"""Runs the fixed workloads of tests/test_gpu_engine_configs.py in a fresh process, so that the engine switches (GPK_*
environment variables, read once per process) take effect.  Usage: python -m tests._engine_worker OUT.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

POTRF_N = [513, 1000, 2048, 4096]
EXTRA = (1024, 2)          # n, extra rows appended below the square part
GPR_N = 2048
TRSM = (2048, 7)           # n, right-hand sides (against the n = 2048 factor)
GEMM32 = (1000, 900, 1300)  # m, n, k: tf32 tensor-core eligible, several row tiles (clusters of 2 row tiles)


def spd(n, seed):
    rng = np.random.default_rng(seed)
    B = rng.standard_normal((n, n + 16))
    d = np.exp(rng.uniform(-3, 3, n))                # rows of different scale: the per-row digit exponents matter
    return (B @ B.T / n + 0.5 * np.eye(n)) * d[:, None] * d[None, :]


def extra_rows(n, p, seed):
    return np.random.default_rng(seed).standard_normal((p, n))


def gemm32_operands():
    rng = np.random.default_rng(77)
    m, n, k = GEMM32
    return rng.standard_normal((m, k)).astype(np.float32), rng.standard_normal((k, n)).astype(np.float32)


def main(out):
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import _lib, ops
    from oracle import gp_oracle as O

    torch.cuda.set_device(0)
    res = {}
    lib = _lib.load()
    for n in POTRF_N:
        A = ops.to_device(spd(n, n))
        ops.potrf(A)
        res[f"potrf{n}"] = np.tril(A.cpu().numpy())
        res[f"slices{n}"] = np.array(lib.gpk_potrf_last_slices())
        if n == TRSM[0]:
            L = A
    n, p = EXTRA
    A = np.concatenate([np.tril(spd(n, n + 1)), extra_rows(n, p, 5)])
    Ad = ops.to_device(A)
    ops.potrf(Ad, n)
    res["extra"] = Ad.cpu().numpy()
    res["extra"][:n] = np.tril(res["extra"][:n])   # (the strict upper triangle of the square part is scratch)
    B = np.random.default_rng(3).standard_normal(TRSM)
    res["trsm"] = ops.trsm(L, ops.to_device(B)).cpu().numpy()
    d = O.make_data(2, GPR_N, 8, 1)
    m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.Matern52(lengthscales=np.sqrt(8.0)), noise_variance=0.1)
    res["lml"] = np.array(float(m.log_marginal_likelihood()))
    res["lml_slices"] = np.array(lib.gpk_potrf_last_slices())
    with gpf.config.as_context(gpf.config.Config(float=np.float32)):
        A32 = ops.to_device(spd(1000, 1000).astype(np.float32))
        ops.potrf(A32)
        res["potrf32"] = np.tril(A32.cpu().numpy())
        Ag, Bg = gemm32_operands()
        res["gemm32"] = ops.gemm(ops.to_device(Ag), ops.to_device(Bg)).cpu().numpy()
    torch.cuda.synchronize()
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
