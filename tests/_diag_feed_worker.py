"""Runs the factorisations of tests/test_gpu_diag_feed.py in a fresh process, so that GPK_DIAG_FEED_MAX_K and
GPK_FP64_ENGINE (read once per process) take effect.  Usage: python -m tests._diag_feed_worker OUT.npz"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EXTRA = [(1000, 3), (4096, 3)]  # n, extra rows appended below the square part
C2_N, C2_NOISE = 8192, 0.1


def spd(n, seed):
    rng = np.random.default_rng(seed)
    B = rng.standard_normal((n, n + 16))
    d = np.exp(rng.uniform(-3, 3, n))                # rows of different scale: the per-row digit exponents matter
    return (B @ B.T / n + 0.5 * np.eye(n)) * d[:, None] * d[None, :]


def extra_input(n, p):
    """The lower triangle of an SPD matrix with p rows below it (the (Y - m)^T rows a GPR factorisation carries)."""
    return np.concatenate([np.tril(spd(n, n + 7)), np.random.default_rng(n).standard_normal((p, n))])


def c2_input():
    """bench.py's C2 matrix: Matern52 (lengthscale sqrt(8)) on its N = 8192, D = 8 inputs plus noise, with Y^T below."""
    from oracle import gp_oracle as O

    d = O.make_data(2, C2_N, 8, 1)
    Xs = d["X"] / np.sqrt(8.0)
    sq = (Xs * Xs).sum(axis=1)
    r = np.sqrt(np.maximum(sq[:, None] + sq[None, :] - 2.0 * (Xs @ Xs.T), 1e-36))
    K = (1.0 + np.sqrt(5.0) * r + (5.0 / 3.0) * r * r) * np.exp(-np.sqrt(5.0) * r)
    K[np.diag_indices(C2_N)] = 1.0 + C2_NOISE
    return np.concatenate([np.tril(K), d["Y"].T]), d


def factor(A, n):
    from gpflow_b200 import ops

    Ad = ops.to_device(A)
    ops.potrf(Ad, n)
    L = Ad.cpu().numpy()
    L[:n] = np.tril(L[:n])  # (the strict upper triangle of the square part is scratch)
    return L


def main(out):
    import torch

    import gpflow_b200 as gpf

    torch.cuda.set_device(0)
    res = {}
    for n, p in EXTRA:
        res[f"extra{n}"] = factor(extra_input(n, p), n)
    A, d = c2_input()
    L = factor(A, C2_N)
    res["c2"] = L
    res["c2_again_sha"] = np.array(hashlib.sha256(factor(A, C2_N).tobytes()).hexdigest())
    res["c2_sha"] = np.array(hashlib.sha256(L.tobytes()).hexdigest())
    m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.Matern52(lengthscales=np.sqrt(8.0)), noise_variance=C2_NOISE)
    res["c2_lml"] = np.array(float(m.log_marginal_likelihood()))
    torch.cuda.synchronize()
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
