"""Time the matrix-free kernel product and the CGLB bound on the device.

    python scripts/cglb_time.py [--reps 5] [--warmup 1] [--out DIR]

1. gpk_kmv ((K(X, X) + s I) V, nothing stored) against gpk_kbuild's fast path (K(X, X) written in full) at N = 16384 and
   32768, D = 8, RBF and Matern52, P = 1 and 4: ms per call and evaluated elements (N^2) per second.
2. CGLB.elbo() at N = 32768, M = 1024, D = 8 with max_cg_iters = 0 and = 10 (ten CG steps: the difference / 10 is the
   time per CG iteration; minus one product at P = 1 it is the preconditioner and the vector updates), and
   elbo_and_grad() with ten steps, next to SGPR.elbo() / elbo_and_grad() and GPR.log_marginal_likelihood() /
   log_marginal_likelihood_and_grad() at the same shape.
3. CGLB.elbo() and elbo_and_grad() at N = 2^17 (GPR would need 137 GB for K + s I), max_cg_iters = 10.
The card name and power limit are read in the same run.  Needs a CUDA device; there is no CPU fallback."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def time_ms(torch, f, reps, warmup):
    for _ in range(warmup):
        f()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        f()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import _lib, ops

    assert torch.cuda.is_available(), "cglb_time.py needs a CUDA device"
    lib = _lib.load()
    res = {"card": card()}
    print("card:", res["card"])
    D = 8
    for N in (16384, 32768):
        X = torch.from_numpy(np.random.default_rng(0).standard_normal((N, D))).cuda()
        K = torch.empty((N, N), dtype=torch.float64, device="cuda")
        for name, kern in (("rbf", gpf.kernels.SquaredExponential(lengthscales=2.0)),
                           ("m52", gpf.kernels.Matern52(lengthscales=2.0))):
            desc = gpf.kernels.compile_kernel(kern, D)

            def kb():
                _lib.check(lib.gpk_kbuild(*desc, ops._p(X), N, D, None, N, D, D, ops._p(K), N, _lib.GPK_F64,
                                          0, 0.1, None, ops._stream()), "gpk_kbuild")

            t_kb = time_ms(torch, kb, args.reps, args.warmup)
            for P in (1, 4):
                V = torch.ones((N, P), dtype=torch.float64, device="cuda")
                out = torch.empty((N, P), dtype=torch.float64, device="cuda")
                ws = ops.scratch_bytes(lib.gpk_kmv_ws(N, N, P))

                def kmv():
                    _lib.check(lib.gpk_kmv(*desc, ops._p(X), N, D, None, N, D, D, ops._p(V), P, P, 0.1, ops._p(out),
                                           P, ops._p(ws), ops._stream()), "gpk_kmv")

                t = time_ms(torch, kmv, args.reps, args.warmup)
                r = {"N": N, "kernel": name, "P": P, "kmv_ms": t, "kmv_elements_per_s": N * N / (t * 1e-3),
                     "kbuild_ms": t_kb, "kbuild_elements_per_s": N * N / (t_kb * 1e-3)}
                print(json.dumps(r))
                res[f"kmv_{name}_N{N}_P{P}"] = r
        del K
        torch.cuda.empty_cache()

    def models(N, M, iters):
        rng = np.random.default_rng(1)
        X = rng.standard_normal((N, D))
        Y = np.sin(X[:, :1]) + 0.1 * rng.standard_normal((N, 1))
        Z = X[rng.choice(N, M, replace=False)]
        k = lambda: gpf.kernels.SquaredExponential(lengthscales=2.0)
        m = gpf.models.CGLB((X, Y), kernel=k(), inducing_variable=Z, noise_variance=0.1, max_cg_iters=iters,
                            cg_tolerance=1e-12)
        return X, Y, Z, k, m

    N, M = 32768, 1024
    X, Y, Z, k, m10 = models(N, M, 10)
    m0 = models(N, M, 0)[4]
    r = {"N": N, "M": M}
    # reset v each call so every evaluation runs the same steps from v = 0
    zero = lambda m: m.aux_vec.assign(np.zeros((1, N)))
    r["elbo_0_iters_ms"] = time_ms(torch, lambda: (zero(m0), m0.elbo()), args.reps, args.warmup)
    r["elbo_10_iters_ms"] = time_ms(torch, lambda: (zero(m10), m10.elbo()), args.reps, args.warmup)
    r["cg_iteration_ms"] = (r["elbo_10_iters_ms"] - r["elbo_0_iters_ms"]) / 10
    r["kmv_rbf_P1_ms"] = res[f"kmv_rbf_N{N}_P1"]["kmv_ms"]
    r["cg_iteration_minus_product_ms"] = r["cg_iteration_ms"] - r["kmv_rbf_P1_ms"]
    r["elbo_and_grad_10_iters_ms"] = time_ms(torch, lambda: (zero(m10), m10.elbo_and_grad(device_arrays=True)),
                                             args.reps, args.warmup)
    s = gpf.models.SGPR((X, Y), kernel=k(), inducing_variable=Z, noise_variance=0.1)
    r["sgpr_elbo_ms"] = time_ms(torch, lambda: s.elbo(), args.reps, args.warmup)
    r["sgpr_elbo_and_grad_ms"] = time_ms(torch, lambda: s.elbo_and_grad(device_arrays=True), args.reps, args.warmup)
    g = gpf.models.GPR((X, Y), kernel=k(), noise_variance=0.1)
    r["gpr_lml_ms"] = time_ms(torch, lambda: g.log_marginal_likelihood(), args.reps, args.warmup)
    r["gpr_lml_and_grad_ms"] = time_ms(torch, lambda: g.log_marginal_likelihood_and_grad(), args.reps, args.warmup)
    print(json.dumps(r))
    res["elbo_N32768"] = r
    del g, s
    torch.cuda.empty_cache()
    N = 1 << 17
    m = models(N, M, 10)[4]
    torch.cuda.reset_peak_memory_stats()
    r = {"N": N, "M": M, "elbo_10_iters_ms": time_ms(torch, lambda: (m.aux_vec.assign(np.zeros((1, N))), m.elbo()),
                                                         max(1, args.reps // 2), 1)}
    r["elbo_and_grad_10_iters_ms"] = time_ms(torch, lambda: (m.aux_vec.assign(np.zeros((1, N))),
                                                              m.elbo_and_grad(device_arrays=True)),
                                             max(1, args.reps // 2), 1)
    r["peak_GiB"] = torch.cuda.max_memory_allocated() / 2 ** 30
    print(json.dumps(r))
    res["elbo_N131072"] = r
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cglb_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
