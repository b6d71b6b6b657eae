"""Time SVGP.elbo_and_grad for a multi-output kernel against the single-output calls that do the same per-latent work.

    python scripts/mo_svgp_time.py [--reps 20] [--warmup 3]

Workload: LinearCoregionalization of L latents (SquaredExponential ARD, Matern32, Matern52, RBF + Linear, repeated for
L > 4) mixed into P outputs, separate Z per latent, float64, Gaussian likelihood, whiten=True, dense q_sqrt.  For each
configuration the script times one multi-output elbo_and_grad (gpk_svgp_mo_elbo_grad) and the sum of L single-output
elbo_and_grad calls with P = 1 at the same B, M and D (latent l's kernel and Z): that sum is the floor of a design that
runs each latent's work in its own launches.  Configurations: L = 4, P = 8, M = 512, B = 2048, D = 8, and the
launch-bound L = 8, P = 8, M = 64, B = 1024, D = 8.  ms per call are CUDA-event times over `reps` calls after `warmup`
calls (each call ends in its one host read).  The card name, power limit and maximum SM clock are read in the same run
and printed in the one JSON line.  Needs a CUDA device; there is no CPU fallback."""
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


def configuration(L, P, M, B, D, reps, warmup):
    import numpy as np
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import ops

    K, IV = gpf.kernels, gpf.inducing_variables
    rng = np.random.default_rng(L * 1000 + M)

    def latent_kernel(l):
        return [lambda: K.SquaredExponential(lengthscales=np.full(D, 2.5)), lambda: K.Matern32(lengthscales=3.0),
                lambda: K.Matern52(lengthscales=2.8),
                lambda: K.SquaredExponential(lengthscales=2.5) + K.Linear(variance=0.1)][l % 4]()

    X = ops.to_device(rng.standard_normal((B, D)))
    Y = ops.to_device(np.sin(rng.standard_normal((B, 1)) @ np.ones((1, P))) + 0.1 * rng.standard_normal((B, P)))
    Zs = [1.5 * rng.standard_normal((M, D)) for _ in range(L)]
    q_mu = 0.3 * rng.standard_normal((M, L))
    q_sqrt = np.stack([np.tril(0.05 * rng.standard_normal((M, M)), -1) + np.eye(M) for _ in range(L)])
    mo = gpf.models.SVGP(K.LinearCoregionalization([latent_kernel(l) for l in range(L)], 0.5 * rng.standard_normal(
        (P, L))), gpf.likelihoods.Gaussian(0.2), IV.SeparateIndependentInducingVariables(
        [IV.InducingPoints(z) for z in Zs]), q_mu=q_mu, q_sqrt=q_sqrt, num_data=100 * B, whiten=True)
    singles = [gpf.models.SVGP(latent_kernel(l), gpf.likelihoods.Gaussian(0.2), Zs[l].copy(), num_latent_gps=1,
                               q_mu=q_mu[:, l:l + 1].copy(), q_sqrt=q_sqrt[l:l + 1].copy(), num_data=100 * B)
               for l in range(L)]
    Y1 = Y[:, :1].contiguous()
    t_mo = time_ms(torch, lambda: mo.elbo_and_grad((X, Y), device_arrays=True), reps, warmup)

    def run_singles():
        for s in singles:
            s.elbo_and_grad((X, Y1), device_arrays=True)

    t_so = time_ms(torch, run_singles, reps, warmup)
    return {"L": L, "P": P, "M": M, "B": B, "D": D, "mo_ms": round(t_mo, 3), "single_sum_ms": round(t_so, 3),
            "ratio": round(t_mo / t_so, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "mo_svgp_time.py needs a CUDA device"
    res = {"card": card(), "configs": [configuration(4, 8, 512, 2048, 8, args.reps, args.warmup),
                                       configuration(8, 8, 64, 1024, 8, args.reps, args.warmup)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
