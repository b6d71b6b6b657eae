"""Time the Bayesian GPLVM bound and its gradient on the device.

    python scripts/bgplvm_time.py [--reps 20] [--warmup 3] [--out DIR]

Four shapes: an oil-flow-like case (N = 1000, Q = 10, M = 32, P = 12), a GPU-sized case (N = 16384, Q = 8, M = 256,
P = 32), and two wide latent spaces (N = 4096, M = 128, P = 16 at Q = 16 and Q = 32, the kernels' other two
instantiations), RBF with ARD lengthscales.  Per shape: BayesianGPLVM.elbo() and elbo_and_grad() in ms per call (CUDA events
over `reps` calls after `warmup`), SGPR.elbo_and_grad at the same N, M, P with X = the latent means for comparison, and
in a torch.profiler run of its own the device time of the psi2 forward (psi2_pair_kernel<.., false>) and of the psi2
adjoint (psi2_pair_kernel<.., true> + psi2_point_kernel).  Pair elements per second count N M (M + 1) / 2 per kernel;
FLOP/s count 3 Q' + 12 fp64 operations per forward element (the exponent and the table exp) and 2 (3 Q' + 12) + 6 Q'
per adjoint element (both adjoint kernels recompute the exponent and exp; 3 Q' accumulations each).  The card name
and power limit are read in the same run.  Needs a CUDA device; there is no CPU fallback."""
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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import gpflow_b200 as gpf

    assert torch.cuda.is_available(), "bgplvm_time.py needs a CUDA device"
    res = {"card": card()}
    print("card:", res["card"])
    for (N, Q, M, P) in [(1000, 10, 32, 12), (16384, 8, 256, 32), (4096, 16, 128, 16), (4096, 32, 128, 16)]:
        rng = np.random.default_rng(0)
        Y = rng.standard_normal((N, P))
        mu = rng.standard_normal((N, Q))
        S = rng.uniform(0.05, 0.5, (N, Q))
        Z = rng.standard_normal((M, Q))
        ls = np.linspace(1.0, 3.0, Q)
        m = gpf.models.BayesianGPLVM(Y, mu, S, gpf.kernels.SquaredExponential(lengthscales=ls), inducing_variable=Z)
        s = gpf.models.SGPR((mu, Y), gpf.kernels.SquaredExponential(lengthscales=ls), Z)
        r = {"N": N, "Q": Q, "M": M, "P": P}
        r["elbo_ms"] = time_ms(torch, lambda: m.elbo(), args.reps, args.warmup)
        r["elbo_and_grad_ms"] = time_ms(torch, lambda: m.elbo_and_grad(device_arrays=True), args.reps, args.warmup)
        r["sgpr_elbo_and_grad_ms"] = time_ms(torch, lambda: s.elbo_and_grad(device_arrays=True), args.reps,
                                             args.warmup)
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                m.elbo_and_grad(device_arrays=True)
            torch.cuda.synchronize()
        fwd = bwd = 0.0
        for e in prof.key_averages():
            t = e.device_time_total / 1e3 / args.reps  # ms per call
            if "psi2_pair_kernel" in e.key and "false" in e.key:
                fwd += t
            elif "psi2_pair_kernel" in e.key or "psi2_point_kernel" in e.key:
                bwd += t
        pairs = N * M * (M + 1) / 2
        r["psi2_fwd_ms"], r["psi2_bwd_ms"] = fwd, bwd
        r["pair_elements"] = pairs
        r["psi2_fwd_pairs_per_s"] = pairs / (fwd * 1e-3) if fwd else None
        r["psi2_fwd_fp64_flops"] = pairs * (3 * Q + 12) / (fwd * 1e-3) if fwd else None
        r["psi2_bwd_fp64_flops"] = pairs * (2 * (3 * Q + 12) + 6 * Q) / (bwd * 1e-3) if bwd else None
        print(json.dumps(r))
        res[f"N{N}_M{M}"] = r
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bgplvm_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
