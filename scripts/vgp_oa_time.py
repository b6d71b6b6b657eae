"""Time VGPOpperArchambeau.elbo_and_grad (gpk_vgp_oa_elbo_grad) per evaluation, split by kernel class.

    python scripts/vgp_oa_time.py [--reps 5] [--warmup 2] [--out DIR]

For N in {1024, 4096, 8192} and P in {1, 3} (RBF, D = 8, Bernoulli likelihood): ms per elbo_and_grad call (host wall
clock over `reps` calls; each call ends in its own device->host read), then one more call with the library's per-class
event timing on (gpk_prof_enable), which reports the device milliseconds and launches of each class: 0 K-build and the
square pass, 1 DMMA / SIMT GEMMs (the weighted product included), 2 potrf leaf, 3 skinny GEMM, 4 elementwise and
reductions, 5 int8 tensor-core updates, 6 panel solve.  The card name, power limit and maximum SM clock are read with the
numbers and printed with them.  Needs a CUDA device; there is no CPU fallback."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.grad_time import card  # noqa: E402

CLASSES = ["kbuild_square", "gemm", "leaf", "skinny", "misc", "int8_tc", "panel"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import _lib

    assert torch.cuda.is_available(), "vgp_oa_time.py needs a CUDA device"
    lib = _lib.load()
    res = {"card": card(), "runs": []}
    print("card:", res["card"])
    D = 8
    for N in (1024, 4096, 8192):
        rng = np.random.default_rng(N)
        X = rng.standard_normal((N, D))
        Y = (np.sin(X[:, :1]) + 0.3 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
        for P in (1, 3):
            m = gpf.models.VGPOpperArchambeau((X, np.tile(Y, (1, P))), gpf.kernels.SquaredExponential(lengthscales=2.0),
                                              gpf.likelihoods.Bernoulli())
            m.q_alpha.assign(0.01 * rng.standard_normal((N, P)))
            m.q_lambda.assign(0.5 + rng.random((N, P)))
            for _ in range(args.warmup):
                m.elbo_and_grad()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.reps):
                m.elbo_and_grad()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / args.reps
            n = len(CLASSES)
            cms, cl = (ctypes.c_double * 8)(), (ctypes.c_int64 * 8)()
            lib.gpk_prof_read(cms, cl, 8)  # clear
            lib.gpk_prof_enable(1)
            m.elbo_and_grad()
            lib.gpk_prof_read(cms, cl, 8)
            lib.gpk_prof_enable(0)
            split = {CLASSES[i]: {"ms": round(cms[i], 3), "launches": int(cl[i])} for i in range(n)}
            row = {"N": N, "P": P, "ms_per_elbo_and_grad": round(ms, 3), "classes": split}
            res["runs"].append(row)
            print(json.dumps(row))
            del m
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "vgp_oa_time.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
