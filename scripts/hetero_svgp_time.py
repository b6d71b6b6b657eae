"""Time SVGP training through HeteroskedasticTFPConditional against the same model with a Gaussian likelihood, and the
heteroskedastic likelihood's operators alone.

    python scripts/hetero_svgp_time.py [--reps 20] [--warmup 3]

SVGP: SeparateIndependent of two SquaredExponential ARD latents (L = 2) with separate Z, D = 4, float64, whiten=True,
dense q_sqrt.  For B in {1e3, 1e4, 1e5} and M in {20, 256} the script times one elbo_and_grad
(gpk_svgp_mo_elbo_grad) with the heteroskedastic likelihood (Y [B, 1]) and with Gaussian(0.2) on P = 2 independent
outputs (Y [B, 2]): the difference is the likelihood's share of a training step.  Operators at B = 1e6 rows of two
latents: variational_expectations (the 20-node sum), predict_mean_and_var, predict_log_density (400 nodes) and the
adjoints of the variational expectations (gpk_lik_varexp_grad).  ms per call are CUDA-event times over `reps` calls
after `warmup` calls.  The card name, power limit and maximum SM clock are read in the same run and printed in the one
JSON line.  Needs a CUDA device; there is no CPU fallback."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.mo_svgp_time import card, time_ms  # noqa: E402


def svgp(B, M, reps, warmup):
    import numpy as np
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import ops

    K, IV, LIK = gpf.kernels, gpf.inducing_variables, gpf.likelihoods
    D = 4
    rng = np.random.default_rng(B + M)
    Xh = rng.standard_normal((B, D))
    X = ops.to_device(Xh)
    Y1 = ops.to_device(np.sin(Xh[:, :1]) + rng.standard_normal((B, 1)) * np.exp(0.5 * np.cos(Xh[:, 1:2])))
    Y2 = ops.to_device(np.sin(Xh[:, :2]) + 0.3 * rng.standard_normal((B, 2)))
    Zs = [1.5 * rng.standard_normal((M, D)) for _ in range(2)]
    q_mu = 0.3 * rng.standard_normal((M, 2))
    q_sqrt = np.stack([np.tril(0.05 * rng.standard_normal((M, M)), -1) + np.eye(M) for _ in range(2)])

    def model(lik):
        return gpf.models.SVGP(K.SeparateIndependent([K.SquaredExponential(lengthscales=np.full(D, 2.0))
                                                      for _ in range(2)]), lik,
                               IV.SeparateIndependentInducingVariables([IV.InducingPoints(z.copy()) for z in Zs]),
                               num_latent_gps=2, q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), num_data=10 * B)

    het, gauss = model(LIK.HeteroskedasticTFPConditional()), model(LIK.Gaussian(0.2))
    t_het = time_ms(torch, lambda: het.elbo_and_grad((X, Y1), device_arrays=True), reps, warmup)
    t_gauss = time_ms(torch, lambda: gauss.elbo_and_grad((X, Y2), device_arrays=True), reps, warmup)
    return {"B": B, "M": M, "hetero_ms": round(t_het, 3), "gaussian_ms": round(t_gauss, 3),
            "ratio": round(t_het / t_gauss, 3)}


def operators(N, reps, warmup):
    import numpy as np
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import ops

    rng = np.random.default_rng(1)
    mu = ops.to_device(np.c_[rng.standard_normal(N), 0.5 * rng.standard_normal(N)])
    var = ops.to_device(0.1 + rng.random((N, 2)))
    Y = ops.to_device(rng.standard_normal((N, 1)))
    lik = gpf.likelihoods.HeteroskedasticTFPConditional()
    desc = lik._lik_desc()
    res = {"N": N}
    for name, f in [("varexp_ms", lambda: ops.lik_varexp_sum(desc, mu, var, Y)),
                    ("varexp_grad_ms", lambda: ops.lik_varexp_grad(desc, mu, var, Y)),
                    ("predict_mean_and_var_ms", lambda: ops.lik_predict_mean_and_var(desc, mu, var)),
                    ("predict_log_density_ms", lambda: ops.lik_predict_log_density(desc, mu, var, Y))]:
        res[name] = round(time_ms(torch, f, reps, warmup), 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "hetero_svgp_time.py needs a CUDA device"
    res = {"card": card(),
           "svgp": [svgp(B, M, args.reps, args.warmup) for B in (1000, 10000, 100000) for M in (20, 256)],
           "operators": operators(1000000, args.reps, args.warmup)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
