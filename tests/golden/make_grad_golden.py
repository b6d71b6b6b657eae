"""Generates tests/golden/grad_golden.npz: loss and gradients of `training_loss_and_gradients` (the optimiser contract,
one gradient per trainable parameter in `trainable_parameters` order) of every model with a device gradient, on small
seeded cases.  tests/test_gpu_grad_golden.py checks that the device gradients keep reproducing them.  Needs a GPU.

    python tests/golden/make_grad_golden.py [output.npz]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import gpflow_b200 as gpf  # noqa: E402
from oracle import gp_oracle as O  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
K = gpf.kernels
LIK = gpf.likelihoods
MF = gpf.mean_functions


def _expr(D):
    s = float(np.sqrt(D))
    return ((K.SquaredExponential(variance=1.1, lengthscales=s) + K.Matern32(variance=1.0, lengthscales=2 * s))
            * K.Linear(variance=0.5))


def _linear(D, P, seed):
    rng = np.random.default_rng(seed)
    return MF.Linear(0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1))


def _q(M, P, q_diag, seed):
    rng = np.random.default_rng(seed)
    q_mu = 0.3 * rng.standard_normal((M, P))
    if q_diag:
        return q_mu, 0.5 + rng.random((M, P))
    return q_mu, np.stack([np.tril(0.1 * rng.standard_normal((M, M))) + np.eye(M) for _ in range(P)])


def _targets(lik, Y, seed):
    rng = np.random.default_rng(seed)
    if lik == "bernoulli":
        return (Y + 0.3 * rng.standard_normal(Y.shape) > 0).astype(np.float64)
    return Y + 0.3 * rng.standard_t(3.0, Y.shape)        # student_t


def cases():
    """{name: (model, args of training_loss_and_gradients)}."""
    out = {}
    d = O.make_data(11, 300, 3, 2)
    out["gpr"] = (gpf.models.GPR((d["X"], d["Y"]), _expr(3), mean_function=_linear(3, 2, 1), noise_variance=0.1), ())
    d = O.make_data(12, 500, 4, 1, M=64)
    out["sgpr"] = (gpf.models.SGPR((d["X"], d["Y"]), _expr(4), d["Z"], mean_function=_linear(4, 1, 2),
                                   noise_variance=0.2), ())
    for lik in ("gaussian", "student_t", "bernoulli"):
        P = 1 if lik == "bernoulli" else 2
        d = O.make_data(13, 400, 4, P, M=40)
        Y = d["Y"] if lik == "gaussian" else _targets(lik, d["Y"], 3)
        settings = [(True, False)] if lik == "bernoulli" else [(w, q) for w in (True, False) for q in (False, True)]
        for whiten, q_diag in settings:
            q_mu, q_sqrt = _q(40, P, q_diag, 4)
            if lik == "gaussian":
                likelihood, mean = LIK.Gaussian(0.15), _linear(4, P, 5)
            elif lik == "student_t":
                likelihood, mean = LIK.StudentT(scale=0.7, df=4.0), MF.Constant(np.array([0.3]))
            else:
                likelihood, mean = LIK.Bernoulli(), None
            m = gpf.models.SVGP(_expr(4), likelihood, d["Z"].copy(), mean_function=mean, num_latent_gps=P,
                                q_mu=q_mu, q_sqrt=q_sqrt, q_diag=q_diag, whiten=whiten, num_data=5000)
            out[f"svgp_{lik}_w{int(whiten)}_d{int(q_diag)}"] = (m, ((d["X"], Y),))
    d = O.make_data(14, 200, 3, 2)
    m = gpf.models.VGP((d["X"], d["Y"]), _expr(3), LIK.Gaussian(0.1), mean_function=_linear(3, 2, 6))
    q_mu, q_sqrt = _q(200, 2, False, 7)
    m.q_mu.assign(q_mu)
    m.q_sqrt.assign(q_sqrt)
    out["vgp"] = (m, ())
    return out


def record():
    res = {}
    for name, (m, args) in cases().items():
        loss, grads = m.training_loss_and_gradients(*args)
        res[f"{name}/loss"] = np.asarray(loss, dtype=np.float64)
        for i, g in enumerate(grads):
            res[f"{name}/g{i}"] = np.asarray(g, dtype=np.float64)
    return res


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "grad_golden.npz")
    res = record()
    np.savez_compressed(path, **res)
    print({k: np.shape(v) for k, v in res.items()})
