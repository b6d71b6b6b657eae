"""Oracle of the scalar likelihoods (test infrastructure, like tests/svgp_grad_oracle.py; not imported by the product):
the targets of csrc/lik.cu, and the likelihoods tests/svgp_grad_oracle.py takes.

The likelihoods restate gpflow/likelihoods/scalar_discrete.py:29-117 (Bernoulli with utils.py::inv_probit, Poisson with
the exp link), scalar_continuous.py:177-213 (StudentT) and logdensities.py:49-102; the quadrature is base.py:279-456 with
NDiagGHQuadrature of 20 points (quadrature/gauss_hermite.py): E[g] ~ sum_k w_k g(mu + sqrt(v) z_k), z = sqrt(2) hermgauss
nodes, w = weights / sqrt(pi), log-space logsumexp_k(log w_k + g).  Every element (n, p) is one scalar likelihood.

Each `ve_grads` returns the exact derivatives of its variational expectations (of the 20-point sum for the quadrature
likelihoods, which is what autodiff of the reference gives).  Pinned by finite differences in
tests/test_oracle_likelihoods.py.
"""
from __future__ import annotations

import os
import re
from typing import Tuple

import numpy as np
from scipy.special import erf, gammaln, logsumexp

from oracle import gp_oracle as O

N_GH = 20
JITTER_PROBIT = 1e-3


def gh_points_and_weights(n_gh: int = N_GH) -> Tuple[np.ndarray, np.ndarray]:
    """gauss_hermite.py:30-46."""
    z, dz = np.polynomial.hermite.hermgauss(n_gh)
    return z * np.sqrt(2), dz / np.sqrt(np.pi)


def cuda_gh_table() -> Tuple[np.ndarray, np.ndarray]:
    """The nodes and weights committed as literals in csrc/lik.cu (GH_Z, GH_W)."""
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpflow_b200", "csrc", "lik.cu")
    text = open(src).read()

    def table(name):
        body = re.search(name + r"\[GH_N\]\s*=\s*\{([^}]*)\}", text).group(1)
        return np.array([float(v) for v in body.replace("\n", " ").split(",") if v.strip()])

    return table("GH_Z"), table("GH_W")


def inv_probit(x):
    """utils.py::inv_probit."""
    return 0.5 * (1.0 + erf(x / np.sqrt(2.0))) * (1 - 2 * JITTER_PROBIT) + JITTER_PROBIT


class Lik:
    """One scalar likelihood: log p(y | f) and its derivatives, elementwise."""
    name = ""
    closed_ve = False

    def logp(self, y, f):
        raise NotImplementedError

    def dlogp(self, y, f):
        """(d/df, d/d(likelihood parameter)) of log p(y | f)."""
        raise NotImplementedError

    def conditional_mean(self, f):
        raise NotImplementedError

    def conditional_variance(self, f):
        raise NotImplementedError

    # ---- base.py:344-400: quadrature ----
    def quad_ve(self, mu, v, y):
        z, w = gh_points_and_weights()
        F = mu[None] + np.sqrt(v)[None] * z[:, None, None]
        return np.sum(w[:, None, None] * self.logp(y[None], F), 0)

    def quad_ve_grads(self, mu, v, y):
        z, w = gh_points_and_weights()
        sd = np.sqrt(v)
        F = mu[None] + sd[None] * z[:, None, None]
        g1, gp = self.dlogp(y[None], F)
        W = w[:, None, None]
        dmu = np.sum(W * g1, 0)
        dv = np.sum(W * g1 * z[:, None, None], 0) / (2.0 * sd)
        return dmu, dv, np.sum(W * gp, 0)

    def quad_log_density(self, mu, v, y):
        z, w = gh_points_and_weights()
        F = mu[None] + np.sqrt(v)[None] * z[:, None, None]
        return np.sum(logsumexp(self.logp(y[None], F) + np.log(w)[:, None, None], axis=0), -1)

    def quad_mean_and_var(self, mu, v):
        z, w = gh_points_and_weights()
        F = mu[None] + np.sqrt(v)[None] * z[:, None, None]
        W = w[:, None, None]
        cm = self.conditional_mean(F)
        ey = np.sum(W * cm, 0)
        ey2 = np.sum(W * (self.conditional_variance(F) + cm ** 2), 0)
        return ey, ey2 - ey ** 2

    # ---- the public forms (closed where the reference has them) ----
    def variational_expectations(self, mu, v, y):
        """Per element [N, P] (the reference sums over P; the device sums over everything)."""
        return self.quad_ve(mu, v, y)

    def ve_grads(self, mu, v, y):
        return self.quad_ve_grads(mu, v, y)

    def predict_log_density(self, mu, v, y):
        return self.quad_log_density(mu, v, y)

    def predict_mean_and_var(self, mu, v):
        return self.quad_mean_and_var(mu, v)


class Gaussian(Lik):
    name = "gaussian"
    closed_ve = True

    def __init__(self, variance=1.0):
        self.variance = float(variance)

    def logp(self, y, f):
        return -0.5 * O.LOG2PI - 0.5 * np.log(self.variance) - 0.5 * (y - f) ** 2 / self.variance

    def dlogp(self, y, f):
        s = self.variance
        return (y - f) / s, -0.5 / s + 0.5 * (y - f) ** 2 / (s * s)

    def conditional_mean(self, f):
        return f

    def conditional_variance(self, f):
        return np.full_like(f, self.variance)

    def variational_expectations(self, mu, v, y):
        s = self.variance
        return -0.5 * O.LOG2PI - 0.5 * np.log(s) - 0.5 * ((y - mu) ** 2 + v) / s

    def ve_grads(self, mu, v, y):
        s = self.variance
        return (y - mu) / s, np.full_like(v, -0.5 / s), -0.5 / s + 0.5 * ((y - mu) ** 2 + v) / (s * s)

    def predict_log_density(self, mu, v, y):
        return O.gaussian_predict_log_density(mu, v, y, self.variance)

    def predict_mean_and_var(self, mu, v):
        return mu, v + self.variance


class Bernoulli(Lik):
    name = "bernoulli"

    def logp(self, y, f):
        p = inv_probit(f)
        return np.log(np.where(y == 1, p, 1 - p))

    def dlogp(self, y, f):
        p = inv_probit(f)
        dp = (1 - 2 * JITTER_PROBIT) * np.exp(-0.5 * f * f) / np.sqrt(2 * np.pi)
        return np.where(y == 1, dp / p, -dp / (1 - p)), np.zeros_like(f)

    def conditional_mean(self, f):
        return inv_probit(f)

    def conditional_variance(self, f):
        p = inv_probit(f)
        return p - p ** 2

    def predict_mean_and_var(self, mu, v):  # scalar_discrete.py:93-101
        p = inv_probit(mu / np.sqrt(1 + v))
        return p, p - p ** 2

    def predict_log_density(self, mu, v, y):  # :103-108
        p = self.predict_mean_and_var(mu, v)[0]
        return np.sum(np.log(np.where(y == 1, p, 1 - p)), -1)


class Poisson(Lik):
    name = "poisson"
    closed_ve = True

    def __init__(self, binsize=1.0):
        self.binsize = float(binsize)

    def logp(self, y, f):  # logdensities.py:58-59 with lam = exp(f) binsize
        lam = np.exp(f) * self.binsize
        return y * np.log(lam) - lam - gammaln(y + 1.0)

    def dlogp(self, y, f):
        return y - np.exp(f) * self.binsize, np.zeros_like(f)

    def conditional_mean(self, f):
        return np.exp(f) * self.binsize

    def conditional_variance(self, f):
        return np.exp(f) * self.binsize

    def variational_expectations(self, mu, v, y):  # scalar_discrete.py:67-78
        b = self.binsize
        return y * mu - np.exp(mu + v / 2) * b - gammaln(y + 1) + y * np.log(b)

    def ve_grads(self, mu, v, y):
        e = np.exp(mu + v / 2) * self.binsize
        return y - e, -0.5 * e, np.zeros_like(mu)


class StudentT(Lik):
    name = "student_t"

    def __init__(self, scale=1.0, df=3.0):
        self.scale, self.df = float(scale), float(df)

    def logp(self, y, f):  # logdensities.py:93-102
        df, sc = self.df, self.scale
        const = gammaln((df + 1.0) * 0.5) - gammaln(df * 0.5) - 0.5 * (np.log(sc ** 2) + np.log(df) + np.log(np.pi))
        return const - 0.5 * (df + 1.0) * np.log(1.0 + (1.0 / df) * ((y - f) / sc) ** 2)

    def dlogp(self, y, f):
        df, sc = self.df, self.scale
        r = y - f
        q = sc * sc * df + r * r
        return (df + 1.0) * r / q, -1.0 / sc + (df + 1.0) * r * r / (sc * q)

    def conditional_mean(self, f):
        return f

    def conditional_variance(self, f):
        return np.full_like(f, self.scale ** 2 * (self.df / (self.df - 2.0)))


def make(name: str, **kw) -> Lik:
    return {"gaussian": Gaussian, "bernoulli": Bernoulli, "poisson": Poisson, "student_t": StudentT}[name](**kw)


def targets(name: str, F: np.ndarray, rng: np.random.Generator) -> np.ndarray:
    """Observations of the likelihood `name` around the latent values F."""
    if name == "bernoulli":
        return (F + 0.3 * rng.standard_normal(F.shape) > 0).astype(np.float64)
    if name == "poisson":
        return rng.poisson(np.exp(np.clip(F, -3, 2))).astype(np.float64)
    return F + 0.3 * rng.standard_t(3.0, F.shape)

