"""Oracle of the scalar likelihoods and of the SVGP ELBO gradient through them (test infrastructure, like
tests/svgp_grad_oracle.py; not imported by the product): the targets of csrc/lik.cu and gpk_svgp_elbo_grad.

The likelihoods restate gpflow/likelihoods/scalar_discrete.py:29-117 (Bernoulli with utils.py::inv_probit, Poisson with
the exp link), scalar_continuous.py:177-213 (StudentT) and logdensities.py:49-102; the quadrature is base.py:279-456 with
NDiagGHQuadrature of 20 points (quadrature/gauss_hermite.py): E[g] ~ sum_k w_k g(mu + sqrt(v) z_k), z = sqrt(2) hermgauss
nodes, w = weights / sqrt(pi), log-space logsumexp_k(log w_k + g).  Every element (n, p) is one scalar likelihood.

The ELBO gradient is tests/svgp_grad_oracle.py's with the constant fvar adjoint w = -c/(2s) replaced by per-element
weights.  With c = num_data / B, R[n,p] = c dVE/dfmean and W[n,p] = c dVE/dfvar (the exact derivatives of the
20-point sum for the quadrature likelihoods, which is what autodiff of the reference gives):
  whiten:     Abar = m R^T + 2 sum_p (S_p S_p^T - I) A diag(W_p),   dF/dKuf = L^-T Abar,
              dF/dKuu = -sym(L^-T Phi(Abar A^T) L^-1),   dF/dS_p = tril(2 (A diag(W_p) A^T) S_p - S_p) + diag(1 / diag S_p)
  otherwise:  Abar = m R^T + 2 sum_p S_p S_p^T A diag(W_p),   dF/dKuf = K^-1 Abar - 2 A diag(sum_p W_p),
              dF/dKuu = sym(-K^-1 Abar A^T) + A diag(sum_p W_p) A^T + 1/2 K^-1 (m m^T + Sig) K^-1 - P/2 K^-1,
              dF/dS_p = tril(2 (A diag(W_p) A^T) S_p - K^-1 S_p) + diag(1 / diag S_p)
  both:       dF/dq_mu = A R - m (whiten) or A R - K^-1 m,   dF/dKdiag[n] = sum_p W[n,p],   dF/dm(X) = R.
Pinned by central finite differences of svgp_elbo_lik in tests/test_oracle_likelihoods.py.
"""
from __future__ import annotations

import os
import re
from typing import Dict, Tuple

import numpy as np
from scipy.special import erf, gammaln, logsumexp

from oracle import gp_oracle as O
from tests.svgp_grad_oracle import _phi, _sym, kernel_and_z_grads

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


# ---- SVGP ------------------------------------------------------------------------------------------------------
def svgp_elbo_lik(X, Y, Z, kernel, q_mu, q_sqrt, lik: Lik, *, whiten=True, num_data=None, mean_function=None,
                  jitter=O.DEFAULT_JITTER) -> float:
    """svgp.py:166-181 with the likelihood `lik`."""
    kl = O.prior_kl(Z, kernel, q_mu, q_sqrt, whiten=whiten, jitter=jitter)
    f_mean, f_var = O.svgp_predict_f(X, Z, kernel, q_mu, q_sqrt, whiten=whiten, full_cov=False,
                                     mean_function=mean_function, jitter=jitter)
    scale = 1.0 if num_data is None else float(num_data) / X.shape[0]
    return float(np.sum(lik.variational_expectations(f_mean, f_var, Y)) * scale - kl)


def svgp_elbo_lik_and_grad(X, Y, kernel, Z, q_mu, q_sqrt, lik: Lik, *, whiten=True, num_data=None,
                           mean_function=None, jitter=O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The ELBO of svgp_elbo_lik and its gradient: {"leaves", "lik" (d/d Gaussian variance or Student-t scale, else 0),
    "mean", "Z", "q_mu", "q_sqrt"} as tests/svgp_grad_oracle.py::svgp_elbo_and_grad_expr."""
    B, P = Y.shape
    M, D = Z.shape
    q_diag = q_sqrt.ndim == 2
    c = 1.0 if num_data is None else float(num_data) / B
    K = O.Kuu(Z, kernel, jitter=jitter)
    L = O.cholesky(K)
    Kuf = O.Kuf(Z, kernel, X)
    Linv = O.tri_solve(L, np.eye(M))
    Kinv = Linv.T @ Linv
    S = np.stack([np.diag(q_sqrt[:, p]) for p in range(P)]) if q_diag else np.tril(q_sqrt)
    Sig = sum(S[p] @ S[p].T for p in range(P))
    A = Linv @ Kuf if whiten else Kinv @ Kuf
    f_mean, f_var = O.svgp_predict_f(X, Z, kernel, q_mu, q_sqrt, whiten=whiten, mean_function=mean_function,
                                     jitter=jitter)
    dmu, dv, dpar = lik.ve_grads(f_mean, f_var, Y)
    R, W = c * dmu, c * dv
    Wsum = W.sum(1)
    I = np.eye(M)
    G = [A @ np.diag(W[:, p]) @ A.T for p in range(P)]
    if whiten:
        Abar = q_mu @ R.T + 2.0 * sum((S[p] @ S[p].T - I) @ A @ np.diag(W[:, p]) for p in range(P))
        Guf = Linv.T @ Abar
        Guu = -_sym(Linv.T @ _phi(Abar @ A.T) @ Linv)
        dq_mu = A @ R - q_mu
        KS = S
    else:
        Abar = q_mu @ R.T + 2.0 * sum(S[p] @ S[p].T @ A @ np.diag(W[:, p]) for p in range(P))
        Guf = Kinv @ Abar - 2.0 * A @ np.diag(Wsum)
        Guu = (_sym(-Kinv @ Abar @ A.T) + A @ np.diag(Wsum) @ A.T + 0.5 * Kinv @ (q_mu @ q_mu.T + Sig) @ Kinv
               - 0.5 * P * Kinv)
        dq_mu = A @ R - Kinv @ q_mu
        KS = np.stack([Kinv @ S[p] for p in range(P)])
    if q_diag:
        kd = np.ones(M) if whiten else np.diag(Kinv)
        dq_sqrt = np.stack([2.0 * q_sqrt[:, p] * np.diag(G[p]) for p in range(P)], 1) - kd[:, None] * q_sqrt \
            + 1.0 / q_sqrt
    else:
        dq_sqrt = np.stack([np.tril(2.0 * G[p] @ S[p] - KS[p]) + np.diag(1.0 / np.diag(S[p])) for p in range(P)])
    per_leaf, dZ = kernel_and_z_grads(kernel, X, Z, Guu, Guf, Wsum)
    dm = R
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = dm.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = dm.sum(0)
        rhs = dm.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else dm
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    elbo = svgp_elbo_lik(X, Y, Z, kernel, q_mu, q_sqrt, lik, whiten=whiten, num_data=num_data,
                         mean_function=mean_function, jitter=jitter)
    return elbo, {"leaves": per_leaf, "lik": float(c * np.sum(dpar)), "mean": mean, "Z": dZ, "q_mu": dq_mu,
                  "q_sqrt": dq_sqrt}
