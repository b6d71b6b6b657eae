"""Oracle of the MultiClass likelihood with the RobustMax inverse link and of the SVGP ELBO gradient through it (test
infrastructure, like tests/lik_oracle.py; not imported by the product): the targets of the MultiClass kernels of
csrc/lik.cu and of gpk_svgp_elbo_grad with a MULTICLASS descriptor.

prob_is_largest restates gpflow/likelihoods/multiclass.py:120-155 for one row with label y, means mu_c and variances v_c:
  x_k, w_k = hermgauss(20) nodes and weights / sqrt(pi),   s_y = sqrt(max(2 v_y, 1e-10)),   s_c = sqrt(max(v_c, 1e-10)),
  d_ck = (mu_y + x_k s_y - mu_c) / s_c,   cdf_ck = Phi(d_ck) (1 - 2e-6) + 1e-6,   p = sum_k w_k prod_{c != y} cdf_ck;
the labels are truncated to integers, and one outside [0, C) has an all-zero one-hot: mu_y = v_y = 0 and every class in
the product.  VE = p log(1 - eps) + (1 - p) log eps_k1 (eps_k1 = eps / (C - 1)), density(y) = p (1 - eps) + (1 - p) eps_k1.

The adjoints, with kappa = log(1 - eps) - log eps_k1, phi the standard normal density, E_ck = prod_{c' != y, c} cdf_c'k
(a prefix times a suffix product) and g_ck = w_k E_ck (1 - 2e-6) phi(d_ck) / s_c:
  dVE/dmu_c = -kappa sum_k g_ck,   dVE/dv_c = -kappa sum_k g_ck d_ck / (2 s_c) (0 where v_c <= 1e-10)   (c != y)
  dVE/dmu_y = kappa sum_k sum_{c != y} g_ck,   dVE/dv_y = kappa sum_k x_k sum_{c != y} g_ck / s_y (0 where 2 v_y <= 1e-10)
  dVE/deps = -p / (1 - eps) + (1 - p) / eps.
The SVGP ELBO gradient is tests/lik_oracle.py::svgp_elbo_lik_and_grad's with these R = c dVE/dfmean, W = c dVE/dfvar and
one label column.  Pinned by central finite differences in tests/test_oracle_multiclass.py.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np
from scipy.special import erf

from oracle import gp_oracle as O
from tests.svgp_grad_oracle import _phi, _sym, kernel_and_z_grads

N_GH = 20
SQUASH = 1e-6


def gh() -> Tuple[np.ndarray, np.ndarray]:
    """hermgauss(20) as prob_is_largest uses it: the raw nodes, the weights / sqrt(pi)."""
    x, w = np.polynomial.hermite.hermgauss(N_GH)
    return x, w / np.sqrt(np.pi)


class MultiClass:
    def __init__(self, num_classes: int, epsilon: float = 1e-3):
        self.num_classes, self.epsilon = int(num_classes), float(epsilon)

    @property
    def eps_k1(self) -> float:
        return self.epsilon / (self.num_classes - 1.0)

    def _one_hot(self, Y):
        y = np.trunc(np.asarray(Y, dtype=np.float64)[:, 0])
        return (y[:, None] == np.arange(self.num_classes)[None]).astype(np.float64)  # all zero outside [0, C)

    def _parts(self, Y, mu, var):
        oh = self._one_hot(Y)
        x, w = gh()
        s_y = np.sqrt(np.maximum(2.0 * np.sum(oh * var, 1), 1e-10))
        X = np.sum(oh * mu, 1)[:, None] + x[None] * s_y[:, None]                      # [N, K]
        s = np.sqrt(np.maximum(var, 1e-10))
        d = (X[:, None, :] - mu[:, :, None]) / s[:, :, None]                          # [N, C, K]
        cdf = 0.5 * (1.0 + erf(d / np.sqrt(2.0))) * (1 - 2 * SQUASH) + SQUASH
        cdf = cdf * (1.0 - oh)[:, :, None] + oh[:, :, None]
        return oh, x, w, s_y, s, d, cdf

    def prob_is_largest(self, Y, mu, var) -> np.ndarray:
        """p per row [N]."""
        _, _, w, _, _, _, cdf = self._parts(Y, mu, var)
        return np.prod(cdf, 1) @ w

    def variational_expectations(self, mu, var, Y) -> np.ndarray:
        """Per row [N] (multiclass.py:201-210)."""
        p = self.prob_is_largest(Y, mu, var)
        return p * np.log(1.0 - self.epsilon) + (1.0 - p) * np.log(self.eps_k1)

    def density(self, mu, var, Y, p=None) -> np.ndarray:
        p = self.prob_is_largest(Y, mu, var) if p is None else p
        return p * (1.0 - self.epsilon) + (1.0 - p) * self.eps_k1

    def predict_log_density(self, mu, var, Y) -> np.ndarray:
        return np.log(self.density(mu, var, Y))

    def predict_mean_and_var(self, mu, var) -> Tuple[np.ndarray, np.ndarray]:
        N = mu.shape[0]
        ps = np.stack([self.density(mu, var, np.full((N, 1), float(c))) for c in range(self.num_classes)], 1)
        return ps, ps - ps ** 2

    def ve_grads(self, mu, var, Y) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(dVE/dmu [N, C], dVE/dvar [N, C], dVE/deps [N])."""
        oh, x, w, s_y, s, d, cdf = self._parts(Y, mu, var)
        ones = np.ones_like(cdf[:, :1])
        pre = np.concatenate([ones, np.cumprod(cdf, 1)[:, :-1]], 1)
        suf = np.concatenate([np.cumprod(cdf[:, ::-1], 1)[:, ::-1][:, 1:], ones], 1)
        E = pre * suf                                                                  # prod_{c' != c} (y factor 1)
        off = (1.0 - oh)[:, :, None]
        g = off * w[None, None] * E * (1 - 2 * SQUASH) * np.exp(-0.5 * d * d) / np.sqrt(2 * np.pi) / s[:, :, None]
        kappa = np.log(1.0 - self.epsilon) - np.log(self.eps_k1)
        dmu = -kappa * g.sum(2)
        dv = np.where(var > 1e-10, -kappa * np.sum(g * d, 2) / (2.0 * s), 0.0) * (1.0 - oh)
        gs = g.sum(1)                                                                  # [N, K]
        dmu = dmu + oh * (kappa * gs.sum(1))[:, None]
        dvy = np.where(2.0 * np.sum(oh * var, 1) > 1e-10, kappa * (gs @ x) / s_y, 0.0)
        dv = dv + oh * dvy[:, None]
        p = np.prod(cdf, 1) @ w
        deps = -p / (1.0 - self.epsilon) + (1.0 - p) / self.epsilon
        return dmu, dv, deps


def labels(rng: np.random.Generator, F: np.ndarray, noise: float = 0.3) -> np.ndarray:
    """Labels [N, 1]: the argmax of the latent values F [N, C] plus Gaussian noise."""
    return np.argmax(F + noise * rng.standard_normal(F.shape), 1)[:, None].astype(np.float64)


# ---- SVGP ------------------------------------------------------------------------------------------------------
def svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, lik: MultiClass, *, whiten=True, num_data=None, mean_function=None,
              jitter=O.DEFAULT_JITTER) -> float:
    """svgp.py:166-181 with the MultiClass likelihood (labels Y [B, 1], P = q_mu.shape[1] latents)."""
    kl = O.prior_kl(Z, kernel, q_mu, q_sqrt, whiten=whiten, jitter=jitter)
    f_mean, f_var = O.svgp_predict_f(X, Z, kernel, q_mu, q_sqrt, whiten=whiten, full_cov=False,
                                     mean_function=mean_function, jitter=jitter)
    scale = 1.0 if num_data is None else float(num_data) / X.shape[0]
    return float(np.sum(lik.variational_expectations(f_mean, f_var, Y)) * scale - kl)


def svgp_elbo_and_grad(X, Y, kernel, Z, q_mu, q_sqrt, lik: MultiClass, *, whiten=True, num_data=None,
                       mean_function=None, jitter=O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The ELBO of svgp_elbo and its gradient: {"leaves", "lik" (d/d epsilon), "mean", "Z", "q_mu", "q_sqrt"} as
    tests/lik_oracle.py::svgp_elbo_lik_and_grad."""
    B = X.shape[0]
    M, P = q_mu.shape
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
    dmu, dv, deps = lik.ve_grads(f_mean, f_var, Y)
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
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = R.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = R.sum(0)
        rhs = R.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else R
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    elbo = svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, lik, whiten=whiten, num_data=num_data,
                     mean_function=mean_function, jitter=jitter)
    return elbo, {"leaves": per_leaf, "lik": float(c * np.sum(deps)), "mean": mean, "Z": dZ, "q_mu": dq_mu,
                  "q_sqrt": dq_sqrt}
