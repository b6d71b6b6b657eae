"""Oracle of the MultiClass likelihood with the RobustMax inverse link (test infrastructure, like tests/lik_oracle.py;
not imported by the product): the target of the MultiClass kernels of csrc/lik.cu, and a likelihood
tests/svgp_grad_oracle.py takes (the target of gpk_svgp_elbo_grad with a MULTICLASS descriptor).

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
tests/svgp_grad_oracle.py::svgp_elbo_and_grad takes these as dVE/dfmean and dVE/dfvar, with one label column.  Pinned by
central finite differences in tests/test_oracle_multiclass.py.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
from scipy.special import erf

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

