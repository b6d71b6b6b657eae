"""Oracle of HeteroskedasticTFPConditional with a Normal distribution (test infrastructure, like tests/lik_oracle.py; not
imported by the product): the target of the HETEROSKEDASTIC descriptor of csrc/lik.cu and of the SVGP gradients
through it.

The reference (gpflow/likelihoods/multilatent.py:95-133 through base.py:279-400 and quadrature/gauss_hermite.py) puts a
20 x 20 tensor grid of NDiagGHQuadrature(2, 20) over the two latents of a row, F = [f, g], y ~ N(f, s(g)^2) with s(g) =
transform(g) + lower.  `Hetero` evaluates that literal grid (`grid_*`), so the tests check the device's factorised form
against it rather than assume it.  The factorised forms and the closed-form adjoints, with z_j, w_j the scaled nodes,
g_j = mu_g + sqrt(v_g) z_j, Q = (y - mu_f)^2 + v_f, A = sum_j w_j log s(g_j), S = sum_j w_j s(g_j)^-2 and h(g) = -log s
- Q / (2 s^2):
    VE = -1/2 log 2 pi - A - Q S / 2
    dVE/dmu_f = (y - mu_f) S,   dVE/dv_f = -S / 2,   dVE/dmu_g = sum_j w_j h'(g_j),
    dVE/dv_g = sum_j w_j h'(g_j) z_j / (2 sqrt v_g), or h''(mu_g) / 2 at v_g = 0,
    h' = (s'/s)(Q/s^2 - 1),   h'' = (s''/s - (s'/s)^2)(Q/s^2 - 1) - 2 Q s'^2 / s^4.
The SVGP ELBO and its gradient come from tests/svgp_grad_oracle.py, which takes any likelihood with
`variational_expectations` and `ve_grads`: every model shape has two latents there (a single-output kernel with two
latents is one shared kernel and one shared Z).
"""
from __future__ import annotations

from typing import Tuple

import numpy as np
from scipy.special import logsumexp

from oracle import gp_oracle as O
from tests.lik_oracle import gh_points_and_weights

TRANSFORMS = [("exp", 0.0), ("softplus", 0.0), ("exp", 1e-3), ("softplus", 0.05)]


def rows(seed=0, N=12):
    """Rows with v_f = 0, v_g = 0 and |mu_g| up to 8 among ordinary ones."""
    rng = np.random.default_rng(seed)
    mu = np.stack([rng.uniform(-2, 2, N), rng.uniform(-1.5, 1.5, N)], 1)
    v = np.stack([rng.uniform(0.05, 1.5, N), rng.uniform(0.01, 0.8, N)], 1)
    mu[0, 1], mu[1, 1], mu[2, 1], mu[3, 1] = 8.0, -8.0, 6.5, -7.0
    v[4, 0] = 0.0
    v[5, 1] = 0.0
    v[1, 1] = 0.0
    v[6, :] = 0.0
    y = mu[:, :1] + rng.standard_normal((N, 1)) * np.exp(0.3 * mu[:, 1:2])
    return mu, v, y


def scale_fn(transform: str, lower: float, g):
    """s(g), s'(g), s''(g) of Exp or Softplus shifted by `lower`."""
    g = np.asarray(g, dtype=np.float64)
    if transform == "exp":
        e = np.exp(g)
        return e + lower, e, e
    if transform == "softplus":
        sig = np.exp(-np.logaddexp(0.0, -g))
        return np.logaddexp(0.0, g) + lower, sig, sig * (1.0 - sig)
    raise ValueError(transform)


class Hetero:
    """One heteroskedastic Normal likelihood; mu, v [N, 2] (location, log-scale latent), y [N, 1]."""

    def __init__(self, transform: str = "exp", lower: float = 0.0):
        self.transform, self.lower = transform, float(lower)

    def s(self, g):
        return scale_fn(self.transform, self.lower, g)[0]

    def logp(self, y, f, g):
        s = self.s(g)
        return -0.5 * O.LOG2PI - np.log(s) - 0.5 * (y - f) ** 2 / s ** 2

    # ---- the literal 20 x 20 grid (base.py:344-400 with NDiagGHQuadrature(2, 20)) ----
    def _grid(self, mu, v):
        z, w = gh_points_and_weights()
        F = mu[:, 0:1, None] + np.sqrt(v[:, 0:1, None]) * z[None, :, None]   # [N, i, 1]
        G = mu[:, 1:2, None] + np.sqrt(v[:, 1:2, None]) * z[None, None, :]   # [N, 1, j]
        return F, G, w[:, None] * w[None, :]

    def grid_ve(self, mu, v, y):
        F, G, W = self._grid(mu, v)
        return np.sum(W[None] * self.logp(y[:, :, None], F, G), axis=(1, 2))

    def grid_mean_and_var(self, mu, v):
        F, G, W = self._grid(mu, v)
        ey = np.sum(W[None] * (F + 0 * G), axis=(1, 2))
        ey2 = np.sum(W[None] * (self.s(G) ** 2 + F ** 2), axis=(1, 2))
        return ey[:, None], (ey2 - ey ** 2)[:, None]

    def grid_log_density(self, mu, v, y):
        F, G, W = self._grid(mu, v)
        t = self.logp(y[:, :, None], F, G) + np.log(W)[None]
        return logsumexp(t.reshape(t.shape[0], -1), axis=1)

    # ---- the factorised forms the device evaluates ----
    def _nodes(self, mu, v):
        z, w = gh_points_and_weights()
        return z, w, mu[:, 1:2] + np.sqrt(v[:, 1:2]) * z[None]

    def factorised_ve(self, mu, v, y):
        _, w, G = self._nodes(mu, v)
        s = self.s(G)
        Q = (y[:, 0] - mu[:, 0]) ** 2 + v[:, 0]
        return -0.5 * O.LOG2PI - np.sum(w * np.log(s), 1) - 0.5 * Q * np.sum(w / s ** 2, 1)

    def factorised_mean_and_var(self, mu, v):
        _, w, G = self._nodes(mu, v)
        return mu[:, 0:1], (np.sum(w * self.s(G) ** 2, 1) + v[:, 0])[:, None]

    # ---- what tests/svgp_grad_oracle.py consumes ----
    def variational_expectations(self, mu, v, y):
        """Per row [N]: the literal grid."""
        return self.grid_ve(mu, v, y)

    def ve_grads(self, mu, v, y) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """(dVE/dmu [N, 2], dVE/dv [N, 2], 0): the closed forms, the v_g = 0 limit included."""
        z, w, G = self._nodes(mu, v)
        s, s1, s2 = scale_fn(self.transform, self.lower, G)
        r = y[:, 0] - mu[:, 0]
        Q = r ** 2 + v[:, 0]
        S = np.sum(w / s ** 2, 1)
        h1 = s1 / s * (Q[:, None] / s ** 2 - 1.0)
        dmu = np.stack([r * S, np.sum(w * h1, 1)], 1)
        vg = v[:, 1]
        with np.errstate(divide="ignore", invalid="ignore"):
            dvg = np.sum(w * h1 * z, 1) / (2.0 * np.sqrt(vg))
        s0, s10, s20 = scale_fn(self.transform, self.lower, mu[:, 1])
        a, qs = s10 / s0, Q / s0 ** 2
        limit = 0.5 * ((s20 / s0 - a * a) * (qs - 1.0) - 2.0 * qs * a * a)
        dv = np.stack([-0.5 * S, np.where(vg > 0, dvg, limit)], 1)
        return dmu, dv, np.zeros_like(mu)

    def predict_mean_and_var(self, mu, v):
        return self.factorised_mean_and_var(mu, v)

    def predict_log_density(self, mu, v, y):
        return self.grid_log_density(mu, v, y)
