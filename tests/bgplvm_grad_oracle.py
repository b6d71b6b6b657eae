"""Gradient oracle of the Bayesian GPLVM bound (test infrastructure): the target of gpk_bgplvm_elbo_grad.  With s the
noise variance, P the output dimension, K = Kuu + jitter I = L L^T, A~ = L^-1 psi2 L^-T, B = I + A~/s = LB LB^T,
c = LB^-1 L^-1 psi1^T Y / s, v = LB^-T c and u = L^-T v:

    dF/dpsi1 = Y u^T / s                   dF/dpsi2 = L^-T [P (I - B^-1) - v v^T] L^-1 / (2s)
    dF/dKuu  = L^-T [P/2 (I - B^-1) - P/2 (B - I) - v v^T / 2] L^-1
    dF/dpsi0 = -P / (2s)
    dF/ds    = [-NP + P (M - tr B^-1) + P psi0/s - P tr(A~)/s + sum Y^2/s - |c|^2 - |v|^2] / (2s)
    dKL/dmu  = (mu - m0) / p,   dKL/dS = -1/(2S) + 1/(2p)

and the psi adjoints: psi1[n,m] = sigma^2 exp(-u1), psi2_n[m,m'] = sigma^4 exp(-u2) with the exponents of csrc/psi.cu,
each differentiated in closed form.  Pinned by central finite differences of tests/bgplvm_oracle.py::bgplvm_elbo in
tests/test_oracle_bgplvm.py."""
from __future__ import annotations

import numpy as np

from oracle import gp_oracle as O
from tests.bgplvm_oracle import _cols, _lengthscales, psi_statistics


def bgplvm_elbo_grad(Y, mu, S, Z, kernel, noise, m0=None, p0=None, jitter=O.DEFAULT_JITTER):
    """{"noise", "variance", "lengthscales" (scalar or [Q']), "mu" [N, Q], "S" [N, Q], "Z" [M, Q]}: dF/d(value)."""
    m0 = np.zeros_like(mu) if m0 is None else m0
    p0 = np.ones_like(mu) if p0 is None else p0
    N, Q = mu.shape
    M, P = Z.shape[0], Y.shape[1]
    s = noise
    cols = _cols(kernel, Q)
    nd = len(cols)
    ell = _lengthscales(kernel, nd)
    l2 = ell ** 2
    var = float(kernel.variance)
    psi0, psi1, psi2 = psi_statistics(mu, S, Z, kernel)
    Kuu = O.Kuu(Z, kernel, jitter=jitter)
    L = np.linalg.cholesky(Kuu)
    Li = np.linalg.inv(L)
    At = Li @ psi2 @ Li.T
    B = np.eye(M) + At / s
    LB = np.linalg.cholesky(B)
    Binv = np.linalg.inv(B)
    c = np.linalg.solve(LB, Li @ psi1.T @ Y) / s
    v = np.linalg.solve(LB.T, c)
    u = Li.T @ v
    G1 = Y @ u.T / s
    G2 = Li.T @ (P * (np.eye(M) - Binv) - v @ v.T) @ Li / (2 * s)
    Gk = Li.T @ (0.5 * P * (np.eye(M) - Binv) - 0.5 * P * (B - np.eye(M)) - 0.5 * v @ v.T) @ Li
    g = {"noise": (-N * P + P * (M - np.trace(Binv)) + P * psi0 / s - P * np.trace(At) / s + np.sum(Y * Y) / s
                   - np.sum(c * c) - np.sum(v * v)) / (2 * s)}
    dmu, dS, dZ = -(mu - m0) / p0, 1.0 / (2 * S) - 1.0 / (2 * p0), np.zeros((M, Q))
    dvar = -P * N / (2 * s)
    dl = np.zeros(nd)
    ma, Sa, Za = mu[:, cols], S[:, cols], Z[:, cols]
    # Kuu: K_ij = sigma^2 exp(-1/2 sum_d (z_id - z_jd)^2 / l_d^2) (the jitter carries no parameter)
    K = Kuu - jitter * np.eye(M)
    dzz = Za[:, None, :] - Za[None, :, :]
    dvar += np.sum(Gk * K) / var
    dl += np.einsum("ij,ijd->d", Gk * K, dzz ** 2) / ell ** 3
    dZ[:, cols] += -2.0 * np.einsum("ij,ijd->id", Gk * K, dzz) / l2
    # psi1
    a = 1.0 / (l2 + Sa)
    d1 = ma[:, None, :] - Za[None, :, :]
    e1 = G1 * psi1
    dmu[:, cols] += -np.einsum("nm,nmd->nd", e1, d1) * a
    dS[:, cols] += 0.5 * a * a * np.einsum("nm,nmd->nd", e1, d1 ** 2) - 0.5 * a * e1.sum(1)[:, None]
    dZ[:, cols] += np.einsum("nm,nmd,nd->md", e1, d1, a)
    dvar += e1.sum() / var
    dl += np.sum(ell * a * a * np.einsum("nm,nmd->nd", e1, d1 ** 2) + Sa * a * e1.sum(1)[:, None] / ell, axis=0)
    # psi2 per point
    b = 1.0 / (l2 + 2 * Sa)
    zbar = 0.5 * (Za[:, None, :] + Za[None, :, :])
    d2 = ma[:, None, None, :] - zbar[None]
    u2 = (np.sum(dzz ** 2 / (4 * l2), axis=-1)[None] + 0.5 * np.sum(np.log1p(2 * Sa / l2), axis=1)[:, None, None]
          + np.einsum("nijd,nd->nij", d2 ** 2, b))
    e2 = G2[None] * var * var * np.exp(-u2)
    E = e2.sum(axis=(1, 2))
    dmu[:, cols] += -2 * b * np.einsum("nij,nijd->nd", e2, d2)
    dS[:, cols] += -b * E[:, None] + 2 * b * b * np.einsum("nij,nijd->nd", e2, d2 ** 2)
    dvar += 2 * e2.sum() / var
    dZ[:, cols] += -2 * (np.einsum("nij,ijd->id", e2, dzz) / (2 * l2) - np.einsum("nij,nijd,nd->id", e2, d2, b))
    dl += (np.einsum("nij,ijd->d", e2, dzz ** 2) / (2 * ell ** 3)
           + np.sum(2 * ell * b * b * np.einsum("nij,nijd->nd", e2, d2 ** 2) + 2 * Sa * b * E[:, None] / ell, axis=0))
    g.update(variance=dvar, mu=dmu, S=dS, Z=dZ)
    g["lengthscales"] = dl if np.ndim(kernel.lengthscales) > 0 else float(dl.sum())
    return g
