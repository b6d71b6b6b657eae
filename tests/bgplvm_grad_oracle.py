"""Gradient oracle of the Bayesian GPLVM bound (test infrastructure): the target of gpk_bgplvm_elbo_grad.  With s the
noise variance, P the output dimension, K = Kuu + jitter I = L L^T, A~ = L^-1 psi2 L^-T, B = I + A~/s = LB LB^T,
c = LB^-1 L^-1 psi1^T Y / s, v = LB^-T c and u = L^-T v:

    dF/dpsi1 = Y u^T / s                   dF/dpsi2 = L^-T [P (I - B^-1) - v v^T] L^-1 / (2s)
    dF/dKuu  = L^-T [P/2 (I - B^-1) - P/2 (B - I) - v v^T / 2] L^-1
    dF/dpsi0 = -P / (2s)
    dF/ds    = [-NP + P (M - tr B^-1) + P psi0/s - P tr(A~)/s + sum Y^2/s - |c|^2 - |v|^2] / (2s)
    dKL/dmu  = (mu - m0) / p,   dKL/dS = -1/(2S) + 1/(2p)

and the psi adjoints (psi_vjp): psi1[n,m] = sigma^2 exp(-u1), psi2_n[m,m'] = sigma^4 exp(-u2) with the exponents of
csrc/psi.cu, each differentiated in closed form.  Pinned by central finite differences of
tests/bgplvm_oracle.py::bgplvm_elbo and, psi_vjp alone, of tests/bgplvm_oracle.py::psi_statistics in
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
    Za = Z[:, cols]
    # Kuu: K_ij = sigma^2 exp(-1/2 sum_d (z_id - z_jd)^2 / l_d^2) (the jitter carries no parameter)
    K = Kuu - jitter * np.eye(M)
    dzz = Za[:, None, :] - Za[None, :, :]
    dvar += np.sum(Gk * K) / var
    dl += np.einsum("ij,ijd->d", Gk * K, dzz ** 2) / ell ** 3
    dZ[:, cols] += -2.0 * np.einsum("ij,ijd->id", Gk * K, dzz) / l2
    pg = psi_vjp(mu, S, Z, kernel, G1, G2)
    dmu += pg["mu"]
    dS += pg["S"]
    dZ += pg["Z"]
    dvar += pg["variance"]
    dl += pg["lengthscales"]
    g.update(variance=dvar, mu=dmu, S=dS, Z=dZ)
    g["lengthscales"] = dl if np.ndim(kernel.lengthscales) > 0 else float(dl.sum())
    return g


def psi_vjp(mu, S, Z, kernel, G1, G2, abs_sums=False, block_elems=1 << 21):
    """The vector-Jacobian product of the psi statistics: with F = sum G1 * psi1 + sum G2 * psi2 (G1 [N, M], G2 [M, M]
    symmetric), {"mu" [N, Q], "S" [N, Q], "Z" [M, Q], "variance", "lengthscales" [nd] (one per active dim, scalar
    lengthscale too)}: dF/d(value), zeros in the columns outside the leaf's active dims.  With diff1 = mu - z_m,
    a = 1/(l^2 + S), e1 = G1 psi1 and diff2 = mu - zbar, b = 1/(l^2 + 2S), e2 = G2 sigma^4 exp(-u2) per point:

        dmu = -a sum_m e1 diff1 - 2 b sum_ij e2 diff2
        dS  = 1/2 a^2 sum_m e1 diff1^2 - 1/2 a sum_m e1 - b sum_ij e2 + 2 b^2 sum_ij e2 diff2^2
        dZ_i = sum_n e1 a diff1 - sum_nj e2 (z_i - z_j) / l^2 + 2 sum_nj e2 b diff2
        dsigma^2 = sum e1 / sigma^2 + 2 sum e2 / sigma^2
        dl = sum_n [l a^2 sum_m e1 diff1^2 + S a sum_m e1 / l] + sum_nij e2 (z_i - z_j)^2 / (2 l^3)
             + sum_n [2 l b^2 sum_ij e2 diff2^2 + 2 S b sum_ij e2 / l]

    evaluated over blocks of points (at most block_elems entries of [points, M, M, nd] at a time).

    With abs_sums the result is (grads, sums), sums[name] = (T, U, C) of the shape of grads[name], per output element
    over the terms t_k behind it (one per point, inducing point or pair and formula term above):
        T = sum_k |t_k|,  U = max u_k over the terms with exp(-u_k) > 0 (u_k the psi1 or psi2 exponent of the term),
        C = sum_k |t_k| kappa_k, kappa_k = 2 sum_d |diff2_d| b_d h_d + p_d h_d / |diff2_d| for a psi2 term carrying
            diff2_d^p_d (0 for psi1 terms), h_d = |mu_d| + |zbar_d|:
    a rounding of diff2 = mu - zbar by eps h (it cancels: the error is absolute, not relative to diff2) moves the
    exponent by up to 2 |diff2| b eps h per dim and the factor diff2^p by p eps h / |diff2| relative, so moves t_k by
    at most eps |t_k| kappa_k."""
    N, Q = mu.shape
    M = Z.shape[0]
    cols = _cols(kernel, Q)
    nd = len(cols)
    ell = _lengthscales(kernel, nd)
    l2 = ell ** 2
    var = float(kernel.variance)
    ma, Sa, Za = mu[:, cols], S[:, cols], Z[:, cols]
    G1 = np.asarray(G1, dtype=np.float64)
    G2 = np.asarray(G2, dtype=np.float64)
    dmu, dS, dZa = np.zeros((N, nd)), np.zeros((N, nd)), np.zeros((M, nd))
    dvar, dl = 0.0, np.zeros(nd)
    dzz = Za[:, None, :] - Za[None, :, :]
    ez = np.sum(dzz ** 2 / (4 * l2), axis=-1)
    zbar = 0.5 * (Za[:, None, :] + Za[None, :, :])
    if abs_sums:
        T = dict(mu=np.zeros((N, nd)), S=np.zeros((N, nd)), Z=np.zeros((M, nd)), variance=0.0, lengthscales=np.zeros(nd))
        C = {k: np.zeros_like(v) if k != "variance" else 0.0 for k, v in T.items()}
        U = {k: np.zeros_like(v) if k != "variance" else 0.0 for k, v in T.items()}
    nb = max(1, block_elems // max(1, M * M * nd))
    for n0 in range(0, N, nb):
        sl = slice(n0, min(N, n0 + nb))
        m_, s_, g1 = ma[sl], Sa[sl], G1[sl]
        # psi1
        a = 1.0 / (l2 + s_)
        d1 = m_[:, None, :] - Za[None, :, :]
        u1 = 0.5 * np.sum(np.log1p(s_ / l2), axis=1)[:, None] + 0.5 * np.einsum("bmd,bd->bm", d1 ** 2, a)
        e1 = g1 * var * np.exp(-u1)
        dmu[sl] += -np.einsum("bm,bmd->bd", e1, d1) * a
        dS[sl] += 0.5 * a * a * np.einsum("bm,bmd->bd", e1, d1 ** 2) - 0.5 * a * e1.sum(1)[:, None]
        dZa += np.einsum("bm,bmd,bd->md", e1, d1, a)
        dvar += e1.sum() / var
        dl += np.sum(ell * a * a * np.einsum("bm,bmd->bd", e1, d1 ** 2) + s_ * a * e1.sum(1)[:, None] / ell, axis=0)
        # psi2 per point
        b = 1.0 / (l2 + 2 * s_)
        d2 = m_[:, None, None, :] - zbar[None]
        u2 = (ez[None] + 0.5 * np.sum(np.log1p(2 * s_ / l2), axis=1)[:, None, None]
              + np.einsum("bijd,bd->bij", d2 ** 2, b))
        e2 = G2[None] * var * var * np.exp(-u2)
        E = e2.sum(axis=(1, 2))
        dmu[sl] += -2 * b * np.einsum("bij,bijd->bd", e2, d2)
        dS[sl] += -b * E[:, None] + 2 * b * b * np.einsum("bij,bijd->bd", e2, d2 ** 2)
        dvar += 2 * e2.sum() / var
        dZa += -2 * (np.einsum("bij,ijd->id", e2, dzz) / (2 * l2) - np.einsum("bij,bijd,bd->id", e2, d2, b))
        dl += (np.einsum("bij,ijd->d", e2, dzz ** 2) / (2 * ell ** 3)
               + np.sum(2 * ell * b * b * np.einsum("bij,bijd->bd", e2, d2 ** 2) + 2 * s_ * b * E[:, None] / ell, axis=0))
        if abs_sums:
            _psi_abs_sums(T, U, C, sl, var, ell, l2, m_, s_, a, d1, u1, np.abs(e1), b, d2, u2, np.abs(e2), dzz, zbar)
    g = {"mu": np.zeros((N, Q)), "S": np.zeros((N, Q)), "Z": np.zeros((M, Q)), "variance": dvar, "lengthscales": dl}
    g["mu"][:, cols], g["S"][:, cols], g["Z"][:, cols] = dmu, dS, dZa
    if not abs_sums:
        return g
    sums = {}
    for k in g:
        if k in ("mu", "S", "Z"):
            full = [np.zeros_like(g[k]) for _ in range(3)]
            for f, x in zip(full, (T[k], U[k], C[k])):
                f[:, cols] = x
            sums[k] = tuple(full)
        else:
            sums[k] = (T[k], U[k], C[k])
    return g, sums


def _psi_abs_sums(T, U, C, sl, var, ell, l2, m_, s_, a, d1, u1, ae1, b, d2, u2, ae2, dzz, zbar):
    """Adds one block of points to the (T, U, C) sums of psi_vjp; ae1 = |e1|, ae2 = |e2|."""
    ad1, ad2, adz = np.abs(d1), np.abs(d2), np.abs(dzz)
    h = np.abs(m_)[:, None, None, :] + np.abs(zbar)[None]             # [B, M, M, nd]
    ku = 2 * np.einsum("bijd,bd->bij", ad2 * h, b)                      # exponent cancellation, relative
    u1m = np.where(np.exp(-u1) > 0, u1, 0.0)
    u2m = np.where(np.exp(-u2) > 0, u2, 0.0)
    S1 = ae1.sum(1)                                                     # [B]
    S2 = ae2.sum((1, 2))
    S2k = (ae2 * ku).sum((1, 2))
    e1d1 = np.einsum("bm,bmd->bd", ae1, ad1)
    e1d1s = np.einsum("bm,bmd->bd", ae1, ad1 ** 2)
    e2d2 = np.einsum("bij,bijd->bd", ae2, ad2)
    e2d2s = np.einsum("bij,bijd->bd", ae2, ad2 ** 2)
    e2d2k = np.einsum("bij,bijd->bd", ae2 * ku, ad2)
    e2d2sk = np.einsum("bij,bijd->bd", ae2 * ku, ad2 ** 2)
    e2h = np.einsum("bij,bijd->bd", ae2, h)
    e2d2h = np.einsum("bij,bijd->bd", ae2, ad2 * h)
    # dmu, dS
    T["mu"][sl] += a * e1d1 + 2 * b * e2d2
    C["mu"][sl] += 2 * b * (e2d2k + e2h)
    T["S"][sl] += 0.5 * a * a * e1d1s + 0.5 * a * S1[:, None] + b * S2[:, None] + 2 * b * b * e2d2s
    C["S"][sl] += b * S2k[:, None] + 2 * b * b * (e2d2sk + 2 * e2d2h)
    upt = np.maximum(u1m.max(1), u2m.max((1, 2)))[:, None]
    U["mu"][sl] = np.maximum(U["mu"][sl], upt)
    U["S"][sl] = np.maximum(U["S"][sl], upt)
    # dZ (row i: the pairs (i, j) over j, twice: the symmetric (j, i) terms)
    T["Z"] += (np.einsum("bm,bmd,bd->md", ae1, ad1, a) + 2 * np.einsum("bij,ijd->id", ae2, adz) / (2 * l2)
               + 2 * np.einsum("bij,bijd,bd->id", ae2, ad2, b))
    C["Z"] += (2 * np.einsum("bij,ijd->id", ae2 * ku, adz) / (2 * l2)
               + 2 * np.einsum("bij,bijd,bd->id", ae2 * ku, ad2, b) + 2 * np.einsum("bij,bijd,bd->id", ae2, h, b))
    U["Z"] = np.maximum(U["Z"], np.maximum(u1m.max(0), u2m.max((0, 2)))[:, None])
    # the kernel parameters
    T["variance"] += S1.sum() / var + 2 * S2.sum() / var
    C["variance"] += 2 * S2k.sum() / var
    T["lengthscales"] += (np.sum(ell * a * a * e1d1s + s_ * a * S1[:, None] / ell, axis=0)
                          + np.einsum("bij,ijd->d", ae2, adz ** 2) / (2 * ell ** 3)
                          + np.sum(2 * ell * b * b * e2d2s + 2 * s_ * b * S2[:, None] / ell, axis=0))
    C["lengthscales"] += (np.einsum("bij,ijd->d", ae2 * ku, adz ** 2) / (2 * ell ** 3)
                          + np.sum(2 * ell * b * b * (e2d2sk + 2 * e2d2h) + 2 * s_ * b * S2k[:, None] / ell, axis=0))
    um = max(float(u1m.max()), float(u2m.max()))
    U["variance"] = max(U["variance"], um)
    U["lengthscales"] = np.maximum(U["lengthscales"], um)
