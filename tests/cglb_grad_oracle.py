"""Gradient oracle for the CGLB bound with any fused kernel expression (test infrastructure, like
tests/sgpr_grad_oracle.py; not imported by the product): the target of gpk_cglb_elbo_grad.

The bound at a given v [P, N] (gpflow/models/cglb.py:83-160, restated in tests/cglb_oracle.py) depends on the kernel
through K^ = K(X, X) + s I, Kuf, Kuu and Kdiag.  Its adjoints in those matrices are tests/cglb_oracle.py::bound_adjoints
(pinned there by finite differences); with z = Q^-1 r, r = e^T - v K^, Q = A'^T A' + s I, A' = L^-1 Kuf, V = v^T:

    dF/dK^   = 1/2 V V^T + 1/2 (z V^T + V z^T)
    dF/dKuf  = L^-T [(-P/s B^-1 - 2 c_t/s I) A' + Az z^T],            Az = A' z
    dF/dKuu  = L^-T [P/2 (I - B^-1) - 1/2 Az Az^T + c_t (B - I)] L^-1
    dF/dKdiag = c_t / s,  c_t = -(P/2) / (1 + t/N),  t = (sum Kdiag - |A'|_F^2) / s
    dF/ds    = sum (V^2/2 + z V) - P/2 (N - M + tr B^-1) / s + |z|^2 / 2 - c_t t / s   (the first sum is sum_i dF/dK^_ii)
    dF/dm    = V + z,   dF/dv = (K^ z - r^T)^T

and dF/dtheta adds the four sources, each leaf's dK by the product rule: the N x N one through
kernel_grad_oracle.weighted_leaf_grads, the other three through kernel_grad_oracle's walk and reduce.  dF/dZ comes from
the Kuf and Kuu sources as in SGPR.

Nothing here is N x N: r, K^ z and the N x N reduction run over row blocks of K(X, X), and z comes from the Woodbury
form of Q^-1 (the Nystrom preconditioner, as the device applies it).  A row block k(X_b, X) evaluated with X2 given
drops the diagonal a White leaf adds to K(X, X), so the block's own columns are evaluated as k(X_b), with X2 = None.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
from scipy.linalg import cho_solve

from oracle import gp_oracle as O
from tests import kernel_grad_oracle as KG

LOG2PI = np.log(2.0 * np.pi)


def _rows(cross, square, r0: int, r1: int):
    """Rows r0:r1 of an N-column matrix from its cross evaluation against all of X, with columns r0:r1 (the block's
    diagonal square) replaced by the X2 = None evaluation; arrays or dicts of arrays, stacks on a leading axis."""
    if isinstance(cross, dict):
        return {name: _rows(cross[name], square[name], r0, r1) for name in cross}
    cross[..., r0:r1] = square
    return cross


def _kv_rows(kernel: O.Kernel, X: np.ndarray, W: np.ndarray, block_rows: int) -> Tuple[np.ndarray, np.ndarray]:
    """(K(X, X) W, |K(X, X)| |W|) for W [N, P], by row blocks."""
    N = X.shape[0]
    out, out_abs = np.empty_like(W), np.empty_like(W)
    for r0 in range(0, N, block_rows):
        r1 = min(N, r0 + block_rows)
        Kb = _rows(kernel(X[r0:r1], X), kernel(X[r0:r1]), r0, r1)
        out[r0:r1] = Kb @ W
        out_abs[r0:r1] = np.abs(Kb) @ np.abs(W)
    return out, out_abs


def _add(acc: List[Dict[str, object]], part: List[Dict[str, object]]) -> List[Dict[str, object]]:
    if not acc:
        return [dict(d) for d in part]
    return [{name: a[name] + b[name] for name in a} for a, b in zip(acc, part)]


def cglb_elbo_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, Z: np.ndarray, s2: float, v: np.ndarray,
                            mean_function=None, jitter: float = O.DEFAULT_JITTER, abs_sums: bool = False,
                            block_rows: int = 256) -> Tuple[float, Dict[str, object]]:
    """The CGLB bound at the given v [P, N] (cglb.py:83-160) and its gradient, v held fixed in K^ and Q only through
    the closed forms above, for any Sum / Product expression of the fused leaves, the Constant / Linear mean functions,
    the inducing points and v.  Returns (elbo, {"leaves": [per leaf in `leaves()` order], "noise_variance": float,
    "mean": {"c"} or {"A", "b"} or {}, "Z": [M, D], "v": [P, N]}).  With `abs_sums` also the sums of |terms| the
    rounding of each gradient entry is relative to: "leaves_abs" (per slot, over the N x N, Kuf, Kuu and Kdiag
    sources), "noise_abs", "Z_abs" [M, D], "v_abs" [P, N] (|K^| |z| + |r|) and "mean_abs" (the mean's layout)."""
    N, P = Y.shape
    M, D = Z.shape
    s = float(s2)
    V = np.asarray(v, dtype=np.float64).T                              # [N, P]
    e = Y - O._mean(mean_function, X, P)
    Kuf = kernel(Z, X)
    L = O.cholesky(kernel(Z) + jitter * np.eye(M))
    Ap = O.tri_solve(L, Kuf)                                           # A' = L^-1 Kuf
    B = np.eye(M) + Ap @ Ap.T / s
    LB = O.cholesky(B)
    Bi = cho_solve((LB, True), np.eye(M))
    kdiag = kernel(X, full_cov=False)
    t = (np.sum(kdiag) - np.sum(Ap * Ap)) / s
    ct = -0.5 * P / (1.0 + t / N)

    KV, _ = _kv_rows(kernel, X, V, block_rows)
    KhV = KV + s * V
    R = e - KhV                                                        # r^T [N, P]
    z = (R - Ap.T @ cho_solve((LB, True), Ap @ R) / s) / s             # Q^-1 r^T by Woodbury
    lb = float(np.sum(V * (R + 0.5 * KhV)))
    rz = float(np.sum(R * z))
    logdet = -P * (np.sum(np.log(np.diag(LB))) + 0.5 * N * np.log(s) + 0.5 * N * np.log(1.0 + t / N))
    elbo = -0.5 * N * P * LOG2PI + logdet - (lb + 0.5 * rz)

    # the N x N source, by row blocks of G = 1/2 (V V^T + z V^T + V z^T)
    nn: List[Dict[str, object]] = []
    nn_abs: List[Dict[str, object]] = []
    for r0 in range(0, N, block_rows):
        r1 = min(N, r0 + block_rows)
        Xb = X[r0:r1]
        G = 0.5 * (V[r0:r1] @ V.T + z[r0:r1] @ V.T + V[r0:r1] @ z.T)
        g, ga = KG.weighted_leaf_grads(
            kernel, G, lambda k: _rows(k(Xb, X), k(Xb), r0, r1),
            lambda k: _rows(KG.leaf_dK_cross(k, Xb, X, with_z=False), KG.leaf_dK(k, Xb), r0, r1), abs_sums)
        nn, nn_abs = _add(nn, g), _add(nn_abs, ga)
    Kz, Kz_abs = _kv_rows(kernel, X, z, block_rows)

    # the Kuf, Kuu and Kdiag sources
    Az = Ap @ z
    Li = O.tri_solve(L, np.eye(M))
    I = np.eye(M)
    Guf = Li.T @ ((-P / s * Bi - 2.0 * ct / s * I) @ Ap + Az @ z.T)
    Guu = Li.T @ (0.5 * P * (I - Bi) - 0.5 * Az @ Az.T + ct * (B - I)) @ Li
    Gdiag = np.full(N, ct / s)
    uu, uf, dg = KG.inducing_stacks(kernel, X, Z)
    per_leaf = nn
    for part in (KG.reduce(Guu, uu), KG.reduce(Guf, uf), KG.reduce(Gdiag, dg)):
        per_leaf = _add(per_leaf, part)
    dZ = np.zeros((M, D))
    dZ_abs = np.zeros((M, D))
    for st in uf:
        dZ += np.einsum("mn,dmn->md", Guf, st["Z"])
        dZ_abs += np.einsum("mn,dmn->md", np.abs(Guf), np.abs(st["Z"]))
    for st in uu:
        dZ += 2.0 * np.einsum("ij,dij->id", Guu, st["Z"])
        dZ_abs += 2.0 * np.einsum("ij,dij->id", np.abs(Guu), np.abs(st["Z"]))

    trBi = float(np.trace(Bi))
    zz = float(np.sum(z * z))
    diag_G = np.sum(0.5 * V * V + z * V, axis=1)
    dnoise = float(np.sum(diag_G)) - 0.5 * P * (N - M + trBi) / s + 0.5 * zz - ct * t / s
    dm = V + z
    out = {"leaves": per_leaf, "noise_variance": dnoise, "mean": KG.mean_grads(mean_function, X, dm), "Z": dZ,
           "v": (Kz + s * z - R).T}
    if abs_sums:
        per_leaf_abs = nn_abs
        for part in (KG.reduce(Guu, uu, True), KG.reduce(Guf, uf, True), KG.reduce(Gdiag, dg, True)):
            per_leaf_abs = _add(per_leaf_abs, part)
        out["leaves_abs"] = per_leaf_abs
        out["noise_abs"] = float(np.sum(np.abs(diag_G)) + 0.5 * P * (N + M + trBi) / s + 0.5 * zz + abs(ct * t / s))
        out["Z_abs"] = dZ_abs
        out["v_abs"] = (Kz_abs + s * np.abs(z) + np.abs(R)).T
        out["mean_abs"] = KG.mean_grads(mean_function, np.abs(X), np.abs(V) + np.abs(z))
    return float(elbo), out
