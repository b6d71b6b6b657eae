"""Gradient oracle for the SGPR bound with any fused kernel expression (test infrastructure, like
tests/grad_expr_oracle.py; not imported by the product): the target of gpk_sgpr_elbo_grad.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/sgpr.py:181-289.  The closed forms
restated here, with s the noise variance, Yc = Y - m(X), K = Kuu + jitter I = L L^T, A' = L^-1 Kuf,
B = I + A'A'^T / s = LB LB^T, c = LB^-1 A' Yc / s and v = LB^-T c:

    dF/dKuu   = L^-T [P/2 (I - B^-1) - P/2 (B - I) - 1/2 v v^T] L^-1
    dF/dKuf   = L^-T [H A' + v Yc^T / s],   H = (P/s)(I - B^-1) - v v^T / s
    dF/dKdiag = -P / (2s)
    dF/ds     = [-NP + P (M - tr B^-1) + P trace_k - P trace_q + sum Yc^2 / s - |c|^2 - |v|^2] / (2s)
    dF/dm     = (Yc - A'^T v) / s

and dF/dtheta = sum G (.) dK/dtheta over the three matrices, each leaf's dK by the product rule of grad_expr_oracle.
dF/dZ adds sum_n G_uf[m, n] dk(z_m, x_n)/dz_m and 2 sum_j G_uu[i, j] dk(z_i, z_j)/dz_i (G_uu is symmetric).  Pinned by
central finite differences of oracle/gp_oracle.py::sgpr_elbo in tests/test_oracle_sgpr_grad.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests.grad_expr_oracle import _leaf_dK, leaves  # noqa: F401  (leaves: the device's leaf order, re-exported)


def _cols(k: O.Kernel, D: int) -> np.ndarray:
    """The input columns a leaf reads, in its active-dims order."""
    return np.arange(D)[k.active_dims] if isinstance(k.active_dims, slice) else np.asarray(k.active_dims, dtype=int)


def _leaf_dK_cross(k: O.Kernel, Z: np.ndarray, X: np.ndarray, with_z: bool = True) -> Dict[str, np.ndarray]:
    """d k(Z, X) / d(parameter) of one leaf, [M, N] (per-dimension parameters: a [D_active, M, N] stack), plus, with
    `with_z`, "Z": d k(z_m, x_n) / d z_{m, d} as a [D, M, N] stack over the full input columns."""
    M, D = Z.shape
    N = X.shape[0]
    Zs, Xs = k.slice(Z, X)
    cols = _cols(k, D)
    dZ = np.zeros((D, M, N)) if with_z else None
    if isinstance(k, O.Stationary):
        K = k(Z, X)
        var = float(k.variance)
        ell = np.asarray(k.lengthscales, dtype=np.float64)
        r2 = np.maximum(k.scaled_squared_euclid_dist(Zs, Xs), 0.0)
        r = np.sqrt(r2)
        with np.errstate(divide="ignore", invalid="ignore"):
            if isinstance(k, O.RationalQuadratic):
                u = r2 / (2.0 * float(k.alpha))
                dkds = -0.5 * K / (1.0 + u)
            elif isinstance(k, O.SquaredExponential):
                dkds = -0.5 * K
            elif isinstance(k, O.Exponential):
                dkds = np.where(r > 0, -K / (4.0 * r), 0.0)
            elif isinstance(k, O.Matern12):
                dkds = np.where(r > 0, -K / (2.0 * r), 0.0)
            elif isinstance(k, O.Matern32):
                dkds = -1.5 * var * np.exp(-np.sqrt(3.0) * r)
            elif isinstance(k, O.Matern52):
                s5 = np.sqrt(5.0)
                dkds = -(5.0 / 6.0) * var * (1.0 + s5 * r) * np.exp(-s5 * r)
            else:
                raise NotImplementedError(type(k).__name__)
        diff = Zs[:, None, :] - Xs[None, :, :]                                      # [M, N, Da]
        ell_d = np.broadcast_to(ell, (len(cols),)) if ell.ndim else np.full(len(cols), float(ell))
        out = {"variance": K / var}
        if ell.ndim == 0:
            out["lengthscales"] = dkds * (-2.0 * r2 / float(ell))
        else:
            out["lengthscales"] = np.stack([dkds * (-2.0 * diff[:, :, d] ** 2 / ell[d] ** 3) for d in range(len(ell))])
        if isinstance(k, O.RationalQuadratic):
            out["alpha"] = K * (u / (1.0 + u) - np.log1p(u))
        if with_z:
            for j, c in enumerate(cols):
                dZ[c] += dkds * 2.0 * diff[:, :, j] / ell_d[j] ** 2
            out["Z"] = dZ
        return out
    if isinstance(k, O.Linear):
        v = np.asarray(k.variance, dtype=np.float64)
        lin = (Zs * v) @ Xs.T
        if isinstance(k, O.Polynomial):
            deg = float(k.degree)
            dbase = deg * (lin + float(k.offset)) ** (deg - 1.0)
        else:
            dbase = np.ones_like(lin)
        out = {"variance": dbase * (Zs @ Xs.T) if v.ndim == 0 else
               np.stack([dbase * np.outer(Zs[:, d], Xs[:, d]) for d in range(Zs.shape[1])])}
        if isinstance(k, O.Polynomial):
            out["offset"] = dbase
        if with_z:
            vd = np.broadcast_to(v, (len(cols),)) if v.ndim else np.full(len(cols), float(v))
            for j, c in enumerate(cols):
                dZ[c] += dbase * vd[j] * Xs[None, :, j]
            out["Z"] = dZ
        return out
    if isinstance(k, (O.White, O.Constant)):
        out = {"variance": np.zeros((M, N)) if isinstance(k, O.White) else np.ones((M, N))}
        if with_z:
            out["Z"] = dZ
        return out
    raise NotImplementedError(type(k).__name__)


def _leaf_dKdiag(k: O.Kernel, X: np.ndarray) -> Dict[str, np.ndarray]:
    """d k(x_n, x_n) / d(parameter) of one leaf, [N] (per-dimension parameters: [D_active, N])."""
    N = X.shape[0]
    Xs = k.slice(X)[0]
    if isinstance(k, O.Stationary):
        ell = np.asarray(k.lengthscales, dtype=np.float64)
        out = {"variance": np.ones(N), "lengthscales": np.zeros(N) if ell.ndim == 0 else np.zeros((ell.shape[0], N))}
        if isinstance(k, O.RationalQuadratic):
            out["alpha"] = np.zeros(N)
        return out
    if isinstance(k, O.Linear):
        v = np.asarray(k.variance, dtype=np.float64)
        lin = np.sum(Xs * Xs * v, axis=1)
        if isinstance(k, O.Polynomial):
            deg = float(k.degree)
            dbase = deg * (lin + float(k.offset)) ** (deg - 1.0)
        else:
            dbase = np.ones(N)
        out = {"variance": dbase * np.sum(Xs * Xs, axis=1) if v.ndim == 0 else (Xs * Xs).T * dbase[None]}
        if isinstance(k, O.Polynomial):
            out["offset"] = dbase
        return out
    if isinstance(k, (O.White, O.Constant)):
        return {"variance": np.ones(N)}
    raise NotImplementedError(type(k).__name__)


def _walk(kernel: O.Kernel, A: np.ndarray, value, dleaf, per_leaf: List[Dict[str, np.ndarray]]) -> None:
    """The product rule: A = d root / d (this node's matrix), elementwise; `value(k)` is a node's matrix, `dleaf(k)` a
    leaf's derivative dict.  Appends, per leaf in device order, {name: G-weighted derivative stack (A applied)}."""
    if isinstance(kernel, O.Sum):
        for c in kernel.kernels:
            _walk(c, A, value, dleaf, per_leaf)
        return
    if isinstance(kernel, O.Product):
        mats = [value(c) for c in kernel.kernels]
        for i, c in enumerate(kernel.kernels):
            others = np.ones_like(A)
            for j, m in enumerate(mats):
                if j != i:
                    others = others * m
            _walk(c, A * others, value, dleaf, per_leaf)
        return
    per_leaf.append({name: A * d for name, d in dleaf(kernel).items()})


def _reduce(G: np.ndarray, stacks: List[Dict[str, np.ndarray]], absolute: bool = False) -> List[Dict[str, object]]:
    """Per leaf {name: sum G (.) stack} (or, `absolute`, sum |G (.) stack|) from _walk's stacks, "Z" left out."""
    f = np.abs if absolute else (lambda a: a)
    out = []
    for st in stacks:
        g = {}
        for name, d in st.items():
            if name == "Z":
                continue
            g[name] = float(np.sum(f(G * d))) if d.ndim == G.ndim else np.array([np.sum(f(G * e)) for e in d])
        out.append(g)
    return out


def sgpr_elbo_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, Z: np.ndarray, s2: float,
                            mean_function=None, jitter: float = O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The SGPR ELBO (sgpr.py:214-289) and its gradient for any Sum / Product expression of the fused leaves, the
    Constant / Linear mean functions and the inducing points.  Returns (elbo, {"leaves": [per leaf in `leaves()` order:
    {"variance", "lengthscales", "alpha", "offset"} as the leaf has them], "noise_variance": float,
    "mean": {"c"} or {"A", "b"} or {}, "Z": [M, D]})."""
    N, P = Y.shape
    M, D = Z.shape
    s = float(s2)
    Yc = Y - O._mean(mean_function, X, P)
    L = O.cholesky(O.Kuu(Z, kernel, jitter=jitter))
    Ap = O.tri_solve(L, O.Kuf(Z, kernel, X))                       # A' = L^-1 Kuf
    B = np.eye(M) + Ap @ Ap.T / s
    LB = O.cholesky(B)
    c = O.tri_solve(LB, Ap @ Yc / s)
    v = O.tri_solve(LB, c, trans=True)
    Linv = O.tri_solve(L, np.eye(M))
    Binv = np.linalg.inv(B)
    I = np.eye(M)
    W = 0.5 * P * (I - Binv) - 0.5 * P * (B - I) - 0.5 * v @ v.T
    H = (P / s) * (I - Binv) - v @ v.T / s
    Guu = Linv.T @ W @ Linv
    Guf = Linv.T @ (H @ Ap + v @ Yc.T / s)
    Gdiag = np.full(N, -P / (2.0 * s))
    elbo = O.sgpr_elbo(X, Y, kernel, Z, s, mean_function=mean_function, jitter=jitter)

    uu: List[Dict[str, np.ndarray]] = []
    uf: List[Dict[str, np.ndarray]] = []
    dg: List[Dict[str, np.ndarray]] = []

    def dleaf_uu(k):
        d = _leaf_dK(k, Z)
        d["Z"] = _leaf_dK_cross(k, Z, Z)["Z"]
        return d

    _walk(kernel, np.ones((M, M)), lambda k: k(Z), dleaf_uu, uu)
    _walk(kernel, np.ones((M, N)), lambda k: k(Z, X), lambda k: _leaf_dK_cross(k, Z, X), uf)
    _walk(kernel, np.ones(N), lambda k: k(X, full_cov=False), lambda k: _leaf_dKdiag(k, X), dg)
    per_leaf = []
    for a, b, d in zip(_reduce(Guu, uu), _reduce(Guf, uf), _reduce(Gdiag, dg)):
        per_leaf.append({name: a[name] + b[name] + d[name] for name in a})
    dZ = np.zeros((M, D))
    for st in uf:
        dZ += np.einsum("mn,dmn->md", Guf, st["Z"])
    for st in uu:
        dZ += 2.0 * np.einsum("ij,dij->id", Guu, st["Z"])

    trace_k = np.sum(kernel(X, full_cov=False)) / s
    trace_q = np.sum(Ap * Ap) / s
    dnoise = (-N * P + P * (M - np.trace(Binv)) + P * trace_k - P * trace_q + np.sum(Yc * Yc) / s
              - np.sum(c * c) - np.sum(v * v)) / (2.0 * s)
    dm = (Yc - Ap.T @ v) / s
    return elbo, {"leaves": per_leaf, "noise_variance": float(dnoise), "mean": _mean_grads(mean_function, X, dm),
                  "Z": dZ}


def _mean_grads(mean_function, X: np.ndarray, dm: np.ndarray) -> Dict[str, np.ndarray]:
    """The Constant / Linear mean function's parameter gradients from dF/dm [N, P]: {"c"} or {"A", "b"} or {}."""
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = dm.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = dm.sum(0)
        rhs = dm.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else dm
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    return mean
