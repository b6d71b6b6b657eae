"""Kernel-gradient building blocks shared by the model gradient oracles (test infrastructure; not imported by the
product): the device's leaf order, each fused leaf's dK/d(parameter) over a square, a cross block and a diagonal, the
product rule through Sum / Product, the reductions sum_ij G_ij dK_ij/dtheta, dF/dZ, the Cholesky-adjoint helpers phi and
sym, and the Constant / Linear mean-function gradients.

The model oracles (tests/grad_expr_oracle.py, sgpr_grad_oracle.py, svgp_grad_oracle.py, vgp_grad_oracle.py,
vgp_oa_grad_oracle.py, cglb_grad_oracle.py, natgrad_oracle.py) build on these; each is pinned by central finite
differences in its tests/test_oracle_*.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from oracle.gp_grad_oracle import stationary_dK


def leaves(kernel: O.Kernel) -> List[O.Kernel]:
    """Leaves of an expression in the order the device numbers them (depth first, left to right)."""
    if isinstance(kernel, O.Combination):
        return [leaf for c in kernel.kernels for leaf in leaves(c)]
    return [kernel]


def phi(T: np.ndarray) -> np.ndarray:
    """tril(T) with its diagonal halved."""
    return np.tril(T, -1) + 0.5 * np.diag(np.diag(T))


def sym(T: np.ndarray) -> np.ndarray:
    return 0.5 * (T + T.T)


def leaf_dK(k: O.Kernel, X: np.ndarray) -> Dict[str, np.ndarray]:
    """dK/d(parameter) of one leaf on the unsliced X (the leaf slices its own active_dims).  Per-dimension parameters
    (ARD lengthscales, ARD Linear / Polynomial variances) give a [D_active, N, N] stack."""
    Xs = k.slice(X)[0]
    if isinstance(k, O.RationalQuadratic):
        K = k(X)
        var, a = float(k.variance), float(k.alpha)
        ell = np.asarray(k.lengthscales, dtype=np.float64)
        r2 = np.maximum(k.scaled_squared_euclid_dist(Xs), 0.0)
        u = r2 / (2.0 * a)
        dkds = -0.5 * K / (1.0 + u)
        if ell.ndim == 0:
            dl = dkds * (-2.0 * r2 / float(ell))
        else:
            diff2 = (Xs[:, None, :] - Xs[None, :, :]) ** 2
            dl = np.stack([dkds * (-2.0 * diff2[:, :, d] / ell[d] ** 3) for d in range(ell.shape[0])])
        return {"variance": K / var, "lengthscales": dl, "alpha": K * (u / (1.0 + u) - np.log1p(u))}
    if isinstance(k, O.Stationary):
        return stationary_dK(k, X)
    if isinstance(k, O.Linear):
        v = np.asarray(k.variance, dtype=np.float64)
        outer = np.stack([np.outer(Xs[:, d], Xs[:, d]) for d in range(Xs.shape[1])])   # [D, N, N]
        lin = (Xs * v) @ Xs.T
        if isinstance(k, O.Polynomial):
            deg = float(k.degree)
            dbase = deg * (lin + float(k.offset)) ** (deg - 1.0)
        else:
            dbase = np.ones_like(lin)
        dv = dbase * (Xs @ Xs.T) if v.ndim == 0 else dbase[None] * outer
        out = {"variance": dv}
        if isinstance(k, O.Polynomial):
            out["offset"] = dbase
        return out
    if isinstance(k, O.White):
        return {"variance": np.eye(X.shape[0])}
    if isinstance(k, O.Constant):
        return {"variance": np.ones((X.shape[0], X.shape[0]))}
    raise NotImplementedError(type(k).__name__)


def _cols(k: O.Kernel, D: int) -> np.ndarray:
    """The input columns a leaf reads, in its active-dims order."""
    return np.arange(D)[k.active_dims] if isinstance(k.active_dims, slice) else np.asarray(k.active_dims, dtype=int)


def leaf_dK_cross(k: O.Kernel, Z: np.ndarray, X: np.ndarray, with_z: bool = True) -> Dict[str, np.ndarray]:
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


def leaf_dKdiag(k: O.Kernel, X: np.ndarray) -> Dict[str, np.ndarray]:
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


def walk(kernel: O.Kernel, A: np.ndarray, value, dleaf, per_leaf: List[Dict[str, np.ndarray]]) -> None:
    """The product rule: A = d root / d (this node's matrix), elementwise; `value(k)` is a node's matrix, `dleaf(k)` a
    leaf's derivative dict.  Appends, per leaf in device order, {name: G-weighted derivative stack (A applied)}."""
    if isinstance(kernel, O.Sum):
        for c in kernel.kernels:
            walk(c, A, value, dleaf, per_leaf)
        return
    if isinstance(kernel, O.Product):
        mats = [value(c) for c in kernel.kernels]
        for i, c in enumerate(kernel.kernels):
            others = np.ones_like(A)
            for j, m in enumerate(mats):
                if j != i:
                    others = others * m
            walk(c, A * others, value, dleaf, per_leaf)
        return
    per_leaf.append({name: A * d for name, d in dleaf(kernel).items()})


def reduce(G: np.ndarray, stacks: List[Dict[str, np.ndarray]], absolute: bool = False) -> List[Dict[str, object]]:
    """Per leaf {name: sum G (.) stack} (or, `absolute`, sum |G (.) stack|) from walk's stacks, "Z" left out."""
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


def weighted_leaf_grads(kernel: O.Kernel, G: np.ndarray, value, dleaf, abs_sums: bool = False
                        ) -> Tuple[List[Dict[str, object]], List[Dict[str, object]]]:
    """sum_ij G_ij dK_ij/dtheta per leaf slot by the product rule (Sum: the upstream adjoint; Product: times the other
    children), on whatever block of K the weight G covers: `value(k)` is a node's matrix on that block and `dleaf(k)`
    a leaf's derivative dict (per-dimension parameters as a [D_active, ...] stack).  Returns (per leaf in `leaves()`
    order {name: float or [D_active]}, the same layout of sum_ij |G_ij A_ij dK_ij/dtheta| with `abs_sums`, else empty
    dicts), A the leaf's adjoint from the product rule."""
    per_leaf: List[Dict[str, object]] = []
    per_leaf_abs: List[Dict[str, object]] = []

    def visit(k: O.Kernel, A: np.ndarray) -> None:   # A = d root / d (this node's matrix), elementwise
        if isinstance(k, O.Sum):
            for c in k.kernels:
                visit(c, A)
            return
        if isinstance(k, O.Product):
            mats = [value(c) for c in k.kernels]
            for i, c in enumerate(k.kernels):
                others = np.ones_like(A)
                for j, m in enumerate(mats):
                    if j != i:
                        others = others * m
                visit(c, A * others)
            return
        GA = G * A
        g, ga = {}, {}
        for name, dK in dleaf(k).items():
            g[name] = float(np.sum(GA * dK)) if dK.ndim == G.ndim else np.array([np.sum(GA * d) for d in dK])
            if abs_sums:
                ga[name] = float(np.sum(np.abs(GA * dK))) if dK.ndim == G.ndim else np.array([np.sum(np.abs(GA * d))
                                                                                            for d in dK])
        per_leaf.append(g)
        per_leaf_abs.append(ga)

    visit(kernel, np.ones_like(G))
    return per_leaf, per_leaf_abs


def inducing_stacks(kernel: O.Kernel, X: np.ndarray, Z: np.ndarray):
    """walk's stacks over Kuu (with "Z": d k(z_i, z_j) / d z_i), Kuf and the diagonal of K(X, X)."""
    M, N = Z.shape[0], X.shape[0]
    uu: List[Dict[str, np.ndarray]] = []
    uf: List[Dict[str, np.ndarray]] = []
    dg: List[Dict[str, np.ndarray]] = []

    def dleaf_uu(k):
        d = leaf_dK(k, Z)
        d["Z"] = leaf_dK_cross(k, Z, Z)["Z"]
        return d

    walk(kernel, np.ones((M, M)), lambda k: k(Z), dleaf_uu, uu)
    walk(kernel, np.ones((M, N)), lambda k: k(Z, X), lambda k: leaf_dK_cross(k, Z, X), uf)
    walk(kernel, np.ones(N), lambda k: k(X, full_cov=False), lambda k: leaf_dKdiag(k, X), dg)
    return uu, uf, dg


def kernel_and_z_grads(kernel: O.Kernel, X: np.ndarray, Z: np.ndarray, Guu: np.ndarray, Guf: np.ndarray,
                       Gdiag: np.ndarray) -> Tuple[List[Dict[str, object]], np.ndarray]:
    """Per leaf (in `leaves()` order) {parameter: sum G (.) dK/dparameter} over Kuu, Kuf and the diagonal of K(X, X), and
    dF/dZ [M, D] (G_uu symmetric)."""
    uu, uf, dg = inducing_stacks(kernel, X, Z)
    per_leaf = []
    for a, b, d in zip(reduce(Guu, uu), reduce(Guf, uf), reduce(Gdiag, dg)):
        per_leaf.append({name: a[name] + b[name] + d[name] for name in a})
    dZ = np.zeros(Z.shape)
    for st in uf:
        dZ += np.einsum("mn,dmn->md", Guf, st["Z"])
    for st in uu:
        dZ += 2.0 * np.einsum("ij,dij->id", Guu, st["Z"])
    return per_leaf, dZ


def mean_grads(mean_function, X: np.ndarray, dm: np.ndarray) -> Dict[str, np.ndarray]:
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
