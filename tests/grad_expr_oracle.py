"""Gradient oracle for GPR with any fused kernel expression (test infrastructure, like oracle/gp_grad_oracle.py; not
imported by the product): the target of gpk_gpr_lml_grad_expr and of the Constant / Linear mean-function gradients.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/gpr.py:91-107.  The closed form
restated here is dLML/dtheta = sum_ij G_ij dK_ij/dtheta, G = 1/2 (alpha alpha^T - P K^-1), alpha = K^-1 (Y - m), with the
expression's dK/d(leaf) by the product rule and dLML/dm = alpha.  It is pinned by central finite differences of
oracle/gp_oracle.py::gpr_log_marginal_likelihood in tests/test_oracle_grad_expr.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from oracle.gp_grad_oracle import stationary_dK

# ----------------------------------------------------------------------------------------------------------------------
# any expression of the fused leaves (target of gpk_gpr_lml_grad_expr)
# ----------------------------------------------------------------------------------------------------------------------
def _leaf_dK(k: O.Kernel, X: np.ndarray) -> Dict[str, np.ndarray]:
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


def leaves(kernel: O.Kernel) -> List[O.Kernel]:
    """Leaves of an expression in the order the device numbers them (depth first, left to right)."""
    if isinstance(kernel, O.Combination):
        return [leaf for c in kernel.kernels for leaf in leaves(c)]
    return [kernel]


def gpr_lml_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, noise_variance: float,
                          mean_function=None) -> Tuple[float, Dict[str, object]]:
    """LML (gpr.py:91-107) and its gradient for any Sum / Product expression of RBF, Matern12/32/52, Exponential,
    RationalQuadratic, Linear, Polynomial, White and Constant leaves (scalar or ARD, with active_dims), and the
    Constant / Linear mean functions.  dLML/dtheta = sum_ij G_ij dK_ij/dtheta with G = 1/2 (alpha alpha^T - P K^-1); the
    expression's dK/d(leaf) follows the product rule (Sum: the upstream adjoint; Product: times the other children).
    Returns (lml, {"leaves": [per leaf in `leaves()` order: {"variance", "lengthscales", "alpha", "offset"} as the leaf
    has them], "noise_variance": float, "mean": {"c"} or {"A", "b"} or {}})."""
    N, P = Y.shape
    Kx = kernel(X)
    L = O.cholesky(O.add_noise_cov(Kx, noise_variance))
    mu = O._mean(mean_function, X, P)
    lml = float(np.sum(O.multivariate_normal(Y, mu, L)))
    alpha = O.tri_solve(L, O.tri_solve(L, Y - mu), trans=True)
    Linv = O.tri_solve(L, np.eye(N, dtype=X.dtype))
    G = 0.5 * (alpha @ alpha.T - P * (Linv.T @ Linv))
    per_leaf: List[Dict[str, object]] = []

    def walk(k: O.Kernel, A: np.ndarray) -> None:   # A = d root / d (this node's matrix), elementwise
        if isinstance(k, O.Sum):
            for c in k.kernels:
                walk(c, A)
            return
        if isinstance(k, O.Product):
            mats = [c(X) for c in k.kernels]
            for i, c in enumerate(k.kernels):
                others = np.ones_like(A)
                for j, m in enumerate(mats):
                    if j != i:
                        others = others * m
                walk(c, A * others)
            return
        GA = G * A
        g = {}
        for name, dK in _leaf_dK(k, X).items():
            g[name] = float(np.sum(GA * dK)) if dK.ndim == 2 else np.array([np.sum(GA * d) for d in dK])
        per_leaf.append(g)

    walk(kernel, np.ones((N, N)))
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = alpha.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = alpha.sum(0)
        rhs = alpha.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else alpha
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    return lml, {"leaves": per_leaf, "noise_variance": float(np.trace(G)), "mean": mean}
