"""Gradient oracle for GPR with any fused kernel expression (test infrastructure, like oracle/gp_grad_oracle.py; not
imported by the product): the target of gpk_gpr_lml_grad_expr and of the Constant / Linear mean-function gradients.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/gpr.py:91-107.  The closed form
restated here is dLML/dtheta = sum_ij G_ij dK_ij/dtheta, G = 1/2 (alpha alpha^T - P K^-1), alpha = K^-1 (Y - m), with the
expression's dK/d(leaf) by the product rule of tests/kernel_grad_oracle.py and dLML/dm = alpha.  It is pinned by central
finite differences of oracle/gp_oracle.py::gpr_log_marginal_likelihood in tests/test_oracle_grad_expr.py.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests import kernel_grad_oracle as KG


def gpr_lml_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, noise_variance: float,
                          mean_function=None, abs_sums: bool = False) -> Tuple[float, Dict[str, object]]:
    """LML (gpr.py:91-107) and its gradient for any Sum / Product expression of RBF, Matern12/32/52, Exponential,
    RationalQuadratic, Linear, Polynomial, White and Constant leaves (scalar or ARD, with active_dims), and the
    Constant / Linear mean functions.  dLML/dtheta = sum_ij G_ij dK_ij/dtheta with G = 1/2 (alpha alpha^T - P K^-1); the
    expression's dK/d(leaf) follows the product rule (Sum: the upstream adjoint; Product: times the other children).
    Returns (lml, {"leaves": [per leaf in `leaves()` order: {"variance", "lengthscales", "alpha", "offset"} as the leaf
    has them], "noise_variance": float, "mean": {"c"} or {"A", "b"} or {}}).  With `abs_sums` also "leaves_abs" (the
    same layout) and "noise_abs": per slot S = sum_ij |G_ij A_ij dK_ij/dtheta| (A the leaf's adjoint), the scale that
    the rounding of the sum and of G is relative to."""
    N, P = Y.shape
    Kx = kernel(X)
    L = O.cholesky(O.add_noise_cov(Kx, noise_variance))
    mu = O._mean(mean_function, X, P)
    lml = float(np.sum(O.multivariate_normal(Y, mu, L)))
    alpha = O.tri_solve(L, O.tri_solve(L, Y - mu), trans=True)
    Linv = O.tri_solve(L, np.eye(N, dtype=X.dtype))
    G = 0.5 * (alpha @ alpha.T - P * (Linv.T @ Linv))
    per_leaf, per_leaf_abs = KG.weighted_leaf_grads(kernel, G, lambda k: k(X), lambda k: KG.leaf_dK(k, X), abs_sums)
    out = {"leaves": per_leaf, "noise_variance": float(np.trace(G)), "mean": KG.mean_grads(mean_function, X, alpha)}
    if abs_sums:
        out["leaves_abs"] = per_leaf_abs
        out["noise_abs"] = float(np.sum(np.abs(np.diag(G))))
    return lml, out
