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

and dF/dtheta = sum G (.) dK/dtheta over the three matrices, each leaf's dK by the product rule of kernel_grad_oracle.
dF/dZ adds sum_n G_uf[m, n] dk(z_m, x_n)/dz_m and 2 sum_j G_uu[i, j] dk(z_i, z_j)/dz_i (G_uu is symmetric).  Pinned by
central finite differences of oracle/gp_oracle.py::sgpr_elbo in tests/test_oracle_sgpr_grad.py.
"""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests import kernel_grad_oracle as KG


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

    per_leaf, dZ = KG.kernel_and_z_grads(kernel, X, Z, Guu, Guf, Gdiag)

    trace_k = np.sum(kernel(X, full_cov=False)) / s
    trace_q = np.sum(Ap * Ap) / s
    dnoise = (-N * P + P * (M - np.trace(Binv)) + P * trace_k - P * trace_q + np.sum(Yc * Yc) / s
              - np.sum(c * c) - np.sum(v * v)) / (2.0 * s)
    dm = (Yc - Ap.T @ v) / s
    return elbo, {"leaves": per_leaf, "noise_variance": float(dnoise), "mean": KG.mean_grads(mean_function, X, dm),
                  "Z": dZ}


def optimal_q(X, Y, kernel, Z, s2, whiten, jitter=O.DEFAULT_JITTER):
    """q* of the collapsed bound (sgpr.py:346-377) as SVGP variational parameters: mean [M, P] and dense q_sqrt
    [P, M, M]; whitened through L (q_mu = L^-1 mu, q_sqrt = chol(L^-1 cov L^-T))."""
    P = Y.shape[1]
    mu, cov = O.sgpr_compute_qu(X, Y, kernel, Z, s2, jitter=jitter)
    if whiten:
        L = O.cholesky(O.Kuu(Z, kernel, jitter=jitter))
        mu = O.tri_solve(L, mu)
        cov = O.tri_solve(L, O.tri_solve(L, cov).T)
    Lq = O.cholesky(0.5 * (cov + cov.T))
    return mu, np.stack([Lq] * P)
