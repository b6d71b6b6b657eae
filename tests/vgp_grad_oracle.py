"""Gradient oracle for the VGP ELBO with any fused kernel expression (test infrastructure, like
tests/svgp_grad_oracle.py; not imported by the product): the target of gpk_vgp_elbo_grad.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/vgp.py:111-143.  The closed forms
restated here, with s the noise variance, w = -1/(2s), Yc = Y - m(X), K = k(X) + jitter I = L L^T, m = q_mu [N, P],
S_p = tril(q_sqrt[p]), Sig = sum_p S_p S_p^T, R = (Yc - L m) / s, Phi(T) = tril(T) with its diagonal halved and
sym(T) = (T + T^T) / 2:

    Lbar     = tril(R m^T + 2w L Sig)                      (dF/dL)
    dF/dK    = sym(L^-T Phi(L^T Lbar) L^-1)                (the Cholesky adjoint; the jitter carries no parameter)
    dF/dq_mu = L^T R - m
    dF/dS_p  = tril(2w (L^T L) S_p - S_p) + diag(1 / diag S_p)
    dF/ds    = sum_np [-1/(2s) + ((Yc - L m)^2 + fvar) / (2 s^2)],   dF/dm(X) = R

The kernel parameters follow from sum_ij dF/dK_ij dK_ij/dtheta over the N x N square, the diagonal included, by the
product rule of tests/sgpr_grad_oracle.py.  Pinned by central finite differences of oracle/gp_oracle.py::vgp_elbo in
tests/test_oracle_vgp_grad.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests.grad_expr_oracle import _leaf_dK, leaves  # noqa: F401  (leaves: the device's leaf order, re-exported)
from tests.sgpr_grad_oracle import _reduce, _walk
from tests.svgp_grad_oracle import _phi, _sym


def vgp_elbo_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, q_mu: np.ndarray, q_sqrt: np.ndarray,
                           s2: float, *, mean_function=None,
                           jitter: float = O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The VGP ELBO (vgp.py:111-143) and its gradient for any Sum / Product expression of the fused leaves, the
    Constant / Linear mean functions and the variational parameters.  q_mu [N, P], q_sqrt [P, N, N] (its strict upper
    part is not read).  Returns (elbo, {"leaves": [per leaf in `leaves()` order], "noise_variance": float,
    "mean": {"c"} or {"A", "b"} or {}, "q_mu": [N, P], "q_sqrt": [P, N, N], "K": dF/dK [N, N]})."""
    N, P = Y.shape
    s = float(s2)
    w = -1.0 / (2.0 * s)
    Yc = Y - O._mean(mean_function, X, P)
    L = O.cholesky(kernel(X) + jitter * np.eye(N))
    Linv = O.tri_solve(L, np.eye(N))
    S = np.tril(q_sqrt)
    Sig = sum(S[p] @ S[p].T for p in range(P))
    Fm = L @ q_mu
    fvar = np.stack([np.sum((L @ S[p]) ** 2, 1) for p in range(P)], 1)
    R = (Yc - Fm) / s
    Lbar = np.tril(R @ q_mu.T + 2.0 * w * L @ Sig)
    GK = _sym(Linv.T @ _phi(L.T @ Lbar) @ Linv)
    LtL = L.T @ L
    dq_mu = L.T @ R - q_mu
    dq_sqrt = np.stack([np.tril(2.0 * w * LtL @ S[p] - S[p]) + np.diag(1.0 / np.diag(S[p])) for p in range(P)])
    stacks: List[Dict[str, np.ndarray]] = []
    _walk(kernel, np.ones((N, N)), lambda k: k(X), lambda k: _leaf_dK(k, X), stacks)
    per_leaf = _reduce(GK, stacks)
    dnoise = np.sum(-0.5 / s + ((Yc - Fm) ** 2 + fvar) / (2.0 * s * s))
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = R.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = R.sum(0)
        rhs = R.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else R
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    elbo = O.vgp_elbo(X, Y, kernel, q_mu, q_sqrt, s, mean_function=mean_function, jitter=jitter)
    return elbo, {"leaves": per_leaf, "noise_variance": float(dnoise), "mean": mean, "q_mu": dq_mu,
                  "q_sqrt": dq_sqrt, "K": GK}
