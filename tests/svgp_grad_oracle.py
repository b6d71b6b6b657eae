"""Gradient oracle for the SVGP ELBO with any fused kernel expression (test infrastructure, like
tests/sgpr_grad_oracle.py; not imported by the product): the target of gpk_svgp_elbo_grad.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/svgp.py:166-181.  The closed forms
restated here, with s the noise variance, c = num_data / B (1 without num_data), w = -c / (2s), Yc = Y - m(X),
K = Kuu + jitter I = L L^T, S_p = tril(q_sqrt[p]), m = q_mu [M, P], Sig = sum_p S_p S_p^T, A = L^-1 Kuf (whiten) or
K^-1 Kuf, Fm = A^T m, R = c (Yc - Fm) / s, Phi(T) = tril(T) with its diagonal halved and sym(T) = (T + T^T) / 2:

  whiten:     Abar = m R^T + 2w (Sig - P I) A
              dF/dKuf = L^-T Abar,   dF/dKuu = -sym(L^-T Phi(Abar A^T) L^-1)   (the Cholesky adjoint)
              dF/dq_mu = A R - m,    dF/dS_p = tril(2w (A A^T) S_p - S_p) + diag(1 / diag S_p)
  otherwise:  Abar = m R^T + 2w Sig A
              dF/dKuf = K^-1 Abar - 2wP A
              dF/dKuu = sym(-K^-1 Abar A^T) + wP A A^T + 1/2 K^-1 (m m^T + Sig) K^-1 - P/2 K^-1
              dF/dq_mu = A R - K^-1 m,   dF/dS_p = tril(2w (A A^T) S_p - K^-1 S_p) + diag(1 / diag S_p)
  both:       dF/dKdiag = P w,   dF/ds = c sum_np [-1/(2s) + ((Yc - Fm)^2 + fvar) / (2 s^2)],   dF/dm(X) = R

With q_diag the q_sqrt forms restricted to the diagonal (Sig = diag(sum_p s_p^2)).  The kernel parameters and Z follow
from dF/dKuu, dF/dKuf and dF/dKdiag exactly as in tests/sgpr_grad_oracle.py.  Pinned by central finite differences of
oracle/gp_oracle.py::svgp_elbo in tests/test_oracle_svgp_grad.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests.grad_expr_oracle import _leaf_dK, leaves  # noqa: F401  (leaves: the device's leaf order, re-exported)
from tests.sgpr_grad_oracle import _leaf_dK_cross, _leaf_dKdiag, _reduce, _walk


def _phi(T: np.ndarray) -> np.ndarray:
    return np.tril(T, -1) + 0.5 * np.diag(np.diag(T))


def _sym(T: np.ndarray) -> np.ndarray:
    return 0.5 * (T + T.T)


def kernel_and_z_grads(kernel: O.Kernel, X: np.ndarray, Z: np.ndarray, Guu: np.ndarray, Guf: np.ndarray,
                       Gdiag: np.ndarray) -> Tuple[List[Dict[str, object]], np.ndarray]:
    """Per leaf (in `leaves()` order) {parameter: sum G (.) dK/dparameter} over Kuu, Kuf and the diagonal of K(X, X), and
    dF/dZ [M, D] (G_uu symmetric)."""
    M, D = Z.shape
    N = X.shape[0]
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
    return per_leaf, dZ


def svgp_elbo_and_grad_expr(X: np.ndarray, Y: np.ndarray, kernel: O.Kernel, Z: np.ndarray, q_mu: np.ndarray,
                            q_sqrt: np.ndarray, s2: float, *, whiten: bool = True, num_data=None, mean_function=None,
                            jitter: float = O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The SVGP ELBO (svgp.py:166-181) on the batch (X, Y) and its gradient for any Sum / Product expression of the fused
    leaves, the Constant / Linear mean functions, the inducing points and the variational parameters.  q_sqrt is
    [P, M, M] or [M, P] (q_diag).  Returns (elbo, {"leaves": [per leaf in `leaves()` order], "noise_variance": float,
    "mean": {"c"} or {"A", "b"} or {}, "Z": [M, D], "q_mu": [M, P], "q_sqrt": the shape of q_sqrt})."""
    B, P = Y.shape
    M, D = Z.shape
    s = float(s2)
    q_diag = q_sqrt.ndim == 2
    c = 1.0 if num_data is None else float(num_data) / B
    w = -c / (2.0 * s)
    Yc = Y - O._mean(mean_function, X, P)
    K = O.Kuu(Z, kernel, jitter=jitter)
    L = O.cholesky(K)
    Kuf = O.Kuf(Z, kernel, X)
    Kd = kernel(X, full_cov=False)
    Linv = O.tri_solve(L, np.eye(M))
    Kinv = Linv.T @ Linv
    S = np.stack([np.diag(q_sqrt[:, p]) for p in range(P)]) if q_diag else np.tril(q_sqrt)
    Sig = sum(S[p] @ S[p].T for p in range(P))
    A = Linv @ Kuf if whiten else Kinv @ Kuf
    Fm = A.T @ q_mu
    if whiten:
        fvar = Kd[:, None] - np.sum(A * A, 0)[:, None] + np.stack([np.sum((S[p].T @ A) ** 2, 0) for p in range(P)], 1)
    else:
        fvar = Kd[:, None] - np.sum(Kuf * A, 0)[:, None] + np.stack([np.sum((S[p].T @ A) ** 2, 0) for p in range(P)], 1)
    R = c * (Yc - Fm) / s
    AAt = A @ A.T
    I = np.eye(M)
    if whiten:
        Abar = q_mu @ R.T + 2.0 * w * (Sig - P * I) @ A
        Guf = Linv.T @ Abar
        Guu = -_sym(Linv.T @ _phi(Abar @ A.T) @ Linv)
        dq_mu = A @ R - q_mu
        KS = S
    else:
        Abar = q_mu @ R.T + 2.0 * w * Sig @ A
        Guf = Kinv @ Abar - 2.0 * w * P * A
        Guu = (_sym(-Kinv @ Abar @ A.T) + w * P * AAt + 0.5 * Kinv @ (q_mu @ q_mu.T + Sig) @ Kinv
               - 0.5 * P * Kinv)
        dq_mu = A @ R - Kinv @ q_mu
        KS = np.stack([Kinv @ S[p] for p in range(P)])
    if q_diag:
        kd = np.ones(M) if whiten else np.diag(Kinv)
        dq_sqrt = 2.0 * w * q_sqrt * np.diag(AAt)[:, None] - kd[:, None] * q_sqrt + 1.0 / q_sqrt
    else:
        dq_sqrt = np.stack([np.tril(2.0 * w * AAt @ S[p] - KS[p]) + np.diag(1.0 / np.diag(S[p])) for p in range(P)])
    Gdiag = np.full(B, P * w)
    per_leaf, dZ = kernel_and_z_grads(kernel, X, Z, Guu, Guf, Gdiag)
    dnoise = c * np.sum(-0.5 / s + ((Yc - Fm) ** 2 + fvar) / (2.0 * s * s))
    dm = R
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = dm.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = dm.sum(0)
        rhs = dm.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else dm
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    elbo = O.svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, s, whiten=whiten, num_data=num_data,
                       mean_function=mean_function, jitter=jitter)
    return elbo, {"leaves": per_leaf, "noise_variance": float(dnoise), "mean": mean, "Z": dZ, "q_mu": dq_mu,
                  "q_sqrt": dq_sqrt}
