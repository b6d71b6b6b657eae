"""Value and gradient oracle for the VGPOpperArchambeau ELBO (test infrastructure, like tests/vgp_grad_oracle.py; not
imported by the product): the target of gpk_vgp_oa_elbo_grad.

The reference obtains these gradients from TensorFlow autodiff through gpflow/models/vgp.py:325-376.  With K = k(X) (no
jitter), alpha = q_alpha [N, P], Lambda_p = diag(q_lambda[:, p]), A_p = I + Lambda_p K Lambda_p, B_p = A_p^-1, the
likelihood's adjoints R = dVE/dfmean and W = dVE/dfvar, D_p = diag(W_p / lambda_p^2) and sym(T) = (T + T^T) / 2:

    Abar_p       = B_p (D_p + 1/2 I) B_p - 1/2 B_p                                       (dF/dA_p)
    dF/dK        = sum_p [sym(R_p alpha_p^T) - 1/2 alpha_p alpha_p^T + Lambda_p Abar_p Lambda_p]
    dF/dalpha    = K (R - alpha),   dF/dm(X) = R
    dF/dlambda_j = -2 W_j (1 - (B_p)_jj) / lambda_j^3 + 2 (K Lambda_p Abar_p)_jj            (the direct form)

The kernel parameters follow from sum_ij dF/dK_ij dK_ij/dtheta over the N x N square by the product rule of
tests/kernel_grad_oracle.py.  `lik` is any likelihood oracle with variational_expectations(mu, v, y) and ve_grads(mu, v,
y) -> (dmu, dv, dpar): tests/lik_oracle.py (Gaussian, Bernoulli, Poisson, StudentT), tests/multiclass_oracle.py and
tests/hetero_oracle.py.  Pinned by central finite differences of `elbo_literal` in tests/test_oracle_vgp_oa_grad.py.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests import kernel_grad_oracle as KG


def elbo_literal(X, Y, kernel, q_alpha, q_lambda, lik, mean_function=None) -> float:
    """vgp.py:343-376 transcribed line by line (the [P, N, N] stacks included)."""
    N, P = q_alpha.shape
    K = kernel(X)
    K_alpha = K @ q_alpha
    f_mean = K_alpha + O._mean(mean_function, X, P)
    I = np.tile(np.eye(N)[None], (P, 1, 1))
    A = I + q_lambda.T[:, None, :] * q_lambda.T[:, :, None] * K
    L = np.linalg.cholesky(A)
    Li = np.stack([np.linalg.solve(L[p], I[p]) for p in range(P)])
    tmp = Li / q_lambda.T[:, None, :]
    f_var = 1.0 / q_lambda ** 2 - np.sum(tmp ** 2, 1).T
    A_logdet = 2.0 * np.sum(np.log(np.diagonal(L, axis1=1, axis2=2)))
    trAi = np.sum(Li ** 2)
    KL = 0.5 * (A_logdet + trAi - N * P + np.sum(K_alpha * q_alpha))
    return float(np.sum(lik.variational_expectations(f_mean, f_var, Y)) - KL)


def moments(X, kernel, q_alpha, q_lambda, mean_function=None):
    """(fmean [N, P], fvar [N, P], [B_p], K) of q(F)."""
    N, P = q_alpha.shape
    K = kernel(X)
    fmean = K @ q_alpha + O._mean(mean_function, X, P)
    Bs, fvar = [], np.empty((N, P))
    for p in range(P):
        lam = q_lambda[:, p]
        Li = O.tri_solve(O.cholesky(np.eye(N) + lam[:, None] * K * lam[None]), np.eye(N))
        Bs.append(Li.T @ Li)
        fvar[:, p] = 1.0 / lam ** 2 - np.sum((Li / lam[None]) ** 2, 0)
    return fmean, fvar, Bs, K


def vgp_oa_elbo_and_grad(X, Y, kernel, q_alpha, q_lambda, lik, *, mean_function=None
                         ) -> Tuple[float, Dict[str, object]]:
    """The ELBO and its gradient: {"leaves": [per leaf in `leaves()` order], "lik": d/d(likelihood parameter) (0 without
    one), "mean": {"c"} or {"A", "b"} or {}, "q_alpha", "q_lambda": [N, P], "K": dF/dK [N, N], "R", "W": [N, P]}."""
    N, P = q_alpha.shape
    fmean, fvar, Bs, K = moments(X, kernel, q_alpha, q_lambda, mean_function)
    R, W, dpar = lik.ve_grads(fmean, fvar, Y)
    GK = np.zeros((N, N))
    dlam = np.empty((N, P))
    for p in range(P):
        lam, a, B = q_lambda[:, p], q_alpha[:, p], Bs[p]
        Abar = B @ np.diag(W[:, p] / lam ** 2 + 0.5) @ B - 0.5 * B
        RA = np.outer(R[:, p], a)
        GK += 0.5 * (RA + RA.T) - 0.5 * np.outer(a, a) + lam[:, None] * Abar * lam[None]
        dlam[:, p] = -2.0 * W[:, p] * (1.0 - np.diag(B)) / lam ** 3 + 2.0 * np.diag(K @ (lam[:, None] * Abar))
    stacks: List[Dict[str, np.ndarray]] = []
    KG.walk(kernel, np.ones((N, N)), lambda k: k(X), lambda k: KG.leaf_dK(k, X), stacks)
    elbo = elbo_literal(X, Y, kernel, q_alpha, q_lambda, lik, mean_function)
    return elbo, {"leaves": KG.reduce(GK, stacks), "lik": float(np.sum(dpar)),
                  "mean": KG.mean_grads(mean_function, X, R),
                  "q_alpha": K @ (R - q_alpha), "q_lambda": dlam, "K": GK, "R": R, "W": W}
