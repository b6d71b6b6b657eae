"""Forward oracle of the Bayesian GPLVM (test infrastructure, not imported by the product): the RBF psi statistics by
the reference's Cholesky formulas (gpflow/expectations/squared_exponentials.py:49-96, 207-292, here with a diagonal
covariance), the bound of gpflow/models/gplvm.py:162-216 and its predict_f (:218-274), in NumPy float64."""
from __future__ import annotations

import numpy as np

from oracle import gp_oracle as O


def _cols(kernel: O.SquaredExponential, Q: int) -> np.ndarray:
    return np.arange(Q)[kernel.active_dims] if isinstance(kernel.active_dims, slice) else np.asarray(kernel.active_dims)


def _lengthscales(kernel: O.SquaredExponential, nd: int) -> np.ndarray:
    return np.broadcast_to(np.asarray(kernel.lengthscales, dtype=np.float64), (nd,)).copy()


def psi_statistics(mu, S, Z, kernel):
    """(psi0, psi1 [N, M], psi2 [M, M] summed over n) of q(x_n) = N(mu_n, diag S_n)."""
    cols = _cols(kernel, mu.shape[1])
    mu, S, Z = mu[:, cols], S[:, cols], Z[:, cols]
    N, M = mu.shape[0], Z.shape[0]
    lam = np.diag(_lengthscales(kernel, len(cols)) ** 2)
    var = float(kernel.variance)
    psi1 = np.empty((N, M))
    psi2 = np.zeros((M, M))
    zbar = 0.5 * (Z[:, None, :] + Z[None, :, :])
    dz = Z[:, None, :] - Z[None, :, :]
    Llam = np.linalg.cholesky(lam)
    t = np.linalg.solve(Llam, dz.reshape(-1, len(cols)).T)
    ez = np.exp(-0.25 * np.sum(t * t, axis=0)).reshape(M, M)       # exp(-1/4 (z - z')^T Lambda^-1 (z - z'))
    for n in range(N):
        Sn = np.diag(S[n])
        L1 = np.linalg.cholesky(lam + Sn)                             # squared_exponentials.py:73-88
        v = np.linalg.solve(L1, (mu[n][None, :] - Z).T)
        det1 = np.prod(np.diag(Llam)) / np.prod(np.diag(L1))
        psi1[n] = var * det1 * np.exp(-0.5 * np.sum(v * v, axis=0))
        L2 = np.linalg.cholesky(0.5 * lam + Sn)                       # squared_exponentials.py:249-290
        w = np.linalg.solve(L2, (zbar - mu[n]).reshape(-1, len(cols)).T)
        det2 = np.prod(np.diag(np.linalg.cholesky(0.5 * lam))) / np.prod(np.diag(L2))
        psi2 += var * var * det2 * ez * np.exp(-0.5 * np.sum(w * w, axis=0)).reshape(M, M)
    return N * var, psi1, psi2


def kl(mu, S, m0, p0) -> float:
    """KL[q(X) || p(X)] (gplvm.py:195-204)."""
    return float(np.sum(0.5 * np.log(p0 / S) - 0.5 + ((mu - m0) ** 2 + S) / (2.0 * p0)))


def _terms(Y, mu, S, Z, kernel, noise, jitter):
    psi0, psi1, psi2 = psi_statistics(mu, S, Z, kernel)
    M = Z.shape[0]
    L = np.linalg.cholesky(O.Kuu(Z, kernel, jitter=jitter))
    A = O.tri_solve(L, psi1.T)
    tmp = O.tri_solve(L, psi2)
    AAT = O.tri_solve(L, tmp.T) / noise
    B = AAT + np.eye(M)
    LB = np.linalg.cholesky(B)
    c = O.tri_solve(LB, A @ Y) / noise
    return psi0, L, LB, AAT, c


def bgplvm_elbo(Y, mu, S, Z, kernel, noise, m0=None, p0=None, jitter=O.DEFAULT_JITTER) -> float:
    m0 = np.zeros_like(mu) if m0 is None else m0
    p0 = np.ones_like(mu) if p0 is None else p0
    psi0, _, LB, AAT, c = _terms(Y, mu, S, Z, kernel, noise, jitter)
    N, P = Y.shape
    bound = -0.5 * N * P * np.log(2 * np.pi * noise)
    bound += -P * np.sum(np.log(np.diag(LB)))
    bound += -0.5 * np.sum(Y * Y) / noise
    bound += 0.5 * np.sum(c * c)
    bound += -0.5 * P * (psi0 / noise - np.trace(AAT))
    return float(bound - kl(mu, S, m0, p0))


def bgplvm_predict_f(Y, mu, S, Z, kernel, noise, Xnew, full_cov=False, jitter=O.DEFAULT_JITTER):
    _, L, LB, _, c = _terms(Y, mu, S, Z, kernel, noise, jitter)
    P = Y.shape[1]
    tmp1 = O.tri_solve(L, O.Kuf(Z, kernel, Xnew))
    tmp2 = O.tri_solve(LB, tmp1)
    mean = tmp2.T @ c
    if full_cov:
        var = kernel(Xnew) + tmp2.T @ tmp2 - tmp1.T @ tmp1
        return mean, np.tile(var[None], (P, 1, 1))
    var = kernel(Xnew, full_cov=False) + np.sum(tmp2 ** 2, axis=0) - np.sum(tmp1 ** 2, axis=0)
    return mean, np.tile(var[:, None], (1, P))
