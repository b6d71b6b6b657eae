"""NumPy restatement of gpflow/models/cglb.py: the Nystrom preconditioner, the CG loop line by line (quirks included),
the bound and prediction.  Vectors are [P, N] as in the reference.  Kernels are evaluated through __call__, so leaves
with active_dims slice their inputs."""
from __future__ import annotations

import numpy as np
from scipy.linalg import solve_triangular

LOG2PI = np.log(2.0 * np.pi)


def common(X, Z, ko, s, jitter=1e-6):
    """sgpr.py:181-209 with A = L^-1 Kuf / sigma: (L, A, LB, AAT)."""
    Kuu = ko(Z) + jitter * np.eye(Z.shape[0])
    L = np.linalg.cholesky(Kuu)
    A = solve_triangular(L, ko(Z, X), lower=True) / np.sqrt(s)
    AAT = A @ A.T
    LB = np.linalg.cholesky(AAT + np.eye(Z.shape[0]))
    return L, A, LB, AAT


def precondition(A, LB, s, v):
    """NystromPreconditioner.__call__ (cglb.py:310-340): (v Q^-1 [B, N], sum v Q^-1 v)."""
    vt = v.T
    Av = A @ vt
    t = solve_triangular(LB, Av, lower=True)
    t = solve_triangular(LB.T, t, lower=False)
    rv = vt - A.T @ t
    return rv.T / s, np.sum(rv * vt) / s


def conjugate_gradient(K, b, initial, A, LB, s, cg_tolerance, max_steps, restart_cg_step):
    """cglb_conjugate_gradient (cglb.py:343-420) -> (v, iterations, final rz).  rz is one scalar over all rows and
    gamma = rz / denom has shape [P]: for P > 1 the step `gamma * p` does not broadcast, as in the reference."""
    v = initial
    r = b - v @ K
    z, rz = precondition(A, LB, s, r)
    p = z
    i = 0
    while 0.5 * rz > cg_tolerance and i < max_steps:
        Ap = p @ K
        denom = np.sum(p * Ap, axis=-1)
        gamma = rz / denom
        if p.shape[0] != 1:
            raise ValueError("CG step: gamma of shape [P] does not broadcast against p [P, N] for P > 1")
        v = v + gamma * p
        restart = i % restart_cg_step == restart_cg_step - 1
        r = b - v @ K if restart else r - gamma * Ap
        z, new_rz = precondition(A, LB, s, r)
        p = z if restart else z + p * new_rz / rz
        rz = new_rz
        i += 1
    return v, i, rz


def bound(X, Y, Z, ko, s, v, jitter=1e-6, mean=None):
    """cglb.py:83-160 at the given v [P, N]: dict(elbo, const, logdet, quad, lb, rz)."""
    N, P = Y.shape
    e = Y - (0.0 if mean is None else mean)
    L, A, LB, AAT = common(X, Z, ko, s, jitter)
    trace = np.sum(ko(X, full_cov=False)) / s - np.trace(AAT)
    logdet = -P * (np.sum(np.log(np.diag(LB))) + 0.5 * N * np.log(s) + 0.5 * N * np.log(1 + trace / N))
    K = ko(X) + s * np.eye(N)
    Kv = v @ K
    r = e.T - Kv
    _, rz = precondition(A, LB, s, r)
    lb = np.sum(v * (r + 0.5 * Kv))
    quad = -(lb + 0.5 * rz)
    const = -0.5 * N * P * LOG2PI
    return dict(elbo=const + logdet + quad, const=const, logdet=logdet, quad=quad, lb=lb, rz=rz)


def run_cg(X, Y, Z, ko, s, v0, tol, max_steps, restart, jitter=1e-6, mean=None):
    _, A, LB, _ = common(X, Z, ko, s, jitter)
    K = ko(X) + s * np.eye(X.shape[0])
    e = Y - (0.0 if mean is None else mean)
    return conjugate_gradient(K, e.T, v0, A, LB, s, tol, max_steps, restart)


def predict_f(X, Y, Z, ko, s, v, Xnew, jitter=1e-6):
    """cglb.py:162-240 with the given v (full_cov=False): (mean [Nnew, P], var [Nnew, P])."""
    L, A, LB, _ = common(X, Z, ko, s, jitter)
    K = ko(X) + s * np.eye(X.shape[0])
    cg_mean = ko(Xnew, X) @ v.T
    res = Y - K @ v.T
    c = solve_triangular(LB, A @ res, lower=True) / np.sqrt(s)
    tmp1 = solve_triangular(L, ko(Z, Xnew), lower=True)
    tmp2 = solve_triangular(LB, tmp1, lower=True)
    mean = tmp2.T @ c + cg_mean
    var = ko(Xnew, full_cov=False) + np.sum(tmp2 ** 2, 0) - np.sum(tmp1 ** 2, 0)
    return mean, np.tile(var[:, None], (1, Y.shape[1]))


# ---- the gradient at fixed v, in the matrices the bound is built from -------------------------------------------
def bound_from(Kh, Kuf, Kuu, kdiag, s, e, v, P=None):
    """The bound as a function of K^ [N, N], Kuf [M, N], Kuu [M, M] (jitter included), Kdiag [N], s, e [N, P], v [P, N]."""
    N, P = e.shape
    L = np.linalg.cholesky(Kuu)
    At = solve_triangular(L, Kuf, lower=True)
    M = Kuu.shape[0]
    B = np.eye(M) + At @ At.T / s
    t = (np.sum(kdiag) - np.sum(At ** 2)) / s
    logdet = -P * (0.5 * np.linalg.slogdet(B)[1] + 0.5 * N * np.log(s) + 0.5 * N * np.log(1 + t / N))
    Q = At.T @ At + s * np.eye(N)
    r = e.T - v @ Kh
    quad = -(np.sum(v * e.T) - 0.5 * np.sum(v * (v @ Kh)) + 0.5 * np.sum(r * np.linalg.solve(Q, r.T).T))
    return -0.5 * N * P * LOG2PI + logdet + quad


def bound_adjoints(Kh, Kuf, Kuu, kdiag, s, e, v):
    """The closed forms of gpk_cglb_elbo_grad (include/gpk.h): dict of dF/dK^, dF/dKuf, dF/dKuu, dF/dKdiag (scalar per
    element), dF/ds (with K^ = K + s I depending on s), dF/de and dF/dv."""
    N, P = e.shape
    M = Kuu.shape[0]
    L = np.linalg.cholesky(Kuu)
    At = solve_triangular(L, Kuf, lower=True)
    B = np.eye(M) + At @ At.T / s
    Bi = np.linalg.inv(B)
    t = (np.sum(kdiag) - np.sum(At ** 2)) / s
    ct = -0.5 * P / (1 + t / N)
    Q = At.T @ At + s * np.eye(N)
    r = e.T - v @ Kh                     # [P, N]
    z = np.linalg.solve(Q, r.T)          # [N, P]
    V = v.T
    Az = At @ z
    Li = np.linalg.inv(L)
    dKh = 0.5 * V @ V.T + 0.5 * (z @ V.T + V @ z.T)
    dKuf = Li.T @ ((-P / s * Bi - 2 * ct / s * np.eye(M)) @ At + Az @ z.T)
    dKuu = Li.T @ (0.5 * P * (np.eye(M) - Bi) - 0.5 * Az @ Az.T + ct * (B - np.eye(M))) @ Li
    ds = np.sum(0.5 * V ** 2 + z * V) - 0.5 * P * (N - M + np.trace(Bi)) / s + 0.5 * np.sum(z ** 2) - ct * t / s
    return dict(Kh=dKh, Kuf=dKuf, Kuu=dKuu, kdiag=ct / s, s=ds, e=-(V + z), v=(Kh @ z - r.T).T)
