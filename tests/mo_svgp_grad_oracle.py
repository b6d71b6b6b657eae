"""Gradient oracle for the multi-output SVGP ELBO (test infrastructure, like tests/svgp_grad_oracle.py; not imported by
the product): the target of gpk_svgp_mo_elbo_grad.

L independent latent GPs g_l, latent l with kernel k_l and inducing inputs Z_l (lists of length 1 are shared), q_mu
[M, L], q_sqrt [L, M, M] or [M, L] (q_diag), and P outputs f = g W^T with W [P, L] (LinearCoregionalization) or f = g
(W None, P = L).  Per latent the forward is the single-output forward with P = 1 (posteriors.py:844-885), then

    fmean = gmean W^T [B, P],   fvar = gvar (W o W)^T [B, P]                 (conditionals/util.py:518-563)

and the KL is the sum of the latents' KLs (kullback_leiblers.py:31-49 with Kuu [L, M, M]).  With c = num_data / B,
R = c dVE/dfmean and Wt = c dVE/dfvar ([B, P] here), the adjoints of the latents and of W are

    Rg = R W [B, L] (dF/dgmean),   Wg = Wt (W o W) [B, L] (dF/dgvar),   dW = R^T gmean + 2 W o (Wt^T gvar)

(Rg = R, Wg = Wt without W).  Latent l's backward is the single-output backward with P = 1 driven by Rg[:, l] and
Wg[:, l] (tests/lik_oracle.py::svgp_elbo_lik_and_grad, restated below for one latent); its kernel gradients and dZ
add into its kernel's and its Z's (summed where one is shared).  dF/dm(X) = R.  Pinned by central finite differences of
mo_svgp_elbo (composed from O.mo_independent_predict_f, O.mix_latent_gp, O.gauss_kl and the likelihood oracles) in
tests/test_oracle_mo_svgp_grad.py.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests.svgp_grad_oracle import _phi, _sym, kernel_and_z_grads


def _latent_q(q_sqrt: np.ndarray, l: int) -> np.ndarray:
    return q_sqrt[:, l:l + 1] if q_sqrt.ndim == 2 else q_sqrt[l:l + 1]


def mo_svgp_elbo(X, Y, Zs: Sequence[np.ndarray], kernels: Sequence[O.Kernel], q_mu, q_sqrt, lik, *, W=None,
                 whiten: bool = True, num_data=None, mean_function=None, jitter: float = O.DEFAULT_JITTER) -> float:
    """svgp.py:166-181 for a multi-output kernel, composed as the reference composes it."""
    L = q_mu.shape[1]
    gm, gv = O.mo_independent_predict_f(X, Zs, kernels, q_mu, q_sqrt, whiten=whiten, jitter=jitter)
    fm, fv = (gm, gv) if W is None else O.mix_latent_gp(W, gm, gv, False, False)
    fm = fm + O._mean(mean_function, X, fm.shape[1])
    if whiten:
        kl = O.gauss_kl(q_mu, q_sqrt, None)
    else:
        K = np.stack([O.Kuu(Zs[l if len(Zs) > 1 else 0], kernels[l if len(kernels) > 1 else 0], jitter=jitter)
                      for l in range(L)])
        kl = O.gauss_kl(q_mu, q_sqrt, K)
    scale = 1.0 if num_data is None else float(num_data) / X.shape[0]
    return float(np.sum(lik.variational_expectations(fm, fv, Y)) * scale - kl)


def _latent_backward(X, kernel, Z, m, qs, R, w, whiten, jitter):
    """One latent's backward (P = 1): m [M, 1], qs [1, M, M] or [M, 1], R [B, 1], w [B] -> (per_leaf, dZ, dq_mu [M],
    dq_sqrt [M, M] or [M])."""
    M = Z.shape[0]
    q_diag = qs.ndim == 2
    K = O.Kuu(Z, kernel, jitter=jitter)
    Lc = O.cholesky(K)
    Kuf = O.Kuf(Z, kernel, X)
    Linv = O.tri_solve(Lc, np.eye(M))
    Kinv = Linv.T @ Linv
    S = np.diag(qs[:, 0]) if q_diag else np.tril(qs[0])
    Sig = S @ S.T
    A = Linv @ Kuf if whiten else Kinv @ Kuf
    AW = A * w[None, :]
    G = AW @ A.T
    if whiten:
        Abar = m @ R.T + 2.0 * (Sig - np.eye(M)) @ AW
        Guf = Linv.T @ Abar
        Guu = -_sym(Linv.T @ _phi(Abar @ A.T) @ Linv)
        dq_mu = A @ R - m
        KS = S
    else:
        Abar = m @ R.T + 2.0 * Sig @ AW
        Guf = Kinv @ Abar - 2.0 * AW
        Guu = _sym(-Kinv @ Abar @ A.T) + G + 0.5 * Kinv @ (m @ m.T + Sig) @ Kinv - 0.5 * Kinv
        dq_mu = A @ R - Kinv @ m
        KS = Kinv @ S
    if q_diag:
        kd = np.ones(M) if whiten else np.diag(Kinv)
        s = qs[:, 0]
        dq_sqrt = 2.0 * s * np.diag(G) - kd * s + 1.0 / s
    else:
        dq_sqrt = np.tril(2.0 * G @ S - KS) + np.diag(1.0 / np.diag(S))
    per_leaf, dZ = kernel_and_z_grads(kernel, X, Z, Guu, Guf, w)
    return per_leaf, dZ, dq_mu[:, 0], dq_sqrt


def mo_svgp_elbo_and_grad(X, Y, Zs: Sequence[np.ndarray], kernels: Sequence[O.Kernel], q_mu, q_sqrt, lik, *, W=None,
                          whiten: bool = True, num_data=None, mean_function=None,
                          jitter: float = O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The ELBO of mo_svgp_elbo and its gradient: {"kernels": [per kernel of `kernels`: per leaf in `leaves()` order],
    "lik" (d/d Gaussian variance or Student-t scale, else 0), "mean", "Z": [per set of `Zs`], "q_mu", "q_sqrt", "W"
    (None without W)}."""
    B = X.shape[0]
    L = q_mu.shape[1]
    c = 1.0 if num_data is None else float(num_data) / B
    gm, gv = O.mo_independent_predict_f(X, Zs, kernels, q_mu, q_sqrt, whiten=whiten, jitter=jitter)
    fm, fv = (gm, gv) if W is None else O.mix_latent_gp(W, gm, gv, False, False)
    P = fm.shape[1]
    fm = fm + O._mean(mean_function, X, P)
    dmu, dv, dpar = lik.ve_grads(fm, fv, Y)
    R, Wt = c * dmu, c * dv
    if W is None:
        Rg, Wg, dW = R, Wt, None
    else:
        Rg, Wg = R @ W, Wt @ (W * W)
        dW = R.T @ gm + 2.0 * W * (Wt.T @ gv)
    kgrads: List[Optional[list]] = [None] * len(kernels)
    dZs = [np.zeros_like(Z) for Z in Zs]
    dq_mu = np.zeros_like(q_mu)
    dq_sqrt = np.zeros_like(q_sqrt)
    for l in range(L):
        ki, zi = (l if len(kernels) > 1 else 0), (l if len(Zs) > 1 else 0)
        per_leaf, dZ, dm_l, ds_l = _latent_backward(X, kernels[ki], Zs[zi], q_mu[:, l:l + 1], _latent_q(q_sqrt, l),
                                                    Rg[:, l:l + 1], Wg[:, l], whiten, jitter)
        if kgrads[ki] is None:
            kgrads[ki] = per_leaf
        else:
            kgrads[ki] = [{n: a[n] + b[n] for n in a} for a, b in zip(kgrads[ki], per_leaf)]
        dZs[zi] += dZ
        dq_mu[:, l] = dm_l
        if q_sqrt.ndim == 2:
            dq_sqrt[:, l] = ds_l
        else:
            dq_sqrt[l] = ds_l
    mean: Dict[str, np.ndarray] = {}
    if isinstance(mean_function, O.ConstantMean):
        cs = R.sum(0)
        mean["c"] = np.array([cs.sum()]) if mean_function.c.size == 1 else cs
    elif isinstance(mean_function, O.LinearMean):
        cs = R.sum(0)
        rhs = R.sum(1, keepdims=True) if mean_function.A.shape[1] == 1 else R
        mean["A"] = X.T @ rhs
        mean["b"] = np.array([cs.sum()]) if mean_function.b.size == 1 else cs
    elbo = mo_svgp_elbo(X, Y, Zs, kernels, q_mu, q_sqrt, lik, W=W, whiten=whiten, num_data=num_data,
                        mean_function=mean_function, jitter=jitter)
    return elbo, {"kernels": kgrads, "lik": float(c * np.sum(dpar)), "mean": mean, "Z": dZs, "q_mu": dq_mu,
                  "q_sqrt": dq_sqrt, "W": dW}
