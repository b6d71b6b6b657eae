"""Value and gradient oracle for the SVGP ELBO with any likelihood and output structure (test infrastructure, like
tests/sgpr_grad_oracle.py; not imported by the product): the target of gpk_svgp_elbo_grad and gpk_svgp_mo_elbo_grad.

L independent latent GPs g_l, latent l with kernel k_l and inducing inputs Z_l (lists of length 1 are shared), q_mu
[M, L], q_sqrt [L, M, M] or [M, L] (q_diag), and P outputs f = g W^T with W [P, L] (LinearCoregionalization) or f = g
(W None, P = L).  Single-output SVGP is one kernel, one Z and no W.  Per latent the forward is gpflow/posteriors.py:
844-885, then

    fmean = gmean W^T [B, P],   fvar = gvar (W o W)^T [B, P]                 (conditionals/util.py:518-563)

and the KL is the sum of the latents' KLs (kullback_leiblers.py:31-49).  The reference obtains the gradient from
TensorFlow autodiff through gpflow/models/svgp.py:166-181.  With c = num_data / B, R = c dVE/dfmean and Wt = c dVE/dfvar
([B, P], from the likelihood's `ve_grads`), the adjoints of the latents and of W are

    Rg = R W [B, L] (dF/dgmean),   Wg = Wt (W o W) [B, L] (dF/dgvar),   dW = R^T gmean + 2 W o (Wt^T gvar)

(Rg = R, Wg = Wt without W), and dF/dm(X) = R.  Latent l's backward, with r = Rg[:, l], w = Wg[:, l], K = Kuu + jitter
I = L L^T, m = q_mu[:, l], S = tril(q_sqrt[l]), A = L^-1 Kuf (whiten) or K^-1 Kuf, Phi(T) = tril(T) with its diagonal
halved and sym(T) = (T + T^T) / 2:

  whiten:     Abar = m r^T + 2 (S S^T - I) A diag(w)
              dF/dKuf = L^-T Abar,   dF/dKuu = -sym(L^-T Phi(Abar A^T) L^-1)   (the Cholesky adjoint)
              dF/dm = A r - m,       dF/dS = tril(2 (A diag(w) A^T) S - S) + diag(1 / diag S)
  otherwise:  Abar = m r^T + 2 S S^T A diag(w)
              dF/dKuf = K^-1 Abar - 2 A diag(w)
              dF/dKuu = sym(-K^-1 Abar A^T) + A diag(w) A^T + 1/2 K^-1 (m m^T + S S^T) K^-1 - 1/2 K^-1
              dF/dm = A r - K^-1 m,  dF/dS = tril(2 (A diag(w) A^T) S - K^-1 S) + diag(1 / diag S)
  both:       dF/dKdiag = w

With q_diag the q_sqrt forms restricted to the diagonal.  The latents that share a kernel and a Z add their dF/dKuu,
dF/dKuf and dF/dKdiag; the kernel parameters and Z follow from those sums as in tests/sgpr_grad_oracle.py.  Pinned by
central finite differences in tests/test_oracle_svgp_grad.py (Gaussian, against oracle/gp_oracle.py::svgp_elbo),
tests/test_oracle_likelihoods.py, tests/test_oracle_multiclass.py, tests/test_oracle_mo_svgp_grad.py and
tests/test_oracle_heteroskedastic.py.
"""
from __future__ import annotations

from typing import Dict, Sequence, Tuple

import numpy as np

from oracle import gp_oracle as O
from tests import kernel_grad_oracle as KG


def _latent_q(q_sqrt: np.ndarray, l: int) -> np.ndarray:
    return q_sqrt[:, l:l + 1] if q_sqrt.ndim == 2 else q_sqrt[l:l + 1]


def _kl(kernels, Zs, q_mu, q_sqrt, whiten, jitter) -> float:
    if whiten:
        return O.gauss_kl(q_mu, q_sqrt, None)
    K = np.stack([O.Kuu(Zs[l if len(Zs) > 1 else 0], kernels[l if len(kernels) > 1 else 0], jitter=jitter)
                  for l in range(q_mu.shape[1])])
    return O.gauss_kl(q_mu, q_sqrt, K)


def _forward(X, kernels, Zs, q_mu, q_sqrt, W, whiten, mean_function, jitter):
    """(gmean, gvar [B, L], fmean, fvar [B, P]) with fmean including m(X)."""
    gm, gv = O.mo_independent_predict_f(X, Zs, kernels, q_mu, q_sqrt, whiten=whiten, jitter=jitter)
    fm, fv = (gm, gv) if W is None else O.mix_latent_gp(W, gm, gv, False, False)
    return gm, gv, fm + O._mean(mean_function, X, fm.shape[1]), fv


def svgp_elbo(X, Y, kernels: Sequence[O.Kernel], Zs: Sequence[np.ndarray], q_mu, q_sqrt, lik, *, W=None,
              whiten: bool = True, num_data=None, mean_function=None, jitter: float = O.DEFAULT_JITTER) -> float:
    """svgp.py:166-181 composed as the reference composes it: O.mo_independent_predict_f, O.mix_latent_gp, O.gauss_kl
    and the likelihood's variational expectations."""
    _, _, fm, fv = _forward(X, kernels, Zs, q_mu, q_sqrt, W, whiten, mean_function, jitter)
    scale = 1.0 if num_data is None else float(num_data) / X.shape[0]
    kl = _kl(kernels, Zs, q_mu, q_sqrt, whiten, jitter)
    return float(np.sum(lik.variational_expectations(fm, fv, Y)) * scale - kl)


def _geometry(X, kernel, Z, whiten, jitter):
    """(L^-1, K^-1, A) of one kernel and inducing set, K = Kuu + jitter I = L L^T."""
    Linv = O.tri_solve(O.cholesky(O.Kuu(Z, kernel, jitter=jitter)), np.eye(Z.shape[0]))
    Kinv = Linv.T @ Linv
    Kuf = O.Kuf(Z, kernel, X)
    return Linv, Kinv, Linv @ Kuf if whiten else Kinv @ Kuf


def _latent_backward(geometry, m, qs, R, w, whiten):
    """One latent's backward: m [M, 1], qs [1, M, M] or [M, 1], R [B, 1], w [B] -> (dF/dKuu, dF/dKuf, dq_mu [M],
    dq_sqrt [M, M] or [M])."""
    Linv, Kinv, A = geometry
    M = Linv.shape[0]
    q_diag = qs.ndim == 2
    S = np.diag(qs[:, 0]) if q_diag else np.tril(qs[0])
    Sig = S @ S.T
    AW = A * w[None, :]
    G = AW @ A.T
    if whiten:
        Abar = m @ R.T + 2.0 * (Sig - np.eye(M)) @ AW
        Guf = Linv.T @ Abar
        Guu = -KG.sym(Linv.T @ KG.phi(Abar @ A.T) @ Linv)
        dq_mu = A @ R - m
        KS = S
    else:
        Abar = m @ R.T + 2.0 * Sig @ AW
        Guf = Kinv @ Abar - 2.0 * AW
        Guu = KG.sym(-Kinv @ Abar @ A.T) + G + 0.5 * Kinv @ (m @ m.T + Sig) @ Kinv - 0.5 * Kinv
        dq_mu = A @ R - Kinv @ m
        KS = Kinv @ S
    if q_diag:
        kd = np.ones(M) if whiten else np.diag(Kinv)
        s = qs[:, 0]
        dq_sqrt = 2.0 * s * np.diag(G) - kd * s + 1.0 / s
    else:
        dq_sqrt = np.tril(2.0 * G @ S - KS) + np.diag(1.0 / np.diag(S))
    return Guu, Guf, dq_mu[:, 0], dq_sqrt


def svgp_elbo_and_grad(X, Y, kernels: Sequence[O.Kernel], Zs: Sequence[np.ndarray], q_mu, q_sqrt, lik, *, W=None,
                       whiten: bool = True, num_data=None, mean_function=None,
                       jitter: float = O.DEFAULT_JITTER) -> Tuple[float, Dict[str, object]]:
    """The ELBO of svgp_elbo and its gradient.  `lik` is any likelihood oracle with variational_expectations(mu, v, y)
    and ve_grads(mu, v, y) -> (dmu, dv, dpar): tests/lik_oracle.py (Gaussian, Bernoulli, Poisson, StudentT),
    tests/multiclass_oracle.py and tests/hetero_oracle.py.  Returns (elbo, {"leaves": [per leaf in `leaves()` order]
    with one kernel, or "kernels": [per kernel of `kernels`: per leaf] with several; "lik": d/d(likelihood parameter)
    (the Gaussian variance, the Student-t scale, the MultiClass epsilon; 0 without one); "mean": {"c"} or {"A", "b"} or
    {}; "Z": [M, D] with one Z, or [per set of `Zs`] with several; "q_mu"; "q_sqrt"; "W" (None without W)})."""
    B = X.shape[0]
    L = q_mu.shape[1]
    c = 1.0 if num_data is None else float(num_data) / B
    gm, gv, fm, fv = _forward(X, kernels, Zs, q_mu, q_sqrt, W, whiten, mean_function, jitter)
    dmu, dv, dpar = lik.ve_grads(fm, fv, Y)
    R, Wt = c * dmu, c * dv
    if W is None:
        Rg, Wg, dW = R, Wt, None
    else:
        Rg, Wg = R @ W, Wt @ (W * W)
        dW = R.T @ gm + 2.0 * W * (Wt.T @ gv)
    geometry: Dict[Tuple[int, int], tuple] = {}
    adj: Dict[Tuple[int, int], list] = {}   # (kernel, Z) -> [dF/dKuu, dF/dKuf, dF/dKdiag] summed over its latents
    dq_mu = np.zeros_like(q_mu)
    dq_sqrt = np.zeros_like(q_sqrt)
    for l in range(L):
        key = (l if len(kernels) > 1 else 0, l if len(Zs) > 1 else 0)
        if key not in geometry:
            geometry[key] = _geometry(X, kernels[key[0]], Zs[key[1]], whiten, jitter)
        Guu, Guf, dq_mu[:, l], ds = _latent_backward(geometry[key], q_mu[:, l:l + 1], _latent_q(q_sqrt, l),
                                                     Rg[:, l:l + 1], Wg[:, l], whiten)
        if q_sqrt.ndim == 2:
            dq_sqrt[:, l] = ds
        else:
            dq_sqrt[l] = ds
        if key in adj:
            for acc, g in zip(adj[key], (Guu, Guf, Wg[:, l])):
                acc += g
        else:
            adj[key] = [Guu, Guf, Wg[:, l].copy()]
    kgrads = [None] * len(kernels)
    dZs = [np.zeros_like(Z) for Z in Zs]
    for (ki, zi), (Guu, Guf, Gdiag) in adj.items():
        per_leaf, dZ = KG.kernel_and_z_grads(kernels[ki], X, Zs[zi], Guu, Guf, Gdiag)
        kgrads[ki] = per_leaf if kgrads[ki] is None else [{n: a[n] + b[n] for n in a}
                                                          for a, b in zip(kgrads[ki], per_leaf)]
        dZs[zi] += dZ
    elbo = float(np.sum(lik.variational_expectations(fm, fv, Y)) * c - _kl(kernels, Zs, q_mu, q_sqrt, whiten, jitter))
    out = {"lik": float(c * np.sum(dpar)), "mean": KG.mean_grads(mean_function, X, R),
           "Z": dZs[0] if len(Zs) == 1 else dZs, "q_mu": dq_mu, "q_sqrt": dq_sqrt, "W": dW}
    if len(kernels) == 1:
        out["leaves"] = kgrads[0]
    else:
        out["kernels"] = kgrads
    return elbo, out
