"""Natural-gradient oracle (test infrastructure, not imported by the product): the target of gpk_natgrad_step.

Three layers, for P latents with m = q_mu[:, p], S = tril(q_sqrt[p]), gm = dF/dm, gS = dF/dS (F the ELBO):
  1. the reference's parameter conversions (gpflow/optimizers/natgrad.py:429-502), restated literally;
  2. the literal `_natgrad_apply_gradients` (natgrad.py:280-367) for XiNat and XiSqrtMeanVar, with dF/deta from the
     analytic Cholesky adjoint Sigbar = sym(S^-T Phi(S^T gS) S^-1): dF/deta2 = Sigbar, dF/deta1 = gm - 2 Sigbar m; the
     XiSqrtMeanVar direction is the forward-mode derivative of natural_to_meanvarsqrt, written analytically;
  3. the rewritten forms the device runs (include/gpk.h), which form neither Sig^-1, S^-1 nor a second Cholesky.
The reference descends -F; every step here ascends F by the same amount: theta' = theta + gamma dF/deta."""
from __future__ import annotations

from typing import Tuple

import numpy as np
import scipy.linalg

from tests.kernel_grad_oracle import phi, sym


def _inv_lower(L: np.ndarray) -> np.ndarray:
    return scipy.linalg.solve_triangular(L, np.eye(L.shape[0]), lower=True)


def concave_grads(M, P, S, rng):
    """gm and gS = tril(2 Sigbar S) of a concave objective in Sig (Sigbar negative definite): every step is valid."""
    gm = rng.standard_normal((M, P))
    gS = np.empty_like(S)
    for p in range(P):
        A = rng.standard_normal((M, M)) / np.sqrt(M)
        Sigbar = -(A @ A.T) - 0.1 * np.eye(M)
        gS[p] = np.tril(2.0 * Sigbar @ np.tril(S[p]))
    return gm, gS


# ---- 1. conversions, natgrad.py:429-502 (GPflow layout: mean [M, P], square roots [P, M, M]) -----------------------
def natural_to_meanvarsqrt(nat1: np.ndarray, nat2: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    mu, sq = np.empty_like(nat1), np.empty_like(nat2)
    for p in range(nat2.shape[0]):
        var_sqrt = _inv_lower(np.linalg.cholesky(-2.0 * nat2[p]))
        S = var_sqrt.T @ var_sqrt
        mu[:, p] = S @ nat1[:, p]
        sq[p] = np.linalg.cholesky(S)
    return mu, sq


def meanvarsqrt_to_natural(mu: np.ndarray, s_sqrt: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    n1, n2 = np.empty_like(mu), np.empty_like(s_sqrt)
    for p in range(s_sqrt.shape[0]):
        s_sqrt_inv = _inv_lower(s_sqrt[p])
        s_inv = s_sqrt_inv.T @ s_sqrt_inv
        n1[:, p] = s_inv @ mu[:, p]
        n2[p] = -0.5 * s_inv
    return n1, n2


def meanvarsqrt_to_expectation(m: np.ndarray, v_sqrt: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    return m, np.stack([v_sqrt[p] @ v_sqrt[p].T + np.outer(m[:, p], m[:, p]) for p in range(v_sqrt.shape[0])])


def expectation_to_meanvarsqrt(eta1: np.ndarray, eta2: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    return eta1, np.stack([np.linalg.cholesky(eta2[p] - np.outer(eta1[:, p], eta1[:, p])) for p in range(eta2.shape[0])])


# ---- 2. the literal step -----------------------------------------------------------------------------------------------
def chol_adjoint(S: np.ndarray, gS: np.ndarray) -> np.ndarray:
    """dF/dSig for F(chol(Sig)) with dF/dS = gS at S = chol(Sig) (one latent)."""
    Si = _inv_lower(S)
    return sym(Si.T @ phi(S.T @ gS) @ Si)


def dF_deta(m: np.ndarray, S: np.ndarray, gm: np.ndarray, gS: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """The chain rule of natgrad.py:345-348: (dF/deta1 [M, P], dF/deta2 [P, M, M]); S with a positive diagonal."""
    d1, d2 = np.empty_like(m), np.empty_like(S)
    for p in range(S.shape[0]):
        d2[p] = chol_adjoint(S[p], gS[p])
        d1[:, p] = gm[:, p] - 2.0 * d2[p] @ m[:, p]
    return d1, d2


def natural_to_meanvarsqrt_tangent(nat1, nat2, t1, t2) -> Tuple[np.ndarray, np.ndarray]:
    """The forward-mode derivative of natural_to_meanvarsqrt at (nat1, nat2) in the direction (t1, t2): with
    Sig = (-2 nat2)^-1 = L L^T, dSig = 2 Sig t2 Sig, dmu = dSig nat1 + Sig t1, dL = L Phi(L^-1 dSig L^-T)."""
    dmu, dL = np.empty_like(nat1), np.empty_like(nat2)
    for p in range(nat2.shape[0]):
        Sig = np.linalg.inv(-2.0 * nat2[p])
        Sig = sym(Sig)
        L = np.linalg.cholesky(Sig)
        Li = _inv_lower(L)
        dSig = 2.0 * Sig @ t2[p] @ Sig
        dmu[:, p] = dSig @ nat1[:, p] + Sig @ t1[:, p]
        dL[p] = L @ phi(Li @ dSig @ Li.T)
    return dmu, dL


def literal_step(xi: str, m, S, gm, gS, gamma: float) -> Tuple[np.ndarray, np.ndarray]:
    """natgrad.py:320-367 with S = tril(q_sqrt) of positive diagonal, ascending F: xi' = xi + gamma (natural gradient)."""
    S = np.tril(S)
    d1, d2 = dF_deta(m, S, gm, gS)
    if xi == "nat":
        n1, n2 = meanvarsqrt_to_natural(m, S)
        return natural_to_meanvarsqrt(n1 + gamma * d1, n2 + gamma * d2)
    n1, n2 = meanvarsqrt_to_natural(m, S)
    t1, t2 = natural_to_meanvarsqrt_tangent(n1, n2, d1, d2)
    return m + gamma * t1, S + gamma * t2


def sign_normalised_literal_step(xi: str, m, S, gm, gS, gamma: float):
    """The literal step applied through the chain rule of q_sqrt: S = S~ D with D = diag(sign diag S), gS~ = gS D."""
    S = np.tril(S)
    D = np.stack([np.where(np.diag(S[p]) < 0, -1.0, 1.0) for p in range(S.shape[0])])
    return literal_step(xi, m, S * D[:, None, :], gm, gS * D[:, None, :], gamma)


# ---- 3. the rewritten forms --------------------------------------------------------------------------------------------
def rewritten_step(xi: str, m, S, gm, gS, gamma: float) -> Tuple[np.ndarray, np.ndarray]:
    """The device's algebra (include/gpk.h, csrc/natgrad.cu).  Raises np.linalg.LinAlgError where the device reports a
    non-positive pivot of J B J."""
    P, M, _ = S.shape
    J = np.eye(M)[::-1]
    m_out, S_out = m.copy(), np.empty_like(S)
    for p in range(P):
        Sp = np.tril(S[p])
        T = Sp.T @ gS[p]
        if xi == "nat":
            d = np.where(np.diag(Sp) < 0, -1.0, 1.0)
            H = sym(phi(T))
            B = np.eye(M) - 2.0 * gamma * d[:, None] * H * d[None, :]
            C = np.linalg.cholesky(J @ B @ J)
            U = J @ C @ J
            Sn = scipy.linalg.solve_triangular(U, (Sp * d[None, :]).T, lower=False).T   # S~ U^-T
            S_out[p] = np.tril(Sn)
        else:
            Sn = Sp
            S_out[p] = np.tril(Sp + gamma * Sp @ phi(T))
        m_out[:, p] = m[:, p] + gamma * Sn @ (Sn.T @ gm[:, p])
    return m_out, S_out
