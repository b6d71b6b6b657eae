"""The natural-gradient oracle (tests/natgrad_oracle.py): its Cholesky adjoint and XiSqrtMeanVar tangent against central
finite differences, the reference's literal step against the rewritten forms the device runs, the rule for negative
entries on diag(q_sqrt), and the exact-step identities of XiNat with gamma = 1 on the VGP and SVGP oracles.  Also the
host-side refusals of NaturalGradient.  No device needed."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from oracle import gp_oracle as O
from tests import natgrad_oracle as NG
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as SV
from tests import vgp_grad_oracle as V

SEED = 20261016


def _q(M, P, rng, neg=False):
    m = 0.5 * rng.standard_normal((M, P))
    S = np.stack([np.tril(0.3 * rng.standard_normal((M, M)) / np.sqrt(M), -1) + np.diag(0.5 + 0.5 * rng.random(M))
                  for _ in range(P)])
    if neg:
        S *= np.where(rng.random(M) < 0.4, -1.0, 1.0)[None, None, :]
    return m, S


def test_cholesky_adjoint_matches_finite_differences():
    rng = np.random.default_rng(SEED)
    M = 6
    _, S = _q(M, 1, rng)
    S = S[0]
    W = rng.standard_normal((M, M))
    Sig = S @ S.T

    def g(Sg):   # a function of the Cholesky factor
        L = np.linalg.cholesky(Sg)
        return np.sum(W * L) + np.sum(np.log(np.diag(L)) ** 2)

    L = np.linalg.cholesky(Sig)
    gS = np.tril(W) + np.diag(2.0 * np.log(np.diag(L)) / np.diag(L))
    Sigbar = NG.chol_adjoint(L, gS)
    h = 1e-6
    for _ in range(5):
        E = rng.standard_normal((M, M))
        E = E + E.T
        fd = (g(Sig + h * E) - g(Sig - h * E)) / (2 * h)
        assert abs(np.sum(Sigbar * E) - fd) <= 1e-7 * max(1.0, abs(fd)), (np.sum(Sigbar * E), fd)


def test_xi_sqrt_mean_var_tangent_matches_finite_differences():
    rng = np.random.default_rng(SEED + 1)
    M, P = 7, 2
    m, S = _q(M, P, rng)
    n1, n2 = NG.meanvarsqrt_to_natural(m, S)
    t1 = rng.standard_normal((M, P))
    t2 = rng.standard_normal((P, M, M))
    t2 = 0.5 * (t2 + t2.transpose(0, 2, 1))
    dmu, dL = NG.natural_to_meanvarsqrt_tangent(n1, n2, t1, t2)
    h = 1e-6
    mp, Lp = NG.natural_to_meanvarsqrt(n1 + h * t1, n2 + h * t2)
    mm, Lm = NG.natural_to_meanvarsqrt(n1 - h * t1, n2 - h * t2)
    np.testing.assert_allclose(dmu, (mp - mm) / (2 * h), rtol=0, atol=3e-7 * np.abs(dmu).max())
    np.testing.assert_allclose(dL, (Lp - Lm) / (2 * h), rtol=0, atol=3e-7 * np.abs(dL).max())


def test_conversions_round_trip():
    rng = np.random.default_rng(SEED + 2)
    m, S = _q(9, 3, rng)
    m2, S2 = NG.natural_to_meanvarsqrt(*NG.meanvarsqrt_to_natural(m, S))
    np.testing.assert_allclose(m2, m, atol=1e-12)
    np.testing.assert_allclose(S2, S, atol=1e-12)
    m3, S3 = NG.expectation_to_meanvarsqrt(*NG.meanvarsqrt_to_expectation(m, S))
    np.testing.assert_allclose(m3, m, atol=1e-12)
    np.testing.assert_allclose(S3, S, atol=1e-12)


@pytest.mark.parametrize("xi", ["nat", "sqrt"])
@pytest.mark.parametrize("M", [1, 2, 7, 33, 128, 300])
@pytest.mark.parametrize("P", [1, 4])
@pytest.mark.parametrize("gamma", [1.0, 0.3, 0.05])
def test_literal_step_equals_rewritten_step(xi, M, P, gamma):
    rng = np.random.default_rng(SEED + 10 * M + P)
    m, S = _q(M, P, rng)
    gm, gS = NG.concave_grads(M, P, S, rng)
    ml, Sl = NG.literal_step(xi, m, S, gm, gS, gamma)
    mr, Sr = NG.rewritten_step(xi, m, S, gm, gS, gamma)
    assert np.abs(mr - ml).max() <= 1e-12 * np.abs(ml).max()
    assert np.abs(Sr - Sl).max() <= 1e-12 * np.abs(Sl).max()


@pytest.mark.parametrize("xi", ["nat", "sqrt"])
def test_negative_diagonal_follows_the_chain_rule_through_q_sqrt(xi):
    rng = np.random.default_rng(SEED + 3)
    M, P, gamma = 40, 3, 0.7
    m, S = _q(M, P, rng, neg=True)
    assert (np.diagonal(S, axis1=1, axis2=2) < 0).any()
    gm, gS = NG.concave_grads(M, P, S, rng)
    ml, Sl = NG.sign_normalised_literal_step(xi, m, S, gm, gS, gamma)
    mr, Sr = NG.rewritten_step(xi, m, S, gm, gS, gamma)
    Sig_l = Sl @ Sl.transpose(0, 2, 1)
    Sig_r = Sr @ Sr.transpose(0, 2, 1)
    assert np.abs(mr - ml).max() <= 1e-12 * np.abs(ml).max()
    assert np.abs(Sig_r - Sig_l).max() <= 1e-12 * np.abs(Sig_l).max()
    if xi == "nat":
        assert (np.diagonal(Sr, axis1=1, axis2=2) > 0).all()
        assert np.abs(Sr - Sl).max() <= 1e-12 * np.abs(Sl).max()


def test_xinat_unit_step_makes_the_vgp_elbo_the_gpr_marginal_likelihood():
    d = O.make_data(3, 30, 3, 2)
    X, Y = d["X"], d["Y"]
    ko = O.SquaredExponential(variance=1.3, lengthscales=0.8)
    s2, jit = 0.1, O.DEFAULT_JITTER
    rng = np.random.default_rng(SEED + 4)
    m, S = _q(30, 2, rng)
    _, g = V.vgp_elbo_and_grad_expr(X, Y, ko, m, S, s2, jitter=jit)
    m1, S1 = NG.rewritten_step("nat", m, S, g["q_mu"], g["q_sqrt"], 1.0)
    elbo = O.vgp_elbo(X, Y, ko, m1, S1, s2, jitter=jit)
    ref = O.gpr_log_marginal_likelihood(X, Y, ko, s2 + jit)
    assert abs(elbo - ref) <= 1e-10 * abs(ref), (elbo, ref)


@pytest.mark.parametrize("whiten", [True, False])
def test_xinat_unit_step_makes_the_full_batch_svgp_elbo_the_sgpr_bound(whiten):
    d = O.make_data(4, 60, 3, 2, M=12)
    X, Y, Z = d["X"], d["Y"], d["Z"]
    ko = O.Sum([O.SquaredExponential(variance=1.1, lengthscales=0.9), O.White(variance=0.05)])
    s2 = 0.2
    rng = np.random.default_rng(SEED + 5)
    m, S = _q(12, 2, rng)
    _, g = SV.svgp_elbo_and_grad(X, Y, [ko], [Z], m, S, LO.Gaussian(s2), whiten=whiten, num_data=60)
    m1, S1 = NG.rewritten_step("nat", m, S, g["q_mu"], g["q_sqrt"], 1.0)
    elbo = O.svgp_elbo(X, Y, Z, ko, m1, S1, s2, whiten=whiten, num_data=60)
    ref = O.sgpr_elbo(X, Y, ko, Z, s2)
    assert abs(elbo - ref) <= 1e-10 * abs(ref), (elbo, ref)


def test_natural_gradient_refusals_on_the_host():
    opt = gpf.optimizers
    for gamma in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="gamma"):
            opt.NaturalGradient(gamma)

    class Custom(opt.XiTransform):
        pass

    with pytest.raises(NotImplementedError, match="XiNat and XiSqrtMeanVar"):
        opt.NaturalGradient(0.1, xi_transform=Custom())
    ng = opt.NaturalGradient(0.1)
    with pytest.raises(ValueError, match="training_loss_closure"):
        ng.minimize(lambda: 0.0, [])
    assert isinstance(ng.xi_transform, opt.XiNat)
    assert opt.XiSqrtMeanVar()._code == gpf._lib.GPK_XI_SQRT_MEAN_VAR
