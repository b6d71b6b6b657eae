"""The device likelihood operators (csrc/lik.cu: gpk_lik_varexp_sum, gpk_lik_predict_mean_and_var,
gpk_lik_predict_log_density) against the oracle (tests/lik_oracle.py) in float64 and float32, and the SVGP value,
predict_y and predict_log_density with Bernoulli / Poisson / StudentT through the public API."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S

pytestmark = pytest.mark.gpu

L = gpf.likelihoods


def _pair(name):
    """(device likelihood, oracle likelihood) with the same values."""
    if name == "bernoulli":
        return L.Bernoulli(), LO.Bernoulli()
    if name == "poisson":
        return L.Poisson(binsize=1.3), LO.Poisson(1.3)
    if name == "student_t":
        return L.StudentT(scale=0.7, df=4.0), LO.StudentT(0.7, 4.0)
    raise ValueError(name)


def _elements(name, N=777, P=3, seed=1):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-2.0, 2.0, (N, P))
    v = rng.uniform(0.01, 1.5, (N, P))
    return mu, v, LO.targets(name, mu, rng)


@pytest.mark.parametrize("dtype,rtol", [(np.float64, 1e-12), (np.float32, 1e-5)])
@pytest.mark.parametrize("name", ["bernoulli", "poisson", "student_t", "gaussian"])
def test_operators_match_oracle(cuda_device, name, dtype, rtol):
    if name == "gaussian":
        desc, lo = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.3), LO.Gaussian(0.3)
    else:
        lp, lo = _pair(name)
        desc = lp._lik_desc()
    mu, v, y = _elements(name)
    if dtype == np.float32:  # the oracle sees the values the device sees
        mu, v, y = (a.astype(np.float32).astype(np.float64) for a in (mu, v, y))
    with gpf.config.as_context(gpf.config.Config(float=dtype, jitter=1e-6)):
        M, V, Y = (ops.to_device(a) for a in (mu, v, y))
        ve = float(ops.lik_varexp_sum(desc, M, V, Y).cpu().numpy()[0])
        pm, pv = ops.lik_predict_mean_and_var(desc, M, V)
        ld = ops.lik_predict_log_density(desc, M, V, Y).cpu().numpy()
    want = float(np.sum(lo.variational_expectations(mu, v, y)))
    assert abs(ve - want) <= rtol * abs(want), (ve, want)
    wm, wv = lo.predict_mean_and_var(mu, v)
    tol = 1e-12 if dtype == np.float64 else 1e-5
    np.testing.assert_allclose(pm.cpu().numpy(), wm, rtol=tol, atol=tol * np.max(np.abs(wm)))
    np.testing.assert_allclose(pv.cpu().numpy(), wv, rtol=tol, atol=tol * np.max(np.abs(wv)))
    wl = lo.predict_log_density(mu, v, y)
    np.testing.assert_allclose(ld, wl, rtol=tol, atol=tol * np.max(np.abs(wl)))


@pytest.mark.parametrize("name", ["bernoulli", "poisson", "student_t"])
@pytest.mark.parametrize("whiten", [True, False])
def test_svgp_value_and_predictions_match_oracle(cuda_device, name, whiten):
    B, D, M, P = 300, 3, 20, 2
    d = O.make_data(2, B, D, P)
    rng = np.random.default_rng(9)
    Y = LO.targets(name, np.sin(d["X"][:, :1] @ np.ones((1, P))), rng)
    Z = d["X"][:M].copy()
    q_mu = 0.3 * rng.standard_normal((M, P))
    q_sqrt = np.stack([np.tril(0.1 * rng.standard_normal((M, M)), -1) + np.diag(0.5 + 0.3 * rng.random(M))
                       for _ in range(P)])
    lp, lo = _pair(name)
    mp, mo = gpf.mean_functions.Constant(np.array([0.1, -0.2])), O.ConstantMean(np.array([0.1, -0.2]))
    m = gpf.models.SVGP(gpf.kernels.Matern52(variance=1.2, lengthscales=1.5), lp, Z, num_latent_gps=P, q_mu=q_mu,
                        q_sqrt=q_sqrt, whiten=whiten, num_data=3000, mean_function=mp)
    ko = O.Matern52(1.2, 1.5)
    jit = gpf.config.default_jitter()
    want = S.svgp_elbo(d["X"], Y, [ko], [Z], q_mu, q_sqrt, lo, whiten=whiten, num_data=3000, mean_function=mo,
                       jitter=jit)
    np.testing.assert_allclose(float(m.elbo((d["X"], Y))), want, rtol=1e-10)
    fm, fv = O.svgp_predict_f(d["X"], Z, ko, q_mu, q_sqrt, whiten=whiten, mean_function=mo, jitter=jit)
    ym, yv = m.predict_y(d["X"])
    wm, wv = lo.predict_mean_and_var(fm, fv)
    np.testing.assert_allclose(ym.cpu().numpy(), wm, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(yv.cpu().numpy(), wv, rtol=1e-8, atol=1e-10)
    ld = m.predict_log_density((d["X"], Y)).cpu().numpy()
    np.testing.assert_allclose(ld, lo.predict_log_density(fm, fv, Y), rtol=1e-8, atol=1e-10)
