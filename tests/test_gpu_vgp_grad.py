"""Device value and gradient of the VGP ELBO for any fused kernel expression, the variational parameters and the
Constant / Linear mean functions (gpk_vgp_elbo_grad: csrc/fused.cu::vgp_elbo_grad, the square pass of
csrc/grad.cu::square_grad_launch) against the oracle (tests/vgp_grad_oracle.py::vgp_elbo_and_grad_expr, pinned by
finite differences in tests/test_oracle_vgp_grad.py), VGP.elbo(), the whitened SVGP gradient at Z = X without jitter,
finite differences of the device ELBO at N = 2048, and the reference's method-equivalence training run."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import ops
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import vgp_grad_oracle as V

pytestmark = pytest.mark.gpu

K = gpf.kernels


def _model(X, Y, kp, q_mu, q_sqrt, s2, mp=None):
    m = gpf.models.VGP((X, Y), kp, gpf.likelihoods.Gaussian(s2), mean_function=mp)
    m.q_mu.assign(q_mu)
    m.q_sqrt.assign(q_sqrt)
    return m


def _check(m, X, Y, ko, q_mu, q_sqrt, s2, mo=None, rtol=1e-6):
    elbo, grads = m.elbo_and_grad()
    ref_elbo, g = V.vgp_elbo_and_grad_expr(X, Y, ko, q_mu, q_sqrt, s2, mean_function=mo,
                                           jitter=gpf.config.default_jitter())
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-8)
    ref = GC.reference_by_param(g, [m.kernel], m.mean_function, [
        (m.likelihood.variance, g["noise_variance"]), (m.q_mu, g["q_mu"]), (m.q_sqrt, g["q_sqrt"])])
    GC.assert_grads_match(grads, ref, rtol, "parameter")
    dq = grads[m.q_sqrt]
    iu = np.triu_indices(dq.shape[1], 1)
    assert np.all(dq[:, iu[0], iu[1]] == 0.0)


@pytest.mark.parametrize("name,N,D,P", [
    ("rbf_plus_white", 17, 3, 1), ("c5", 64, 8, 3), ("c5", 200, 8, 1), ("rq", 200, 3, 3), ("rq_ard", 64, 4, 1),
    ("polynomial_ard", 17, 4, 3), ("linear_ard", 200, 4, 3), ("constant_times_matern52", 200, 5, 1),
    ("additive_active_dims", 64, 4, 3), ("k_plus_k", 17, 4, 1)])
def test_vgp_grad_matches_oracle(cuda_device, name, N, D, P):
    d = O.make_data(5, N, D, P)
    q_mu, q_sqrt = GC.q(N, P)
    kp, ko = GC.case(name, D)
    m = _model(d["X"], d["Y"], kp, q_mu, q_sqrt, 0.15)
    _check(m, d["X"], d["Y"], ko, q_mu, q_sqrt, 0.15)


@pytest.mark.parametrize("N,P", [(200, 3), (700, 1)])
def test_value_agrees_with_elbo(cuda_device, N, P):
    """out[0] of the fused call against VGP.elbo() on the same model."""
    d = O.make_data(6, N, 4, P)
    kp, _ = GC.case("c5", 4)
    m = _model(d["X"], d["Y"], kp, *GC.q(N, P, seed=5), 0.2)
    elbo, _ = m.elbo_and_grad()
    np.testing.assert_allclose(float(elbo), float(m.elbo()), rtol=1e-10)


def test_vgp_equals_whitened_svgp_at_z_equal_x_without_jitter(cuda_device):
    """With zero jitter, Z = X and num_data = N, the whitened SVGP ELBO is the VGP ELBO, so the kernel, noise and q
    gradients of the two device entry points agree."""
    N, D, P = 120, 3, 2
    d = O.make_data(7, N, D, P)
    q_mu, q_sqrt = GC.q(N, P, seed=6)
    s2 = 0.2
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=0.0)):
        kp = K.SquaredExponential(variance=1.3, lengthscales=0.8) + K.Linear(variance=0.3)
        vg = _model(d["X"], d["Y"], kp, q_mu, q_sqrt, s2)
        sv = gpf.models.SVGP(kp, gpf.likelihoods.Gaussian(s2), d["X"].copy(), num_latent_gps=P, q_mu=q_mu.copy(),
                             q_sqrt=q_sqrt.copy(), whiten=True, num_data=N)
        e_v, g_v = vg.elbo_and_grad()
        e_s, g_s = sv.elbo_and_grad((d["X"], d["Y"]))
    np.testing.assert_allclose(float(e_v), float(e_s), rtol=1e-9)
    pairs = [(vg.likelihood.variance, sv.likelihood.variance), (vg.q_mu, sv.q_mu), (vg.q_sqrt, sv.q_sqrt)]
    pairs += [(p, p) for p in g_v if any(p is q for q in kp.trainable_parameters)]
    assert len(pairs) == len(g_v)
    scale = max(float(np.max(np.abs(g))) for g in g_v.values())
    for pv, ps in pairs:
        np.testing.assert_allclose(np.asarray(g_v[pv]), np.asarray(g_s[ps]), rtol=0, atol=1e-7 * scale)


@pytest.mark.parametrize("mean", ["constant", "linear"])
def test_mean_function_grads_match_oracle(cuda_device, mean):
    N, D, P = 150, 4, 2
    d = O.make_data(3, N, D, P)
    rng = np.random.default_rng(11)
    if mean == "constant":
        c = 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    else:
        A, b = 0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    kp, ko = GC.case("c5", D)
    q_mu, q_sqrt = GC.q(N, P)
    m = _model(d["X"], d["Y"], kp, q_mu, q_sqrt, 0.2, mp)
    _check(m, d["X"], d["Y"], ko, q_mu, q_sqrt, 0.2, mo)


def test_n2048_finite_difference_of_device_elbo(cuda_device):
    """N = 2048 (a multi-block factorisation on its tensor-core path): the analytic device gradient against central
    finite differences of VGP.elbo() for the noise, a lengthscale, one q_mu and one off-diagonal q_sqrt entry (the ELBO
    is quadratic in both, so their differences are exact up to rounding)."""
    N, D, P = 2048, 8, 1
    d = O.make_data(8, N, D, P)
    rng = np.random.default_rng(13)
    q_mu = 0.3 * rng.standard_normal((N, P))
    q_sqrt = (np.tril(0.01 * rng.standard_normal((N, N)), -1) + np.diag(0.5 + 0.5 * rng.random(N)))[None]
    kp = K.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) + K.White(variance=0.05)
    m = _model(d["X"], d["Y"], kp, q_mu, q_sqrt, 0.1)
    _, grads = m.elbo_and_grad()
    rbf = kp.kernels[0]
    cases = [(m.likelihood.variance, (), 1e-5), (rbf.lengthscales, (), 1e-4), (m.q_mu, (700, 0), 1e-2),
             (m.q_sqrt, (0, 1500, 300), 1e-2)]
    for p, idx, t in cases:
        base = np.array(p.numpy(), dtype=np.float64)

        def at(s):
            v = base.copy()
            v[idx] += s
            p.assign(v)
            return float(m.elbo())

        fd = (at(t) - at(-t)) / (2 * t)
        p.assign(base)
        got = float(np.asarray(grads[p]).reshape(base.shape)[idx])
        np.testing.assert_allclose(got, fd, rtol=1e-5, atol=1e-6, err_msg=str(idx))


def test_method_equivalence_vgp_trained_with_scipy(cuda_device):
    """tests/integration/test_method_equivalence.py::test_equivalence for VGP: SquaredExponential, Constant mean, Scipy
    with maxiter = 3000 on both GPR and VGP, then the reference's own bars."""
    data = (GC.Datum.X, GC.Datum.Y)
    gpr = gpf.models.GPR(data, kernel=K.SquaredExponential(), mean_function=gpf.mean_functions.Constant())
    vgp = gpf.models.VGP(data, kernel=K.SquaredExponential(), likelihood=gpf.likelihoods.Gaussian(),
                         mean_function=gpf.mean_functions.Constant())
    for m in (gpr, vgp):
        gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options=dict(maxiter=3000))
    np.testing.assert_allclose(float(vgp.maximum_log_likelihood_objective()), float(gpr.log_marginal_likelihood()),
                               rtol=1e-6)
    np.testing.assert_allclose(vgp.kernel.lengthscales.numpy(), gpr.kernel.lengthscales.numpy(), rtol=2e-4)
    np.testing.assert_allclose(vgp.kernel.variance.numpy(), gpr.kernel.variance.numpy(), rtol=1e-3)
    gpr_mu, gpr_var = gpr.predict_y(GC.Datum.Xtest)
    vgp_mu, vgp_var = vgp.predict_y(GC.Datum.Xtest)
    np.testing.assert_allclose(vgp_mu.cpu().numpy(), gpr_mu.cpu().numpy(), rtol=1e-3)
    np.testing.assert_allclose(vgp_var.cpu().numpy(), gpr_var.cpu().numpy(), rtol=1e-4)


class _NotGaussian(gpf.likelihoods.ScalarLikelihood):
    pass


class _Quadratic(gpf.mean_functions.MeanFunction):
    def __call__(self, X):
        return ops.to_device(X)[:, :1] * 0.0


def test_refusals(cuda_device):
    d = O.make_data(1, 30, 2, 1)
    data = (d["X"], d["Y"])
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = gpf.models.VGP(data, K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1))
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients()
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        m = gpf.models.VGP(data, kern, gpf.likelihoods.Gaussian(0.1))
        with pytest.raises(NotImplementedError, match=cls):
            m.elbo_and_grad()
    m = gpf.models.VGP(data, K.SharedIndependent(K.SquaredExponential(), 1), gpf.likelihoods.Gaussian(0.1))
    with pytest.raises(NotImplementedError, match="single-output"):
        m.elbo_and_grad()
    m = gpf.models.VGP(data, K.SquaredExponential(), _NotGaussian())
    with pytest.raises(NotImplementedError, match="Gaussian"):
        m.elbo_and_grad()
    lik = gpf.likelihoods.Gaussian(variance=gpf.mean_functions.Linear(A=np.array([[0.05], [0.0]]), b=np.array([0.08])))
    m = gpf.models.VGP(data, K.SquaredExponential(), lik)
    with pytest.raises(NotImplementedError):
        m.elbo_and_grad()
    m = gpf.models.VGP(data, K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1), mean_function=_Quadratic())
    with pytest.raises(NotImplementedError, match="mean function"):
        m.elbo_and_grad()
    m = gpf.models.VGP(data, K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1))
    m.kernel.variance.prior = object()
    with pytest.raises(NotImplementedError, match="prior"):
        gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options={"maxiter": 2})
