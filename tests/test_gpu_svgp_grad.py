"""Device value and gradient of the SVGP ELBO for any fused kernel expression, both whiten and both q_diag settings, the
inducing points, the variational parameters and the Constant / Linear mean functions (gpk_svgp_elbo_grad:
csrc/fused.cu::svgp_elbo_grad, the passes of csrc/grad.cu::inducing_grad_launch) against the oracle
(tests/svgp_grad_oracle.py::svgp_elbo_and_grad, pinned by finite differences in tests/test_oracle_svgp_grad.py),
the value entry point, the SGPR gradient at the optimal q(u), finite differences of the device ELBO at the C4 shape,
an L-BFGS-B run and a minibatch loop."""
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S
from tests.sgpr_grad_oracle import optimal_q

pytestmark = pytest.mark.gpu

K = gpf.kernels


def _model(kp, Z, q_mu, q_sqrt, whiten, q_diag, s2, num_data=None, mp=None):
    return gpf.models.SVGP(kp, gpf.likelihoods.Gaussian(s2), Z.copy(), num_latent_gps=q_mu.shape[1], q_mu=q_mu.copy(),
                           q_sqrt=q_sqrt.copy(), whiten=whiten, q_diag=q_diag, num_data=num_data, mean_function=mp)


def _check(m, X, Y, ko, Z, q_mu, q_sqrt, s2, mo=None, rtol=1e-6):
    elbo, grads = m.elbo_and_grad((X, Y))
    ref_elbo, g = S.svgp_elbo_and_grad(X, Y, [ko], [Z], q_mu, q_sqrt, LO.Gaussian(s2), whiten=m.whiten,
                                       num_data=m.num_data, mean_function=mo, jitter=gpf.config.default_jitter())
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-8)
    ref = GC.reference_by_param(g, [m.kernel], m.mean_function, [
        (m.likelihood.variance, g["lik"]), (m.inducing_variable.Z, g["Z"]), (m.q_mu, g["q_mu"]),
        (m.q_sqrt, g["q_sqrt"])])
    GC.assert_grads_match(grads, ref, rtol, "parameter")
    if not m.q_diag:
        dq = grads[m.q_sqrt]
        assert np.all(dq[:, np.triu_indices(dq.shape[1], 1)[0], np.triu_indices(dq.shape[1], 1)[1]] == 0.0)


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("name,B,M,D,P,num_data", [
    ("rbf_plus_white", 600, 17, 3, 1, None), ("c5", 500, 64, 8, 3, 20000), ("c5", 400, 200, 8, 1, None),
    ("rq_ard", 300, 64, 4, 3, None), ("polynomial_ard", 500, 17, 4, 1, 5000), ("linear_ard", 400, 64, 4, 1, None),
    ("constant_times_matern52", 300, 200, 5, 3, 10000), ("additive_active_dims", 700, 64, 4, 1, None),
    ("k_plus_k", 300, 17, 4, 3, None)])
def test_svgp_grad_matches_oracle(cuda_device, name, B, M, D, P, num_data, whiten, q_diag):
    d = O.make_data(5, B, D, P)
    Z = GC.z(M, D)
    q_mu, q_sqrt = GC.q(M, P, q_diag)
    kp, ko = GC.case(name, D)
    m = _model(kp, Z, q_mu, q_sqrt, whiten, q_diag, 0.15, num_data)
    _check(m, d["X"], d["Y"], ko, Z, q_mu, q_sqrt, 0.15)


@pytest.mark.parametrize("kernel", ["matern12", "rbf"])
def test_coincident_inducing_points(cuda_device, kernel):
    """Z = X[:M]: every stationary leaf's derivative at a coincident pair is exactly 0 (the 1e-36 clip passes none)."""
    d = O.make_data(4, 800, 3, 2)
    Z = d["X"][:64].copy()
    if kernel == "matern12":
        kp, ko = K.Matern12(variance=0.9, lengthscales=1.4), O.Matern12(0.9, 1.4)
    else:
        kp, ko = K.SquaredExponential(variance=1.2, lengthscales=1.1), O.SquaredExponential(1.2, 1.1)
    q_mu, q_sqrt = GC.q(64, 2, False)
    m = _model(kp, Z, q_mu, q_sqrt, True, False, 0.1, 8000)
    _check(m, d["X"], d["Y"], ko, Z, q_mu, q_sqrt, 0.1)


@pytest.mark.parametrize("with_mean", [False, True])
@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, True)])
def test_value_entry_point_agrees_with_the_gradient_entry_point(cuda_device, whiten, q_diag, with_mean):
    """out[0..3] of gpk_svgp_elbo_grad against gpk_svgp_elbo on the same inputs: a Gaussian descriptor, the raw Y and
    m(X) [B, P] apart (or NULL)."""
    lib = _lib.load()
    T = ops.torch()
    B, M, D, P = 1000, 200, 8, 3
    d = O.make_data(5, B, D, P)
    X, Y, Z = ops.to_device(d["X"]), ops.to_device(d["Y"]), ops.to_device(GC.z(M, D))
    q_mu, q_sqrt = (ops.to_device(a) for a in GC.q(M, P, q_diag))
    mX = ops.to_device(0.2 * np.sin(d["X"][:, :P]) + 0.1 * np.arange(1, P + 1)) if with_mean else None
    kp, _ = GC.case("c5", D)
    nodes, n, dims, ard = gpf.kernels.compile_kernel(kp, D)
    n_out = 5 + lib.gpk_gpr_lml_grad_slots(nodes, n, dims, ard, D)
    a = T.empty((4,), dtype=T.float64, device=X.device)
    b = T.empty((n_out,), dtype=T.float64, device=X.device)
    dZ = T.empty((M, D), dtype=T.float64, device=X.device)
    dq_mu, dq_sqrt = T.empty_like(q_mu), T.empty_like(q_sqrt)
    ws = ops.scratch_bytes(lib.gpk_svgp_elbo_ws(B, M, P, _lib.GPK_F64))
    gauss = ctypes.byref(_lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1))
    gws = ops.scratch_bytes(lib.gpk_svgp_elbo_grad_ws(B, M, P, gauss, _lib.GPK_F64))
    head = (nodes, n, dims, ard, ops._p(X), B, D, D, ops._p(Y))
    tail = (ops._p(Z), M, D, ops._p(q_mu), ops._p(q_sqrt), int(q_diag), int(whiten))
    _lib.check(lib.gpk_svgp_elbo(*head, ops._p(mX), P, *tail, gauss, 50.0, 1e-6, 0, P, _lib.GPK_F64, ops._p(a),
                                 ops._p(ws), ops._stream()), "gpk_svgp_elbo")
    _lib.check(lib.gpk_svgp_elbo_grad(*head, ops._p(mX), P, *tail, gauss, 50.0, 1e-6, _lib.GPK_F64, ops._p(b), n_out,
                                      ops._p(dZ), ops._p(dq_mu), ops._p(dq_sqrt), ops._p(gws), ops._stream()),
               "gpk_svgp_elbo_grad")
    a, b = a.cpu().numpy(), b.cpu().numpy()
    np.testing.assert_allclose(b[:4], a, rtol=1e-12)
    for t in (b, dZ, dq_mu, dq_sqrt):
        assert np.all(np.isfinite(np.asarray(t.cpu().numpy() if hasattr(t, "cpu") else t)))


@pytest.mark.parametrize("whiten", [True, False])
def test_envelope_identity_with_sgpr_on_the_device(cuda_device, whiten):
    """At the optimal q(u) of the collapsed bound, with num_data = N on the full data, the SVGP ELBO's kernel, noise and
    Z gradients are the SGPR bound's, and its q gradients vanish."""
    N, M, D, P = 800, 40, 3, 2
    d = O.make_data(6, N, D, P)
    Z = GC.z(M, D)
    kp = K.SquaredExponential(variance=1.3, lengthscales=1.7) + K.Linear(variance=0.3)
    ko = O.SquaredExponential(1.3, 1.7) + O.Linear(0.3)
    s2 = 0.2
    q_mu, q_sqrt = optimal_q(d["X"], d["Y"], ko, Z, s2, whiten, jitter=gpf.config.default_jitter())
    sv = _model(kp, Z, q_mu, q_sqrt, whiten, False, s2, N)
    sg = gpf.models.SGPR((d["X"], d["Y"]), kp, sv.inducing_variable.Z, noise_variance=s2)
    sg.likelihood = sv.likelihood
    e_sv, g_sv = sv.elbo_and_grad((d["X"], d["Y"]))
    e_sg, g_sg = sg.elbo_and_grad()
    np.testing.assert_allclose(float(e_sv), float(e_sg), rtol=1e-9)
    scale = max(float(np.max(np.abs(g))) for g in g_sg.values())
    assert len(g_sg) == len(g_sv) - 2   # the same keys but q_mu and q_sqrt; SGPR holds its own copy of Z
    for p, g in g_sg.items():
        q = sv.inducing_variable.Z if p is sg.inducing_variable.Z else p
        np.testing.assert_allclose(np.asarray(g_sv[q]), np.asarray(g), rtol=0, atol=1e-6 * scale)
    for p in (sv.q_mu, sv.q_sqrt):
        assert float(np.max(np.abs(g_sv[p]))) < 1e-6 * scale


@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("mean", ["constant", "linear"])
def test_mean_function_grads_match_oracle(cuda_device, whiten, mean):
    B, D, M, P = 600, 4, 40, 2
    d = O.make_data(3, B, D, P)
    rng = np.random.default_rng(11)
    if mean == "constant":
        c = 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    else:
        A, b = 0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    kp, ko = GC.case("c5", D)
    Z = GC.z(M, D)
    q_mu, q_sqrt = GC.q(M, P, False)
    m = _model(kp, Z, q_mu, q_sqrt, whiten, False, 0.2, 6000, mp)
    _check(m, d["X"], d["Y"], ko, Z, q_mu, q_sqrt, 0.2, mo)


def test_c4_full_size_finite_difference_of_device_elbo(cuda_device):
    """BASELINE config 4's shape in float64 (B = 4096, M = 2048, P = 8, D = 16, num_data = 1e6; RBF + White, whitened,
    dense q_sqrt): the analytic device gradient against central finite differences of the device ELBO along random
    directions of the kernel parameters, Z, q_mu and q_sqrt."""
    B, M, P, D = 4096, 2048, 8, 16
    d = O.make_data(4, B, D, P, M=M)
    q_mu, q_sqrt = O.make_q(4, M, P)
    data = (ops.to_device(d["X"]), ops.to_device(d["Y"]))
    rng = np.random.default_rng(12)
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
        kp = K.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) + K.White(variance=0.01)
        m = gpf.models.SVGP(kp, gpf.likelihoods.Gaussian(0.1), d["Z"], num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt,
                            whiten=True, num_data=1000000)
        _, grads = m.elbo_and_grad(data)
        rbf, white = kp.kernels
        groups = {
            "kernel": ([rbf.variance, rbf.lengthscales, white.variance], [0.3, 1.0, 0.002], 1e-4),
            "Z": ([m.inducing_variable.Z], [rng.standard_normal((M, D))], 1e-4),
            "q_mu": ([m.q_mu], [rng.standard_normal((M, P))], 1e-3),
            "q_sqrt": ([m.q_sqrt], [np.tril(rng.standard_normal((P, M, M)))], 1e-3),
        }
        for key, (params, dirs, t) in groups.items():
            dirs = [np.broadcast_to(np.asarray(dv, dtype=np.float64), p.shape) for p, dv in zip(params, dirs)]
            analytic = sum(float(np.sum(np.asarray(grads[p]).reshape(p.shape) * dv)) for p, dv in zip(params, dirs))
            fd = GC.fd_along(m, data, params, dirs, t)
            np.testing.assert_allclose(analytic, fd, rtol=1e-5, err_msg=key)


def test_scipy_trains_svgp_with_every_parameter_trainable(cuda_device):
    B, D, M, P = 500, 3, 15, 2
    d = O.make_data(5, B, D, P)
    Z = d["X"][:M].copy()
    k = K.SquaredExponential(variance=1.0, lengthscales=2.0) + K.Linear(variance=0.5)
    m = gpf.models.SVGP(k, gpf.likelihoods.Gaussian(1.0), Z, num_latent_gps=P, whiten=True)
    names = {id(m.q_mu), id(m.q_sqrt), id(m.inducing_variable.Z), id(m.likelihood.variance)}
    assert names <= {id(p) for p in m.trainable_parameters}
    data = (d["X"], d["Y"])
    loss0 = -float(m.elbo(data))
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(data), m.trainable_variables,
                                          options={"maxiter": 40})
    loss1 = -float(m.elbo(data))
    assert loss1 < loss0 - 1.0
    np.testing.assert_allclose(loss1, res.fun, rtol=1e-8)


def test_minibatch_loop_over_an_iterator(cuda_device):
    """value_and_gradients draws ONE batch per call and returns the loss and gradients of that batch, between small
    gradient steps on the stochastic gradients."""
    N, D, M, P, Bs = 1200, 3, 20, 1, 200
    d = O.make_data(7, N, D, P)
    X, Y = d["X"], d["Y"]
    m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=2.0), gpf.likelihoods.Gaussian(1.0),
                        X[:M].copy(), num_latent_gps=P, num_data=N)
    batches = [(X[i:i + Bs], Y[i:i + Bs]) for i in range(0, N, Bs)]
    closure = m.training_loss_closure(iter(batches))
    variables = m.trainable_variables
    for batch in batches:
        want = -float(m.elbo(batch))
        _, ref = m.training_loss_and_gradients(batch)
        loss, grads = closure.value_and_gradients(variables)
        np.testing.assert_allclose(loss, want, rtol=1e-10)
        scale = max(float(np.max(np.abs(r))) for r in ref)
        for p, g, r in zip(variables, grads, ref):
            np.testing.assert_allclose(np.asarray(g), np.asarray(r), rtol=0, atol=1e-9 * scale)
            p.assign_unconstrained(p.unconstrained_variable - 1e-5 * np.asarray(g).reshape(p.shape))
    with pytest.raises(StopIteration):   # one batch per call: the iterator is exhausted
        closure.value_and_gradients(variables)


class _NotGaussian(gpf.likelihoods.ScalarLikelihood):
    pass


class _Quadratic(gpf.mean_functions.MeanFunction):
    def __call__(self, X):
        return ops.to_device(X)[:, :1] * 0.0


def test_refusals(cuda_device):
    d = O.make_data(1, 200, 2, 1)
    Z = d["X"][:10].copy()
    data = (d["X"], d["Y"])
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = gpf.models.SVGP(K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1), Z.copy(), num_latent_gps=1)
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients(data)
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        m = gpf.models.SVGP(kern, gpf.likelihoods.Gaussian(0.1), Z.copy(), num_latent_gps=1)
        with pytest.raises(NotImplementedError, match=cls):
            m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SharedIndependent(K.SquaredExponential(), 1), gpf.likelihoods.Gaussian(0.1), Z.copy(),
                        num_latent_gps=1)
    with pytest.raises(NotImplementedError, match="single-output"):
        m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SquaredExponential(), _NotGaussian(), Z.copy(), num_latent_gps=1)
    with pytest.raises(NotImplementedError, match="Gaussian"):
        m.elbo_and_grad(data)
    lik = gpf.likelihoods.Gaussian(variance=gpf.mean_functions.Linear(A=np.array([[0.05], [0.0]]), b=np.array([0.08])))
    m = gpf.models.SVGP(K.SquaredExponential(), lik, Z.copy(), num_latent_gps=1)
    with pytest.raises(NotImplementedError):
        m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1), Z.copy(), num_latent_gps=1,
                        mean_function=_Quadratic())
    with pytest.raises(NotImplementedError, match="mean function"):
        m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SquaredExponential(), gpf.likelihoods.Gaussian(0.1), Z.copy(), num_latent_gps=1)
    m.kernel.variance.prior = object()
    with pytest.raises(NotImplementedError, match="prior"):
        gpf.optimizers.Scipy().minimize(m.training_loss_closure(data), m.trainable_variables, options={"maxiter": 2})
