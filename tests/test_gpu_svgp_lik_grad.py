"""Device value and gradient of the SVGP ELBO with Bernoulli / Poisson / StudentT likelihoods (gpk_svgp_elbo_grad:
csrc/fused.cu::svgp_elbo_grad, csrc/lik.cu) against the oracle (tests/lik_oracle.py, pinned by finite differences in
tests/test_oracle_likelihoods.py) and the unfused SVGP.elbo; the mean-shift convention of its Gaussian case;
finite differences of the device ELBO at the C4 shape; L-BFGS-B training of a Bernoulli classifier against the same run
driven by the oracle; a Student-t minibatch loop; and the refusals."""
import copy
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from gpflow_b200.base import Parameter
from oracle import gp_oracle as O
from tests import lik_oracle as LO
from tests.test_gpu_grad_expr import ATTRS, _case, _py_leaves
from tests.test_gpu_svgp_grad import _fd_along, _q, _z

pytestmark = pytest.mark.gpu

K = gpf.kernels
LIK = gpf.likelihoods


def _pair(name):
    if name == "bernoulli":
        return LIK.Bernoulli(), LO.Bernoulli()
    if name == "poisson":
        return LIK.Poisson(binsize=1.3), LO.Poisson(1.3)
    return LIK.StudentT(scale=0.7, df=4.0), LO.StudentT(0.7, 4.0)


def _reference(m, X, Y, ko, Z, q_mu, q_sqrt, lo, mo=None):
    """Oracle gradients keyed by id(Parameter), summed over the leaves a Parameter occurs in."""
    elbo, g = LO.svgp_elbo_lik_and_grad(X, Y, ko, Z, q_mu, q_sqrt, lo, whiten=m.whiten, num_data=m.num_data,
                                        mean_function=mo, jitter=gpf.config.default_jitter())
    ref = {id(m.inducing_variable.Z): g["Z"], id(m.q_mu): g["q_mu"], id(m.q_sqrt): g["q_sqrt"]}
    if isinstance(m.likelihood, LIK.StudentT):
        ref[id(m.likelihood.scale)] = np.asarray(g["lik"])
    for leaf, gd in zip(_py_leaves(m.kernel), g["leaves"]):
        for a in ATTRS:
            p = getattr(leaf, a, None)
            if isinstance(p, Parameter) and a in gd:
                v = np.asarray(gd[a], dtype=np.float64).reshape(p.shape)
                ref[id(p)] = ref[id(p)] + v if id(p) in ref else v
    mf = m.mean_function
    for name, v in g["mean"].items():
        ref[id(getattr(mf, name))] = np.asarray(v).reshape(getattr(mf, name).shape)
    return elbo, ref


def _check(m, X, Y, ko, Z, q_mu, q_sqrt, lo, mo=None, rtol=1e-6):
    elbo, grads = m.elbo_and_grad((X, Y))
    ref_elbo, ref = _reference(m, X, Y, ko, Z, q_mu, q_sqrt, lo, mo)
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-8)
    # out[0] is the unfused route's value (prior_kl, predict_f, variational_expectations)
    np.testing.assert_allclose(float(elbo), float(m.elbo((X, Y))), rtol=1e-12)
    assert {id(p) for p in grads} == set(ref)
    scale = max(float(np.max(np.abs(v))) for v in ref.values())
    for p, g in grads.items():
        g = np.asarray(g, dtype=np.float64).reshape(p.shape)
        assert np.all(np.isfinite(g))
        r = ref[id(p)]
        atol = rtol * max(float(np.max(np.abs(r))), 1e-3 * scale)
        np.testing.assert_allclose(g, r, rtol=0, atol=atol)


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("lik", ["bernoulli", "poisson", "student_t"])
@pytest.mark.parametrize("name,B,M,D,P,num_data", [
    ("rbf_plus_white", 400, 17, 3, 1, None), ("c5", 300, 64, 8, 3, 20000), ("rq_ard", 300, 200, 4, 1, 5000),
    ("constant_times_matern52", 250, 64, 5, 2, None)])
def test_svgp_lik_grad_matches_oracle(cuda_device, name, B, M, D, P, num_data, lik, whiten, q_diag):
    d = O.make_data(5, B, D, P)
    rng = np.random.default_rng(M + P)
    Y = LO.targets(lik, np.sin(d["X"][:, :1] @ np.ones((1, P))), rng)
    Z = _z(M, D)
    q_mu, q_sqrt = _q(M, P, q_diag)
    kp, ko = _case(name, D)
    lp, lo = _pair(lik)
    m = gpf.models.SVGP(kp, lp, Z.copy(), num_latent_gps=P, q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), whiten=whiten,
                        q_diag=q_diag, num_data=num_data)
    _check(m, d["X"], Y, ko, Z, q_mu, q_sqrt, lo)


@pytest.mark.parametrize("lik", ["bernoulli", "student_t"])
@pytest.mark.parametrize("mean", ["constant", "linear"])
def test_mean_function_grads_match_oracle(cuda_device, lik, mean):
    B, D, M, P = 400, 4, 30, 2
    d = O.make_data(3, B, D, P)
    rng = np.random.default_rng(11)
    Y = LO.targets(lik, np.sin(d["X"][:, :1] @ np.ones((1, P))), rng)
    if mean == "constant":
        c = np.array([0.3])
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    else:
        A, b = 0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    kp, ko = _case("c5", D)
    Z = _z(M, D)
    q_mu, q_sqrt = _q(M, P, False)
    lp, lo = _pair(lik)
    m = gpf.models.SVGP(kp, lp, Z.copy(), num_latent_gps=P, q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), num_data=6000,
                        mean_function=mp)
    _check(m, d["X"], Y, ko, Z, q_mu, q_sqrt, lo, mo)


def _lik_grad_call(lib, desc, kp, X, Y, mX, Z, q_mu, q_sqrt, q_diag, whiten, scale):
    B, D = X.shape
    M, P = Z.shape[0], Y.shape[1]
    nodes, n_nodes, dims, ard = K.compile_kernel(kp, D)
    n_out = 5 + lib.gpk_gpr_lml_grad_slots(nodes, n_nodes, dims, ard, D)
    T = ops.torch()
    out = T.empty((n_out,), dtype=T.float64, device=X.device)
    dZ, dq_mu, dq_sqrt = (T.empty(tuple(a.shape), dtype=T.float64, device=X.device) for a in (Z, q_mu, q_sqrt))
    ws = ops.scratch_bytes(lib.gpk_svgp_elbo_grad_ws(B, M, P, ctypes.byref(desc), _lib.GPK_F64))
    _lib.check(lib.gpk_svgp_elbo_grad(nodes, n_nodes, dims, ard, ops._p(X), B, ops._ld(X), D, ops._p(Y), ops._p(mX), P,
                                      ops._p(Z), M, ops._ld(Z), ops._p(q_mu), ops._p(q_sqrt), int(q_diag), int(whiten),
                                      ctypes.byref(desc), scale, 1e-6, _lib.GPK_F64, ops._p(out), n_out, ops._p(dZ),
                                      ops._p(dq_mu), ops._p(dq_sqrt), ops._p(ws), ops._stream()), "gpk_svgp_elbo_grad")
    dm = ws[lib.gpk_svgp_elbo_grad_dm(B, M, P, _lib.GPK_F64):][:8 * B * P].view(T.float64).view(B, P)
    return [a.cpu().numpy() for a in (out, dZ, dq_mu, dq_sqrt, dm)]


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("M", [17, 64, 200])
def test_gaussian_descriptor_with_mean_equals_centred_targets(cuda_device, M, whiten, q_diag):
    """The Gaussian descriptor with raw Y and m(X) apart against the same entry with Y - m(X) and no mean: every
    output.  This pins the mean-shift convention SVGP uses for every likelihood, Gaussian included."""
    B, D, P = 500, 4, 2
    d = O.make_data(6, B, D, P)
    kp, _ = _case("c5", D)
    Z = ops.to_device(_z(M, D))
    q_mu, q_sqrt = (ops.to_device(a) for a in _q(M, P, q_diag))
    X, Y = ops.to_device(d["X"]), ops.to_device(d["Y"])
    mX = ops.to_device(np.tile(np.array([[0.2, -0.1]]), (B, 1)))
    Yc = ops.to_device(d["Y"] - np.array([[0.2, -0.1]]))
    lib = _lib.load()
    desc = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.15)
    got = _lik_grad_call(lib, desc, kp, X, Y, mX, Z, q_mu, q_sqrt, q_diag, whiten, 7.0)
    want = _lik_grad_call(lib, desc, kp, X, Yc, None, Z, q_mu, q_sqrt, q_diag, whiten, 7.0)
    for what, a, b in zip(["out", "dZ", "dq_mu", "dq_sqrt", "dm"], got, want):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12 * max(1.0, float(np.max(np.abs(b)))), err_msg=what)


def test_c4_full_size_finite_difference_of_device_elbo(cuda_device):
    """The C4 shape in float64 (B = 4096, M = 2048, D = 16, num_data = 1e6; RBF + White, whitened, dense q_sqrt) with a
    Bernoulli likelihood at P = 1: the analytic device gradient against central finite differences of the device ELBO
    (the unfused route) along random directions of the kernel parameters, Z, q_mu and q_sqrt."""
    B, M, P, D = 4096, 2048, 1, 16
    d = O.make_data(4, B, D, P, M=M)
    q_mu, q_sqrt = O.make_q(4, M, P)
    rng = np.random.default_rng(12)
    Y = (d["Y"] + 0.3 * rng.standard_normal(d["Y"].shape) > np.median(d["Y"])).astype(np.float64)
    data = (ops.to_device(d["X"]), ops.to_device(Y))
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
        kp = K.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) + K.White(variance=0.01)
        m = gpf.models.SVGP(kp, LIK.Bernoulli(), d["Z"], num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt, whiten=True,
                            num_data=1000000)
        elbo, grads = m.elbo_and_grad(data)
        np.testing.assert_allclose(float(elbo), float(m.elbo(data)), rtol=1e-12)
        rbf, white = kp.kernels
        groups = {
            "kernel": ([rbf.variance, rbf.lengthscales, white.variance], [0.3, 1.0, 0.002], 1e-4),
            "Z": ([m.inducing_variable.Z], [rng.standard_normal((M, D))], 1e-4),
            "q_mu": ([m.q_mu], [rng.standard_normal((M, P))], 1e-3),
            # unlike the Gaussian ELBO, the Bernoulli one is not quadratic in q_sqrt: a shorter step keeps the central
            # difference's t^2 term under the tolerance
            "q_sqrt": ([m.q_sqrt], [np.tril(rng.standard_normal((P, M, M)))], 2.5e-4),
        }
        for key, (params, dirs, t) in groups.items():
            dirs = [np.broadcast_to(np.asarray(dv, dtype=np.float64), p.shape) for p, dv in zip(params, dirs)]
            analytic = sum(float(np.sum(np.asarray(grads[p]).reshape(p.shape) * dv)) for p, dv in zip(params, dirs))
            fd = _fd_along(m, data, params, dirs, t)
            np.testing.assert_allclose(analytic, fd, rtol=1e-5, err_msg=key)


def _classifier(X, Z):
    return gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=1.0), LIK.Bernoulli(), Z.copy(),
                           num_latent_gps=1, whiten=True)


def test_scipy_trains_a_bernoulli_classifier(cuda_device):
    """L-BFGS-B with Z, the kernel and q trainable on 2-D data split by a line, against the same run whose value and
    gradient come from the oracle.  The labels carry noise near the line: on labels that are exactly separable the ELBO
    keeps rising as the latent function steepens, and the optimiser has no optimum to converge to."""
    rng = np.random.default_rng(21)
    N, M = 200, 12
    X = rng.standard_normal((N, 2))
    clean = X[:, :1] + 0.7 * X[:, 1:] > 0
    Y = (X[:, :1] + 0.7 * X[:, 1:] + 0.3 * rng.standard_normal((N, 1)) > 0).astype(np.float64)
    Z = X[:M].copy()
    data = (X, Y)
    m = _classifier(X, Z)
    loss0 = -float(m.elbo(data))
    opts = {"maxiter": 2000}
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(data), m.trainable_variables, options=opts)
    loss1 = -float(m.elbo(data))
    assert res.success, res.message
    assert loss1 < loss0 - 10.0
    np.testing.assert_allclose(loss1, res.fun, rtol=1e-10)
    pm, _ = m.predict_y(X)
    acc = float(np.mean((pm.cpu().numpy() > 0.5) == clean))
    assert acc > 0.95, acc

    o = _classifier(X, Z)
    lo = LO.Bernoulli()

    def oracle_objective_and_grad(batch):
        rbf = o.kernel
        ko = O.SquaredExponential(float(rbf.variance.numpy()), float(rbf.lengthscales.numpy()))
        Zv, qm, qs = (np.asarray(p.numpy(), dtype=np.float64) for p in (o.inducing_variable.Z, o.q_mu, o.q_sqrt))
        elbo, g = LO.svgp_elbo_lik_and_grad(X, Y, ko, Zv, qm, qs, lo, whiten=True,
                                            jitter=gpf.config.default_jitter())
        grads = {o.inducing_variable.Z: g["Z"], o.q_mu: g["q_mu"], o.q_sqrt: g["q_sqrt"],
                 rbf.variance: np.asarray(g["leaves"][0]["variance"]),
                 rbf.lengthscales: np.asarray(g["leaves"][0]["lengthscales"])}
        return elbo, grads

    o._objective_and_grad = oracle_objective_and_grad
    res_o = gpf.optimizers.Scipy().minimize(o.training_loss_closure(data), o.trainable_variables, options=opts)
    assert res_o.success, res_o.message
    # the bound is flat along Z and q here: where L-BFGS-B's default stopping rule ends a converged run moves by up to a
    # few 1e-5 (the device run itself is not bitwise repeatable: its reductions add through atomics), and tighter
    # tolerances run into the iteration limit with the bound still creeping down by 1e-5 per thousand steps
    np.testing.assert_allclose(res.fun, res_o.fun, rtol=1e-4)


def test_student_t_minibatch_loop_over_an_iterator(cuda_device):
    """value_and_gradients draws ONE batch per call and returns the loss and gradients of that batch, the Student-t
    scale included, between small gradient steps."""
    N, D, M, P, Bs = 1200, 3, 20, 1, 200
    d = O.make_data(7, N, D, P)
    X = d["X"]
    Y = d["Y"] + 0.3 * np.random.default_rng(3).standard_t(3.0, d["Y"].shape)
    m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=2.0), LIK.StudentT(scale=0.5), X[:M].copy(),
                        num_latent_gps=P, num_data=N)
    assert id(m.likelihood.scale) in {id(p) for p in m.trainable_parameters}
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
    with pytest.raises(StopIteration):
        closure.value_and_gradients(variables)


class _NotGaussian(gpf.likelihoods.ScalarLikelihood):
    pass


def test_refusals(cuda_device):
    d = O.make_data(1, 200, 2, 1)
    Z = d["X"][:10].copy()
    Yb = (d["Y"] > 0).astype(np.float64)
    data = (d["X"], Yb)
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = gpf.models.SVGP(K.SquaredExponential(), LIK.Bernoulli(), Z.copy(), num_latent_gps=1)
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients(data)
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        m = gpf.models.SVGP(kern, LIK.Poisson(), Z.copy(), num_latent_gps=1)
        with pytest.raises(NotImplementedError, match=cls):
            m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SharedIndependent(K.SquaredExponential(), 1), LIK.StudentT(), Z.copy(), num_latent_gps=1)
    with pytest.raises(NotImplementedError, match="single-output"):
        m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SquaredExponential(), _NotGaussian(), Z.copy(), num_latent_gps=1)
    with pytest.raises(NotImplementedError, match="Gaussian"):
        m.elbo_and_grad(data)
    with pytest.raises(NotImplementedError, match="Function"):
        LIK.StudentT(scale=gpf.mean_functions.Constant(np.array([0.5])))
    with pytest.raises(NotImplementedError, match="probit"):
        LIK.Bernoulli(invlink=copy.copy(np.exp))
    # VGP keeps its Gaussian-only gradient
    m = gpf.models.VGP(data, K.SquaredExponential(), LIK.Bernoulli())
    with pytest.raises(NotImplementedError):
        m.elbo_and_grad()
