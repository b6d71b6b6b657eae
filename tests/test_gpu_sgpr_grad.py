"""Device value and gradient of the SGPR bound for any fused kernel expression, the inducing points and the Constant /
Linear mean functions (gpk_sgpr_elbo_grad: csrc/fused.cu::sgpr_elbo_grad, csrc/grad.cu::sgpr_grad_kernel) against the
oracle (tests/sgpr_grad_oracle.py::sgpr_elbo_and_grad_expr, pinned by finite differences in
tests/test_oracle_sgpr_grad.py), the value entry point, finite differences of the device ELBO at the C3 shape, and an
L-BFGS-B run with trainable inducing points."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from gpflow_b200.base import Parameter
from oracle import gp_oracle as O
from tests import sgpr_grad_oracle as S
from tests.test_gpu_grad_expr import ATTRS, _case, _py_leaves

pytestmark = pytest.mark.gpu

K = gpf.kernels


def _z(M, D, seed=3):
    return 1.1 * np.random.default_rng(seed).standard_normal((M, D))


def _reference(m, X, Y, ko, Z, s2, mo=None):
    """Oracle gradients keyed by id(Parameter), summed over the leaves a Parameter occurs in."""
    elbo, g = S.sgpr_elbo_and_grad_expr(X, Y, ko, Z, s2, mean_function=mo, jitter=gpf.config.default_jitter())
    ref = {id(m.likelihood.variance): np.asarray(g["noise_variance"]), id(m.inducing_variable.Z): g["Z"]}
    pl = _py_leaves(m.kernel)
    assert len(pl) == len(g["leaves"])
    for leaf, gd in zip(pl, g["leaves"]):
        for a in ATTRS:
            p = getattr(leaf, a, None)
            if isinstance(p, Parameter) and a in gd:
                v = np.asarray(gd[a], dtype=np.float64).reshape(p.shape)
                ref[id(p)] = ref[id(p)] + v if id(p) in ref else v
    mf = m.mean_function
    for name, v in g["mean"].items():
        ref[id(getattr(mf, name))] = np.asarray(v).reshape(getattr(mf, name).shape)
    return elbo, ref


def _check(m, X, Y, ko, Z, s2, mo=None, rtol=1e-6):
    elbo, grads = m.elbo_and_grad()
    ref_elbo, ref = _reference(m, X, Y, ko, Z, s2, mo)
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-8)
    assert {id(p) for p in grads} == set(ref)
    for p, g in grads.items():
        assert np.all(np.isfinite(g))
    scale = max(float(np.max(np.abs(v))) for v in ref.values())
    for p, g in grads.items():
        np.testing.assert_allclose(np.asarray(g, dtype=np.float64).reshape(p.shape), ref[id(p)], rtol=0,
                                   atol=rtol * scale)


@pytest.mark.parametrize("name,N,M,D,P", [
    ("rbf_plus_white", 1500, 17, 3, 1), ("c5", 2000, 64, 8, 1), ("c5", 1200, 200, 8, 2), ("rq", 900, 17, 3, 2),
    ("rq_ard", 1000, 64, 4, 1), ("polynomial_ard", 1500, 17, 4, 1), ("linear_ard", 1000, 64, 4, 2),
    ("constant_times_matern52", 1200, 200, 5, 1), ("additive_active_dims", 2500, 64, 4, 1), ("k_plus_k", 800, 17, 4, 1)])
def test_sgpr_grad_matches_oracle(cuda_device, name, N, M, D, P):
    d = O.make_data(5, N, D, P)
    Z = _z(M, D)
    kp, ko = _case(name, D)
    m = gpf.models.SGPR((d["X"], d["Y"]), kp, Z.copy(), noise_variance=0.15)
    _check(m, d["X"], d["Y"], ko, Z, 0.15)


@pytest.mark.parametrize("kernel", ["matern12", "rbf"])
def test_coincident_inducing_points(cuda_device, kernel):
    """Z = X[:M]: every stationary leaf's derivative at a coincident pair is exactly 0 (the 1e-36 clip passes none)."""
    d = O.make_data(4, 1000, 3, 1)
    Z = d["X"][:64].copy()
    if kernel == "matern12":
        kp, ko = K.Matern12(variance=0.9, lengthscales=1.4), O.Matern12(0.9, 1.4)
    else:
        kp, ko = K.SquaredExponential(variance=1.2, lengthscales=1.1), O.SquaredExponential(1.2, 1.1)
    m = gpf.models.SGPR((d["X"], d["Y"]), kp, Z.copy(), noise_variance=0.1)
    _check(m, d["X"], d["Y"], ko, Z, 0.1)


def test_value_agrees_with_the_value_entry_point(cuda_device):
    """out[0..7] of gpk_sgpr_elbo_grad against gpk_sgpr_elbo on the same inputs."""
    lib = _lib.load()
    T = ops.torch()
    N, M, D, P = 3000, 200, 8, 2
    d = O.make_data(5, N, D, P)
    X, Y, Z = ops.to_device(d["X"]), ops.to_device(d["Y"]), ops.to_device(_z(M, D))
    kp, _ = _case("c5", D)
    nodes, n, dims, ard = gpf.kernels.compile_kernel(kp, D)
    n_out = 9 + lib.gpk_gpr_lml_grad_slots(nodes, n, dims, ard, D)
    a = T.empty((8,), dtype=T.float64, device=X.device)
    b = T.empty((n_out,), dtype=T.float64, device=X.device)
    dZ = T.empty((M, D), dtype=T.float64, device=X.device)
    ws = ops.scratch_bytes(lib.gpk_sgpr_elbo_ws(N, M, P, _lib.GPK_F64))
    gws = ops.scratch_bytes(lib.gpk_sgpr_elbo_grad_ws(N, M, P, _lib.GPK_F64))
    _lib.check(lib.gpk_sgpr_elbo(nodes, n, dims, ard, ops._p(X), N, D, D, ops._p(Y), P, ops._p(Z), M, D, 0.1, 1e-6,
                                 _lib.GPK_F64, ops._p(a), None, None, None, ops._p(ws), ops._stream()), "gpk_sgpr_elbo")
    _lib.check(lib.gpk_sgpr_elbo_grad(nodes, n, dims, ard, ops._p(X), N, D, D, ops._p(Y), P, ops._p(Z), M, D, 0.1, 1e-6,
                                      _lib.GPK_F64, ops._p(b), n_out, ops._p(dZ), ops._p(gws), ops._stream()),
               "gpk_sgpr_elbo_grad")
    a, b = a.cpu().numpy(), b.cpu().numpy()
    np.testing.assert_allclose(b[:8], a, rtol=1e-12)
    assert np.all(np.isfinite(b)) and np.all(np.isfinite(dZ.cpu().numpy()))


@pytest.mark.parametrize("kernel", ["matern52", "c5"])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("mean", ["constant", "linear"])
def test_mean_function_grads_match_oracle(cuda_device, kernel, P, mean):
    N, D, M = 800, 4, 40
    d = O.make_data(3, N, D, P)
    rng = np.random.default_rng(11)
    if mean == "constant":
        c = 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    else:
        A, b = 0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    if kernel == "matern52":
        kp, ko = K.Matern52(variance=1.1, lengthscales=1.9), O.Matern52(1.1, 1.9)
    else:
        kp, ko = _case("c5", D)
    Z = _z(M, D)
    m = gpf.models.SGPR((d["X"], d["Y"]), kp, Z.copy(), mean_function=mp, noise_variance=0.2)
    _check(m, d["X"], d["Y"], ko, Z, 0.2, mo)


def test_c3_full_size_finite_difference_of_device_elbo(cuda_device):
    """BASELINE configs[2] in float64 (RBF, N = 100000, M = 1024, D = 16): the analytic device gradient against a
    central finite difference of the device ELBO along the lengthscale, the variance, the noise variance and the three
    entries of Z with the largest gradients."""
    N, M, D = 100000, 1024, 16
    d = O.make_data(3, N, D, 1, M=M)
    X, Y = ops.to_device(d["X"]), ops.to_device(d["Y"])
    Z0 = d["Z"]
    s = float(np.sqrt(D))

    def model(ell=s, var=1.0, s2=0.1, Z=Z0):
        return gpf.models.SGPR((X, Y), K.SquaredExponential(variance=var, lengthscales=ell), Z.copy(), noise_variance=s2)

    m = model()
    _, grads = m.elbo_and_grad()
    base = dict(ell=s, var=1.0, s2=0.1)
    for key, p in [("ell", m.kernel.lengthscales), ("var", m.kernel.variance), ("s2", m.likelihood.variance)]:
        h = 1e-4 * base[key]
        hi, lo = dict(base), dict(base)
        hi[key] += h
        lo[key] -= h
        fd = (float(model(**hi).elbo()) - float(model(**lo).elbo())) / (2 * h)
        np.testing.assert_allclose(float(grads[p]), fd, rtol=1e-5, err_msg=key)
    gz = grads[m.inducing_variable.Z]
    for flat in np.argsort(-np.abs(gz).reshape(-1))[:3]:
        idx = np.unravel_index(flat, gz.shape)
        h = 1e-3
        Zp, Zm = Z0.copy(), Z0.copy()
        Zp[idx] += h
        Zm[idx] -= h
        fd = (float(model(Z=Zp).elbo()) - float(model(Z=Zm).elbo())) / (2 * h)
        np.testing.assert_allclose(float(gz[idx]), fd, rtol=1e-5, err_msg=str(idx))


def test_scipy_trains_sgpr_with_trainable_inducing_points_and_linear_mean(cuda_device):
    N, D, M = 600, 3, 15
    d = O.make_data(5, N, D, 1)
    Z = d["X"][:M].copy()
    k = K.SquaredExponential(variance=1.0, lengthscales=2.0) + K.Linear(variance=0.5)
    mf = gpf.mean_functions.Linear(np.zeros((D, 1)), np.zeros(1))
    m = gpf.models.SGPR((d["X"], d["Y"]), k, Z, mean_function=mf, noise_variance=1.0)
    assert any(p is m.inducing_variable.Z for p in m.trainable_parameters)
    loss0 = -float(m.elbo())
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options={"maxiter": 25})
    loss1 = -float(m.elbo())
    assert loss1 < loss0 - 1.0
    np.testing.assert_allclose(loss1, res.fun, rtol=1e-8)
    _, grads = m.training_loss_and_gradients()
    rbf, lin = k.kernels
    ko = O.SquaredExponential(float(rbf.variance.numpy()), float(rbf.lengthscales.numpy())) \
        + O.Linear(float(lin.variance.numpy()))
    mo = O.LinearMean(mf.A.numpy().copy(), mf.b.numpy().copy())
    Zf = np.asarray(m.inducing_variable.Z.numpy()).copy()
    _, ref = _reference(m, d["X"], d["Y"], ko, Zf, float(m.likelihood.variance.numpy()), mo)
    want = [-p.unconstrained_gradient(ref[id(p)]) for p in m.trainable_parameters]
    scale = max(float(np.max(np.abs(w))) for w in want)
    for p, gu, w in zip(m.trainable_parameters, grads, want):
        np.testing.assert_allclose(np.asarray(gu).reshape(-1), np.asarray(w).reshape(-1), rtol=1e-5, atol=1e-6 * scale)


def test_refusals(cuda_device):
    d = O.make_data(1, 200, 2, 1)
    Z = d["X"][:10].copy()
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = gpf.models.SGPR((d["X"], d["Y"]), K.SquaredExponential(), Z.copy(), noise_variance=0.1)
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients()
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic")]:
        m = gpf.models.SGPR((d["X"], d["Y"]), kern, Z.copy(), noise_variance=0.1)
        with pytest.raises(NotImplementedError, match=cls):
            m.elbo_and_grad()
    lik = gpf.likelihoods.Gaussian(variance=gpf.mean_functions.Linear(A=np.array([[0.05], [0.0]]), b=np.array([0.08])))
    m = gpf.models.SGPR((d["X"], d["Y"]), K.SquaredExponential(), Z.copy(), likelihood=lik)
    with pytest.raises(NotImplementedError):
        m.training_loss_and_gradients()
    f = gpf.models.GPRFITC((d["X"], d["Y"]), K.SquaredExponential(), Z.copy(), noise_variance=0.1)
    with pytest.raises(NotImplementedError, match="fitc"):
        f.training_loss_and_gradients()
    with pytest.raises(NotImplementedError):
        gpf.optimizers.Scipy().minimize(f.training_loss_closure(), f.trainable_variables, options={"maxiter": 2})
