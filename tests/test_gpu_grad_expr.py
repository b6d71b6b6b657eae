"""Device gradient of the GPR LML for any fused kernel expression (gpk_gpr_lml_grad_expr, csrc/grad.cu::
gpr_grad_expr_kernel) and of the Constant / Linear mean functions, against the expression oracle
(tests/grad_expr_oracle.py::gpr_lml_and_grad_expr, pinned by finite differences in tests/test_oracle_grad_expr.py)."""
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import grad_expr_oracle as G

pytestmark = pytest.mark.gpu

K = gpf.kernels


def _check(m, X, Y, ko, s2, mo=None, rtol=1e-6):
    lml, grads = m.log_marginal_likelihood_and_grad()
    ref_lml, g = G.gpr_lml_and_grad_expr(X, Y, ko, s2, mean_function=mo)
    # the value comes from the forward path (norm-expansion K-build): with Matern12 / Exponential leaves its diagonal
    # rounding noise under the square root moves the LML by a few 1e-9 relative
    np.testing.assert_allclose(float(lml), ref_lml, rtol=2e-8)
    ref = GC.reference_by_param(g, [m.kernel], m.mean_function, [(m.likelihood.variance, g["noise_variance"])])
    GC.assert_grads_match(grads, ref, rtol, "model")


@pytest.mark.parametrize("name,N,D,P", [
    ("rbf_plus_white", 300, 3, 1), ("c5", 700, 8, 1), ("c5", 1500, 8, 2), ("rq", 400, 3, 2), ("rq_ard", 500, 4, 1),
    ("polynomial_ard", 500, 4, 1), ("linear_ard", 600, 4, 2), ("constant_times_matern52", 600, 5, 1),
    ("additive_active_dims", 800, 4, 1), ("k_plus_k", 300, 4, 1)])
def test_expr_grad_matches_oracle(cuda_device, name, N, D, P):
    d = O.make_data(5, N, D, P)
    kp, ko = GC.case(name, D)
    m = gpf.models.GPR((d["X"], d["Y"]), kp, noise_variance=0.15)
    _check(m, d["X"], d["Y"], ko, 0.15)


@pytest.mark.parametrize("kernel", ["matern52", "c5"])
@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("mean", ["constant", "constant_per_output", "linear", "linear_one_column"])
def test_mean_function_grads_match_oracle(cuda_device, kernel, P, mean):
    N, D = 500, 4
    d = O.make_data(3, N, D, P)
    rng = np.random.default_rng(11)
    if mean == "constant":
        mp, mo = gpf.mean_functions.Constant(np.array([0.3])), O.ConstantMean(np.array([0.3]))
    elif mean == "constant_per_output":
        c = 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    elif mean == "linear":
        A, b = 0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    else:
        A, b = 0.2 * rng.standard_normal((D, 1)), np.array([0.4])
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    if kernel == "matern52":  # a single stationary leaf: gpr_grad_kernel, alpha read from the same workspace
        kp, ko = K.Matern52(variance=1.1, lengthscales=1.9), O.Matern52(1.1, 1.9)
    else:
        kp, ko = GC.case("c5", D)
    m = gpf.models.GPR((d["X"], d["Y"]), kp, mean_function=mp, noise_variance=0.2)
    _check(m, d["X"], d["Y"], ko, 0.2, mo)


def _under_one_child_sum(nodes, n):
    """The node array with a Sum node over its root appended: the same kernel, but no longer a bare leaf."""
    wrapped = (_lib.KNode * (n + 1))()
    ctypes.memmove(wrapped, nodes, ctypes.sizeof(_lib.KNode) * n)
    wrapped[n].op = _lib.K_SUM
    wrapped[n].n_children = 1
    wrapped[n].child[0] = n - 1
    return wrapped, n + 1


def test_single_leaf_kernel_agrees_with_expression_kernel(cuda_device):
    """gpk_gpr_lml_grad_expr on one bare stationary leaf (n_nodes = 1: gpr_grad_kernel) against the same leaf under a
    one-child Sum (n_nodes = 2: gpr_grad_expr_kernel), same inputs, within 1e-10 of the largest component."""
    lib = _lib.load()
    T = ops.torch()
    for kp, nl in [(K.Matern52(variance=1.2, lengthscales=1.7), 1), (K.SquaredExponential(lengthscales=GC.ELL4), 4),
                   (K.Matern12(variance=0.8, lengthscales=1.3), 1)]:
        d = O.make_data(2, 900, 4, 2)
        X, Y = ops.to_device(d["X"]), ops.to_device(d["Y"])
        N, D, P = 900, 4, 2
        nodes, n, dims, ard = gpf.kernels.compile_kernel(kp, D)
        assert n == 1
        ws = ops.scratch_bytes(lib.gpk_gpr_lml_grad_ws(N, P, _lib.GPK_F64))
        res = []
        for nd, nn in [(nodes, n), _under_one_child_sum(nodes, n)]:
            out = T.empty((5 + 1 + nl,), dtype=T.float64, device=X.device)
            _lib.check(lib.gpk_gpr_lml_grad_expr(nd, nn, dims, ard, ops._p(X), N, D, D, ops._p(Y), P, 0.1,
                                                 _lib.GPK_F64, ops._p(out), 6 + nl, ops._p(ws), ops._stream()),
                       "gpk_gpr_lml_grad_expr")
            res.append(out.cpu().numpy())
        a, b = res
        np.testing.assert_allclose(b[:3], a[:3], rtol=1e-12)
        scale = np.max(np.abs(a[4:]))
        np.testing.assert_allclose(b[4:], a[4:], rtol=0, atol=1e-10 * scale)


def test_c5_full_size_finite_difference_of_device_lml(cuda_device):
    """BASELINE configs[4], output 0 (N = 4096, D = 32: 32 staged columns): the analytic device gradient against a central
    finite difference of the device LML along the RBF lengthscale, the Matern32 variance, the Linear variance and the
    noise variance."""
    d = O.make_data(5, 4096, 32, 4)
    X, Y = d["X"], np.ascontiguousarray(d["Y"][:, :1])
    s = float(np.sqrt(32))

    def model(l_rbf=s, v_m32=1.0, v_lin=1.0, s2=0.1):
        k = (K.SquaredExponential(variance=1.0, lengthscales=l_rbf) + K.Matern32(variance=v_m32, lengthscales=2 * s)) \
            * K.Linear(variance=v_lin)
        return gpf.models.GPR((X, Y), k, noise_variance=s2)

    m = model()
    _, grads = m.log_marginal_likelihood_and_grad()
    rbf, m32 = m.kernel.kernels[0].kernels
    lin = m.kernel.kernels[1]
    base = dict(l_rbf=s, v_m32=1.0, v_lin=1.0, s2=0.1)
    for key, p in [("l_rbf", rbf.lengthscales), ("v_m32", m32.variance), ("v_lin", lin.variance),
                   ("s2", m.likelihood.variance)]:
        h = 1e-4 * base[key]
        hi, lo = dict(base), dict(base)
        hi[key] += h
        lo[key] -= h
        fd = (float(model(**hi).log_marginal_likelihood()) - float(model(**lo).log_marginal_likelihood())) / (2 * h)
        np.testing.assert_allclose(float(grads[p]), fd, rtol=1e-5, err_msg=key)


def test_scipy_trains_c5_shaped_kernel_with_linear_mean(cuda_device):
    N, D = 500, 4
    d = O.make_data(5, N, D, 1)
    s = float(np.sqrt(D))
    k = (K.SquaredExponential(variance=1.0, lengthscales=s) + K.Matern32(variance=1.0, lengthscales=2 * s)) \
        * K.Linear(variance=1.0)
    mf = gpf.mean_functions.Linear(np.zeros((D, 1)), np.zeros(1))
    m = gpf.models.GPR((d["X"], d["Y"]), k, mean_function=mf, noise_variance=1.0)
    loss0 = -float(m.log_marginal_likelihood())
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options={"maxiter": 20})
    loss1 = -float(m.log_marginal_likelihood())
    assert loss1 < loss0 - 1.0
    np.testing.assert_allclose(loss1, res.fun, rtol=1e-8)
    _, grads = m.training_loss_and_gradients()
    rbf, m32 = k.kernels[0].kernels
    lin = k.kernels[1]
    ko = (O.SquaredExponential(float(rbf.variance.numpy()), float(rbf.lengthscales.numpy()))
          + O.Matern32(float(m32.variance.numpy()), float(m32.lengthscales.numpy()))) * O.Linear(float(lin.variance.numpy()))
    mo = O.LinearMean(mf.A.numpy().copy(), mf.b.numpy().copy())
    _, g = G.gpr_lml_and_grad_expr(d["X"], d["Y"], ko, float(m.likelihood.variance.numpy()), mean_function=mo)
    ref = GC.reference_by_param(g, [m.kernel], mf, [(m.likelihood.variance, g["noise_variance"])])
    want = [-p.unconstrained_gradient(ref[id(p)]) for p in m.trainable_parameters]
    scale = max(float(np.max(np.abs(w))) for w in want)
    for p, gu, w in zip(m.trainable_parameters, grads, want):
        np.testing.assert_allclose(np.asarray(gu).reshape(-1), np.asarray(w).reshape(-1), rtol=1e-5, atol=1e-6 * scale)


def test_materialised_kernels_raise_naming_the_class(cuda_device):
    d = O.make_data(1, 64, 2, 1)
    for kern, cls in [(K.Cosine() + K.White(), "Cosine"), (K.Periodic(K.SquaredExponential()), "Periodic"),
                      (K.ChangePoints([K.SquaredExponential(), K.Matern52()], locations=[0.0]), "ChangePoints")]:
        m = gpf.models.GPR((d["X"], d["Y"]), kern, noise_variance=0.1)
        with pytest.raises(NotImplementedError, match=cls):
            m.log_marginal_likelihood_and_grad()
