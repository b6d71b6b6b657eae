"""MultiClass (RobustMax) on the device: the operators of csrc/lik.cu against the oracle (tests/multiclass_oracle.py
and tests/svgp_grad_oracle.py, pinned by finite differences in tests/test_oracle_multiclass.py), SVGP.elbo / predict_y /
predict_log_density, the value and gradient of gpk_svgp_elbo_grad over fused expressions, finite differences of the device ELBO at a large shape,
L-BFGS-B training of a 3-class classifier against the same run driven by the oracle, a minibatch loop and the
refusals."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import multiclass_oracle as MO
from tests import svgp_grad_oracle as S

pytestmark = pytest.mark.gpu

K = gpf.kernels
LIK = gpf.likelihoods


def _rows(C, N=67, seed=0):
    rng = np.random.default_rng(seed + C)
    mu = rng.uniform(-1.5, 1.5, (N, C))
    var = rng.uniform(0.05, 1.2, (N, C))
    var[0, :2] = 3e-11                   # inside the clamps of s_c and s_y
    var[1, :] = 0.0
    Y = np.argmax(mu + 0.5 * rng.standard_normal(mu.shape), 1)[:, None].astype(np.float64)
    Y[0, 0] = 1.0
    Y[2, 0] = C + 3.0                    # outside [0, C)
    Y[3, 0] = -1.0
    Y[4, 0] += 0.6                       # truncated
    return mu, var, Y


@pytest.mark.parametrize("C", [2, 3, 10, 100])
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_operators_match_the_oracle(cuda_device, C, dtype):
    T = ops.torch()
    td = getattr(T, dtype)
    mu, var, Y = _rows(C)
    mu, var = (a.astype(dtype).astype(np.float64) for a in (mu, var))
    dev = [T.tensor(a, dtype=td, device=cuda_device) for a in (mu, var, Y)]
    eps = 0.013
    desc = _lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0.0, 0.0, 0.0, 0.0, eps, C)
    lo = MO.MultiClass(C, eps)
    rtol = 1e-12 if dtype == "float64" else 1e-5
    ve = float(ops.lik_varexp_sum(desc, *dev)[0])
    # the variational expectations sum in fp64 from the stored inputs whatever the storage type
    np.testing.assert_allclose(ve, np.sum(lo.variational_expectations(mu, var, Y)), rtol=1e-12)
    ld = ops.lik_predict_log_density(desc, *dev).cpu().numpy().astype(np.float64)
    np.testing.assert_allclose(ld, lo.predict_log_density(mu, var, Y), rtol=rtol, atol=0)
    m, v = (a.cpu().numpy().astype(np.float64) for a in ops.lik_predict_mean_and_var(desc, dev[0], dev[1]))
    mo, vo = lo.predict_mean_and_var(mu, var)
    assert m.shape == (mu.shape[0], C)
    np.testing.assert_allclose(m, mo, rtol=rtol, atol=0)
    np.testing.assert_allclose(v, vo, rtol=rtol, atol=1e-15)


def test_operators_refuse_a_bad_descriptor(cuda_device):
    mu, var, Y = (ops.to_device(a) for a in _rows(3, N=5))
    with pytest.raises(ValueError, match="one latent per class"):
        ops.lik_varexp_sum(_lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0, 0, 0, 0, 1e-3, 4), mu, var, Y)
    with pytest.raises(ValueError, match="epsilon"):
        ops.lik_predict_log_density(_lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0, 0, 0, 0, 1.5, 3), mu, var, Y)


# ---- SVGP ------------------------------------------------------------------------------------------------------
def _labelled(C, B, D, seed=5):
    d = O.make_data(seed, B, D, 1)
    rng = np.random.default_rng(seed + C)
    Y = MO.labels(rng, np.sin(d["X"][:, :1] + 0.7 * np.arange(C)[None]))
    Y[0, 0] = float(C)                   # one label outside the classes
    return d["X"], Y


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_svgp_value_and_predictions_match_the_oracle(cuda_device, dtype):
    C, B, D, M = 4, 300, 3, 20
    X, Y = _labelled(C, B, D)
    Z = GC.z(M, D)
    q_mu, q_sqrt = GC.q(M, C, False)
    ko = O.SquaredExponential(1.3, 1.7) + O.White(0.05)
    lo = MO.MultiClass(C, 0.02)
    tol, atol = (1e-10, 1e-13) if dtype == np.float64 else (2e-4, 1e-5)
    with gpf.config.as_context(gpf.config.Config(float=dtype, jitter=1e-6)):
        kp = K.SquaredExponential(variance=1.3, lengthscales=1.7) + K.White(variance=0.05)
        m = gpf.models.SVGP(kp, LIK.MultiClass(C, invlink=LIK.RobustMax(C, 0.02)), Z.copy(), num_latent_gps=C,
                            q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), num_data=5000)
        elbo = float(m.elbo((X, Y)))
        ref = S.svgp_elbo(X, Y, [ko], [Z], q_mu, q_sqrt, lo, num_data=5000, jitter=1e-6)
        np.testing.assert_allclose(elbo, ref, rtol=tol)
        fm, fv = O.svgp_predict_f(X, Z, ko, q_mu, q_sqrt, whiten=True, jitter=1e-6)
        pm, pv = (a.cpu().numpy() for a in m.predict_y(X))
        om, ov = lo.predict_mean_and_var(fm, fv)
        np.testing.assert_allclose(pm, om, rtol=tol, atol=atol)
        np.testing.assert_allclose(pv, ov, rtol=tol, atol=atol)
        np.testing.assert_allclose(pm.sum(1), 1.0, rtol=1e-2)   # close to a distribution over the classes
        ld = m.predict_log_density((X, Y)).cpu().numpy()
        np.testing.assert_allclose(ld, lo.predict_log_density(fm, fv, Y), rtol=tol)
        if dtype == np.float64:
            value, _ = m.elbo_and_grad((X, Y))
            np.testing.assert_allclose(float(value), elbo, rtol=1e-12)


def _check(m, X, Y, ko, Z, q_mu, q_sqrt, lo, mo=None, rtol=1e-6):
    elbo, grads = m.elbo_and_grad((X, Y))
    ref_elbo, g = S.svgp_elbo_and_grad(X, Y, [ko], [Z], q_mu, q_sqrt, lo, whiten=m.whiten, num_data=m.num_data,
                                       mean_function=mo, jitter=gpf.config.default_jitter())
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-8)
    np.testing.assert_allclose(float(elbo), float(m.elbo((X, Y))), rtol=1e-12)
    ref = GC.reference_by_param(g, [m.kernel], m.mean_function, [
        (m.inducing_variable.Z, g["Z"]), (m.q_mu, g["q_mu"]), (m.q_sqrt, g["q_sqrt"]),
        (m.likelihood.invlink.epsilon, g["lik"])])
    GC.assert_grads_match(grads, ref, rtol, "parameter")


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("name,B,M,D,C,num_data", [
    ("rbf_plus_white", 400, 17, 3, 3, None), ("c5", 300, 64, 8, 5, 20000), ("rq_ard", 300, 200, 4, 3, 5000),
    ("constant_times_matern52", 250, 64, 5, 5, None)])
def test_svgp_multiclass_grad_matches_oracle(cuda_device, name, B, M, D, C, num_data, whiten, q_diag):
    X, Y = _labelled(C, B, D)
    Z = GC.z(M, D)
    q_mu, q_sqrt = GC.q(M, C, q_diag)
    kp, ko = GC.case(name, D)
    m = gpf.models.SVGP(kp, LIK.MultiClass(C, invlink=LIK.RobustMax(C, 0.03)), Z.copy(), num_latent_gps=C,
                        q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), whiten=whiten, q_diag=q_diag, num_data=num_data)
    _check(m, X, Y, ko, Z, q_mu, q_sqrt, MO.MultiClass(C, 0.03))


@pytest.mark.parametrize("mean", ["constant", "linear"])
def test_mean_function_and_epsilon_grads_match_oracle(cuda_device, mean):
    C, B, D, M = 3, 400, 4, 30
    X, Y = _labelled(C, B, D, seed=3)
    rng = np.random.default_rng(11)
    if mean == "constant":
        c = np.array([0.3])
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    else:
        A, b = 0.2 * rng.standard_normal((D, C)), 0.1 * np.arange(1, C + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    kp, ko = GC.case("c5", D)
    Z = GC.z(M, D)
    q_mu, q_sqrt = GC.q(M, C, False)
    m = gpf.models.SVGP(kp, LIK.MultiClass(C, invlink=LIK.RobustMax(C, 0.2)), Z.copy(), num_latent_gps=C,
                        q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), num_data=6000, mean_function=mp)
    _check(m, X, Y, ko, Z, q_mu, q_sqrt, MO.MultiClass(C, 0.2), mo)


def test_large_shape_finite_difference_of_device_elbo(cuda_device):
    """B = 4096, M = 1024, D = 16, C = 10 in float64 (RBF + White, whitened, dense q_sqrt, num_data = 1e6): the
    analytic device gradient against central finite differences of the device ELBO (the unfused route) along random
    directions of the kernel parameters, Z, q_mu and q_sqrt."""
    B, M, C, D = 4096, 1024, 10, 16
    d = O.make_data(4, B, D, 1, M=M)
    q_mu, q_sqrt = O.make_q(4, M, C)
    rng = np.random.default_rng(12)
    Y = MO.labels(rng, np.sin(d["X"][:, :C]))
    data = (ops.to_device(d["X"]), ops.to_device(Y))
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
        kp = K.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) + K.White(variance=0.01)
        m = gpf.models.SVGP(kp, LIK.MultiClass(C), d["Z"], num_latent_gps=C, q_mu=q_mu, q_sqrt=q_sqrt, whiten=True,
                            num_data=1000000)
        elbo, grads = m.elbo_and_grad(data)
        np.testing.assert_allclose(float(elbo), float(m.elbo(data)), rtol=1e-12)
        rbf, white = kp.kernels
        groups = {
            "kernel": ([rbf.variance, rbf.lengthscales, white.variance], [0.3, 1.0, 0.002], 1e-4),
            "Z": ([m.inducing_variable.Z], [rng.standard_normal((M, D))], 1e-4),
            "q_mu": ([m.q_mu], [rng.standard_normal((M, C))], 1e-3),
            "q_sqrt": ([m.q_sqrt], [np.tril(rng.standard_normal((C, M, M)))], 2.5e-4),
        }
        for key, (params, dirs, t) in groups.items():
            dirs = [np.broadcast_to(np.asarray(dv, dtype=np.float64), p.shape) for p, dv in zip(params, dirs)]
            analytic = sum(float(np.sum(np.asarray(grads[p]).reshape(p.shape) * dv)) for p, dv in zip(params, dirs))
            fd = GC.fd_along(m, data, params, dirs, t)
            np.testing.assert_allclose(analytic, fd, rtol=1e-5, err_msg=key)


def _classifier(Z, C):
    return gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=1.0), LIK.MultiClass(C), Z.copy(),
                           num_latent_gps=C, whiten=True)


def test_scipy_trains_a_three_class_classifier(cuda_device):
    """L-BFGS-B with the kernel, Z and q trainable (epsilon keeps its default, untrainable) on 2-D data in three angular
    sectors with noisy labels, against the same run whose value and gradient come from the oracle.

    Neither run converges: the RobustMax bound is nearly flat along some directions (with whiten, fmean scales with the
    square root of the kernel variance and fvar with it, and the class probabilities depend only on their ratios), and
    L-BFGS-B creeps along them past 3000 iterations whichever gradient drives it.  Both runs stop at the same iteration
    budget instead.  Their paths separate (a 1e-12 relative perturbation of the gradient moves the objective after 100
    steps by 3e-3), but both end in the same flat basin, a few 1e-4 apart."""
    rng = np.random.default_rng(21)
    N, M, C = 240, 12, 3
    X = rng.standard_normal((N, 2))
    ang = np.arctan2(X[:, 1], X[:, 0])
    clean = np.floor((ang + np.pi) / (2 * np.pi / C)).astype(int) % C
    noisy = np.floor((ang + 0.25 * rng.standard_normal(N) + np.pi) / (2 * np.pi / C)).astype(int) % C
    Y = noisy[:, None].astype(np.float64)
    Z = X[:M].copy()
    data = (X, Y)
    m = _classifier(Z, C)
    loss0 = -float(m.elbo(data))
    opts = {"maxiter": 1000}
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(data), m.trainable_variables, options=opts)
    loss1 = -float(m.elbo(data))
    assert res.nit == 1000, res.message
    assert loss1 < loss0 - 10.0
    np.testing.assert_allclose(loss1, res.fun, rtol=1e-10)
    pm, _ = m.predict_y(X)
    acc = float(np.mean(np.argmax(pm.cpu().numpy(), 1) == clean))
    assert acc > 0.9, acc

    o = _classifier(Z, C)
    lo = MO.MultiClass(C)

    def oracle_objective_and_grad(batch):
        rbf = o.kernel
        ko = O.SquaredExponential(float(rbf.variance.numpy()), float(rbf.lengthscales.numpy()))
        Zv, qm, qs = (np.asarray(p.numpy(), dtype=np.float64) for p in (o.inducing_variable.Z, o.q_mu, o.q_sqrt))
        elbo, g = S.svgp_elbo_and_grad(X, Y, [ko], [Zv], qm, qs, lo, whiten=True, jitter=gpf.config.default_jitter())
        grads = {o.inducing_variable.Z: g["Z"], o.q_mu: g["q_mu"], o.q_sqrt: g["q_sqrt"],
                 rbf.variance: np.asarray(g["leaves"][0]["variance"]),
                 rbf.lengthscales: np.asarray(g["leaves"][0]["lengthscales"])}
        return elbo, grads

    o._objective_and_grad = oracle_objective_and_grad
    res_o = gpf.optimizers.Scipy().minimize(o.training_loss_closure(data), o.trainable_variables, options=opts)
    assert res_o.nit == 1000, res_o.message
    np.testing.assert_allclose(res.fun, res_o.fun, rtol=2e-3)


def test_minibatch_loop_over_an_iterator(cuda_device):
    """value_and_gradients draws ONE batch per call and returns the loss and gradients of that batch."""
    N, D, M, C, Bs = 1200, 3, 20, 4, 200
    X, Y = _labelled(C, N, D, seed=7)
    m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=2.0), LIK.MultiClass(C), X[:M].copy(),
                        num_latent_gps=C, num_data=N)
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


def test_refusals(cuda_device):
    C = 3
    X, Y = _labelled(C, 200, 2)
    Z = X[:10].copy()
    data = (X, Y)
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m = gpf.models.SVGP(K.SquaredExponential(), LIK.MultiClass(C), Z.copy(), num_latent_gps=C)
        with pytest.raises(NotImplementedError, match="float64"):
            m.training_loss_and_gradients(data)
    m = gpf.models.SVGP(K.SharedIndependent(K.SquaredExponential(), C), LIK.MultiClass(C), Z.copy(), num_latent_gps=C)
    with pytest.raises(NotImplementedError, match="single-output"):
        m.elbo_and_grad(data)
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.MultiClass(C), Z.copy(), num_latent_gps=C)
    with pytest.raises(ValueError, match=r"\[B, 1\]"):
        m.elbo_and_grad((X, np.tile(Y, (1, C))))
    with pytest.raises(NotImplementedError, match="sharding"):
        m.elbo(data, latent_range=(0, 1))
    with pytest.raises(NotImplementedError, match="sharding"):
        m.elbo(data, batch_total=400)
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.MultiClass(C), Z.copy(), num_latent_gps=C + 1)
    with pytest.raises(ValueError, match="one latent GP per class"):
        m.elbo_and_grad(data)
    m = gpf.models.VGP(data, K.SquaredExponential(), LIK.MultiClass(C), num_latent_gps=C)
    with pytest.raises(NotImplementedError):
        m.elbo_and_grad()
    m = gpf.models.SVGP(K.SquaredExponential(), LIK.MultiClass(C), Z.copy(), num_latent_gps=C)
    m.likelihood.invlink.epsilon.trainable = True
    with pytest.raises(NotImplementedError, match="prior"):
        m.training_loss_and_gradients(data)
