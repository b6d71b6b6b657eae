"""SVGP.elbo_and_grad for multi-output kernels on the device (gpk_svgp_mo_elbo_grad): every kernel / inducing-variable
pair against the oracle (tests/svgp_grad_oracle.py) in both whiten and both q_diag settings, a Gaussian and a
Poisson likelihood, the Constant / Linear mean functions; cross-checks with the single-output entry (SharedIndependent
with a shared Z takes it, L equal SeparateIndependent kernels, MultiClass), W = I against SeparateIndependent, the
value against the unfused elbo(); a finite-difference check at L = 4, P = 8, M = 256, B = 1024; training with Scipy,
Adam over an iterator and NaturalGradient alternating with Adam; and the refusals."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import ops
from gpflow_b200.base import Parameter
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S

pytestmark = pytest.mark.gpu

K = gpf.kernels
IV = gpf.inducing_variables
LIK = gpf.likelihoods
ROWS = ["shared_shared", "shared_separate", "separate_shared", "separate_separate", "coregionalization"]


def _problem(row, whiten, q_diag, lik="gaussian", B=300, M=20, D=3, P=4, seed=0, mean=None):
    """(model, data, oracle arguments) for one row of the kernel / inducing-variable table with L = 3 latents."""
    rng = np.random.default_rng(100 + ROWS.index(row) + 7 * seed)
    L = 3
    kp, ko = GC.latent_kernel_pairs(D)
    X = rng.standard_normal((B, D))
    Zs = [1.1 * rng.standard_normal((M, D)) for _ in range(L)]
    shared_k = row.startswith("shared_")
    shared_z = row in ("shared_shared", "separate_shared")
    W = 0.7 * rng.standard_normal((P, L)) if row == "coregionalization" else None
    Pout = P if W is not None else L
    if shared_k:
        kern, ok = K.SharedIndependent(kp[0], L), [ko[0]]
    elif W is not None:
        kern, ok = K.LinearCoregionalization(kp, W.copy()), ko
    else:
        kern, ok = K.SeparateIndependent(kp), ko
    if shared_z:
        iv, oz = IV.SharedIndependentInducingVariables(IV.InducingPoints(Zs[0].copy())), Zs[:1]
    else:
        iv, oz = IV.SeparateIndependentInducingVariables([IV.InducingPoints(z.copy()) for z in Zs]), Zs
    F = np.sin(X[:, :1] @ np.ones((1, Pout))) + 0.3 * rng.standard_normal((B, Pout))
    if lik == "gaussian":
        Y, lp, lo = F + 0.1 * rng.standard_normal(F.shape), LIK.Gaussian(0.2), LO.Gaussian(0.2)
    else:
        Y, lp, lo = LO.targets("poisson", F, rng), LIK.Poisson(), LO.Poisson()
    q_mu, q_sqrt = GC.q(M, L, q_diag, rng, upper_noise=False)
    mp = mo = None
    if mean == "constant":
        c = 0.1 * np.arange(1, Pout + 1)
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    elif mean == "linear":
        A, b = 0.2 * rng.standard_normal((D, Pout)), 0.1 * np.arange(1, Pout + 1)
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    m = gpf.models.SVGP(kern, lp, iv, num_latent_gps=L, q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), whiten=whiten,
                        q_diag=q_diag, num_data=5000, mean_function=mp)
    return m, (X, Y), dict(Zs=oz, kernels=ok, q_mu=q_mu, q_sqrt=q_sqrt, lik=lo, W=W, mean_function=mo)


def _latent_kernels(m):
    k = m.kernel
    return [k.kernel] if isinstance(k, K.SharedIndependent) else list(k.kernels)


def _check(m, data, o, rtol=1e-8):
    elbo, grads = m.elbo_and_grad(data)
    ref_elbo, g = S.svgp_elbo_and_grad(data[0], data[1], o["kernels"], o["Zs"], o["q_mu"], o["q_sqrt"], o["lik"],
                                       W=o["W"], whiten=m.whiten, num_data=m.num_data, mean_function=o["mean_function"],
                                       jitter=gpf.config.default_jitter())
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-9)
    zs = [v.Z for v in m.inducing_variable.inducing_variables]
    extra = [(m.q_mu, g["q_mu"]), (m.q_sqrt, g["q_sqrt"])] + list(zip(zs, [g["Z"]] if len(zs) == 1 else g["Z"]))
    if isinstance(m.likelihood, LIK.Gaussian):
        extra.append((m.likelihood.variance, g["lik"]))
    if o["W"] is not None:
        extra.append((m.kernel.W, g["W"]))
    ref = GC.reference_by_param(g, _latent_kernels(m), m.mean_function, extra)
    GC.assert_grads_match(grads, ref, rtol, "parameter")


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("row", ROWS)
def test_mo_grad_matches_oracle_gaussian(cuda_device, row, whiten, q_diag):
    m, data, o = _problem(row, whiten, q_diag)
    _check(m, data, o)


@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, True)])
@pytest.mark.parametrize("row", ROWS[1:])
def test_mo_grad_matches_oracle_poisson(cuda_device, row, whiten, q_diag):
    m, data, o = _problem(row, whiten, q_diag, lik="poisson")
    _check(m, data, o)


@pytest.mark.parametrize("mean", ["constant", "linear"])
@pytest.mark.parametrize("row", ["separate_shared", "coregionalization"])
def test_mo_grad_mean_functions(cuda_device, row, mean):
    m, data, o = _problem(row, False, False, mean=mean)
    _check(m, data, o)


def test_shared_independent_with_shared_z_is_the_single_output_call(cuda_device, monkeypatch):
    """One kernel and one Z for every latent: elbo_and_grad makes the single-output call on the inner kernel, so the
    results are the single-output model's up to the run-to-run spread of its atomic reductions."""
    rng = np.random.default_rng(5)
    B, M, D, L = 400, 30, 3, 3
    X, Y = rng.standard_normal((B, D)), rng.standard_normal((B, L))
    Z = rng.standard_normal((M, D))
    q_mu, q_sqrt = GC.q(M, L, False, rng, upper_noise=False)
    k = K.Matern52(variance=1.1, lengthscales=1.4) + K.Linear(variance=0.3)
    so = gpf.models.SVGP(k, LIK.Gaussian(0.3), Z.copy(), num_latent_gps=L, q_mu=q_mu, q_sqrt=q_sqrt, num_data=2000)
    mo = gpf.models.SVGP(K.SharedIndependent(k, L), so.likelihood, IV.SharedIndependentInducingVariables(
        IV.InducingPoints(Z.copy())), num_latent_gps=L, q_mu=q_mu, q_sqrt=q_sqrt, num_data=2000)

    def refuse(*args, **kwargs):
        raise AssertionError("SharedIndependent with a shared Z took the multi-output entry")

    monkeypatch.setattr(mo, "_mo_elbo_and_grad", refuse)
    e_so, g_so = so.elbo_and_grad((X, Y))
    e_mo, g_mo = mo.elbo_and_grad((X, Y))
    np.testing.assert_allclose(float(e_mo), float(e_so), rtol=1e-14)
    pairs = [(so.q_mu, mo.q_mu), (so.q_sqrt, mo.q_sqrt), (so.inducing_variable.Z,
                                                          mo.inducing_variable.inducing_variables[0].Z)]
    pairs += [(p, p) for p in k.trainable_parameters] + [(so.likelihood.variance, mo.likelihood.variance)]
    for a, b in pairs:
        ref = np.asarray(g_so[a])
        np.testing.assert_allclose(np.asarray(g_mo[b]), ref, rtol=0, atol=1e-13 * np.max(np.abs(ref)))


@pytest.mark.parametrize("lik", ["gaussian", "multiclass"])
def test_separate_independent_of_equal_kernels_matches_single_output(cuda_device, lik):
    """L copies of one kernel with a shared Z is the single-output SVGP with P = L latents: the value, and the kernel
    gradients summed over the copies.  MultiClass takes one latent per class."""
    rng = np.random.default_rng(6)
    B, M, D, L = 500, 40, 3, 3
    X = rng.standard_normal((B, D))
    Y = rng.standard_normal((B, L)) if lik == "gaussian" else rng.integers(0, L, (B, 1)).astype(np.float64)
    Z = rng.standard_normal((M, D))
    q_mu, q_sqrt = GC.q(M, L, False, rng, upper_noise=False)

    def kern():
        return K.SquaredExponential(variance=1.2, lengthscales=[0.9, 1.3, 1.7]) + K.White(variance=0.05)

    def lk():
        return LIK.Gaussian(0.3) if lik == "gaussian" else LIK.MultiClass(L)

    k = kern()
    so = gpf.models.SVGP(k, lk(), Z.copy(), num_latent_gps=L, q_mu=q_mu, q_sqrt=q_sqrt, num_data=3000, whiten=False)
    copies = [kern() for _ in range(L)]
    mo = gpf.models.SVGP(K.SeparateIndependent(copies), lk(), IV.SharedIndependentInducingVariables(
        IV.InducingPoints(Z.copy())), num_latent_gps=L, q_mu=q_mu, q_sqrt=q_sqrt, num_data=3000, whiten=False)
    e_so, g_so = so.elbo_and_grad((X, Y))
    e_mo, g_mo = mo.elbo_and_grad((X, Y))
    np.testing.assert_allclose(float(e_mo), float(e_so), rtol=1e-12)
    for i, p in enumerate(k.trainable_parameters):
        tot = sum(np.asarray(g_mo[c.trainable_parameters[i]]) for c in copies)
        np.testing.assert_allclose(tot, np.asarray(g_so[p]), rtol=1e-11, atol=1e-12 * np.max(np.abs(g_so[p])))
    for a, b in [(so.q_mu, mo.q_mu), (so.q_sqrt, mo.q_sqrt),
                 (so.inducing_variable.Z, mo.inducing_variable.inducing_variables[0].Z)]:
        r = np.asarray(g_so[a])
        np.testing.assert_allclose(np.asarray(g_mo[b]), r, rtol=0, atol=1e-11 * np.max(np.abs(r)))


@pytest.mark.parametrize("lik", ["gaussian", "poisson"])
def test_coregionalization_with_identity_mixing_matches_separate_independent(cuda_device, lik):
    m, data, _ = _problem("separate_separate", True, False, lik=lik)
    kp, _ = GC.latent_kernel_pairs(3)
    lc = gpf.models.SVGP(K.LinearCoregionalization(kp, np.eye(3)), m.likelihood, m.inducing_variable,
                         num_latent_gps=3, q_mu=m.q_mu.numpy(), q_sqrt=m.q_sqrt.numpy(), num_data=m.num_data)
    kp2, _ = GC.latent_kernel_pairs(3)
    si = gpf.models.SVGP(K.SeparateIndependent(kp2), m.likelihood, m.inducing_variable, num_latent_gps=3,
                         q_mu=m.q_mu.numpy(), q_sqrt=m.q_sqrt.numpy(), num_data=m.num_data)
    e_lc, g_lc = lc.elbo_and_grad(data)
    e_si, g_si = si.elbo_and_grad(data)
    np.testing.assert_allclose(float(e_lc), float(e_si), rtol=1e-12)
    for a, b in zip(_latent_kernels(lc), _latent_kernels(si)):
        for pa, pb in zip(a.trainable_parameters, b.trainable_parameters):
            np.testing.assert_allclose(np.asarray(g_lc[pa]), np.asarray(g_si[pb]), rtol=1e-10, atol=1e-12)
    pairs = [(lc.q_mu, si.q_mu), (lc.q_sqrt, si.q_sqrt)] + [(v.Z, v.Z) for v in lc.inducing_variable.inducing_variables]
    for a, b in pairs:
        r = np.asarray(g_si[b])
        np.testing.assert_allclose(np.asarray(g_lc[a]), r, rtol=0, atol=1e-11 * np.max(np.abs(r)))
    assert g_lc[lc.kernel.W].shape == (3, 3)


@pytest.mark.parametrize("row", ROWS)
def test_value_agrees_with_unfused_elbo(cuda_device, row):
    m, data, _ = _problem(row, row != "separate_shared", row == "shared_separate", lik="poisson" if row ==
                          "coregionalization" else "gaussian")
    e, _ = m.elbo_and_grad(data)
    np.testing.assert_allclose(float(e), float(m.elbo(data)), rtol=1e-10)


def test_realistic_size_finite_difference_of_device_elbo(cuda_device):
    """L = 4, P = 8, M = 256, B = 1024, D = 8: the analytic device gradient against central finite differences of the
    device ELBO along random directions of every parameter group, W included."""
    B, M, P, L, D = 1024, 256, 8, 4, 8
    rng = np.random.default_rng(21)
    X = rng.standard_normal((B, D))
    Y = np.sin(X[:, :1] @ np.ones((1, P))) + 0.1 * rng.standard_normal((B, P))
    ks = [K.SquaredExponential(variance=1.0, lengthscales=np.full(D, 2.5)), K.Matern32(lengthscales=3.0),
          K.Matern52(lengthscales=2.8), K.SquaredExponential(lengthscales=2.5) + K.Linear(variance=0.1)]
    W = 0.5 * rng.standard_normal((P, L))
    iv = IV.SeparateIndependentInducingVariables([IV.InducingPoints(1.5 * rng.standard_normal((M, D)))
                                                  for _ in range(L)])
    q_mu, q_sqrt = GC.q(M, L, False, rng, upper_noise=False)
    m = gpf.models.SVGP(K.LinearCoregionalization(ks, W), LIK.Gaussian(0.2), iv, num_latent_gps=L, q_mu=q_mu,
                        q_sqrt=q_sqrt, num_data=100000)
    data = (ops.to_device(X), ops.to_device(Y))
    _, grads = m.elbo_and_grad(data)
    kparams = [p for k in ks for p in k.trainable_parameters]
    groups = {
        "kernel": (kparams, [0.05 * np.ones(p.shape) for p in kparams], 1e-4),
        "noise": ([m.likelihood.variance], [0.01], 1e-4),
        "Z": ([v.Z for v in iv.inducing_variables], [rng.standard_normal((M, D)) for _ in range(L)], 1e-4),
        "q_mu": ([m.q_mu], [rng.standard_normal((M, L))], 1e-3),
        "q_sqrt": ([m.q_sqrt], [np.tril(rng.standard_normal((L, M, M)))], 1e-3),
        "W": ([m.kernel.W], [rng.standard_normal((P, L))], 1e-4),
    }
    for key, (params, dirs, t) in groups.items():
        dirs = [np.broadcast_to(np.asarray(dv, dtype=np.float64), p.shape) for p, dv in zip(params, dirs)]
        analytic = sum(float(np.sum(np.asarray(grads[p]).reshape(p.shape) * dv)) for p, dv in zip(params, dirs))
        fd = GC.fd_along(m, data, params, dirs, t)
        np.testing.assert_allclose(analytic, fd, rtol=1e-5, err_msg=key)


def _notebook_model():
    """multioutput.pct.py:111-340: N = 100, D = 1, M = 15, L = 2, P = 3, SquaredExponential + Linear latents."""
    rng = np.random.default_rng(0)
    N, M, L, P = 100, 15, 2, 3
    X = rng.random(N)[:, None] * 10 - 5
    G = np.hstack((0.5 * np.sin(3 * X) + X, 3.0 * np.cos(X) - X))
    Wt = np.array([[0.5, -0.3, 1.5], [-0.4, 0.43, 0.0]])
    Y = G @ Wt + rng.standard_normal((N, P)) * 0.2
    kern = K.LinearCoregionalization([K.SquaredExponential() + K.Linear() for _ in range(L)],
                                     W=rng.standard_normal((P, L)))
    iv = IV.SeparateIndependentInducingVariables([IV.InducingPoints(np.linspace(-5, 5, M)[:, None])
                                                  for _ in range(L)])
    m = gpf.models.SVGP(kern, LIK.Gaussian(), iv, q_mu=np.zeros((M, L)),
                        q_sqrt=np.repeat(np.eye(M)[None], L, axis=0))
    return m, (X, Y)


def test_scipy_fits_the_coregionalization_notebook(cuda_device):
    m, data = _notebook_model()
    assert m.kernel.W in set(m.trainable_parameters)
    e0 = float(m.elbo(data))
    _, g0 = m.training_loss_and_gradients(data)
    res = gpf.optimizers.Scipy().minimize(m.training_loss_closure(data), m.trainable_variables,
                                          options={"maxiter": 20000})
    assert res.success, res.message
    e1 = float(m.elbo(data))
    assert e1 > e0 + 100.0, (e0, e1)
    _, g1 = m.training_loss_and_gradients(data)
    n0 = np.sqrt(sum(float(np.sum(np.square(g))) for g in g0))
    n1 = np.sqrt(sum(float(np.sum(np.square(g))) for g in g1))
    assert n1 < 1e-2 * n0, (n0, n1)


def test_adam_minibatch_loop_keeps_the_arrays_on_the_device(cuda_device):
    m, (X, Y) = _notebook_model()
    m.num_data = X.shape[0]
    Xd, Yd = ops.to_device(X), ops.to_device(Y)
    batches = [(Xd[i:i + 25], Yd[i:i + 25]) for i in range(0, 100, 25)] * 10
    arrays = [v.Z for v in m.inducing_variable.inducing_variables] + [m.q_mu, m.q_sqrt, m.kernel.W]
    _, g = m.elbo_and_grad(batches[0], device_arrays=True)
    for p in arrays:
        assert hasattr(g[p], "data_ptr") and g[p].is_cuda and tuple(g[p].shape) == tuple(p.shape)
    e0 = float(m.elbo((Xd, Yd)))
    before = [np.array(p.numpy()) for p in arrays]
    closure = m.training_loss_closure(iter(batches))
    opt = gpf.optimizers.Adam(0.02)
    for _ in range(len(batches)):
        opt.minimize(closure, m.trainable_variables)
    assert float(m.elbo((Xd, Yd))) > e0
    for p, b in zip(arrays, before):
        assert not np.array_equal(np.array(p.numpy()), b)


def test_natural_gradient_alternates_with_adam(cuda_device):
    m, data = _notebook_model()
    m.q_mu.trainable = False
    m.q_sqrt.trainable = False
    closure = m.training_loss_closure(data)
    ng, adam = gpf.optimizers.NaturalGradient(gamma=0.1), gpf.optimizers.Adam(0.01)
    e0 = float(m.elbo(data))
    for _ in range(20):
        ng.minimize(closure, [(m.q_mu, m.q_sqrt)])
        adam.minimize(closure, m.trainable_variables)
    assert float(m.elbo(data)) > e0 + 50.0


def test_refusals(cuda_device):
    m, data, _ = _problem("coregionalization", True, False)
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m32, data32, _ = _problem("separate_separate", True, False)
        with pytest.raises(NotImplementedError, match="float64"):
            m32.elbo_and_grad(tuple(np.asarray(d, dtype=np.float32) for d in data32))
    kp, _ = GC.latent_kernel_pairs(3)
    bad = gpf.models.SVGP(K.SeparateIndependent([kp[0], K.Cosine(), kp[2]]), LIK.Gaussian(0.2), m.inducing_variable,
                          num_latent_gps=3)
    with pytest.raises(NotImplementedError, match="Cosine"):
        bad.elbo_and_grad((data[0], data[1][:, :3]))
    with pytest.raises(ValueError, match="columns"):
        m.elbo_and_grad((data[0], data[1][:, :3]))
    wrong = gpf.models.SVGP(K.LinearCoregionalization(kp, np.ones((4, 3))), LIK.Gaussian(0.2), m.inducing_variable,
                            num_latent_gps=3)
    wrong.kernel.W = Parameter(np.ones((4, 2)))
    with pytest.raises(ValueError):
        wrong.elbo_and_grad(data)
    two = IV.SeparateIndependentInducingVariables([IV.InducingPoints(np.zeros((20, 3))) for _ in range(2)])
    mism = gpf.models.SVGP(K.SeparateIndependent(kp), LIK.Gaussian(0.2), two, num_latent_gps=3)
    with pytest.raises(ValueError):
        mism.elbo_and_grad((data[0], data[1][:, :3]))
