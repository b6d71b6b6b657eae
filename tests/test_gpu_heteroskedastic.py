"""HeteroskedasticTFPConditional on the device: the likelihood operators and adjoints against the literal-grid oracle
(tests/hetero_oracle.py) in fp64 and fp32 for every scale transform; equivalence with the Gaussian likelihood at a
constant scale; SVGP value and gradient through the likelihood against tests/svgp_grad_oracle.py for every model
shape with two outputs (SeparateIndependent, SharedIndependent with one Z, a plain kernel with two latents,
LinearCoregionalization with L = 3); consistency with the unfused ELBO and finite differences at B = 4096; the
reference's notebook loop (NaturalGradient alternating with Adam) against the same loop driven on the host by the
oracles; and the refusals."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import ops
from gpflow_b200.base import Exp
from oracle import gp_oracle as O
from tests import adam_oracle as AO
from tests import grad_check as GC
from tests import hetero_oracle as HO
from tests import lik_oracle as LO
from tests import natgrad_oracle as NG
from tests import svgp_grad_oracle as S

pytestmark = pytest.mark.gpu

K = gpf.kernels
IV = gpf.inducing_variables
LIK = gpf.likelihoods
SHAPES = ["separate", "shared", "plain", "coregionalization"]


def _host(t):
    return np.asarray(t.cpu().numpy(), dtype=np.float64)


# ---- 1. the operators ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("transform,lower", HO.TRANSFORMS)
def test_operators_match_the_oracle(cuda_device, dtype, transform, lower):
    lik, o = GC.hetero_pair(transform, lower)
    mu, v, y = HO.rows(7, N=300)
    mu, v, y = (a.astype(dtype).astype(np.float64) for a in (mu, v, y))   # the oracle sees the stored values
    f64 = dtype == np.float64
    with gpf.config.as_context(gpf.config.Config(float=dtype)):   # the storage dtype the operators keep
        Fmu, Fvar, Y = (ops.to_device(a) for a in (mu, v, y))
        ve = float(_host(lik.variational_expectations(None, Fmu, Fvar, Y))[0])
        mean, var = lik.predict_mean_and_var(None, Fmu, Fvar)
        ld = lik.predict_log_density(None, Fmu, Fvar, Y)
    assert Fmu.dtype == ops.torch_dtype(dtype)
    np.testing.assert_allclose(ve, np.sum(o.grid_ve(mu, v, y)), rtol=1e-12)
    assert tuple(mean.shape) == tuple(var.shape) == (300, 1) and mean.dtype == Fmu.dtype
    m_ref, v_ref = o.grid_mean_and_var(mu, v)
    np.testing.assert_allclose(_host(mean), m_ref, rtol=1e-14 if f64 else 1e-7, atol=0)
    np.testing.assert_allclose(_host(var), v_ref, rtol=1e-12 if f64 else 1e-6, atol=0)
    assert tuple(ld.shape) == (300,)
    np.testing.assert_allclose(_host(ld), o.grid_log_density(mu, v, y), rtol=1e-12 if f64 else 1e-6,
                               atol=1e-12 if f64 else 1e-5)


@pytest.mark.parametrize("transform,lower", HO.TRANSFORMS)
def test_adjoints_match_the_oracle(cuda_device, transform, lower):
    lik, o = GC.hetero_pair(transform, lower)
    mu, v, y = HO.rows(8, N=257)
    R, W, dpar = ops.lik_varexp_grad(lik._lik_desc(), ops.to_device(mu), ops.to_device(v), ops.to_device(y), scale=1.7)
    dmu, dv, _ = o.ve_grads(mu, v, y)
    for got, ref in ((R, 1.7 * dmu), (W, 1.7 * dv)):
        got = _host(got)
        for p in range(2):
            np.testing.assert_allclose(got[:, p], ref[:, p], rtol=1e-11, atol=1e-13 * np.max(np.abs(ref[:, p])))
    assert float(_host(dpar)[0]) == 0.0


def test_constant_scale_is_the_gaussian_likelihood(cuda_device):
    """g = log(sigma^2) / 2 with v_g = 0 is Gaussian(sigma^2): the factorised forms are algebraically identical."""
    rng = np.random.default_rng(11)
    N, s2 = 1000, 0.345
    mu_f, v_f = rng.standard_normal((N, 1)), rng.random((N, 1)) ** 2
    y = rng.standard_normal((N, 1))
    mu = np.c_[mu_f, np.full((N, 1), np.log(s2) / 2)]
    v = np.c_[v_f, np.zeros((N, 1))]
    X = np.zeros((N, 1))
    het, gauss = LIK.HeteroskedasticTFPConditional(), LIK.Gaussian(s2)
    a = float(_host(het.variational_expectations(X, mu, v, y))[0])
    b = float(_host(gauss.variational_expectations(X, mu_f, v_f, y))[0])
    np.testing.assert_allclose(a, b, rtol=1e-12)
    for x, r in zip(het.predict_mean_and_var(X, ops.to_device(mu), ops.to_device(v)),
                    gauss.predict_mean_and_var(X, ops.to_device(mu_f), ops.to_device(v_f))):
        np.testing.assert_allclose(_host(x), _host(r), rtol=1e-12)
    Rh, Wh, _ = ops.lik_varexp_grad(het._lik_desc(), ops.to_device(mu), ops.to_device(v), ops.to_device(y))
    Rg, Wg, _ = ops.lik_varexp_grad(gauss._lik_desc(), ops.to_device(mu_f), ops.to_device(v_f), ops.to_device(y))
    np.testing.assert_allclose(_host(Rh)[:, :1], _host(Rg), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(_host(Wh)[:, :1], _host(Wg), rtol=1e-12)
    # the log density is the 20-point quadrature of the Gaussian's closed form
    ld = _host(het.predict_log_density(X, mu, v, y))
    np.testing.assert_allclose(ld, LO.Gaussian(s2).quad_log_density(mu_f, v_f, y), rtol=1e-12, atol=1e-12)


# ---- 3. SVGP value and gradient ------------------------------------------------------------------------------------
def _problem(shape, whiten, q_diag, transform="exp", lower=0.0, mean=None, B=300, M=20, D=3, seed=0):
    """(model, data, oracle arguments) of one model shape with P = 2 outputs."""
    rng = np.random.default_rng(500 + SHAPES.index(shape) + 11 * seed)
    L = 3 if shape == "coregionalization" else 2
    kp, ko = GC.latent_kernel_pairs(D)
    X = rng.standard_normal((B, D))
    Y = np.sin(X[:, :1]) + 0.5 * rng.standard_normal((B, 1)) * np.exp(0.5 * np.cos(X[:, 1:2]))
    Zs = [1.1 * rng.standard_normal((M, D)) for _ in range(L)]
    W = None
    if shape == "separate":
        kern, ok = K.SeparateIndependent(kp[:2]), ko[:2]
        iv, oz = IV.SeparateIndependentInducingVariables([IV.InducingPoints(z.copy()) for z in Zs]), Zs
    elif shape == "shared":
        kern, ok = K.SharedIndependent(kp[1], L), [ko[1]]
        iv, oz = IV.SharedIndependentInducingVariables(IV.InducingPoints(Zs[0].copy())), Zs[:1]
    elif shape == "plain":
        kern, ok = kp[0], [ko[0]]
        iv, oz = Zs[0].copy(), Zs[:1]
    else:
        W = 0.7 * rng.standard_normal((2, L))
        kern, ok = K.LinearCoregionalization(kp, W.copy()), ko
        iv, oz = IV.SeparateIndependentInducingVariables([IV.InducingPoints(z.copy()) for z in Zs]), Zs
    lp, lo = GC.hetero_pair(transform, lower)
    q_mu, q_sqrt = GC.q(M, L, q_diag, rng, upper_noise=False)
    mp = mo = None
    if mean == "constant":
        c = np.array([0.2, -0.4])
        mp, mo = gpf.mean_functions.Constant(c), O.ConstantMean(c)
    elif mean == "linear":
        A, b = 0.2 * rng.standard_normal((D, 2)), np.array([0.1, -0.3])
        mp, mo = gpf.mean_functions.Linear(A, b), O.LinearMean(A, b)
    m = gpf.models.SVGP(kern, lp, iv, num_latent_gps=L, q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy(), whiten=whiten,
                        q_diag=q_diag, num_data=5000, mean_function=mp)
    return m, (X, Y), dict(Zs=oz, kernels=ok, q_mu=q_mu, q_sqrt=q_sqrt, lik=lo, W=W, mean_function=mo)


def _check(m, data, o, rtol=1e-8):
    elbo, grads = m.elbo_and_grad(data)
    ref_elbo, g = S.svgp_elbo_and_grad(data[0], data[1], o["kernels"], o["Zs"], o["q_mu"], o["q_sqrt"], o["lik"],
                                       W=o["W"], whiten=m.whiten, num_data=m.num_data, mean_function=o["mean_function"],
                                       jitter=gpf.config.default_jitter())
    np.testing.assert_allclose(float(elbo), ref_elbo, rtol=1e-9)
    iv, k = m.inducing_variable, m.kernel
    zs = [v.Z for v in iv.inducing_variables] if hasattr(iv, "inducing_variables") else [iv.Z]
    extra = [(m.q_mu, g["q_mu"]), (m.q_sqrt, g["q_sqrt"])] + list(zip(zs, [g["Z"]] if len(zs) == 1 else g["Z"]))
    if o["W"] is not None:
        extra.append((k.W, g["W"]))
    kernels = [k.kernel] if isinstance(k, K.SharedIndependent) else (
        list(k.kernels) if isinstance(k, K.MultioutputKernel) else [k])
    GC.assert_grads_match(grads, GC.reference_by_param(g, kernels, m.mean_function, extra), rtol, "parameter")


@pytest.mark.parametrize("transform,lower", [("exp", 0.0), ("softplus", 1e-3)])
@pytest.mark.parametrize("mean", [None, "constant", "linear"])
@pytest.mark.parametrize("whiten,q_diag", [(True, False), (False, False), (True, True), (False, True)])
@pytest.mark.parametrize("shape", SHAPES)
def test_svgp_gradient_matches_the_oracle(cuda_device, shape, whiten, q_diag, mean, transform, lower):
    m, data, o = _problem(shape, whiten, q_diag, transform, lower, mean)
    _check(m, data, o)


def test_shapes_take_the_expected_entry(cuda_device, monkeypatch):
    """A plain kernel and SharedIndependent with one Z take the single-output entry, the others the multi-output one."""
    for shape, so in [("plain", True), ("shared", True), ("separate", False), ("coregionalization", False)]:
        m, data, _ = _problem(shape, True, False)

        def refuse(*args, **kwargs):
            raise AssertionError(shape)

        monkeypatch.setattr(m, "_mo_elbo_and_grad" if so else "_so_elbo_and_grad", refuse)
        m.elbo_and_grad(data)


# ---- 4. consistency and scale --------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES)
def test_value_agrees_with_unfused_elbo_and_predictions(cuda_device, shape):
    m, data, o = _problem(shape, shape != "shared", shape == "plain", "softplus", 1e-3, "linear")
    e, _ = m.elbo_and_grad(data)
    np.testing.assert_allclose(float(e), float(m.elbo_unfused(data)), rtol=1e-12)
    np.testing.assert_allclose(float(e), float(m.elbo(data)), rtol=1e-12)
    X, Y = data
    fm, fv = m.predict_f(X)
    fm, fv = _host(fm), _host(fv)
    mean, var = m.predict_y(X)
    rm, rv = o["lik"].grid_mean_and_var(fm, fv)
    np.testing.assert_allclose(_host(mean), rm, rtol=1e-13, atol=1e-14)
    np.testing.assert_allclose(_host(var), rv, rtol=1e-11)
    np.testing.assert_allclose(_host(m.predict_log_density((X, Y))), o["lik"].grid_log_density(fm, fv, Y),
                               rtol=1e-12, atol=1e-12)


def test_realistic_size_finite_difference_of_device_elbo(cuda_device):
    """B = 4096, M = 64, L = 2 (SeparateIndependent): the device gradient against central finite differences of the
    device ELBO along random directions of every parameter group."""
    B, M, D = 4096, 64, 4
    rng = np.random.default_rng(31)
    X = rng.standard_normal((B, D))
    Y = np.sin(X[:, :1]) + rng.standard_normal((B, 1)) * np.exp(0.5 * np.cos(X[:, 1:2]))
    ks = [K.SquaredExponential(variance=1.0, lengthscales=np.full(D, 2.0)), K.Matern52(lengthscales=2.5)]
    iv = IV.SeparateIndependentInducingVariables([IV.InducingPoints(1.5 * rng.standard_normal((M, D)))
                                                  for _ in range(2)])
    q_mu, q_sqrt = GC.q(M, 2, False, rng, upper_noise=False)
    m = gpf.models.SVGP(K.SeparateIndependent(ks), LIK.HeteroskedasticTFPConditional(), iv, num_latent_gps=2,
                        q_mu=q_mu, q_sqrt=q_sqrt, num_data=100000, mean_function=gpf.mean_functions.Constant([0.1, -0.2]))
    data = (ops.to_device(X), ops.to_device(Y))
    _, grads = m.elbo_and_grad(data)
    kparams = [p for k in ks for p in k.trainable_parameters]
    groups = {
        "kernel": (kparams, [0.05 * np.ones(p.shape) for p in kparams], 1e-4),
        "Z": ([v.Z for v in iv.inducing_variables], [rng.standard_normal((M, D)) for _ in range(2)], 1e-4),
        "q_mu": ([m.q_mu], [rng.standard_normal((M, 2))], 1e-5),   # the log-scale latent makes the ELBO far from
        "q_sqrt": ([m.q_sqrt], [np.tril(rng.standard_normal((2, M, M)))], 1e-5),  # quadratic in q: short steps
        "mean": ([m.mean_function.c], [np.array([1.0, -0.5])], 1e-5),
    }
    for key, (params, dirs, t) in groups.items():
        dirs = [np.broadcast_to(np.asarray(dv, dtype=np.float64), p.shape) for p, dv in zip(params, dirs)]
        analytic = sum(float(np.sum(np.asarray(grads[p]).reshape(p.shape) * dv)) for p, dv in zip(params, dirs))
        fd = GC.fd_along(m, data, params, dirs, t)
        np.testing.assert_allclose(analytic, fd, rtol=1e-5, err_msg=key)


# ---- 5. the notebook loop ------------------------------------------------------------------------------------------
EPOCHS, LOG_EVERY = 100, 20


def _notebook_data():
    """heteroskedastic.pct.py: N = 1001, loc = sin x, scale = exp(cos x), seed 0; M = 20 inducing points per latent."""
    N, M = 1001, 20
    np.random.seed(0)
    X = np.linspace(0, 4 * np.pi, N)[:, None]
    Y = np.random.normal(np.sin(X), np.exp(np.cos(X)))
    Z = np.linspace(X.min(), X.max(), M)[:, None]
    return X, Y, Z


def _oracle_loop(X, Y, Z):
    """The notebook's loop driven on the host: the rewritten natural-gradient step (tests/natgrad_oracle.py) on (q_mu,
    q_sqrt) alternating with Adam (tests/adam_oracle.py) on the kernels and Z, the gradients from the oracles."""
    M = Z.shape[0]
    val = {"variance0": np.array(1.0), "lengthscales0": np.array(1.0), "variance1": np.array(1.0),
           "lengthscales1": np.array(1.0), "Z0": Z.copy(), "Z1": Z.copy()}
    kinds = {k: (AO.IDENTITY if k.startswith("Z") else AO.SOFTPLUS) for k in val}
    state = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in val.items()}
    q_mu, q_sqrt = np.zeros((M, 2)), np.repeat(np.eye(M)[None], 2, axis=0)
    lik = HO.Hetero()
    jitter = gpf.config.default_jitter()
    hyper = dict(AO.KERAS_DEFAULTS, lr=0.01)

    def grad():
        ks = [O.SquaredExponential(float(val[f"variance{l}"]), float(val[f"lengthscales{l}"])) for l in range(2)]
        return S.svgp_elbo_and_grad(X, Y, ks, [val["Z0"], val["Z1"]], q_mu, q_sqrt, lik, whiten=True, jitter=jitter)

    losses = []
    for t in range(1, EPOCHS + 1):
        _, g = grad()
        q_mu, q_sqrt = NG.rewritten_step("nat", q_mu, q_sqrt, g["q_mu"], g["q_sqrt"], 0.1)
        _, g = grad()
        flat = {"Z0": g["Z"][0], "Z1": g["Z"][1]}
        for l in range(2):
            flat[f"variance{l}"] = g["kernels"][l][0]["variance"]
            flat[f"lengthscales{l}"] = g["kernels"][l][0]["lengthscales"]
        for k in val:
            gk = np.asarray(flat[k], dtype=np.float64).reshape(val[k].shape)
            val[k], *state[k] = AO.constrained_step(val[k], gk, *state[k], t, kinds[k], 0.0, -1.0, **hyper)
        if t % LOG_EVERY == 0:
            losses.append(-grad()[0])
    return val, q_mu, q_sqrt, losses


def test_notebook_loop_matches_the_host_loop(cuda_device):
    X, Y, Z = _notebook_data()
    lik = LIK.HeteroskedasticTFPConditional(distribution_class=LIK.Normal, scale_transform=Exp())
    assert lik.latent_dim == 2
    kern = K.SeparateIndependent([K.SquaredExponential(), K.SquaredExponential()])
    iv = IV.SeparateIndependentInducingVariables([IV.InducingPoints(Z.copy()), IV.InducingPoints(Z.copy())])
    m = gpf.models.SVGP(kernel=kern, likelihood=lik, inducing_variable=iv, num_latent_gps=lik.latent_dim)
    data = (X, Y)
    loss_fn = m.training_loss_closure(data)
    m.q_mu.trainable = False
    m.q_sqrt.trainable = False
    natgrad, adam = gpf.optimizers.NaturalGradient(gamma=0.1), gpf.optimizers.Adam(0.01)
    losses = []
    for epoch in range(1, EPOCHS + 1):
        natgrad.minimize(loss_fn, [(m.q_mu, m.q_sqrt)])
        adam.minimize(loss_fn, m.trainable_variables)
        if epoch % LOG_EVERY == 0:
            losses.append(float(loss_fn()))
    val, q_mu, q_sqrt, ref_losses = _oracle_loop(X, Y, Z)
    print("hetero-notebook losses", losses, ref_losses)
    np.testing.assert_allclose(losses, ref_losses, rtol=1e-8)
    assert losses[-1] < losses[0]
    got = {"Z0": iv.inducing_variables[0].Z, "Z1": iv.inducing_variables[1].Z}
    for l in range(2):
        got[f"variance{l}"] = kern.kernels[l].variance
        got[f"lengthscales{l}"] = kern.kernels[l].lengthscales
    for k, p in got.items():
        np.testing.assert_allclose(np.asarray(p.numpy(), dtype=np.float64).reshape(val[k].shape), val[k], rtol=1e-7,
                                   atol=1e-9, err_msg=k)
    np.testing.assert_allclose(m.q_mu.numpy(), q_mu, rtol=0, atol=1e-7 * np.max(np.abs(q_mu)))
    np.testing.assert_allclose(np.tril(m.q_sqrt.numpy()), np.tril(q_sqrt), rtol=0, atol=1e-7)
    # the trained model's predictions against the oracle's, from the oracle's parameters
    ks = [O.SquaredExponential(float(val[f"variance{l}"]), float(val[f"lengthscales{l}"])) for l in range(2)]
    fm, fv = O.mo_independent_predict_f(X, [val["Z0"], val["Z1"]], ks, q_mu, q_sqrt, whiten=True,
                                        jitter=gpf.config.default_jitter())
    mean, var = m.predict_y(X)
    rm, rv = HO.Hetero().grid_mean_and_var(fm, fv)
    np.testing.assert_allclose(_host(mean), rm, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(_host(var), rv, rtol=1e-6)
    np.testing.assert_allclose(_host(m.predict_log_density(data)), HO.Hetero().grid_log_density(fm, fv, Y),
                               rtol=1e-6, atol=1e-7)


# ---- 6. refusals ---------------------------------------------------------------------------------------------------
def test_refusals(cuda_device):
    m, (X, Y), _ = _problem("separate", True, False)
    with pytest.raises(ValueError, match="Y \\[B, 1\\]"):
        m.elbo_and_grad((X, np.c_[Y, Y]))
    lik = m.likelihood
    F = np.zeros((X.shape[0], 2))
    with pytest.raises(ValueError, match="Y \\[N, 1\\]"):
        lik.variational_expectations(X, F, F, np.c_[Y, Y])
    with pytest.raises(ValueError, match="F \\[N, 2\\]"):
        lik.predict_mean_and_var(X, np.zeros((X.shape[0], 3)), np.zeros((X.shape[0], 3)))
    with pytest.raises(ValueError, match="Y \\[N, 1\\]"):
        lik.predict_log_density(X, F, F, np.c_[Y, Y])
    kp, _ = GC.latent_kernel_pairs(3)
    three = gpf.models.SVGP(K.SeparateIndependent(kp), LIK.HeteroskedasticTFPConditional(),
                            IV.SeparateIndependentInducingVariables([IV.InducingPoints(np.zeros((20, 3)) + i)
                                                                     for i in range(3)]), num_latent_gps=3)
    with pytest.raises(ValueError, match="P = 2"):
        three.elbo_and_grad((X, Y))
    plain3 = gpf.models.SVGP(kp[0], LIK.HeteroskedasticTFPConditional(), np.zeros((20, 3)), num_latent_gps=3)
    with pytest.raises(ValueError, match="P = 2"):
        plain3.elbo_and_grad((X, Y))
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-4)):
        m32, data32, _ = _problem("separate", True, False)
        with pytest.raises(NotImplementedError, match="float64"):
            m32.elbo_and_grad(tuple(np.asarray(d, dtype=np.float32) for d in data32))
    v = gpf.models.VGP((X, Y), K.SquaredExponential(), LIK.HeteroskedasticTFPConditional(), num_latent_gps=2)
    with pytest.raises(NotImplementedError, match="Gaussian likelihood"):
        gpf.optimizers.NaturalGradient(0.1).minimize(v.training_loss, [(v.q_mu, v.q_sqrt)])
    so, data, _ = _problem("plain", True, False)
    for kw in (dict(latent_range=(0, 1)), dict(batch_total=600), dict(include_kl=False)):
        with pytest.raises(NotImplementedError, match="sharding"):
            so.elbo(data, **kw)
