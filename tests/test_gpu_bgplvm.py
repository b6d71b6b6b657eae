"""Bayesian GPLVM on the device: the RBF psi statistics (gpk_rbf_psi) element by element against the oracle within a
bound derived from their operation counts, the fused bound and its gradient against tests/bgplvm_oracle.py and
tests/bgplvm_grad_oracle.py, finite differences of the device bound, a cross-check against SGPR, prediction, the
reference's three BayesianGPLVM tests (tests/gpflow/models/test_gplvm.py), device Adam, and the refusals."""

import zlib

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests import adam_oracle as AO
from tests.bgplvm_grad_oracle import bgplvm_elbo_grad
from tests.bgplvm_oracle import _cols, _lengthscales, bgplvm_elbo, bgplvm_predict_f, psi_statistics

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps


def _data(N, Q, M, P, seed=0, svar=(0.05, 0.5)):
    rng = np.random.default_rng(seed)
    return dict(Y=rng.standard_normal((N, P)), mu=rng.standard_normal((N, Q)), S=rng.uniform(*svar, (N, Q)),
                Z=rng.standard_normal((M, Q)))


def _kernels(ls, variance=1.3, active_dims=None):
    return (gpf.kernels.SquaredExponential(variance=variance, lengthscales=ls, active_dims=active_dims),
            O.SquaredExponential(variance, ls, active_dims=active_dims))


def _model(d, kp, **kw):
    m = gpf.models.BayesianGPLVM(d["Y"], d["mu"], d["S"], kp, inducing_variable=d["Z"], **kw)
    m.likelihood.variance.assign(0.3)
    return m


# ---- psi statistics ----------------------------------------------------------------------------------------------
def psi_bounds(mu, S, Z, ko):
    """Per-element error bounds of the device psi1 and psi2.  Each exponent u is a sum of 3 nd + 2 rounded operations
    on non-negative terms (plus the log1p shifts), so |du| <= (3 nd + 4) eps u + 2 eps; exp(-u) adds at most 2 eps
    (the K-build exp is pinned to the ulp by test_gpu_kbuild_accuracy.py) and the variance product 2 eps.  psi2 sums N
    non-negative terms, in chunks and then across chunks: at most N eps more, relative to the sum."""
    cols = _cols(ko, mu.shape[1])
    nd = len(cols)
    l2 = _lengthscales(ko, nd) ** 2
    ma, Sa, Za = mu[:, cols], S[:, cols], Z[:, cols]
    var = float(ko.variance)
    c = (3 * nd + 4) * EPS
    u1 = (0.5 * np.sum(np.log1p(Sa / l2), 1)[:, None]
          + 0.5 * np.sum((ma[:, None] - Za[None]) ** 2 / (l2 + Sa)[:, None], -1))
    b1 = var * np.exp(-u1) * (c * u1 + 6 * EPS)
    zbar = 0.5 * (Za[:, None] + Za[None])
    ez = np.sum((Za[:, None] - Za[None]) ** 2 / (4 * l2), -1)
    b2 = np.zeros((Z.shape[0],) * 2)
    tot = np.zeros_like(b2)
    for n in range(mu.shape[0]):
        u2 = ez + 0.5 * np.sum(np.log1p(2 * Sa[n] / l2)) + np.sum((ma[n] - zbar) ** 2 / (l2 + 2 * Sa[n]), -1)
        t = var * var * np.exp(-u2)
        b2 += t * (c * u2 + 6 * EPS)
        tot += t
    return b1, b2 + mu.shape[0] * EPS * tot


def device_psi(mu, S, Z, kp):
    lib = _lib.load()
    T = ops.torch()
    N, Q = mu.shape
    M = Z.shape[0]
    mu_d, S_d, Z_d = ops.to_device(mu), ops.to_device(S), ops.to_device(Z)
    p0 = T.empty((1,), dtype=T.float64, device=mu_d.device)
    p1 = T.empty((N, M), dtype=T.float64, device=mu_d.device)
    p2 = T.empty((M, M), dtype=T.float64, device=mu_d.device)
    # the workspace exactly as sized, followed by a guard region that must come back untouched
    need, guard = lib.gpk_rbf_psi_ws(N, M), 1 << 20
    ws = ops.scratch_bytes(need + guard)
    ws[need:].fill_(0xA5)
    _lib.check(lib.gpk_rbf_psi(*gpf.kernels.compile_kernel(kp, Q), ops._p(mu_d), ops._p(S_d), N, Q, ops._p(Z_d), M,
                               Q, ops._p(p0), ops._p(p1), ops._p(p2), ops._p(ws), ops._stream()), "gpk_rbf_psi")
    assert bool((ws[need:] == 0xA5).all()), "gpk_rbf_psi wrote past gpk_rbf_psi_ws bytes"
    return float(p0.cpu()[0]), p1.cpu().numpy(), p2.cpu().numpy()


PSI_CASES = {
    "scalar": (37, 3, 11, 0.9, None),
    "ard": (37, 3, 11, [0.7, 1.2, 2.0], None),
    "active_dims": (37, 4, 11, [0.8, 1.5], [3, 1]),
    "off_tile_edges": (1031, 5, 67, 1.1, None),
    "m_one": (50, 2, 1, 1.0, None),
    "q_one": (80, 1, 9, 0.6, None),
    "q_32": (40, 32, 13, list(np.linspace(2.0, 6.0, 32)), None),
    "q_12_ard": (300, 12, 40, list(np.linspace(0.8, 3.0, 12)), None),
    "n_split": (6000, 3, 4, 1.0, None),
    # few active dims and many pairs: four pairs per thread and many point chunks, the largest psi2 chunk buffer
    "many_chunks_q2": (1000, 2, 256, 0.9, None),
    "many_chunks_q1": (700, 1, 160, 0.8, None),
}
RATIOS = {}


@pytest.mark.parametrize("name", list(PSI_CASES))
def test_rbf_psi_within_derived_bound(cuda_device, name):
    N, Q, M, ls, ad = PSI_CASES[name]
    d = _data(N, Q, M, 1, seed=zlib.crc32(name.encode()) % 1000)
    kp, ko = _kernels(np.asarray(ls) if isinstance(ls, list) else ls, active_dims=ad)
    p0, p1, p2 = device_psi(d["mu"], d["S"], d["Z"], kp)
    r0, r1, r2 = psi_statistics(d["mu"], d["S"], d["Z"], ko)
    b1, b2 = psi_bounds(d["mu"], d["S"], d["Z"], ko)
    # the oracle's own rounding (Cholesky forms, per-point sums) is of the same order: the bound is taken twice
    ratio1 = np.max(np.abs(p1 - r1) / (2 * b1 + 1e-300))
    ratio2 = np.max(np.abs(p2 - r2) / (2 * b2 + 1e-300))
    RATIOS[name] = (ratio1, ratio2)
    print(f"{name}: max error / bound psi1 {ratio1:.3f} psi2 {ratio2:.3f}")
    assert p0 == pytest.approx(r0, rel=1e-15)
    assert ratio1 <= 1.0 and ratio2 <= 1.0
    np.testing.assert_array_equal(p2, p2.T)


def test_rbf_psi_refuses_other_kernels(cuda_device):
    d = _data(10, 2, 3, 1)
    with pytest.raises(ValueError, match="SquaredExponential"):
        device_psi(d["mu"], d["S"], d["Z"], gpf.kernels.Matern32())


# ---- bound and gradient ------------------------------------------------------------------------------------------
GRAD_CASES = {
    "scalar": (40, 3, 9, 2, 0.9, None),
    "ard": (40, 3, 9, 3, [0.7, 1.2, 2.0], None),
    "active_dims": (40, 4, 9, 2, [0.8, 1.5], [3, 1]),
    "wide_q": (60, 20, 17, 2, list(np.linspace(1.5, 4.0, 20)), None),
    "many_chunks": (700, 1, 160, 2, 0.15, None),
    # the 9-16 kernel bucket, and both halves of the ND = 32 split with 1 and 16 live dims in the second
    "ard_q9": (50, 9, 11, 2, list(np.linspace(1.2, 3.0, 9)), None),
    "ard_q16": (45, 16, 12, 2, list(np.linspace(1.5, 4.0, 16)), None),
    "ard_q17": (45, 17, 12, 2, list(np.linspace(1.5, 4.0, 17)), None),
    "ard_q32": (60, 32, 13, 2, list(np.linspace(2.0, 6.0, 32)), None),
}


def _spread(d, half_width, seed):
    """Z on a regular grid of spacing about 0.5 over [-half_width, half_width]^Q and the latent means uniform over the
    same box: with lengthscales well under the spacing, Kuu stays well conditioned at large M."""
    M, Q = d["Z"].shape
    side = int(np.ceil(M ** (1.0 / Q)))
    axes = np.meshgrid(*([np.linspace(-half_width, half_width, side)] * Q), indexing="ij")
    d["Z"] = np.stack([a.reshape(-1) for a in axes], 1)[:M].copy()
    d["mu"] = np.random.default_rng(seed).uniform(-half_width, half_width, d["mu"].shape)
    return d


def _prior(N, Q, seed=5):
    rng = np.random.default_rng(seed)
    return 0.1 * rng.standard_normal((N, Q)), rng.uniform(0.5, 2.0, (N, Q))


@pytest.mark.parametrize("name", list(GRAD_CASES))
def test_elbo_and_gradient_against_oracle(cuda_device, name):
    N, Q, M, P, ls, ad = GRAD_CASES[name]
    d = _data(N, Q, M, P, seed=3)
    if name == "many_chunks":
        d = _spread(d, 40.0, 4)
    m0, p0 = _prior(N, Q)
    kp, ko = _kernels(np.asarray(ls) if isinstance(ls, list) else ls, active_dims=ad)
    m = _model(d, kp, X_prior_mean=m0, X_prior_var=p0)
    ref = bgplvm_elbo(d["Y"], d["mu"], d["S"], d["Z"], ko, 0.3, m0, p0)
    val = float(m.elbo())
    assert val == pytest.approx(ref, rel=1e-10)
    v2, g = m.elbo_and_grad()
    assert float(v2) == pytest.approx(val, rel=1e-12)
    go = bgplvm_elbo_grad(d["Y"], d["mu"], d["S"], d["Z"], ko, 0.3, m0, p0)
    pairs = [(m.likelihood.variance, go["noise"]), (kp.variance, go["variance"]), (kp.lengthscales, go["lengthscales"]),
             (m.X_data_mean, go["mu"]), (m.X_data_var, go["S"]), (m.inducing_variable.Z, go["Z"])]
    for p, ref_g in pairs:
        ref_g = np.asarray(ref_g)
        got = np.asarray(g[p]).reshape(ref_g.shape)
        np.testing.assert_allclose(got, ref_g, rtol=1e-8, atol=1e-8 * max(1.0, np.max(np.abs(ref_g))))


def test_elbo_at_many_point_chunks(cuda_device):
    """N = 1000, M = 256, Q = 2: the psi2 chunk buffer is at its largest relative to the rest of the workspace."""
    N, Q, M, P = 1000, 2, 256, 3
    d = _spread(_data(N, Q, M, P, seed=17), 4.0, 18)
    kp, ko = _kernels(np.array([0.18, 0.22]))
    m = _model(d, kp)
    ref = bgplvm_elbo(d["Y"], d["mu"], d["S"], d["Z"], ko, 0.3)
    assert float(m.elbo()) == pytest.approx(ref, rel=1e-10)
    v, g = m.elbo_and_grad()
    assert float(v) == pytest.approx(ref, rel=1e-10)
    assert all(np.all(np.isfinite(np.asarray(x))) for x in g.values())


FD_LENGTHSCALES = {4: np.array([0.9, 1.4, 2.0, 1.1]), 12: np.linspace(1.2, 3.0, 12), 24: np.linspace(2.0, 5.0, 24)}


def test_device_elbo_finite_differences(cuda_device):
    _check_device_finite_differences(4)


@pytest.mark.parametrize("Q", [12, 24])
def test_device_elbo_finite_differences_wide_latent(cuda_device, Q):
    """As test_device_elbo_finite_differences, in the 9-16 kernel bucket and across the ND = 32 split."""
    _check_device_finite_differences(Q)


def _check_device_finite_differences(Q):
    """Central differences of the device bound against elbo_and_grad at three entries of every parameter."""
    N, M, P = 300, 24, 3
    d = _data(N, Q, M, P, seed=11)
    kp, _ = _kernels(FD_LENGTHSCALES[Q])
    m = _model(d, kp)
    _, g = m.elbo_and_grad()
    h = 1e-5
    for p in (m.X_data_mean, m.X_data_var, m.inducing_variable.Z, kp.lengthscales, kp.variance,
              m.likelihood.variance):
        base = p.numpy().copy()
        flat = np.asarray(g[p]).reshape(-1)
        for idx in np.random.default_rng(0).choice(base.size, size=min(3, base.size), replace=False):
            step = h * max(1.0, abs(base.reshape(-1)[idx]))
            vals = []
            for sgn in (1, -1):
                x = base.copy().reshape(-1)
                x[idx] += sgn * step
                p.assign(x.reshape(base.shape))
                vals.append(float(m.elbo()))
            p.assign(base)
            fd = (vals[0] - vals[1]) / (2 * step)
            assert flat[idx] == pytest.approx(fd, rel=1e-5, abs=1e-5 * max(1.0, np.max(np.abs(flat))))


def test_tiny_latent_variance_matches_sgpr(cuda_device):
    """With S -> 0 the psi statistics become Kuf^T, Kuf Kuf^T and sum Kdiag: elbo() + KL is SGPR's bound at X = mu."""
    N, Q, M, P = 200, 3, 20, 2
    d = _data(N, Q, M, P, seed=7, svar=(1e-14, 1e-14 * (1 + 1e-9)))
    kp, _ = _kernels(1.2)
    m = _model(d, kp)
    kl = float(m.elbo().unchecked().new_tensor(0.0)) + float(np.sum(0.5 * np.log(1.0 / d["S"]) - 0.5
                                                                     + (d["mu"] ** 2 + d["S"]) / 2.0))
    s = gpf.models.SGPR((d["mu"], d["Y"]), gpf.kernels.SquaredExponential(variance=1.3, lengthscales=1.2), d["Z"],
                        noise_variance=0.3)
    assert float(m.elbo()) + kl == pytest.approx(float(s.elbo()), rel=1e-9)


# ---- prediction --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("full_cov", [False, True])
def test_predict_f_and_y_against_oracle(cuda_device, full_cov):
    N, Q, M, P = 60, 2, 10, 3
    d = _data(N, Q, M, P, seed=13)
    kp, ko = _kernels(np.array([0.9, 1.6]))
    m = _model(d, kp)
    Xnew = np.random.default_rng(1).standard_normal((17, Q))
    mean, var = m.predict_f(Xnew, full_cov=full_cov)
    mo, vo = bgplvm_predict_f(d["Y"], d["mu"], d["S"], d["Z"], ko, 0.3, Xnew, full_cov=full_cov)
    np.testing.assert_allclose(mean.cpu().numpy(), mo, rtol=1e-9, atol=1e-10)
    np.testing.assert_allclose(var.cpu().numpy(), vo, rtol=1e-9, atol=1e-10)
    if full_cov:
        _, vd = m.predict_f(Xnew)
        for p in range(P):  # the reference's consistency check
            np.testing.assert_allclose(np.diag(var.cpu().numpy()[p]), vd.cpu().numpy()[:, p], rtol=1e-10, atol=1e-12)
    else:
        ym, yv = m.predict_y(Xnew)
        np.testing.assert_allclose(ym.cpu().numpy(), mo, rtol=1e-9, atol=1e-10)
        np.testing.assert_allclose(yv.cpu().numpy(), vo + 0.3, rtol=1e-9, atol=1e-10)


# ---- the reference's tests (tests/gpflow/models/test_gplvm.py) ---------------------------------------------------
class _Data:
    rng = np.random.RandomState(999)
    N = 20
    D = 5
    Y = rng.randn(N, D)
    Q = 2
    M = 10
    X = np.linspace(0, 1, N)[:, None]


def _raises_elbo(m, maxiter=2):
    before = float(m.elbo())
    gpf.optimizers.Scipy().minimize(m.training_loss_closure(), m.trainable_variables, options=dict(maxiter=maxiter))
    assert float(m.elbo()) > before


def test_bayesian_gplvm_1d(cuda_device):
    Q = 1
    kernel = gpf.kernels.SquaredExponential()
    inducing = np.linspace(0, 1, _Data.M)[:, None]
    m = gpf.models.BayesianGPLVM(_Data.Y, np.zeros((_Data.N, Q)), np.ones((_Data.N, Q)), kernel,
                                 inducing_variable=inducing)
    assert m.inducing_variable.num_inducing == _Data.M
    _raises_elbo(m)


def test_bayesian_gplvm_2d(cuda_device):
    Q = 2
    X_data_mean = gpf.utilities.ops.pca_reduce(_Data.Y, Q)
    kernel = gpf.kernels.SquaredExponential()
    m = gpf.models.BayesianGPLVM(_Data.Y, X_data_mean, np.ones((_Data.N, Q)), kernel,
                                 num_inducing_variables=_Data.M)
    assert m.inducing_variable.num_inducing == _Data.M
    _raises_elbo(m)
    mu, var = m.predict_f(np.random.RandomState(0).randn(3, Q))
    assert mu.shape == (3, _Data.D) and var.shape == (3, _Data.D)
    with pytest.raises(NotImplementedError):
        m.predict_log_density((np.zeros((3, Q)), np.zeros((3, _Data.D))))


def test_gplvm_constructor_checks(cuda_device):
    with pytest.raises(ValueError):
        assert _Data.X.shape[1] == 1
        gpf.models.BayesianGPLVM(_Data.Y, np.zeros((_Data.N, 1)), np.ones((_Data.N, 1)), gpf.kernels.SquaredExponential())
    with pytest.raises(ValueError):
        gpf.models.BayesianGPLVM(_Data.Y, np.zeros((_Data.N, 1)), np.ones((_Data.N, 1)),
                                 gpf.kernels.SquaredExponential(), num_inducing_variables=3,
                                 inducing_variable=np.zeros((3, 1)))
    m = gpf.models.BayesianGPLVM(_Data.Y, _Data.X, np.ones((_Data.N, 1)), gpf.kernels.SquaredExponential(),
                                 num_inducing_variables=5)
    Z = m.inducing_variable.Z.numpy()
    assert all(np.any(np.all(_Data.X == z, axis=1)) for z in Z)  # rows of X_data_mean
    assert float(m.likelihood.variance.numpy()) == 1.0
    assert type(m.X_data_var.transform).__name__ in ("Softplus", "Shifted", "Exp")
    np.testing.assert_array_equal(m.X_prior_mean, 0.0)
    np.testing.assert_array_equal(m.X_prior_var, 1.0)


# ---- Adam with the latent arrays and Z resident on the device ----------------------------------------------------
def test_adam_matches_oracle_loop(cuda_device):
    N, Q, M, P, K = 50, 3, 8, 2, 6
    d = _data(N, Q, M, P, seed=21)
    kp, ko = _kernels(np.array([0.9, 1.3, 1.7]))
    m = _model(d, kp)
    gpf.utilities.set_trainable(m.kernel, False)
    gpf.utilities.set_trainable(m.likelihood, False)
    opt = gpf.optimizers.Adam(0.01)
    var_list = [m.X_data_mean, m.X_data_var, m.inducing_variable.Z]
    loss = m.training_loss_closure()
    opt.minimize(loss, var_list)
    dev = ops.require_cuda()
    mirrors = [p.device(dev).data_ptr() for p in var_list]
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(K - 1):
            opt.minimize(loss, var_list)
        torch.cuda.synchronize()
    # after the first step nothing is uploaded: mu, S, Z, their moments and the prior stay on the device, and the
    # values stay in the same device mirrors
    htod = [e.name for e in prof.events() if "HtoD" in e.name]
    assert not htod, htod
    assert [p.device(dev).data_ptr() for p in var_list] == mirrors
    lower = gpf.config.default_positive_minimum()
    mu, S, Z = d["mu"].copy(), d["S"].copy(), d["Z"].copy()
    state = {k: (np.zeros_like(v), np.zeros_like(v)) for k, v in (("mu", mu), ("S", S), ("Z", Z))}
    hyper = dict(lr=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
    for t in range(1, K + 1):
        g = bgplvm_elbo_grad(d["Y"], mu, S, Z, ko, 0.3)
        mu, *state["mu"] = AO.constrained_step(mu, g["mu"], *state["mu"], t, AO.IDENTITY, 0.0, -1.0, **hyper)
        S, *state["S"] = AO.constrained_step(S, g["S"], *state["S"], t, AO.SOFTPLUS, lower, -1.0, **hyper)
        Z, *state["Z"] = AO.constrained_step(Z, g["Z"], *state["Z"], t, AO.IDENTITY, 0.0, -1.0, **hyper)
    np.testing.assert_allclose(m.X_data_mean.numpy(), mu, rtol=1e-8, atol=1e-8)
    np.testing.assert_allclose(m.X_data_var.numpy(), S, rtol=1e-8, atol=1e-8)
    np.testing.assert_allclose(m.inducing_variable.Z.numpy(), Z, rtol=1e-8, atol=1e-8)


# ---- refusals ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["Matern32", "SumWhite", "Periodic"])
def test_refuses_other_kernels(cuda_device, kernel):
    d = _data(20, 2, 5, 2)
    k = {"Matern32": lambda: gpf.kernels.Matern32(),
         "SumWhite": lambda: gpf.kernels.SquaredExponential() + gpf.kernels.White(),
         "Periodic": lambda: gpf.kernels.Periodic(gpf.kernels.SquaredExponential())}[kernel]()
    m = _model(d, k)
    name = type(k).__name__
    for f in (m.elbo, m.elbo_and_grad, lambda: m.predict_f(np.zeros((2, 2)))):
        with pytest.raises(NotImplementedError, match=name):
            f()


def test_refuses_float32_priors_and_output_cov(cuda_device):
    d = _data(20, 2, 5, 2)
    m = _model(d, gpf.kernels.SquaredExponential())
    m.data = ops.to_device(d["Y"], dtype=np.float32)
    with pytest.raises(NotImplementedError, match="float64"):
        m.elbo()
    m = _model(d, gpf.kernels.SquaredExponential())
    m.kernel.variance.prior = object()
    with pytest.raises(NotImplementedError, match="prior"):
        m.elbo()
    m.kernel.variance.prior = None
    with pytest.raises(NotImplementedError):
        m.predict_f(np.zeros((2, 2)), full_output_cov=True)
    with pytest.raises(NotImplementedError):
        m.predict_log_density((np.zeros((2, 2)), np.zeros((2, 2))))
