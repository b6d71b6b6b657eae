"""Numerical-edge parity of the digit-sliced (wgmma int8) Cholesky path and the non-positive-definite behaviour.

The fp64 trailing updates carry a digit-truncation error (csrc/planes.cuh); these tests sit where it meets the reference's
own limits: likelihood variance at its 1e-6 lower bound (gpflow/likelihoods/scalar_continuous.py:70-77,
utilities/bijectors.py:37-45), a long-lengthscale RBF (lambda_min of K + s2 I ~ 1e-6 against diagonal 1), N >= 2048 so that
the int8 tensor-core levels are engaged, and rows of very different magnitude.  Bars: 1e-5 relative on the LML and the
posterior mean (north star), posterior variance 1e-5 of the prior variance (the variance itself is ~1e-6 here and fp64
LAPACK does not resolve it to 1e-5 relative either: eps * cond ~ 1e-16 * 4e9)."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N", [2048, 4096])
def test_gpr_noise_at_lower_bound_long_lengthscale(cuda_device, N):
    D = 8
    d = O.make_data(2, N, D, 1, n_new=64)
    ell = 4.0 * np.sqrt(D)
    s2 = 1e-6
    kp, ko = gpf.kernels.SquaredExponential(lengthscales=ell), O.SquaredExponential(lengthscales=ell)
    m = gpf.models.GPR((d["X"], d["Y"]), kp, likelihood=gpf.likelihoods.Gaussian(s2 * (1 + 1e-9)))
    s2 = float(m.likelihood.variance.numpy())
    lml = float(m.log_marginal_likelihood())
    assert _lib.load().gpk_potrf_last_slices() == 7  # cond hint (1 + s2) / s2 = 1e6 -> 7 base-256 digit planes
    ref = O.gpr_log_marginal_likelihood(d["X"], d["Y"], ko, s2)
    np.testing.assert_allclose(lml, ref, rtol=1e-5)
    mean, var = m.predict_f(d["Xnew"])
    mo, vo = O.gpr_predict_f(d["X"], d["Y"], ko, s2, d["Xnew"])
    np.testing.assert_allclose(mean.cpu().numpy(), mo, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(var.cpu().numpy(), vo, rtol=1e-5, atol=1e-5)


def test_gpr_engine_follows_conditioning_hint(cuda_device):
    """(kernel variance + noise) / noise selects S = 6 base-256 digit planes (<= 1e4) or S = 7 (as accurate as fp64
    arithmetic: no DMMA fallback); all agree with the oracle at the model tolerance."""
    d = O.make_data(2, 1536, 8, 1)
    lib = _lib.load()
    for s2, want in ((0.1, 6), (1e-5, 7), (2e-7, 7)):
        kp, ko = gpf.kernels.Matern52(lengthscales=3.0), O.Matern52(lengthscales=3.0)
        m = gpf.models.GPR((d["X"], d["Y"]), kp, likelihood=gpf.likelihoods.Gaussian(s2, variance_lower_bound=1e-7))
        lml = float(m.log_marginal_likelihood())
        assert lib.gpk_potrf_last_slices() == want
        np.testing.assert_allclose(lml, O.gpr_log_marginal_likelihood(d["X"], d["Y"], ko, s2), rtol=1e-6)


def test_potrf_rows_spanning_ten_decades(cuda_device):
    """A = D K D with D = diag(10^u), u in [-5, 5]: every row of L has its own scale |L_ij| <= d_i sqrt(K_ii); the static
    per-row exponents of the digit planes follow it.  Compared with LAPACK row by row in relative terms."""
    rng = np.random.default_rng(5)
    n = 2048
    B = rng.standard_normal((n, n + 64))
    K = B @ B.T / n + 0.5 * np.eye(n)
    dsc = 10.0 ** rng.uniform(-5, 5, n)
    A = K * dsc[:, None] * dsc[None, :]
    Ad = ops.to_device(A.copy())
    L, _ = ops.cholesky(Ad)
    Lref = np.linalg.cholesky(A)
    got = L.cpu().numpy()
    np.testing.assert_allclose(got / dsc[:, None], Lref / dsc[:, None], rtol=0, atol=2e-9)
    np.testing.assert_allclose(np.sum(np.log(np.diag(got))), np.sum(np.log(np.diag(Lref))), rtol=1e-10)


def test_fused_objectives_raise_on_non_positive_definite(cuda_device):
    """tf.linalg.cholesky raises InvalidArgumentError in the reference (gpflow/models/gpr.py:102); here the evaluation is
    asynchronous and the error surfaces when the scalar is read on the host."""
    import scipy.linalg

    rng = np.random.default_rng(0)
    X = rng.standard_normal((300, 2))
    Xd, Yd = np.concatenate([X, X]), rng.standard_normal((600, 1))   # duplicated inputs: K is exactly rank deficient
    big = 1e12                                                       # noise 1e-6 is 1e-18 of the diagonal: lost in fp64
    kp, ko = gpf.kernels.SquaredExponential(variance=big), O.SquaredExponential(variance=big)
    m = gpf.models.GPR((Xd, Yd), kp, likelihood=gpf.likelihoods.Gaussian(1e-6 * (1 + 1e-9)))
    v = m.log_marginal_likelihood()          # enqueued, no error yet
    with pytest.raises(ops.NonPositiveDefiniteError):
        float(v)
    assert m.cholesky_info() > 0
    _, info = scipy.linalg.lapack.dpotrf(O.add_noise_cov(ko(Xd), 1e-6), lower=1)
    assert info > 0                          # LAPACK gives up on the same matrix (first failing pivots need not coincide)
    with pytest.raises(ops.NonPositiveDefiniteError):
        m.log_marginal_likelihood().item()
    assert np.isfinite(float(m.log_marginal_likelihood().unchecked().cpu())) or True  # unchecked read never raises
    # SGPR / SVGP: Kuu of a Linear kernel on 2-D inputs has rank 2; with zero jitter 38 of its 40 pivots are rounding
    # noise around zero, so one of them is non-positive (all 38 positive: probability 2^-38)
    gpf.config.set_default_jitter(0.0)
    try:
        Z = rng.standard_normal((40, 2))
        s = gpf.models.SGPR((X, Yd[:300]), gpf.kernels.Linear(), Z, noise_variance=0.1)
        with pytest.raises(ops.NonPositiveDefiniteError):
            float(s.elbo())
        q = gpf.models.SVGP(gpf.kernels.Linear(), gpf.likelihoods.Gaussian(0.1), Z, num_data=300)
        with pytest.raises(ops.NonPositiveDefiniteError):
            float(q.elbo((X, Yd[:300])))
    finally:
        gpf.config.set_default_jitter(1e-6)


def test_earlier_objective_survives_re_evaluation(cuda_device):
    """ADVICE r1: the scalar returned by one evaluation must not change when the model is evaluated again."""
    d = O.make_data(1, 400, 2, 1)
    m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.SquaredExponential(lengthscales=1.0), noise_variance=0.1)
    a = m.log_marginal_likelihood()
    m.kernel.lengthscales.assign(2.0)
    b = m.log_marginal_likelihood()
    assert abs(float(a) - float(b)) > 1e-3
    np.testing.assert_allclose(float(a), O.gpr_log_marginal_likelihood(d["X"], d["Y"], O.SquaredExponential(lengthscales=1.0), 0.1), rtol=1e-9)


def test_single_column_mean_broadcasts_over_outputs(cuda_device):
    """ADVICE r1: Constant(c=[0.5]) with a 3-column Y centres EVERY column (broadcast of gpflow/models/gpr.py:98)."""
    d = O.make_data(1, 300, 2, 3)
    mf = gpf.mean_functions.Constant(np.array([0.5]))
    m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.SquaredExponential(), mean_function=mf, noise_variance=0.1)
    ref = O.gpr_log_marginal_likelihood(d["X"], d["Y"] - 0.5, O.SquaredExponential(), 0.1)
    np.testing.assert_allclose(float(m.log_marginal_likelihood()), ref, rtol=1e-9)
    mean, _ = m.predict_f(d["X"][:10])
    mo, _ = O.gpr_predict_f(d["X"], d["Y"] - 0.5, O.SquaredExponential(), 0.1, d["X"][:10])
    np.testing.assert_allclose(mean.cpu().numpy(), mo + 0.5, rtol=1e-8, atol=1e-9)
    with pytest.raises(ValueError):
        ops.axpby(1.0, ops.to_device(np.zeros((5, 2))), 1.0, ops.to_device(np.zeros((5, 3))))


def test_concurrent_factorisations_on_four_streams(cuda_device):
    """Four GPR models evaluated on four CUDA streams (bench.py's independent-outputs arm of BASELINE configs[4]): the panel
    kernels of only ONE factorisation at a time may poll their leaf's completion counter (potrf.cu::potrf_t) -- four
    grids of polling CTAs would fill the GPU and lock the leaves out.  Values must equal the one-at-a-time results."""
    import torch
    models, ref = [], []
    for i in range(4):
        d = O.make_data(20 + i, 4096, 8, 1)
        m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.Matern52(lengthscales=2.0 + 0.3 * i), noise_variance=0.1)
        models.append(m)
        ref.append(float(m.log_marginal_likelihood()))
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in models]
    cur = torch.cuda.current_stream()
    for _ in range(3):
        vals = []
        for m, s_ in zip(models, streams):
            s_.wait_stream(cur)
            with torch.cuda.stream(s_):
                vals.append(m.log_marginal_likelihood())
        for s_ in streams:
            cur.wait_stream(s_)
        torch.cuda.synchronize()
        np.testing.assert_allclose([float(v) for v in vals], ref, rtol=1e-12)
