"""The heteroskedastic oracle (tests/hetero_oracle.py) on the CPU: the factorised form the device evaluates against the
reference's literal 20 x 20 grid, the closed-form adjoints against finite differences of the grid sum (the v_g = 0
limit included), the reference's tests restated (tests/gpflow/likelihoods/test_heteroskedastic.py and the Gaussian cases
of test_heteroskedastic_constant_variance.py), the SVGP gradient through the likelihood against finite differences,
the descriptor's layout against the C struct, the host-side checks of a HETEROSKEDASTIC descriptor and the constructor's
refusals.  No device needed."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from gpflow_b200.base import Exp, Shifted, Sigmoid, Softplus, positive
from oracle import gp_oracle as O
from tests import hetero_oracle as HO
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
@pytest.mark.parametrize("transform,lower", HO.TRANSFORMS)
def test_factorised_form_agrees_with_the_grid(transform, lower):
    lik = HO.Hetero(transform, lower)
    mu, v, y = HO.rows()
    np.testing.assert_allclose(lik.factorised_ve(mu, v, y), lik.grid_ve(mu, v, y), rtol=1e-14, atol=0)
    m_f, v_f = lik.factorised_mean_and_var(mu, v)
    m_g, v_g = lik.grid_mean_and_var(mu, v)
    np.testing.assert_allclose(m_f, m_g, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(v_f, v_g, rtol=1e-12, atol=0)


@pytest.mark.parametrize("transform,lower", HO.TRANSFORMS)
def test_adjoints_agree_with_finite_differences_of_the_grid(transform, lower):
    lik = HO.Hetero(transform, lower)
    mu, v, y = HO.rows(1)
    dmu, dv, dpar = lik.ve_grads(mu, v, y)
    assert not np.any(dpar)
    for n in range(mu.shape[0]):
        def f(m, vv):
            return float(lik.grid_ve(m[None], vv[None], y[n:n + 1])[0])

        for p in range(2):
            h = 1e-6
            e = np.eye(2)[p]
            fd = (f(mu[n] + h * e, v[n]) - f(mu[n] - h * e, v[n])) / (2 * h)
            scale = max(1.0, abs(fd))
            assert abs(dmu[n, p] - fd) <= 2e-7 * scale, (n, p, dmu[n, p], fd)
            if v[n, p] > 0:
                hv = 1e-6 * v[n, p]
                fd = (f(mu[n], v[n] + hv * e) - f(mu[n], v[n] - hv * e)) / (2 * hv)
                tol = 2e-6
            else:  # one-sided at v = 0; the error is O(h f'')
                hv = 1e-8
                fd = (f(mu[n], v[n] + hv * e) - f(mu[n], v[n])) / hv
                tol = 1e-5
            assert abs(dv[n, p] - fd) <= tol * max(1.0, abs(fd)), (n, p, dv[n, p], fd)


def test_location_adjoints_are_exact_at_zero_variance():
    lik = HO.Hetero()
    mu, v, y = HO.rows(2)
    v[:, 0] = 0.0
    dmu, dv, _ = lik.ve_grads(mu, v, y)
    S = np.sum(LO.gh_points_and_weights()[1] * np.exp(-2 * (mu[:, 1:2] + np.sqrt(v[:, 1:2])
                                                            * LO.gh_points_and_weights()[0])), 1)
    np.testing.assert_allclose(dmu[:, 0], (y[:, 0] - mu[:, 0]) * S, rtol=1e-14)
    np.testing.assert_allclose(dv[:, 0], -0.5 * S, rtol=1e-14)
    assert np.all(np.isfinite(dv))


# ---- the reference's tests -------------------------------------------------------------------------------------
def test_analytic_mean_and_var():
    """test_heteroskedastic.py::test_analytic_mean_and_var: N(y | f1, exp(f2)^2) has Var[y] = exp(mu_2 + v_2)^2 + v_1."""
    rng = np.random.RandomState(123)
    N = 5
    _ = np.linspace(0, 1, num=N)[:, None]
    _ = rng.randn(N, 1)
    f_mean = rng.randn(N, 2)
    f_var = rng.randn(N, 2) ** 2
    analytic_mean = f_mean[:, [0]]
    analytic_variance = np.exp(f_mean[:, [1]] + f_var[:, [1]]) ** 2 + f_var[:, [0]]
    lik = HO.Hetero()
    for mean, var in (lik.grid_mean_and_var(f_mean, f_var), lik.factorised_mean_and_var(f_mean, f_var)):
        np.testing.assert_allclose(mean, analytic_mean)
        np.testing.assert_allclose(var, analytic_variance, rtol=1.5e-6)


class _ConstantVariance:
    """test_heteroskedastic_constant_variance.py::Data: g = log(0.345) / 2 with v_g = 0 is Gaussian(0.345)."""
    g_var = 0.345
    rng = np.random.RandomState(123)
    N = 5
    X = rng.randn(N, 2)
    Y = rng.randn(N, 1)
    f_mean = rng.randn(N, 1)
    f_var = rng.randn(N, 1) ** 2
    F2_mean = np.c_[f_mean, np.full((N, 1), np.log(g_var) / 2)]
    F2_var = np.c_[f_var, np.zeros((N, 1))]


def test_constant_variance_is_the_gaussian_likelihood():
    D = _ConstantVariance
    gauss, het = LO.Gaussian(D.g_var), HO.Hetero()
    np.testing.assert_allclose(het.grid_ve(D.F2_mean, D.F2_var, D.Y),
                               gauss.variational_expectations(D.f_mean, D.f_var, D.Y)[:, 0], rtol=1e-13)
    np.testing.assert_allclose(het.predict_mean_and_var(D.F2_mean, D.F2_var),
                               gauss.predict_mean_and_var(D.f_mean, D.f_var), rtol=1e-14)
    # the log density is a 20-point quadrature of the Gaussian's closed form (the reference checks 1 decimal)
    np.testing.assert_array_almost_equal(het.predict_log_density(D.F2_mean, D.F2_var, D.Y),
                                         gauss.predict_log_density(D.f_mean, D.f_var, D.Y), decimal=1)
    np.testing.assert_allclose(het.predict_log_density(D.F2_mean, D.F2_var, D.Y),
                               LO.Gaussian(D.g_var).quad_log_density(D.f_mean, D.f_var, D.Y), rtol=1e-13)


# ---- the SVGP gradient through the likelihood --------------------------------------------------------------------
@pytest.mark.parametrize("whiten", [True, False])
def test_svgp_gradient_agrees_with_finite_differences(whiten):
    rng = np.random.default_rng(3)
    B, M, D, L = 25, 6, 2, 3
    X = rng.standard_normal((B, D))
    Y = np.sin(X[:, :1]) + 0.4 * rng.standard_normal((B, 1))
    Zs = [rng.standard_normal((M, D)) for _ in range(L)]
    ks = [O.SquaredExponential(1.1, 0.9), O.Matern32(0.7, 1.2), O.SquaredExponential(0.5, 1.4)]
    W = 0.6 * rng.standard_normal((2, L))
    q_mu = 0.3 * rng.standard_normal((M, L))
    q_sqrt = np.stack([np.tril(0.1 * rng.standard_normal((M, M)), -1) + np.diag(0.4 + 0.3 * rng.random(M))
                       for _ in range(L)])
    lik = HO.Hetero("softplus", 1e-3)
    mf = O.LinearMean(0.2 * rng.standard_normal((D, 2)), np.array([0.1, -0.3]))
    _, g = S.svgp_elbo_and_grad(X, Y, ks, Zs, q_mu, q_sqrt, lik, W=W, whiten=whiten, num_data=100, mean_function=mf)

    def f(qm=q_mu, WW=W, Zl=Zs):
        return S.svgp_elbo(X, Y, ks, Zl, qm, q_sqrt, lik, W=WW, whiten=whiten, num_data=100, mean_function=mf)

    h = 1e-6
    for name, arr, ref, fn in [("q_mu", q_mu, g["q_mu"], lambda a: f(qm=a)), ("W", W, g["W"], lambda a: f(WW=a)),
                               ("Z0", Zs[0], g["Z"][0], lambda a: f(Zl=[a] + Zs[1:]))]:
        for idx in [(0, 0), (1, 1), (arr.shape[0] - 1, arr.shape[1] - 1)]:
            p, m = arr.copy(), arr.copy()
            p[idx] += h
            m[idx] -= h
            fd = (fn(p) - fn(m)) / (2 * h)
            assert abs(ref[idx] - fd) <= 1e-6 * max(1.0, abs(fd)), (name, idx, ref[idx], fd)
    A = mf.A
    for idx in [(0, 0), (1, 1)]:
        p, m = A.copy(), A.copy()
        p[idx] += h
        m[idx] -= h
        fp = S.svgp_elbo(X, Y, ks, Zs, q_mu, q_sqrt, lik, W=W, whiten=whiten, num_data=100,
                         mean_function=O.LinearMean(p, mf.b))
        fm = S.svgp_elbo(X, Y, ks, Zs, q_mu, q_sqrt, lik, W=W, whiten=whiten, num_data=100,
                         mean_function=O.LinearMean(m, mf.b))
        fd = (fp - fm) / (2 * h)
        assert abs(g["mean"]["A"][idx] - fd) <= 1e-6 * max(1.0, abs(fd))


# ---- the descriptor ---------------------------------------------------------------------------------------------
def test_descriptor_mirror_has_the_c_layout(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "a host C compiler (the one nvcc drives) is needed"
    src = tmp_path / "size.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gpk.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %d %d %d\\n", sizeof(gpk_lik), '
                   'offsetof(gpk_lik, epsilon), offsetof(gpk_lik, num_classes), offsetof(gpk_lik, scale_transform), '
                   'offsetof(gpk_lik, scale_lower), GPK_LIK_HETEROSKEDASTIC, GPK_LIK_SCALE_EXP, '
                   'GPK_LIK_SCALE_SOFTPLUS); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    vals = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    size, off_eps, off_c, off_t, off_l, het, sexp, ssp = vals
    assert ctypes.sizeof(_lib.LikDesc) == size
    assert (_lib.LikDesc.epsilon.offset, _lib.LikDesc.num_classes.offset) == (off_eps, off_c)
    assert (_lib.LikDesc.scale_transform.offset, _lib.LikDesc.scale_lower.offset) == (off_t, off_l)
    assert (_lib.LIK_HETEROSKEDASTIC, _lib.LIK_SCALE_EXP, _lib.LIK_SCALE_SOFTPLUS) == (het, sexp, ssp)
    # the existing positional constructions keep their meaning
    d = _lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0.0, 0.0, 0.0, 0.0, 0.01, 7)
    assert (d.epsilon, d.num_classes, d.scale_transform, d.scale_lower) == (0.01, 7, 0, 0.0)


def _het(transform=_lib.LIK_SCALE_EXP, lower=0.0, n_gh=20):
    return _lib.LikDesc(_lib.LIK_HETEROSKEDASTIC, n_gh, 0.0, 0.0, 0.0, 0.0, 0.0, 0, transform, lower)


def _grad_call(lik, P):
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential(), 3)
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: the checks run on the host before the first launch
    st = lib.gpk_svgp_elbo_grad(nodes, n, dims, ard, fake, 100, 3, 3, fake, None, P, fake, 10, 3, fake, fake, 0, 1,
                                ctypes.byref(lik), 1.0, 1e-6, _lib.GPK_F64, fake, 64, fake, fake, fake, fake, None)
    return st, lib.gpk_last_error().decode()


def test_host_checks_of_the_descriptor():
    for bad, P, word in [(_het(), 1, "P = 1"), (_het(), 3, "P = 3"), (_het(2), 2, "scale transform"),
                         (_het(-1), 2, "scale transform"), (_het(lower=-1e-3), 2, "scale_lower"),
                         (_het(lower=float("inf")), 2, "scale_lower"), (_het(lower=float("nan")), 2, "scale_lower"),
                         (_het(n_gh=10), 2, "Gauss-Hermite")]:
        st, msg = _grad_call(bad, P)
        assert st == -1 and word in msg, msg
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    out = ctypes.c_double(0.0)
    for fn, args in [(lib.gpk_lik_varexp_sum, (fake, fake, fake, 10, 1, 1.0, 0, ctypes.byref(out))),
                     (lib.gpk_lik_predict_mean_and_var, (fake, fake, 10, 3, fake, fake)),
                     (lib.gpk_lik_predict_log_density, (fake, fake, fake, 10, 1, fake))]:
        st = fn(ctypes.byref(_het()), *args, _lib.GPK_F64, None)
        assert st == -1 and "2 latents" in lib.gpk_last_error().decode()
    st = lib.gpk_lik_varexp_grad(ctypes.byref(_het()), fake, fake, fake, 10, 1, 1.0, fake, fake, fake, None)
    assert st == -1 and "2 latents" in lib.gpk_last_error().decode()
    st = lib.gpk_lik_varexp_grad(ctypes.byref(_het()), fake, fake, fake, 10, 2, 1.0, fake, fake, None, None)
    assert st == -1 and "null" in lib.gpk_last_error().decode()
    # a latent sub-range of the value entry
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential(), 3)
    st = lib.gpk_svgp_elbo_staged(nodes, n, dims, ard, fake, 100, 3, 3, fake, None, 2, fake, 10, 3, fake, fake, 0, 1,
                                  ctypes.byref(_het()), 1.0, 1e-6, 0, 1, 0, 0, 100, _lib.GPK_F64, fake, fake, None)
    assert st == -1 and "couples the latents" in lib.gpk_last_error().decode()
    # the gradient workspace has the per-latent scratch of a non-Gaussian likelihood
    gauss = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1)
    assert lib.gpk_svgp_elbo_grad_ws(1000, 64, 2, ctypes.byref(_het()), _lib.GPK_F64) > \
        lib.gpk_svgp_elbo_grad_ws(1000, 64, 2, ctypes.byref(gauss), _lib.GPK_F64)


# ---- the Python class ----------------------------------------------------------------------------------------------
def test_constructor_and_descriptor():
    L = gpf.likelihoods
    lik = L.HeteroskedasticTFPConditional()
    assert lik.latent_dim == 2 and lik.observation_dim == 1 and lik.distribution_class is L.Normal
    assert isinstance(lik.scale_transform, Exp) and lik.parameters == ()
    d = lik._lik_desc()
    assert (d.type, d.n_gh, d.scale_transform, d.scale_lower) == (_lib.LIK_HETEROSKEDASTIC, 20, _lib.LIK_SCALE_EXP, 0.0)
    for t, code, lower in [(Softplus(), _lib.LIK_SCALE_SOFTPLUS, 0.0), (Shifted(Exp(), 1e-3), _lib.LIK_SCALE_EXP, 1e-3),
                           (positive(lower=0.01, base="softplus"), _lib.LIK_SCALE_SOFTPLUS, 0.01),
                           (np.exp, _lib.LIK_SCALE_EXP, 0.0)]:
        d = L.HeteroskedasticTFPConditional(scale_transform=t)._lik_desc()
        assert (d.scale_transform, d.scale_lower) == (code, lower)


def test_constructor_refusals():
    L = gpf.likelihoods

    class StudentT:
        pass

    with pytest.raises(NotImplementedError, match="StudentT"):
        L.HeteroskedasticTFPConditional(distribution_class=StudentT)
    with pytest.raises(NotImplementedError, match="Sigmoid"):
        L.HeteroskedasticTFPConditional(scale_transform=Sigmoid())
    with pytest.raises(NotImplementedError, match="square"):
        L.HeteroskedasticTFPConditional(scale_transform=np.square)
    with pytest.raises(NotImplementedError, match="quadrature"):
        L.HeteroskedasticTFPConditional(quadrature=object())
    with pytest.raises(ValueError, match="lower"):
        L.HeteroskedasticTFPConditional(scale_transform=Shifted(Exp(), -1.0))
