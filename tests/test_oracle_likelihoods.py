"""The likelihood oracle (tests/lik_oracle.py) on the CPU: the Gauss-Hermite table committed in csrc/lik.cu, the
reference's likelihood tests restated (tests/gpflow/likelihoods/test_likelihoods.py: variational expectations at zero
variance, closed forms against the quadrature fallback, conditional moments), and the SVGP ELBO gradient oracle
(tests/svgp_grad_oracle.py) through Bernoulli / Poisson / Student-t (and Gaussian) against central finite differences
of its ELBO; the host-side refusals of the likelihood classes and of gpk_svgp_elbo_grad.  No device needed."""
import copy
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import kernel_grad_oracle as KG
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as S

LIKS = ["bernoulli", "poisson", "student_t", "gaussian"]


def _lik(name):
    return {"bernoulli": LO.Bernoulli(), "poisson": LO.Poisson(binsize=1.3), "student_t": LO.StudentT(0.7, 4.0),
            "gaussian": LO.Gaussian(0.3)}[name]


def test_committed_gauss_hermite_table_is_hermgauss_20():
    z, w = LO.cuda_gh_table()
    x, wx = np.polynomial.hermite.hermgauss(20)
    np.testing.assert_array_equal(z, x * np.sqrt(2))
    np.testing.assert_array_equal(w, wx / np.sqrt(np.pi))
    assert abs(w.sum() - 1.0) < 1e-14


def _elements(name, shape=(7, 3), seed=0):
    rng = np.random.default_rng(seed)
    mu = rng.uniform(-1.5, 1.5, shape)
    v = rng.uniform(0.05, 1.2, shape)
    return mu, v, LO.targets(name, mu, rng)


@pytest.mark.parametrize("name", LIKS)
def test_variational_expectations_at_zero_variance_equal_log_prob(name):
    lik = _lik(name)
    mu, _, y = _elements(name)
    np.testing.assert_allclose(lik.variational_expectations(mu, np.zeros_like(mu), y), lik.logp(y, mu), rtol=1e-12,
                               atol=1e-12)


def test_poisson_closed_form_variational_expectations_equal_quadrature():
    lik = _lik("poisson")
    mu, v, y = _elements("poisson")
    np.testing.assert_allclose(lik.variational_expectations(mu, v, y), lik.quad_ve(mu, v, y), rtol=1e-6, atol=1e-6)


def test_bernoulli_closed_forms_equal_quadrature():
    lik = _lik("bernoulli")
    mu, v, y = _elements("bernoulli")
    np.testing.assert_allclose(lik.predict_log_density(mu, v, y), lik.quad_log_density(mu, v, y), rtol=1e-6,
                               atol=1e-6)
    for a, b in zip(lik.predict_mean_and_var(mu, v), lik.quad_mean_and_var(mu, v)):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", LIKS)
def test_conditional_moments_equal_predict_mean_and_var_at_zero_variance(name):
    lik = _lik(name)
    mu, _, _ = _elements(name)
    m, v = lik.predict_mean_and_var(mu, np.zeros_like(mu))
    np.testing.assert_allclose(m, lik.conditional_mean(mu), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(v, lik.conditional_variance(mu), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", LIKS)
def test_variational_expectation_derivatives_match_finite_differences(name):
    lik = _lik(name)
    mu, v, y = _elements(name)
    dmu, dv, dpar = lik.ve_grads(mu, v, y)
    h = 1e-6
    np.testing.assert_allclose(dmu, (lik.variational_expectations(mu + h, v, y)
                                     - lik.variational_expectations(mu - h, v, y)) / (2 * h), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(dv, (lik.variational_expectations(mu, v + h, y)
                                    - lik.variational_expectations(mu, v - h, y)) / (2 * h), rtol=1e-6, atol=1e-7)
    if name in ("student_t", "gaussian"):
        attr = "scale" if name == "student_t" else "variance"
        lp, lm = copy.deepcopy(lik), copy.deepcopy(lik)
        setattr(lp, attr, getattr(lik, attr) + h)
        setattr(lm, attr, getattr(lik, attr) - h)
        fd = (lp.variational_expectations(mu, v, y) - lm.variational_expectations(mu, v, y)) / (2 * h)
        np.testing.assert_allclose(dpar, fd, rtol=1e-6, atol=1e-7)
    else:
        assert np.all(dpar == 0.0)


# ---- the SVGP ELBO gradient ------------------------------------------------------------------------------------
def _data(name, P, B=9, M=5, D=3, q_diag=False, seed=20261016):
    rng = np.random.default_rng(seed + P + 10 * q_diag)
    X = rng.standard_normal((B, D))
    Y = LO.targets(name, np.sin(X[:, :1] @ np.ones((1, P))), rng)
    Z = 1.2 * rng.standard_normal((M, D)) + 0.1
    q_mu = 0.5 * rng.standard_normal((M, P))
    if q_diag:
        q_sqrt = 0.3 + 0.5 * rng.random((M, P))
    else:
        q_sqrt = np.stack([np.tril(0.2 * rng.standard_normal((M, M)), -1) + np.diag(0.4 + 0.5 * rng.random(M))
                           for _ in range(P)])
        q_sqrt += np.triu(rng.standard_normal((M, M)), 1)[None]   # band_part drops the strict upper part
    return X, Y, Z, q_mu, q_sqrt


def _check_all(name, kernel, X, Y, Z, q_mu, q_sqrt, whiten, num_data, tol=5e-6, h=1e-5):
    lik = _lik(name)

    def f(k=kernel, Zv=Z, qm=q_mu, qs=q_sqrt, lk=lik):
        return S.svgp_elbo(X, Y, [k], [Zv], qm, qs, lk, whiten=whiten, num_data=num_data)

    elbo, g = S.svgp_elbo_and_grad(X, Y, [kernel], [Z], q_mu, q_sqrt, lik, whiten=whiten, num_data=num_data)
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    for li, _ in enumerate(KG.leaves(kernel)):
        for pname, got in g["leaves"][li].items():
            for idx in np.ndindex(np.shape(got)):
                fd = (f(k=GC.perturb(kernel, li, pname, idx, h))
                      - f(k=GC.perturb(kernel, li, pname, idx, -h))) / (2 * h)
                GC.close(float(np.asarray(got)[idx]), fd, tol, (li, pname, idx))
    if name in ("student_t", "gaussian"):
        attr = "scale" if name == "student_t" else "variance"
        lp, lm = copy.deepcopy(lik), copy.deepcopy(lik)
        setattr(lp, attr, getattr(lik, attr) + h)
        setattr(lm, attr, getattr(lik, attr) - h)
        GC.close(g["lik"], (f(lk=lp) - f(lk=lm)) / (2 * h), tol, attr)
    else:
        assert g["lik"] == 0.0
    for idx in np.ndindex(Z.shape):
        GC.close(g["Z"][idx], GC.fd_array(lambda v: f(Zv=v), Z, idx, h), tol, ("Z", idx))
    for idx in np.ndindex(q_mu.shape):
        GC.close(g["q_mu"][idx], GC.fd_array(lambda v: f(qm=v), q_mu, idx, h), tol, ("q_mu", idx))
    assert g["q_sqrt"].shape == q_sqrt.shape
    for idx in np.ndindex(q_sqrt.shape):
        if q_sqrt.ndim == 3 and idx[2] > idx[1]:
            assert g["q_sqrt"][idx] == 0.0
            continue
        GC.close(g["q_sqrt"][idx], GC.fd_array(lambda v: f(qs=v), q_sqrt, idx, h), tol, ("q_sqrt", idx))


@pytest.mark.parametrize("name", LIKS)
@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("q_diag", [False, True])
@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("num_data", [None, 40])
def test_svgp_lik_gradient_matches_finite_differences(name, whiten, q_diag, P, num_data):
    X, Y, Z, q_mu, q_sqrt = _data(name, P, q_diag=q_diag)
    _check_all(name, O.SquaredExponential(1.3, 1.7) + O.White(0.05), X, Y, Z, q_mu, q_sqrt, whiten, num_data)


EXPRESSIONS = {
    "c5": lambda: (O.SquaredExponential(1.1, 2.1) + O.Matern32(1.0, 4.0)) * O.Linear(0.5),
    "rq_ard": lambda: O.RationalQuadratic(1.2, np.array([1.1, 1.9, 0.7]), alpha=2.5),
    "polynomial_ard": lambda: O.Polynomial(degree=2.0, variance=np.array([0.2, 0.1, 0.3]), offset=1.3),
    "constant_times_matern52": lambda: O.Constant(1.7) * O.Matern52(0.9, 1.8),
}


@pytest.mark.parametrize("expr", list(EXPRESSIONS))
@pytest.mark.parametrize("name", ["bernoulli", "student_t"])
def test_svgp_lik_gradient_of_every_hyperparameter(expr, name):
    X, Y, Z, q_mu, q_sqrt = _data(name, 2)
    _check_all(name, EXPRESSIONS[expr](), X, Y, Z, q_mu, q_sqrt, whiten=expr != "rq_ard", num_data=30)


@pytest.mark.parametrize("name", ["bernoulli", "poisson", "student_t"])
@pytest.mark.parametrize("kind", ["constant_per_output", "linear", "linear_one_column"])
def test_svgp_lik_mean_function_gradient_matches_finite_differences(name, kind):
    P = 2
    X, Y, Z, q_mu, q_sqrt = _data(name, P)
    D = X.shape[1]
    kernel = O.SquaredExponential(1.3, 1.7) + O.Linear(0.2)
    rng = np.random.default_rng(5)
    if kind == "constant_per_output":
        mf = O.ConstantMean(0.1 * np.arange(1, P + 1))
        params = {"c": mf.c}
    elif kind == "linear":
        mf = O.LinearMean(0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1))
        params = {"A": mf.A, "b": mf.b}
    else:
        mf = O.LinearMean(0.2 * rng.standard_normal((D, 1)), np.array([0.4]))
        params = {"A": mf.A, "b": mf.b}
    lik = _lik(name)
    _, g = S.svgp_elbo_and_grad(X, Y, [kernel], [Z], q_mu, q_sqrt, lik, num_data=30, mean_function=mf)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = S.svgp_elbo(X, Y, [kernel], [Z], q_mu, q_sqrt, lik, num_data=30, mean_function=mf)
            arr[idx] -= 2 * h
            fm = S.svgp_elbo(X, Y, [kernel], [Z], q_mu, q_sqrt, lik, num_data=30, mean_function=mf)
            arr[idx] += h
            GC.close(g["mean"][pname][idx], (fp - fm) / (2 * h), 1e-6, (pname, idx))


# ---- host-side refusals ---------------------------------------------------------------------------------------
def test_likelihood_classes_refuse_what_the_device_does_not_cover():
    L = gpf.likelihoods
    with pytest.raises(NotImplementedError, match="probit"):
        L.Bernoulli(invlink=np.exp)
    with pytest.raises(NotImplementedError, match="exp"):
        L.Poisson(invlink=np.square)
    with pytest.raises(NotImplementedError, match="Function"):
        L.StudentT(scale=gpf.mean_functions.Constant(1.0))
    for cls in (L.Bernoulli, L.Poisson, L.StudentT):
        with pytest.raises(NotImplementedError, match="quadrature"):
            cls(quadrature=object())
    t = L.StudentT(scale=0.5, df=4.0)
    assert float(t.scale.numpy()) == pytest.approx(0.5) and t.df == 4.0
    assert L.Poisson(binsize=2.0).binsize == 2.0


def test_svgp_grad_entry_point_rejects_bad_likelihood_descriptors():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    good = _lib.LikDesc(_lib.LIK_BERNOULLI, 20, 0.0, 0.0, 0.0, 0.0)
    st, msg = GC.svgp_grad_status(nodes, n, dims, ard, 3, good, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = GC.svgp_grad_status(nodes, n, dims, ard, 3, good, n_out=7)
    assert st == -1 and "n_out" in msg and "8" in msg
    st, msg = GC.svgp_grad_status(nodes, n, dims, ard, 3, good, dZ=False)
    assert st == -1 and "dZ" in msg
    for bad, word in [(_lib.LikDesc(9, 20, 0, 0, 0, 0), "unknown"),
                      (_lib.LikDesc(_lib.LIK_BERNOULLI, 10, 0, 0, 0, 0), "Gauss-Hermite"),
                      (_lib.LikDesc(_lib.LIK_STUDENT_T, 20, -1.0, 3.0, 0, 0), "Student-t"),
                      (_lib.LikDesc(_lib.LIK_POISSON, 20, 0, 0, 0.0, 0), "binsize"),
                      (_lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0, 0, 0, 0.0), "noise")]:
        st, msg = GC.svgp_grad_status(nodes, n, dims, ard, 3, bad)
        assert st == -1 and word in msg, msg
    lib = _lib.load()
    # the value entry: MultiClass couples the latents of a row, so a latent sub-range is refused
    fake = ctypes.c_void_p(256)
    three = _lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0.0, 0.0, 0.0, 0.0, 0.01, 3)
    st = lib.gpk_svgp_elbo(nodes, n, dims, ard, fake, 100, 3, 3, fake, None, 3, fake, 10, 3, fake, fake, 0, 1,
                           ctypes.byref(three), 1.0, 1e-6, 0, 2, _lib.GPK_F64, fake, fake, None)
    assert st == -1 and "latent range" in lib.gpk_last_error().decode()
    student_t = _lib.LikDesc(_lib.LIK_STUDENT_T, 20, 0.7, 4.0, 0.0, 0.0)
    gauss = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1)
    ws = lib.gpk_svgp_elbo_grad_ws(1000, 64, 2, ctypes.byref(student_t), _lib.GPK_F64)
    assert ws > lib.gpk_svgp_elbo_grad_ws(1000, 64, 2, ctypes.byref(gauss), _lib.GPK_F64)
    off = lib.gpk_svgp_elbo_grad_dm(1000, 64, 2, _lib.GPK_F64)
    assert off % 256 == 0 and off + 8 * 1000 * 2 <= ws
