"""The MultiClass oracle (tests/multiclass_oracle.py) on the CPU: the reference's RobustMax tests restated
(tests/gpflow/likelihoods/test_multiclass.py: symmetric inputs, a mocked probability, eps_k1 after reassignment), the
adjoints and the SVGP ELBO gradient against central finite differences, the host-side checks of a MULTICLASS descriptor,
the descriptor's layout, the Sigmoid transform and the MultiClass / RobustMax constructors.  No device needed."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
from scipy.special import erf

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from gpflow_b200.base import Sigmoid
from oracle import gp_oracle as O
from tests import multiclass_oracle as MO
from tests import svgp_grad_oracle as S
from tests.test_oracle_likelihoods import _call, _close, _fd_array, _perturb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the reference's RobustMax tests ---------------------------------------------------------------------------
def test_symmetric_inputs_give_equal_class_probabilities():
    C, N, eps = 10, 3, 1e-3
    lik = MO.MultiClass(C, eps)
    F = np.ones((N, C))
    Y = np.random.RandomState(1).randint(C, size=(N, 1)).astype(np.float64)
    p = 1.0 / C
    expected = p * (1 - eps) + (1 - p) * eps / (C - 1)
    mean, _ = lik.predict_mean_and_var(F, F)
    assert np.allclose(mean, expected, 1e-4, 1e-4)
    assert np.allclose(lik.predict_log_density(F, F, Y), np.log(expected), 1e-3, 1e-3)
    ve = p * np.log(1 - eps) + (1 - p) * np.log(eps / (C - 1))
    np.testing.assert_allclose(lik.variational_expectations(F, F, Y), np.full(N, ve), 1e-4, 1e-4)


def test_log_density_of_a_mocked_probability():
    lik = MO.MultiClass(5, 0.231)
    np.testing.assert_allclose(np.log(lik.density(None, None, None, p=np.full(100, 0.73))), -0.5499780059,
                               rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("C", [5, 100])
def test_eps_k1_follows_a_reassigned_epsilon(C):
    link = gpf.likelihoods.RobustMax(C, 1e-3)
    np.testing.assert_allclose(link.eps_k1, 1e-3 / (C - 1))
    link.epsilon = 0.412
    np.testing.assert_allclose(link.eps_k1, 0.412 / (C - 1))
    lik = gpf.likelihoods.MultiClass(C, invlink=link)
    assert lik._lik_desc().epsilon == 0.412


# ---- the adjoints ----------------------------------------------------------------------------------------------
def _rows(C, N=6, seed=0):
    rng = np.random.default_rng(seed + C)
    mu = rng.uniform(-1.5, 1.5, (N, C))
    var = rng.uniform(0.05, 1.2, (N, C))
    var[0, 1] = 3e-11                    # inside the clamp of s_c
    var[1, :] = 2e-11                    # 2 v_y inside the clamp of s_y, whatever the label
    Y = np.argmax(mu + 0.5 * rng.standard_normal(mu.shape), 1)[:, None].astype(np.float64)
    Y[2, 0] = C + 1.0                    # outside [0, C): no class left out of the product
    Y[3, 0] = -1.0
    Y[4, 0] += 0.7                       # truncated
    return mu, var, Y


@pytest.mark.parametrize("C", [2, 3, 5, 40])
def test_adjoints_match_finite_differences(C):
    lik = MO.MultiClass(C, 0.02)
    mu, var, Y = _rows(C)
    dmu, dv, deps = lik.ve_grads(mu, var, Y)
    h = 1e-6
    for idx in np.ndindex(mu.shape):
        fd = _fd_array(lambda m: lik.variational_expectations(m, var, Y)[idx[0]], mu, idx, h)
        _close(dmu[idx], fd, 1e-7, ("mu", idx))
        if var[idx] < 1e-9:  # inside the clamp (of s_c, and of s_y for a label): the expectation does not move with it
            assert dv[idx] == 0.0
            continue
        fd = _fd_array(lambda v: lik.variational_expectations(mu, v, Y)[idx[0]], var, idx, h)
        _close(dv[idx], fd, 1e-6, ("var", idx))
    for n in range(mu.shape[0]):
        lp, lm = MO.MultiClass(C, 0.02 + h), MO.MultiClass(C, 0.02 - h)
        fd = (lp.variational_expectations(mu, var, Y)[n] - lm.variational_expectations(mu, var, Y)[n]) / (2 * h)
        _close(deps[n], fd, 1e-7, ("eps", n))


def test_label_outside_the_classes_leaves_every_class_in_the_product():
    lik = MO.MultiClass(4, 0.01)
    mu, var, Y = _rows(4)
    p = lik.prob_is_largest(Y[2:3], mu[2:3], var[2:3])
    x, w = MO.gh()
    d = (x[None, :] * 1e-5 - mu[2][:, None]) / np.sqrt(var[2])[:, None]
    cdf = 0.5 * (1 + erf(d / np.sqrt(2))) * (1 - 2e-6) + 1e-6
    np.testing.assert_allclose(p, np.prod(cdf, 0) @ w, rtol=1e-14)


def test_exclusive_products_survive_many_classes():
    """At 100 classes the full product underflows where the exclusive products do not, so dividing the full product by
    cdf_ck would give 0 / 0; the prefix-suffix form stays finite."""
    C = 100
    lik = MO.MultiClass(C)
    mu = np.full((1, C), 3.0)
    mu[0, 0] = -3.0
    var = np.full((1, C), 0.01)
    dmu, dv, deps = lik.ve_grads(mu, var, np.zeros((1, 1)))
    assert np.all(np.isfinite(dmu)) and np.all(np.isfinite(dv)) and np.isfinite(deps).all()


# ---- the SVGP ELBO gradient ------------------------------------------------------------------------------------
def _data(C, B=9, M=5, D=3, q_diag=False, seed=20261016):
    rng = np.random.default_rng(seed + C + 10 * q_diag)
    X = rng.standard_normal((B, D))
    Y = MO.labels(rng, np.sin(X[:, :1] + np.arange(C)[None]))
    Y[0, 0] = float(C)                   # one label outside the classes
    Z = 1.2 * rng.standard_normal((M, D)) + 0.1
    q_mu = 0.5 * rng.standard_normal((M, C))
    if q_diag:
        q_sqrt = 0.3 + 0.5 * rng.random((M, C))
    else:
        q_sqrt = np.stack([np.tril(0.2 * rng.standard_normal((M, M)), -1) + np.diag(0.4 + 0.5 * rng.random(M))
                           for _ in range(C)])
        q_sqrt += np.triu(rng.standard_normal((M, M)), 1)[None]
    return X, Y, Z, q_mu, q_sqrt


def _check_all(kernel, X, Y, Z, q_mu, q_sqrt, whiten, num_data, eps=0.05, mean_function=None, tol=5e-6, h=1e-5):
    C = q_mu.shape[1]

    def f(k=kernel, Zv=Z, qm=q_mu, qs=q_sqrt, e=eps):
        return MO.svgp_elbo(X, Y, Zv, k, qm, qs, MO.MultiClass(C, e), whiten=whiten, num_data=num_data,
                            mean_function=mean_function)

    elbo, g = MO.svgp_elbo_and_grad(X, Y, kernel, Z, q_mu, q_sqrt, MO.MultiClass(C, eps), whiten=whiten,
                                    num_data=num_data, mean_function=mean_function)
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    for li, _ in enumerate(S.leaves(kernel)):
        for pname, got in g["leaves"][li].items():
            for idx in np.ndindex(np.shape(got)):
                fd = (f(k=_perturb(kernel, li, pname, idx, h)) - f(k=_perturb(kernel, li, pname, idx, -h))) / (2 * h)
                _close(float(np.asarray(got)[idx]), fd, tol, (li, pname, idx))
    _close(g["lik"], (f(e=eps + h) - f(e=eps - h)) / (2 * h), tol, "epsilon")
    for idx in np.ndindex(Z.shape):
        _close(g["Z"][idx], _fd_array(lambda v: f(Zv=v), Z, idx, h), tol, ("Z", idx))
    for idx in np.ndindex(q_mu.shape):
        _close(g["q_mu"][idx], _fd_array(lambda v: f(qm=v), q_mu, idx, h), tol, ("q_mu", idx))
    assert g["q_sqrt"].shape == q_sqrt.shape
    for idx in np.ndindex(q_sqrt.shape):
        if q_sqrt.ndim == 3 and idx[2] > idx[1]:
            assert g["q_sqrt"][idx] == 0.0
            continue
        _close(g["q_sqrt"][idx], _fd_array(lambda v: f(qs=v), q_sqrt, idx, h), tol, ("q_sqrt", idx))
    return g


@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("q_diag", [False, True])
@pytest.mark.parametrize("C", [3, 5])
@pytest.mark.parametrize("num_data", [None, 40])
def test_svgp_multiclass_gradient_matches_finite_differences(whiten, q_diag, C, num_data):
    X, Y, Z, q_mu, q_sqrt = _data(C, q_diag=q_diag)
    _check_all(O.SquaredExponential(1.3, 1.7) + O.White(0.05), X, Y, Z, q_mu, q_sqrt, whiten, num_data)


@pytest.mark.parametrize("kind", ["constant", "linear"])
def test_svgp_multiclass_mean_function_gradient_matches_finite_differences(kind):
    C = 3
    X, Y, Z, q_mu, q_sqrt = _data(C)
    rng = np.random.default_rng(5)
    if kind == "constant":
        mf = O.ConstantMean(0.1 * np.arange(1, C + 1))
        params = {"c": mf.c}
    else:
        mf = O.LinearMean(0.2 * rng.standard_normal((X.shape[1], C)), 0.1 * np.arange(1, C + 1))
        params = {"A": mf.A, "b": mf.b}
    kernel = O.SquaredExponential(1.3, 1.7) + O.Linear(0.2)
    g = _check_all(kernel, X, Y, Z, q_mu, q_sqrt, True, 30, mean_function=mf)
    lik = MO.MultiClass(C, 0.05)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = MO.svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, lik, num_data=30, mean_function=mf)
            arr[idx] -= 2 * h
            fm = MO.svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, lik, num_data=30, mean_function=mf)
            arr[idx] += h
            _close(g["mean"][pname][idx], (fp - fm) / (2 * h), 1e-6, (pname, idx))


# ---- the descriptor ---------------------------------------------------------------------------------------------
def _mc(C, eps=1e-3, n_gh=20):
    return _lib.LikDesc(_lib.LIK_MULTICLASS, n_gh, 0.0, 0.0, 0.0, 0.0, eps, C)


def test_svgp_grad_entry_point_checks_the_multiclass_descriptor():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    # _call passes P = 1
    for bad, word in [(_mc(1), "classes"), (_mc(_lib.LIK_MAX_CLASSES + 1), "classes"), (_mc(3, 0.0), "epsilon"),
                      (_mc(3, 1.0), "epsilon"), (_mc(3, float("nan")), "epsilon"), (_mc(3), "one latent per class"),
                      (_mc(3, n_gh=10), "Gauss-Hermite")]:
        st, msg = _call(nodes, n, dims, ard, 3, bad)
        assert st == -1 and word in msg, msg
    lib = _lib.load()
    mc = _mc(4)
    gauss = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1)
    assert lib.gpk_svgp_elbo_grad_ws(1000, 64, 4, ctypes.byref(mc), _lib.GPK_F64) > \
        lib.gpk_svgp_elbo_grad_ws(1000, 64, 4, ctypes.byref(gauss), _lib.GPK_F64)


def test_the_bound_admits_the_reference_tests_hundred_classes():
    assert _lib.LIK_MAX_CLASSES >= 100


def test_descriptor_mirror_has_the_c_layout(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc") or shutil.which("g++")
    assert cc, "a host C compiler (the one nvcc drives) is needed"
    src = tmp_path / "size.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "gpk.h"\n'
                   'int main(void) { printf("%zu %zu %zu %d\\n", sizeof(gpk_lik), offsetof(gpk_lik, epsilon), '
                   'offsetof(gpk_lik, num_classes), GPK_LIK_MAX_CLASSES); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, off_eps, off_c, bound = (int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True,
                                                                  check=True).stdout.split())
    assert ctypes.sizeof(_lib.LikDesc) == size
    assert _lib.LikDesc.epsilon.offset == off_eps and _lib.LikDesc.num_classes.offset == off_c
    assert _lib.LIK_MAX_CLASSES == bound


# ---- the Python classes ----------------------------------------------------------------------------------------
def test_sigmoid_round_trip_and_derivative():
    t = Sigmoid()
    x = np.array([-30.0, -3.0, -0.2, 0.0, 0.7, 4.0, 12.0])  # past 12, 1 - sigmoid(x) keeps too few digits
    np.testing.assert_allclose(t.inverse(t.forward(x)), x, rtol=1e-9, atol=1e-12)
    h = 1e-6
    np.testing.assert_allclose(t.forward_grad(x), (t.forward(x + h) - t.forward(x - h)) / (2 * h), rtol=1e-7,
                               atol=1e-10)
    assert t.forward(0.0) == 0.5
    for bad in (0.0, 1.0, -0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="Sigmoid"):
            gpf.base.Parameter(bad, transform=Sigmoid())
    p = gpf.base.Parameter(0.25, transform=Sigmoid())
    np.testing.assert_allclose(p.unconstrained_variable, np.log(0.25 / 0.75))


def test_multiclass_and_robustmax_constructors():
    L = gpf.likelihoods
    lik = L.MultiClass(7)
    assert lik.num_classes == 7 and lik.num_gauss_hermite_points == 20
    assert isinstance(lik.invlink, L.RobustMax) and lik.invlink.num_classes == 7
    eps = lik.invlink.epsilon
    assert float(eps) == pytest.approx(1e-3) and not eps.trainable and isinstance(eps.transform, Sigmoid)
    assert (eps.prior.concentration1, eps.prior.concentration0) == (0.2, 5.0)
    assert [id(p) for p in lik.parameters] == [id(eps)] and lik.trainable_parameters == ()
    d = lik._lik_desc()
    assert (d.type, d.n_gh, d.num_classes) == (_lib.LIK_MULTICLASS, 20, 7) and d.epsilon == pytest.approx(1e-3)
    with pytest.raises(NotImplementedError, match="RobustMax"):
        L.MultiClass(3, invlink=L.inv_probit)
    with pytest.raises(ValueError, match="classes"):
        L.MultiClass(3, invlink=L.RobustMax(4))
    with pytest.raises(ValueError, match="Sigmoid"):
        L.RobustMax(3, epsilon=1.0)
