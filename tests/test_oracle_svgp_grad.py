"""The SVGP gradient oracle (tests/svgp_grad_oracle.py::svgp_elbo_and_grad) with a Gaussian likelihood against central
finite differences of the ELBO oracle (oracle/gp_oracle.py::svgp_elbo) for every hyperparameter, the noise, every entry
of Z, q_mu and the lower q_sqrt, and the mean function parameters, under both whiten and both q_diag settings; the
envelope identity with the SGPR oracle at the optimal q(u); and the argument checks of gpk_svgp_elbo_grad.  No device needed."""
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import kernel_grad_oracle as KG
from tests import lik_oracle as LO
from tests import sgpr_grad_oracle as SG
from tests import svgp_grad_oracle as S

RNG_SEED = 20261016


def _data(P, B=9, M=5, D=3, q_diag=False):
    rng = np.random.default_rng(RNG_SEED + P + 10 * q_diag)
    X = rng.standard_normal((B, D))
    Y = np.sin(X[:, :1] @ np.ones((1, P))) + 0.1 * rng.standard_normal((B, P))
    Z = 1.2 * rng.standard_normal((M, D)) + 0.1   # away from X: no coincident pairs in the finite differences
    q_mu = 0.5 * rng.standard_normal((M, P))
    if q_diag:
        q_sqrt = 0.3 + 0.5 * rng.random((M, P))
    else:
        q_sqrt = np.stack([np.tril(0.2 * rng.standard_normal((M, M)), -1) + np.diag(0.4 + 0.5 * rng.random(M))
                           for _ in range(P)])
        q_sqrt += np.triu(rng.standard_normal((M, M)), 1)[None]   # band_part drops the strict upper part
    return X, Y, Z, q_mu, q_sqrt


def _cases():
    ell3 = np.array([1.1, 1.9, 0.7])
    return {
        "rbf_plus_white": (O.SquaredExponential(1.3, 1.7) + O.White(0.05), 5e-6, 1e-5),
        "c5": ((O.SquaredExponential(1.1, 2.1) + O.Matern32(1.0, 4.0)) * O.Linear(0.5), 5e-6, 1e-5),
        "rq_ard": (O.RationalQuadratic(1.2, ell3, alpha=2.5), 5e-6, 1e-5),
        "polynomial_ard": (O.Polynomial(degree=2.0, variance=np.array([0.2, 0.1, 0.3]), offset=1.3), 5e-6, 1e-5),
        "constant_times_matern52": (O.Constant(1.7) * O.Matern52(0.9, 1.8), 5e-6, 1e-5),
    }


CASES = _cases()


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("q_diag", [False, True])
@pytest.mark.parametrize("num_data", [None, 40])
def test_svgp_gradient_matches_finite_differences(name, whiten, q_diag, num_data):
    P = 2
    kernel, tol, h = CASES[name]
    X, Y, Z, q_mu, q_sqrt = _data(P, q_diag=q_diag)
    s2 = 0.3

    def f(k=kernel, Zv=Z, s=s2, qm=q_mu, qs=q_sqrt):
        return O.svgp_elbo(X, Y, Zv, k, qm, qs, s, whiten=whiten, num_data=num_data)

    elbo, g = S.svgp_elbo_and_grad(X, Y, [kernel], [Z], q_mu, q_sqrt, LO.Gaussian(s2), whiten=whiten,
                                   num_data=num_data)
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    lv = KG.leaves(kernel)
    for li, leaf in enumerate(lv):
        for pname, got in g["leaves"][li].items():
            for idx in np.ndindex(np.shape(got)):
                fd = (f(k=GC.perturb(kernel, li, pname, idx, h))
                      - f(k=GC.perturb(kernel, li, pname, idx, -h))) / (2 * h)
                GC.close(float(np.asarray(got)[idx]), fd, tol, (name, li, pname, idx))
    GC.close(g["lik"], (f(s=s2 + h) - f(s=s2 - h)) / (2 * h), tol, "noise")
    for idx in np.ndindex(Z.shape):
        GC.close(g["Z"][idx], GC.fd_array(lambda v: f(Zv=v), Z, idx, h), tol, ("Z", idx))
    for idx in np.ndindex(q_mu.shape):
        GC.close(g["q_mu"][idx], GC.fd_array(lambda v: f(qm=v), q_mu, idx, h), tol, ("q_mu", idx))
    assert g["q_sqrt"].shape == q_sqrt.shape
    for idx in np.ndindex(q_sqrt.shape):
        if not q_diag and idx[2] > idx[1]:
            assert g["q_sqrt"][idx] == 0.0
            continue
        GC.close(g["q_sqrt"][idx], GC.fd_array(lambda v: f(qs=v), q_sqrt, idx, h), tol, ("q_sqrt", idx))


@pytest.mark.parametrize("whiten", [True, False])
@pytest.mark.parametrize("kind", ["constant_per_output", "linear", "linear_one_column"])
def test_svgp_mean_function_gradient_matches_finite_differences(whiten, kind):
    P = 2
    X, Y, Z, q_mu, q_sqrt = _data(P)
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
    _, g = S.svgp_elbo_and_grad(X, Y, [kernel], [Z], q_mu, q_sqrt, LO.Gaussian(0.2), whiten=whiten, num_data=30,
                                mean_function=mf)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = O.svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, 0.2, whiten=whiten, num_data=30, mean_function=mf)
            arr[idx] -= 2 * h
            fm = O.svgp_elbo(X, Y, Z, kernel, q_mu, q_sqrt, 0.2, whiten=whiten, num_data=30, mean_function=mf)
            arr[idx] += h
            GC.close(g["mean"][pname][idx], (fp - fm) / (2 * h), 1e-6, (pname, idx))


@pytest.mark.parametrize("whiten", [True, False])
def test_envelope_identity_with_sgpr_at_the_optimal_q(whiten):
    """At q* with num_data = N on the full data, the SVGP ELBO equals the SGPR bound and touches it from below, so the
    kernel, noise and Z gradients agree and dF/dq is about 0."""
    P = 2
    rng = np.random.default_rng(7)
    N, M, D = 25, 6, 3
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1] @ np.ones((1, P))) + 0.1 * rng.standard_normal((N, P))
    Z = 1.1 * rng.standard_normal((M, D))
    kernel = O.SquaredExponential(1.3, 1.7) + O.Linear(0.3)
    s2 = 0.25
    q_mu, q_sqrt = SG.optimal_q(X, Y, kernel, Z, s2, whiten)
    e_sv, gs = S.svgp_elbo_and_grad(X, Y, [kernel], [Z], q_mu, q_sqrt, LO.Gaussian(s2), whiten=whiten, num_data=N)
    e_sg, gg = SG.sgpr_elbo_and_grad_expr(X, Y, kernel, Z, s2)
    np.testing.assert_allclose(e_sv, e_sg, rtol=1e-9)
    np.testing.assert_allclose(gs["lik"], gg["noise_variance"], rtol=1e-7, atol=1e-8)
    np.testing.assert_allclose(gs["Z"], gg["Z"], rtol=1e-7, atol=1e-8)
    for a, b in zip(gs["leaves"], gg["leaves"]):
        for name in a:
            np.testing.assert_allclose(a[name], b[name], rtol=1e-7, atol=1e-8, err_msg=name)
    np.testing.assert_allclose(gs["q_mu"], 0.0, atol=1e-8)
    np.testing.assert_allclose(gs["q_sqrt"], 0.0, atol=1e-8)


# ---- argument checks: status -1 and a readable error, before anything reaches a device ------------------------------
def _call(nodes, n, dims, ard, D, dtype=_lib.GPK_F64, n_out=64, dZ=True, dq_mu=True, dq_sqrt=True):
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every check below runs on the host before the first launch
    gauss = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1)
    st = lib.gpk_svgp_elbo_grad(nodes, n, dims, ard, fake, 100, D, D, fake, None, 1, fake, 10, D, fake, fake, 0, 1,
                                ctypes.byref(gauss), 1.0, 1e-6, dtype, fake, n_out, fake if dZ else None,
                                fake if dq_mu else None, fake if dq_sqrt else None, fake, None)
    return st, lib.gpk_last_error().decode()


def test_svgp_grad_entry_point_rejects_bad_arguments_with_a_gaussian_descriptor():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    st, msg = _call(nodes, n, dims, ard, 3, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = _call(nodes, n, dims, ard, 3, n_out=7)   # 5 + 3 slots needed
    assert st == -1 and "n_out" in msg and "8" in msg
    for missing in ["dZ", "dq_mu", "dq_sqrt"]:
        st, msg = _call(nodes, n, dims, ard, 3, **{missing: False})
        assert st == -1 and missing in msg and "svgp_elbo_grad" in msg
    # 33 staged columns: two groups (different active dims) of 17 and 16
    k = K.SquaredExponential(active_dims=list(range(17))) + K.Matern52(active_dims=list(range(17, 33)))
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 33)
    st, msg = _call(nodes, n, dims, ard, 33)
    assert st == -1 and "33" in msg and "32" in msg and "svgp_elbo_grad" in msg
    # the workspace and the offset of dF/dm(X) are host arithmetic
    lib = _lib.load()
    gauss = ctypes.byref(_lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.1))
    ws = lib.gpk_svgp_elbo_grad_ws(1000, 64, 2, gauss, _lib.GPK_F64)
    assert ws > lib.gpk_svgp_elbo_ws(1000, 64, 2, _lib.GPK_F64)
    off = lib.gpk_svgp_elbo_grad_dm(1000, 64, 2, _lib.GPK_F64)
    assert off % 256 == 0 and off + 8 * 1000 * 2 <= ws
