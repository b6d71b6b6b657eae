"""The VGP gradient oracle (tests/vgp_grad_oracle.py::vgp_elbo_and_grad_expr) against central finite differences of the
ELBO oracle (oracle/gp_oracle.py::vgp_elbo) for every hyperparameter of the GPR / SVGP expression list, the noise, q_mu,
the lower q_sqrt and the mean function parameters, at P = 1 and P = 3; its identity with the whitened SVGP oracle at
Z = X and zero jitter; and the argument checks of gpk_vgp_elbo_grad.  No device needed."""
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import kernel_grad_oracle as KG
from tests import lik_oracle as LO
from tests import svgp_grad_oracle as SV
from tests import vgp_grad_oracle as V

RNG_SEED = 20261017
NAMES = ["rbf_plus_white", "c5", "rq", "rq_ard", "polynomial_ard", "linear_ard", "constant_times_matern52",
         "additive_active_dims", "k_plus_k"]
NON_SMOOTH = {"linear_ard", "additive_active_dims"}   # a Matern12 / Exponential leaf


def _data(P, N=9, D=4, seed=0):
    rng = np.random.default_rng(RNG_SEED + P + 100 * seed)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :1] @ np.ones((1, P))) + 0.1 * rng.standard_normal((N, P))
    q_mu = 0.5 * rng.standard_normal((N, P))
    q_sqrt = np.stack([np.tril(0.2 * rng.standard_normal((N, N)), -1) + np.diag(0.4 + 0.5 * rng.random(N))
                       for _ in range(P)])
    q_sqrt += np.triu(rng.standard_normal((N, N)), 1)[None]   # band_part drops the strict upper part
    return X, Y, q_mu, q_sqrt


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("P", [1, 3])
def test_vgp_gradient_matches_finite_differences(name, P):
    _, kernel = GC.case(name, 4)
    X, Y, q_mu, q_sqrt = _data(P)
    s2, tol, h = 0.3, 5e-6, 1e-5

    def f(k=kernel, s=s2, qm=q_mu, qs=q_sqrt):
        return O.vgp_elbo(X, Y, k, qm, qs, s)

    elbo, g = V.vgp_elbo_and_grad_expr(X, Y, kernel, q_mu, q_sqrt, s2)
    assert abs(elbo - f()) < 1e-12 * max(1.0, abs(elbo))
    # Matern12 / Exponential take sqrt(r2) of the oracle's rounded zero on the diagonal (about 1e-8): differences over
    # h = 1e-5 see that noise, so these leaves step by 1e-3 (truncation about 1e-5 relative)
    ktol, kh = (5e-5, 1e-3) if name in NON_SMOOTH else (tol, h)
    lv = KG.leaves(kernel)
    for li, leaf in enumerate(lv):
        for pname in g["leaves"][li]:
            if any(lj < li for lj, l2 in enumerate(lv) if l2 is leaf):
                continue
            # a shared leaf object (k + k) moves in every occurrence: its gradient is the sum over them
            total = sum(np.asarray(g["leaves"][lj][pname]) for lj, l2 in enumerate(lv) if l2 is leaf)
            for idx in np.ndindex(np.shape(total)):
                fd = (f(k=GC.perturb(kernel, li, pname, idx, kh))
                      - f(k=GC.perturb(kernel, li, pname, idx, -kh))) / (2 * kh)
                GC.close(float(np.asarray(total)[idx]), fd, ktol, (name, li, pname, idx))
    GC.close(g["noise_variance"], (f(s=s2 + h) - f(s=s2 - h)) / (2 * h), tol, "noise")
    for idx in np.ndindex(q_mu.shape):
        GC.close(g["q_mu"][idx], GC.fd_array(lambda v: f(qm=v), q_mu, idx, h), tol, ("q_mu", idx))
    assert g["q_sqrt"].shape == q_sqrt.shape
    for idx in np.ndindex(q_sqrt.shape):
        if idx[2] > idx[1]:
            assert g["q_sqrt"][idx] == 0.0
            assert GC.fd_array(lambda v: f(qs=v), q_sqrt, idx, h) == 0.0   # the strict upper part is never read
            continue
        GC.close(g["q_sqrt"][idx], GC.fd_array(lambda v: f(qs=v), q_sqrt, idx, h), tol, ("q_sqrt", idx))


@pytest.mark.parametrize("kind", ["constant", "constant_per_output", "linear", "linear_one_column"])
def test_vgp_mean_function_gradient_matches_finite_differences(kind):
    P = 2
    X, Y, q_mu, q_sqrt = _data(P, seed=1)
    D = X.shape[1]
    kernel = O.SquaredExponential(1.3, 1.7) + O.Linear(0.2)
    rng = np.random.default_rng(5)
    if kind == "constant":
        mf = O.ConstantMean(np.array([0.3]))
        params = {"c": mf.c}
    elif kind == "constant_per_output":
        mf = O.ConstantMean(0.1 * np.arange(1, P + 1))
        params = {"c": mf.c}
    elif kind == "linear":
        mf = O.LinearMean(0.2 * rng.standard_normal((D, P)), 0.1 * np.arange(1, P + 1))
        params = {"A": mf.A, "b": mf.b}
    else:
        mf = O.LinearMean(0.2 * rng.standard_normal((D, 1)), np.array([0.4]))
        params = {"A": mf.A, "b": mf.b}
    _, g = V.vgp_elbo_and_grad_expr(X, Y, kernel, q_mu, q_sqrt, 0.2, mean_function=mf)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = O.vgp_elbo(X, Y, kernel, q_mu, q_sqrt, 0.2, mean_function=mf)
            arr[idx] -= 2 * h
            fm = O.vgp_elbo(X, Y, kernel, q_mu, q_sqrt, 0.2, mean_function=mf)
            arr[idx] += h
            GC.close(g["mean"][pname][idx], (fp - fm) / (2 * h), 1e-6, (pname, idx))


@pytest.mark.parametrize("P", [1, 3])
def test_vgp_equals_whitened_svgp_at_z_equal_x_without_jitter(P):
    """With zero jitter, Z = X and num_data = N, the whitened SVGP ELBO is the VGP ELBO as a function of the kernel
    parameters, the noise and q (A = L^-1 K = L^T, Kdiag - diag(A^T A) = 0), so every shared gradient agrees."""
    X, Y, q_mu, q_sqrt = _data(P, N=7, D=3, seed=2)
    kernel = O.SquaredExponential(1.3, 1.2) + O.Linear(0.3)
    s2 = 0.25
    e_v, gv = V.vgp_elbo_and_grad_expr(X, Y, kernel, q_mu, q_sqrt, s2, jitter=0.0)
    e_s, gs = SV.svgp_elbo_and_grad(X, Y, [kernel], [X], q_mu, q_sqrt, LO.Gaussian(s2), whiten=True,
                                    num_data=X.shape[0], jitter=0.0)
    np.testing.assert_allclose(e_v, e_s, rtol=1e-10)
    np.testing.assert_allclose(gv["noise_variance"], gs["lik"], rtol=1e-8)
    np.testing.assert_allclose(gv["q_mu"], gs["q_mu"], rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(gv["q_sqrt"], gs["q_sqrt"], rtol=1e-8, atol=1e-10)
    for a, b in zip(gv["leaves"], gs["leaves"]):
        for name in a:
            np.testing.assert_allclose(a[name], b[name], rtol=1e-7, atol=1e-9, err_msg=name)


# ---- argument checks: status -1 and a readable error, before anything reaches a device ------------------------------
def _call(nodes, n, dims, ard, D, N=100, dtype=_lib.GPK_F64, n_out=64, dq_mu=True, dq_sqrt=True):
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every check below runs on the host before the first launch
    st = lib.gpk_vgp_elbo_grad(nodes, n, dims, ard, fake, N, D, D, fake, 1, fake, fake, 0.1, 1e-6, dtype, fake, n_out,
                               fake if dq_mu else None, fake if dq_sqrt else None, fake, None)
    return st, lib.gpk_last_error().decode()


def test_vgp_grad_entry_point_rejects_bad_arguments():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    st, msg = _call(nodes, n, dims, ard, 3, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = _call(nodes, n, dims, ard, 3, n_out=7)   # 5 + 3 slots needed
    assert st == -1 and "n_out" in msg and "8" in msg
    for missing in ["dq_mu", "dq_sqrt"]:
        st, msg = _call(nodes, n, dims, ard, 3, **{missing: False})
        assert st == -1 and missing in msg and "vgp_elbo_grad" in msg
    # 33 staged columns: two groups (different active dims) of 17 and 16
    k = K.SquaredExponential(active_dims=list(range(17))) + K.Matern52(active_dims=list(range(17, 33)))
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 33)
    st, msg = _call(nodes, n, dims, ard, 33)
    assert st == -1 and "33" in msg and "32" in msg and "vgp_elbo_grad" in msg
    # a very wide X on very few points outgrows the square pass's scratch
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential(active_dims=[0]), 500)
    st, msg = _call(nodes, n, dims, ard, 500, N=2)
    assert st == -1 and "500 columns" in msg
    # the workspace and the offset of dF/dm(X) are host arithmetic
    lib = _lib.load()
    ws = lib.gpk_vgp_elbo_grad_ws(1000, 2, _lib.GPK_F64)
    assert ws > 6 * 8 * 1000 * 1000
    off = lib.gpk_vgp_elbo_grad_dm(1000, 2, _lib.GPK_F64)
    assert off % 256 == 0 and off + 8 * 1000 * 2 <= ws
