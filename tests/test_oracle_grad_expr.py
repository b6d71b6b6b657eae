"""The expression gradient oracle (tests/grad_expr_oracle.py::gpr_lml_and_grad_expr) against central finite differences
of the LML oracle, the Python slot map against gpk_gpr_lml_grad_slots, and the argument checks of the new entry points.
No device needed."""
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import grad_check as GC
from tests import grad_expr_oracle as G
from tests import kernel_grad_oracle as KG

RNG_SEED = 20240611


def _data(P, N=40, D=4):
    rng = np.random.default_rng(RNG_SEED + P)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :P] @ np.ones((P, P))) + 0.1 * rng.standard_normal((N, P))
    return X, Y


# name -> (oracle expression, whether its finite differences are smooth: the sqrt-type kernels see the rounding noise of
# the reference's norm-expansion distance on the diagonal, see tests/test_oracle_grad.py)
def _cases():
    ell4 = np.array([1.1, 1.9, 0.7, 2.5])
    shared = O.SquaredExponential(variance=0.9, lengthscales=1.4)
    return {
        "rbf": (O.SquaredExponential(1.3, 1.7), True),
        "rbf_ard": (O.SquaredExponential(1.3, ell4), True),
        "matern12": (O.Matern12(0.8, 1.5), False),
        "matern32_ard": (O.Matern32(0.8, ell4), True),
        "matern52": (O.Matern52(1.1, 2.0), True),
        "exponential": (O.Exponential(0.7, 1.2), False),
        "rq": (O.RationalQuadratic(1.2, 1.6, alpha=0.8), True),
        "rq_ard": (O.RationalQuadratic(1.2, ell4, alpha=2.5), True),
        "linear": (O.Linear(0.6), True),
        "linear_ard": (O.Linear(np.array([0.3, 0.5, 0.9, 0.2])), True),
        "polynomial": (O.Polynomial(degree=2.0, variance=0.4, offset=0.7), True),
        "polynomial_ard": (O.Polynomial(degree=3.0, variance=np.array([0.2, 0.1, 0.3, 0.25]), offset=1.3), True),
        "rbf_plus_white": (O.SquaredExponential(1.3, 1.7) + O.White(0.05), True),
        "constant_times_matern52": (O.Constant(1.7) * O.Matern52(0.9, 1.8), True),
        "c5": ((O.SquaredExponential(1.1, 2.1) + O.Matern32(1.0, 4.0)) * O.Linear(0.5), True),
        "nested": (O.Product([O.Sum([O.SquaredExponential(1.0, 1.5, active_dims=[0, 1]), O.Constant(0.3)]),
                              O.Sum([O.Linear(0.4, active_dims=[2, 3]), O.White(0.1)]),
                              O.RationalQuadratic(0.9, 2.2, alpha=1.5)]), True),
        "additive_active_dims": (O.SquaredExponential(1.0, 0.9, active_dims=[0]) + O.Matern52(0.7, 1.3, active_dims=[1])
                                 + O.Linear(np.array([0.3, 0.4]), active_dims=[2, 3]), True),
        "shared_parameter": (shared + shared, True),
    }


CASES = _cases()
PARAMS = ("variance", "lengthscales", "alpha", "offset")


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("P", [1, 2])
def test_expression_gradient_matches_finite_differences(name, P):
    kernel, smooth = CASES[name]
    X, Y = _data(P)
    _check_fd(X, Y, kernel, smooth, name)


@pytest.mark.parametrize("name", list(GC.wide_cases()))
def test_wide_expression_gradient_matches_finite_differences(name):
    kernel, D = GC.wide_cases()[name]
    X, Y = _data(1, N=50, D=D)
    _check_fd(X, Y, kernel, True, name)


def _check_fd(X, Y, kernel, smooth, name):
    s2 = 0.2
    lml, g = G.gpr_lml_and_grad_expr(X, Y, kernel, s2)
    assert abs(lml - O.gpr_log_marginal_likelihood(X, Y, kernel, s2)) < 1e-9 * max(1.0, abs(lml))
    h = 1e-5
    tol = 5e-6 if smooth else 2e-3
    lv = KG.leaves(kernel)
    seen = set()
    for li, leaf in enumerate(lv):
        for pname, gval in g["leaves"][li].items():
            key = (id(leaf), pname)
            if key in seen:
                continue
            seen.add(key)
            # a shared leaf object: its gradient is the sum over its occurrences
            total = sum(np.asarray(g["leaves"][lj][pname]) for lj, l2 in enumerate(lv) if l2 is leaf)
            for idx in np.ndindex(np.shape(total)):
                fp = O.gpr_log_marginal_likelihood(X, Y, GC.perturb(kernel, li, pname, idx, h), s2)
                fm = O.gpr_log_marginal_likelihood(X, Y, GC.perturb(kernel, li, pname, idx, -h), s2)
                fd = (fp - fm) / (2 * h)
                got = float(np.asarray(total)[idx]) if np.ndim(total) else float(total)
                assert abs(got - fd) <= tol * max(1.0, abs(fd)), (name, li, pname, idx, got, fd)
    fd_n = (O.gpr_log_marginal_likelihood(X, Y, kernel, s2 + h) - O.gpr_log_marginal_likelihood(X, Y, kernel, s2 - h)) / (2 * h)
    assert abs(g["noise_variance"] - fd_n) <= tol * max(1.0, abs(fd_n))


@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("kind", ["constant_scalar", "constant_per_output", "linear", "linear_one_column"])
def test_mean_function_gradient_matches_finite_differences(P, kind):
    X, Y = _data(P)
    D = X.shape[1]
    kernel = O.SquaredExponential(1.3, 1.7) + O.Linear(0.2)
    rng = np.random.default_rng(5)
    if kind == "constant_scalar":
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
    _, g = G.gpr_lml_and_grad_expr(X, Y, kernel, 0.2, mean_function=mf)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = O.gpr_log_marginal_likelihood(X, Y, kernel, 0.2, mean_function=mf)
            arr[idx] -= 2 * h
            fm = O.gpr_log_marginal_likelihood(X, Y, kernel, 0.2, mean_function=mf)
            arr[idx] += h
            fd = (fp - fm) / (2 * h)
            assert abs(g["mean"][pname][idx] - fd) <= 1e-6 * max(1.0, abs(fd)), (pname, idx, g["mean"][pname][idx], fd)


# ---- the Python slot map against the library's --------------------------------------------------------------------
def _product_cases(D=4):
    K = gpf.kernels
    ell = np.array([1.1, 1.9, 0.7, 2.5])
    shared = K.SquaredExponential(variance=0.9, lengthscales=1.4)
    rq = K.RationalQuadratic(variance=1.2, lengthscales=ell, alpha=2.5)
    return {
        "rbf_plus_white": K.SquaredExponential() + K.White(variance=0.05),
        "c5": (K.SquaredExponential(lengthscales=2.0) + K.Matern32(lengthscales=4.0)) * K.Linear(variance=0.5),
        "rq_ard": rq,
        "polynomial_ard": K.Polynomial(degree=3.0, variance=np.array([0.2, 0.1, 0.3, 0.25]), offset=1.3),
        "linear_ard": K.Linear(variance=np.array([0.3, 0.5, 0.9, 0.2])),
        "constant_times_matern52": K.Constant(variance=1.7) * K.Matern52(),
        "additive_active_dims": (K.SquaredExponential(active_dims=[0]) + K.Matern52(active_dims=[1])
                                 + K.Linear(variance=np.array([0.3, 0.4]), active_dims=[2, 3])),
        "shared_parameter": shared + shared,
        "nested": (K.SquaredExponential(active_dims=[0, 1]) + K.Constant()) * (K.Linear(active_dims=[2, 3]) + K.White())
                  * K.RationalQuadratic(lengthscales=ell),
        "rbf_ard_plus_matern_ard_same_values": K.SquaredExponential(lengthscales=ell) + K.Matern32(lengthscales=ell),
    }


@pytest.mark.parametrize("name", list(_product_cases()))
def test_python_slot_map_agrees_with_library(name):
    kern = _product_cases()[name]
    D = 4
    lib = _lib.load()
    nodes, n, dims, ard = gpf.kernels.compile_kernel(kern, D)
    n_slots = lib.gpk_gpr_lml_grad_slots(nodes, n, dims, ard, D)
    slots = gpf.kernels.gradient_slots(kern, D)
    assert n_slots == sum(c for _, _, c in slots)
    pos = 0
    for p, off, cnt in slots:
        assert off == pos and cnt == p.numpy().size
        pos += cnt


def test_slot_map_names_materialised_kernels():
    K = gpf.kernels
    for kern, cls in [(K.Cosine(), "Cosine"), (K.Periodic(K.SquaredExponential()) + K.White(), "Periodic"),
                      (K.ArcCosine() * K.Linear(), "ArcCosine"), (K.Coregion(output_dim=2, rank=1, active_dims=[0]), "Coregion"),
                      (K.ChangePoints([K.SquaredExponential(), K.Matern52()], locations=[0.0]), "ChangePoints")]:
        with pytest.raises(NotImplementedError, match=cls):
            gpf.kernels.gradient_slots(kern, 2)


# ---- argument checks: status -1 and a readable error, before anything reaches a device ------------------------------
def _call_expr(nodes, n, dims, ard, D, dtype=_lib.GPK_F64, n_out=64):
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every check below runs on the host before the first launch
    st = lib.gpk_gpr_lml_grad_expr(nodes, n, dims, ard, fake, 100, D, D, fake, 1, 0.1, dtype, fake, n_out, fake, None)
    return st, lib.gpk_last_error().decode()


def test_expr_entry_point_rejects_bad_arguments():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    st, msg = _call_expr(nodes, n, dims, ard, 3, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = _call_expr(nodes, n, dims, ard, 3, n_out=7)   # 5 + 3 slots needed
    assert st == -1 and "n_out" in msg and "8" in msg
    # an op without a fused record (the materialised kernels have none)
    bad = (_lib.KNode * 1)()
    bad[0].op = 12
    st, msg = _call_expr(bad, 1, dims, ard, 3)
    assert st == -1 and "op 12" in msg
    assert _lib.load().gpk_gpr_lml_grad_slots(bad, 1, dims, ard, 3) == -1
    # 33 staged columns: two groups (different active dims) of 17 and 16
    k = K.SquaredExponential(active_dims=list(range(17))) + K.Matern52(active_dims=list(range(17, 33)))
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 33)
    st, msg = _call_expr(nodes, n, dims, ard, 33)
    assert st == -1 and "33" in msg and "32" in msg
    assert _lib.load().gpk_gpr_lml_grad_slots(nodes, n, dims, ard, 33) == -1
    # 32 columns (C5's shape) are accepted by the slot query
    k = (K.SquaredExponential() + K.Matern32()) * K.Linear()
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 32)
    assert _lib.load().gpk_gpr_lml_grad_slots(nodes, n, dims, ard, 32) == 5
    # more than 32 per-dimension slots: two ARD leaves of 20 dims on one group
    ell = np.linspace(1.0, 2.0, 20)
    k = K.SquaredExponential(lengthscales=ell) + K.Matern32(lengthscales=ell)
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 20)
    assert _lib.load().gpk_gpr_lml_grad_slots(nodes, n, dims, ard, 20) == -1
    assert "per-dimension" in _lib.load().gpk_last_error().decode()
