"""The SGPR gradient oracle (tests/sgpr_grad_oracle.py::sgpr_elbo_and_grad_expr) against central finite differences of
the ELBO oracle (oracle/gp_oracle.py::sgpr_elbo) for every hyperparameter, the noise, every entry of Z and the mean
function parameters, and the argument checks of gpk_sgpr_elbo_grad.  No device needed."""
import copy
import ctypes

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import sgpr_grad_oracle as S

RNG_SEED = 20261015


def _data(P, N=30, M=7, D=4):
    rng = np.random.default_rng(RNG_SEED + P)
    X = rng.standard_normal((N, D))
    Y = np.sin(X[:, :P] @ np.ones((P, P))) + 0.1 * rng.standard_normal((N, P))
    Z = 1.2 * rng.standard_normal((M, D)) + 0.1   # away from X: no coincident pairs in the finite differences
    return X, Y, Z


# name -> (oracle expression, finite-difference tolerance, step).  Matern12 sees the rounding noise of the reference's
# norm-expansion distance on the Kuu diagonal under its square root, and so does Exponential (see
# tests/test_oracle_grad_expr.py): a longer step keeps that noise below the tolerance.
def _cases():
    ell4 = np.array([1.1, 1.9, 0.7, 2.5])
    shared = O.Matern32(0.9, ell4)
    return {
        "rbf_plus_white": (O.SquaredExponential(1.3, 1.7) + O.White(0.05), 5e-6, 1e-5),
        "c5": ((O.SquaredExponential(1.1, 2.1) + O.Matern32(1.0, 4.0)) * O.Linear(0.5), 5e-6, 1e-5),
        "rq_ard": (O.RationalQuadratic(1.2, ell4, alpha=2.5), 5e-6, 1e-5),
        "polynomial_ard_plus_white": (O.Polynomial(degree=2.0, variance=np.array([0.2, 0.1, 0.3, 0.25]), offset=1.3)
                                      + O.White(0.1), 5e-6, 1e-5),
        "linear_ard_plus_matern12": (O.Linear(np.array([0.3, 0.5, 0.9, 0.2])) + O.Matern12(0.5, 1.5), 2e-3, 1e-3),
        "constant_times_matern52": (O.Constant(1.7) * O.Matern52(0.9, 1.8), 5e-6, 1e-5),
        "additive_active_dims": (O.SquaredExponential(1.0, 0.9, active_dims=[0]) + O.Matern52(0.7, 1.3, active_dims=[1])
                                 + O.Exponential(0.4, np.array([1.2, 0.8]), active_dims=[2, 3])
                                 + O.Linear(np.array([0.3, 0.4]), active_dims=[2, 3]), 2e-3, 1e-3),
        "k_plus_k": (shared + shared, 5e-6, 1e-5),
    }


CASES = _cases()


def _perturb(kernel, leaf, name, idx, h):
    k2 = copy.deepcopy(kernel)
    target = S.leaves(k2)[leaf]   # a shared leaf (k + k) stays one object after deepcopy: both occurrences move
    v = np.array(getattr(target, name), dtype=np.float64)
    if v.ndim == 0:
        v = v + h
    else:
        v = v.copy()
        v[idx] += h
    setattr(target, name, v if v.ndim else float(v))
    return k2


def _close(got, fd, tol, what):
    assert abs(got - fd) <= tol * max(1.0, abs(fd)), (what, got, fd)


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("P", [1, 2])
def test_sgpr_gradient_matches_finite_differences(name, P):
    kernel, tol, h = CASES[name]
    X, Y, Z = _data(P)
    s2 = 0.2
    elbo, g = S.sgpr_elbo_and_grad_expr(X, Y, kernel, Z, s2)
    assert abs(elbo - O.sgpr_elbo(X, Y, kernel, Z, s2)) < 1e-12 * max(1.0, abs(elbo))
    f = lambda k=kernel, Zv=Z, s=s2: O.sgpr_elbo(X, Y, k, Zv, s)  # noqa: E731
    lv = S.leaves(kernel)
    seen = set()
    for li, leaf in enumerate(lv):
        for pname in g["leaves"][li]:
            if (id(leaf), pname) in seen:
                continue
            seen.add((id(leaf), pname))
            total = sum(np.asarray(g["leaves"][lj][pname]) for lj, l2 in enumerate(lv) if l2 is leaf)
            for idx in np.ndindex(np.shape(total)):
                fd = (f(k=_perturb(kernel, li, pname, idx, h)) - f(k=_perturb(kernel, li, pname, idx, -h))) / (2 * h)
                _close(float(np.asarray(total)[idx]), fd, tol, (name, li, pname, idx))
    _close(g["noise_variance"], (f(s=s2 + h) - f(s=s2 - h)) / (2 * h), tol, "noise")
    for idx in np.ndindex(Z.shape):
        Zp, Zm = Z.copy(), Z.copy()
        Zp[idx] += h
        Zm[idx] -= h
        _close(g["Z"][idx], (f(Zv=Zp) - f(Zv=Zm)) / (2 * h), tol, ("Z", idx))


@pytest.mark.parametrize("P", [1, 2])
@pytest.mark.parametrize("kind", ["constant_scalar", "constant_per_output", "linear", "linear_one_column"])
def test_sgpr_mean_function_gradient_matches_finite_differences(P, kind):
    X, Y, Z = _data(P)
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
    _, g = S.sgpr_elbo_and_grad_expr(X, Y, kernel, Z, 0.2, mean_function=mf)
    h = 1e-6
    for pname, arr in params.items():
        assert g["mean"][pname].shape == arr.shape
        for idx in np.ndindex(arr.shape):
            arr[idx] += h
            fp = O.sgpr_elbo(X, Y, kernel, Z, 0.2, mean_function=mf)
            arr[idx] -= 2 * h
            fm = O.sgpr_elbo(X, Y, kernel, Z, 0.2, mean_function=mf)
            arr[idx] += h
            _close(g["mean"][pname][idx], (fp - fm) / (2 * h), 1e-6, (pname, idx))


# ---- argument checks: status -1 and a readable error, before anything reaches a device ------------------------------
def _call(nodes, n, dims, ard, D, dtype=_lib.GPK_F64, n_out=64, dZ=True):
    lib = _lib.load()
    fake = ctypes.c_void_p(256)  # never dereferenced: every check below runs on the host before the first launch
    st = lib.gpk_sgpr_elbo_grad(nodes, n, dims, ard, fake, 100, D, D, fake, 1, fake, 10, D, 0.1, 1e-6, dtype, fake,
                                n_out, fake if dZ else None, fake, None)
    return st, lib.gpk_last_error().decode()


def test_sgpr_grad_entry_point_rejects_bad_arguments():
    K = gpf.kernels
    nodes, n, dims, ard = gpf.kernels.compile_kernel(K.SquaredExponential() + K.White(), 3)
    st, msg = _call(nodes, n, dims, ard, 3, dtype=_lib.GPK_F32)
    assert st == -1 and "float64" in msg
    st, msg = _call(nodes, n, dims, ard, 3, n_out=11)   # 9 + 3 slots needed
    assert st == -1 and "n_out" in msg and "12" in msg
    st, msg = _call(nodes, n, dims, ard, 3, dZ=False)
    assert st == -1 and "dZ" in msg
    # 33 staged columns: two groups (different active dims) of 17 and 16
    k = K.SquaredExponential(active_dims=list(range(17))) + K.Matern52(active_dims=list(range(17, 33)))
    nodes, n, dims, ard = gpf.kernels.compile_kernel(k, 33)
    st, msg = _call(nodes, n, dims, ard, 33)
    assert st == -1 and "33" in msg and "32" in msg and "sgpr_elbo_grad" in msg
    # the workspace and the offset of dF/dm are host arithmetic
    lib = _lib.load()
    assert lib.gpk_sgpr_elbo_grad_ws(1000, 64, 2, _lib.GPK_F64) > lib.gpk_sgpr_elbo_ws(1000, 64, 2, _lib.GPK_F64)
    off = lib.gpk_sgpr_elbo_grad_dm(1000, 64, 2, _lib.GPK_F64)
    assert off % 256 == 0 and off + 8 * 1000 * 2 <= lib.gpk_sgpr_elbo_grad_ws(1000, 64, 2, _lib.GPK_F64)

