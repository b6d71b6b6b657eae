"""CPU self-checks of tests/kbuild_bounds.py: the per-element intervals must hold for the reference's own norm-expansion
formulation (oracle square_distance, in fp64 and fp32) and must not be loose; the fast path's x emulation must be
the rounding chain it claims to be."""
from fractions import Fraction

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import kbuild_bounds as B

ORACLE = {_lib.K_RBF: O.SquaredExponential, _lib.K_MATERN12: O.Matern12, _lib.K_MATERN32: O.Matern32,
          _lib.K_MATERN52: O.Matern52, _lib.K_EXPONENTIAL: O.Exponential}


def inputs(D, dtype, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((300, D)) + 1.5
    X[5] = X[4]
    X[7] = X[6] + 1e-6 * rng.standard_normal(D)
    X2 = rng.standard_normal((170, D)) + 1.0
    return X.astype(dtype), X2.astype(dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("D", [1, 8, 9, 17, 64])
def test_x_bound_holds_for_oracle_square_distance(D, dtype):
    """The oracle's norm expansion (gpflow/utilities/ops.py) on inputs scaled by 1/lengthscale lies within Bx of the
    direct-difference reference, and its worst error reaches a meaningful fraction of the bound."""
    X, X2 = inputs(D, dtype, D)
    ell = np.sqrt(D) * (0.4 + np.random.default_rng(1).random(D))
    worst = 0.0
    for Xb in (X2, None):
        Xs, Xbs = (X / ell.astype(dtype)), (None if Xb is None else Xb / ell.astype(dtype))
        got = O.square_distance(Xs, Xbs).astype(np.float64)
        r2, na, nb = B.r2_ref(X.astype(np.float64) / ell, (X if Xb is None else Xb).astype(np.float64) / ell)
        bx = B.gamma(D, dtype) * (na[:, None] + nb[None, :])
        err = np.abs(got - r2)
        assert np.all(err <= bx), float((err / bx).max())
        worst = max(worst, float((err / bx).max()))
    assert worst > 1e-3, worst


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("op", B.STATIONARY, ids=[B.NAMES[t] for t in B.STATIONARY])
@pytest.mark.parametrize("D", [1, 9, 33])
def test_oracle_kernel_lies_in_interval(op, D, dtype):
    """The oracle's K (its own exp / sqrt on the norm-expansion distance) lies in the helper's interval, built from the
    compiled kernel as the device tests build it."""
    X, X2 = inputs(D, dtype, 100 + D)
    ell = np.sqrt(D) * 0.7
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        kp = getattr(gpf.kernels, "SquaredExponential" if op == _lib.K_RBF else ORACLE[op].__name__)(
            variance=1.3, lengthscales=ell)
    desc = gpf.kernels.compile_kernel(kp, D)
    ko = ORACLE[op](variance=desc[0][0].variance, lengthscales=desc[0][0].lengthscale)
    for Xb in (X2, None):
        got = ko(X, Xb).astype(np.float64)
        cen, lo, hi = B.expr_interval(desc, X, Xb, dtype=dtype)
        assert np.all((got >= lo) & (got <= hi)), float(B.ratio(got, cen, lo, hi).max())


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
def test_composed_interval_holds_for_oracle(dtype):
    """Sum / Product of ARD stationary and Linear leaves over several groups: the oracle lies in the interval."""
    rng = np.random.default_rng(5)
    D = 50
    X, X2 = (rng.standard_normal((120, D)) + 0.5).astype(dtype), (rng.standard_normal((90, D)) + 0.5).astype(dtype)
    l1, l2 = 5.0 * (0.5 + rng.random(40)), 5.0 * (0.5 + rng.random(36))
    exprs = []
    for mod in (gpf.kernels, O):
        with gpf.config.as_context(gpf.config.Config(float=dtype)):
            rbf = mod.SquaredExponential(variance=1.2, lengthscales=l1, active_dims=list(range(40)))
            lin = mod.Linear(variance=0.3, active_dims=list(range(40, 46)))
            m52 = mod.Matern52(variance=0.7, lengthscales=l2, active_dims=list(range(5, 41)))
            exprs.append(mod.Sum([mod.Product([rbf, lin]), m52]))
    desc = gpf.kernels.compile_kernel(exprs[0], D)
    for Xb in (X2, None):
        got = exprs[1](X, Xb).astype(np.float64)
        cen, lo, hi = B.expr_interval(desc, X, Xb, dtype=dtype)
        assert np.all((got >= lo) & (got <= hi)), float(B.ratio(got, cen, lo, hi).max())


def test_fast_x_emulation_is_the_rounding_chain():
    """fast_x reproduces fl(fl(fl(v w)^2) + fl(fl(t w)^2)) computed with exact rationals and one rounding per step."""
    rnd = lambda q: Fraction(float(q))  # noqa: E731  (float() of a Fraction rounds to nearest)
    for op, ell in [(_lib.K_MATERN52, 1.7), (_lib.K_RBF, 0.3), (_lib.K_EXPONENTIAL, 2.9)]:
        w = B.fast_weight(op, ell)
        assert w == np.sqrt(float(rnd(rnd(Fraction(1) / rnd(Fraction(ell) * Fraction(ell))) * Fraction(B.FOLD[op]))))
        v, t = np.array([0.1, 3.3, 1e-19, 17.0]), np.array([0.7, 0.0, 2.2e-3, 250.0])
        x = B.fast_x(v, t, w, np.float64)
        for i, vi in enumerate(v):
            for j, tj in enumerate(t):
                a, b = rnd(Fraction(vi) * Fraction(w)), rnd(Fraction(tj) * Fraction(w))
                assert x[i, j] == float(rnd(a * a) + rnd(b * b))


def test_function_bars_cover_the_cpu_model():
    """The fp64 fast-path bars are built on the CPU model's bounds; the model's exp times a premultiplied table entry
    stays inside them."""
    from tests.test_fast_math_model import fast_exp_neg

    u = np.linspace(0, 700, 200001)
    var = 1.3
    tab_var = B.k_of_x(_lib.K_RBF, u, var)
    got = fast_exp_neg(u) * var
    rel = np.abs(got - np.asarray(tab_var, np.float64)) / np.asarray(tab_var, np.float64)
    a, b = B.fast_bar(_lib.K_RBF, np.float64)
    assert rel.max() <= a * B.U64
    for op in B.STATIONARY:
        assert B.fn_bar(op, np.float64) >= B.fast_bar(op, np.float64)
        assert B.fn_bar(op, np.float32)[0] >= B.generic_bar(op, np.float32)[0]
