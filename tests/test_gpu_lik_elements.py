"""The likelihood kernels of csrc/lik.cu element by element, against the exact oracle and the per-element bars of
tests/lik_bounds.py (their soundness and sharpness are shown on the CPU in tests/test_lik_bounds.py).

The C ABI is called directly.  Every input, output and workspace is a view into a NaN-filled buffer with GUARD elements
on both sides, and the guards must still be NaN afterwards: a padding lane writing R[n P + c] with c >= C, or a
grid-stride loop running past its end, shows there.
  a. gpk_lik_varexp_grad of the scalar likelihoods: R, Wt [P][B] and dpar at P = 1 / 3 / 7, B not a multiple of 256,
     scale 1.7, the tails and v from 0 to 1e4 (dpar per element through one-element calls as well);
  b. gpk_lik_varexp_sum per element (one-element views, each writing its own out[i]) and over the whole table;
  c. the predictions per element, fp64 and fp32 storage (fp32: the fp64 result rounded once);
  d. MultiClass at C = 2 ... 128, on both sides of every 32-class chunk edge: R, Wt, dVE/deps, per-row VE, predictions;
  e. grid-stride launches past every cap (scalar 2048 x 256 elements, MultiClass 8192 x 4 rows, heteroskedastic
     2048 x 256 rows);
  f. the case table reaches every kernel instantiation of lik.cu;
  g. the worst |device - exact| / bar per kernel and likelihood."""
import ctypes
import functools
import math
import os
import re

import numpy as np
import pytest

from gpflow_b200 import _lib
from tests import hetero_oracle as HO
from tests import lik_bounds as LB
from tests import multiclass_oracle as MO

pytestmark = pytest.mark.gpu

GUARD = 4096
CS = 1.7
EPS = 1e-3
REPORT = {}
REACHED = set()
SCALAR = LB.scalar_cases()
IDS = [LB.case_name(*c) for c in SCALAR]
F32_MAX = float(np.finfo(np.float32).max)


def _torch():
    import torch
    return torch


def _desc(kind, par):
    return _lib.LikDesc(LB.TYPE[kind], 20, par.get("scale", 0.0), par.get("df", 0.0), par.get("binsize", 0.0),
                        par.get("noise", 0.0), 0.0, 0, 0, 0.0)


def _mc_desc(C):
    return _lib.LikDesc(_lib.LIK_MULTICLASS, 20, 0.0, 0.0, 0.0, 0.0, EPS, C, 0, 0.0)


class Guarded:
    """A view of n elements inside a NaN-filled device buffer with GUARD elements on each side."""

    def __init__(self, values, dtype=np.float64, n=None):
        T = _torch()
        td = T.float64 if dtype == np.float64 else T.float32
        n = len(values) if values is not None else n
        self.buf = T.full((2 * GUARD + n,), float("nan"), dtype=td, device="cuda")
        self.view = self.buf[GUARD:GUARD + n]
        if values is not None:
            self.view.copy_(T.from_numpy(np.ascontiguousarray(values, dtype=dtype)))
        self.n, self.size = n, self.buf.element_size()

    def ptr(self, i=0):
        return ctypes.c_void_p(self.view.data_ptr() + i * self.size)

    def host(self):
        return self.view.cpu().numpy().astype(np.float64)

    def guards_intact(self):
        T = _torch()
        return bool(T.isnan(self.buf[:GUARD]).all()) and bool(T.isnan(self.buf[GUARD + self.n:]).all())


def _ok(status, what):
    if status != 0:
        raise _lib.GpkError(f"{what}: {_lib.load().gpk_last_error().decode()}")


def _sync():
    _torch().cuda.synchronize()


def _ratio(got, want, bar):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.abs(got - want) / bar
    r = np.where(got == want, 0.0, r)
    return np.where(np.isnan(r), np.inf, r)


def _check(key, got, want, bar, where=""):
    r = _ratio(got, want, bar)
    REPORT[key] = max(REPORT.get(key, 0.0), float(r.max()) if r.size else 0.0)
    if r.size and not r.max() <= 1.0:
        i = int(np.argmax(r))
        raise AssertionError(f"{key} {where}: element {i} device {np.ravel(got)[i]!r} exact {np.ravel(want)[i]!r} "
                             f"bar {np.ravel(bar)[i]:.3g} ratio {r.ravel()[i]:.3g} ({int((r > 1).sum())} elements out)")


def _sum_bar(terms, bars, scale=1.0):
    """The bar of scale * sum_i terms_i summed in any order: the terms' bars, (n + 2) u sum |term| for the order and the
    final scaling, and the exact per-element values' own rounding to double."""
    n = len(terms)
    a = float(np.sum(np.abs(terms)))
    return abs(scale) * (float(np.sum(bars)) + (n + 3) * LB.U * a)


def _f32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


# ---- the exact references, once per session ------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _exact_scalar(i, f32=False):
    kind, par = SCALAR[i]
    y, mu, v = LB.scalar_elements(kind)
    if f32:
        y, mu, v = _f32(y), _f32(mu), _f32(v)
    return (y, mu, v), LB.exact_scalar(kind, par, y, mu, v)


@functools.lru_cache(maxsize=None)
def _exact_predict(i, f32=False):
    kind, par = SCALAR[i]
    y, mu, v = LB.predict_elements(kind)
    if f32:
        y, mu, v = _f32(y), _f32(mu), _f32(v)
    return (y, mu, v), LB.exact_scalar_predict(kind, par, y, mu, v)


@functools.lru_cache(maxsize=None)
def _mc_case(C):
    """The MultiClass rows with fp32-representable inputs, so that one exact reference serves both storage types."""
    y, mu, v = LB.mc_rows(C)
    y, mu, v = y, _f32(mu), _f32(v)
    return (y, mu, v), LB.exact_mc(C, EPS, y, mu, v)


# ---- a. scalar adjoints --------------------------------------------------------------------------------------------
def _grad_call(kind, par, y, mu, v, B, P):
    """gpk_lik_varexp_grad on element i = b P + p of (y, mu, v): (R [B*P], Wt [P*B], dpar)."""
    idx = np.arange(B * P)
    fvar_t = v.reshape(B, P).T.reshape(-1)
    Fm, Fv, Y = Guarded(mu), Guarded(fvar_t), Guarded(y)
    R, Wt, dp = Guarded(None, n=B * P), Guarded(None, n=B * P), Guarded(np.zeros(1))
    _ok(_lib.load().gpk_lik_varexp_grad(ctypes.byref(_desc(kind, par)), Fm.ptr(), Fv.ptr(), Y.ptr(), B, P, CS,
                                        R.ptr(), Wt.ptr(), dp.ptr(), None), "gpk_lik_varexp_grad")
    _sync()
    for g in (Fm, Fv, Y, R, Wt, dp):
        assert g.guards_intact(), "a guard region was written"
    return R.host(), Wt.host().reshape(P, B).T.reshape(-1)[idx], dp.host()[0]


@pytest.mark.parametrize("P", [1, 3, 7])
@pytest.mark.parametrize("i", range(len(SCALAR)), ids=IDS)
def test_scalar_adjoints(cuda_device, i, P):
    kind, par = SCALAR[i]
    (y, mu, v), ex = _exact_scalar(i)
    n = len(y)
    B = -(-n // P)
    if B % 256 == 0:
        B += 1
    idx = np.arange(B * P) % n
    em = LB.scalar_ve(kind, par, y, mu, v)
    R, W, dpar = _grad_call(kind, par, y[idx], mu[idx], v[idx], B, P)
    REACHED.add("lik_grad_kernel")
    cR, cW = CS * em["dmu"], CS * em["dv"]
    _check(f"grad R {kind}", R, CS * ex["dmu"][idx], LB.bar(cR)[idx], f"P={P} {IDS[i]}")
    _check(f"grad Wt {kind}", W, CS * ex["dv"][idx], LB.bar(cW)[idx], f"P={P} {IDS[i]}")
    if kind in ("gaussian", "student_t"):
        want = CS * math.fsum(ex["dpar"][idx])
        _check(f"grad dpar sum {kind}", dpar, want, _sum_bar(ex["dpar"][idx], LB.bar(em["dpar"])[idx], CS))
    else:
        assert dpar == 0.0
    if P == 1:   # dpar element by element: one call per element, each adding into its own zeroed slot
        Fm, Fv, Y = Guarded(mu), Guarded(v), Guarded(y)
        R1, W1, D1 = Guarded(None, n=n), Guarded(None, n=n), Guarded(np.zeros(n))
        lib, d = _lib.load(), _desc(kind, par)
        for j in range(n):
            _ok(lib.gpk_lik_varexp_grad(ctypes.byref(d), Fm.ptr(j), Fv.ptr(j), Y.ptr(j), 1, 1, CS, R1.ptr(j), W1.ptr(j),
                                        D1.ptr(j), None), "gpk_lik_varexp_grad")
        _sync()
        assert all(g.guards_intact() for g in (Fm, Fv, Y, R1, W1, D1))
        np.testing.assert_array_equal(R1.host(), R[:n])   # one element or many: the same arithmetic
        np.testing.assert_array_equal(W1.host(), W[:n])
        if kind in ("gaussian", "student_t"):
            _check(f"grad dpar {kind}", D1.host(), CS * ex["dpar"], LB.bar(CS * em["dpar"]))


def test_scalar_dv_at_zero_variance_is_the_limit(cuda_device):
    """At v = 0 d/dv is g''(mu) / 2, finite, for every quadrature likelihood (0/0 before the limit was taken)."""
    for i, (kind, par) in enumerate(SCALAR):
        (y, mu, v), ex = _exact_scalar(i)
        z = v == 0.0
        _, W, _ = _grad_call(kind, par, y[z], mu[z], v[z], int(z.sum()), 1)
        assert np.all(np.isfinite(W)), (kind, W)


# ---- b. variational expectations -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("i", range(len(SCALAR)), ids=IDS)
def test_scalar_varexp(cuda_device, i, dtype):
    kind, par = SCALAR[i]
    (y, mu, v), ex = _exact_scalar(i, dtype == np.float32)
    em = LB.scalar_ve(kind, par, y, mu, v, grad=False)["ve"]
    n, code = len(y), _lib.GPK_F64 if dtype == np.float64 else _lib.GPK_F32
    Fm, Fv, Y, out = Guarded(mu, dtype), Guarded(v, dtype), Guarded(y, dtype), Guarded(None, n=n)
    lib, d = _lib.load(), _desc(kind, par)
    for j in range(n):
        _ok(lib.gpk_lik_varexp_sum(ctypes.byref(d), Fm.ptr(j), Fv.ptr(j), Y.ptr(j), 1, 1, 1.0, 0, out.ptr(j), code,
                                   None), "gpk_lik_varexp_sum")
    REACHED.add(f"lik_varexp_kernel<{'double' if dtype == np.float64 else 'float'}>")
    tot = Guarded(None, n=1)
    _ok(lib.gpk_lik_varexp_sum(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), n, 1, CS, 0, tot.ptr(), code, None),
        "gpk_lik_varexp_sum")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, out, tot))
    _check(f"varexp {kind}", out.host(), ex["ve"], LB.bar(em), IDS[i])
    _check(f"varexp sum {kind}", tot.host(), CS * math.fsum(ex["ve"]), _sum_bar(ex["ve"], LB.bar(em), CS))


# ---- c. predictions ------------------------------------------------------------------------------------------------
def _pred_bar(exact, em, f32):
    b = LB.bar(em)
    return LB.round32_bar(exact, b) if f32 else b


def _pred_check(key, got, exact, em, f32):
    """fp32: where every value within the fp64 bar overflows fp32, the device must give the rounded exact value's
    infinity; where only some do, an infinity of either sign or a value inside the bar."""
    if f32:
        b64 = LB.bar(em)
        over = np.abs(exact) - b64 > F32_MAX
        np.testing.assert_array_equal(got[over], np.float32(exact[over]).astype(np.float64))
        edge = (np.abs(exact) + b64 > F32_MAX) & ~over
        assert not np.any(np.isnan(got[edge]))
        keep = ~over & ~(edge & np.isinf(got))
        got, exact, em = got[keep], exact[keep], LB.Err(em.v[keep], em.e[keep])
    _check(key, got, exact, _pred_bar(exact, em, f32))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("i", range(len(SCALAR)), ids=IDS)
def test_scalar_predictions(cuda_device, i, dtype):
    kind, par = SCALAR[i]
    f32 = dtype == np.float32
    (y, mu, v), ex = _exact_predict(i, f32)
    n, code, tn = len(y), _lib.GPK_F32 if f32 else _lib.GPK_F64, "float" if f32 else "double"
    lib, d = _lib.load(), _desc(kind, par)
    Fm, Fv, Y = Guarded(mu, dtype), Guarded(v, dtype), Guarded(y, dtype)
    mean, var, ld = Guarded(None, dtype, n), Guarded(None, dtype, n), Guarded(None, dtype, n)
    st = lib.gpk_lik_predict_mean_and_var(ctypes.byref(d), Fm.ptr(), Fv.ptr(), n, 1, mean.ptr(), var.ptr(), code, None)
    if kind == "student_t" and par["df"] <= 2:
        assert st != 0 and b"df > 2" in lib.gpk_last_error()
    else:
        _ok(st, "gpk_lik_predict_mean_and_var")
        REACHED.add(f"lik_predict_mv_kernel<{tn}>")
    _ok(lib.gpk_lik_predict_log_density(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), n, 1, ld.ptr(), code, None),
        "gpk_lik_predict_log_density")
    REACHED.add(f"lik_predict_ld_kernel<{tn}>")
    # the row sum over P = 3 latents
    P = 3
    N = n // P
    ld3 = Guarded(None, dtype, N)
    _ok(lib.gpk_lik_predict_log_density(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), N, P, ld3.ptr(), code, None),
        "gpk_lik_predict_log_density")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, mean, var, ld, ld3))
    em_ld = LB.scalar_predict_ld(kind, par, y, mu, v)
    _pred_check(f"predict ld {kind} {tn}", ld.host(), ex["ld"], em_ld, f32)
    terms, bars = ex["ld"][:N * P].reshape(N, P), LB.bar(em_ld)[:N * P].reshape(N, P)
    want3 = np.array([math.fsum(t) for t in terms])
    row = LB.Err(want3, bars.sum(1) / LB.SAFETY + (P + 2) * LB.U * np.abs(terms).sum(1))
    _pred_check(f"predict ld rows {kind} {tn}", ld3.host(), want3, row, f32)
    if kind != "student_t" or par["df"] > 2:
        m, vv = LB.scalar_predict_mv(kind, par, mu, v)
        _pred_check(f"predict mean {kind} {tn}", mean.host(), ex["mean"], m, f32)
        _pred_check(f"predict var {kind} {tn}", var.host(), ex["var"], vv, f32)


# ---- d. MultiClass -------------------------------------------------------------------------------------------------
def _mc_grad_call(C, y, mu, v):
    B = mu.shape[0]
    Fm, Fv, Y = Guarded(mu.reshape(-1)), Guarded(v.T.reshape(-1)), Guarded(y)
    R, Wt, ge = Guarded(None, n=B * C), Guarded(None, n=B * C), Guarded(np.zeros(1))
    _ok(_lib.load().gpk_lik_varexp_grad(ctypes.byref(_mc_desc(C)), Fm.ptr(), Fv.ptr(), Y.ptr(), B, C, CS, R.ptr(),
                                        Wt.ptr(), ge.ptr(), None), "gpk_lik_varexp_grad")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, R, Wt, ge)), "a guard region was written"
    return R.host().reshape(B, C), Wt.host().reshape(C, B).T, ge.host()[0]


def _mc_check_grad(C, y, mu, v, ex, rows, tag):
    em = LB.mc_grad(C, EPS, y, mu, v, CS)
    R, W, geps = _mc_grad_call(C, y[rows], mu[rows], v[rows])
    REACHED.add(f"mc_grad_kernel<{(C + 31) // 32}>")
    _check("multiclass R", R, CS * ex["R"][rows], LB.bar(em["R"])[rows], tag)
    _check("multiclass Wt", W, CS * ex["W"][rows], LB.bar(em["W"])[rows], tag)
    _check("multiclass geps", geps, CS * math.fsum(ex["deps"][rows]),
           _sum_bar(ex["deps"][rows], LB.bar(em["deps"])[rows], CS), tag)


def _mc_values(C, y, mu, v, dtype, rows):
    """(per-row VE through one-row views, the VE sum, predictive mean and var [N, C], log density [N])."""
    code, tn = (_lib.GPK_F64, "double") if dtype == np.float64 else (_lib.GPK_F32, "float")
    lib, d = _lib.load(), _mc_desc(C)
    N = len(rows)
    Fm, Fv, Y = Guarded(mu[rows].reshape(-1), dtype), Guarded(v[rows].reshape(-1), dtype), Guarded(y[rows], dtype)
    out, tot = Guarded(None, n=min(N, 64)), Guarded(None, n=1)
    for j in range(out.n):
        _ok(lib.gpk_lik_varexp_sum(ctypes.byref(d), Fm.ptr(j * C), Fv.ptr(j * C), Y.ptr(j), 1, C, 1.0, 0, out.ptr(j),
                                   code, None), "gpk_lik_varexp_sum")
    _ok(lib.gpk_lik_varexp_sum(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), N, C, CS, 0, tot.ptr(), code, None),
        "gpk_lik_varexp_sum")
    mean, var, ld = Guarded(None, dtype, N * C), Guarded(None, dtype, N * C), Guarded(None, dtype, N)
    _ok(lib.gpk_lik_predict_mean_and_var(ctypes.byref(d), Fm.ptr(), Fv.ptr(), N, C, mean.ptr(), var.ptr(), code, None),
        "gpk_lik_predict_mean_and_var")
    _ok(lib.gpk_lik_predict_log_density(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), N, C, ld.ptr(), code, None),
        "gpk_lik_predict_log_density")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, out, tot, mean, var, ld)), "a guard region was written"
    NJ = (C + 31) // 32
    REACHED.update({f"mc_varexp_kernel<{tn}, {NJ}>", f"mc_predict_mv_kernel<{tn}, {NJ}>",
                    f"mc_predict_ld_kernel<{tn}, {NJ}>"})
    return out.host(), tot.host()[0], mean.host().reshape(N, C), var.host().reshape(N, C), ld.host()


def _mc_check_values(C, y, mu, v, ex, dtype, rows, tag):
    f32 = dtype == np.float32
    tn = "float" if f32 else "double"
    ve1, tot, mean, var, ld = _mc_values(C, y, mu, v, dtype, rows)
    ve = LB.mc_ve(C, EPS, y, mu, v)
    k = len(ve1)
    _check(f"multiclass varexp {tn}", ve1, ex["ve"][rows][:k], LB.bar(ve)[rows][:k], tag)
    _check(f"multiclass varexp sum {tn}", tot, CS * math.fsum(ex["ve"][rows]),
           _sum_bar(ex["ve"][rows], LB.bar(ve)[rows], CS), tag)
    em_m, em_v, em_ld = LB.mc_predict(C, EPS, y, mu, v)
    # the float64 oracle's class probabilities, inside one bar of the exact ones (tests/test_lik_bounds.py): two bars
    wm, wv = MO.MultiClass(C, EPS).predict_mean_and_var(mu, v)
    _pred_check(f"multiclass predict mean {tn}", mean, wm[rows], LB.Err(em_m.v[rows], 2 * em_m.e[rows]), f32)
    _pred_check(f"multiclass predict var {tn}", var, wv[rows], LB.Err(em_v.v[rows], 2 * em_v.e[rows]), f32)
    _pred_check(f"multiclass predict ld {tn}", ld, ex["ld"][rows], LB.Err(em_ld.v[rows], em_ld.e[rows]), f32)


@pytest.mark.parametrize("C", LB.MC_CLASSES)
def test_multiclass_adjoints(cuda_device, C):
    (y, mu, v), ex = _mc_case(C)
    _mc_check_grad(C, y, mu, v, ex, np.arange(len(y)), f"C={C}")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("C", LB.MC_CLASSES)
def test_multiclass_values(cuda_device, C, dtype):
    (y, mu, v), ex = _mc_case(C)
    _mc_check_values(C, y, mu, v, ex, dtype, np.arange(len(y)), f"C={C}")


# ---- e. grid-stride launches ---------------------------------------------------------------------------------------
LIK_CAP = 2048 * 256     # lik_grid: 2048 CTAs of 256 threads, one element (heteroskedastic: one row) per thread
MC_CAP = 8192 * 4        # mc_grid: 8192 CTAs of 4 warps, one row per warp


@pytest.mark.parametrize("kind", ["bernoulli", "student_t"])
def test_scalar_grid_stride(cuda_device, kind):
    i = next(j for j, (k, p) in enumerate(SCALAR) if k == kind and p.get("df", 3.0) == 3.0
             and p.get("scale", 0.7) == 0.7)
    _, par = SCALAR[i]
    (y, mu, v), ex = _exact_scalar(i)
    P = 3
    B = LIK_CAP // P + 1001
    idx = np.arange(B * P) % len(y)
    assert B * P > LIK_CAP
    em = LB.scalar_ve(kind, par, y, mu, v)
    R, W, dpar = _grad_call(kind, par, y[idx], mu[idx], v[idx], B, P)
    _check(f"grid-stride R {kind}", R, CS * ex["dmu"][idx], LB.bar(CS * em["dmu"])[idx])
    _check(f"grid-stride Wt {kind}", W, CS * ex["dv"][idx], LB.bar(CS * em["dv"])[idx])
    if kind == "student_t":
        _check(f"grid-stride dpar {kind}", dpar, CS * math.fsum(ex["dpar"][idx]),
               _sum_bar(ex["dpar"][idx], LB.bar(em["dpar"])[idx], CS))
    Fm, Fv, Y, out = Guarded(mu[idx]), Guarded(v[idx]), Guarded(y[idx]), Guarded(None, n=1)
    _ok(_lib.load().gpk_lik_varexp_sum(ctypes.byref(_desc(kind, par)), Fm.ptr(), Fv.ptr(), Y.ptr(), B, P, CS, 0,
                                       out.ptr(), _lib.GPK_F64, None), "gpk_lik_varexp_sum")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, out))
    ve = LB.scalar_ve(kind, par, y, mu, v, grad=False)["ve"]
    _check(f"grid-stride varexp sum {kind}", out.host(), CS * math.fsum(ex["ve"][idx]),
           _sum_bar(ex["ve"][idx], LB.bar(ve)[idx], CS))


@pytest.mark.parametrize("C", [3, 33])
def test_multiclass_grid_stride(cuda_device, C):
    y, mu, v = LB.mc_rows(C)
    y, mu, v = y, _f32(mu), _f32(v)
    ex = LB.exact_mc(C, EPS, y, mu, v)
    rows = np.arange(MC_CAP + 77) % len(y)
    _mc_check_grad(C, y, mu, v, ex, rows, f"grid-stride C={C}")
    _mc_check_values(C, y, mu, v, ex, np.float64, rows, f"grid-stride C={C}")


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_heteroskedastic_grid_stride(cuda_device, dtype):
    rng = np.random.default_rng(21)
    n0, B = 257, LIK_CAP + 1001
    mu = np.c_[rng.standard_normal(n0), 0.5 * rng.standard_normal(n0)]
    v = np.c_[rng.uniform(0, 1, n0), rng.uniform(0, 0.5, n0)]
    v[:7, 1] = 0.0
    y = rng.standard_normal(n0)
    if dtype == np.float32:
        mu, v, y = _f32(mu), _f32(v), _f32(y)
    idx = np.arange(B) % n0
    d = _lib.LikDesc(_lib.LIK_HETEROSKEDASTIC, 20, 0.0, 0.0, 0.0, 0.0, 0.0, 0, _lib.LIK_SCALE_EXP, 0.0)
    h = HO.Hetero()
    code = _lib.GPK_F64 if dtype == np.float64 else _lib.GPK_F32
    Fm, Fv, Y, out = Guarded(mu[idx].reshape(-1), dtype), Guarded(v[idx].reshape(-1), dtype), Guarded(y[idx], dtype), \
        Guarded(None, n=1)
    lib = _lib.load()
    _ok(lib.gpk_lik_varexp_sum(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), B, 2, 1.0, 0, out.ptr(), code, None),
        "gpk_lik_varexp_sum")
    _sync()
    assert all(g.guards_intact() for g in (Fm, Fv, Y, out))
    REACHED.add(f"het_varexp_kernel<{'double' if code == _lib.GPK_F64 else 'float'}>")
    want = math.fsum(h.factorised_ve(mu, v, y[:, None])[idx].ravel())
    np.testing.assert_allclose(out.host()[0], want, rtol=1e-12)
    if dtype == np.float64:
        Fm, Fv, Y = Guarded(mu[idx].reshape(-1)), Guarded(v[idx].T.reshape(-1)), Guarded(y[idx])
        R, Wt, dp = Guarded(None, n=2 * B), Guarded(None, n=2 * B), Guarded(np.zeros(1))
        _ok(lib.gpk_lik_varexp_grad(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), B, 2, CS, R.ptr(), Wt.ptr(), dp.ptr(),
                                    None), "gpk_lik_varexp_grad")
        _sync()
        assert all(g.guards_intact() for g in (Fm, Fv, Y, R, Wt, dp))
        REACHED.add("het_grad_kernel")
        dmu, dv, _ = h.ve_grads(mu, v, y[:, None])
        for got, ref in ((R.host().reshape(B, 2), CS * dmu[idx]), (Wt.host().reshape(2, B).T, CS * dv[idx])):
            for p in range(2):
                np.testing.assert_allclose(got[:, p], ref[:, p], rtol=1e-11, atol=1e-13 * np.max(np.abs(ref[:, p])))
        assert dp.host()[0] == 0.0


def test_heteroskedastic_predictions_reach_both_storage_types(cuda_device):
    """The heteroskedastic prediction kernels' values are covered in tests/test_gpu_heteroskedastic.py; here one
    launch of each per storage type, for the instantiation table."""
    rng = np.random.default_rng(4)
    mu, v, y = rng.standard_normal((50, 2)), rng.uniform(0, 1, (50, 2)), rng.standard_normal(50)
    d = _lib.LikDesc(_lib.LIK_HETEROSKEDASTIC, 20, 0.0, 0.0, 0.0, 0.0, 0.0, 0, _lib.LIK_SCALE_EXP, 0.0)
    h = HO.Hetero()
    lib = _lib.load()
    for dtype, code, tn in ((np.float64, _lib.GPK_F64, "double"), (np.float32, _lib.GPK_F32, "float")):
        m_, v_, y_ = (np.asarray(a, dtype).astype(np.float64) for a in (mu, v, y))
        Fm, Fv, Y = Guarded(m_.reshape(-1), dtype), Guarded(v_.reshape(-1), dtype), Guarded(y_, dtype)
        mean, var, ld = Guarded(None, dtype, 50), Guarded(None, dtype, 50), Guarded(None, dtype, 50)
        _ok(lib.gpk_lik_predict_mean_and_var(ctypes.byref(d), Fm.ptr(), Fv.ptr(), 50, 2, mean.ptr(), var.ptr(), code,
                                             None), "gpk_lik_predict_mean_and_var")
        _ok(lib.gpk_lik_predict_log_density(ctypes.byref(d), Fm.ptr(), Fv.ptr(), Y.ptr(), 50, 2, ld.ptr(), code, None),
            "gpk_lik_predict_log_density")
        _sync()
        assert all(g.guards_intact() for g in (Fm, Fv, Y, mean, var, ld))
        rt = 1e-12 if dtype == np.float64 else 1e-6
        wm, wv = h.grid_mean_and_var(m_, v_)
        np.testing.assert_allclose(mean.host(), np.ravel(wm), rtol=rt)
        np.testing.assert_allclose(var.host(), np.ravel(wv), rtol=rt)
        np.testing.assert_allclose(ld.host(), h.grid_log_density(m_, v_, y_[:, None]), rtol=rt, atol=rt)
        REACHED.update({f"het_predict_mv_kernel<{tn}>", f"het_predict_ld_kernel<{tn}>"})


# ---- f. instantiation coverage -------------------------------------------------------------------------------------
def _instantiations_in_source():
    """Every kernel instantiation of lik.cu: the __global__ templates with their argument ranges."""
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpflow_b200", "csrc",
                            "lik.cu")).read()
    names = re.findall(r"__global__ void __launch_bounds__\([^)]*\)\s*(\w+)\(", src)
    want = set()
    for nm in names:
        if nm.startswith("mc_") and nm != "mc_grad_kernel":
            want |= {f"{nm}<{t}, {nj}>" for t in ("float", "double") for nj in (1, 2, 3, 4)}
        elif nm == "mc_grad_kernel":
            want |= {f"mc_grad_kernel<{nj}>" for nj in (1, 2, 3, 4)}
        elif nm in ("lik_grad_kernel", "het_grad_kernel"):
            want.add(nm)
        else:
            want |= {f"{nm}<{t}>" for t in ("float", "double")}
    return want


def test_case_table_reaches_every_instantiation():
    """From the case parameters: the dtypes, the class counts' chunk counts and the likelihood types the tests above
    launch (REACHED records the same names as they run)."""
    reach = {"lik_grad_kernel", "het_grad_kernel"}
    for tn in ("float", "double"):
        reach |= {f"lik_varexp_kernel<{tn}>", f"lik_predict_mv_kernel<{tn}>", f"lik_predict_ld_kernel<{tn}>",
                  f"het_varexp_kernel<{tn}>", f"het_predict_mv_kernel<{tn}>", f"het_predict_ld_kernel<{tn}>"}
        for C in LB.MC_CLASSES:
            nj = (C + 31) // 32
            reach |= {f"mc_varexp_kernel<{tn}, {nj}>", f"mc_predict_mv_kernel<{tn}, {nj}>",
                      f"mc_predict_ld_kernel<{tn}, {nj}>", f"mc_grad_kernel<{nj}>"}
    want = _instantiations_in_source()
    assert len(want) == 42, sorted(want)
    assert reach == want, (sorted(want - reach), sorted(reach - want))
    # every chunk count with a class count on each side of its upper edge (31 | 32 | 33, ...)
    for nj in (1, 2, 3):
        assert 32 * nj in LB.MC_CLASSES and 32 * nj + 1 in LB.MC_CLASSES
    if REACHED:   # the GPU tests of this session ran: what they launched is the table
        assert REACHED == want, (sorted(want - REACHED), sorted(REACHED - want))


# ---- g. report -----------------------------------------------------------------------------------------------------
def test_report_worst_ratios():
    """Prints the worst |device - exact| / bar of every kernel and likelihood measured in this session."""
    print("\nworst |device - exact| / bar:")
    for k in sorted(REPORT):
        print(f"  {k:44s} {REPORT[k]:.3g}")
