"""Error-bounded references for the K-build (csrc/kbuild.cu), CPU only.

Instead of one blanket rtol, every element of a device K gets an interval that a correct kernel must hit.

Function bars.  A stationary leaf is evaluated as k(x) with x = c r2 (c from `FOLD`, r2 the squared distance of the
inputs scaled by 1/lengthscale) and u = sqrt(x) (u = x for RBF).  The bar on |k_dev - k(x)| / k(x) has the form
(a + b u) eps, eps = 2^-53 (fp64) or 2^-24 (fp32), plus an absolute term for underflow:

fp64 fast path (`stationary_value4`).  From the CPU model of tests/test_fast_math_model.py: the table-driven
exp(-u), i.e. table rounding, polynomial, the product t * p, is within E_EXP = 4.5e-16 / eps, and the Newton / Heron
sqrt within E_SQRT = 3.4e-16 / eps.  On top of that:
  - the table premultiplied by the variance (RBF, Matern12, Exponential) or the product pre * t (Matern): +1;
  - Matern32 prefactor fma(var, u, var): its rounding +1, and the sqrt error enters as u d / (1 + u) <= d: +E_SQRT;
  - Matern52 prefactor fma(var3, x, fma(var, u, var)): +1 for the outer rounding and the larger of var3 = var * (1/3)
    (2 roundings) and the inner fma (1 + E_SQRT);
  - the sqrt error d = E_SQRT eps carried through exp(-u) gives exp(-u) (1 - u d): b = E_SQRT (b = 0 for RBF).
fp64 generic path (`leaf_value`): library exp (1 ulp = 2 eps) and sqrt, constants s3 / s5 (0.5), products and sums of
the prefactor: a = 3 (RBF, Matern12, Exponential), 7.5 (Matern32), 10.5 (Matern52); b = 2.5.
fp32 fast path (`stationary_value_f32`): __expf is within 2 + 1.173 u ulps (1 ulp <= 2 eps): a = 4, b = 2.346; the
product with var or the prefactor +1; sqrtf is correctly rounded: b += 1; prefactor Matern32 +2 (fmaf rounding, u),
Matern52 +3.  fp32 generic: expf within 2 ulps, so the fp64 generic numbers + 2.
A test uses the larger of the fast and generic bars, so one helper bounds both paths.

Absolute terms: fp64 adds 2^-1074 (results in the subnormal range round to that grid) and, for u > 708, var exp(-708)
(both paths return 0 there); fp32 adds var 2^-126 + 2^-149 (__expf flushes results below 2^-126 to zero).

Bound on x.  With the weighted inputs z = x_input * w (w = sqrt(c) / lengthscale per dimension) and the scaled norms
na = |z_i|^2, nb = |z_j|^2, the device forms x = na + nb - 2 <z_i, z_j>.  Per element, with u_T the unit roundoff of the
dtype and D the number of active dimensions:
  - each norm is a D-term sum of rounded squares (sequential fmas, or 8-lane butterflies plus one add per 8-dim
    chunk): (D + 3) u_T na;
  - the D-term dot product: D u_T sum |z_id z_jd| <= D u_T (na + nb) / 2, counted twice;
  - the sum na + nb and the final fma: u_T (na + nb) + u_T |x| <= 3 u_T (na + nb);
  - the generic path's `scale *` after the expansion (scale itself rounded): 4 u_T (na + nb);
  - the weighted inputs are rounded (relative 2 u_T + 4 u_64, including the fp32 cast and the host's rounding of w):
    x moves by at most 4 * that * (na + nb) (Cauchy-Schwarz);
  - the reference x_ref = sum_d (z_id - z_jd)^2 in fp64 (rounded z, differences, squares, sum): (2 D + 30) u_64
    (na + nb) covers it with the weight terms.
So |x_dev - x_ref| <= Bx = gamma (na + nb), gamma = (2 D + 18) u_T + (2 D + 30) u_64.  The bound is stated for the
scaled norms, so it also holds for the generic path, which applies the scale after the norm expansion.

Interval on k.  Every stationary leaf decreases monotonically in x >= 0, so k_dev must lie in
[k(x_ref + Bx) (1 - e_f) - atol, k(max(x_ref - Bx, clip)) (1 + e_f) + atol], e_f the function bar at u(x_ref + Bx),
clip = c 1e-36 (none for RBF, whose generic path does not clip).  Linear leaves, Sum and Product combine intervals.

The other fused leaves (generic kernel only, `leaf_value`; parameters are rounded to the dtype, T(var), T(alpha),
T(offset), and the references use the rounded values):
  - RationalQuadratic var (1 + x / (2 alpha))^-alpha, x = r2 (c = 1), decreases in x: the same Bx, then the base
    1 + fl(fl(0.5 x) / alpha) carries 2 roundings, which the power amplifies by alpha (a factor exp(2.01 alpha u_T)),
    plus pow's ulp bound (`ULP`) and the product with var.
  - Polynomial (var <x, x'> + offset)^degree: the Linear dot interval, plus the offset (one rounding), then the power
    at both ends of the interval (0 inside it for even degrees), plus pow's ulp bound.
  - Constant is exactly T(var) everywhere; White exactly T(var) on the diagonal of the symmetric form and +0 elsewhere,
    the rectangular call with X2 = X included.
K_diag (`kdiag_kernel`): exactly T(var) for stationary, Constant and White leaves; a running sum
sum_d fl(fl(T(w_d) x_d) x_d) for Linear / Polynomial, within (D + 4) u_T sum_d |w_d| x_d^2, then as above.

`ULP` collects the maximum errors of the CUDA Math API (CUDA C++ Programming Guide, appendix "Mathematical Functions":
double and single precision tables, default -prec-sqrt=true, no fast math), in ulps of the result; k ulps are at most
2 k u relative for a normal result."""
from __future__ import annotations

import numpy as np

from gpflow_b200 import _lib

U64, U32 = 2.0 ** -53, 2.0 ** -24
FOLD = {_lib.K_RBF: 0.5, _lib.K_MATERN12: 1.0, _lib.K_EXPONENTIAL: 0.25, _lib.K_MATERN32: 3.0, _lib.K_MATERN52: 5.0}
STATIONARY = tuple(FOLD)
NAMES = {_lib.K_RBF: "rbf", _lib.K_MATERN12: "m12", _lib.K_EXPONENTIAL: "exp", _lib.K_MATERN32: "m32",
         _lib.K_MATERN52: "m52"}
E_EXP, E_SQRT = 4.5e-16 / U64, 3.4e-16 / U64
ULP = {"exp": 1, "expf": 2, "pow": 2, "powf": 4, "sin": 2, "sinf": 2, "cos": 2, "cosf": 2, "acos": 2, "acosf": 2,
       "sqrt": 0, "sqrtf": 0}
FUSED_NAMES = {**NAMES, _lib.K_RQ: "rq", _lib.K_LINEAR: "lin", _lib.K_POLYNOMIAL: "poly",
               _lib.K_CONSTANT: "const", _lib.K_WHITE: "white"}


def rnd(x, dtype):
    """x rounded to the dtype, back in fp64 (parameters as the kernels see them)."""
    return float(np.dtype(dtype).type(x))


def pow_ulp(dtype):
    return ULP["pow"] if np.dtype(dtype) == np.float64 else ULP["powf"]


def tiny_abs(dtype):
    return 2.0 ** -1074 if np.dtype(dtype) == np.float64 else 2.0 ** -149


def unit(dtype):
    return U64 if np.dtype(dtype) == np.float64 else U32


def fast_bar(op, dtype):
    """(a, b) of the fast path's function bar (a + b u) eps, see the module docstring."""
    sq = op != _lib.K_RBF
    if np.dtype(dtype) == np.float64:
        pre = {_lib.K_MATERN32: 1 + E_SQRT, _lib.K_MATERN52: 1 + max(2.0, 1 + E_SQRT)}.get(op, 0.0)
        return E_EXP + 1 + pre, E_SQRT if sq else 0.0
    pre = {_lib.K_MATERN32: 2.0, _lib.K_MATERN52: 3.0}.get(op, 0.0)
    return 4 + 1 + pre, 2.346 + (1.0 if sq else 0.0)


def generic_bar(op, dtype):
    a = {_lib.K_MATERN32: 7.5, _lib.K_MATERN52: 10.5}.get(op, 3.0)
    b = 2.5 if op != _lib.K_RBF else 0.0
    return (a, b) if np.dtype(dtype) == np.float64 else (a + 2, b)


def fn_bar(op, dtype):
    """Function bar covering both the fast and the generic path."""
    (a1, b1), (a2, b2) = fast_bar(op, dtype), generic_bar(op, dtype)
    return max(a1, a2), max(b1, b2)


def u_of_x(op, x):
    x = np.asarray(x, np.float64)
    return np.maximum(x, 0.0) if op == _lib.K_RBF else np.sqrt(np.maximum(x, 0.0))


def k_of_x(op, x, var):
    """var * k(x) in long double (64-bit or wider significand)."""
    x = np.asarray(x, np.longdouble)
    v = np.longdouble(var)
    if op == _lib.K_RBF:
        return v * np.exp(-x)
    u = np.sqrt(np.maximum(x, np.longdouble(0)))
    e = np.exp(-u)
    if op == _lib.K_MATERN32:
        return v * (1 + u) * e
    if op == _lib.K_MATERN52:
        return v * (1 + u + x / 3) * e
    return v * e


def atol_fn(dtype, var, u):
    if np.dtype(dtype) == np.float64:
        return np.where(np.asarray(u) > 708.0, var * np.exp(-708.0), 0.0) + 2.0 ** -1074
    return var * 2.0 ** -126 + 2.0 ** -149 + 0.0 * np.asarray(u)


def clip_of(op):
    return 0.0 if op == _lib.K_RBF else FOLD[op] * 1e-36


# ---- x reference -------------------------------------------------------------------------------------------------
def gamma(D, dtype):
    return (2 * D + 18) * unit(dtype) + (2 * D + 30) * U64


def r2_ref(Z, Z2, rows=None):
    """sum_d (Z_id - Z2_jd)^2 in fp64 for the given rows of Z (all columns of Z2), plus the squared norms."""
    Za = Z if rows is None else Z[rows]
    acc = np.zeros((Za.shape[0], Z2.shape[0]))
    for d in range(Z.shape[1]):
        acc += np.square(Za[:, d, None] - Z2[None, :, d])
    return acc, np.square(Za).sum(1), np.square(Z2).sum(1)


def stationary_interval(op, var, D, dtype, r2, na, nb):
    """(center, lo, hi) of one stationary leaf from c = 1 distances r2 and norms (of inputs scaled by 1/lengthscale)."""
    c = FOLD[op]
    x = c * r2
    bx = gamma(D, dtype) * c * (na[:, None] + nb[None, :])
    xhi, xlo = x + bx, x - bx
    if op != _lib.K_RBF:
        xlo = np.maximum(xlo, clip_of(op))
    a, b = fn_bar(op, dtype)
    uh = u_of_x(op, xhi)
    ef = (a + b * uh) * unit(dtype)
    at = atol_fn(dtype, var, uh)
    lo = np.asarray(k_of_x(op, xhi, var), np.float64) * (1 - ef) - at
    hi = np.asarray(k_of_x(op, xlo, var), np.float64) * (1 + ef) + at
    cen = np.asarray(k_of_x(op, np.maximum(x, clip_of(op)) if op != _lib.K_RBF else x, var), np.float64)
    return cen, lo, hi


# ---- compiled kernel expressions (kernels.compile_kernel output) -> intervals -----------------------------------
def _leaf_inputs(nd, dims, ard, D):
    cols = np.arange(D) if nd.n_dims == 0 else np.array([dims[nd.dims_off + i] for i in range(nd.n_dims)])
    if nd.n_ard > 0:
        par = np.array([ard[nd.ard_off + i] for i in range(nd.n_ard)], np.float64)
    else:
        par = np.full(len(cols), nd.lengthscale if nd.op in STATIONARY or nd.op == _lib.K_RQ else 1.0)
    return cols, par


def combine(op, kids, u):
    """Sum / Product of child intervals, left to right as the postfix fold evaluates them, one rounding per step."""
    cen, lo, hi = kids[0]
    for kc, kl, kh in kids[1:]:
        if op == _lib.K_SUM:
            cen, lo, hi = cen + kc, lo + kl, hi + kh
        else:
            p = np.stack([lo * kl, lo * kh, hi * kl, hi * kh])
            cen, lo, hi = cen * kc, p.min(0), p.max(0)
        m = u * np.maximum(np.abs(lo), np.abs(hi))     # rounding of this Sum / Product step
        lo, hi = lo - m, hi + m
    return cen, lo, hi


def rq_of_x(x, var, alpha):
    """var (1 + x / (2 alpha))^-alpha in long double."""
    a = np.longdouble(alpha)
    return np.longdouble(var) * (1 + np.asarray(x, np.longdouble) / (2 * a)) ** (-a)


def rq_interval(var, alpha, D, dtype, r2, na, nb):
    """(center, lo, hi) of a RationalQuadratic leaf from c = 1 distances and norms (module docstring)."""
    u = unit(dtype)
    var, alpha = rnd(var, dtype), rnd(alpha, dtype)
    bx = gamma(D, dtype) * (na[:, None] + nb[None, :])
    xlo = np.maximum(r2 - bx, -alpha)               # the device's x may be slightly negative
    amp = np.exp(2.01 * alpha * u)                  # the base's two roundings, amplified by the power
    e = (2 * pow_ulp(dtype) + 1.01) * u
    at = var * 2.0 ** -126 + 2.0 ** -149 if np.dtype(dtype) == np.float32 else 2.0 ** -1074
    lo = np.asarray(rq_of_x(r2 + bx, var, alpha), np.float64) / amp * (1 - e) - at
    hi = np.asarray(rq_of_x(xlo, var, alpha), np.float64) * amp * (1 + e) + at
    return np.asarray(rq_of_x(r2, var, alpha), np.float64), lo, hi


def int_degree(deg):
    return float(deg) == np.floor(deg)


def power_interval(y, ylo, yhi, deg, dtype):
    """(center, lo, hi) of y^deg for y in [ylo, yhi] (y < 0 only for integer degrees), plus pow's ulp bound."""
    u = unit(dtype)
    f = lambda t: np.asarray(np.power(np.asarray(t, np.longdouble), np.longdouble(deg)), np.float64)  # noqa: E731
    a, b = f(ylo), f(yhi)
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    if int_degree(deg) and int(deg) % 2 == 0:
        lo = np.where((ylo < 0) & (yhi > 0), 0.0, lo)
    e = 2 * pow_ulp(dtype) * u
    return f(y), lo - e * np.abs(lo) - tiny_abs(dtype), hi + e * np.abs(hi) + tiny_abs(dtype)


def expr_interval(desc, X, X2=None, rows=None, dtype=None, cache=None, sym=None):
    """(center, lo, hi) of K(X, X2)[rows] for a compiled expression of any fused leaves, Sum and Product nodes.
    X2=None: the symmetric form (same values; White is T(var) on its diagonal).  `sym` overrides which form White sees
    (a symmetric K whose columns are passed as X2).  `cache` (a dict) keeps the reference distances of the same inputs
    across calls, e.g. across kernel types: x for another c is a rescale of r2."""
    nodes, n_nodes, dims, ard = desc
    dtype = np.dtype(dtype or X.dtype)
    sym = X2 is None if sym is None else sym
    X = np.asarray(X, np.float64)
    X2 = X if X2 is None else np.asarray(X2, np.float64)
    D = X.shape[1]
    rows = np.arange(X.shape[0]) if rows is None else np.asarray(rows)
    u = unit(dtype)
    memo = {} if cache is None else cache

    def linear(nd, cols, par):
        v = par if nd.n_ard > 0 else np.full(len(cols), nd.variance)
        A, B = X[rows][:, cols] * v, X2[:, cols]
        cen = A @ B.T
        half = ((len(cols) + 3) * u + (len(cols) + 3) * U64) * (np.abs(A) @ np.abs(B).T)
        return cen, cen - half, cen + half

    def rec(i):
        nd = nodes[i]
        if nd.op in (_lib.K_SUM, _lib.K_PRODUCT):
            return combine(nd.op, [rec(nd.child[c]) for c in range(nd.n_children)], u)
        shape = (len(rows), X2.shape[0])
        if nd.op == _lib.K_CONSTANT:
            c = np.full(shape, rnd(nd.variance, dtype))
            return c, c, c
        if nd.op == _lib.K_WHITE:
            c = np.where(sym & (rows[:, None] == np.arange(shape[1])[None, :]), rnd(nd.variance, dtype), 0.0)
            return c, c, c
        cols, par = _leaf_inputs(nd, dims, ard, D)
        if nd.op == _lib.K_LINEAR:
            return linear(nd, cols, par)
        if nd.op == _lib.K_POLYNOMIAL:
            cen, lo, hi = linear(nd, cols, par)
            off = rnd(nd.lengthscale, dtype)
            m = u * np.maximum(np.abs(lo + off), np.abs(hi + off))
            return power_interval(cen + off, lo + off - m, hi + off + m, rnd(nd.alpha, dtype), dtype)
        if nd.op not in STATIONARY and nd.op != _lib.K_RQ:
            raise ValueError(f"no interval for kernel op {nd.op}")
        key = (tuple(cols), tuple(par))
        if key not in memo:
            memo[key] = r2_ref(X[:, cols] / par, X2[:, cols] / par, rows)
        r2, na, nb = memo[key]
        if nd.op == _lib.K_RQ:
            return rq_interval(nd.variance, nd.alpha, len(cols), dtype, r2, na, nb)
        return stationary_interval(nd.op, nd.variance, len(cols), dtype, r2, na, nb)

    return rec(n_nodes - 1)


def kdiag_interval(desc, X, dtype=None):
    """(center, lo, hi) of K_diag(X) as `kdiag_kernel` forms it (module docstring)."""
    nodes, n_nodes, dims, ard = desc
    dtype = np.dtype(dtype or X.dtype)
    X = np.asarray(X, np.float64)
    u = unit(dtype)

    def rec(i):
        nd = nodes[i]
        if nd.op in (_lib.K_SUM, _lib.K_PRODUCT):
            return combine(nd.op, [rec(nd.child[c]) for c in range(nd.n_children)], u)
        if nd.op not in (_lib.K_LINEAR, _lib.K_POLYNOMIAL):
            c = np.full(X.shape[0], rnd(nd.variance, dtype))
            return c, c, c
        cols, par = _leaf_inputs(nd, dims, ard, X.shape[1])
        w = par if nd.n_ard > 0 else np.ones(len(cols))
        var = 1.0 if nd.n_ard > 0 else nd.variance
        s = np.square(X[:, cols]) @ w * var
        half = ((len(cols) + 4) * u + 4 * U64) * np.abs(s)
        if nd.op == _lib.K_LINEAR:
            return s, s - half, s + half
        off = rnd(nd.lengthscale, dtype)
        y, ylo, yhi = s + off, s - half + off, s + half + off
        m = u * np.maximum(np.abs(ylo), np.abs(yhi))
        return power_interval(y, ylo - m, yhi + m, rnd(nd.alpha, dtype), dtype)

    return rec(n_nodes - 1)


def ratio(dev, cen, lo, hi):
    """|dev - center| relative to the interval's half-width on dev's side (> 1: outside)."""
    dev = np.asarray(dev, np.float64)
    up = dev >= cen
    w = np.where(up, hi - cen, cen - lo)
    return np.where(dev == cen, 0.0, np.abs(dev - cen) / np.where(w > 0, w, np.inf))


# ---- the fast path's x for axis-aligned inputs (part 1) ---------------------------------------------------------
def fast_weight(op, ell):
    """The folded weight sqrt((1 / (ell * ell)) * c) as compile_kprog / kbuild_fast_launch form it (fp64)."""
    return np.sqrt(np.float64(1.0) / (np.float64(ell) * np.float64(ell)) * np.float64(FOLD[op]))


def fast_x(v, t, w, dtype):
    """x_ij of rows (v_i, 0) against rows (0, t_j), D = 2, bit for bit: fl(fl(fl(v w)^2) + fl(fl(t w)^2)) in the
    dtype (the gram term is exactly zero, the norm butterflies add exact zeros)."""
    T = np.dtype(dtype).type
    wt = T(w)
    a = np.asarray(v, T) * wt
    b = np.asarray(t, T) * wt
    return (a * a)[:, None] + (b * b)[None, :]


def sweep_targets(op, n, umax, specials=True):
    """n target values of one axis' share of x, dense near zero: x = p_i + q_j then covers u in [0, umax]."""
    xmax = umax if op == _lib.K_RBF else umax * umax
    c = FOLD[op]
    sp = [0.0, 0.0, c * 1e-38, c * 0.5e-36, c * 0.99e-36, c * 2e-36, 1e-300 * xmax, 1e-20] if specials else []
    g = np.geomspace(xmax * 1e-16, xmax / 2, n - len(sp))
    return np.concatenate([sp, g])
