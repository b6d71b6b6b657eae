"""Error-bounded references for the materialised kernels (csrc/kaux.cu) and their compositions, CPU only.

`kaux_eval` works in fp64 on inputs converted exactly from the dtype, with the parameters as fp64 host values, and
rounds the result to the dtype once.  Each element gets an interval by interval propagation through the kernel's
operation order (u = 2^-53, `ULP` of tests/kbuild_bounds.py for the library functions, k ulps <= 2 k u relative):
  - Cosine: s = sum_d (x_d - x'_d) scale_d is within (D + 2) u sum_d |(x_d - x'_d) scale_d| of the exact sum, 2 pi s
    adds one rounding; cos over that interval (its extrema included), then cos's ulps, var * and the rounding to T.  The
    absolute error grows with |s|, as it does in the reference.
  - Periodic: per dimension the argument pi (x_d - x'_d) / p_d carries 3 roundings (relative), sin over that interval,
    sin's ulps, * scale_d, then |.| or the square; the running sum adds one rounding per term.  The base is monotone
    decreasing in that sum: its value at the two ends, widened by its own operations ((a + b r) u, as the generic
    K-build's bars, RQ through the amplified base as in kbuild_bounds.rq_interval).
  - ArcCosine: num, |x|^2, |x'|^2 within (D + 2) u of their absolute sums; sqrt, two divisions; the jittered argument
    1e-15 + (1 - 2e-15) c; acos over the interval (its slope is unbounded near |c| = 1, which the interval shows) and
    its ulps; J_n decreases on [0, pi]; J's own evaluation error is absolute (24 u times its largest term); |x|^n |x'|^n
    and var / pi.  Rows that are bitwise equal on the active dims give num = |x|^2 = |x'|^2 bit for bit, so
    c = fl(fl(n / fl(sqrt n)) / fl(sqrt n)) is within 5 u of 1 there: that tighter interval shows the jitter.
  - Coregion: exactly T(B[i, j]) with the indices truncated toward zero like tf.cast; an index whose truncation lies
    outside [0, O), or NaN, gives NaN.
  - ChangePoints weights: sigma(x) = 1 / (1 + exp(-s (x - x0))) and the reference's own 1 - sigma, evaluated exactly,
    against the device's fp64 chain (relative (2.01 |t| + 4.1) u on sigma, one rounding on 1 - sigma and on the
    product), rounded to T.  K = sum_i diag(a_i) K_i diag(a_i') then counts the roundings of scale_rows_ and
    scale_cols_ (one each) and of the accumulating axpby (one per term), all in T.

The NumPy emulations at the end evaluate leaf_value / kbuild_kernel's generic path, kdiag_kernel and kaux_eval in the
device's operation order; their named mutants are the defects the bars must catch."""
from __future__ import annotations

import types

import numpy as np

from gpflow_b200 import _lib
from tests import kbuild_bounds as KB

U64 = KB.U64
PI = np.pi                          # the double the kernels use (3.14159265358979323846 rounds to it)
S3, S5, C53 = np.sqrt(3.0), np.sqrt(5.0), 5.0 / 3.0
JIT = 1e-15
R_BASES = (_lib.K_EXPONENTIAL, _lib.K_MATERN12, _lib.K_MATERN32, _lib.K_MATERN52)   # bases with K_r
L = np.longdouble


# ---- descriptors ---------------------------------------------------------------------------------------------------
def params(kernel, D):
    """The descriptor of a materialised kernel as a plain namespace (Coregion's table from the host, no device)."""
    from gpflow_b200.kernels import materialised as M

    if isinstance(kernel, M.Coregion):
        dims = kernel._dims(D)
        return types.SimpleNamespace(op=_lib.KAUX_COREGION, dims=np.asarray(dims), table=kernel.output_covariance(),
                                     table_dim=int(kernel.output_dim))
    d = kernel._desc(D)
    n = d.n_dims
    return types.SimpleNamespace(op=d.op, base=d.base, order=d.order, variance=d.variance, alpha=d.alpha, bias=d.bias,
                                 dims=np.array(d.dims[:n]), scale=np.array(d.scale[:n]), period=np.array(d.period[:n]))


def _finish(cen, lo, hi, dtype):
    """The final rounding of the fp64 value to the dtype."""
    u = KB.unit(dtype) if np.dtype(dtype) == np.float32 else 0.0
    t = KB.tiny_abs(dtype)
    return cen, lo - u * np.abs(lo) - t, hi + u * np.abs(hi) + t


def _widen(lo, hi, e):
    m = e * np.maximum(np.abs(lo), np.abs(hi))
    return lo - m, hi + m


def _mul(al, ah, bl, bh):
    p = np.stack([al * bl, al * bh, ah * bl, ah * bh])
    return p.min(0), p.max(0)


def _trig_range(fn, lo, hi):
    """Range of sin / cos over [lo, hi] (elementwise), extrema inside the interval included."""
    a, b = fn(lo), fn(hi)
    rl, rh = np.minimum(a, b), np.maximum(a, b)
    shift = 0.0 if fn is np.cos else PI / 2           # cos(x) peaks at 2 k pi, sin(x) at pi / 2 + 2 k pi
    kmax = np.floor((hi - shift) / (2 * PI))
    has_max = kmax * 2 * PI + shift >= lo
    kmin = np.floor((hi - shift - PI) / (2 * PI))
    has_min = kmin * 2 * PI + shift + PI >= lo
    return np.where(has_min, -1.0, rl), np.where(has_max, 1.0, rh)


def _trig_ulp(lo, hi, name):
    return _widen(lo, hi, 2 * KB.ULP[name] * U64)


# ---- base kernels of Periodic --------------------------------------------------------------------------------------
def base_value(base, var, alpha, r):
    """base.K_r(r) / K_r2(r) in long double with the kernels' double constants."""
    r = np.asarray(r, L)
    v = L(var)
    if base == _lib.K_RBF:
        return v * np.exp(L(-0.5) * r)
    if base == _lib.K_RQ:
        return KB.rq_of_x(r, var, alpha)
    if base == _lib.K_EXPONENTIAL:
        return v * np.exp(L(-0.5) * r)
    if base == _lib.K_MATERN12:
        return v * np.exp(-r)
    if base == _lib.K_MATERN32:
        return v * (1 + L(S3) * r) * np.exp(-L(S3) * r)
    return v * (1 + L(S5) * r + L(C53) * r * r) * np.exp(-L(S5) * r)


BASE_BAR = {_lib.K_RBF: (3.02, 0.0), _lib.K_EXPONENTIAL: (3.02, 0.0), _lib.K_MATERN12: (3.02, 0.0),
            _lib.K_MATERN32: (7.5, 2.5), _lib.K_MATERN52: (10.5, 2.5)}


def base_interval(base, var, alpha, r, rlo, rhi):
    f = lambda t: np.asarray(base_value(base, var, alpha, t), np.float64)  # noqa: E731
    if base == _lib.K_RQ:
        amp = np.exp(2.01 * alpha * U64)
        e = (2 * KB.ULP["pow"] + 1.01) * U64
        return f(r), f(rhi) / amp * (1 - e), f(rlo) * amp * (1 + e)
    a, b = BASE_BAR[base]
    e = (a + b * rhi) * U64
    return f(r), f(rhi) * (1 - e) - 2.0 ** -1074, f(rlo) * (1 + e) + 2.0 ** -1074


# ---- intervals -----------------------------------------------------------------------------------------------------
def _pairs(p, X, X2):
    A = np.asarray(X, np.float64)[:, p.dims]
    B = A if X2 is None else np.asarray(X2, np.float64)[:, p.dims]
    return A, B


def cosine_interval(p, X, X2, dtype):
    A, B = _pairs(p, X, X2)
    diff = A.astype(L)[:, None, :] - B.astype(L)[None, :, :]
    terms = diff * p.scale.astype(L)
    s = terms.sum(-1)
    es = (len(p.dims) + 2) * 1.01 * U64 * np.asarray(np.abs(terms).sum(-1), np.float64)
    arg = np.asarray(2 * L(PI) * s, np.float64)
    e = 2 * PI * es + 1.01 * U64 * np.abs(arg) + 1e-300
    lo, hi = _trig_range(np.cos, arg - e, arg + e)
    lo, hi = _trig_ulp(lo, hi, "cos")
    lo, hi = _mul(lo, hi, p.variance, p.variance)
    lo, hi = _widen(lo, hi, U64)
    cen = np.asarray(L(p.variance) * np.cos(2 * L(PI) * s), np.float64)
    return _finish(cen, lo, hi, dtype)


def periodic_interval(p, X, X2, dtype):
    A, B = _pairs(p, X, X2)
    use_r = p.base in R_BASES
    n1, n2 = A.shape[0], B.shape[0]
    acc, alo, ahi = np.zeros((n1, n2), L), np.zeros((n1, n2)), np.zeros((n1, n2))
    for q in range(len(p.dims)):
        arg = L(PI) * (A[:, None, q].astype(L) - B[None, :, q].astype(L)) / L(p.period[q])
        sn = np.sin(arg) * L(p.scale[q])
        acc = acc + (np.abs(sn) if use_r else sn * sn)
        a = np.asarray(arg, np.float64)
        ea = 3.01 * U64 * np.abs(a)
        slo, shi = _trig_range(np.sin, a - ea, a + ea)
        slo, shi = _trig_ulp(slo, shi, "sin")
        slo, shi = _widen(slo * p.scale[q], shi * p.scale[q], U64)
        mlo = np.where((slo <= 0) & (shi >= 0), 0.0, np.minimum(np.abs(slo), np.abs(shi)))
        mhi = np.maximum(np.abs(slo), np.abs(shi))
        if not use_r:
            mlo, mhi = mlo * mlo * (1 - U64), mhi * mhi * (1 + U64)
        alo, ahi = (alo + mlo) * (1 - U64), (ahi + mhi) * (1 + U64)
    r = np.asarray(acc, np.float64)
    cen, lo, hi = base_interval(p.base, p.variance, p.alpha, r, np.maximum(alo, 0.0), ahi)
    return _finish(cen, lo, hi, dtype)


def arccos_J(order, theta):
    if order == 0:
        return PI - theta
    if order == 1:
        return np.sin(theta) + (PI - theta) * np.cos(theta)
    return 3.0 * np.sin(theta) * np.cos(theta) + (PI - theta) * (1.0 + 2.0 * np.cos(theta) ** 2)


J_TERMS = {0: 2 * PI, 1: 1 + PI, 2: 1.5 + 3 * PI}    # bounds on the sum of |terms| of J_n over [0, pi]


def arccos_interval(p, X, X2, dtype, tight_coincident=True):
    A, B = _pairs(p, X, X2)
    D = len(p.dims)
    w = p.scale
    AL, BL = A.astype(L), B.astype(L)
    num = L(p.bias) + (AL * w.astype(L)) @ BL.T
    na = L(p.bias) + (AL * AL) @ w.astype(L)
    nb = L(p.bias) + (BL * BL) @ w.astype(L)
    g = (D + 2) * 1.01 * U64
    nabs = p.bias + np.abs(A * w) @ np.abs(B).T
    n_, na_, nb_ = (np.asarray(t, np.float64) for t in (num, na, nb))
    nlo, nhi = n_ - g * nabs, n_ + g * nabs
    dal, dah = np.sqrt(na_ * (1 - g)) * (1 - U64), np.sqrt(na_ * (1 + g)) * (1 + U64)
    dbl, dbh = np.sqrt(nb_ * (1 - g)) * (1 - U64), np.sqrt(nb_ * (1 + g)) * (1 + U64)
    dal, dah, dbl, dbh = dal[:, None], dah[:, None], dbl[None, :], dbh[None, :]
    clo, chi = _mul(nlo, nhi, 1 / dah, 1 / dal)
    clo, chi = _widen(clo, chi, U64)
    clo, chi = _mul(clo, chi, 1 / dbh, 1 / dbl)
    clo, chi = _widen(clo, chi, U64)
    if tight_coincident:
        same = np.all(A[:, None, :] == B[None, :, :], axis=-1)
        clo, chi = np.where(same, 1 - 5 * U64, clo), np.where(same, 1 + 5 * U64, chi)
    k = 1.0 - 2.0 * JIT
    xlo, xhi = JIT + k * clo, JIT + k * chi
    xlo, xhi = _widen(xlo, xhi, 2.01 * U64)
    xlo, xhi = np.clip(xlo, -1.0, 1.0), np.clip(xhi, -1.0, 1.0)
    tlo, thi = np.arccos(xhi), np.arccos(xlo)
    e = 2 * KB.ULP["acos"] * U64
    tlo, thi = tlo * (1 - e), thi * (1 + e)
    eJ = 24 * U64 * J_TERMS[p.order]
    Jlo, Jhi = arccos_J(p.order, thi) - eJ, arccos_J(p.order, tlo) + eJ
    plo, phi = np.ones_like(Jlo), np.ones_like(Jhi)
    for _ in range(p.order):
        plo, phi = plo * dal * dbl * (1 - 2.01 * U64), phi * dah * dbh * (1 + 2.01 * U64)
    vp = p.variance * (1.0 / PI)
    lo, hi = _mul(Jlo, Jhi, plo, phi)
    lo, hi = _widen(lo * vp, hi * vp, 3.01 * U64)
    c = num / np.sqrt(na)[:, None] / np.sqrt(nb)[None, :]
    th = np.arccos(L(JIT) + L(k) * c)
    pw = (np.sqrt(na)[:, None] * np.sqrt(nb)[None, :]) ** p.order
    cen = np.asarray(L(vp) * arccos_J(p.order, th) * pw, np.float64)
    return _finish(cen, lo, hi, dtype)


def coregion_index(x, table_dim):
    """tf.cast(x, tf.int32) toward zero; -1 for an index that is NaN or outside [0, table_dim)."""
    x = np.asarray(x, np.float64)
    ok = (x > -1.0) & (x < table_dim)
    return np.where(ok, np.trunc(np.where(ok, x, 0.0)), -1).astype(np.int64)


def coregion_value(p, X, X2, dtype):
    """The exact device result: T(B[i, j]), NaN for an invalid index."""
    A, B = _pairs(p, X, X2)
    i, j = coregion_index(A[:, 0], p.table_dim), coregion_index(B[:, 0], p.table_dim)
    v = p.table[np.maximum(i, 0)[:, None], np.maximum(j, 0)[None, :]]
    v = np.where((i[:, None] >= 0) & (j[None, :] >= 0), v, np.nan)
    return v.astype(dtype)


def kaux_interval(p, X, X2, dtype):
    """(center, lo, hi) of gpk_kaux's K(X, X2) (X2=None: the symmetric form; the values are the same)."""
    if p.op == _lib.KAUX_COSINE:
        return cosine_interval(p, X, X2, dtype)
    if p.op == _lib.KAUX_PERIODIC:
        return periodic_interval(p, X, X2, dtype)
    if p.op == _lib.KAUX_ARCCOS:
        return arccos_interval(p, X, X2, dtype)
    v = coregion_value(p, X, X2, dtype).astype(np.float64)
    return v, v, v


def kaux_diag_interval(p, X, dtype):
    """gpk_kaux_diag: the variance (Cosine, Periodic), var / pi J_n(0) |x|^(2n) (ArcCosine), B[i, i] (Coregion)."""
    X = np.asarray(X, np.float64)
    if p.op == _lib.KAUX_COREGION:
        i = coregion_index(X[:, p.dims[0]], p.table_dim)
        v = np.where(i >= 0, np.diag(p.table)[np.maximum(i, 0)], np.nan).astype(dtype).astype(np.float64)
        return v, v, v
    if p.op != _lib.KAUX_ARCCOS:
        v = p.variance if p.op == _lib.KAUX_COSINE else float(base_value(p.base, p.variance, p.alpha, 0.0))
        v = np.full(X.shape[0], np.dtype(dtype).type(v), np.float64)
        return v, v, v
    A = X[:, p.dims]
    na = L(p.bias) + (A.astype(L) ** 2) @ p.scale.astype(L)
    n_ = np.asarray(na, np.float64)
    g = (len(p.dims) + 2) * 1.01 * U64
    vp = p.variance * (1.0 / PI) * arccos_J(p.order, 0.0)
    cen = np.asarray(L(vp) * na ** p.order, np.float64)
    lo, hi = vp * (n_ * (1 - g)) ** p.order, vp * (n_ * (1 + g)) ** p.order
    lo, hi = _widen(lo, hi, (p.order + 4.01) * U64)
    return _finish(cen, lo, hi, dtype)


# ---- ChangePoints ----------------------------------------------------------------------------------------------------
def sigmoid_exact(x, loc, steep):
    return 1 / (1 + np.exp(-L(steep) * (np.asarray(x, L) - L(loc))))


def cp_weight_interval(x, has_lo, loc_lo, steep_lo, has_hi, loc_hi, steep_hi, dtype):
    """(center, lo, hi) of cp_weights_kernel: sig_lo(x) (1 - sig_hi(x)) in fp64, rounded to T."""
    x = np.asarray(x, np.float64)
    cen = np.ones(x.shape, L)
    lo, hi = np.ones(x.shape), np.ones(x.shape)
    for on, loc, st, upper in ((has_lo, loc_lo, steep_lo, False), (has_hi, loc_hi, steep_hi, True)):
        if not on:
            continue
        s = sigmoid_exact(x, loc, st)
        t = np.abs(st * (x - loc))
        d = (2.01 * t + 4.1) * U64
        sv = np.asarray(s, np.float64)
        slo, shi = sv * (1 - d), np.minimum(sv * (1 + d), 1.0)
        if upper:
            s = 1 - s
            slo, shi = _widen(1 - shi, 1 - slo, U64)
        cen = cen * s
        lo, hi = _mul(lo, hi, slo, shi)
        lo, hi = _widen(lo, hi, U64)
    return _finish(np.asarray(cen, np.float64), lo, hi, dtype)


def cp_weight_args(locs, steeps, i):
    """has_lo, loc_lo, steep_lo, has_hi, loc_hi, steep_hi of kernel i, as ChangePoints._weights passes them."""
    n = len(locs)
    return (int(i > 0), float(locs[i - 1]) if i > 0 else 0.0, float(steeps[i - 1]) if i > 0 else 1.0,
            int(i < n), float(locs[i]) if i < n else 0.0, float(steeps[i]) if i < n else 1.0)


def scaled_sum_interval(parts, dtype, diag=False):
    """sum_i a_i K_i a'_i from (a, a', (cen, lo, hi) of K_i) per term: scale_rows_, scale_cols_, accumulating axpby.
    diag: K_i is a column [N, 1] and a' scales its rows again (K_diag)."""
    u = KB.unit(dtype)
    acc = None
    for (ac, al, ah), (bc, bl, bh), (kc, kl, kh) in parts:
        col = (slice(None), None) if diag else (None, slice(None))
        cen = ac[:, None] * kc * bc[col]
        lo, hi = _mul(kl, kh, al[:, None], ah[:, None])
        lo, hi = _widen(lo, hi, u)
        lo, hi = _mul(lo, hi, bl[col], bh[col])
        lo, hi = _widen(lo, hi, u)
        if acc is None:
            acc = cen, lo, hi
        else:
            acc = KB.combine(_lib.K_SUM, [acc, (cen, lo, hi)], u)
    return acc


# ---- public kernels, composed as the Python layer composes them ----------------------------------------------------
def kernel_interval(kernel, X, X2, dtype, full_cov=True):
    """(center, lo, hi) of kernel(X, X2) or kernel(X, full_cov=False) through the public K / K_diag: fused expressions,
    materialised leaves, Sum / Product with materialised children (axpby / hadamard_) and ChangePoints."""
    from gpflow_b200 import kernels as K
    from gpflow_b200.kernels import materialised as M

    D = np.asarray(X).shape[1]
    u = KB.unit(dtype)
    if kernel.is_fusable():
        desc = K.compile_kernel(kernel, D)
        return KB.expr_interval(desc, X, X2, dtype=dtype) if full_cov else KB.kdiag_interval(desc, X, dtype)
    if isinstance(kernel, M.ChangePoints):
        locs = np.asarray(kernel.locations.numpy(), np.float64).reshape(-1)
        st = np.asarray(kernel.steepness.numpy(), np.float64).reshape(-1)
        st = np.full(len(locs), float(st[0])) if st.size == 1 else st
        parts = []
        for i, k in enumerate(kernel.kernels):
            args = cp_weight_args(locs, st, i)
            a = cp_weight_interval(np.asarray(X, np.float64)[:, 0], *args, dtype)
            if full_cov:
                b = a if X2 is None else cp_weight_interval(np.asarray(X2, np.float64)[:, 0], *args, dtype)
                parts.append((a, b, kernel_interval(k, X, X2, dtype)))
            else:
                kc, kl, kh = kernel_interval(k, X, None, dtype, full_cov=False)
                parts.append((a, a, (kc[:, None], kl[:, None], kh[:, None])))
        cen, lo, hi = scaled_sum_interval(parts, dtype, diag=not full_cov)
        return (cen, lo, hi) if full_cov else (cen[:, 0], lo[:, 0], hi[:, 0])
    if isinstance(kernel, M._Materialised):
        p = params(kernel, D)
        return kaux_interval(p, X, X2, dtype) if full_cov else kaux_diag_interval(p, X, dtype)
    # Sum / Product with a materialised child: materialised children first, the fused ones as one group last
    fus = [k for k in kernel.kernels if k.is_fusable()]
    kids = [kernel_interval(k, X, X2, dtype, full_cov) for k in kernel.kernels if not k.is_fusable()]
    if fus:
        grp = fus[0] if len(fus) == 1 else kernel.__class__(fus)
        kids.append(kernel_interval(grp, X, X2, dtype, full_cov))
    return KB.combine(kernel._op, kids, u)


# ---- emulations of the device's operation order, with named mutants --------------------------------------------------
def _fma(a, b, c, T):
    return T(np.float64(a) * np.float64(b) + np.float64(c)) if T is np.float32 else T(a * b + c)


def emulate_kbuild(desc, X, X2=None, dtype=np.float64, mutant=None, sym=None):
    """kbuild_kernel's generic path in the dtype: staged weighted inputs, sequential fma norms and dots, leaf_value and
    the postfix fold.  mutant in {"rq_no_half", "poly_no_offset", "poly_offset_after", "white_rect"}."""
    nodes, n_nodes, dims, ard = desc
    T = np.dtype(dtype).type
    sym = X2 is None if sym is None else sym
    X = np.asarray(X, T)
    X2 = X if X2 is None else np.asarray(X2, T)
    D = X.shape[1]
    n1, n2 = X.shape[0], X2.shape[0]

    def leaf(nd):
        var, alpha = T(nd.variance), T(nd.alpha)
        if nd.op == _lib.K_CONSTANT:
            return np.full((n1, n2), var)
        if nd.op == _lib.K_WHITE:
            on = (sym or mutant == "white_rect") & (np.arange(n1)[:, None] == np.arange(n2)[None, :])
            return np.where(on, var, T(0))
        cols, par = KB._leaf_inputs(nd, dims, ard, D)
        lin = nd.op in (_lib.K_LINEAR, _lib.K_POLYNOMIAL)
        scale = T(1.0)
        if nd.n_ard > 0:
            w = par if lin else 1.0 / par
            if lin:
                var = T(1.0)
        else:
            w = np.ones(len(cols))
            if not lin:
                scale = T(1.0 / (nd.lengthscale * nd.lengthscale))
        w = w.astype(T)
        A = X[:, cols] * w
        B = X2[:, cols] * w if (nd.n_ard > 0 and not lin) else X2[:, cols]
        dot, na, nb = np.zeros((n1, n2), T), np.zeros(n1, T), np.zeros(n2, T)
        for d in range(len(cols)):
            dot = _fma(A[:, None, d], B[None, :, d], dot, T)
            na, nb = _fma(A[:, d], A[:, d], na, T), _fma(B[:, d], B[:, d], nb, T)
        if nd.op == _lib.K_LINEAR:
            return var * dot
        if nd.op == _lib.K_POLYNOMIAL:
            off = T(nd.lengthscale)
            if mutant == "poly_no_offset":
                return np.power(var * dot, alpha)
            if mutant == "poly_offset_after":
                return np.power(var * dot, alpha) + off
            return np.power(var * dot + off, alpha)
        r2 = scale * (na[:, None] + nb[None, :] - T(2) * dot)
        if nd.op == _lib.K_RQ:
            h = r2 / alpha if mutant == "rq_no_half" else T(0.5) * r2 / alpha
            return var * np.power(T(1) + h, -alpha)
        if nd.op == _lib.K_RBF:
            return var * np.exp(T(-0.5) * r2)
        r = np.sqrt(np.maximum(r2, T(1e-36)))
        if nd.op == _lib.K_MATERN52:
            s5 = T(S5)
            return var * (T(1) + s5 * r + T(C53) * r * r) * np.exp(-s5 * r)
        if nd.op == _lib.K_MATERN32:
            s3 = T(S3)
            return var * (T(1) + s3 * r) * np.exp(-s3 * r)
        if nd.op == _lib.K_MATERN12:
            return var * np.exp(-r)
        return var * np.exp(T(-0.5) * r)

    def rec(i):
        nd = nodes[i]
        if nd.op in (_lib.K_SUM, _lib.K_PRODUCT):
            acc = rec(nd.child[0])
            for c in range(1, nd.n_children):
                k = rec(nd.child[c])
                acc = acc + k if nd.op == _lib.K_SUM else acc * k
            return acc
        return leaf(nd)

    with np.errstate(all="ignore"):
        return rec(n_nodes - 1)


def emulate_kdiag(desc, X, dtype=np.float64, mutant=None):
    """kdiag_kernel in the dtype; mutant "ard_squared" squares the ARD weight."""
    nodes, n_nodes, dims, ard = desc
    T = np.dtype(dtype).type
    X = np.asarray(X, T)

    def rec(i):
        nd = nodes[i]
        if nd.op in (_lib.K_SUM, _lib.K_PRODUCT):
            acc = rec(nd.child[0])
            for c in range(1, nd.n_children):
                acc = acc + rec(nd.child[c]) if nd.op == _lib.K_SUM else acc * rec(nd.child[c])
            return acc
        v = np.full(X.shape[0], T(nd.variance))
        if nd.op in (_lib.K_LINEAR, _lib.K_POLYNOMIAL):
            cols, par = KB._leaf_inputs(nd, dims, ard, X.shape[1])
            w = (par if nd.n_ard > 0 else np.ones(len(cols))).astype(T)
            if nd.n_ard > 0:
                v = np.full(X.shape[0], T(1))
            acc = np.zeros(X.shape[0], T)
            for d, c in enumerate(cols):
                wd = w[d] * w[d] if mutant == "ard_squared" else w[d]
                acc = acc + wd * X[:, c] * X[:, c]
            v = v * acc
            if nd.op == _lib.K_POLYNOMIAL:
                v = np.power(v + T(nd.lengthscale), T(nd.alpha))
        return v

    return rec(n_nodes - 1)


def emulate_kaux(p, X, X2=None, dtype=np.float64, mutant=None):
    """kaux_eval / the Coregion lookup in fp64, rounded to the dtype.  mutant in {"periodic_sin2", "arccos_no_jitter",
    "coregion_nearest", "in_float" (the arithmetic in fp32), "cosine_no_2"}."""
    W = np.float32 if mutant == "in_float" else np.float64
    A, B = _pairs(p, X, X2)
    A, B = A.astype(W), B.astype(W)
    pi = W(PI)
    with np.errstate(all="ignore"):
        if p.op == _lib.KAUX_COREGION:
            if mutant == "coregion_nearest":
                i, j = np.rint(A[:, 0]).astype(np.int64), np.rint(B[:, 0]).astype(np.int64)
                ok = (i[:, None] >= 0) & (i[:, None] < p.table_dim) & (j[None, :] >= 0) & (j[None, :] < p.table_dim)
                v = np.where(ok, p.table[np.clip(i, 0, p.table_dim - 1)[:, None], np.clip(j, 0, p.table_dim - 1)[None, :]],
                             np.nan)
                return v.astype(dtype)
            return coregion_value(p, X, X2, dtype)
        if p.op == _lib.KAUX_COSINE:
            s = np.zeros((A.shape[0], B.shape[0]), W)
            for q in range(len(p.dims)):
                s = s + (A[:, None, q] - B[None, :, q]) * W(p.scale[q])
            v = W(p.variance) * np.cos((pi if mutant == "cosine_no_2" else W(2.0) * pi) * s)
            return v.astype(dtype)
        if p.op == _lib.KAUX_PERIODIC:
            use_r = p.base in R_BASES and mutant != "periodic_sin2"
            acc = np.zeros((A.shape[0], B.shape[0]), W)
            for q in range(len(p.dims)):
                sn = np.sin(pi * (A[:, None, q] - B[None, :, q]) / W(p.period[q])) * W(p.scale[q])
                acc = acc + (np.abs(sn) if use_r else sn * sn)
            return _base_emulated(p.base, W(p.variance), W(p.alpha), acc, W).astype(dtype)
        num = np.full((A.shape[0], B.shape[0]), W(p.bias))
        na, nb = np.full(A.shape[0], W(p.bias)), np.full(B.shape[0], W(p.bias))
        for q in range(len(p.dims)):
            w = W(p.scale[q])
            num = num + w * A[:, None, q] * B[None, :, q]
            na, nb = na + w * A[:, q] * A[:, q], nb + w * B[:, q] * B[:, q]
        da, db = np.sqrt(na), np.sqrt(nb)
        c = num / da[:, None] / db[None, :]
        jit = W(0.0) if mutant == "arccos_no_jitter" else W(JIT)
        theta = np.arccos(jit + (W(1.0) - W(2.0) * jit) * c)
        pw = np.ones_like(theta)
        for _ in range(p.order):
            pw = pw * (da[:, None] * db[None, :])
        return (W(p.variance) * (W(1.0) / pi) * arccos_J(p.order, theta).astype(W) * pw).astype(dtype)


def _base_emulated(base, var, alpha, r, W):
    if base == _lib.K_RBF:
        return var * np.exp(W(-0.5) * r)
    if base == _lib.K_RQ:
        return var * np.power(W(1.0) + W(0.5) * r / alpha, -alpha)
    if base == _lib.K_EXPONENTIAL:
        return var * np.exp(W(-0.5) * r)
    if base == _lib.K_MATERN12:
        return var * np.exp(-r)
    if base == _lib.K_MATERN32:
        return var * (W(1.0) + W(S3) * r) * np.exp(-W(S3) * r)
    return var * (W(1.0) + W(S5) * r + W(C53) * r * r) * np.exp(-W(S5) * r)


def emulate_changepoints(kernel, X, X2, dtype, mutant=None):
    """ChangePoints._materialise in the dtype with the children's exact intervals' centers rounded to T as K_i;
    mutant "x_weights_on_cols" scales X2's columns by X's weights."""
    T = np.dtype(dtype).type
    locs = np.asarray(kernel.locations.numpy(), np.float64).reshape(-1)
    st = np.asarray(kernel.steepness.numpy(), np.float64).reshape(-1)
    st = np.full(len(locs), float(st[0])) if st.size == 1 else st
    acc = None
    for i, k in enumerate(kernel.kernels):
        args = cp_weight_args(locs, st, i)
        a = _cp_weight_emulated(np.asarray(X, np.float64)[:, 0], *args).astype(T)
        b = a if (X2 is None or mutant == "x_weights_on_cols") else \
            _cp_weight_emulated(np.asarray(X2, np.float64)[:, 0], *args).astype(T)
        Ki = kernel_interval(k, X, X2, dtype)[0].astype(T)
        if mutant == "x_weights_on_cols" and X2 is not None:
            b = np.resize(a, len(np.asarray(X2)))
        Ki = (Ki * a[:, None]) * b[None, :]
        acc = Ki if acc is None else Ki + acc
    return acc


def _cp_weight_emulated(x, has_lo, loc_lo, steep_lo, has_hi, loc_hi, steep_hi):
    w = np.ones_like(x)
    if has_lo:
        w = w * (1.0 / (1.0 + np.exp(-steep_lo * (x - loc_lo))))
    if has_hi:
        w = w * (1.0 - 1.0 / (1.0 + np.exp(-steep_hi * (x - loc_hi))))
    return w
