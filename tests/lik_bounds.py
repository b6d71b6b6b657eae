"""Exact references and per-element error bars for the likelihood kernels (csrc/lik.cu), CPU only.

Oracle.  mpmath at 113 bits evaluates the same 20-point sums the device evaluates: the committed node / weight table
(`lik_oracle.cuda_gh_table()`) and the stored inputs taken as exact doubles, every constant (1/sqrt 2, the 1e-3 probit
jitter, 1/sqrt(2 pi), log pi, ...) as the exact real the source names.  Targets: per element the variational
expectation, d/dmu, d/dv and d/d(likelihood parameter); the predictive mean / variance and log density; for MultiClass
p, VE, R_c, W_c, R_y, W_y, dVE/deps and the predictions, with the 1e-10 clamps and the label rules of
tests/multiclass_oracle.py.  At v = 0 the d/dv target of a quadrature likelihood is the limit of the derivative of the
20-point sum, g''(mu) sum_k w_k z_k^2 / 2 (the device takes sum_k w_k z_k^2 = 1; the bar carries the difference).

Bars: a running error analysis of the kernel's own operation order.  `Err` carries a value and a bound on its distance
from the exact real, and every operation adds the propagated input errors (first order in the inputs' bars, exact
for + and -) and its own rounding:
  - + - * / fma sqrt correctly rounded: u |result| (fma also u |a b|, so one bar covers a fused and an unfused fma);
  - the CUDA Math API's maximum errors for double: exp 1, log 1, erf 2, lgamma (x > 0) 4, rsqrt 1 ulp, 1 ulp <= 2u |x|,
    plus 2^-1074 for results in the subnormal range; a function's input error enters through a bound on its
    derivative over the input's interval;
  - a compile-time constant (1/sqrt 2, 1 - 2e-3, ...) is the nearest double: u relative to the real it names.
So node placement f_k = fma(sqrt v, z_k, mu) contributes |g'(f_k)| (|sqrt(v) z_k| + |f_k|) u per node through the
function that consumes it, the function error is measured against absolute term sizes (Poisson's VE bar scales with
|y mu| + e + lgamma(y + 1), not with |VE|), and a 20-term fma sum adds u per term to sum_k w_k |term_k| (at most
gamma_20 sum_k w_k |term_k|).  d/dv = dz / (2 sqrt v) with dz = sum_k w_k g_k z_k: that sum cancels (the table is
symmetric), and its bar, divided by 2 sqrt v, is carried in full.  The reference's autodiff forms the same sum, so at
v = 1e-300 the 20-point derivative is itself meaningless to about 1e-16 |g'(mu)| / sqrt(v); the bar says so.
MultiClass products: the relative bar of each cdf factor adds, plus one u per multiplication (C - 1 + the chunk totals +
the scan's depth, all counted by the running analysis).  The warp and block sums of a VE or dpar sum over n terms in an
unknown order add (n - 1) u sum |term|.

fp32 storage: the operators compute in fp64 from the rounded inputs and round once, so an fp32 output's bar is half an
fp32 ulp of the result plus the fp64 bar at the rounded inputs; the sums (fp64 outputs) keep the fp64 bar.

The same code, run on float64 NumPy values in the kernel's operation order, is the emulation tests/test_lik_bounds.py
holds inside every bar (and whose mutants it shows outside).  First-order terms are exact for the operations here up to
O(u^2) relative, which a factor 2 on every bar (`SAFETY`) covers.
"""
from __future__ import annotations

import contextlib
import math
from fractions import Fraction
from typing import Dict, List, Tuple

import mpmath
import numpy as np
from scipy.special import digamma, erf, gammaln

from tests import lik_oracle as LO

U = 2.0 ** -53
TINY = 2.0 ** -1074
SAFETY = 2.0
ULP = {"exp": 1, "log": 1, "erf": 2, "lgamma": 4, "rsqrt": 1}
PREC = 113

GH_Z, GH_W = LO.cuda_gh_table()
# |sum_k w_k z_k^2 - 1| of the committed table, exactly; the v = 0 limit of the device takes the sum as 1
S2_EXCESS = abs(float(sum(Fraction(w) * Fraction(z) ** 2 for z, w in zip(GH_Z, GH_W)) - 1))

SQRT1_2 = 0.70710678118654752440
RSQRT2PI = 0.39894228040143267794
LOG2PI = 1.8378770664093454835606594728112
LOGPI = 1.1447298858494001741434273513531
JIT = 1e-3          # inv_probit's jitter
SQUASH = 1e-6       # RobustMax._squash


_ARITH = [None]   # None: fp64 arithmetic; np.float32: every result rounded to fp32 (a mutant of the operators)


@contextlib.contextmanager
def arithmetic(dtype):
    """Run the emulation with every operation's result rounded to `dtype`."""
    _ARITH[0] = dtype
    try:
        yield
    finally:
        _ARITH[0] = None


def _c(v):
    return v if _ARITH[0] is None else np.asarray(v).astype(_ARITH[0])


def _ulp(x):
    return 2.0 * U * np.abs(x) + TINY


class Err:
    """A computed value and a bound on its distance from the exact real it stands for."""
    __slots__ = ("v", "e")
    __array_ufunc__ = None   # ndarray op Err defers to Err

    def __init__(self, v, e=None):
        self.v = np.asarray(v)
        self.e = np.zeros(self.v.shape) if e is None else np.asarray(e)

    @staticmethod
    def const(c, exact=False):
        """A literal: the nearest double to the real it names (exact: the literal is the real)."""
        return Err(np.float64(c), 0.0 if exact else U * abs(c))

    def _w(self, o):
        return o if isinstance(o, Err) else Err(o)   # plain numbers are exact

    def _r(self, v, e):
        return Err(_c(v), e + U * np.abs(v) + TINY)

    def __add__(self, o):
        o = self._w(o)
        return self._r(self.v + o.v, self.e + o.e)

    __radd__ = __add__

    def __sub__(self, o):
        o = self._w(o)
        return self._r(self.v - o.v, self.e + o.e)

    def __rsub__(self, o):
        return self._w(o) - self

    def __neg__(self):
        return Err(-self.v, self.e)

    def __mul__(self, o):
        o = self._w(o)
        return self._r(self.v * o.v, np.abs(o.v) * self.e + np.abs(self.v) * o.e + self.e * o.e)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = self._w(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            q = self.v / o.v
            den = np.maximum(np.abs(o.v) - o.e, 0.0)
            e = np.where(self.e + o.e == 0, 0.0, (self.e + np.abs(q) * o.e) / den)
        return self._r(q, e)

    def __rtruediv__(self, o):
        return self._w(o) / self

    def fma(self, b, c):
        """self * b + c in one rounding (bar also valid for two roundings)."""
        b, c = self._w(b), self._w(c)
        ab = self.v * b.v
        v = ab + c.v
        return Err(_c(v), np.abs(b.v) * self.e + np.abs(self.v) * b.e + self.e * b.e + c.e + U * np.abs(ab) +
                   U * np.abs(v) + 2 * TINY)


def where(cond, a: Err, b: Err) -> Err:
    a, b = (x if isinstance(x, Err) else Err(x) for x in (a, b))
    return Err(np.where(cond, a.v, b.v), np.where(cond, a.e, b.e))


def sqrt(a: Err) -> Err:
    v = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(a.e == 0, 0.0, a.e / (v + np.sqrt(np.maximum(a.v - a.e, 0.0))))
        e = np.where(np.isfinite(e), e, np.sqrt(a.e))
    return Err(_c(v), e + U * np.abs(v) + TINY)


def rsqrt(a: Err) -> Err:
    v = 1.0 / np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(a.e == 0, 0.0, 0.5 * np.abs(v) * a.e / np.maximum(a.v - a.e, 0.0))
    return Err(_c(v), e + ULP["rsqrt"] * _ulp(v))


def exp(a: Err) -> Err:
    with np.errstate(over="ignore", invalid="ignore"):
        v = np.exp(a.v)
        e = np.exp(a.v + a.e) - np.exp(a.v)
        e = np.where(a.e == 0, 0.0, e)
    return Err(_c(v), e + ULP["exp"] * _ulp(v))


def log(a: Err) -> Err:
    with np.errstate(divide="ignore", invalid="ignore"):
        v = np.log(a.v)
        e = np.where(a.e == 0, 0.0, a.e / np.maximum(np.abs(a.v) - a.e, 0.0))
    return Err(_c(v), e + ULP["log"] * _ulp(v))


def erf_(a: Err) -> Err:
    v = erf(a.v)
    lo = np.maximum(np.abs(a.v) - a.e, 0.0)
    return Err(_c(v), 2.0 / math.sqrt(math.pi) * np.exp(-lo * lo) * a.e + ULP["erf"] * _ulp(v))


def lgamma(a: Err) -> Err:
    """lgamma(x), x > 0."""
    v = gammaln(a.v)
    hi = np.abs(a.v) + a.e
    dg = np.maximum(np.abs(digamma(np.maximum(a.v - a.e, 1e-300))), np.abs(digamma(hi)))
    return Err(_c(v), dg * a.e + ULP["lgamma"] * _ulp(v))


def bar(x: Err):
    return SAFETY * x.e


def round32_bar(exact, bar64):
    """The bar of a fp64 result rounded once to fp32."""
    m = np.abs(exact) + bar64
    return bar64 + 0.5 * np.where(m >= 2.0 ** -126, 2.0 ** (np.floor(np.log2(np.maximum(m, 1e-300))) - 23), 2.0 ** -149)


# ==== scalar likelihoods ===========================================================================================
SCALAR_KINDS = ("gaussian", "bernoulli", "poisson", "student_t")
TYPE = {"gaussian": 0, "bernoulli": 1, "poisson": 2, "student_t": 3}


def c0(kind: str, par: Dict[str, float]) -> Err:
    """lik_prepare's host constant (glibc's log / lgamma held to the same budget as the device's)."""
    if kind == "gaussian":
        return Err.const(-0.5 * LOG2PI) - 0.5 * log(Err(par["noise"]))
    if kind == "poisson":
        return log(Err(par["binsize"]))
    if kind == "student_t":
        s, df = Err(par["scale"]), Err(par["df"])
        return (lgamma(0.5 * (df + 1.0)) - lgamma(0.5 * df)) - 0.5 * ((log(s * s) + log(df)) + Err.const(LOGPI))
    return Err(0.0)


def _inv_probit(f: Err) -> Err:
    return (0.5 * (1.0 + erf_(f * Err.const(SQRT1_2)))) * Err.const(1.0 - 2e-3) + Err.const(JIT)


def _dphi(f: Err) -> Err:
    """(1 - 2 jitter) phi(f); the compiler folds the two constants into one."""
    c = Err(np.float64((1.0 - 2e-3) * RSQRT2PI), 3 * U * (1.0 - 2e-3) * RSQRT2PI)
    return c * exp((-0.5 * f) * f)


def logp(kind, par, c, y, f: Err) -> Err:
    if kind == "bernoulli":
        p = _inv_probit(f)
        return where(y == 1.0, log(p), log(1.0 - p))
    if kind == "poisson":
        lam = exp(f) * par["binsize"]
        return (y * log(lam) - lam) - lgamma(Err(y + 1.0))
    if kind == "student_t":
        r = (y - f) / par["scale"]
        return c - (0.5 * (par["df"] + 1.0)) * log(1.0 + (r * r) / par["df"])
    r = y - f
    return c - (0.5 * (r * r)) / par["noise"]


def dlogp(kind, par, y, f: Err, mutation=None) -> Tuple[Err, Err]:
    if kind == "bernoulli":
        p, dp = _inv_probit(f), _dphi(f)
        return where(y == 1.0, dp / p, -(dp / (1.0 - p))), Err(np.zeros(np.shape(f.v)))
    if kind == "poisson":
        return y - exp(f) * par["binsize"], Err(np.zeros(np.shape(f.v)))
    if kind == "student_t":
        s, df = par["scale"], par["df"]
        r = y - f
        s2df = (Err(s) * s) * df
        q = s2df + r * r
        ds = (((df + 1.0) * r) * r) / (s * q)
        if mutation != "dscale_no_inv_scale":
            ds = (-1.0 / Err(s)) + ds
        return ((df + 1.0) * r) / q, ds
    return (y - f) / par["noise"], Err(np.zeros(np.shape(f.v)))


def d2logp(kind, par, y, f: Err) -> Err:
    if kind == "bernoulli":
        p, dp = _inv_probit(f), _dphi(f)
        a1, a0 = dp / p, dp / (1.0 - p)
        return where(y == 1.0, -a1 * (f + a1), a0 * (f - a0))
    s, df = par["scale"], par["df"]   # Student-t
    r = y - f
    s2df = (Err(s) * s) * df
    q = s2df + r * r
    return ((df + 1.0) * (r * r - s2df)) / (q * q)


def scalar_ve(kind: str, par: Dict[str, float], y, mu, v, *, grad=True, table=None, mutation=None):
    """lik_ve<GRAD> on arrays of elements: {"ve", "dmu", "dv", "dpar"} as Err."""
    y, mu_e, v_e = np.asarray(y), Err(mu), Err(v)
    c = c0(kind, par)
    zero = Err(np.zeros(np.shape(mu_e.v)))
    if kind == "gaussian":
        s = par["noise"]
        r = y - mu_e
        rv = r * r + v_e
        return {"ve": c - (0.5 * rv) / s, "dmu": r / s, "dv": Err(np.full(np.shape(mu_e.v), -0.5 / s)),
                "dpar": -0.5 / Err(s) + (0.5 * rv) / (Err(s) * s)}
    if kind == "poisson":
        e = exp(mu_e + 0.5 * v_e) * par["binsize"]
        return {"ve": (((y * mu_e) - e) - lgamma(Err(y + 1.0))) + y * c, "dmu": y - e, "dv": -0.5 * e,
                "dpar": zero}
    Z, W = (GH_Z, GH_W) if table is None else table
    sd = sqrt(v_e)
    ve, dmu, dz, dpar = zero, zero, zero, zero
    for k in range(len(Z)):
        f = sd.fma(Z[k], mu_e)
        wk = W[k]
        if grad:
            g1, ds = dlogp(kind, par, y, f, mutation)
            dmu = Err(wk).fma(g1, dmu)
            dz = (wk * g1).fma(Z[k], dz)
            dpar = Err(wk).fma(ds, dpar)
        ve = Err(wk).fma(logp(kind, par, c, y, f), ve)
    out = {"ve": ve, "dmu": dmu, "dz": dz, "dpar": dpar}
    if grad:
        two = 1.0 if mutation == "dv_no_half" else 2.0
        with np.errstate(divide="ignore", invalid="ignore"):
            dv_q = dz / (two * sd)
        lim = 0.5 * d2logp(kind, par, y, mu_e)
        lim = Err(lim.v, lim.e + 0.5 * np.abs(lim.v) * S2_EXCESS)
        out["dv"] = where(v_e.v > 0.0, dv_q, lim) if mutation != "no_v0_limit" else dv_q
    return out


def scalar_predict_mv(kind, par, mu, v) -> Tuple[Err, Err]:
    """lik_predict_mv_kernel's arithmetic on the stored inputs."""
    mu_e, v_e = Err(np.asarray(mu, np.float64)), Err(np.asarray(v, np.float64))
    if kind == "gaussian":
        return mu_e, v_e + par["noise"]
    if kind == "bernoulli":
        p = _inv_probit(mu_e / sqrt(1.0 + v_e))
        return p, p - p * p
    sd = sqrt(v_e)
    cvar = (Err(par["scale"]) * par["scale"]) * (Err(par["df"]) / (Err(par["df"]) - 2.0)) \
        if kind == "student_t" else None
    ey = ey2 = Err(np.zeros(np.shape(mu_e.v)))
    for k in range(20):
        f = sd.fma(GH_Z[k], mu_e)
        if kind == "poisson":
            cm = exp(f) * par["binsize"]
            cv = cm
        else:
            cm, cv = f, cvar
        ey = Err(GH_W[k]).fma(cm, ey)
        ey2 = Err(GH_W[k]).fma(cv + cm * cm, ey2)
    return ey, ey2 - ey * ey


def scalar_predict_ld(kind, par, y, mu, v) -> Err:
    """lik_predict_ld_kernel's per-element term (the kernel sums them over a row)."""
    y, mu_e, v_e = np.asarray(y, np.float64), Err(np.asarray(mu, np.float64)), Err(np.asarray(v, np.float64))
    if kind == "gaussian":
        tv = v_e + par["noise"]
        r = y - mu_e
        return -0.5 * ((Err.const(LOG2PI) + log(tv)) + (r * r) / tv)
    if kind == "bernoulli":
        pr = _inv_probit(mu_e / sqrt(1.0 + v_e))
        return log(where(y == 1.0, pr, 1.0 - pr))
    c = c0(kind, par)
    sd = sqrt(v_e)
    gmax = se = None
    for k in range(20):
        g = logp(kind, par, c, y, sd.fma(GH_Z[k], mu_e)) + log(Err(GH_W[k]))
        if gmax is None:
            gmax, se = g, Err(np.ones(np.shape(g.v)))
            continue
        up = g.v > gmax.v
        se_up = se.fma(exp(gmax - g), 1.0)
        se_dn = se + exp(g - gmax)
        se, gmax = where(up, se_up, se_dn), where(up, g, gmax)
    return gmax + log(se)


# ---- the exact scalar references ----------------------------------------------------------------------------------
def _mp_logp_terms(kind, par, y, f):
    """(log p, g', d/dpar log p) at f, exact."""
    mp = mpmath
    if kind == "bernoulli":
        J = mp.mpf("0.001")
        p = (1 + mp.erf(f / mp.sqrt(2))) / 2 * (1 - 2 * J) + J
        dp = (1 - 2 * J) * mp.exp(-f * f / 2) / mp.sqrt(2 * mp.pi)
        if y == 1:
            return mp.log(p), dp / p, mp.mpf(0)
        return mp.log(1 - p), -dp / (1 - p), mp.mpf(0)
    if kind == "poisson":
        lam = mp.exp(f) * mp.mpf(par["binsize"])
        return y * mp.log(lam) - lam - mp.loggamma(y + 1), y - lam, mp.mpf(0)
    s, df = mp.mpf(par["scale"]), mp.mpf(par["df"])
    r = y - f
    c = mp.loggamma((df + 1) / 2) - mp.loggamma(df / 2) - (mp.log(s * s) + mp.log(df) + mp.log(mp.pi)) / 2
    q = s * s * df + r * r
    return (c - (df + 1) / 2 * mp.log(1 + r * r / (s * s * df)), (df + 1) * r / q,
            -1 / s + (df + 1) * r * r / (s * q))


def _mp_g2(kind, par, y, f):
    mp = mpmath
    if kind == "bernoulli":
        J = mp.mpf("0.001")
        p = (1 + mp.erf(f / mp.sqrt(2))) / 2 * (1 - 2 * J) + J
        dp = (1 - 2 * J) * mp.exp(-f * f / 2) / mp.sqrt(2 * mp.pi)
        if y == 1:
            a = dp / p
            return -a * (f + a)
        a = dp / (1 - p)
        return a * (f - a)
    s, df = mp.mpf(par["scale"]), mp.mpf(par["df"])
    r = y - f
    q = s * s * df + r * r
    return (df + 1) * (r * r - s * s * df) / (q * q)


def exact_scalar(kind: str, par: Dict[str, float], y, mu, v) -> Dict[str, np.ndarray]:
    """The exact ve, dmu, dv, dpar of every element (the 20-point sums of the committed table; closed forms for the
    Gaussian and Poisson), rounded to double at the end."""
    mp = mpmath
    out = {k: np.empty(len(mu)) for k in ("ve", "dmu", "dv", "dpar")}
    with mp.workprec(PREC):
        Z = [mp.mpf(z) for z in GH_Z]
        W = [mp.mpf(w) for w in GH_W]
        S2 = mp.fsum(w * z * z for z, w in zip(Z, W))
        for i, (yi, mi, vi) in enumerate(zip(y, mu, v)):
            # the nodes differ from mu by sqrt(v) z_k: dz's cancellation needs that many more bits
            mp.prec = PREC + (int(-math.log2(math.sqrt(vi))) + 20 if 0.0 < vi < 1.0 else 0)
            yi, mi, vi = mp.mpf(float(yi)), mp.mpf(float(mi)), mp.mpf(float(vi))
            if kind == "gaussian":
                s = mp.mpf(par["noise"])
                r = yi - mi
                vals = (-mp.log(2 * mp.pi) / 2 - mp.log(s) / 2 - (r * r + vi) / (2 * s), r / s, -1 / (2 * s),
                        -1 / (2 * s) + (r * r + vi) / (2 * s * s))
            elif kind == "poisson":
                b = mp.mpf(par["binsize"])
                e = mp.exp(mi + vi / 2) * b
                vals = (yi * mi - e - mp.loggamma(yi + 1) + yi * mp.log(b), yi - e, -e / 2, mp.mpf(0))
            else:
                sd = mp.sqrt(vi)
                ve = dmu = dz = dpar = mp.mpf(0)
                for z, w in zip(Z, W):
                    lp, g1, gp = _mp_logp_terms(kind, par, yi, mi + sd * z)
                    ve += w * lp
                    dmu += w * g1
                    dz += w * g1 * z
                    dpar += w * gp
                dv = dz / (2 * sd) if vi > 0 else _mp_g2(kind, par, yi, mi) * S2 / 2
                vals = (ve, dmu, dv, dpar)
            for key, val in zip(("ve", "dmu", "dv", "dpar"), vals):
                out[key][i] = float(val)
    return out


def exact_scalar_predict(kind: str, par: Dict[str, float], y, mu, v) -> Dict[str, np.ndarray]:
    """The exact predictive mean, variance and log density of every element."""
    mp = mpmath
    out = {k: np.empty(len(mu)) for k in ("mean", "var", "ld")}
    with mp.workprec(PREC):
        Z = [mp.mpf(z) for z in GH_Z]
        W = [mp.mpf(w) for w in GH_W]
        J = mp.mpf("0.001")
        for i, (yi, mi, vi) in enumerate(zip(y, mu, v)):
            # E[y^2] - E[y]^2 cancels by about exp(2 mu) (Poisson) times 1 / v: carry those bits as well
            mp.prec = PREC + int(3 * abs(mi)) + (int(-math.log2(vi)) + 20 if 0.0 < vi < 1.0 else 0)
            yi, mi, vi = mp.mpf(float(yi)), mp.mpf(float(mi)), mp.mpf(float(vi))
            if kind == "gaussian":
                s = mp.mpf(par["noise"])
                tv = vi + s
                vals = (mi, tv, -(mp.log(2 * mp.pi) + mp.log(tv) + (yi - mi) ** 2 / tv) / 2)
            elif kind == "bernoulli":
                a = mi / mp.sqrt(1 + vi)
                p = (1 + mp.erf(a / mp.sqrt(2))) / 2 * (1 - 2 * J) + J
                vals = (p, p - p * p, mp.log(p if yi == 1 else 1 - p))
            else:
                sd = mp.sqrt(vi)
                ey = ey2 = dens = mp.mpf(0)
                for z, w in zip(Z, W):
                    f = mi + sd * z
                    if kind == "poisson":
                        cm = mp.exp(f) * mp.mpf(par["binsize"])
                        cv = cm
                    else:
                        cm = f
                        cv = mp.mpf(par["scale"]) ** 2 * mp.mpf(par["df"]) / (mp.mpf(par["df"]) - 2)
                    ey += w * cm
                    ey2 += w * (cv + cm * cm)
                    dens += w * mp.exp(_mp_logp_terms(kind, par, yi, f)[0])
                vals = (ey, ey2 - ey * ey, mp.log(dens))
            for key, val in zip(("mean", "var", "ld"), vals):
                out[key][i] = float(val)
    return out


# ---- the case table -----------------------------------------------------------------------------------------------
V_LIST = (0.0, 1e-300, 1e-30, 1e-12, 1e-6, 1.0, 1e2, 1e4)


def scalar_cases() -> List[Tuple[str, Dict[str, float]]]:
    """(kind, parameters) of every scalar configuration the tests run."""
    cases = [("gaussian", {"noise": 0.3}), ("bernoulli", {}), ("poisson", {"binsize": 1.3})]
    for df in (0.7, 3.0, 30.0):
        for scale in (1e-3, 0.7):
            cases.append(("student_t", {"df": df, "scale": scale}))
    return cases


def case_name(kind, par) -> str:
    return kind + "".join(f"-{k}{v:g}" for k, v in sorted(par.items()))


def scalar_elements(kind: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(y, mu, v) of the adjoint / VE case table of a likelihood: the tails of the issue list and every v of V_LIST."""
    rows = []
    if kind == "bernoulli":
        for mu in (-40.0, -8.5, -3.0, -0.3, 0.0, 0.7, 5.0, 12.0, 40.0):
            for y in (1.0, 0.0, -1.0):
                rows += [(y, mu, v) for v in V_LIST]
    elif kind == "poisson":
        for mu in (-30.0, -5.0, 0.0, 3.0, 13.5, 200.0, 650.0):
            for y in (0.0, 1.0, 7.0, 1e3, 1e6):
                rows += [(y, mu, v) for v in V_LIST if mu + v / 2 <= 700.0]
        rows += [(1e6, math.log(1e6 / 1.3), v) for v in V_LIST[:6]]   # y log lam - lam - lgamma(y+1) at 1e7 sizes
        rows += [(y, 700.0 - v / 2, v) for y in (0.0, 3.0) for v in (0.0, 1.0, 1e2, 1e3)]
    elif kind == "student_t":
        for mu in (0.3, -2.0):
            for r in (0.0, 1e-3, -0.5, 3.0, 1e3, 1e8, -1e8):
                rows += [(mu + r, mu, v) for v in V_LIST]
    else:
        for mu in (-3.0, 0.0, 2.0):
            for r in (0.0, 0.4, -7.0):
                rows += [(mu + r, mu, v) for v in V_LIST]
    a = np.array(rows)
    return a[:, 0].copy(), a[:, 1].copy(), a[:, 2].copy()


def predict_elements(kind: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(y, mu, v) of the prediction table: the adjoint table, for Poisson only where every quadrature node keeps
    exp(2 f_k) finite (|f_k| <= 350), so that E[y^2] is a double."""
    y, mu, v = scalar_elements(kind)
    if kind == "poisson":
        keep = np.abs(mu) + np.sqrt(v) * GH_Z[-1] <= 350.0
        y, mu, v = y[keep], mu[keep], v[keep]
    return y, mu, v


# ==== MultiClass ===================================================================================================
MC_CLASSES = (2, 31, 32, 33, 64, 65, 96, 97, 128)


def mc_rows(C: int, seed: int = 0) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(labels [N], mu [N, C], v [N, C]) of the MultiClass case table for C classes: the labels at both sides of every
    chunk edge, out of range and truncated; variances 0 and 3e-11 on label and non-label classes, with a non-label
    mean equal to the label's so that the clamped classes' terms are not negligible."""
    rng = np.random.default_rng(1000 + C + seed)
    labels = sorted({c for c in (0, 31, 32, 63, 64, 95, 96, C - 1) if c < C})
    labels += [float(C), float(C + 3), -1.0, 32.7, -0.5]
    rows_y, rows_mu, rows_v = [], [], []

    def base():
        return 0.6 * rng.standard_normal(C), rng.uniform(0.05, 1.0, C)

    for y in labels:
        mu, v = base()
        yi = int(y) if -1.0 < y < C else -1
        if yi >= 0:
            mu[yi] += 0.8
        rows_y.append(float(y)), rows_mu.append(mu), rows_v.append(v)
    for vy in (0.0, 3e-11, 0.4):
        for y in (0, C - 1):
            mu, v = base()
            others = [c for c in range(C) if c != y]
            for j, c in enumerate(others[:4] + others[-2:]):
                v[c] = (0.0, 3e-11)[j % 2]
                mu[c] = mu[y]
            v[y] = vy
            rows_y.append(float(y)), rows_mu.append(mu), rows_v.append(v)
    return np.array(rows_y), np.array(rows_mu), np.array(rows_v)


class McConsts:
    """mc_desc's host constants and the device's 1 - eps and kappa."""

    def __init__(self, C, eps):
        e = Err(np.float64(eps))
        self.eps_k1 = e / (C - 1.0)
        self.log1m = log(1.0 - e)
        self.logk1 = log(self.eps_k1)
        self.inv1m = 1.0 / (1.0 - e)
        self.inveps = 1.0 / e
        self.kappa = self.log1m - self.logk1
        self.one_m = 1.0 - e


def _scan_up(x: Err, mutation=None) -> Err:
    """mc_scan_up along the last axis (32 lanes): x *= shfl_up(x, o) where lane >= o."""
    v, e = x.v.copy(), x.e.copy()
    for o in (1, 2, 4, 8, 16):
        t = Err(v[..., :-o], e[..., :-o]) * Err(v[..., o:], e[..., o:])
        v = np.concatenate([v[..., :o], t.v], -1)
        e = np.concatenate([e[..., :o], t.e], -1)
    return Err(v, e)


def _scan_down(x: Err) -> Err:
    v, e = x.v.copy(), x.e.copy()
    for o in (1, 2, 4, 8, 16):
        t = Err(v[..., :-o], e[..., :-o]) * Err(v[..., o:], e[..., o:])
        v = np.concatenate([t.v, v[..., -o:]], -1)
        e = np.concatenate([t.e, e[..., -o:]], -1)
    return Err(v, e)


def _warp_sum(x: Err) -> Err:
    """warp_sum: xor butterflies; lane 0's tree folds halves."""
    while x.v.shape[-1] > 1:
        h = x.v.shape[-1] // 2
        x = Err(x.v[..., :h], x.e[..., :h]) + Err(x.v[..., h:], x.e[..., h:])
    return Err(x.v[..., 0], x.e[..., 0])


def mc_label(y, C):
    y = np.asarray(y)
    return np.where((y > -1.0) & (y < C), np.trunc(np.clip(y, -1.0, C)), -1).astype(np.int64)


def mc_prob(C, lab, mu, v, *, grad=False, mutation=None):
    """mc_load + mc_selected + mc_prob<NJ, GRAD> for rows [N]: p and, with grad, G, H [N, NJ*32], gs, gx (warp sums)
    and is (1 / s_c), is_y, v_y."""
    N = mu.shape[0]
    NJ = (C + 31) // 32
    L = 32 * NJ
    MU = np.zeros((N, L))
    V = np.ones((N, L))
    MU[:, :C], V[:, :C] = mu, v
    cls = np.arange(L)[None]
    valid = (cls < C) & (cls != lab[:, None])
    mu_e = Err(MU)
    is_ = rsqrt(Err(np.maximum(V, 1e-10)))
    rows = np.arange(N)
    has = lab >= 0
    mu_y = Err(np.where(has, MU[rows, np.maximum(lab, 0)], 0.0))
    v_y = np.where(has, V[rows, np.maximum(lab, 0)], 0.0)
    two = 1.0 if mutation == "s_y_v" else 2.0
    q = Err(np.maximum(two * v_y, 1e-10))
    is_y = rsqrt(q)
    s_y = q * is_y
    shape = (N, NJ, 32)
    z3 = lambda a: Err(a.v.reshape(shape), a.e.reshape(shape))
    valid3 = valid.reshape(shape)
    p = Err(np.zeros(N))
    G = H = Err(np.zeros(shape))
    gs = gx = Err(np.zeros((N, 32)))
    for k in range(20):
        xk = Err(GH_Z[k]) * Err.const(SQRT1_2)
        wk = GH_W[k]
        X = xk.fma(s_y, mu_y)
        d = (Err(X.v[:, None], X.e[:, None]) - mu_e) * is_
        d3 = z3(d)
        cdf = (0.5 * (1.0 + erf_(d3 * Err.const(SQRT1_2)))).fma(Err.const(1.0 - 2.0 * SQUASH), Err.const(SQUASH))
        cdf = where(valid3, cdf, Err(np.ones(shape)))
        incl = _scan_up(cdf)
        tot = [Err(incl.v[:, j, 31], incl.e[:, j, 31]) for j in range(NJ)]
        allp = Err(np.ones(N))
        for j in range(NJ):
            allp = allp * tot[j]
        p = Err(wk).fma(allp, p)
        if not grad:
            continue
        dn_all = _scan_down(cdf)
        before = Err(np.ones(N))
        gk = Err(np.zeros((N, 32)))
        Gs, Hs = [], []
        for j in range(NJ):
            after = Err(np.ones(N))
            last = NJ - 1 if mutation == "after_missing_last" else NJ
            for i in range(j + 1, last):
                after = after * tot[i]
            ij = Err(incl.v[:, j], incl.e[:, j])
            dj = Err(dn_all.v[:, j], dn_all.e[:, j])
            up = Err(np.concatenate([ij.v[:, :1] if mutation == "own_cdf_lane0" else np.ones((N, 1)), ij.v[:, :-1]], 1),
                     np.concatenate([ij.e[:, :1] if mutation == "own_cdf_lane0" else np.zeros((N, 1)), ij.e[:, :-1]], 1))
            dn = Err(np.concatenate([dj.v[:, 1:], dj.v[:, 31:] if mutation == "own_cdf_lane31" else np.ones((N, 1))], 1),
                     np.concatenate([dj.e[:, 1:], dj.e[:, 31:] if mutation == "own_cdf_lane31" else np.zeros((N, 1))], 1))
            ba = before * after
            E = (Err(ba.v[:, None], ba.e[:, None]) * up) * dn
            dj3 = Err(d3.v[:, j], d3.e[:, j])
            phi = exp((-0.5 * dj3) * dj3)
            g = ((((wk * E) * Err.const(1.0 - 2.0 * SQUASH)) * Err.const(RSQRT2PI)) * phi) * \
                Err(is_.v.reshape(shape)[:, j], is_.e.reshape(shape)[:, j])
            g = where(valid3[:, j], g, Err(np.zeros((N, 32))))
            Gs.append(Err(G.v[:, j], G.e[:, j]) + g)
            Hs.append(g.fma(dj3, Err(H.v[:, j], H.e[:, j])))
            gk = gk + g
            before = before * tot[j]
        G = Err(np.stack([a.v for a in Gs], 1), np.stack([a.e for a in Gs], 1))
        H = Err(np.stack([a.v for a in Hs], 1), np.stack([a.e for a in Hs], 1))
        gs = gs + gk
        gx = Err(xk.v, xk.e).fma(gk, gx)
    out = {"p": p, "is": is_, "is_y": is_y, "v_y": v_y, "V": V}
    if grad:
        out.update(G=Err(G.v.reshape(N, L), G.e.reshape(N, L)), H=Err(H.v.reshape(N, L), H.e.reshape(N, L)),
                   gs=_warp_sum(gs), gx=_warp_sum(gx))
    return out


def mc_grad(C, eps, y, mu, v, cs, *, mutation=None):
    """mc_grad_kernel for rows: R [N, C], W [N, C] (Err), per-row dVE/deps terms, VE (Err)."""
    M = McConsts(C, eps)
    lab = mc_label(y, C)
    o = mc_prob(C, lab, mu, v, grad=True, mutation=mutation)
    N = mu.shape[0]
    k = ((-cs) * M.kappa)
    R = k * o["G"]
    kh = (((-0.5) * cs) * M.kappa)
    Wc = (kh * o["H"]) * o["is"]
    if mutation != "no_w_clamp":
        Wc = where(o["V"] > 1e-10, Wc, Err(np.zeros(Wc.v.shape)))
    rows = np.arange(N)
    has = lab >= 0
    Ry = (cs * M.kappa) * o["gs"]
    Wy = ((cs * M.kappa) * o["gx"]) * o["is_y"]
    Wy = where(2.0 * o["v_y"] > 1e-10, Wy, Err(np.zeros(N)))
    Rv, Re = R.v[:, :C].copy(), R.e[:, :C].copy()
    Wv, We = Wc.v[:, :C].copy(), Wc.e[:, :C].copy()
    li = np.maximum(lab, 0)
    Rv[rows[has], li[has]], Re[rows[has], li[has]] = Ry.v[has], Ry.e[has]
    Wv[rows[has], li[has]], We[rows[has], li[has]] = Wy.v[has], Wy.e[has]
    p = o["p"]
    deps = (-p) * M.inv1m + (1.0 - p) * M.inveps
    ve = p * M.log1m + (1.0 - p) * M.logk1
    return {"R": Err(Rv, Re), "W": Err(Wv, We), "deps": deps, "ve": ve, "p": p}


def mc_ve(C, eps, y, mu, v):
    M = McConsts(C, eps)
    p = mc_prob(C, mc_label(y, C), mu, v)["p"]
    return p * M.log1m + (1.0 - p) * M.logk1


def mc_predict(C, eps, y, mu, v):
    """mc_predict_mv_kernel (mean, var [N, C]) and mc_predict_ld_kernel (ld [N]) on the stored inputs."""
    M = McConsts(C, eps)
    N = mu.shape[0]
    mv, me, vv, vve = (np.zeros((N, C)) for _ in range(4))
    for c in range(C):
        p = mc_prob(C, np.full(N, c), mu, v)["p"]
        dens = p.fma(M.one_m, (1.0 - p) * M.eps_k1)
        var = dens - dens * dens
        mv[:, c], me[:, c], vv[:, c], vve[:, c] = dens.v, dens.e, var.v, var.e
    p = mc_prob(C, mc_label(y, C), mu, v)["p"]
    ld = log(p.fma(M.one_m, (1.0 - p) * M.eps_k1))
    return Err(mv, me), Err(vv, vve), ld


def exact_mc(C, eps, y, mu, v, *, grad=True) -> Dict[str, np.ndarray]:
    """Exact p, VE, density(y), R = dVE/dmu, W = dVE/dv [N, C] and dVE/deps per row (tests/multiclass_oracle.py's
    formulas with its clamps and label rules), at 113 bits."""
    mp = mpmath
    N = mu.shape[0]
    out = {"p": np.empty(N), "ve": np.empty(N), "ld": np.empty(N), "deps": np.empty(N), "R": np.zeros((N, C)),
           "W": np.zeros((N, C))}
    lab = mc_label(y, C)
    with mp.workprec(PREC):
        X = [mp.mpf(z) / mp.sqrt(2) for z in GH_Z]
        Wt = [mp.mpf(w) for w in GH_W]
        e = mp.mpf(float(eps))
        ek1 = e / (C - 1)
        kappa = mp.log(1 - e) - mp.log(ek1)
        S = mp.mpf("1e-6")
        clamp = mp.mpf("1e-10")
        for n in range(N):
            yl = int(lab[n])
            m = [mp.mpf(float(a)) for a in mu[n]]
            vv = [mp.mpf(float(a)) for a in v[n]]
            m_y, v_y = (m[yl], vv[yl]) if yl >= 0 else (mp.mpf(0), mp.mpf(0))
            s_y = mp.sqrt(max(2 * v_y, clamp))
            s = [mp.sqrt(max(a, clamp)) for a in vv]
            others = [c for c in range(C) if c != yl]
            p = mp.mpf(0)
            G = [mp.mpf(0)] * C
            Hs = [mp.mpf(0)] * C
            gx = gsum = mp.mpf(0)
            for xk, wk in zip(X, Wt):
                Xv = m_y + xk * s_y
                d = {c: (Xv - m[c]) / s[c] for c in others}
                cdf = [(1 + mp.erf(d[c] / mp.sqrt(2))) / 2 * (1 - 2 * S) + S for c in others]
                pre = [mp.mpf(1)]
                for a in cdf:
                    pre.append(pre[-1] * a)
                p += wk * pre[-1]
                if not grad:
                    continue
                suf = [mp.mpf(1)] * (len(cdf) + 1)
                for i in range(len(cdf) - 1, -1, -1):
                    suf[i] = suf[i + 1] * cdf[i]
                gk = mp.mpf(0)
                for i, c in enumerate(others):
                    g = wk * pre[i] * suf[i + 1] * (1 - 2 * S) * mp.exp(-d[c] ** 2 / 2) / mp.sqrt(2 * mp.pi) / s[c]
                    G[c] += g
                    Hs[c] += g * d[c]
                    gk += g
                gsum += gk
                gx += xk * gk
            out["p"][n] = float(p)
            out["ve"][n] = float(p * mp.log(1 - e) + (1 - p) * mp.log(ek1))
            out["ld"][n] = float(mp.log(p * (1 - e) + (1 - p) * ek1))
            out["deps"][n] = float(-p / (1 - e) + (1 - p) / e)
            if grad:
                for c in others:
                    out["R"][n, c] = float(-kappa * G[c])
                    out["W"][n, c] = float(-kappa * Hs[c] / (2 * s[c])) if vv[c] > clamp else 0.0
                if yl >= 0:
                    out["R"][n, yl] = float(kappa * gsum)
                    out["W"][n, yl] = float(kappa * gx / s_y) if 2 * v_y > clamp else 0.0
    return out
