"""Error bars, a schedule mirror and a NumPy emulation of the blocked Cholesky (csrc/potrf.cu), CPU only.

Schedule.  `schedule` mirrors potrf_t -> potrf_rec -> potrf_block -> trailing_update and returns the launches of one
factorisation in issue order: every leaf (slim or full inverse), every panel (plain, fused K = 128, diagonal feed or the
inverse GEMM of a full leaf; polled or event-ordered), the older-column kernel of a feed, and every trailing update (int8
with its S and k-range, or DMMA; which extra rows it slices with dynamic scales and whether a panel sliced them already).

Residual.  For the computed factor F (L in the first n rows, X = Y L^-T in the extra rows) `exact_residual` returns
R = A - L L^T (lower triangle) and R_Y = Y - X L^T without rounding error: every row of F is scaled by a power of two and
split into four 17-bit integer slices; a slice product summed over k < 2^17 stays an integer below 2^53, so fp64 BLAS
returns it exactly in any order, and the seven groups of equal weight are recombined in long double.  The slices keep 68
bits of the row maximum; what they drop, t, is known exactly, and 2 (|t| |F|^T + |F| |t|^T) plus the long double
recombination (8 2^-64 |F| |F|^T) are added to every bar.

Worst-case bar of element (i, j), u the unit roundoff of the arithmetic (2^-53 fp64, 2^-24 fp32):
  * gamma(c_ij) (|F| |F|^T)_ij with c_ij = min(i, j) + 2 (updates touching (i, j)) + 10: the left-looking sums of the leaf
    (one rounding per product, three more for the four partial sums), one rounding per product of every DMMA or fused
    update plus the subtraction from C, and the pivot (rsqrt step and product, a few ulps);
  * for every int8 update touching (i, j): K (S + 1) 2^(-8S+2) s_i s_j, s = 2^e with e the static row exponent from the
    original diagonal (tests/test_digit_slicing_model.py); extra rows use their dynamic scale, the maximum over the
    update's k-range (every row when the scales are not static: that maximum is never above the static one);
  * for rows solved by a panel: the inverse-based residual of dense64_bounds.trsm_check, per 64-column sub-block k of the
    slim panel (128 columns for a full inverse): (eta_k + gamma(w) kappa_k + 2 gamma(w + 2)) max_{j' in k} (|x_i| |L_JJ|^T)_j'
    with kappa_k = || |L_kk| |L_kk^-1| ||_inf from the computed block and eta_k <= 2 gamma(w) kappa_k the residual of the
    leaf's inverse of that block (Higham ch. 14);
  * an absolute term 4 (c_ij + 2 w kappa) 2^-1074 (fp64) for roundings in the subnormal range.

Statistical bars.  z_ij = R_ij / (u (|F| |F|^T)_ij).  Modelling each rounding as an independent error of at most u of
its result, the panel term TP as a random walk of w contributions (TP / sqrt(w)), and an int8 update's truncation as
its S - 1 dropped digit products of order S per k, each 2^-12 2^-8S d_s d_t s_i s_j with digits uniform in [-128, 128)
(RMS 2^0.415 2^-8S s_i s_j per product, independent over k): V8 = sum over the updates of 4 K (S - 1) 2^(0.83 - 16 S)
(s_i s_j)^2 (a factor 2 of margin on the RMS), the RMS of z over a group of elements is at most
sqrt(mean(c_ij + V8_ij / (u M_ij)^2 + (TP_ij / (u M_ij))^2 / w)) (groups: block columns of >= 1e4 elements), and
the mean of z over the d diagonal elements is at most 6 RMS_diag / sqrt(d): a rounding error of the kernels is zero-mean,
a dropped (3,3) digit product or a short rsqrt step is not."""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

from tests.dense64_bounds import NB, U, gamma, split_point
from tests.test_digit_slicing_model import row_exponents, slice_rows, syrk_i8_epilogue

U_LD = 2.0 ** -64
U32 = 2.0 ** -24
TINY = 2.0 ** -1074
PR, PCR = 64, 16                  # panel rows per CTA, rows per critical CTA (potrf.cu)
SLICE_BITS, NSLICE = 17, 4


# ---- schedule mirror -----------------------------------------------------------------------------------------------------
class Config:
    """The engine switches potrf_t reads (defaults = a bare gpk_potrf on an H100 with 132 SMs)."""

    def __init__(self, S=7, sms=132, tc=True, lookahead=True, fuse=True, flaghop=True, slim=True, static=True,
                 feed_max=512, tc_min_k=256, f64=True):
        self.S, self.sms, self.tc, self.lookahead, self.fuse, self.flaghop = S, sms, tc, lookahead, fuse, flaghop
        self.slim, self.static, self.feed_max, self.tc_min_k, self.f64 = slim, static, feed_max, tc_min_k, f64


def tc_update_eligible(cfg, planes, m, n, K):
    """potrf.cu::tc_update_eligible (int32 headroom: 128 * 128 * K * S < 2^31)."""
    return cfg.f64 and planes and K >= cfg.tc_min_k and K % 32 == 0 and n <= m and K * cfg.S * 16384 < 2 ** 31


def schedule(n, rows=None, cfg=None):
    """Launches of potrf_t(n, rows) in issue order, as dicts with a "kind" of leaf / panel / feed_old / update."""
    cfg = cfg or Config()
    rows = n if rows is None else rows
    out = []
    enabled = cfg.lookahead and n > NB
    slim = cfg.f64 and n > NB and cfg.slim
    fuse = slim and enabled and cfg.fuse
    flaghop = slim and enabled and cfg.flaghop
    planes = bool(cfg.tc and slim and split_point(n) >= cfg.tc_min_k)
    st = dict(follow_k0=-1, follow_K=0, dyn_k0=-1, dyn_K=0, feed=False)

    def update(m, nn, K, col0):
        tc = tc_update_eligible(cfg, planes, m, nn, K)
        r0 = col0 + K
        slice_rows = None
        if tc:
            dyn0 = max(n, r0) if cfg.static else r0
            if dyn0 < r0 + m:
                by_panel = cfg.static and st["dyn_k0"] == col0 and st["dyn_K"] == K
                slice_rows = (dyn0, r0 + m, "panel" if by_panel else "update")
        skip = NB if st["feed"] else 0
        st["feed"] = False
        eng = "int8" if tc else "dmma"
        headroom = (not tc and cfg.f64 and planes and K >= cfg.tc_min_k and K % 32 == 0 and nn <= m)
        out.append(dict(kind="update", k0=col0, K=K, r0=r0, m=m, n=nn, engine=eng, S=cfg.S if tc else 0,
                        row_skip=skip, slice=slice_rows, headroom_dmma=headroom))

    def block(nb, rows_, col0, fuse_cols):
        st["feed"] = False
        out.append(dict(kind="leaf", c0=col0, nb=nb, slim=slim))
        if rows_ <= nb:
            return
        prow = rows_ - nb
        fk0, fK = st["follow_k0"], st["follow_K"]
        feed = (fuse and fuse_cols == 0 and nb == NB and NB < fK <= cfg.feed_max and fk0 + fK == col0 + nb
                and prow >= NB)
        ncrit = -(-min(fuse_cols, prow) // PCR) if fuse_cols > 0 else (NB // PCR if feed else 0)
        if feed:
            out.append(dict(kind="feed_old", c0=col0, k0=fk0, kold=fK - nb))
        polled = None
        if flaghop:
            polled = ncrit + -(-prow // PR) <= cfg.sms - 8
        emit = slim and planes and cfg.static
        if slim and fuse_cols > 0:
            below = prow - ncrit * PCR
            ctas = ncrit + (-(-below // PR) if below > 0 else 0)
            out.append(dict(kind="panel", c0=col0, nb=nb, rows=prow, type="fused", fuse_cols=fuse_cols, ncrit=ncrit,
                            ctas=ctas, polled=polled, dyn=None))
            return
        st["dyn_K"] = 0
        dyn = None
        if slim and emit and nb == NB and fK > 0 and fk0 + fK == col0 + nb and rows_ > n - col0:
            st["dyn_k0"], st["dyn_K"] = fk0, fK
            dyn = (fk0, fK)
        if feed:
            st["feed"] = True
        ctas = ncrit + -(-(prow - ncrit * PCR) // PR)
        out.append(dict(kind="panel", c0=col0, nb=nb, rows=prow, type=("feed" if feed else "plain") if slim else "gemm",
                        fuse_cols=0, ncrit=ncrit, ctas=ctas, polled=polled, dyn=dyn))

    def rec(n_, rows_, col0, fk0=-1, fK=0):
        if n_ <= NB:
            st["follow_k0"], st["follow_K"] = fk0, fK
            return block(n_, rows_, col0, 0)
        n1 = split_point(n_)
        if n_ <= 2 * NB and fuse:
            st["follow_K"] = 0
            block(n1, rows_, col0, n_ - n1)
            return rec(n_ - n1, rows_ - n1, col0 + n1, fk0, fK)
        tc = tc_update_eligible(cfg, planes, rows_ - n1, n_ - n1, n1)
        rec(n1, rows_, col0, col0, n1 if tc else 0)
        update(rows_ - n1, n_ - n1, n1, col0)
        return rec(n_ - n1, rows_ - n1, col0 + n1, fk0, fK)

    if n > 0:
        rec(n, rows, 0)
    return out


def branches(launches, n, rows):
    """The code paths of potrf_rec / potrf_block / trailing_update a launch list takes."""
    b = set()
    for L in launches:
        if L["kind"] == "leaf":
            b.add("leaf_slim" if L["slim"] else "leaf_full")
            if L["nb"] < NB and L["c0"] > 0:
                b.add("ragged_last_block")
        elif L["kind"] == "feed_old":
            b.add("feed_old")
        elif L["kind"] == "panel":
            b.add("panel_" + L["type"])
            if L["polled"] is not None:
                b.add("panel_polled" if L["polled"] else "panel_event_ordered")
            if L["dyn"] is not None:
                b.add("extra_rows_sliced_by_panel")
        else:
            if L["engine"] == "int8":
                b.add("update_int8_fed" if L["row_skip"] else "update_int8")
                if L["K"] >= 640 and not L["row_skip"]:
                    b.add("update_int8_k640_plus")
                if L["slice"] and L["slice"][2] == "update":
                    b.add("extra_rows_sliced_by_update")
            else:
                b.add("update_dmma_k128" if L["K"] == NB else "update_dmma")
                if L["headroom_dmma"]:
                    b.add("update_dmma_int32_headroom")
    if rows > n:
        b.add("extra_rows")
    return b


# ---- exact residual ------------------------------------------------------------------------------------------------------
def _slices(F):
    """F = 2^e_i (sum_a s_a 2^(-17 (a + 1)) + t 2^-68) per row, |s_a| <= 2^17, |t| <= 1/2; every step exact.  Returns
    the slices, e and the truncation t 2^(e_i - 68) itself."""
    mx = np.abs(F).max(axis=1) if F.shape[1] else np.zeros(F.shape[0])
    e = np.where(mx > 0, np.frexp(mx)[1], 0).astype(np.int64)
    r = np.ldexp(F, -e[:, None])
    out = []
    for _ in range(NSLICE):
        r = r * 2.0 ** SLICE_BITS
        s = np.rint(r)
        out.append(s)
        r = r - s
    return out, e, np.ldexp(r, (e - SLICE_BITS * NSLICE)[:, None])


def exact_residual(T, F, n, ri):
    """(R, M, trunc) on the rows `ri` of the target T (A's lower triangle in rows < n, Y below) and the factor F (rows x n,
    lower in its first n rows): R = T - F F[:n]^T in long double from exact slice products (meaningful on keep_mask), M =
    |F| |F[:n]|^T and the bound of the slicing truncation."""
    Fl = np.where(np.tri(F.shape[0], n, dtype=bool), F, 0.0)
    assert n < 2 ** SLICE_BITS
    P, Q = Fl[ri], Fl[:n]
    sp, ep, tp = _slices(P)
    sq, eq, tq = _slices(Q)
    acc = np.zeros((len(ri), n), dtype=np.longdouble)
    for g in range(2 * NSLICE - 1):
        pairs = [(a, g - a) for a in range(NSLICE) if 0 <= g - a < NSLICE]
        G = np.concatenate([sp[a] for a, _ in pairs], axis=1) @ np.concatenate([sq[b] for _, b in pairs], axis=1).T
        acc += G.astype(np.longdouble) * np.longdouble(2.0) ** (-SLICE_BITS * (g + 2))
    scale = np.ldexp(1.0, ep)[:, None] * np.ldexp(1.0, eq)[None, :]
    R = (T[ri][:, :n].astype(np.longdouble) - acc * scale.astype(np.longdouble)).astype(np.float64)
    M = np.abs(P) @ np.abs(Q).T
    trunc = 2 * (np.abs(tp) @ np.abs(Q).T + np.abs(P) @ np.abs(tq).T)
    return R, M, trunc


def sample_rows(n, rows, rng, extra=48):
    """Every row at a 32 / 64 / 128 block edge of the square part, the extra rows' edges and `extra` random rows."""
    idx = set()
    for e in range(0, n + 1, 32):
        idx.update(i for i in (e - 1, e) if 0 <= i < n)
    idx.update(i for i in (n, n + 1, rows - 1) if n <= i < rows)
    idx.update(rng.integers(0, rows, size=min(extra, rows)).tolist())
    return np.array(sorted(idx), dtype=np.int64)


# ---- bars ----------------------------------------------------------------------------------------------------------------
def static_exponents(diagA):
    """gemm_tc.cu::row_exp_kernel: e_i = ilogb(sqrt(A_ii)) + 1, 0 for a non-positive or non-finite pivot (row_exponents of
    the one-column matrix sqrt(A_ii); its -1017 floor never applies to a square root)."""
    d = np.asarray(diagA, dtype=np.float64)
    ok = (d > 0) & np.isfinite(d)
    return row_exponents(np.sqrt(np.where(ok, d, 0.0))[:, None])


def _sub_block_terms(F, n, c0, nb, w, ri, u):
    """Panel term of the rows ri (all below block [c0, c0 + nb)) per sub-block of width w: [len(ri), nb]."""
    Ljj = np.tril(F[c0:c0 + nb, c0:c0 + nb])
    out = np.zeros((len(ri), nb))
    H = np.abs(F[ri, c0:c0 + nb]) @ np.abs(Ljj).T
    for o in range(0, nb, w):
        ww = min(w, nb - o)
        B = Ljj[o:o + ww, o:o + ww]
        with np.errstate(all="ignore"):
            X = sla.solve_triangular(B, np.eye(ww), lower=True, check_finite=False)
            kap = float(np.max((np.abs(B) @ np.abs(X)).sum(axis=1)))
        if not np.isfinite(kap):
            kap = np.inf
        coef = 2 * gamma(w, u) * kap + gamma(w, u) * kap + 2 * gamma(w + 2, u)
        tiny = 4 * 2 * w * kap * (TINY if u == U else 2.0 ** -149)
        out[:, o:o + ww] = coef * H[:, o:o + ww].max(axis=1, keepdims=True) + tiny
    return out


def bars(launches, F, n, ri, diagA, M, u=U, S=7):
    """Worst-case bar [len(ri), n] and the pieces the statistical bars need: (bar, c, V8, TP, W), V8 already in units
    of (u M)^2."""
    ri = np.asarray(ri)
    r = len(ri)
    cols = np.arange(n)
    cnt = np.zeros((r, n))
    T8 = np.zeros((r, n))
    V8 = np.zeros((r, n))
    TP = np.zeros((r, n))
    W = np.ones((r, n))
    es = static_exponents(diagA)
    for L in launches:
        if L["kind"] == "update":
            r0, m, nn, k0, K = L["r0"], L["m"], L["n"], L["k0"], L["K"]
            rin = (ri >= r0) & (ri < r0 + m)
            cin = (cols >= r0) & (cols < r0 + nn)
            hit = rin[:, None] & cin[None, :]
            cnt += 2 * hit
            if L["engine"] == "int8":
                ei = es[np.minimum(ri, n - 1)].copy()
                ext = ri >= (n if L["slice"] is None or L["slice"][0] >= n else L["slice"][0])
                if ext.any():
                    ei[ext] = row_exponents(F[ri[ext], k0:k0 + K])
                si = np.ldexp(1.0, ei)[:, None]
                sj = np.ldexp(1.0, es)[None, :]
                Sd = L["S"]
                T8 += hit * (K * (Sd + 1) * 2.0 ** (-8 * Sd + 2)) * si * sj
                with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
                    q = np.where(hit & (M > 0), 2 * np.sqrt(K * (Sd - 1)) * 2.0 ** (0.415 - 8 * Sd) * si * sj
                                 / (u * np.where(M > 0, M, 1.0)), 0.0)
                V8 += q * q
        elif L["kind"] == "panel":
            c0, nb = L["c0"], L["nb"]
            below = ri >= c0 + nb
            if below.any():
                w = 64 if L["type"] != "gemm" else NB
                TP[np.ix_(below, np.arange(c0, c0 + nb))] += _sub_block_terms(F, n, c0, nb, w, ri[below], u)
                W[np.ix_(below, np.arange(c0, c0 + nb))] = w
            if L["type"] == "fused":
                hit = below[:, None] & ((cols >= c0 + nb) & (cols < c0 + nb + L["fuse_cols"]))[None, :]
                cnt += 2 * hit
            if L["type"] == "feed":
                hit = ((ri >= c0 + nb) & (ri < c0 + nb + NB))[:, None] & ((cols >= c0 + nb) & (cols < c0 + nb + NB))[None, :]
                cnt += 4 * hit
    c = np.minimum(ri[:, None], cols[None, :]) + cnt + 10
    tiny = TINY if u == U else 2.0 ** -149
    bar = gamma(c, u) * M + T8 + TP + 4 * c * tiny
    return bar, c, V8, TP, W


def slice_trunc_bar(M, trunc):
    return 8 * U_LD * M + trunc


def keep_mask(ri, n):
    """The residual entries that exist: j <= i in the square part, every column in the extra rows."""
    ri = np.asarray(ri)
    return (ri[:, None] >= np.arange(n)[None, :]) | (ri >= n)[:, None]


def worst_ratio(R, bar, keep):
    """max |R| / bar over `keep`; inf when any kept residual is not finite (a NaN or Inf never passes)."""
    q = np.abs(R[keep]) / bar[keep]
    if not np.all(np.isfinite(q)):
        return float("inf")
    return float(q.max()) if q.size else 0.0


def stats(R, M, ri, n, c, V8, TP, W, u=U, group_min=10_000):
    """(worst RMS ratio over the groups, diagonal mean ratio or None): each statistic over its derived bound."""
    ri = np.asarray(ri)
    tiny = TINY if u == U else 2.0 ** -149
    uM = u * M
    use = keep_mask(ri, n) & (uM > 64 * tiny)
    with np.errstate(divide="ignore", invalid="ignore"):
        z = np.where(use, R / np.where(use, uM, 1.0), 0.0)
        v = np.where(use, c + V8 + (TP / np.where(use, uM, 1.0)) ** 2 / W, 0.0)
    use &= np.isfinite(v)              # (a panel term beyond 1e154 u M: the element carries no statistical weight)
    z = np.where(use, z, 0.0)
    v = np.where(use, v, 0.0)
    worst = 0.0
    groups, acc = [], []
    for o in range(0, n, NB):
        acc.append(np.arange(o, min(n, o + NB)))
        if use[:, np.concatenate(acc)].sum() >= group_min:
            groups.append(np.concatenate(acc))
            acc = []
    if acc and groups:
        groups[-1] = np.concatenate([groups[-1]] + acc)
    for gcols in groups:
        k = use[:, gcols]
        rms = np.sqrt(np.mean(z[:, gcols][k] ** 2))
        worst = max(worst, rms / np.sqrt(np.mean(v[:, gcols][k])))
    dmean = None
    di = np.nonzero(ri < n)[0]
    if len(di):
        d = (di, ri[di])
        dk = use[d]
        if dk.sum() >= 256:
            zd = z[d][dk]
            dmean = abs(float(zd.mean())) / (6 * np.sqrt(np.mean(v[d][dk])) / np.sqrt(dk.sum()))
    return worst, dmean


def check(T, F, n, rows, ri, launches, diagA, u=U, S=7):
    """Every check of one computed factor: dict of worst ratios (worst-case, RMS, diagonal mean; <= 1 passes)."""
    R, M, trunc = exact_residual(T, F, n, ri)
    bar, c, V8, TP, W = bars(launches, F, n, ri, diagA, M, u, S)
    bar = bar * (1 + 4 * u) + slice_trunc_bar(M, trunc)
    out = dict(worst=worst_ratio(R, bar, keep_mask(ri, n)))
    rms, dm = stats(R, M, ri, n, c, V8, TP, W, u)
    out["rms"] = rms
    if dm is not None:
        out["diag_mean"] = dm
    return out


# ---- test matrices -------------------------------------------------------------------------------------------------------
def random_spd(n, rng):
    B = rng.standard_normal((n, n + 16))
    return B @ B.T / n + 0.5 * np.eye(n)


def gpr_matrix(n, rng, kind="rbf", noise=1e-6, variance=1.0, clusters=None):
    """RBF / Matern52 gram matrix on clustered 2-d inputs plus noise: cond ~ variance n / noise."""
    k = clusters or max(2, n // 20)
    centres = rng.uniform(-3, 3, (k, 2))
    X = centres[rng.integers(0, k, n)] + 0.05 * rng.standard_normal((n, 2))
    r = np.sqrt(np.maximum(((X[:, None, :] - X[None, :, :]) ** 2).sum(-1), 0.0))
    if kind == "rbf":
        K = variance * np.exp(-0.5 * r * r)
    else:
        s = np.sqrt(5.0) * r
        K = variance * (1 + s + s * s / 3) * np.exp(-s)
    return K + noise * np.eye(n)


def dad(n, rng, span=500):
    d = np.ldexp(1.0, rng.integers(-span, span + 1, n))
    return random_spd(n, rng) * d[:, None] * d[None, :]


def integer_factor(n, rng, p_max=3):
    """L0 with a power-of-two diagonal, diagonal 128 x 128 diagonal blocks and entries in {-1, 0, 1} elsewhere below
    the diagonal: L0 L0^T and every product of the blocked factorisation are integers below 2^53."""
    L = np.tril(rng.integers(-1, 2, (n, n)).astype(np.float64), -1)
    for o in range(0, n, NB):
        L[o:o + NB, o:o + NB] = 0.0
    L[np.diag_indices(n)] = np.ldexp(1.0, rng.integers(0, p_max + 1, n))
    return L


# ---- NumPy emulation of the blocked factorisation -------------------------------------------------------------------------
def _rsqrt(d, mutant):
    if mutant == "newton1":   # a 2^-22 seed and one Newton step: the result is short by ~ (3/2) e^2
        y0 = (1.0 / np.sqrt(d)) * (1.0 + 2.0 ** -22 * (0.5 + 0.5 * np.random.default_rng(int(d * 1e6) % 997).random()))
        return y0 * (1.5 - 0.5 * d * y0 * y0)
    return 1.0 / np.sqrt(d)


def _leaf(A, c0, nb, mutant):
    """Factor A[c0:c0+nb, c0:c0+nb] in place like potrf_leaf_kernel: 32-column steps; in each, the 32 x 32 block left-
    looking with four partial sums, the rows below by per-row forward substitution, then the in-leaf update."""
    Bk = A[c0:c0 + nb, c0:c0 + nb]
    for jb in range(0, nb, 32):
        w = min(32, nb - jb)
        D = Bk[jb:jb + w, jb:jb + w]
        for j in range(w):
            if j >= 2:
                ks = np.arange(j - 1)
                part = [D[j:, ks[ks % 4 == q]] @ D[j, ks[ks % 4 == q]] for q in range(4)]
                D[j:, j] -= (part[0] + part[1]) + (part[2] + part[3])
            if j >= 1:
                D[j:, j] -= D[j:, j - 1] * D[j, j - 1]
            d = D[j, j]
            if not d > 0:
                d = 1.0
            y = _rsqrt(d, mutant)
            D[j + 1:, j] *= y
            D[j, j] = d * y
        if jb + w < nb:
            Bk[jb + w:, jb:jb + w] = sla.solve_triangular(np.tril(D), Bk[jb + w:, jb:jb + w].T, lower=True,
                                                          check_finite=False).T
            P = Bk[jb + w:, jb:jb + w]
            Bk[jb + w:, jb + w:] -= np.tril(P @ P.T)
    A[c0:c0 + nb, c0:c0 + nb] = np.tril(Bk)


def _int8_update(C, P, nn, S, e, mutant):
    D, rs, _ = slice_rows(P, S, e=e, wrap=True)       # (the top digit wraps like the kernel's int8 when e is too small)
    Df = D.astype(np.float64)
    accs = []
    for g in range(S):
        pairs = [(s, g - s) for s in range(g + 1)]
        if mutant == "drop_digit" and g == S - 1:
            pairs = pairs[1:]                                 # the (0, S-1) product of order S - 1
        lhs = np.concatenate([Df[s] for s, _ in pairs], axis=1)
        rhs = np.concatenate([Df[t][:nn] for _, t in pairs], axis=1)
        accs.append(lhs @ rhs.T)
    if S == 6 and mutant != "drop33":
        accs.append(Df[3] @ Df[3][:nn].T)
    return syrk_i8_epilogue(np.stack(accs), rs, C)


def emulate(A, n, Y=None, cfg=None, mutant=None):
    """The factor F (L in rows < n, X = Y L^-T below) of the launches of `schedule`, on float64 values in the kernels'
    blocking.  `mutant` names a defect to inject (tests/test_chol_bounds.py)."""
    cfg = cfg or Config()
    rows = n + (0 if Y is None else Y.shape[0])
    F = np.zeros((rows, n))
    F[:n] = np.tril(A)
    F[:n] = F[:n] + np.tril(F[:n], -1).T          # work on the full symmetric square part
    if Y is not None:
        F[n:] = Y
    es = static_exponents(np.diag(A))
    if mutant == "exp_small":
        es = es - 1
    launches = schedule(n, rows, cfg)
    dinv_prev = None
    first_int8 = True
    ext_scale = {}
    nxt = [next((M["c0"] for M in launches[i:] if M["kind"] == "leaf"), None) for i in range(len(launches))]
    snap, early_done = {}, False
    for idx, L in enumerate(launches):
        b = nxt[idx]
        unit = (slice(b + 96, b + 128), slice(b + 96, b + 128)) if b is not None and b > 0 else None
        before = F[unit].copy() if unit is not None and L["kind"] != "leaf" else None
        if L["kind"] == "leaf":
            if mutant == "leaf_early" and not early_done and b in snap:
                F[unit] = snap[b]          # the leaf read its block before the last update of its last 32 x 32 unit
                early_done = True
            _leaf(F, L["c0"], L["nb"], mutant)
        elif L["kind"] == "feed_old":
            c0 = L["c0"]
            t = slice(c0 + NB, c0 + 2 * NB)
            Lold = F[t, L["k0"]:c0]
            F[t, t] -= Lold @ Lold.T
        elif L["kind"] == "panel":
            c0, nb = L["c0"], L["nb"]
            Ljj = np.tril(F[c0:c0 + nb, c0:c0 + nb])
            B = F[c0 + nb:, c0:c0 + nb]
            if L["type"] == "gemm":
                B[:] = B @ sla.solve_triangular(Ljj, np.eye(nb), lower=True, check_finite=False).T
            else:
                w1 = max(nb - 64, 0)
                inv = [sla.solve_triangular(Ljj[o:o + w, o:o + w], np.eye(w), lower=True, check_finite=False)
                       for o, w in ((0, min(nb, 64)), (64, w1))]
                use = dinv_prev if (mutant == "stale_dinv" and dinv_prev is not None and nb == NB) else inv
                dinv_prev = inv
                X1 = B[:, :64] @ use[0].T
                Tm = B[:, 64:] - X1 @ Ljj[64:, :64].T
                B[:, :64], B[:, 64:] = X1, Tm @ use[1].T
            if L["type"] == "fused":
                fc = L["fuse_cols"]
                X = F[c0 + nb:, c0:c0 + nb]
                F[c0 + nb:, c0 + nb:c0 + nb + fc] -= X @ X[:fc].T
            if L["type"] == "feed":
                Xt = F[c0 + nb:c0 + 2 * NB, c0:c0 + nb]
                F[c0 + nb:c0 + 2 * NB, c0 + nb:c0 + 2 * NB] -= Xt @ Xt.T
        else:
            k0, K, r0, m, nn = L["k0"], L["K"], L["r0"], L["m"], L["n"]
            skip = L["row_skip"]
            P = F[r0:r0 + m, k0:k0 + K]
            C = F[r0 + skip:r0 + m, r0:r0 + nn]
            if L["engine"] == "int8":
                e = es[np.minimum(np.arange(r0, r0 + m), n - 1)].copy()
                ext = np.arange(r0, r0 + m) >= (n if cfg.static else 0)
                if ext.any():
                    dyn = row_exponents(P[ext])
                    if mutant == "extra_static":      # the scale of the row's first slicing, kept for later k-ranges
                        for i, gi in enumerate(np.nonzero(ext)[0] + r0):
                            ext_scale.setdefault(gi, dyn[i])
                        dyn = np.array([ext_scale[gi] for gi in np.nonzero(ext)[0] + r0])
                    e[ext] = dyn
                new = _int8_update(np.zeros((m, nn)), P, nn, L["S"], e, mutant)
                upd = -new[skip:]
            else:
                upd = P[skip:] @ P[:nn].T
            if mutant in ("tile_twice", "tile_skip") and first_int8 and L["engine"] == "int8":
                t = np.zeros_like(upd)
                t[NB - skip:2 * NB - skip, :32] = upd[NB - skip:2 * NB - skip, :32]
                upd = upd + t if mutant == "tile_twice" else upd - t
            if L["engine"] == "int8":
                first_int8 = False
            C -= upd
        if before is not None and before.size and not np.array_equal(before, F[unit]):
            snap[b] = before
    return np.where(np.tri(rows, n, dtype=bool), F, 0.0)
