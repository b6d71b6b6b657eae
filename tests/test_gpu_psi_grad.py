"""The adjoints of the RBF psi statistics on the device (psi.cu::psi_backward, through gpk_debug_rbf_psi_grad) element
by element against the exact vector-Jacobian product tests/bgplvm_grad_oracle.py::psi_vjp, within per-element bars
derived below, at every kernel instantiation and chunking edge the launch geometry picks.

Bars.  Every output element is a signed sum of terms t_k (psi_vjp's formulas: one per point, inducing point or pair and
formula term).  With EPS the double epsilon and, from psi_vjp(abs_sums=True), T = sum |t_k|, U the largest exponent
behind the element and C = sum |t_k| kappa_k (the cancellation of diff2 = mu - zbar):
  - the exponent u of a term is a sum of non-negative parts (the log-determinant shifts, (z - z')^2 / 4l^2 and
    diff^2 / (l^2 + S) or / (l^2 + 2S) per active dim), each with at most a few roundings, summed at depth 2 nd + 2:
    |du| <= (3 nd + 8) EPS u, apart from diff2's rounding.  diff2 = mu - zbar cancels, so its error is absolute,
    EPS (|mu| + |zbar|) (zbar = (z + z') / 2 rounded, then the subtraction), and moves the term by at most EPS |t_k|
    kappa_k: through the exponent and through the powers of diff2 the term carries (psi_vjp's docstring).
    psi1's diff = mu - z subtracts stored values: its rounding is relative and counted among the roundings below;
  - exp(-u) is the K-build's table exp, within an ulp (test_gpu_kbuild_accuracy.py), so e = exp(-u) (1 + du + 2 EPS);
  - the products around e (G, sigma^2 twice, the pair weight, diff, a or b and their squares, l, S) add at most 12
    roundings per term: 16 EPS |t_k| with the exp's 2 EPS and the rest;
  - the sums: a term reaches its output through a chain of additions whose depth K the launch geometry fixes (the
    fma chain of the owning thread, the warp and CTA tree of block_add, the atomics across chunks and blocks, and the
    value the output held before the call): at most gamma_K (T + |pre|) <= K EPS (T + |pre|).  K per output is
    computed from the geometry the library reports (depth() below);
  - subnormal results of exp (u > 708) are within one subnormal ulp of the true value, and 0 past u = 1416 where the
    true value is below 2^-2043: their absolute error, times the coefficients of these inputs (below 1e10) summed over
    fewer than 1e10 terms, is below TINY = 1e-300.
So |device - (pre + oracle)| <= (3 nd + 8) EPS U T + EPS C + (16 + K) EPS (T + |pre|) + TINY, and the oracle's own
rounding is of the same kind and size: the bar is taken twice, as test_rbf_psi_within_derived_bound does.

Inputs.  G1 and G2 have mixed signs and magnitudes over six decades, G2 exactly symmetric; G1t, G2 and Z have padded
leading dimensions holding NaN, and with active_dims the columns mu, S and Z do not use hold NaN; the outputs are
pre-filled with non-zero values (the entry ADDS), and every output and the workspace have a guard region behind them;
the workspace starts as NaN.  S runs from 1e-12 l^2 to 1e2 l^2; a few points lie far from every inducing point, so
that exponents pass 624 (the slow path of the table exp), 708 (subnormal results) and 1416 (exact zero)."""
import ctypes
import math
import zlib

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests.bgplvm_grad_oracle import psi_vjp

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
TINY = 1e-300
SENT = -7.25e300
GUARD = 512
OUTS = ("mu", "S", "Z", "variance", "lengthscales")

# name: (N, Q, M, lengthscale kind, active dims (None: all Q), ldz)
CASES = {
    "nd1_n3_m1": (3, 1, 1, "scalar", None, 1),
    "nd8_ard_n29_m2": (29, 8, 2, "ard", None, 8),
    "nd9_ard_ldz": (200, 9, 11, "ard", None, 13),
    "nd12_active_dims": (131, 14, 7, "scalar", [13, 0, 2, 5, 6, 7, 11, 3, 9, 10, 1, 8], 17),
    "nd16_ard": (77, 16, 23, "ard", None, 16),
    "nd17_ard_ldz": (300, 17, 5, "ard", None, 20),
    "nd20_active_dims": (45, 23, 13, "ard", [22, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 15, 16, 17, 18, 19, 21], 23),
    "nd32_ard_ldz": (260, 32, 30, "ard", None, 33),
    "nd32_scalar_n5_m1": (5, 32, 1, "scalar", None, 32),
    "nd2_many_pairs": (1000, 2, 70, "ard", None, 2),
}
# distances (in lengthscales) of the far points: psi1 exponents about r^2 / 2, psi2 exponents about r^2
FAR = (26.0, 36.0, 27.5, 38.0, 54.0)
RATIOS = {}
_CACHE = {}


def _T():
    import torch
    return torch


def _inputs(name):
    N, Q, M, kind, ad, ldz = CASES[name]
    rng = np.random.default_rng(zlib.crc32(name.encode()) % 10000)
    cols = np.arange(Q) if ad is None else np.asarray(ad)
    nd = len(cols)
    ell = math.sqrt(nd) / 2 * (np.full(nd, 1.1) if kind == "scalar" else rng.uniform(0.6, 1.6, nd))
    mu, S, Z = np.full((N, Q), np.nan), np.full((N, Q), np.nan), np.full((M, Q), np.nan)
    mu[:, cols] = rng.standard_normal((N, nd))
    Z[:, cols] = rng.standard_normal((M, nd))
    S[:, cols] = ell ** 2 * 10.0 ** rng.uniform(-12, 2, (N, nd))
    for i, r in enumerate(FAR[:min(len(FAR), max(1, N // 4))]):
        n = N - 1 - i
        v = rng.standard_normal(nd)
        mu[n, cols] = r * ell * v / np.linalg.norm(v)
        S[n, cols] = ell ** 2 * 10.0 ** rng.uniform(-12, -3, nd)
    G1 = rng.choice([-1.0, 1.0], (N, M)) * 10.0 ** rng.uniform(-3, 3, (N, M))
    A = rng.choice([-1.0, 1.0], (M, M)) * 10.0 ** rng.uniform(-3, 3, (M, M))
    G2 = 0.5 * (A + A.T)
    ls = float(ell[0]) if kind == "scalar" else ell
    kp = gpf.kernels.SquaredExponential(variance=1.3, lengthscales=ls, active_dims=ad)
    ko = O.SquaredExponential(1.3, ls, active_dims=ad)
    return dict(N=N, Q=Q, M=M, nd=nd, cols=cols, ldz=ldz, mu=mu, S=S, Z=Z, G1=G1, G2=G2, kp=kp, ko=ko, ell=ell)


def _exponents(c):
    """All psi1 and psi2 exponents of the case (u1 [N, M], u2 [N, M, M])."""
    cols, l2 = c["cols"], c["ell"] ** 2
    ma, Sa, Za = c["mu"][:, cols], c["S"][:, cols], c["Z"][:, cols]
    u1 = 0.5 * np.sum(np.log1p(Sa / l2), 1)[:, None] + 0.5 * np.sum((ma[:, None] - Za[None]) ** 2 / (l2 + Sa)[:, None], -1)
    zbar = 0.5 * (Za[:, None] + Za[None])
    ez = np.sum((Za[:, None] - Za[None]) ** 2 / (4 * l2), -1)
    u2 = np.stack([ez + 0.5 * np.sum(np.log1p(2 * Sa[n] / l2)) + np.sum((ma[n] - zbar) ** 2 / (l2 + 2 * Sa[n]), -1)
                   for n in range(ma.shape[0])])
    return u1, u2


def _guarded(host):
    """A device fp64 copy of host (flattened) followed by GUARD sentinels; returns (view, full)."""
    T = _T()
    n = host.size
    full = T.full((n + GUARD,), SENT, dtype=T.float64, device="cuda")
    full[:n] = T.from_numpy(np.ascontiguousarray(host, dtype=np.float64).reshape(-1)).cuda()
    return full[:n], full


def _device_psi_grad(c, pre):
    """gpk_debug_rbf_psi_grad on the case's inputs, adding into pre; returns ({output: array}, geometry [9])."""
    lib = _lib.load()
    T = _T()
    N, Q, M, ldz, nd = c["N"], c["Q"], c["M"], c["ldz"], c["nd"]
    ldg1, ldg2 = N + 3, M + 2
    Zp = np.full((M, ldz), np.nan)
    Zp[:, :Q] = c["Z"]
    G1t = np.full((M, ldg1), np.nan)
    G1t[:, :N] = c["G1"].T
    G2p = np.full((M, ldg2), np.nan)
    G2p[:, :M] = c["G2"]
    dev = lambda a: T.from_numpy(np.ascontiguousarray(a)).cuda()
    mu_d, S_d, Z_d, G1_d, G2_d = dev(c["mu"]), dev(c["S"]), dev(Zp), dev(G1t), dev(G2p)
    gpar_pre = np.concatenate([[pre["variance"]], pre["lengthscales"]])
    outs = {k: _guarded(pre[k]) for k in ("mu", "S", "Z")}
    outs["gpar"] = _guarded(gpar_pre)
    need, wguard = lib.gpk_rbf_psi_ws(N, M), 1 << 16
    ws = ops.scratch_bytes(need + wguard)
    ws[:need].fill_(0xFF)  # NaN doubles: nothing may be read before it is written
    ws[need:].fill_(0xA5)
    geom = (ctypes.c_int64 * 9)()
    _lib.check(lib.gpk_debug_rbf_psi_grad(*gpf.kernels.compile_kernel(c["kp"], Q), ops._p(mu_d), ops._p(S_d), N, Q,
                                          ops._p(Z_d), M, ldz, ops._p(G1_d), ldg1, ops._p(G2_d), ldg2,
                                          ops._p(outs["mu"][0]), ops._p(outs["S"][0]), ops._p(outs["Z"][0]),
                                          ops._p(outs["gpar"][0]), ops._p(ws), geom, ops._stream()),
               "gpk_debug_rbf_psi_grad")
    T.cuda.synchronize()
    assert bool((ws[need:] == 0xA5).all()), "gpk_debug_rbf_psi_grad wrote past gpk_rbf_psi_ws bytes"
    for k, (view, full) in outs.items():
        assert bool((full[view.numel():] == SENT).all()), f"gpk_debug_rbf_psi_grad wrote past {k}"
    got = {k: outs[k][0].cpu().numpy().reshape(pre[k].shape) for k in ("mu", "S", "Z")}
    gp = outs["gpar"][0].cpu().numpy()
    got["variance"], got["lengthscales"] = gp[0], gp[1:]
    assert gp.size == 1 + nd
    return got, np.array(list(geom), dtype=np.int64)


def depth(geom, N, M):
    """Summation depth K per output: the longest chain of additions from a term to the output, for the launches of
    psi_backward with this geometry (see the module docstring)."""
    ND, PP, tiles, nch, nlen, gn, pch, plen, launches = (int(x) for x in geom)
    point = M + 1 + plen + pch + 2                                # psi1 fma chain, psi2 chain, pair-chunk atomics, pre
    z = 4 * -(-N // 512) + 9 + nlen + (M + 1) * nch + 2            # psi1 thread chain and tree, psi2 atomics per row
    par = max(M, PP * nlen, plen) + PP + 13 + gn + tiles * nch + gn * pch + 2   # thread chains, tree, atomics
    return {"mu": point, "S": point, "Z": z, "variance": par, "lengthscales": par}


def _case(name):
    """Inputs, oracle with magnitude sums, pre-fill, device result and geometry of a case (computed once)."""
    if name in _CACHE:
        return _CACHE[name]
    c = _inputs(name)
    g, sums = psi_vjp(c["mu"], c["S"], c["Z"], c["ko"], c["G1"], c["G2"], abs_sums=True)
    rng = np.random.default_rng(7)
    pre = {}
    for k in OUTS:
        Tk = np.asarray(sums[k][0], dtype=np.float64)
        r = rng.choice([-1.0, 1.0], Tk.shape) * rng.uniform(0.5, 1.5, Tk.shape)
        pre[k] = np.where(Tk > 0, Tk * r, 0.75 * r)     # of the size of the element's terms: no add hides it
    got, geom = _device_psi_grad(c, pre)
    _CACHE[name] = dict(c=c, g=g, sums=sums, pre=pre, got=got, geom=geom)
    return _CACHE[name]


def error_ratios(r):
    """{output: |device - (pre + oracle)| / bar} per element for a case of _case, and (device, want) per output."""
    c, g, sums, pre, got = r["c"], r["g"], r["sums"], r["pre"], r["got"]
    K = depth(r["geom"], c["N"], c["M"])
    nd = c["nd"]
    ratios, pairs = {}, {}
    for k in OUTS:
        T, U, C = (np.asarray(x, dtype=np.float64) for x in sums[k])
        want = np.asarray(pre[k]) + np.asarray(g[k])
        dev = np.asarray(got[k], dtype=np.float64)
        bar = 2 * ((3 * nd + 8) * EPS * U * T + EPS * C + (16 + K[k]) * EPS * (T + np.abs(pre[k]))) + TINY
        with np.errstate(invalid="ignore"):
            ratios[k] = np.where(np.isfinite(dev), np.abs(dev - want) / bar, np.inf)
        pairs[k] = (dev, want)
    return ratios, pairs


@pytest.mark.parametrize("name", list(CASES))
def test_psi_adjoints_within_derived_bars(cuda_device, name):
    r = _case(name)
    ratios, pairs = error_ratios(r)
    worst = {k: float(np.max(v)) for k, v in ratios.items()}
    RATIOS[name] = worst
    print(f"{name}: geometry {list(map(int, r['geom']))}; max error / bar " +
          " ".join(f"d{k} {v:.3g}" for k, v in worst.items()))
    for k, v in ratios.items():
        i = np.unravel_index(np.argmax(v), np.shape(v)) if np.ndim(v) else ()
        dev, want = (np.asarray(x)[i] for x in pairs[k])
        assert worst[k] <= 1.0, f"{name} d{k}{list(i)}: device {dev!r}, oracle {want!r}, error / bar {worst[k]:.3g}"


def test_case_table_reaches_every_launch_shape(cuda_device):
    """From the geometry the library reports: all three buckets and both halves of the ND = 32 split (with 1 and 16
    live dims in the second), one point chunk and several with a partial last one, one pair chunk and several with a
    partial last 64-pair staging group, a partial last pair tile and a partial last point block; and exponents past
    624, 708 and 1416 in psi1 and psi2."""
    seen = dict(buckets=set(), second_half=set(), one_point_chunk=False, point_chunks_partial=False,
                one_pair_chunk=False, pair_chunks_partial_group=False, partial_tile=False, several_tiles=False,
                partial_point_block=False)
    u1_all, u2_all = [], []
    for name in CASES:
        r = _case(name)
        N, M, nd = r["c"]["N"], r["c"]["M"], r["c"]["nd"]
        ND, PP, tiles, nch, nlen, gn, pch, plen, launches = (int(x) for x in r["geom"])
        np_ = M * (M + 1) // 2
        # the geometry is the one the rules give: every point and pair covered once, chunks in whole staging groups
        assert ND == (8 if nd <= 8 else 16 if nd <= 16 else 32) and PP == {8: 4, 16: 2, 32: 1}[ND]
        assert launches == (2 if ND == 32 else 1)
        assert tiles == -(-np_ // (256 * PP)) and gn == -(-N // 128)
        assert nlen % 32 == 0 and (nch - 1) * nlen < N <= nch * nlen
        assert plen % 64 == 0 and (pch - 1) * plen < np_ <= pch * plen
        seen["buckets"].add(ND)
        if ND == 32:
            seen["second_half"].add(nd - 16)
        seen["one_point_chunk"] |= nch == 1
        seen["point_chunks_partial"] |= nch > 1 and N % nlen != 0
        seen["one_pair_chunk"] |= pch == 1
        seen["pair_chunks_partial_group"] |= pch > 1 and (np_ - (pch - 1) * plen) % 64 != 0
        seen["partial_tile"] |= np_ % (256 * PP) != 0
        seen["several_tiles"] |= tiles > 1
        seen["partial_point_block"] |= gn > 1 and N % 128 != 0
        u1, u2 = _exponents(r["c"])
        u1_all.append(u1.reshape(-1))
        u2_all.append(u2.reshape(-1))
    assert seen.pop("buckets") == {8, 16, 32}
    assert {1, 16} <= seen.pop("second_half")
    assert all(seen.values()), seen
    for u in (np.concatenate(u1_all), np.concatenate(u2_all)):
        for lo, hi in ((624, 708), (708, 745), (1416, np.inf)):
            assert np.any((u > lo) & (u < hi)), (lo, hi)
