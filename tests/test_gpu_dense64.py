"""The fp64 dense linear algebra under the device gradients, element by element against the derived bars of
tests/dense64_bounds.py: the tiled GEMM on every tile shape, transposition and flag, the inverse-based triangular
solve, the inverse chain (POTRI, LAUUM, the whitened Cholesky adjoint) through gpk_debug_inverse_chain, and the public
GEMM's in-place rule.  tests/_dense64_worker.py runs the same GEMM / TRSM / POTRI cases under GPK_FP64_SIMT=1."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dense64_bounds as DB

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64, F32 = 1, 0
SENT = -777.25
# One step of the fp32 paths.  3xTF32 with truncating splits: a = hi + lo + e with |e| <= 2^-20 |a|, the dropped
# lo * lo term another 2^-20 |a b|, the fp32 accumulation one 2^-24 rounding per step: u = 2^-18 bounds a step; the
# CUDA-core fp32 kernel (u = 2^-24) is inside the same bound
U_TF32 = 2.0 ** -18


def _t():
    import torch
    return torch


def lib():
    from gpflow_b200 import _lib
    return _lib.load()


def dev(a, dtype=np.float64):
    return _t().from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def ptr(x, off=0):
    return ctypes.c_void_p(x.data_ptr() + off * x.element_size())


def sync():
    _t().cuda.synchronize()


def err():
    return lib().gpk_last_error().decode()


# ---- GEMM ------------------------------------------------------------------------------------------------------------
def run_gemm(A, B, C0, alpha, beta, ta, tb, flags, ldpad=0, offset=0, dtype=np.float64, ld_parity=None):
    """C = alpha op(A) op(B) + beta C0 through gpk_gemm, every operand a view with leading dimension + ldpad (rounded
    up to the parity ld_parity if given) at element `offset` of row 1 of a sentinel-filled parent.  Returns (C, parent
    of C after the call, parent before)."""
    m, n = C0.shape
    def parent(M):
        w = M.shape[1] + ldpad + offset + 1
        if ld_parity is not None and w % 2 != ld_parity:
            w += 1
        P = np.full((M.shape[0] + 2, w), SENT)
        P[1:1 + M.shape[0], offset:offset + M.shape[1]] = M
        return P
    PA, PB, PC = parent(A), parent(B), parent(C0)
    dA, dB, dC = dev(PA, dtype), dev(PB, dtype), dev(PC, dtype)
    def view(d, P):
        return ptr(d, P.shape[1] + offset), P.shape[1]
    (pa, lda), (pb, ldb), (pc, ldc) = view(dA, PA), view(dB, PB), view(dC, PC)
    rc = lib().gpk_gemm(ta, tb, m, n, A.shape[0] if ta else A.shape[1], alpha, pa, lda, pb, ldb, beta, pc,
                        ldc, F64 if dtype == np.float64 else F32, flags, None)
    assert rc == 0, err()
    sync()
    out = dC.cpu().numpy().astype(np.float64)
    return out[1:1 + m, offset:offset + n], out, PC


def check_gemm(A, B, C0, alpha, beta, ta, tb, flags, C, rng):
    """Worst error / bar of the device C: long double on every tile-edge row and column plus random ones, and over
    the whole matrix against the fp64 BLAS product (bar doubled: BLAS has the same bound)."""
    m, n = C0.shape
    rows, cols = DB.edge_indices(m, rng), DB.edge_indices(n, rng)
    a_lower = bool(flags & DB.GEMM_A_LOWER)
    C0z = np.nan_to_num(C0) if beta == 0 else C0
    ref, bar = DB.gemm_ref(A, B, C0z, alpha, beta, ta, tb, rows, cols, a_lower)
    r = DB.ratio(np.abs(C[np.ix_(rows, cols)].astype(np.longdouble) - ref), bar)
    As = np.tril(A) if a_lower else A
    oa, ob = DB.opmat(np.nan_to_num(As), ta), DB.opmat(B, tb)
    full = alpha * (oa @ ob) + (beta * C0 if beta != 0 else 0.0)
    k = oa.shape[1]
    mag = abs(alpha) * (np.abs(oa) @ np.abs(ob)) + (abs(beta) * np.abs(C0) if beta != 0 else 0.0)
    rf = DB.ratio(np.abs(C - full), 2 * DB.gamma(k + 2) * mag * (1 + 1e-6) + np.finfo(float).tiny)
    return max(r, rf)


def operands(m, n, k, ta, tb, rng, a_lower=False):
    A = rng.standard_normal((k, m) if ta else (m, k))
    if a_lower:
        A[np.triu_indices(A.shape[0], 1, A.shape[1])] = np.nan   # the stored strict upper part is never read
    B = rng.standard_normal((n, k) if tb else (k, n))
    return A, B, rng.standard_normal((m, n))


# (m, n, k) per tile shape: ragged, and the k of each transposition from the issue's list
TILE_SHAPES = {
    (128, 128): (1401, 1403, [16, 77, 1000, 17]),
    (128, 64): (100, 6343, [17, 1000, 3, 77]),
    (128, 32): (127, 301, [4099, 3, 15, 0]),
    (64, 128): (1001, 903, [15, 1000, 1, 77]),
    (32, 128): (301, 123, [1, 0, 4099, 16]),
}
TRANS = [(0, 0), (0, 1), (1, 0), (1, 1)]
GEMM_CASES = [(tile, ta, tb, TILE_SHAPES[tile][2][i]) for tile in TILE_SHAPES for i, (ta, tb) in enumerate(TRANS)]
WORST = {}


def record(name, r):
    lo, hi = WORST.get(name, (np.inf, 0.0))
    WORST[name] = (min(lo, r), max(hi, r))


def gemm_case(tile, ta, tb, k, seed):
    m, n, _ = TILE_SHAPES[tile]
    assert DB.dmma_tile(m, n, 0, None, tb, k) == tile
    rng = np.random.default_rng(seed)
    A, B, C0 = operands(m, n, k, ta, tb, rng)
    beta = [0.0, 1.0, 0.3, 0.0][(ta * 2 + tb)]
    if beta == 0:
        C0[:] = np.nan                                                  # beta = 0: C is never read
    return A, B, C0, -0.7 if ta else 1.3, beta


@pytest.mark.parametrize("tile,ta,tb,k", GEMM_CASES)
def test_gemm_tile_shapes_inside_bar(cuda_device, tile, ta, tb, k):
    A, B, C0, alpha, beta = gemm_case(tile, ta, tb, k, hash((tile, ta, tb)) % 1000)
    rng = np.random.default_rng(1)
    C, _, _ = run_gemm(A, B, C0, alpha, beta, ta, tb, 0)
    r = check_gemm(A, B, C0, alpha, beta, ta, tb, 0, C, rng)
    record("gemm", r)
    assert r <= 1.0, r


def test_gemm_cases_reach_every_tile_shape_in_every_transposition():
    assert {(t, ta, tb) for t, ta, tb, _ in GEMM_CASES} == {(t, ta, tb) for t in DB.TILES for ta, tb in TRANS}


LOWER_ONLY_SHAPES = [((128, 128), 1400, 1400), ((128, 64), 100, 6400), ((128, 32), 120, 300), ((64, 128), 1000, 900),
                     ((32, 128), 300, 300)]
LOWER_ONLY_VARIANTS = ["plain", "a_lower_syrk", "beta1"]


@pytest.mark.parametrize("tile,m,n", LOWER_ONLY_SHAPES)
@pytest.mark.parametrize("variant", LOWER_ONLY_VARIANTS)
def test_gemm_lower_only_leaves_untouched_tiles_bit_identical(cuda_device, tile, m, n, variant):
    """LOWER_ONLY: tiles whose columns start right of their last row keep the sentinel bit for bit; every entry of the
    other tiles is inside the bar.  a_lower_syrk is lauum's leaf (A_LOWER | LOWER_ONLY, A^T A with NaN above A's
    diagonal), beta1 dense_sig's accumulation (beta = 1)."""
    rng = np.random.default_rng(m + n)
    flags = DB.GEMM_LOWER_ONLY
    k = 77
    ta, tb, beta = 0, 1, 0.0
    if variant == "a_lower_syrk":
        flags |= DB.GEMM_A_LOWER
        k, ta, tb = m, 1, 0
    A, B, C0 = operands(m, n, k, ta, tb, rng, a_lower=variant == "a_lower_syrk")
    if variant == "beta1":
        beta = 1.0
    else:
        C0[:] = SENT
    assert DB.dmma_tile(m, n, flags, None, tb, k) == tile
    C, _, _ = run_gemm(A, B, C0, 1.0, beta, ta, tb, flags)
    mask = DB.tiles_written(m, n, tile, flags)
    assert (~mask).any()
    assert np.array_equal(C[~mask].view(np.int64), C0[~mask].view(np.int64))
    C2 = np.where(mask, C, np.nan)
    rows, cols = DB.edge_indices(m, rng), DB.edge_indices(n, rng)
    keep = mask[np.ix_(rows, cols)]
    ref, bar = DB.gemm_ref(np.nan_to_num(A), B, C0, 1.0, beta, ta, tb, rows, cols, bool(flags & DB.GEMM_A_LOWER))
    r = DB.ratio(np.abs(C2[np.ix_(rows, cols)].astype(np.longdouble) - ref)[keep], bar[keep])
    record("gemm", r)
    assert r <= 1.0, r


A_LOWER_SHAPES = [(300, 203, 300), (1401, 1403, 1401), (100, 6343, 100)]


@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("m,n,k", A_LOWER_SHAPES)
def test_gemm_a_lower_never_reads_the_stored_upper_part(cuda_device, ta, m, n, k):
    rng = np.random.default_rng(m * 3 + ta)
    A, B, C0 = operands(m, n, k, ta, 0, rng, a_lower=True)
    C, _, _ = run_gemm(A, B, C0, -1.1, 0.5, ta, 0, DB.GEMM_A_LOWER)
    assert np.isfinite(C).all()
    r = check_gemm(A, B, C0, -1.1, 0.5, ta, 0, DB.GEMM_A_LOWER, C, rng)
    record("gemm", r)
    assert r <= 1.0, r


@pytest.mark.parametrize("ta", [0, 1])
def test_tf32_gemm_a_lower_never_reads_the_stored_upper_part(cuda_device, ta):
    """The 3xTF32 fp32 path makes the same promise as the DMMA kernel."""
    m = n = k = 640
    assert DB.dmma_tile(m, n, DB.GEMM_A_LOWER, None, 0, k, np.float32) == "tf32"
    rng = np.random.default_rng(40 + ta)
    A, B, C0 = operands(m, n, k, ta, 0, rng, a_lower=True)
    A, B, C0 = (x.astype(np.float32).astype(np.float64) for x in (A, B, C0))
    C, _, _ = run_gemm(A, B, C0, 1.0, 0.0, ta, 0, DB.GEMM_A_LOWER, dtype=np.float32)
    assert np.isfinite(C).all()
    oa = DB.opmat(np.tril(np.nan_to_num(A)), ta)
    bar = (DB.gamma(k + 2, U_TF32)) * (np.abs(oa) @ np.abs(B))
    assert DB.ratio(np.abs(C - oa @ B), bar) <= 1.0


COLSUMSQ_SHAPES = [(301, 203, 77), (127, 1030, 17)]


@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("m,n,k", COLSUMSQ_SHAPES)
def test_gemm_colsumsq_accumulates_inside_bar(cuda_device, ta, m, n, k):
    rng = np.random.default_rng(m + n + ta)
    A, B, _ = operands(m, n, k, ta, 0, rng)
    v0 = rng.uniform(0.5, 2.0, n)
    dA, dB, dv = dev(A), dev(B), dev(v0)
    assert lib().gpk_gemm(ta, 0, m, n, k, 0.9, ptr(dA), A.shape[1], ptr(dB), n, 0.0, ptr(dv), 0, F64,
                          DB.GEMM_COLSUMSQ, None) == 0, err()
    sync()
    got = dv.cpu().numpy()
    oa = DB.opmat(A, ta)
    P = oa.astype(np.longdouble) @ B.astype(np.longdouble) * np.longdouble(0.9)
    ref = v0 + (P ** 2).sum(axis=0)
    mag = ((0.9 * (np.abs(oa) @ np.abs(B))) ** 2).sum(axis=0)
    bar = (2 * DB.gamma(k + 1) + DB.gamma(m + 1)) * mag + DB.gamma(1) * (v0 + mag) + 1e-300
    r = DB.ratio(np.abs(got - ref), bar * (1 + 1e-6))
    record("colsumsq", r)
    assert r <= 1.0, r


VIEW_CASES = [(tile, layout) for tile in [(128, 32), (64, 128), (128, 128)] for layout in ("odd_ld", "unaligned_base")]


@pytest.mark.parametrize("tile,layout", VIEW_CASES)
def test_gemm_unaligned_views_keep_their_sentinels(cuda_device, tile, layout):
    """The two halves of the epilogue's vector test, each alone: an odd leading dimension with a 16-byte aligned C
    base, and an even leading dimension with a C base one element past a 16-byte boundary.  Both take the scalar
    stores; nothing outside the views is written."""
    m, n, ks = TILE_SHAPES[tile]
    rng = np.random.default_rng(7)
    A, B, C0 = operands(m, n, 77, 0, 1, rng)
    parity = 1 if layout == "odd_ld" else 0
    C, after, before = run_gemm(A, B, C0, 0.8, 1.0, 0, 1, 0, ldpad=2, offset=1, ld_parity=parity)
    ldc, base = after.shape[1], after.shape[1] + 1              # C starts at row 1, column 1 of its parent
    assert ldc % 2 == parity and base % 2 == (1 if layout == "unaligned_base" else 0)
    inside = np.zeros(after.shape, dtype=bool)
    inside[1:1 + m, 1:1 + n] = True
    assert np.array_equal(after[~inside], before[~inside])
    r = check_gemm(A, B, C0, 0.8, 1.0, 0, 1, 0, C, rng)  # (torch allocations are 256-byte aligned)
    record("gemm", r)
    assert r <= 1.0, r


@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("n", [1, 16])
def test_gemm_skinny_kernel_inside_bar(cuda_device, ta, n):
    m, k = 300, 1029                                         # k not a multiple of 8 x 128
    assert DB.dmma_tile(m, n, 0, None, 0, k) == "skinny"
    rng = np.random.default_rng(n + ta)
    A, B, C0 = operands(m, n, k, ta, 0, rng)
    C, _, _ = run_gemm(A, B, C0, -0.6, 0.4, ta, 0, 0)
    r = check_gemm(A, B, C0, -0.6, 0.4, ta, 0, 0, C, rng)
    record("gemm", r)
    assert r <= 1.0, r


IN_PLACE_CASES = [("B", 100, 300, (128, 32)), ("B", 128, 15500, (128, 128)), ("A", 2000, 100, (32, 128)),
                  ("A", 15400, 128, (128, 128))]


@pytest.mark.parametrize("which,m,n,tile", IN_PLACE_CASES)
def test_gemm_in_place_within_the_rule(cuda_device, which, m, n, tile):
    """C == B with m <= 128 and C == A with n <= 128 through the public entry, the aliased leaf on 128 x 128 tiles
    included."""
    rng = np.random.default_rng(m + n)
    if which == "B":
        A, X = rng.standard_normal((m, m)), rng.standard_normal((m, n))
        ref = A.astype(np.longdouble) @ X.astype(np.longdouble)
        mag = np.abs(A) @ np.abs(X)
        k = m
    else:
        X, Bm = rng.standard_normal((m, n)), rng.standard_normal((n, n))
        ref = X.astype(np.longdouble) @ Bm.astype(np.longdouble)
        mag = np.abs(X) @ np.abs(Bm)
        k = n
    assert DB.dmma_tile(m, n, 0, which, 0, k) == tile
    dX = dev(X)
    if which == "B":
        dA = dev(A)
        rc = lib().gpk_gemm(0, 0, m, n, m, 1.0, ptr(dA), m, ptr(dX), n, 0.0, ptr(dX), n, F64, 0, None)
    else:
        dBm = dev(Bm)
        rc = lib().gpk_gemm(0, 0, m, n, n, 1.0, ptr(dX), n, ptr(dBm), n, 0.0, ptr(dX), n, F64, 0, None)
    assert rc == 0, err()
    sync()
    r = DB.ratio(np.abs(dX.cpu().numpy() - ref), DB.gamma(k + 2) * mag + 1e-300)
    record("gemm", r)
    assert r <= 1.0, r


@pytest.mark.parametrize("which,m,n,k,trans,ld_off", [
    ("B", 300, 50, 300, 0, 0), ("B", 129, 129, 129, 0, 0),    # no tile spans m
    ("A", 50, 300, 300, 0, 0),                                # no tile spans n
    ("AB", 64, 64, 64, 0, 0),                                 # no tile spans both
    ("B", 64, 256, 64, 1, 0),                                 # transb: column CTAs read rows other CTAs store
    ("A", 256, 64, 64, 1, 0),                                 # transa: likewise
    ("B", 64, 100, 64, 0, 1),                                 # ldb != ldc: the same pointer, another matrix
    ("A", 100, 64, 64, 0, 1)])
def test_gemm_refuses_in_place_it_cannot_honour(cuda_device, which, m, n, k, trans, ld_off):
    """Outside the in-place rule the CTAs would read elements other CTAs overwrite: gpk_gemm refuses and launches
    nothing."""
    X = dev(np.ones((512, 512)))
    Y = dev(np.ones((512, 512)))
    A = X if "A" in which else Y
    B = X if "B" in which else Y
    ta = trans if which == "A" else 0
    tb = trans if which == "B" else 0
    lda = 512 - (ld_off if which == "A" else 0)
    ldb = 512 - (ld_off if which == "B" else 0)
    rc = lib().gpk_gemm(ta, tb, m, n, k, 1.0, ptr(A), lda, ptr(B), ldb, 0.0, ptr(X), 512, F64, 0, None)
    assert rc == -1
    assert "in place needs C == B with transb = 0, ldb == ldc, m <= 128 or C == A with transa = 0" in err()
    assert float(X.sum()) == X.numel()


# ---- TRSM ------------------------------------------------------------------------------------------------------------
def factor_on_device(L0, dtype=np.float64, ldpad=3):
    """gpk_potrf on K = L0 L0^T stored lower with NaN above the diagonal, in a buffer of leading dimension n + ldpad.
    Returns (device buffer, ld, L as factored (NaN / scratch above the diagonal), dinv blocks)."""
    n = L0.shape[0]
    K = L0 @ L0.T
    ld = n + ldpad
    P = np.full((n, ld), np.nan)
    P[:, :n] = np.where(np.tri(n, dtype=bool), K, np.nan)
    dP = dev(P, dtype)
    dc = F64 if dtype == np.float64 else F32
    ws = _t().empty(int(lib().gpk_potrf_ws(n, n, dc)), dtype=_t().uint8, device="cuda")
    info = _t().zeros(1, dtype=_t().int32, device="cuda")
    assert lib().gpk_potrf(ptr(dP), n, n, ld, dc, ptr(info), ptr(ws), None) == 0, err()
    sync()
    assert int(info.item()) == 0
    return dP, ld, ws, dinv_blocks(ws, n, dtype)


def load_factor(L0, ldpad=3):
    """L0 stored lower with NaN above the diagonal, its block inverses recomputed by gpk_trsm (dinv = NULL) into the
    workspace: the route for factors whose K = L0 L0^T is too ill-conditioned to factor on the int8 engine."""
    n = L0.shape[0]
    ld = n + ldpad
    P = np.full((n, ld), np.nan)
    P[:, :n] = np.where(np.tri(n, dtype=bool), L0, np.nan)
    dP = dev(P)
    ws = _t().empty(int(lib().gpk_trsm_ws(n, F64)), dtype=_t().uint8, device="cuda")
    b = dev(np.zeros((n, 1)))
    assert lib().gpk_trsm(0, ptr(dP), n, ld, ptr(b), 1, 1, F64, None, ptr(ws), None) == 0, err()
    sync()
    return dP, ld, ws, dinv_blocks(ws, n)


def dinv_blocks(ws, n, dtype=np.float64):
    nb = -(-n // DB.NB)
    isz = np.dtype(dtype).itemsize
    raw = ws[: nb * DB.NB * DB.NB * isz].cpu().numpy().view(dtype).astype(np.float64).reshape(nb, DB.NB, DB.NB)
    return [raw[b, : min(DB.NB, n - b * DB.NB), : min(DB.NB, n - b * DB.NB)] for b in range(nb)]


def rhs_sample(nrhs, rng):
    if nrhs <= 256:
        return DB.edge_indices(nrhs, rng, extra=4)
    head = [i for e in range(0, 513, 32) for i in (e - 1, e) if 0 <= i < nrhs]
    tail = [nrhs - 1, nrhs - 2, (nrhs // 128) * 128, (nrhs // 128) * 128 - 1]
    return np.array(sorted(i for i in set(head + tail + rng.integers(0, nrhs, 6).tolist()) if 0 <= i < nrhs))


def run_trsm(dP, ld, L, ws, n, nrhs, trans, cached, rng, dtype=np.float64):
    """gpk_trsm on a strided view of B inside a sentinel-filled parent; returns (B0, X, dinv blocks used)."""
    B0 = rng.standard_normal((n, nrhs))
    if dtype == np.float32:
        B0 = B0.astype(np.float32).astype(np.float64)
    P = np.full((n + 2, nrhs + 3), SENT)
    P[1:n + 1, 1:nrhs + 1] = B0
    dB = dev(P, dtype)
    dc = F64 if dtype == np.float64 else F32
    tws = None if cached else _t().empty(int(lib().gpk_trsm_ws(n, dc)), dtype=_t().uint8, device="cuda")
    rc = lib().gpk_trsm(trans, ptr(dP), n, ld, ptr(dB, nrhs + 4), nrhs, nrhs + 3, dc,
                        ptr(ws) if cached else None, ptr(tws) if tws is not None else None, None)
    assert rc == 0, err()
    sync()
    out = dB.cpu().numpy().astype(np.float64)
    inside = np.zeros(P.shape, dtype=bool)
    inside[1:n + 1, 1:nrhs + 1] = True
    assert np.array_equal(out[~inside], P[~inside])
    return B0, out[1:n + 1, 1:nrhs + 1], dinv_blocks(ws if cached else tws, n, dtype)


TRSM_N = [1, 127, 128, 129, 255, 256, 257, 640, 1000, 2048, 4099]
TRSM_CASES = [(n, r) for n in TRSM_N for r in (1, 17, 200)] + [(n, r) for n in (128, 257, 2048) for r in (16, 4096, 15500)]
ENGINE_TRSM = [(129, 17), (257, 200), (1000, 200), (2048, 17), (2048, 4096), (128, 15500)]
COND = {640: 1e6, 1000: 1e4, 2048: 1e6, 257: 1e3}
_FACTORS = {}


def factor(n, dtype=np.float64):
    if (n, dtype) not in _FACTORS:
        rng = np.random.default_rng(n)
        L0 = DB.factor_with_block_cond(n, rng, COND.get(n, 1.0))
        dP, ld, ws, Xb = load_factor(L0) if n in COND else factor_on_device(L0, dtype)
        L = dP.cpu().numpy().astype(np.float64)[:, :n]
        _FACTORS[(n, dtype)] = (dP, ld, ws, np.where(np.tri(n, dtype=bool), L, 0.0))
    return _FACTORS[(n, dtype)]


@pytest.mark.parametrize("n,nrhs", TRSM_CASES)
@pytest.mark.parametrize("trans", [0, 1])
def test_trsm_residual_inside_bar(cuda_device, n, nrhs, trans):
    dP, ld, ws, L = factor(n)
    rng = np.random.default_rng(n * 7 + nrhs + trans)
    cached = (n + nrhs + trans) % 2 == 0 or n in (128, 2048)
    for c in ([True, False] if n in (128, 257, 2048) and nrhs == 17 else [cached]):
        B0, X, Xb = run_trsm(dP, ld, L, ws, n, nrhs, trans, c, rng)
        assert np.isfinite(X).all()
        r, kap, eta = DB.trsm_check(L, B0, X, Xb, trans, rhs_sample(nrhs, rng))
        record("trsm", r)
        assert r <= 1.0, (r, kap, eta)
        if n in COND and COND[n] >= 1e6:
            assert kap > 1e5


TRSM32_CASES = [(640, 17), (1000, 200), (128, 12208), (100, 20000)]


@pytest.mark.parametrize("n,nrhs", TRSM32_CASES)
@pytest.mark.parametrize("trans", [0, 1])
def test_trsm_fp32_inside_bar(cuda_device, n, nrhs, trans):
    """fp32 under the same residual bar with u = U_TF32: n >= 512 solves with the block inverses of the widened
    (fp64-factored) factor; 64 <= n <= 128 with nrhs >= 12208 runs the in-place leaf on 3xTF32 with C aliasing B."""
    if n <= 128:
        assert DB.dmma_tile(n, nrhs, 0, "B", 0, n, np.float32) == "tf32"
    rng = np.random.default_rng(n + nrhs)
    L0 = DB.factor_with_block_cond(n, rng, 1.0).astype(np.float32).astype(np.float64)
    dP, ld, ws, _ = factor_on_device(L0, np.float32)
    L = np.where(np.tri(n, dtype=bool), dP.cpu().numpy().astype(np.float64)[:, :n], 0.0)
    B0, X, Xb = run_trsm(dP, ld, L, ws, n, nrhs, trans, True, rng, np.float32)
    r, _, _ = DB.trsm_check(L, B0, X, Xb, trans, rhs_sample(nrhs, rng), u=U_TF32)
    record("trsm_fp32", r)
    assert r <= 1.0, r


# ---- inverse chain ---------------------------------------------------------------------------------------------------
CHAIN_N = [1, 64, 127, 128, 129, 200, 256, 257, 383, 1000, 2048, 2500]


def chain(op, dL, n, ld, ws, out_ld, T=None):
    out = _t().full((n, out_ld), SENT, dtype=_t().float64, device="cuda")
    tmp = _t().empty(max(1, int(lib().gpk_debug_inverse_chain_ws(op, n))), dtype=_t().uint8, device="cuda")
    rc = lib().gpk_debug_inverse_chain(op, ptr(dL), n, ld, ptr(ws), ptr(T) if T is not None else None, ptr(out),
                                       out_ld, ptr(tmp), None)
    assert rc == 0, err()
    sync()
    return out.cpu().numpy()


def diag_blocks(n):
    blk = np.zeros((n, n), dtype=bool)
    for o in range(0, n, DB.NB):
        blk[o:o + DB.NB, o:o + DB.NB] = True
    return blk


def nan_above(dP, n):
    up = _t().from_numpy(np.triu(np.ones((n, n), dtype=bool), 1)).cuda()
    dP[:, :n][up] = float("nan")


@pytest.mark.parametrize("n", CHAIN_N)
def test_potri_and_lauum_inside_bars(cuda_device, n):
    """POTRI: L <- L^-1 (diagonal blocks = the cached inverses bit for bit, zero above their diagonal, NaN kept above
    the other blocks: never read, never written), every split's identity inside its bar; out <- K^-1 inside the lauum
    bar against the device's own L^-1, out's entries above the diagonal outside the diagonal blocks untouched.  LAUUM
    alone on that L^-1, given NaN everywhere above its diagonal except the zero strict upper parts of the diagonal
    blocks that it requires, gives the same lower triangle."""
    rng = np.random.default_rng(n)
    ill = n in (1000, 2048)
    L0 = DB.factor_with_block_cond(n, rng, 1e6 if ill else 1.0)
    dP, ld, ws, Xb = load_factor(L0) if ill else factor_on_device(L0, ldpad=3 if n % 2 else 0)
    nan_above(dP, n)
    L = np.tril(dP.cpu().numpy()[:, :n])
    out_ld = n + 1
    K = chain(0, dP, n, ld, ws, out_ld)
    X = dP.cpu().numpy()[:, :n]
    up, blk = np.triu(np.ones((n, n), dtype=bool), 1), diag_blocks(n)
    assert np.isnan(X[up & ~blk]).all()
    assert (X[up & blk] == 0).all()
    for b, Xi in enumerate(Xb):
        o = b * DB.NB
        nb = Xi.shape[0]
        assert np.array_equal(np.tril(X[o:o + nb, o:o + nb]), np.tril(Xi))
    Xl = np.where(up, 0.0, X)
    r = DB.trtri_check(L, Xl, rng)
    record("trtri", r)
    assert r <= 1.0, r
    rows, cols = DB.edge_indices(n, rng), DB.edge_indices(n, rng)
    lcheck = DB.lauum_check(Xl, rows, cols)
    assert (K[:, :n][up & ~blk] == SENT).all() and (K[:, n:] == SENT).all()
    r = lcheck(K[:, :n])
    record("lauum", r)
    assert r <= 1.0, r
    up_d = _t().from_numpy(up).cuda()
    blk_d = _t().from_numpy(blk).cuda()
    dP[:, :n][up_d & ~blk_d] = float("nan")                      # LAUUM's input, written here rather than taken
    dP[:, :n][up_d & blk_d] = 0.0                                # from POTRI
    K2 = chain(1, dP, n, ld, ws, out_ld)
    low = ~up
    assert np.array_equal(K2[:, :n][low], K[:, :n][low])
    assert (K2[:, :n][up & ~blk] == SENT).all()


@pytest.mark.parametrize("n", [1, 127, 129, 257, 383, 1000, 2048])
def test_chol_adjoint_symmetric_and_inside_bar(cuda_device, n):
    rng = np.random.default_rng(n + 5)
    L0 = DB.factor_with_block_cond(n, rng, 1e4 if n >= 1000 else 1.0)
    dP, ld, ws, Xb = load_factor(L0) if n >= 1000 else factor_on_device(L0)
    nan_above(dP, n)
    L = np.tril(dP.cpu().numpy()[:, :n])
    T = rng.standard_normal((n, n))
    Tp = np.zeros((n, ld))
    Tp[:, :n] = T
    dT = dev(Tp)
    G = chain(2, dP, n, ld, ws, ld, T=dT)[:, :n]
    assert np.array_equal(G, G.T)
    kap, eta = DB.block_stats(L, Xb, 1)
    bar = DB.chol_adjoint_bar(L, T, kap.max(), eta.max())
    r = DB.ratio(np.abs(G - DB.chol_adjoint_ref(L, T)), bar)
    record("chol_adjoint", r)
    assert r <= 1.0, r


def test_inverse_chain_rejects_bad_arguments(cuda_device):
    x = dev(np.eye(4))
    assert lib().gpk_debug_inverse_chain(7, ptr(x), 4, 4, ptr(x), None, ptr(x), 4, ptr(x), None) == -1
    assert lib().gpk_debug_inverse_chain(2, ptr(x), 4, 4, ptr(x), ptr(x), ptr(x), 5, None, None) == -1


# ---- engine switch ---------------------------------------------------------------------------------------------------
# The cases the fp64 CUDA-core engine reruns: every GEMM list (the tri mask, COLSUMSQ, LOWER_ONLY sentinels, views and
# in-place aliasing each have their own code in that kernel; the skinny kernel does not depend on the switch and runs
# as a control), TRSM over every recursion depth up to 2048 and the aliased 128 x 128 leaf, POTRI / LAUUM at ill- and
# well-conditioned sizes.
def engine_cases():
    m = sys.modules[__name__]
    g = [(m.test_gemm_tile_shapes_inside_bar, c) for c in GEMM_CASES]
    g += [(m.test_gemm_lower_only_leaves_untouched_tiles_bit_identical, (t, mm, nn, v))
          for (t, mm, nn) in LOWER_ONLY_SHAPES for v in LOWER_ONLY_VARIANTS]
    g += [(m.test_gemm_a_lower_never_reads_the_stored_upper_part, (ta, *s_)) for s_ in A_LOWER_SHAPES for ta in (0, 1)]
    g += [(m.test_gemm_colsumsq_accumulates_inside_bar, (ta, *s_)) for s_ in COLSUMSQ_SHAPES for ta in (0, 1)]
    g += [(m.test_gemm_unaligned_views_keep_their_sentinels, c) for c in VIEW_CASES]
    g += [(m.test_gemm_skinny_kernel_inside_bar, (ta, n)) for n in (1, 16) for ta in (0, 1)]
    g += [(m.test_gemm_in_place_within_the_rule, c) for c in IN_PLACE_CASES]
    g += [(m.test_trsm_residual_inside_bar, (n, r, t)) for (n, r) in ENGINE_TRSM for t in (0, 1)]
    g += [(m.test_potri_and_lauum_inside_bars, (n,)) for n in (129, 383, 1000, 2048)]
    return g


def test_fp64_cuda_core_engine_inside_the_same_bars(cuda_device, tmp_path):
    """GPK_FP64_SIMT=1 (read once per process): engine_cases() run on the fp64 CUDA-core kernel in a worker process,
    each through the same assertions and bars as here."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    env["GPK_FP64_SIMT"] = "1"
    out = str(tmp_path / "simt.json")
    r = subprocess.run([sys.executable, "-m", "tests._dense64_worker", out], cwd=ROOT, env=env, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    import json
    with open(out) as f:
        res = json.load(f)
    assert res["cases"] == len(engine_cases())
    assert not res["failed"], res["failed"]
    print("fp64 SIMT worst ratios:", res["worst"])


def test_report_worst_ratios():
    """Prints the (smallest, largest) per-case error / bar of every operator measured in this session."""
    print("worst ratios:", {k: (float(a), float(b)) for k, (a, b) in WORST.items()})
