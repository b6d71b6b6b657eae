"""The int8 digit-sliced trailing update (gemm_tc.cu::syrk_i8_kernel) against a NumPy emulation of its arithmetic, bit for bit.

gpk_debug_syrk_i8 runs ONE update as gpk_potrf issues it for rows with row-maximum scales.  The emulation
(tests/test_digit_slicing_model.py::syrk_i8_emulate) slices the same rows, forms the int32 accumulators exactly and recombines
them in the kernel's order, so the kernel must reproduce it exactly: a lost digit product, a wrong plane offset, a wrong
epilogue weight or a stage refilled early shows up as a mismatch even where it moves the result by 2^(-8(S-1)) of the row
scale only -- far below the tolerance of any comparison with LAPACK.  Every instantiation <S, CL> (S = 6, 7, 8 digit planes,
clusters of 1, 2, 4 CTAs) runs, with and without the lower-triangle tile restriction."""
import functools

import numpy as np
import pytest

from gpflow_b200 import _lib
from tests.test_digit_slicing_model import slice_rows, syrk_i8_accumulators, syrk_i8_epilogue
from tests.test_tile_iterators_model import diag_units_total, tc_units

pytestmark = pytest.mark.gpu

TC_BM, TC_BN = 128, 32
SENTINEL = -7.25e3
S_ALL, CL_ALL = [6, 7, 8], [1, 2, 4]


def dev_matmul(a, b):
    """fp64 GEMM of integer-valued digit planes on the device: exact like any other order of the same integer sums."""
    import torch
    return (torch.from_numpy(np.ascontiguousarray(a)).cuda() @ torch.from_numpy(np.ascontiguousarray(b)).cuda()).cpu().numpy()


@functools.lru_cache(maxsize=None)
def stored_mask(m, n, lower):
    """Elements of C the kernel stores: the valid tiles of every unit of the TcTileIter mirror (one cluster walks them all)."""
    mask = np.zeros((-(-m // TC_BM) * TC_BM, -(-n // TC_BN) * TC_BN), dtype=bool)
    for cl in CL_ALL:
        tiles = {(u["tm"], u["tn"]) for b in range(cl) for u in tc_units(m, n, lower, cl, cl, b) if u["valid"]}
        part = np.zeros_like(mask)
        for tm, tn in tiles:
            part[tm * TC_BM:(tm + 1) * TC_BM, tn * TC_BN:(tn + 1) * TC_BN] = True
        assert cl == 1 or np.array_equal(part, mask)          # the same tile set for every cluster width
        mask = part
    return mask[:m, :n]


def run_kernel(P, n, S, cl, lower, C0, *, r0=None, k0=0, ldc=None, c_offset=0, head_flag=False):
    """C0 - P P[:n]^T on the GPU: P [m, K] becomes columns [k0, k0 + K) of a device matrix of row stride k0 + K + 3 (the
    other columns are never read and stay uninitialised), sliced as rows [r0, r0 + m) of the plane store.  C lives at
    `c_offset` doubles into its buffer with row stride `ldc`.  Returns (C, rowscale, flag)."""
    import torch

    m, K = P.shape
    r0 = r0 if r0 is not None else -(-(k0 + K) // TC_BM) * TC_BM
    lda = k0 + K + 3
    A = torch.empty((m, lda), dtype=torch.float64, device="cuda")
    A[:, k0:k0 + K] = torch.from_numpy(P).cuda()
    ldc = ldc or n
    buf = torch.full((c_offset + m * ldc,), np.nan, dtype=torch.float64, device="cuda")
    cv = buf[c_offset:].view(m, ldc)
    cv[:, :n] = torch.from_numpy(np.ascontiguousarray(C0)).cuda()
    rs = torch.zeros(m, dtype=torch.float64, device="cuda")
    flag = torch.zeros(2, dtype=torch.int32, device="cuda") if head_flag else None
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.gpk_debug_syrk_i8(A.data_ptr(), lda, r0, k0, K, buf.data_ptr() + 8 * c_offset, ldc, m, n, lower, S, cl,
                                     rs.data_ptr(), flag.data_ptr() if flag is not None else None, stream),
               "gpk_debug_syrk_i8")
    out = cv.cpu().numpy()
    assert np.isnan(out[:, n:]).all(), "stored beyond column n"
    if c_offset:
        assert np.isnan(buf[:c_offset].cpu().numpy()).all()
    return out[:, :n], rs.cpu().numpy(), (flag.cpu().numpy() if flag is not None else None)


def expected(P, n, S, C0, lower):
    acc, rs = syrk_i8_accumulators(P, n, S)
    full = syrk_i8_epilogue(acc, rs, C0)
    return np.where(stored_mask(P.shape[0], n, lower), full, C0), rs


def check(P, n, S, cl, lower, C0, want=None, **kw):
    got, rs, flag = run_kernel(P, n, S, cl, lower, C0, **kw)
    if want is None:
        want, _ = expected(P, n, S, C0, lower)
    else:
        want = np.where(stored_mask(P.shape[0], n, lower), want, C0)
    np.testing.assert_array_equal(rs, slice_rows(P, S)[1])
    np.testing.assert_array_equal(got, want)
    return flag


def sentinel_c(m, n, rng):
    C = np.full((m, n), SENTINEL)
    C[::3] = rng.standard_normal((len(C[::3]), n))
    return C


def mixed_rows(m, K, rng):
    """Gaussian rows of very different scale (1e-30 .. 1e30), rows whose entries span 1e-30 .. 1e30, and zero rows."""
    P = rng.standard_normal((m, K)) * 10.0 ** rng.uniform(-30, 30, size=(m, 1))
    P[1::7] = rng.standard_normal((len(P[1::7]), K)) * 10.0 ** rng.uniform(-30, 30, size=(len(P[1::7]), K))
    P[5::11] = 0.0
    return P


# (m, n, r0, k0, K): tile edges of n (32, 33, 96, 130, 640) and m (128, 200, 1000); column-tile counts that are no multiple
# of CL (2, 3, 5 tiles); r0 > k0 + K and k0 > 0 (non-zero plane-tile offsets)
SHAPES = [(128, 32, 128, 0, 128), (200, 33, 256, 64, 96), (128, 96, 384, 128, 224), (1000, 130, 512, 32, 480),
          (1000, 640, 1024, 256, 512), (200, 200, 128, 0, 64)]


@functools.lru_cache(maxsize=None)
def _case(S, shape):
    m, n, r0, k0, K = shape
    rng = np.random.default_rng(hash((S,) + shape) % 2 ** 32)
    P = mixed_rows(m, K, rng)
    C0 = sentinel_c(m, n, rng)
    acc, rs = syrk_i8_accumulators(P, n, S)
    return P, C0, syrk_i8_epilogue(acc, rs, C0)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "m%d_n%d_r%d_k%d_K%d" % s)
@pytest.mark.parametrize("lower", [0, 1])
@pytest.mark.parametrize("cl", CL_ALL)
@pytest.mark.parametrize("S", S_ALL)
def test_syrk_i8_bit_exact(cuda_device, S, cl, lower, shape):
    P, C0, want = _case(S, shape)
    m, n, r0, k0, K = shape
    check(P, n, S, cl, lower, C0, want=want, r0=r0, k0=k0)


@pytest.mark.parametrize("S", S_ALL)
def test_syrk_i8_persistent_ctas_loop(cuda_device, S):
    """m = n = 4096: ~2000 lower tiles for 130 CTAs, so every CTA walks many units and the pipeline wraps its stages."""
    rng = np.random.default_rng(S)
    m = n = 4096
    P = mixed_rows(m, 128, rng)
    C0 = sentinel_c(m, n, rng)
    acc, rs = syrk_i8_accumulators(P, n, S, matmul=dev_matmul)
    full = syrk_i8_epilogue(acc, rs, C0)
    for cl in CL_ALL:
        for lower in (0, 1):
            check(P, n, S, cl, lower, C0, want=full)


@pytest.mark.parametrize("cl", CL_ALL)
def test_syrk_i8_scalar_epilogue(cuda_device, cl):
    """Odd ldc and a C that starts one double past a 16-byte boundary: the epilogue's scalar branch."""
    rng = np.random.default_rng(cl)
    for S in S_ALL:
        P = mixed_rows(200, 96, rng)
        C0 = sentinel_c(200, 130, rng)
        check(P, 130, S, cl, 1, C0, ldc=133, c_offset=1, k0=32)
        check(P, 130, S, cl, 0, C0, ldc=131, c_offset=1)


def constructed(S, digits):
    """One value (exactly representable, with e = 0) whose digits are `digits` (most significant first) where fp64 can hold
    them: sum_s d_s 2^(-8s) 2^-6."""
    from fractions import Fraction
    return float(sum(Fraction(int(d), 256 ** s) for s, d in enumerate(digits)) / 64)


def edge_rows(S, K, rng):
    """Digit-pattern edges, one kind per block of rows."""
    rows = []
    r = rng.standard_normal(K)
    rows.append(np.zeros(K))                                          # zero row
    top = np.clip(r, -0.5, 0.5); top[3] = 1 - 2.0 ** -53; top[9] = -top[3]   # top digit rounds up to +-64 (never 65: see below)
    rows.append(top)
    rows.append(np.full(K, constructed(S, [-63] + [-128] * (S - 1))))   # lower digits all -128
    rows.append(np.full(K, constructed(S, [63] + [127] * (S - 1))))     # lower digits all 127
    rows.append(np.where(np.arange(K) % 2, 1, -1) * constructed(S, [-63] + [-128] * (S - 1)))
    ties = rng.integers(-2 ** 20, 2 ** 20, size=K) + 0.5                  # exact ties at the last digit: rint to even
    tie = ties * 2.0 ** (-6 - 8 * (S - 1)); tie[0] = 0.75
    rows.append(tie)
    rows.append(rng.standard_normal(K) * 10.0 ** rng.uniform(-30, 30, size=K))
    rows.append(-r * 2.0 ** -40)
    return np.array(rows)


@pytest.mark.parametrize("cl", CL_ALL)
@pytest.mark.parametrize("S", S_ALL)
def test_syrk_i8_digit_pattern_edges(cuda_device, S, cl):
    """Zero rows, top digits at +-64, lower digits all -128 / all 127, exact rounding ties at the last digit, entries over
    1e-30 .. 1e30.  (The top digit of a row-maximum slicing is at most 64 in magnitude: x 2^(6-e) < 64.)"""
    rng = np.random.default_rng(S * 10 + cl)
    K = 256
    E = edge_rows(S, K, rng)
    P = np.concatenate([E, rng.standard_normal((200 - len(E), K)), E[::-1] * 3.0])
    D, _, _ = slice_rows(P, S)
    assert np.abs(D[0]).max() == 64
    if S < 8:   # (fp64 holds 53 bits: all lower digits -128 fit up to S = 7, all 127 at S = 6)
        assert (D[1:, 2] == -128).all()
    if S == 6:
        assert (D[1:, 3] == 127).all()
    C0 = sentinel_c(len(P), 160, rng)
    check(P, 160, S, cl, 1, C0)
    check(P, 160, S, cl, 0, C0)


@pytest.mark.parametrize("S", S_ALL)
def test_syrk_i8_extreme_row_scales(cuda_device, S):
    """Row maxima at the ends of the fp64 range, below the first n rows (so that every product stays finite): 1e301 and
    DBL_MAX (a 'd >= 1e300 means no scale' guard digitised them at scale 2^-6, far out of the digitiser's range), and
    subnormal / sub-2^-1018 maxima (2^(6-e) overflowed to inf)."""
    rng = np.random.default_rng(S)
    K, n = 128, 96
    big = np.finfo(float).max
    # column rows at 2^-400 for the huge rows ...
    Q = rng.standard_normal((n, K)) * 2.0 ** -400
    huge = rng.standard_normal((4, K))
    huge[0] *= 1e301
    huge[1] = huge[1] / np.abs(huge[1]).max() * big
    huge[2] *= 1e305
    huge[3] = np.where(np.arange(K) % 3, 1e300, -big)
    P = np.concatenate([Q, huge, rng.standard_normal((30, K))])
    C0 = sentinel_c(len(P), n, rng)
    for cl in CL_ALL:
        check(P, n, S, cl, 1, C0)
    # ... and at 2^400 for the tiny ones
    Q = rng.standard_normal((n, K)) * 2.0 ** 400
    tiny = rng.standard_normal((4, K))
    tiny[0] *= 1e-310                                    # subnormal maximum
    tiny[1] *= 2.0 ** -1030
    tiny[2] = tiny[2] / np.abs(tiny[2]).max() * 2.0 ** -1018 * (1 - 2.0 ** -52)
    tiny[3] *= 1e-300
    P = np.concatenate([Q, tiny, rng.standard_normal((30, K)) * 2.0 ** 300])
    C0 = sentinel_c(len(P), n, rng)
    for cl in CL_ALL:
        check(P, n, S, cl, 1, C0)


@pytest.mark.parametrize("S,K", [(6, 21824), (7, 18720), (8, 16352)])
def test_syrk_i8_int32_headroom_at_the_largest_k(cuda_device, S, K):
    """The largest K potrf sends to the int8 kernel (K S 2^14 < 2^31) with digits that drive the accumulators as high as
    that bound allows: rows whose every digit product has the same sign (top digit -63, lower digits -128)."""
    rng = np.random.default_rng(S)
    m = n = 256
    P = rng.standard_normal((m, K))
    P[::2] = constructed(S, [-63] + [-128] * (S - 1))
    acc, rs = syrk_i8_accumulators(P, n, S, matmul=dev_matmul)
    assert np.abs(acc).max() > (0.74 if S == 8 else 0.82) * 2.0 ** 31   # within a few percent of what int32 holds
    C0 = sentinel_c(m, n, rng)
    want = syrk_i8_epilogue(acc, rs, C0)
    check(P, n, S, 2, 1, C0, want=want)
    with pytest.raises(ValueError):                     # one k-step more is refused (potrf uses DMMA there)
        run_kernel(P[:, :1] * np.ones((1, K + 32)), n, S, 2, 1, C0)


@pytest.mark.parametrize("cl", CL_ALL)
@pytest.mark.parametrize("m,n", [(128, 96), (200, 33), (1000, 130), (640, 640), (128, 128)])
def test_syrk_i8_head_flag_counts(cuda_device, cl, m, n):
    """flag[0] = the head tiles the kernel publishes (padding tiles of a unit included), flag[1] = diag_units_total(m, n),
    the count the waiting look-ahead leaf needs (test_tile_iterators_model mirrors)."""
    rng = np.random.default_rng(m + n + cl)
    P = rng.standard_normal((m, 64))
    C0 = sentinel_c(m, n, rng)
    flag = check(P, n, 7, cl, 1, C0, head_flag=True)
    heads = sum(u["head"] for b in range(cl) for u in tc_units(m, n, 1, cl, cl, b))
    assert flag.tolist() == [heads, diag_units_total(m, n)]
