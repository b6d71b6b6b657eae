"""NumPy model of the fp64 -> int8 digit slicing of gpflow_b200/csrc/gemm_tc.cu (planes.cuh::tc_digits + the weighted
recombination of the int8 tensor-core int32 accumulators): checks, without a GPU, the error bound DESIGN.md 4.3 states for the
tensor-core trailing update, the exactness of the digit expansion (including the conversion-free rounding the kernels
use), and the int32 headroom of the accumulators."""
import numpy as np
import pytest


def slice_rows(P: np.ndarray, S: int):
    """Per row: e = ilogb(max|row|) + 1; the S balanced base-256 digits (most significant first) of
    I = rint(x 2^(6-e) 2^(8(S-1))): d = ((I + 128) & 255) - 128 from the low end, the top digit is what remains
    (planes.cuh::tc_digits, slice_rows_kernel).  Returns digits [S, m, K] (int64) and rowscale [m] = 2^(e-6)."""
    mx = np.abs(P).max(axis=1)
    e = np.where(mx > 0, np.floor(np.log2(np.where(mx > 0, mx, 1.0))).astype(np.int64) + 1, 0)
    v = P * np.exp2(6.0 - e)[:, None]                       # |v| < 64
    I = np.rint(v * 2.0 ** (8 * (S - 1))).astype(np.int64)  # exact product (power of two), one rounding
    digits = np.empty((S,) + P.shape, dtype=np.int64)
    for s in range(S - 1, 0, -1):
        d = ((I + 128) & 255) - 128
        digits[s] = d
        I = (I - d) >> 8
    digits[0] = I
    assert np.abs(digits[0]).max() <= 65 and digits.min() >= -128 and digits.max() <= 127   # int8
    return digits, np.exp2(e - 6.0), e


def syrk_model(P: np.ndarray, S: int) -> np.ndarray:
    """sum_{s+t<S} 2^(-8(s+t)) D_s D_t^T (+ 2^(-8S) D_{S/2} D_{S/2}^T for S = 6), recombined with the row scales
    (syrk_i8_kernel epilogue)."""
    D, rs, _ = slice_rows(P, S)
    m = P.shape[0]
    out = np.zeros((m, m))
    for g in range(S):
        acc = np.zeros((m, m), dtype=np.int64)
        for s in range(g + 1):
            acc += D[s] @ D[g - s].T                      # exact integer accumulation (int32 on the tensor cores)
        assert np.abs(acc).max() < 2 ** 31, "int32 accumulator would overflow"
        out += acc.astype(np.float64) * 2.0 ** (-8 * g)
    if S == 6:
        out += (D[3] @ D[3].T).astype(np.float64) * 2.0 ** (-8 * S)
    return out * rs[:, None] * rs[None, :]


@pytest.mark.parametrize("S", [6, 7, 8])
@pytest.mark.parametrize("K", [512, 4096])
def test_digit_sliced_syrk_error_bound(S, K):
    rng = np.random.default_rng(S * 1000 + K)
    m = 96
    P = rng.standard_normal((m, K)) * np.exp2(rng.integers(-20, 20, size=(m, 1)))   # rows of very different scale
    got = syrk_model(P, S)
    Pl = P.astype(np.longdouble)
    exact = (Pl @ Pl.T).astype(np.float64)
    _, _, e = slice_rows(P, S)
    scale = np.exp2(e)[:, None] * np.exp2(e)[None, :]
    # dropped digit products of order >= S: (S + 1) pairs of |d| <= 128 each, 2^(-8S) relative to 64 x 64, per k
    bound = 4.0 * K * (S + 1) * 2.0 ** (-8 * S) * scale + 4 * np.finfo(float).eps * np.abs(exact) + K * 2.0 ** -53 * scale
    assert np.all(np.abs(got - exact) <= bound)
    if S == 6:   # the default for well-conditioned problems: ~1e-11 relative to the row scales at K = 4096
        assert (np.abs(got - exact) / scale).max() < 3e-11
    if S == 7:
        assert (np.abs(got - exact) / scale).max() < 2e-13


def test_square_term_removes_the_bias_of_the_diagonal():
    """Without the (3,3) product the diagonal of P P^T is short by sum_k d_3(i,k)^2 2^-48 > 0 (a systematic error of
    sum log diag L, scripts/radix_study.py); with it the diagonal error is zero-mean."""
    rng = np.random.default_rng(11)
    P = rng.standard_normal((128, 2048))
    got = syrk_model(P, 6)
    Pl = P.astype(np.longdouble)
    exact = (Pl @ Pl.T).astype(np.float64)
    D, rs, _ = slice_rows(P, 6)
    sq = (D[3] ** 2).sum(axis=1) * 2.0 ** -48 * rs ** 2
    err = np.diag(got) - np.diag(exact)
    assert abs(err.mean()) < 0.1 * sq.mean()
    assert np.all(sq > 10 * np.abs(err).mean())


def test_digit_expansion_is_exact_up_to_the_last_digit():
    rng = np.random.default_rng(0)
    P = rng.standard_normal((8, 64))
    for S in (6, 7, 8):
        D, rs, _ = slice_rows(P, S)
        recon = sum(D[s] * 2.0 ** (-8 * s) for s in range(S)) * rs[:, None]
        assert np.abs(recon - P).max() <= 0.5 * 2.0 ** (-8 * (S - 1)) * rs.max() * 1.0000001
    D, rs, e = slice_rows(P, 7)            # 2^-55 of 2^e: entries within a factor 4 of 2^e keep every bit
    recon = sum(D[s] * 2.0 ** (-8 * s) for s in range(7)) * rs[:, None]
    big = np.abs(P) >= np.exp2(e - 2.0)[:, None]
    assert big.any() and np.array_equal(recon[big], P[big])


def digit_bytes(v: np.ndarray, S: int) -> np.ndarray:
    """planes.cuh::TcDigitizer::bytes in uint64 arithmetic: X = (I + flip) ^ flip with I read off the bit pattern of
    x + 1.5 2^52 (no conversion instruction); byte j of X is the int8 digit of plane S - 1 - j."""
    magic = 6755399441055744.0
    M = (1 << 64) - 1
    flip = 0x8080808080808080 >> (8 * (9 - S))
    c = (flip - 0x4330000000000000 - 0x0008000000000000) & M
    low = 8 * (S - 1) if S <= 6 else 8 * (S - 1) - 16
    v = np.asarray(v, dtype=np.float64)
    if S <= 6:
        bits = (v * 2.0 ** low + magic).view(np.uint64)
        return np.array([((int(b) + c) & M) ^ flip for b in bits], dtype=np.uint64)
    xh = v * 65536.0
    th = xh + magic
    r = xh - (th - magic)
    bits = (r * 2.0 ** low + magic).view(np.uint64)
    hi = (th.view(np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32)      # __double2loint
    return np.array([(((int(b) + c) + (int(h) << low)) & M) ^ flip for b, h in zip(bits, hi)], dtype=np.uint64)


def test_conversion_free_digit_bytes_match_the_digit_model():
    rng = np.random.default_rng(1)
    v = np.concatenate([rng.uniform(-64, 64, 20000), rng.uniform(-1e-6, 1e-6, 2000),
                        [63.999999999, -63.999999999, 0.5, -0.5, 1.5, 2.5, 0.0, 2.0 ** -41, -(2.0 ** -41), 3 * 2.0 ** -42]])
    for S in (6, 7, 8):
        X = digit_bytes(v, S)
        # reference digits from exact integer arithmetic (ties to even like the fp64 adder)
        scaled = [np.longdouble(x) * np.longdouble(2.0) ** (8 * (S - 1)) for x in v]
        I = np.array([int(np.rint(x)) for x in scaled], dtype=object)
        # digit-by-digit from the low end, as in slice_rows()
        rest = [int(i) for i in I]
        for j in range(S - 1):
            d = [((i + 128) & 255) - 128 for i in rest]
            rest = [(i - dd) >> 8 for i, dd in zip(rest, d)]
            byte = ((X >> np.uint64(8 * j)) & np.uint64(0xFF)).astype(np.uint8).view(np.int8).astype(np.int64)
            assert np.array_equal(byte, np.array(d, dtype=np.int64)), (S, j)
        top = ((X >> np.uint64(8 * (S - 1))) & np.uint64(0xFF)).astype(np.uint8).view(np.int8).astype(np.int64)
        assert np.array_equal(top, np.array(rest, dtype=np.int64)) and np.abs(top).max() <= 65


def test_byte_transpose_selectors():
    """planes.cuh::tc_transpose4: two PRMT stages (selectors 0x5140 / 0x7362, then 0x5410 / 0x7632)."""
    def prmt(a, b, sel):
        src = [(a >> (8 * i)) & 0xFF for i in range(4)] + [(b >> (8 * i)) & 0xFF for i in range(4)]
        return sum(src[(sel >> (4 * i)) & 0xF] << (8 * i) for i in range(4))
    a = [0x03020100, 0x13121110, 0x23222120, 0x33323130]
    l01, h01 = prmt(a[0], a[1], 0x5140), prmt(a[0], a[1], 0x7362)
    l23, h23 = prmt(a[2], a[3], 0x5140), prmt(a[2], a[3], 0x7362)
    o = [prmt(l01, l23, 0x5410), prmt(l01, l23, 0x7632), prmt(h01, h23, 0x5410), prmt(h01, h23, 0x7632)]
    assert o == [0x30201000, 0x31211101, 0x32221202, 0x33231303]


def test_int32_headroom_at_the_largest_k():
    """Worst case |digit| = 128 everywhere and (g+1) <= S digit pairs per accumulator: 128*128*K*S must stay below 2^31,
    i.e. K <= 2^17 / S (21845 at S = 6).  potrf.cu::trailing_update falls back to the DMMA kernel beyond that."""
    assert 128 * 128 * 4096 * 7 < 2 ** 31                # BASELINE config 2: K <= N/2 = 4096
    assert 128 * 128 * 16384 * 8 >= 2 ** 31 > 128 * 128 * 16383 * 8
