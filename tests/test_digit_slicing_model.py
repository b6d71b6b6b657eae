"""NumPy model of the fp64 -> int8 digit slicing of gpflow_b200/csrc/gemm_tc.cu (planes.cuh::tc_digits + the weighted
recombination of the int8 tensor-core int32 accumulators): checks, without a GPU, the error bound DESIGN.md 4.3 states for the
tensor-core trailing update, the exactness of the digit expansion (including the conversion-free rounding the kernels
use), and the int32 headroom of the accumulators."""
import numpy as np
import pytest


def row_exponents(P: np.ndarray) -> np.ndarray:
    """planes.cuh::tc_slice_row_cta: e = ilogb(max|row|) + 1 (max|row| 2^-e in [0.5, 1)), held at -1017 below 2^-1018 so
    that 2^(6-e) stays finite; 0 for an all-zero (or non-finite) row.  frexp, not log2: log2 rounds up just below a power of
    two and is inexact for subnormals."""
    mx = np.abs(P).max(axis=1)
    e = np.frexp(mx)[1].astype(np.int64)
    return np.where((mx > 0) & np.isfinite(mx), np.maximum(e, -1017), 0)


def slice_rows(P: np.ndarray, S: int):
    """Per row: e = ilogb(max|row|) + 1 (row_exponents); the S balanced base-256 digits (most significant first) of
    I = rint(x 2^(6-e) 2^(8(S-1))): d = ((I + 128) & 255) - 128 from the low end, the top digit is what remains
    (planes.cuh::TcDigitizer, slice_rows_kernel).  Returns digits [S, m, K] (int64), rowscale [m] = 2^(e-6) and e."""
    e = row_exponents(P)
    v = P * np.ldexp(1.0, 6 - e)[:, None]                   # |v| < 64, the kernel's product x * 2^(6-e)
    I = np.rint(v * 2.0 ** (8 * (S - 1))).astype(np.int64)  # exact product (power of two), one rounding
    digits = np.empty((S,) + P.shape, dtype=np.int64)
    for s in range(S - 1, 0, -1):
        d = ((I + 128) & 255) - 128
        digits[s] = d
        I = (I - d) >> 8
    digits[0] = I
    assert np.abs(digits[0]).max() <= 65 and digits.min() >= -128 and digits.max() <= 127   # int8
    return digits, np.ldexp(1.0, e - 6), e


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


def syrk_i8_accumulators(P: np.ndarray, n: int, S: int, matmul=np.matmul):
    """The int32 accumulators of gemm_tc.cu::syrk_i8_kernel for C[m, n] -= P P[:n]^T: acc[g] = sum_{s+t=g} D_s D_t^T
    (g < S), plus D_3 D_3^T at index 6 for S = 6.  Computed as float64 matmuls of the digit planes: every partial sum is an
    integer below 2^53, so any fp64 GEMM (`matmul`) returns them exactly in any summation order.
    Returns (acc [NACC, m, n], rowscale [m])."""
    D, rs, _ = slice_rows(P, S)
    Df = D.astype(np.float64)
    accs = []
    for g in range(S):
        lhs = np.concatenate([Df[s] for s in range(g + 1)], axis=1)
        rhs = np.concatenate([Df[g - s][:n] for s in range(g + 1)], axis=1)
        accs.append(matmul(lhs, rhs.T))
    if S == 6:
        accs.append(matmul(Df[3], Df[3][:n].T))
    acc = np.stack(accs)
    assert np.abs(acc).max(initial=0) < 2.0 ** 31, "int32 accumulator would overflow"
    return acc, rs


def syrk_i8_epilogue(acc: np.ndarray, rs: np.ndarray, C: np.ndarray) -> np.ndarray:
    """The kernel's epilogue in its order: v = 0; v = fma(acc_g, 2^-8g, v) for g = 0 .. NACC-1; C += (-(rs_i rs_j)) v.
    Every acc_g 2^-8g and every (rs_i rs_j) v is a power-of-two scaling (exact while the result is a normal number), so each
    fma rounds like the multiply-then-add below: the result is bit for bit what the kernel stores."""
    m, n = acc.shape[1:]
    v = np.zeros((m, n))
    for g in range(acc.shape[0]):
        v = v + acc[g] * 2.0 ** (-8 * g)
    with np.errstate(over="ignore", invalid="ignore"):
        return C + (-(rs[:, None] * rs[None, :n])) * v


def syrk_i8_emulate(P: np.ndarray, n: int, S: int, C: np.ndarray) -> np.ndarray:
    """C - P P[:n]^T exactly as syrk_i8_kernel computes it from row-maximum scales (every tile stored)."""
    acc, rs = syrk_i8_accumulators(P, n, S)
    return syrk_i8_epilogue(acc, rs, C)


@pytest.mark.parametrize("S", [6, 7, 8])
def test_kernel_emulation_matches_the_digit_model(S):
    """The bit-level emulation of syrk_i8_kernel (tests/test_gpu_syrk_i8.py) is the digit model: the same products as
    syrk_model within the rounding of the recombination, the digits of digit_bytes (the conversion-free digitiser) exactly,
    and within DESIGN.md 4.3's bound K (S + 1) 2^(-8S+2) of the exact product relative to the row scales."""
    rng = np.random.default_rng(40 + S)
    m, n, K = 96, 64, 512
    P = rng.standard_normal((m, K)) * np.ldexp(1.0, rng.integers(-20, 20, size=(m, 1)))
    got = -syrk_i8_emulate(P, n, S, np.zeros((m, n)))
    model = syrk_model(P, S)[:, :n]
    _, _, e = slice_rows(P, S)
    scale = np.ldexp(1.0, e)[:, None] * np.ldexp(1.0, e[:n])[None, :]
    assert np.all(np.abs(got - model) <= 8 * np.finfo(float).eps * (np.abs(model) + scale))
    # digits: byte j of digit_bytes(x 2^(6-e)) is plane S - 1 - j of slice_rows
    D, _, _ = slice_rows(P, S)
    v = (P * np.ldexp(1.0, 6 - e)[:, None]).ravel()
    X = digit_bytes(v[:4000], S)
    for j in range(S):
        byte = ((X >> np.uint64(8 * j)) & np.uint64(0xFF)).astype(np.uint8).view(np.int8).astype(np.int64)
        assert np.array_equal(byte, D[S - 1 - j].ravel()[:4000]), (S, j)
    Pl = P.astype(np.longdouble)
    exact = Pl @ Pl[:n].T
    err = np.abs(got.astype(np.longdouble) - exact) / scale
    rounding = 4 * np.finfo(float).eps * np.abs(exact) / scale          # the fp64 recombination of the accumulators
    assert np.all(err <= K * (S + 1) * 2.0 ** (-8 * S + 2) + rounding), err.max()


def test_row_exponents_follow_frexp_over_the_whole_range():
    """Row exponents at the ends of the fp64 range: a maximum just below a power of two (where log2 rounds up), 1e300 and
    DBL_MAX (no 'no scale' cut-off), subnormal maxima (held at -1017) and zero rows."""
    big = np.finfo(float).max
    rows = np.array([[1 - 2.0 ** -53, 0.25], [1e300, -1.0], [-big, 1.0], [5e-324, 0.0], [2.0 ** -1019, 0.0],
                     [2.0 ** -1018, 0.0], [0.0, 0.0], [-0.75, 0.5]])
    assert row_exponents(rows).tolist() == [0, 997, 1024, -1017, -1017, -1017, 0, 0]
    for S in (6, 7, 8):
        D, rs, _ = slice_rows(rows, S)
        assert np.all(np.isfinite(rs)) and np.abs(D[0]).max() <= 64


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
