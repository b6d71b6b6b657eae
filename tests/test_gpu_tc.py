"""GPU tests of the wgmma (int8-sliced fp64) symmetric rank-k update against NumPy fp64, through
gpk_potrf's recursion (engine on) and directly via a Cholesky whose trailing updates use it."""
import os

import numpy as np
import pytest
import scipy.linalg as sla
from numpy.testing import assert_allclose

import gpflow_b200 as gpf
from gpflow_b200 import ops
from tests.helpers import to_np

pytestmark = pytest.mark.gpu


def _spd(n, rng, cond_shift=0.5):
    A = rng.standard_normal((n, n + 5))
    return A @ A.T / n + cond_shift * np.eye(n)


@pytest.mark.parametrize("n", [512, 640, 1000, 1536, 2048])
def test_potrf_with_tcgen05_trailing_update(cuda_device, n):
    """n >= 512 engages the int8 tensor-core path for the top level(s) of the recursion (K >= 256)."""
    rng = np.random.default_rng(n)
    K = _spd(n, rng)
    L, _ = ops.cholesky(ops.to_device(K))
    ref = sla.cholesky(K, lower=True)
    # digit truncation: K * S * 2^-49 relative to row maxima (S = 7) -> ~1e-11 on L
    assert_allclose(to_np(L), ref, rtol=2e-9, atol=2e-10)
    Ld = to_np(L)
    resid = np.linalg.norm(Ld @ Ld.T - K) / np.linalg.norm(K)
    assert resid < 1e-11, resid


def test_potrf_tc_extra_rows_and_scaling(cuda_device):
    """Rows with very different magnitudes exercise the per-row power-of-two scales."""
    rng = np.random.default_rng(7)
    n, p = 1024, 2
    D = np.exp(rng.uniform(-6, 6, n))                      # row/column scaling over 5 decades
    K = _spd(n, rng) * D[:, None] * D[None, :]
    Y = rng.standard_normal((n, p)) * D[:, None]
    A = np.zeros((n + p, n))
    A[:n] = np.tril(K)
    A[n:] = Y.T
    Ad = ops.to_device(A)
    ops.potrf(Ad, n)
    L = sla.cholesky(K, lower=True)
    got = to_np(Ad)
    assert_allclose(np.tril(got[:n]) / D[:, None], L / D[:, None], rtol=1e-7, atol=1e-9)
    alpha = sla.solve_triangular(L, Y, lower=True).T
    assert_allclose(got[n:], alpha, rtol=1e-7, atol=1e-8)


def test_potrf_diagonal_beyond_1e300(cuda_device):
    """One row and column scaled by 1e150 (A_ii ~ 1e300): its static row exponent is ~500, not 'no scale'.  A guard that
    treated a diagonal >= 1e300 as unscaled digitised that row of L at 2^-6 and corrupted every update it enters.
    Compared with LAPACK row by row in relative terms, as test_gpu_edge.py::test_potrf_rows_spanning_ten_decades."""
    rng = np.random.default_rng(13)
    n = 1024
    dsc = np.ones(n)
    dsc[300] = 1e150
    dsc[301] = 1e-150
    A = _spd(n, rng) * dsc[:, None] * dsc[None, :]
    assert A[300, 300] > 1e300
    L, _ = ops.cholesky(ops.to_device(A))
    Lref = np.linalg.cholesky(A)
    got = to_np(L)
    assert np.isfinite(got).all()
    assert_allclose(got / dsc[:, None], Lref / dsc[:, None], rtol=0, atol=2e-9)


# ---- fp32 GEMM on wgmma tf32 (3xTF32) ----------------------------------------------------------
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("m,n,k", [(512, 768, 640), (300, 1000, 777), (1024, 1024, 20000), (128, 5000, 128)])
def test_gemm_tf32_tcgen05_matches_fp64(cuda_device, ta, tb, m, n, k):
    """Shapes above the eligibility threshold run on the tensor cores; the 3xTF32 compensation keeps fp32
    accuracy (error ~ sqrt(k) * 2^-23 relative to |a||b|).  (1024,1024,20000) exercises split-K atomics."""
    rng = np.random.default_rng(m + n + k)
    A = rng.standard_normal((k, m) if ta else (m, k)).astype(np.float32)
    B = rng.standard_normal((n, k) if tb else (k, n)).astype(np.float32)
    C = rng.standard_normal((m, n)).astype(np.float32)
    ref = 0.7 * (A.T if ta else A).astype(np.float64) @ (B.T if tb else B).astype(np.float64) - 0.3 * C
    with gpf.config.as_context(gpf.config.Config(float=np.float32)):
        Cd = ops.to_device(C.copy())
        ops.gemm(ops.to_device(A), ops.to_device(B), transa=bool(ta), transb=bool(tb), alpha=0.7, beta=-0.3, out=Cd)
    err = np.abs(to_np(Cd) - ref).max()
    assert err < 4e-6 * np.sqrt(k) * 3.0, err     # plain TF32 (10-bit mantissa) would be ~1e-3 * sqrt(k)


@pytest.mark.parametrize("beta", [0.5, 1.0, 0.0])
def test_gemm_tf32_lower_only_split_k_leaves_the_upper_tiles(cuda_device, beta):
    """m = n = 512, k = 8192 runs split-K (8 splits on 132 SMs): C is pre-scaled by beta and the splits add atomically.
    GPK_GEMM_LOWER_ONLY promises that the 128 x 128 tiles strictly above the diagonal stay untouched, the pre-scaling
    included."""
    from gpflow_b200 import _lib

    rng = np.random.default_rng(17)
    m, k = 512, 8192
    A = rng.standard_normal((m, k)).astype(np.float32)
    C0 = rng.standard_normal((m, m)).astype(np.float32)
    upper = (np.arange(m)[None, :] // 128) > (np.arange(m)[:, None] // 128)
    C0[upper] = 12345.0
    with gpf.config.as_context(gpf.config.Config(float=np.float32)):
        Cd = ops.to_device(C0.copy())
        ops.gemm(ops.to_device(A), ops.to_device(A), transb=True, beta=beta, out=Cd, flags=_lib.GPK_GEMM_LOWER_ONLY)
    got = to_np(Cd)
    assert np.all(got[upper] == 12345.0)
    ref = A.astype(np.float64) @ A.T.astype(np.float64) + beta * C0.astype(np.float64)
    scale = np.abs(A).astype(np.float64) @ np.abs(A).T.astype(np.float64) + np.abs(C0)
    err = (np.abs(got - ref) / scale)[~upper].max()
    assert err < 1e-6, err                                   # fp32 rounding of a k = 8192 dot product: ~1e-7 of |a||b|


@pytest.mark.parametrize("ta,tb", [(0, 0), (1, 1), (0, 1)])
def test_gemm_tf32_strided_views(cuda_device, ta, tb):
    """Operands and C as views into larger buffers: odd leading dimensions (ops._ld is the row stride) and base pointers
    off 16-byte alignment, so the pre-pass and the epilogue take their scalar branches.  C outside the view stays intact."""
    rng = np.random.default_rng(3 + ta + 2 * tb)
    m, n, k = 300, 1000, 777
    ar, ac = (k, m) if ta else (m, k)
    br, bc = (n, k) if tb else (k, n)
    odd = lambda c: c + 3 if (c + 3) % 2 else c + 4          # noqa: E731  (odd row stride, room for the column offset)
    with gpf.config.as_context(gpf.config.Config(float=np.float32)):
        Abuf = ops.to_device(rng.standard_normal((ar + 2, odd(ac))).astype(np.float32))
        Bbuf = ops.to_device(rng.standard_normal((br + 1, odd(bc))).astype(np.float32))
        Cbuf = ops.to_device(rng.standard_normal((m + 3, odd(n + 5))).astype(np.float32))
        Av, Bv, Cv = Abuf[1:1 + ar, 2:2 + ac], Bbuf[1:1 + br, 2:2 + bc], Cbuf[2:2 + m, 5:5 + n]
        for v in (Av, Bv, Cv):   # odd stride: (row offset * ld + odd column offset) * 4 bytes is never a multiple of 8
            assert ops._ld(v) % 2 == 1 and v.data_ptr() % 8 == 4
        C0 = to_np(Cbuf).astype(np.float64)
        ops.gemm(Av, Bv, transa=bool(ta), transb=bool(tb), alpha=0.7, beta=-0.3, out=Cv)
        a, b = to_np(Av).astype(np.float64), to_np(Bv).astype(np.float64)
    ref = 0.7 * (a.T if ta else a) @ (b.T if tb else b) - 0.3 * C0[2:2 + m, 5:5 + n]
    got = to_np(Cbuf)
    assert np.abs(got[2:2 + m, 5:5 + n] - ref).max() < 4e-6 * np.sqrt(k) * 3.0
    outside = np.ones(got.shape, bool)
    outside[2:2 + m, 5:5 + n] = False
    assert np.array_equal(got[outside], C0[outside].astype(np.float32))


def test_gemm_tf32_flags(cuda_device):
    from gpflow_b200 import _lib

    rng = np.random.default_rng(5)
    with gpf.config.as_context(gpf.config.Config(float=np.float32)):
        m, k = 1500, 900
        A = rng.standard_normal((m, k)).astype(np.float32)
        C = ops.full((m, m), 5.0, dtype=np.float32)
        ops.gemm(ops.to_device(A), ops.to_device(A), transb=True, out=C, flags=_lib.GPK_GEMM_LOWER_ONLY)
        ref = A.astype(np.float64) @ A.T.astype(np.float64)
        il = np.tril_indices(m)
        assert np.all(np.abs(to_np(C)[il] - ref[il]) < 2e-6 * np.abs(ref[il]) + 2e-4)
        assert np.all(to_np(C)[:128, 256:] == 5.0)           # tiles strictly above the diagonal untouched
        kq, n = 1100, 2000
        Q = rng.standard_normal((kq, kq)).astype(np.float32)
        Bm = rng.standard_normal((kq, n)).astype(np.float32)
        ref = np.tril(Q).T.astype(np.float64) @ Bm.astype(np.float64)
        got = ops.gemm(ops.to_device(Q), ops.to_device(Bm), transa=True, flags=_lib.GPK_GEMM_A_LOWER)
        assert np.all(np.abs(to_np(got) - ref) < 2e-6 * np.abs(ref) + 2e-4)
        # lower-triangular A used untransposed: the K range ABOVE each row tile is skipped (tri = 1)
        ref1 = np.tril(Q).astype(np.float64) @ Bm.astype(np.float64)
        got1 = ops.gemm(ops.to_device(Q), ops.to_device(Bm), flags=_lib.GPK_GEMM_A_LOWER)
        assert np.all(np.abs(to_np(got1) - ref1) < 2e-6 * np.abs(ref1) + 2e-4)
        v = ops.full((n,), 1.5, dtype=np.float32)
        ops.gemm(ops.to_device(Q), ops.to_device(Bm), transa=True, out=v,
                 flags=_lib.GPK_GEMM_A_LOWER | _lib.GPK_GEMM_COLSUMSQ)
        assert_allclose(to_np(v), 1.5 + (ref ** 2).sum(0), rtol=2e-5)
