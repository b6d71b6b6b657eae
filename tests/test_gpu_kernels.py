"""GPU parity tests of the individual CUDA operators against the CPU oracle / NumPy, through the
C ABI (ctypes) exactly as the product calls them."""
import numpy as np
import pytest
import scipy.linalg as sla
from numpy.testing import assert_allclose

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from oracle import gp_oracle as O
from tests.helpers import build, to_np, tol, tol_for

pytestmark = pytest.mark.gpu

EXPRS = {
    "rbf": "rbf", "rbf_ard": "rbf_ard", "m12": "m12", "m32": "m32", "m52": "m52", "rq": "rq", "exp": "exp",
    "lin": "lin", "lin_ard": "lin_ard", "const": "const", "white": "white", "poly": "poly", "poly_ard": "poly_ard",
    "poly*rbf+white": ("sum", ("prod", ("poly_ard", [1, 2]), "rbf"), "white"),
    "rbf+white": ("sum", "rbf", "white"),
    "sum3": ("sum", "rbf", "m32", "lin"),
    "prod": ("prod", "m52", "lin"),
    "(rbf+m32)*lin": ("prod", ("sum", "rbf", "m32"), "lin"),
    "active_dims": ("sum", ("m32", [0, 2]), ("rbf", [1])),
    "ard_groups": ("prod", ("rbf_ard", [0, 1, 3]), ("sum", ("lin_ard", [2, 3]), "const")),
    "four_groups": ("sum", ("rbf", [0]), ("m12", [1]), ("m32", [2]), ("m52", [3])),
    "deep": ("sum", ("prod", ("sum", "rbf", "const"), ("sum", "m12", "white")), "lin"),
}


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", sorted(EXPRS))
def test_kbuild_matches_oracle(cuda_device, name, dtype):
    rng = np.random.default_rng(1)
    N, N2, D = 150, 97, 4
    X, X2 = rng.standard_normal((N, D)).astype(dtype), rng.standard_normal((N2, D)).astype(dtype)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        ko, kp = build(EXPRS[name], D, [O, gpf.kernels])
        Xd, X2d = ops.to_device(X), ops.to_device(X2)
        t = tol_for(EXPRS[name], dtype)
        assert_allclose(to_np(kp(Xd)), ko(X), **t)                      # symmetric (White active)
        assert_allclose(to_np(kp(Xd, X2d)), ko(X, X2), **tol(dtype))   # rectangular (White == 0)
        assert_allclose(to_np(kp(Xd, Xd)), ko(X, X), **t)               # X2 given: White stays 0
        assert_allclose(to_np(kp(Xd, full_cov=False)), ko(X, full_cov=False), **tol(dtype))


@pytest.mark.parametrize("N,N2", [(1, 1), (63, 65), (64, 64), (130, 1), (3, 257)])
def test_kbuild_ragged_shapes(cuda_device, N, N2):
    rng = np.random.default_rng(2)
    D = 3
    X, X2 = rng.standard_normal((N, D)), rng.standard_normal((N2, D))
    ko, kp = build(("sum", "m52", "white"), D, [O, gpf.kernels])
    assert_allclose(to_np(kp(X, X2)), ko(X, X2), rtol=1e-11, atol=1e-12)
    assert_allclose(to_np(kp(X)), ko(X), rtol=1e-11, atol=1e-12)


def test_kbuild_lower_and_diag_shift(cuda_device):
    rng = np.random.default_rng(3)
    N, D = 200, 8
    X = rng.standard_normal((N, D))
    ko, kp = build("m52", D, [O, gpf.kernels])
    Xd = ops.to_device(X)
    desc = gpf.kernels.compile_kernel(kp, D)
    noise = ops.to_device(0.1 + rng.random(N))
    out = ops.full((N, N), -7.0, like=Xd)
    ops.kbuild(desc, Xd, None, uplo=_lib.GPK_LOWER, diag_scalar=0.25, diag_vec=noise, out=out)
    ref = ko(X) + np.diag(0.25 + to_np(noise))
    got = to_np(out)
    il = np.tril_indices(N)
    assert_allclose(got[il], ref[il], rtol=1e-12, atol=1e-13)
    # tiles strictly above the diagonal are never touched
    assert np.all(got[:64, 64:] == -7.0)
    # unaligned leading dimension falls back to scalar stores
    buf = ops.full((N, N + 1), 0.0, like=Xd)
    ops.kbuild(desc, Xd, None, out=buf[:, :N])
    assert_allclose(to_np(buf[:, :N]), ko(X), rtol=1e-12, atol=1e-13)


def test_kbuild_large_D_chunks(cuda_device):
    rng = np.random.default_rng(4)
    N, D = 70, 100
    X = rng.standard_normal((N, D))
    ko, kp = build(("sum", "rbf_ard", "lin"), D, [O, gpf.kernels])
    assert_allclose(to_np(kp(X)), ko(X), rtol=1e-11, atol=1e-11)


def test_separate_independent_stack(cuda_device):
    rng = np.random.default_rng(5)
    X = rng.standard_normal((40, 3))
    kos, kps = zip(*[build(e, 3, [O, gpf.kernels], seed=i) for i, e in enumerate(["rbf", "m32", ("prod", "m52", "lin")])])
    mo_o, mo_p = O.SeparateIndependent(kos), gpf.kernels.SeparateIndependent(kps)
    assert_allclose(to_np(mo_p.K(X)), mo_o.K(X), rtol=1e-11, atol=1e-12)
    assert_allclose(to_np(mo_p.K_diag(X)), mo_o.K_diag(X), rtol=1e-11, atol=1e-12)


# ---- GEMM ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("ta,tb", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("m,n,k", [(128, 128, 128), (300, 200, 77), (1, 5, 3), (129, 257, 130), (64, 3, 500)])
def test_gemm_matches_numpy(cuda_device, dtype, ta, tb, m, n, k):
    rng = np.random.default_rng(6)
    A = rng.standard_normal((k, m) if ta else (m, k)).astype(dtype)
    B = rng.standard_normal((n, k) if tb else (k, n)).astype(dtype)
    C = rng.standard_normal((m, n)).astype(dtype)
    ref = 0.7 * (A.T if ta else A).astype(np.float64) @ (B.T if tb else B).astype(np.float64) - 0.3 * C
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Cd = ops.to_device(C.copy())
        ops.gemm(ops.to_device(A), ops.to_device(B), transa=bool(ta), transb=bool(tb), alpha=0.7, beta=-0.3, out=Cd)
    t = dict(rtol=1e-11, atol=1e-11) if dtype == np.float64 else dict(rtol=1e-4, atol=1e-4 * np.sqrt(k))
    assert_allclose(to_np(Cd), ref, **t)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_gemm_flags(cuda_device, dtype):
    rng = np.random.default_rng(7)
    m, k, n = 300, 260, 190
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        t = dict(rtol=1e-10, atol=1e-10) if dtype == np.float64 else dict(rtol=2e-4, atol=2e-3)
        # SYRK lower-only
        A = rng.standard_normal((m, k)).astype(dtype)
        C = ops.full((m, m), 5.0, dtype=dtype)
        ops.gemm(ops.to_device(A), ops.to_device(A), transb=True, out=C, flags=_lib.GPK_GEMM_LOWER_ONLY)
        ref = A.astype(np.float64) @ A.T.astype(np.float64)
        il = np.tril_indices(m)
        assert_allclose(to_np(C)[il], ref[il], **t)
        assert np.all(to_np(C)[:128, 128:] == 5.0)
        # lower-triangular A^T (q_sqrt^T A) with and without the fused column-sum-of-squares epilogue
        Q = rng.standard_normal((k, k)).astype(dtype)
        Bm = rng.standard_normal((k, n)).astype(dtype)
        ref = np.tril(Q).T.astype(np.float64) @ Bm.astype(np.float64)
        got = ops.gemm(ops.to_device(Q), ops.to_device(Bm), transa=True, flags=_lib.GPK_GEMM_A_LOWER)
        assert_allclose(to_np(got), ref, **t)
        v = ops.full((n,), 1.5, dtype=dtype)
        ops.gemm(ops.to_device(Q), ops.to_device(Bm), transa=True, out=v,
                 flags=_lib.GPK_GEMM_A_LOWER | _lib.GPK_GEMM_COLSUMSQ)
        assert_allclose(to_np(v), 1.5 + (ref ** 2).sum(0), rtol=1e-9 if dtype == np.float64 else 1e-4)
        # lower-triangular A, not transposed
        got = ops.gemm(ops.to_device(Q), ops.to_device(Bm), flags=_lib.GPK_GEMM_A_LOWER)
        assert_allclose(to_np(got), np.tril(Q).astype(np.float64) @ Bm.astype(np.float64), **t)


# ---- Cholesky / triangular solves ------------------------------------------------------------------
def _spd(n, rng, dtype):
    A = rng.standard_normal((n, n + 5))
    return (A @ A.T / n + 0.5 * np.eye(n)).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", [1, 5, 31, 32, 33, 127, 128, 129, 300, 513, 1000])
def test_potrf_matches_lapack(cuda_device, dtype, n):
    rng = np.random.default_rng(8)
    K = _spd(n, rng, dtype)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        L, _ = ops.cholesky(ops.to_device(K))
    ref = sla.cholesky(K.astype(np.float64), lower=True)
    t = dict(rtol=1e-10, atol=1e-11) if dtype == np.float64 else dict(rtol=5e-4, atol=5e-5)
    assert_allclose(to_np(L), ref, **t)
    assert np.all(np.triu(to_np(L), 1) == 0)


def test_potrf_extra_rows_give_solves(cuda_device):
    rng = np.random.default_rng(9)
    n, p = 333, 3
    K = _spd(n, rng, np.float64)
    Y = rng.standard_normal((n, p))
    A = np.full((n + p, n), np.nan)
    A[:n][np.tril_indices(n)] = K[np.tril_indices(n)]   # only the lower triangle is ever read
    A[n:] = Y.T
    Ad = ops.to_device(np.nan_to_num(A, nan=123.0))
    ops.potrf(Ad, n)
    L = sla.cholesky(K, lower=True)
    got = to_np(Ad)
    assert_allclose(np.tril(got[:n]), L, rtol=1e-10, atol=1e-11)
    assert_allclose(got[n:], sla.solve_triangular(L, Y, lower=True).T, rtol=1e-9, atol=1e-10)
    assert np.all(np.triu(got[:n], 1)[:128, 128:] == 123.0)  # strict upper tiles untouched


def test_potrf_panel_grid_larger_than_the_gpu(cuda_device):
    """n = 9856: the panel kernels below the first diagonal blocks have more CTAs than the GPU has SMs.  Those launches are
    ordered behind their leaf by an event; smaller grids poll the leaf's completion counter (a grid that fills every SM
    with polling CTAs would lock the leaf out -- potrf.cu::potrf_block).  The factor is checked through L L^T = A on a
    sample of rows and through log det against LAPACK."""
    rng = np.random.default_rng(12)
    n = 9856
    B = rng.standard_normal((n, 64))
    d = 1.0 + rng.uniform(0, 1, n)
    K = B @ B.T / 64 + np.diag(d)
    L, _ = ops.cholesky(ops.to_device(K))
    Ln = to_np(L)
    rows = rng.choice(n, 40, replace=False)
    assert_allclose(Ln[rows] @ Ln.T, K[rows], rtol=0, atol=2e-10)
    sign, logdet = np.linalg.slogdet(K)
    assert_allclose(2.0 * np.log(np.diag(Ln)).sum(), logdet, rtol=1e-11)


def test_debug_trace_records_the_chain_of_a_factorisation(cuda_device):
    """gpk_debug_trace: %globaltimer marks of the leaf / panel / update kernels of one factorisation (n = 1024: 8 leaves,
    4 fused + 3 plain panels, 3 int8 tensor-core updates); switching it off stops the recording; the factor is unaffected."""
    import ctypes
    import torch
    from gpflow_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(13)
    n = 1024
    K = _spd(n, rng, np.float64)
    ref = sla.cholesky(K, lower=True)
    cap = 512
    buf = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.gpk_debug_trace(ctypes.c_void_p(buf.data_ptr()), ctypes.c_void_p(pos.data_ptr()), cap) == 0
    try:
        L, _ = ops.cholesky(ops.to_device(K))
        torch.cuda.synchronize()
    finally:
        assert lib.gpk_debug_trace(None, None, 0) == 0
    assert_allclose(to_np(L), ref, rtol=1e-10, atol=1e-11)
    nmarks = int(pos.item())
    assert 0 < nmarks <= cap
    b = buf.cpu().numpy()[: 2 * nmarks].reshape(nmarks, 2)
    kid, phase = b[:, 1] >> 8, b[:, 1] & 255
    assert np.sum((kid == 1) & (phase == 0)) == 8 and np.sum((kid == 1) & (phase == 2)) == 8      # leaves: started, done
    assert np.sum((kid == 2) & (phase == 0)) == 4 and np.sum((kid == 3) & (phase == 0)) >= 3      # fused / plain panels
    assert np.sum((kid == 4) & (phase == 0)) == 3                                                    # K = 256, 512, 256
    t = b[:, 0]
    assert t.max() - t.min() < 50_000_000                                                            # one factorisation: << 50 ms
    ops.cholesky(ops.to_device(K))
    torch.cuda.synchronize()
    assert int(pos.item()) == nmarks                                                                 # off: nothing appended


def test_potrf_reports_non_positive_definite(cuda_device):
    rng = np.random.default_rng(10)
    n = 200
    K = _spd(n, rng, np.float64)
    K[150, 150] = -1.0
    with pytest.raises(ops.NonPositiveDefiniteError) as e:
        ops.cholesky(ops.to_device(K))
    assert "151" in str(e.value)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("trans", [False, True])
@pytest.mark.parametrize("n,nrhs", [(5, 3), (128, 1), (129, 40), (300, 257), (700, 2)])
def test_trsm_matches_lapack(cuda_device, dtype, trans, n, nrhs):
    rng = np.random.default_rng(11)
    K = _spd(n, rng, np.float64)
    L = sla.cholesky(K, lower=True)
    B = rng.standard_normal((n, nrhs))
    ref = sla.solve_triangular(L, B, lower=True, trans=1 if trans else 0)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Ld, Bd = ops.to_device(L.astype(dtype)), ops.to_device(B.astype(dtype))
        ops.trsm(Ld, Bd, trans=trans)                       # diagonal-block inverses recomputed
        t = dict(rtol=1e-9, atol=1e-10) if dtype == np.float64 else dict(rtol=2e-3, atol=2e-3)
        assert_allclose(to_np(Bd), ref, **t)
        Kd = ops.to_device(K.astype(dtype))
        L2, dinv = ops.cholesky(Kd)
        B2 = ops.to_device(B.astype(dtype))
        ops.trsm(L2, B2, trans=trans, dinv=dinv)            # cached inverses from potrf
        assert_allclose(to_np(B2), ref, **t)


# ---- reductions / elementwise -----------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_reductions_and_gaussian_varexp(cuda_device, dtype):
    rng = np.random.default_rng(12)
    A = rng.standard_normal((301, 77)).astype(dtype)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Ad = ops.to_device(A)
        r = 1e-12 if dtype == np.float64 else 1e-5
        assert_allclose(to_np(ops.colsumsq(Ad, scale=-2.0)), -2.0 * (A.astype(np.float64) ** 2).sum(0), rtol=r)
        assert_allclose(to_np(ops.reduce(ops.SUM, Ad, A.size)), A.astype(np.float64).sum(), rtol=1e-6, atol=1e-6)
        assert_allclose(to_np(ops.reduce(ops.SUMSQ, Ad, A.size)), (A.astype(np.float64) ** 2).sum(), rtol=1e-6)
        P = np.abs(A[:77, :77]) + 0.1
        Pd = ops.to_device(P)
        assert_allclose(to_np(ops.reduce(ops.SUMLOG, Pd, 77, 78)), np.log(np.diag(P).astype(np.float64)).sum(), rtol=1e-6)
        assert_allclose(to_np(ops.reduce(ops.SUMLOGSQ, Pd, 77, 78)), np.log(np.diag(P).astype(np.float64) ** 2).sum(), rtol=1e-6)
        Q = rng.standard_normal((3, 50, 50)).astype(dtype)
        assert_allclose(to_np(ops.tril_sumsq(ops.to_device(Q))), (np.tril(Q).astype(np.float64) ** 2).sum(), rtol=1e-6)
        assert_allclose(to_np(ops.transpose(Ad)), A.T)
        Y = ops.to_device(A.copy())
        ops.axpby(2.0, Ad, -1.0, Y)
        assert_allclose(to_np(Y), A, rtol=1e-6)
        s = (np.abs(rng.standard_normal(77)) + 0.5).astype(dtype)
        assert_allclose(to_np(ops.scale_cols_(ops.to_device(A.copy()), ops.to_device(s), invert=True)), A / s, rtol=1e-6)
        s = (np.abs(rng.standard_normal(301)) + 0.5).astype(dtype)
        assert_allclose(to_np(ops.scale_rows_(ops.to_device(A.copy()), ops.to_device(s))), A * s[:, None], rtol=1e-6)
        Fmu, Fvar, Yv = rng.standard_normal((40, 3)).astype(dtype), rng.random((40, 3)).astype(dtype), rng.standard_normal((40, 3)).astype(dtype)
        gauss = _lib.LikDesc(_lib.LIK_GAUSSIAN, 20, 0.0, 0.0, 0.0, 0.3)
        got = ops.lik_varexp_sum(gauss, ops.to_device(Fmu), ops.to_device(Fvar), ops.to_device(Yv), scale=2.0)
        assert_allclose(to_np(got), 2.0 * O.gaussian_variational_expectations(Fmu.astype(np.float64), Fvar.astype(np.float64), Yv.astype(np.float64), 0.3).sum(), rtol=1e-6)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["rbf", "rbf_ard", "m12", "m32", "m52", "exp"])
def test_kbuild_fast_path_modes(cuda_device, name, dtype):
    """Single-stationary-leaf fast path: rectangular, symmetric full (mirrored tiles) and lower-only, ragged N,
    far-apart points (exp underflow) and coincident points (the 1e-36 clip)."""
    rng = np.random.default_rng(21)
    N, N2, D = 333, 190, 5
    X = rng.standard_normal((N, D)) * np.where(rng.random((N, 1)) < 0.1, 8.0 if dtype == np.float64 else 3.0, 1.0)  # outliers
    X[5] = X[4]                                                                       # duplicate row
    X2 = rng.standard_normal((N2, D))
    X, X2 = X.astype(dtype), X2.astype(dtype)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        ko, kp = build(EXPRS[name], D, [O, gpf.kernels])
        Xd, X2d = ops.to_device(X), ops.to_device(X2)
        t = tol_for(EXPRS[name], dtype)
        if dtype == np.float32:  # eps * |x|^2 noise of the norm-expansion distance with |x| up to ~7
            t = dict(rtol=max(t["rtol"], 1e-4), atol=max(t["atol"], 1e-4))
        elif name in ("m12", "exp"):  # sqrt(eps * |x|^2) with the |x|~18 outliers
            t = dict(rtol=1e-6, atol=1e-6)
        full = to_np(kp(Xd))
        ref = ko(X)
        chk, rchk = full.copy(), ref.copy()
        if dtype == np.float32:  # the coincident pair carries the reference formulation's own eps*|x|^2 noise
            chk[4, 5] = chk[5, 4] = rchk[4, 5] = rchk[5, 4] = 0.0
        assert_allclose(chk, rchk, **t)
        bad = np.argwhere(full != full.T)  # mirrored tiles are copies; diagonal tiles round symmetrically
        assert len(bad) == 0, f"asymmetric entries, first: {bad[:6].tolist()} count {len(bad)}"
        assert_allclose(to_np(kp(Xd, X2d)), ko(X, X2), **tol(dtype))
        desc = gpf.kernels.compile_kernel(kp, D)
        low = ops.full((N, N), -3.0, like=Xd)
        ops.kbuild(desc, Xd, None, uplo=_lib.GPK_LOWER, diag_scalar=0.5, out=low)
        il = np.tril_indices(N)
        lchk, lref = to_np(low), ref + 0.5 * np.eye(N)
        if dtype == np.float32:
            lchk[5, 4] = lref[5, 4] = 0.0
        assert_allclose(lchk[il], lref[il], **t)
        assert np.all(to_np(low)[:64, 64:] == -3.0)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("n", [1, 37, 128, 300])
def test_potrf_batched_matches_lapack(cuda_device, dtype, n):
    """gpk_potrf_batched: a stack [L, n, n] (multi-output Kuu, covariances/multioutput/kuus.py:62-122); n <= 128 is one
    launch with one CTA per matrix, larger n runs the factorisations back to back."""
    rng = np.random.default_rng(n)
    Lb = 5
    mats = []
    for _ in range(Lb):
        B = rng.standard_normal((n, n + 3))
        mats.append(B @ B.T / n + 0.5 * np.eye(n))
    A = np.stack(mats).astype(dtype)
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Ad = ops.to_device(A.copy())
        ops.potrf_batched(Ad)
    got = np.tril(Ad.cpu().numpy().astype(np.float64))
    ref = np.stack([np.linalg.cholesky(m) for m in A.astype(np.float64)])
    assert_allclose(got, ref, rtol=0, atol=2e-11 if dtype == np.float64 else 3e-4)
    bad = A.copy()
    bad[3, n - 1, n - 1] = -1.0
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        with pytest.raises(ops.NonPositiveDefiniteError):
            ops.potrf_batched(ops.to_device(bad))
