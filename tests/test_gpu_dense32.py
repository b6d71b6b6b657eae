"""The fp32 dense products of the SGPR and SVGP objectives element by element against the bars of
tests/dense32_bounds.py: the 3xTF32 GEMM (every transposition, ragged shapes, one and two row tiles per cluster,
split-K up to 64 splits, A_LOWER, LOWER_ONLY, strided views), the statistical bars (RMS of the relative error, the
truncation bias of the C3 product A A^T at K = 1e5), the batched column sums of squares of the SVGP variance through
gpk_debug_gemm_tf32_batched, the SVGP forward's fmean / fvar read from its workspace, and the skinny kernel at the
depths the objectives run it.  tests/_dense32_worker.py reruns the GEMM, COLSUMSQ and SVGP lists under
GPK_FP32_ENGINE=simt and under GPK_TF32_CLUSTER=1 with GPK_SVGP_BATCHED=0."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import dense32_bounds as D
from tests import dense64_bounds as DB
from tests import test_gpu_dense64 as G

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = 0
SENT = -777.25
ENGINE = "simt" if os.environ.get("GPK_FP32_ENGINE") == "simt" else "tf32"
CLUSTER = 1 if os.environ.get("GPK_TF32_CLUSTER", "").startswith("1") else 2
BATCHED = os.environ.get("GPK_SVGP_BATCHED", "1") != "0"
TINY = np.finfo(np.float64).tiny
WORST = {}


def record(name, r):
    lo, hi = WORST.get(name, (np.inf, 0.0))
    WORST[name] = (min(lo, r), max(hi, r))


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def _t():
    import torch
    return torch


# ---- GEMM ------------------------------------------------------------------------------------------------------------
GEMM_CASES = {
    # name: (m, n, k, ta, tb, alpha, beta, flags, view)
    "t00": (1401, 1403, 777, 0, 0, 1.3, 0.0, 0, None),
    "t01": (1401, 1403, 777, 0, 1, -0.7, 1.0, 0, None),
    "t10": (1401, 1403, 777, 1, 0, 0.9, 0.3, 0, None),
    "t11": (1401, 1403, 777, 1, 1, 1.0, 0.0, 0, None),
    "one_row_tile": (100, 20011, 301, 0, 1, 1.0, 0.3, 0, None),
    "splitk2": (1280, 1280, 4096, 1, 0, 1.0, 0.0, 0, None),
    "splitk8_beta1": (512, 512, 8192, 0, 1, 1.0, 1.0, 0, None),
    "splitk8_beta03": (300, 1000, 8192, 0, 0, -1.1, 0.3, 0, None),
    "splitk64": (128, 128, 65536, 0, 1, 1.0, 1.0, 0, None),
    "splitk4_lower_beta03": (1024, 1024, 20000, 0, 1, 1.0, 0.3, DB.GEMM_LOWER_ONLY, None),
    "splitk8_lower_beta0": (512, 512, 8192, 0, 1, 1.0, 0.0, DB.GEMM_LOWER_ONLY, None),
    "splitk8_lower_beta1": (640, 640, 16384, 0, 1, 1.0, 1.0, DB.GEMM_LOWER_ONLY, None),
    "lower_beta1": (1500, 1500, 900, 0, 1, 1.0, 1.0, DB.GEMM_LOWER_ONLY, None),
    "a_lower_tri1": (1100, 2000, 1100, 0, 0, 1.0, 0.5, DB.GEMM_A_LOWER, None),
    "a_lower_tri2": (1100, 2000, 1100, 1, 0, -0.8, 0.0, DB.GEMM_A_LOWER, None),
    "a_lower_tri2_lower": (1100, 1100, 1100, 1, 0, 1.0, 0.0, DB.GEMM_A_LOWER | DB.GEMM_LOWER_ONLY, None),
    "view_odd_ld": (1401, 1403, 777, 0, 1, 0.8, 1.0, 0, 1),
    "view_unaligned_base": (1401, 1403, 777, 1, 0, 0.8, 1.0, 0, 0),
}


def gemm_case(name):
    m, n, k, ta, tb, alpha, beta, flags, view = GEMM_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    A, B, C0 = G.operands(m, n, k, ta, tb, rng, a_lower=bool(flags & DB.GEMM_A_LOWER))
    A, B, C0 = f32(A), f32(B), f32(C0)
    if beta == 0:
        C0[:] = np.nan                                      # beta = 0: C is never read
    if flags & DB.GEMM_LOWER_ONLY:
        C0[DB.tiles_written(m, n, (128, 128), flags) == 0] = SENT
    return A, B, C0


def kernel_of(m, n, k, flags, tb):
    return D.gemm_kernel(m, n, k, flags, None, tb, ENGINE)


def check32(A, B, C0, alpha, beta, ta, tb, flags, C, rng, kernel, nsplit, name):
    """Worst error / bar of the device C: long double on tile-edge rows and columns plus random ones (fp64 with its own
    bar added above k = 8192), the whole matrix against fp64 with the bar doubled, and on tf32 the RMS statistic over
    every written entry.  Returns (ratio, rms / rms bar or None)."""
    m, n = C.shape
    a_lower = bool(flags & DB.GEMM_A_LOWER)
    As = np.tril(np.nan_to_num(A)) if a_lower else A
    oa, ob = DB.opmat(As, ta), DB.opmat(B, tb)
    k = oa.shape[1]
    g = D.g_tf32(k, nsplit) if kernel == "tf32" else D.g_simt(k)
    tile = (128, 128) if kernel == "tf32" else DB.dmma_tile(m, n, flags, None, tb, k)
    mask = DB.tiles_written(m, n, tile, flags)
    if flags & DB.GEMM_LOWER_ONLY:
        assert (~mask).any()
        assert np.array_equal(C[~mask], C0[~mask], equal_nan=True), "LOWER_ONLY wrote a skipped tile"
    C0z = np.nan_to_num(C0) if beta == 0 else C0
    rows, cols = D.edge_indices(m, rng), D.edge_indices(n, rng)
    keep = mask[np.ix_(rows, cols)]
    sa, sb = oa[rows], ob[:, cols]
    if k <= 8192:
        ref = np.longdouble(alpha) * (sa.astype(np.longdouble) @ sb.astype(np.longdouble))
        gr = (k + 2) * DB.U_LD
    else:
        ref = alpha * (sa @ sb)
        gr = D.g_ref(k)
    mag = abs(alpha) * (np.abs(sa) @ np.abs(sb))
    if beta != 0:
        ref = ref + beta * C0z[np.ix_(rows, cols)].astype(np.longdouble)
        mag = mag + abs(beta) * np.abs(C0z[np.ix_(rows, cols)])
    err = np.abs(C[np.ix_(rows, cols)].astype(np.longdouble) - ref).astype(np.float64)
    r = DB.ratio(err[keep], ((g + gr) * mag * (1 + 1e-6) + TINY)[keep])
    full = alpha * (oa @ ob) + (beta * C0z if beta != 0 else 0.0)
    fmag = abs(alpha) * (np.abs(oa) @ np.abs(ob)) + (abs(beta) * np.abs(C0z) if beta != 0 else 0.0)
    ferr = np.abs(C - full)
    rf = DB.ratio(ferr[mask], (2 * (g + D.g_ref(k)) * fmag * (1 + 1e-6) + TINY)[mask])
    rms = None
    if kernel == "tf32" and mask.sum() >= 100000:
        rms = D.rms_rel(ferr[mask], fmag[mask]) / D.rms_bar(k)
        record("gemm_tf32_rms", rms)
    record(f"gemm_{kernel}", max(r, rf))
    return max(r, rf), rms


def run_gemm_case(name):
    m, n, k, ta, tb, alpha, beta, flags, view = GEMM_CASES[name]
    A, B, C0 = gemm_case(name)
    kernel = kernel_of(m, n, k, flags, tb)
    cl, nsplit = D.tf32_launch(m, n, k, flags, 1, CLUSTER)
    if view is None:
        C, _, _ = G.run_gemm(A, B, C0, alpha, beta, ta, tb, flags, dtype=np.float32)
    else:
        C, after, before = G.run_gemm(A, B, C0, alpha, beta, ta, tb, flags, ldpad=2, offset=1, ld_parity=view,
                                      dtype=np.float32)
        inside = np.zeros(after.shape, dtype=bool)
        inside[1:1 + m, 1:1 + n] = True
        assert after.shape[1] % 2 == view
        assert np.array_equal(after[~inside], before[~inside]), "a sentinel outside the view was overwritten"
    tile = (128, 128) if kernel == "tf32" else DB.dmma_tile(m, n, flags, None, tb, k)
    assert np.isfinite(C[DB.tiles_written(m, n, tile, flags)]).all()
    r, rms = check32(A, B, C0, alpha, beta, ta, tb, flags, C, np.random.default_rng(1), kernel, nsplit, name)
    assert r <= 1.0, r
    if rms is not None:
        assert rms <= 1.0, rms
    return kernel, cl, nsplit


@pytest.mark.parametrize("name", sorted(GEMM_CASES))
def test_gemm_fp32_inside_bar(cuda_device, name):
    run_gemm_case(name)


def test_gemm_cases_reach_every_configuration():
    """Under the default switches the list reaches the tf32 kernel in all four transpositions, both cluster widths,
    split-K from 2 to 64 (the largest the rule picks) with beta 0, 1 and 0.3 with and without LOWER_ONLY, and both
    triangular forms of A_LOWER."""
    seen = set()
    for name, (m, n, k, ta, tb, alpha, beta, flags, view) in GEMM_CASES.items():
        assert D.gemm_kernel(m, n, k, flags, None, tb) == "tf32", name
        cl, nsplit = D.tf32_launch(m, n, k, flags)
        seen |= {("trans", ta, tb), ("cl", cl), ("nsplit", nsplit)}
        if nsplit > 1:
            seen.add(("splitk", beta, bool(flags & DB.GEMM_LOWER_ONLY)))
        if flags & DB.GEMM_A_LOWER:
            seen.add(("tri", 2 if ta else 1))
    want = {("trans", a, b) for a in (0, 1) for b in (0, 1)} | {("cl", 1), ("cl", 2), ("tri", 1), ("tri", 2)}
    want |= {("nsplit", s) for s in (2, 8, 64)} | {("splitk", b, lo) for b in (0.0, 1.0, 0.3) for lo in (False, True)}
    assert want <= seen, want - seen


def test_c3_syrk_bias_and_rms(cuda_device):
    """A A^T at the SGPR shape (m = 1024, k = 1e5, LOWER_ONLY, split-K): every written entry inside the bar, the RMS
    statistic, and the mean signed relative error of the diagonal, where every product is positive and a truncating
    accumulation cannot cancel."""
    torch = _t()
    m, k = 1024, 100000
    kernel = kernel_of(m, m, k, DB.GEMM_LOWER_ONLY, 1)
    cl, nsplit = D.tf32_launch(m, m, k, DB.GEMM_LOWER_ONLY, 1, CLUSTER)
    g = torch.Generator(device="cuda").manual_seed(11)
    dA = torch.randn((m, k), generator=g, device="cuda", dtype=torch.float32)
    dC = torch.full((m, m), SENT, device="cuda", dtype=torch.float32)
    assert G.lib().gpk_gemm(0, 1, m, m, k, 1.0, G.ptr(dA), k, G.ptr(dA), k, 0.0, G.ptr(dC), m, F32,
                            DB.GEMM_LOWER_ONLY, None) == 0, G.err()
    G.sync()
    C = dC.cpu().numpy().astype(np.float64)
    A = dA.cpu().numpy().astype(np.float64)
    del dA, dC
    tile = (128, 128) if kernel == "tf32" else DB.dmma_tile(m, m, DB.GEMM_LOWER_ONLY, None, 1, k)
    mask = DB.tiles_written(m, m, tile, DB.GEMM_LOWER_ONLY)
    assert (C[~mask] == SENT).all()
    ref = A @ A.T
    mag = np.abs(A) @ np.abs(A).T
    gk = D.g_tf32(k, nsplit) if kernel == "tf32" else D.g_simt(k)
    err = np.abs(C - ref)
    r = DB.ratio(err[mask], ((gk + D.g_ref(k)) * mag + TINY)[mask])
    record(f"gemm_{kernel}", r)
    assert r <= 1.0, r
    if kernel == "tf32":
        rms = D.rms_rel(err[mask], mag[mask]) / D.rms_bar(k)
        bias = D.signed_bias(np.diag(C), np.diag(ref))
        record("gemm_tf32_rms", rms)
        record("c3_diag_bias", abs(bias) / D.BIAS_BAR)
        print(f"C3 A A^T: rms {rms * D.rms_bar(k):.3e} (bar {D.rms_bar(k):.3e}), diagonal bias {bias:.3e} "
              f"(bar {D.BIAS_BAR:.1e}), worst ratio {r:.3e}, nsplit {nsplit}, cl {cl}")
        assert rms <= 1.0, rms
        assert abs(bias) <= D.BIAS_BAR, bias


# ---- batched COLSUMSQ ------------------------------------------------------------------------------------------------
COLSUMSQ_CASES = [(2, 256, 1000), (3, 512, 4099), (8, 2048, 4096), (16, 256, 4099), (2, 2048, 1000), (3, 256, 4096),
                  (16, 512, 1000)]


def q_factors(P, M, rng):
    q = np.tril(rng.standard_normal((P, M, M))) * (1 / np.sqrt(M)) + np.eye(M)[None]
    q = f32(q)
    q[:, np.triu(np.ones((M, M), dtype=bool), 1)] = np.nan   # never read
    return q


def colsumsq_ref(q, A, cols, v0, alpha=1.0):
    """fp64 v0 + sum_i (alpha tril(q_p)^T A)_ij^2 on the columns `cols`, and its bar (the fp64 reference's own error
    added to the GEMM's)."""
    P, M, _ = q.shape
    ref, bar = [], []
    g = D.g_tf32(M) + D.g_ref(M)
    for p in range(P):
        L = np.tril(np.nan_to_num(q[p]))
        y = alpha * (L.T @ A[:, cols])
        s = abs(alpha) * (np.abs(L).T @ np.abs(A[:, cols]))
        ref.append(v0[p][cols] + (y ** 2).sum(axis=0))
        bar.append(D.colsumsq_bar(y, s, g, M, v0[p][cols]) + D.g_ref(M) * (s ** 2).sum(axis=0))
    return np.array(ref), np.array(bar) * (1 + 1e-6) + TINY


@pytest.mark.parametrize("P,M,B", COLSUMSQ_CASES)
def test_batched_colsumsq_inside_bar(cuda_device, P, M, B):
    """fvar_p = v0_p + colsum((tril(q_p)^T A)^2) for P latents in one launch: NaN above every q_p's diagonal, the
    output prefilled, its batch stride past B with sentinels in the gaps that must survive."""
    rng = np.random.default_rng(P * 100 + M + B)
    q = q_factors(P, M, rng)
    ldb, cst = B + 3, B + 5
    A = f32(rng.standard_normal((M, B)))
    Ap = np.full((M, ldb), SENT)
    Ap[:, :B] = A
    v0 = f32(rng.uniform(0.5, 2.0, (P, B)))
    out0 = np.full((P, cst), SENT)
    out0[:, :B] = v0
    torch = _t()
    dq, dA, dout = G.dev(q, np.float32), G.dev(Ap, np.float32), G.dev(out0, np.float32)
    rc = G.lib().gpk_debug_gemm_tf32_batched(1, 0, M, B, M, 1.0, G.ptr(dq), M, G.ptr(dA), ldb, 0.0, G.ptr(dout), 0,
                                             DB.GEMM_A_LOWER | DB.GEMM_COLSUMSQ, P, M * M, cst, None)
    assert rc == 0, G.err()
    G.sync()
    out = dout.cpu().numpy().astype(np.float64)
    del dq, dA, dout
    torch.cuda.empty_cache()
    assert (out[:, B:] == SENT).all(), "a gap between the batches was written"
    got = out[:, :B]
    assert np.isfinite(got).all()
    cols = D.edge_indices(B, rng, extra=64)
    ref, bar = colsumsq_ref(q, A, cols, v0)
    r = DB.ratio(np.abs(got[:, cols] - ref), bar)
    record("colsumsq_batched", r)
    assert r <= 1.0, r


def test_batched_colsumsq_refusals(cuda_device):
    x = G.dev(np.ones((512, 512)), np.float32)
    lib = G.lib()
    for flags, m, want in [(DB.GEMM_A_LOWER, 256, "batched form needs COLSUMSQ"),
                           (DB.GEMM_A_LOWER | DB.GEMM_COLSUMSQ, 128, "m % 256 == 0"),
                           (DB.GEMM_COLSUMSQ, 300, "m % 256 == 0")]:
        rc = lib.gpk_debug_gemm_tf32_batched(1, 0, m, 256, m, 1.0, G.ptr(x), 512, G.ptr(x), 512, 0.0, G.ptr(x), 0,
                                             flags, 2, 0, 256, None)
        assert rc == -1 and want in G.err(), (flags, m, G.err())
    G.sync()
    assert float(x.sum()) == x.numel()


# ---- SVGP forward ----------------------------------------------------------------------------------------------------
# (B, M, P, p_begin, p_end, q_diag): rows reaching every fvar path (dense64_bounds-style mirror: D.svgp_fvar_path)
SVGP_CASES = [(1000, 512, 3, 0, 3, False), (1000, 512, 4, 1, 3, False), (1000, 640, 3, 0, 3, False),
              (1000, 512, 3, 1, 2, False), (700, 512, 3, 0, 3, False), (1000, 512, 3, 0, 3, True),
              (4096, 2048, 8, 0, 8, False)]


def svgp_setup(B, M, P, q_diag, seed):
    import gpflow_b200 as gpf
    from gpflow_b200.kernels import compile_kernel

    rng = np.random.default_rng(seed)
    Dd = 3
    X, Z = f32(rng.uniform(-2, 2, (B, Dd))), f32(rng.uniform(-2, 2, (M, Dd)))
    Y = f32(rng.standard_normal((B, P)))
    q_mu = f32(rng.standard_normal((M, P)))
    if q_diag:
        q_sqrt = f32(rng.uniform(0.2, 1.2, (M, P)))
    else:
        q_sqrt = np.nan_to_num(q_factors(P, M, rng))            # the layout the model stores (strict upper part 0)
    with gpf.config.as_context(gpf.config.Config(float=np.float32, jitter=1e-3)):
        k = gpf.kernels.SquaredExponential(lengthscales=1.3)
        nodes = compile_kernel(k, Dd)
        lik = gpf.likelihoods.Gaussian(0.3)._lik_desc()
    return dict(X=X, Y=Y, Z=Z, q_mu=q_mu, q_sqrt=q_sqrt, nodes=nodes, lik=lik, D=Dd)


def svgp_run(s, B, M, P, p0, p1, q_diag, whiten, stage, ws=None, A=None):
    """gpk_svgp_elbo_staged in fp32; with A given, planted in the workspace before stage 2.  Returns (fmu [B, Pl],
    fvar [Pl, B], A [M, B] from the workspace, ws)."""
    torch = _t()
    lib = G.lib()
    need = int(lib.gpk_svgp_elbo_ws(B, M, P, F32))
    if ws is None:
        ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    ld = ctypes.c_int64(0)
    offA = int(lib.gpk_svgp_elbo_A(B, M, P, F32, ctypes.byref(ld)))
    Aw = ws[offA:offA + M * ld.value * 4].view(torch.float32).view(M, ld.value)
    if A is not None:
        Aw[:, :B] = torch.from_numpy(A.astype(np.float32)).cuda()
    fo, vo = ctypes.c_int64(0), ctypes.c_int64(0)
    assert lib.gpk_svgp_elbo_fmu_fvar(B, M, P, F32, ctypes.byref(fo), ctypes.byref(vo)) == 0, G.err()
    d = {k: G.dev(v, np.float32) for k, v in s.items() if k in ("X", "Y", "Z", "q_mu", "q_sqrt")}
    out = torch.zeros(4, dtype=torch.float64, device="cuda")
    nodes, n_nodes, dims, ard = s["nodes"]
    rc = lib.gpk_svgp_elbo_staged(nodes, n_nodes, dims, ard, G.ptr(d["X"]), B, s["D"], s["D"], G.ptr(d["Y"]), None, P,
                                  G.ptr(d["Z"]), M, s["D"], G.ptr(d["q_mu"]), G.ptr(d["q_sqrt"]), int(q_diag),
                                  int(whiten), ctypes.byref(s["lik"]), 1.0, 1e-3, p0, p1, stage, 0, B, F32,
                                  G.ptr(out), G.ptr(ws), None)
    assert rc == 0, G.err()
    G.sync()
    Pl = p1 - p0
    fmu = ws[fo.value:fo.value + B * Pl * 4].view(torch.float32).cpu().numpy().astype(np.float64).reshape(B, Pl)
    fvar = ws[vo.value:vo.value + Pl * B * 4].view(torch.float32).cpu().numpy().astype(np.float64).reshape(Pl, B)
    return fmu, fvar, Aw[:, :B].cpu().numpy().astype(np.float64), ws


def fvar_parts(s, A, fmu, fvar, p0, p1, q_diag, path, v0=None):
    """fmean's worst ratio, and per latent the fvar error and bar, against fp64 from exactly the fp32 A, q_mu, q_sqrt.
    v0 = None: fvar0 = Kdiag - sum A^2 with Kdiag = 1 (SquaredExponential, variance 1) and a bar for colsumsq_kernel's
    fp32 atomics (at most one rounding per row); otherwise the given fvar0, without error of its own."""
    M, B = A.shape
    qm = s["q_mu"][:, p0:p1]
    r_mu = DB.ratio(np.abs(fmu - A.T @ qm), (D.g_simt(M) + D.g_ref(M)) * (np.abs(A).T @ np.abs(qm)) + TINY)
    sumA2 = (A ** 2).sum(axis=0)
    if v0 is None:
        v0, v0_bar = 1.0 - sumA2, D.gamma(M + 2) * (1.0 + sumA2)
    else:
        v0_bar = np.zeros(B)
    g = (D.g_tf32(M) if path in ("batched", "tf32") else D.g_simt(M)) + D.g_ref(M)
    errs, bars = [], []
    for i, p in enumerate(range(p0, p1)):
        if q_diag:
            y = s["q_sqrt"][:, p][:, None] * A
            bar = v0_bar + D.gamma(M + 2) * (np.abs(v0) + (y ** 2).sum(axis=0))
        else:
            L = s["q_sqrt"][p]
            y, sm = L.T @ A, np.abs(L).T @ np.abs(A)
            bar = v0_bar + D.colsumsq_bar(y, sm, g, M, v0) + D.g_ref(M) * (sm ** 2).sum(axis=0)
        errs.append(np.abs(fvar[i] - (v0 + (y ** 2).sum(axis=0))))
        bars.append(bar * (1 + 1e-6) + TINY)
    return r_mu, errs, bars


def fvar_check(s, A, fmu, fvar, p0, p1, q_diag, path):
    r_mu, errs, bars = fvar_parts(s, A, fmu, fvar, p0, p1, q_diag, path)
    return r_mu, max(DB.ratio(e, b) for e, b in zip(errs, bars))


@pytest.mark.parametrize("B,M,P,p0,p1,q_diag", SVGP_CASES)
def test_svgp_forward_fmean_fvar_inside_bars(cuda_device, B, M, P, p0, p1, q_diag):
    """Stage 2 with a planted A (whiten): fmean and fvar against fp64 from the same fp32 A, q_mu and q_sqrt.  Stage 0,
    whitened: its fvar and that of stage 2 on the device's own A (read back from the workspace) inside the same bar.
    Stage 0 without whitening (A in the workspace is then K^-1 Kuf, fvar0 is gone): fmean, and fvar_p - fvar_p0."""
    path = D.svgp_fvar_path(B, M, p1 - p0, q_diag, np.float32, BATCHED, ENGINE)
    s = svgp_setup(B, M, P, q_diag, B + M + P + p0)
    rng = np.random.default_rng(M)
    A = f32(rng.standard_normal((M, B)) * (0.8 / np.sqrt(M)))
    fmu, fvar, _, ws = svgp_run(s, B, M, P, p0, p1, q_diag, True, 2, A=A)
    assert np.isfinite(fmu).all() and np.isfinite(fvar).all()
    r_mu, r_var = fvar_check(s, A, fmu, fvar, p0, p1, q_diag, path)
    record("svgp_fmean", r_mu)
    record(f"svgp_fvar_{path}", r_var)
    assert r_mu <= 1.0 and r_var <= 1.0, (r_mu, r_var, path)
    fmu0, fvar0, A0, _ = svgp_run(s, B, M, P, p0, p1, q_diag, True, 0, ws=ws)
    _, fvar2, _, _ = svgp_run(s, B, M, P, p0, p1, q_diag, True, 2, ws=ws, A=A0)
    for fm, fv in ((fmu0, fvar0), (fmu0, fvar2)):
        r_mu, r_var = fvar_check(s, A0, fm, fv, p0, p1, q_diag, path)
        record("svgp_fmean", r_mu)
        record(f"svgp_fvar_{path}", r_var)
        assert r_mu <= 1.0 and r_var <= 1.0, (r_mu, r_var, path)
    fmu1, fvar1, A1, _ = svgp_run(s, B, M, P, p0, p1, q_diag, False, 0, ws=ws)
    y0 = s["q_sqrt"][:, p0][:, None] * A1 if q_diag else s["q_sqrt"][p0].T @ A1
    v0 = fvar1[0] - (y0 ** 2).sum(axis=0)
    r_mu, errs, bars = fvar_parts(s, A1, fmu1, fvar1, p0, p1, q_diag, path, v0=v0)
    r_var = max([DB.ratio(e, b + bars[0]) for e, b in zip(errs[1:], bars[1:])] + [0.0])
    record("svgp_fmean", r_mu)
    record(f"svgp_fvar_{path}", r_var)
    assert r_mu <= 1.0 and r_var <= 1.0, (r_mu, r_var, path)


def test_svgp_cases_reach_every_fvar_path():
    paths = {D.svgp_fvar_path(B, M, p1 - p0, qd) for B, M, P, p0, p1, qd in SVGP_CASES}
    assert paths == {"batched", "tf32", "simt", "q_diag"}
    assert any(p0 > 0 and p1 - p0 >= 2 and D.svgp_fvar_path(B, M, p1 - p0, qd) == "batched"
               for B, M, P, p0, p1, qd in SVGP_CASES)


# ---- skinny products -------------------------------------------------------------------------------------------------
SKINNY_CASES = [("sgpr_A_Yc", 1024, 1, 100000, 0), ("svgp_At_qmu", 4096, 8, 2048, 1)]


@pytest.mark.parametrize("name,m,n,k,ta", SKINNY_CASES)
def test_skinny_fp32_at_objective_depth(cuda_device, name, m, n, k, ta):
    assert D.gemm_kernel(m, n, k) == "skinny"
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(m + k)
    dA = torch.randn((k, m) if ta else (m, k), generator=g, device="cuda", dtype=torch.float32)
    dB = torch.randn((k, n), generator=g, device="cuda", dtype=torch.float32)
    dC = torch.randn((m, n), generator=g, device="cuda", dtype=torch.float32)
    A, Bm, C0 = (x.cpu().numpy().astype(np.float64) for x in (dA, dB, dC))
    alpha, beta = -0.6, 0.4
    assert G.lib().gpk_gemm(ta, 0, m, n, k, alpha, G.ptr(dA), m if ta else k, G.ptr(dB), n, beta, G.ptr(dC), n, F32,
                            0, None) == 0, G.err()
    G.sync()
    C = dC.cpu().numpy().astype(np.float64)
    oa = A.T if ta else A
    ref = alpha * (oa @ Bm) + beta * C0
    mag = abs(alpha) * (np.abs(oa) @ np.abs(Bm)) + abs(beta) * np.abs(C0)
    r = DB.ratio(np.abs(C - ref), (D.g_simt(k) + D.g_ref(k)) * mag * (1 + 1e-6) + TINY)
    record("skinny", r)
    assert r <= 1.0, r


# ---- engine switches -------------------------------------------------------------------------------------------------
def engine_cases():
    m = sys.modules[__name__]
    g = [(m.test_gemm_fp32_inside_bar, (name,)) for name in sorted(GEMM_CASES)]
    g += [(m.test_c3_syrk_bias_and_rms, ())]
    g += [(m.test_batched_colsumsq_inside_bar, c) for c in COLSUMSQ_CASES[:4]]
    g += [(m.test_svgp_forward_fmean_fvar_inside_bars, c) for c in SVGP_CASES]
    return g


@pytest.mark.parametrize("env", [{"GPK_FP32_ENGINE": "simt"}, {"GPK_TF32_CLUSTER": "1", "GPK_SVGP_BATCHED": "0"}],
                         ids=["simt", "cluster1_unbatched"])
def test_fp32_switches_inside_the_same_bars(cuda_device, tmp_path, env):
    """The switches are read once per process: engine_cases() run in a worker process under each, through the same
    assertions; the bars follow the kernel the mirrors say the switches select."""
    e = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    e.update(env)
    out = str(tmp_path / "w.json")
    r = subprocess.run([sys.executable, "-m", "tests._dense32_worker", out], cwd=ROOT, env=e, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    with open(out) as f:
        res = json.load(f)
    assert res["cases"] == len(engine_cases())
    assert not res["failed"], res["failed"]
    print(env, "worst ratios:", res["worst"])


def test_report_worst_ratios():
    """Prints the (smallest, largest) per-case error / bar of every operator measured in this session."""
    print("worst ratios:", {k: (float(a), float(b)) for k, (a, b) in WORST.items()})
