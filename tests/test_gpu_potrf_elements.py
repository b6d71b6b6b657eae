"""The Cholesky factorisation (csrc/potrf.cu) element by element: every element of R = A - L L^T and R_Y = Y - X L^T, computed
without rounding error, inside the worst-case bar that tests/chol_bounds.py derives from the schedule of the launches that
produced it, and the statistical bars on the RMS and on the diagonal mean of R / (u |L| |L|^T).  The case table reaches
every branch of the schedule mirror (test_case_table_reaches_every_branch).  Every case runs on a view inside a NaN
parent (leading dimension n + 5, NaN guard rows below): the guards and the strict upper triangle outside the 128 x 128
diagonal blocks stay bit-unchanged, and a second run is bit-identical.  Integer-exact factors (every product of the
blocked factorisation exact) must come back exactly, up to n = 37504 where the K = 18816 update falls back to DMMA."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from tests import _potrf_worker as PW
from tests import chol_bounds as CB
from tests import dense64_bounds as DB

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FULL_MAX = 1152              # exact residual of every element up to this n, sampled rows above
WORST = {}


def record(name, r):
    WORST[name] = max(WORST.get(name, 0.0), float(r))


def _t():
    import torch
    return torch


def sms():
    return _t().cuda.get_device_properties(0).multi_processor_count


def rows_for(n, rows, rng):
    return np.arange(rows) if n <= FULL_MAX else CB.sample_rows(n, rows, rng)


def check_factor(T, F, n, rows, diagA, cfg, family, u=CB.U, S=7):
    rng = np.random.default_rng(n + rows)
    ri = rows_for(n, rows, rng)
    r = CB.check(T, F, n, rows, ri, CB.schedule(n, rows, cfg), diagA, u=u, S=S)
    for k, v in r.items():
        record(f"{k}/{family}", v)
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, (n, rows, family, r)


def check_guards(out, before, n, rows):
    """Guard rows, padding columns and the strict upper triangle outside the 128 x 128 diagonal blocks: bit-unchanged."""
    keep = np.ones(out.shape, dtype=bool)
    keep[:rows, :n] = False
    up = np.triu(np.ones((n, n), dtype=bool), 1)
    for o in range(0, n, DB.NB):
        up[o:o + DB.NB, o:o + DB.NB] = False
    keep[:n, :n] |= up
    w = 8 if out.dtype == np.float64 else 4
    iv = np.int64 if w == 8 else np.int32
    assert np.array_equal(out[keep].view(iv), before[keep].view(iv))


def run_and_check(A, Y, n, family, cfg=None, dtype=np.float64):
    rows = n + (0 if Y is None else Y.shape[0])
    T = PW.target(A, Y)
    F, out, before, info, S = PW.factor(T, n, rows, dtype)
    assert info == 0
    check_guards(out, before, n, rows)
    F2, out2, _, _, _ = PW.factor(T, n, rows, dtype)
    assert np.array_equal(out.view(np.uint8), out2.view(np.uint8)), "second run differs"
    if cfg is None and dtype == np.float64:
        # the default engine: int8 updates with S = 7 from n >= 384 (split_point(n) >= 256), so the mirror's branches are
        # the launches that ran
        assert S == (7 if n > DB.NB and DB.split_point(n) >= 256 else 0), (n, S)
    cfg = cfg or CB.Config(S=S or 7, sms=sms(), tc=S > 0, f64=dtype == np.float64)
    u = CB.U if dtype == np.float64 else CB.U32
    Tq = T.astype(dtype).astype(np.float64)
    check_factor(Tq, F, n, rows, np.diag(Tq[:n, :n]), cfg, family, u=u, S=S or 7)
    return F


# ---- the case table --------------------------------------------------------------------------------------------------------
SIZES = [1, 2, 31, 32, 33, 64, 65, 127, 128, 129, 200, 256, 257, 300, 384, 385, 512, 640, 1000, 1152, 2048, 2049, 4096]
EXTRA = [(n, p) for n in (333, 1000, 2049) for p in (1, 2, 3, 127, 128, 129, 300)] + [(100, 5), (128, 129)]
FAMILIES = ["gpr_rbf", "gpr_m52", "dad", "block_cond", "scale_p1000", "scale_m1000", "scale_m1060"]
FAMILY_SIZES = [300, 1000, 2049]
INTEGER = [(n, 0, 0) for n in SIZES] + [(1000, 3, 0), (2049, 129, 0), (300, 0, -1000), (1000, 0, -1000), (2049, 2, -1000),
                                        (300, 0, -1060), (1000, 0, -1060), (2049, 2, -1060)]


def event_ordered_sizes(n_sms):
    """The first n whose first panel grid exceeds n_sms - 8 (by the mirror), and one past it."""
    n = 4096
    while "panel_event_ordered" not in CB.branches(CB.schedule(n, n, CB.Config(sms=n_sms)), n, n):
        n += 1
    return [n, n + 1]


def family_matrix(family, n, rng):
    if family == "spd":
        return CB.random_spd(n, rng)
    if family.startswith("gpr"):
        return CB.gpr_matrix(n, rng, family[4:], 1e-6)
    if family == "dad":
        return CB.dad(n, rng)
    if family == "block_cond":
        L = DB.factor_with_block_cond(n, rng, 1e3)
        return L @ L.T
    e = {"scale_p1000": 1000, "scale_m1000": -1000, "scale_m1060": -1060}[family]
    return np.ldexp(CB.random_spd(n, rng), e)


def table_branches(n_sms):
    b = set()
    for n in SIZES:
        b |= CB.branches(CB.schedule(n, n, CB.Config(sms=n_sms)), n, n)
    for n, p in EXTRA:
        b |= CB.branches(CB.schedule(n, n + p, CB.Config(sms=n_sms)), n, n + p)
    for n in event_ordered_sizes(n_sms) + [37504]:
        b |= CB.branches(CB.schedule(n, n, CB.Config(sms=n_sms)), n, n)
    return b


ALL_BRANCHES = {"leaf_full", "leaf_slim", "ragged_last_block", "panel_fused", "panel_plain", "panel_feed", "panel_gemm",
                "panel_polled", "panel_event_ordered", "feed_old", "update_dmma_k128", "update_dmma",
                "update_dmma_int32_headroom", "update_int8", "update_int8_fed", "update_int8_k640_plus",
                "extra_rows", "extra_rows_sliced_by_panel"}


def test_case_table_reaches_every_branch(cuda_device):
    """Every branch of potrf_rec / potrf_block / trailing_update in the default configuration is taken by some case
    (the dynamic slicing by the update itself is the GPK_TC_STATIC=0 path: test_engine_configuration_inside_bars)."""
    got = table_branches(sms())
    assert got == ALL_BRANCHES, (ALL_BRANCHES - got, got - ALL_BRANCHES)


@pytest.mark.parametrize("n", SIZES)
def test_random_spd_inside_bars(cuda_device, n):
    rng = np.random.default_rng(n)
    run_and_check(CB.random_spd(n, rng), None, n, "spd")


@pytest.mark.parametrize("n,p", EXTRA)
def test_extra_rows_inside_bars(cuda_device, n, p):
    rng = np.random.default_rng(7 * n + p)
    A = CB.random_spd(n, rng)
    Y = rng.standard_normal((p, n)) * np.exp2(rng.integers(-8, 8, (p, 1)))
    run_and_check(A, Y, n, "spd_extra")


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("n", FAMILY_SIZES)
def test_matrix_families_inside_bars(cuda_device, family, n):
    rng = np.random.default_rng(zlib.crc32(f"{family}/{n}".encode()))
    A = family_matrix(family, n, rng)
    Y = rng.standard_normal((3, n)) @ np.linalg.cholesky(A).T if n == 1000 else None     # X = Y L^-T of order one
    run_and_check(A, Y, n, family)


def test_block_cond_at_the_edge_of_lapack(cuda_device):
    """Diagonal blocks of condition 1e4 at n = 300 (cond(A) ~ 4e10).  From n = 1000 at 1e4, and at 1e6 for every size
    of the table, L L^T has cond ~ 1e16 and LAPACK's own factorisation fails: no bar exists to check there."""
    rng = np.random.default_rng(300)
    L = DB.factor_with_block_cond(300, rng, 1e4)
    A = L @ L.T
    assert np.isfinite(np.linalg.cholesky(A)).all()
    run_and_check(A, None, 300, "block_cond")


# ---- integer-exact factors --------------------------------------------------------------------------------------------------
def integer_factor_device(n, seed, p_max=3):
    """chol_bounds.integer_factor built on the device: L0 and its lower A = L0 L0^T (exact integer sums)."""
    torch = _t()
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = torch.randint(-1, 2, (n, n), generator=g, device="cuda", dtype=torch.float64).tril_(-1)
    for o in range(0, n, DB.NB):
        L[o:o + DB.NB, o:o + DB.NB] = 0.0
    d = torch.randint(0, p_max + 1, (n,), generator=g, device="cuda").to(torch.float64)
    L.diagonal().copy_(torch.exp2(d))
    return L


def check_integer(n, p, scale, seed):
    torch = _t()
    L0 = integer_factor_device(n, seed)
    X0 = torch.randint(-3, 4, (p, n), device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 1)
                       ).to(torch.float64) if p else None
    big = n > 20000
    ld = n if big else n + PW.LDPAD
    guard = 0 if big else PW.GUARD
    if big:                     # A built in place (only its lower triangle is read): L0 and A are the whole footprint
        dP = torch.empty((n, n), dtype=torch.float64, device="cuda")
        torch.matmul(L0, L0.T, out=dP)
    else:
        dP = torch.full((n + p + guard, ld), float("nan"), dtype=torch.float64, device="cuda")
        dP[:n, :n] = torch.where(torch.ones(n, n, dtype=torch.bool, device="cuda").tril_(), L0 @ L0.T, dP[:n, :n])
    if p:
        dP[n:n + p, :n] = X0 @ L0.T
    if scale:
        dP.mul_(2.0 ** scale)
    before = None if big else dP.clone()
    info, ws = PW.run_parent(dP, n, n + p)
    del ws
    assert info == 0
    s = 2.0 ** (scale // 2)
    worst = 0.0
    for o in range(0, n, 4096):                         # in row chunks: max |L - L0| per row over the row's maximum
        got = torch.tril(dP[o:min(o + 4096, n), :n], diagonal=o)
        ref = torch.tril(L0[o:o + 4096], diagonal=o) * s
        err = (got - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)
        worst = max(worst, float(err.max()))
    if p:
        err = (dP[n:n + p, :n] - X0 * s).abs().amax(dim=1) / (X0 * s).abs().amax(dim=1)
        worst = max(worst, float(err.nan_to_num(0.0).max()))
    record("integer_exact_rel", worst)
    assert worst <= 4 * 2.0 ** -52, (n, p, scale, worst)
    if before is not None:
        check_guards(dP.cpu().numpy(), before.cpu().numpy(), n, n + p)
        dP2 = before.clone()
        PW.run_parent(dP2, n, n + p)
        assert torch.equal(dP.view(torch.int64), dP2.view(torch.int64))
    return worst


@pytest.mark.parametrize("n,p,scale", INTEGER)
def test_integer_exact_factor(cuda_device, n, p, scale):
    """L0 with a power-of-two diagonal, diagonal 128 x 128 blocks and small integers elsewhere: every block inverse, panel
    product, DMMA and digit product is exact, so L comes back as L0 (scale = -1000: A near the bottom of the normal range,
    L = 2^-500 L0; scale = -1060: A and every pivot subnormal, L = 2^-530 L0 normal)."""
    check_integer(n, p, scale, n + p)


def test_integer_exact_event_ordered_panels(cuda_device):
    for n in event_ordered_sizes(sms()):
        assert "panel_event_ordered" in CB.branches(CB.schedule(n, n, CB.Config(sms=sms())), n, n)
        check_integer(n, 0, 0, n)


def test_integer_exact_int32_headroom_fallback(cuda_device):
    """n = 37504: the top-level update has K = 18816 columns, 128^2 K S >= 2^31 at S = 7, so it runs on DMMA."""
    n = 37504
    assert "update_dmma_int32_headroom" in CB.branches(CB.schedule(n, n), n, n)
    free, _ = _t().cuda.mem_get_info()
    if free < 36e9:             # L0 and A (11.25 GB each), the digit planes (~5 GB), row chunks of the comparison
        pytest.skip(f"needs 36 GB of free device memory, {free / 1e9:.0f} GB free")
    check_integer(n, 0, 0, 5)


# ---- subnormal pivots --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 33, 128, 129, 300])
def test_subnormal_pivots_factor(cuda_device, n):
    """A PD matrix scaled by 2^-1060 has subnormal pivots (the rsqrt seed flushes them to zero): the factor is finite, info
    is 0 and every element is inside its bar, as LAPACK factors it."""
    rng = np.random.default_rng(n)
    A = np.ldexp(CB.random_spd(n, rng), -1060)
    assert np.isfinite(np.linalg.cholesky(A)).all()
    F = run_and_check(A, None, n, "scale_m1060")
    assert np.isfinite(F).all()


def test_subnormal_pivots_among_normal_ones(cuda_device):
    """D A D with D = 2^-530 on a few rows only: their pivots are subnormal inside blocks whose other pivots are normal."""
    n = 300
    rng = np.random.default_rng(5)
    d = np.ones(n)
    d[[0, 40, 41, 127, 200, 299]] = 2.0 ** -530
    A = CB.random_spd(n, rng) * d[:, None] * d[None, :]
    assert np.isfinite(np.linalg.cholesky(A)).all()
    F = run_and_check(A, None, n, "subnormal_pivot")
    assert np.isfinite(F).all()


# ---- info ------------------------------------------------------------------------------------------------------------------
INFO_N = 2049
INFO_J = [0, 31, 32, 127, 128, 260, 1030, 1925, 2048]


def test_info_positions_cover_the_update_kinds():
    """The pivots of INFO_J sit in: the first leaf, after a fused panel, after a fed int8 update, after a K >= 1024 update,
    after a DMMA K = 128 update, and in the ragged last block."""
    L = CB.schedule(INFO_N, INFO_N)
    prev = {}
    last = None
    for x in L:
        if x["kind"] == "leaf":
            prev[x["c0"]] = last
        else:
            last = x
    def before(j):
        c0 = max(c for c in prev if c <= j)
        return c0, prev[c0]
    assert before(128)[1]["type"] == "fused"
    assert before(260)[1]["engine"] == "int8" and before(260)[1]["row_skip"]
    assert before(1030)[1]["K"] >= 1024
    assert before(1925)[1]["engine"] == "dmma" and before(1925)[1]["K"] == 128
    assert before(2048)[0] == 2048


@pytest.mark.parametrize("j", INFO_J + ["nan"])
def test_info_names_the_first_failing_pivot(cuda_device, j):
    torch = _t()
    n = INFO_N
    L0 = integer_factor_device(n, 99)
    A = L0 @ L0.T
    jj = 500 if j == "nan" else j
    if j == "nan":
        A[jj, jj] = float("nan")
    else:
        A[jj, jj] -= L0[jj, jj] ** 2              # A - L0 L0^T = -L0_jj^2 e_j e_j^T: pivot j is exactly 0
    dP = torch.full((n + PW.GUARD, n + PW.LDPAD), float("nan"), dtype=torch.float64, device="cuda")
    dP[:n, :n] = torch.where(torch.ones(n, n, dtype=torch.bool, device="cuda").tril_(), A, dP[:n, :n])
    info, _ = PW.run_parent(dP, n, n)
    assert info == jj + 1
    assert torch.equal(dP[:jj, :jj].tril(), L0[:jj, :jj])


# ---- fp32 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [512, 1000, 2049])
def test_fp32_detour_is_the_rounded_fp64_factor(cuda_device, n):
    """n >= 512, square: the fp32 factor is float(L64), L64 the fp64 factor (S = 7) of the widened matrix; the fp32 block
    inverses recomputed from it are inside trsm_check's bars."""
    torch = _t()
    rng = np.random.default_rng(n)
    A32 = CB.random_spd(n, rng).astype(np.float32)
    F32, out, before, info, _ = PW.factor(A32.astype(np.float64), n, n, np.float32)
    assert info == 0
    check_guards(out, before, n, n)
    F64, _, _, info64, S = PW.factor(A32.astype(np.float64), n, n)
    assert info64 == 0 and S == 7
    assert np.array_equal(F32.astype(np.float32), F64.astype(np.float32))
    P = PW.parent_of(A32.astype(np.float64), n, n, np.float32)
    dP = torch.from_numpy(P).cuda()
    _, ws = PW.run_parent(dP, n, n, np.float32)
    nb = -(-n // DB.NB)
    raw = ws[: nb * DB.NB * DB.NB * 4].cpu().numpy().view(np.float32).astype(np.float64).reshape(nb, DB.NB, DB.NB)
    Xb = [raw[b, : min(DB.NB, n - b * DB.NB), : min(DB.NB, n - b * DB.NB)] for b in range(nb)]
    kap, eta = DB.block_stats(F32, Xb, 0)
    bound = 2 * DB.gamma(DB.NB, CB.U32) * kap
    record("fp32_dinv_eta", float((eta / bound).max()))
    assert np.all(eta <= bound), (eta, bound)


@pytest.mark.parametrize("n,p", [(1, 0), (100, 0), (300, 0), (300, 3), (600, 5)])
def test_fp32_native_inside_bars(cuda_device, n, p):
    rng = np.random.default_rng(n + p)
    A = CB.random_spd(n, rng)
    Y = rng.standard_normal((p, n)) if p else None
    run_and_check(A, Y, n, "fp32", dtype=np.float32)


# ---- batched ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,batch", [(1, 1000), (33, 1000), (128, 1000), (129, 3), (300, 3)])
def test_batched_info_words_are_per_matrix(cuda_device, n, batch):
    """gpk_potrf_batched: matrices at a stride beyond n * lda; every third matrix is non-PD at its own pivot (integer
    factors, pivot exactly 0), each info word names its own; the PD ones are the integer factor or inside the bars."""
    torch = _t()
    lda = n + 3
    stride = n * lda + 7
    rng = np.random.default_rng(n)
    buf = np.full(stride * batch + lda, np.nan)
    want_info, mats = [], []
    for b in range(batch):
        L0 = CB.integer_factor(n, rng)
        A = L0 @ L0.T
        j = int(rng.integers(0, n)) if b % 3 == 1 else -1
        if j >= 0:
            A[j, j] -= L0[j, j] ** 2
        want_info.append(j + 1)
        view = buf[b * stride: b * stride + n * lda].reshape(n, lda)
        view[:, :n] = np.where(np.tri(n, dtype=bool), A, np.nan)
        mats.append(L0)
    d = torch.from_numpy(buf).cuda()
    ws = torch.empty(int(PW.lib().gpk_potrf_batched_ws(n, batch, PW.F64)), dtype=torch.uint8, device="cuda")
    info = torch.full((batch,), -7, dtype=torch.int32, device="cuda")
    rc = PW.lib().gpk_potrf_batched(PW.ptr(d), n, lda, stride, batch, PW.F64, PW.ptr(info), PW.ptr(ws), None)
    assert rc == 0, PW.lib().gpk_last_error().decode()
    torch.cuda.synchronize()
    assert info.cpu().numpy().tolist() == want_info
    out = d.cpu().numpy()
    gaps = np.ones(out.shape, dtype=bool)           # everything but the matrices' lower triangles: bit-unchanged
    for b in range(batch):
        view = out[b * stride: b * stride + n * lda].reshape(n, lda)
        g = gaps[b * stride: b * stride + n * lda].reshape(n, lda)
        g[:, :n] &= ~np.tri(n, dtype=bool)
        if want_info[b] == 0:
            assert np.array_equal(np.tril(view[:, :n]), mats[b]), b
        else:
            j = want_info[b] - 1
            assert np.array_equal(np.tril(view[:j, :j]), mats[b][:j, :j]), b
    assert np.array_equal(out[gaps].view(np.int64), buf[gaps].view(np.int64))


# ---- engine configurations ----------------------------------------------------------------------------------------------------
CONFIGS = {
    "slices6": ({"GPK_TC_SLICES": "6"}, dict(S=6)),
    "slices8": ({"GPK_TC_SLICES": "8"}, dict(S=8)),
    "dmma": ({"GPK_FP64_ENGINE": "dmma"}, dict(tc=False)),
    "dynamic_scales": ({"GPK_TC_STATIC": "0"}, dict(static=False)),
    "no_flag_hops": ({"GPK_FLAG_HOPS": "0"}, dict(flaghop=False)),
}


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("potrf_configs"))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_engine_configuration_inside_bars(cuda_device, tmp, name):
    envs, kw = CONFIGS[name]
    env = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    env.update(envs)
    out = os.path.join(tmp, f"{name}.npz")
    r = subprocess.run([sys.executable, "-m", "tests._potrf_worker", out], cwd=ROOT, env=env, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    res = np.load(out)
    reached = set()
    for n, p, fam, seed in PW.CONFIG_CASES:
        A, Y = PW.config_case(n, p, fam, seed)
        key = f"{n}_{p}_{fam}"
        assert int(res[f"info_{key}"]) == 0
        S = int(res[f"S_{key}"])
        assert S == kw.get("S", 0 if kw.get("tc") is False else 7), (name, S)
        cfg = CB.Config(sms=sms(), **kw)
        reached |= CB.branches(CB.schedule(n, n + p, cfg), n, n + p)
        check_factor(PW.target(A, Y), res[f"F_{key}"], n, n + p, np.diag(A), cfg, f"config_{name}", S=S or 7)
    if name == "dynamic_scales":
        assert "extra_rows_sliced_by_update" in reached
    if name == "dmma":
        assert "update_dmma" in reached and "update_int8" not in reached
    if name == "no_flag_hops":
        assert "panel_polled" not in reached


def test_report_worst_ratios(cuda_device):
    """Prints the worst ratio per bar and matrix family over the tests that ran before it (run the file as a whole)."""
    torch = _t()
    p = torch.cuda.get_device_properties(0)
    print(f"\nworst ratios on {p.name} ({p.multi_processor_count} SMs):")
    for k in sorted(WORST):
        print(f"  {k:32s} {WORST[k]:.3g}")
