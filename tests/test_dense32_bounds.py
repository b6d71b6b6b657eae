"""CPU self-tests of tests/dense32_bounds.py: the model of the 3xTF32 kernel inside every bar with margin, each
modelled mutant (a lost correction MMA, hi*hi only, one promotion per K range) outside the statistical bars by at least
10x at K = 2048 and at the SGPR depth K = 1e5 (a strip of entries), and the dispatch mirrors against hand-written
tables."""
import numpy as np
import pytest

from tests import dense32_bounds as D

MUTANTS = [("2x", D.TF_KP), ("1x", D.TF_KP), ("3x", None)]


def _case(K, m, n, seed):
    rng = np.random.default_rng(seed)
    a = rng.standard_normal((m, K)).astype(np.float32)
    b = rng.standard_normal((n, K)).astype(np.float32)
    sq = rng.standard_normal((16, K)).astype(np.float32)
    return a, b, sq


def _stats(a, b, sq, mode, run):
    c = D.emulate_tf32(a[:, None, :], b[None, :, :], mode, run)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ref, mag = a64 @ b64.T, np.abs(a64) @ np.abs(b64).T
    dg = D.emulate_tf32(sq, sq, mode, run)
    dref = (sq.astype(np.float64) ** 2).sum(axis=1)
    K = a.shape[1]
    worst = float(np.max(np.abs(c - ref) / (D.g_tf32(K) * mag)))
    return D.rms_rel(c - ref, mag) / D.rms_bar(K), abs(D.signed_bias(dg, dref)) / D.BIAS_BAR, worst


@pytest.mark.parametrize("K,m,n", [(2048, 48, 40), (100000, 6, 8)])
def test_model_inside_bars_and_mutants_outside(K, m, n):
    a, b, sq = _case(K, m, n, K)
    rms, bias, worst = _stats(a, b, sq, "3x", D.TF_KP)
    assert worst <= 0.1, worst                    # the worst-case bar with a decade of margin
    assert rms <= 0.1 and bias <= 0.5, (rms, bias)
    for mode, run in MUTANTS:
        r, bi, _ = _stats(a, b, sq, mode, run)
        if run is None:
            assert bi >= 10, (mode, run, r, bi)   # truncation bias: only a positive sum shows it at K = 2048
        else:
            assert r >= 10, (mode, run, r, bi)


def test_split_error_is_within_2_to_the_minus_20():
    rng = np.random.default_rng(4)
    x = (rng.standard_normal(200000) * np.exp2(rng.integers(-30, 30, 200000))).astype(np.float32)
    y = rng.standard_normal(200000).astype(np.float32)
    xh, xl = (v.astype(np.float64) for v in D.split(x))
    yh, yl = (v.astype(np.float64) for v in D.split(y))
    three = xl * yh + xh * yl + xh * yh
    exact = x.astype(np.float64) * y.astype(np.float64)
    assert np.all(np.abs(three - exact) <= D.U_SPLIT * np.abs(exact))


def test_one_mma_step_stays_within_u_mma():
    rng = np.random.default_rng(5)
    d = (rng.standard_normal(20000) * 30).astype(np.float32).astype(np.float64)
    p = np.stack([D.rna_tf32(rng.standard_normal(20000).astype(np.float32)).astype(np.float64)
                  * D.rna_tf32(rng.standard_normal(20000).astype(np.float32)).astype(np.float64) for _ in range(8)], 1)
    got = D.mma(d, p)
    assert np.all(got.astype(np.float32) == got)                         # an fp32 value
    exact = d + p.sum(axis=1)
    assert np.all(np.abs(got - exact) <= D.U_MMA * (np.abs(d) + np.abs(p).sum(axis=1)))
    pos = np.abs(p)
    assert np.all(D.mma(np.abs(d), pos) <= np.abs(d) + pos.sum(axis=1))   # positive addends: truncation only loses


@pytest.mark.parametrize("m", [16, 100, 256])
def test_colsumsq_model_inside_bar(m):
    rng = np.random.default_rng(m)
    K, n = 256, 40
    a = rng.standard_normal((m, K)).astype(np.float32)
    b = rng.standard_normal((n, K)).astype(np.float32)
    Y = D.emulate_tf32(a[:, None, :], b[None, :, :])
    v0 = rng.uniform(0.5, 2.0, n).astype(np.float32)
    got = D.emulate_colsumsq(Y, v0)
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    y, s = a64 @ b64.T, np.abs(a64) @ np.abs(b64).T
    ref = v0 + (y ** 2).sum(axis=0)
    bar = D.colsumsq_bar(y, s, D.g_tf32(K), m, v0)
    assert np.all(np.abs(got - ref) <= 0.5 * bar)
    # the batch written into the wrong output (another column's sums) is far outside
    assert np.max(np.abs(got[::-1] - ref) / bar) > 1e3


# (m, n, k, flags, alias, tb, engine) -> the kernel gemm.cu::gemm_t runs for fp32, worked out from gemm_t and
# gemm_tf32_eligible
KERNEL_TABLE = [
    ((1024, 1, 100000, 0, None, 0, "tf32"), "skinny"),          # A'.Yc of SGPR
    ((4096, 8, 2048, 0, None, 0, "tf32"), "skinny"),            # A^T q_mu of SVGP
    ((4096, 16, 2048, 0, None, 0, "tf32"), "skinny"),
    ((4096, 17, 2048, 0, None, 0, "tf32"), "simt"),             # n > 16, and n < 64: no tf32
    ((4096, 8, 2048, 0, None, 1, "tf32"), "simt"),              # transb: no skinny kernel
    ((300, 16, 2048, D.GEMM_A_LOWER, None, 0, "tf32"), "simt"),  # flags: no skinny kernel
    ((1024, 1024, 100000, D.GEMM_LOWER_ONLY, None, 1, "tf32"), "tf32"),
    ((1024, 1024, 100000, D.GEMM_LOWER_ONLY, None, 1, "simt"), "simt"),
    ((1000, 1000, 200, 0, None, 0, "tf32"), "tf32"),             # exactly 2e8
    ((1000, 1000, 199, 0, None, 0, "tf32"), "simt"),
    ((63, 100000, 100000, 0, None, 0, "tf32"), "simt"),          # m < 64
    ((4096, 4096, 63, 0, None, 0, "tf32"), "simt"),              # k < 64
    ((128, 12208, 128, 0, "B", 0, "tf32"), "tf32"),
]


@pytest.mark.parametrize("args,want", KERNEL_TABLE)
def test_gemm_kernel_mirror_matches_table(args, want):
    m, n, k, flags, alias, tb, engine = args
    assert D.gemm_kernel(m, n, k, flags, alias, tb, engine) == want


# (m, n, k, flags, batch, cluster) -> (cl, nsplit) of gemm_tf32 on 132 SMs, worked out by hand
LAUNCH_TABLE = [
    ((1024, 1024, 100000, D.GEMM_LOWER_ONLY, 1, 2), (2, 4)),     # 20 units of 2 tiles: 40, 80, 160 CTAs
    ((1024, 1024, 100000, D.GEMM_LOWER_ONLY, 1, 1), (1, 4)),     # 36 tiles: 36, 72, 144
    ((1024, 1024, 20000, 0, 1, 2), (2, 4)),                      # 32 units: 64, 128, 256
    ((512, 512, 8192, 0, 1, 2), (2, 8)),                         # 8 units; KB = 512: 16, 32, 64, 128, 256
    ((128, 5000, 128, 0, 1, 2), (1, 1)),                         # one row tile; KB = 8
    ((640, 640, 640, 0, 1, 2), (2, 1)),                          # KB = 40 < 128
    ((2048, 4096, 2048, D.GEMM_COLSUMSQ | D.GEMM_A_LOWER, 8, 2), (2, 1)),
    ((256, 1000, 256, D.GEMM_COLSUMSQ, 2, 2), (2, 1)),
    ((300, 1000, 8192, 0, 1, 2), (2, 8)),                        # 3 row tiles: units (0, 1), (2, pad)
]


@pytest.mark.parametrize("args,want", LAUNCH_TABLE)
def test_tf32_launch_mirror_matches_table(args, want):
    m, n, k, flags, batch, cluster = args
    assert D.tf32_launch(m, n, k, flags, batch, cluster) == want


# (B, M, Pl, q_diag, batched_env, engine) -> fvar path of fused.cu::svgp_forward in fp32
SVGP_TABLE = [
    ((4096, 2048, 8, False, True, "tf32"), "batched"),           # C4
    ((4096, 2048, 8, False, False, "tf32"), "tf32"),             # GPK_SVGP_BATCHED=0
    ((4096, 2048, 1, False, True, "tf32"), "tf32"),              # one latent
    ((1000, 640, 3, False, True, "tf32"), "tf32"),               # M % 256 != 0
    ((1000, 512, 3, False, True, "tf32"), "batched"),            # 512 * 1000 * 512 = 2.6e8
    ((700, 512, 3, False, True, "tf32"), "simt"),                # 1.8e8 < 2e8
    ((4096, 2048, 8, True, True, "tf32"), "q_diag"),
    ((4096, 2048, 8, False, True, "simt"), "simt"),              # GPK_FP32_ENGINE=simt
]


@pytest.mark.parametrize("args,want", SVGP_TABLE)
def test_svgp_fvar_path_mirror_matches_table(args, want):
    B, M, Pl, q_diag, env, engine = args
    assert D.svgp_fvar_path(B, M, Pl, q_diag, np.float32, env, engine) == want
