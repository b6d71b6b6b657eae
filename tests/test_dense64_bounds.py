"""CPU self-tests of tests/dense64_bounds.py: the tile-selection mirror against a hand-written table, and fp64 NumPy
emulations of trsm_rec / trtri_rec / lauum_rec (same splits, inverse-based leaves) inside every bar, ill-conditioned
diagonal blocks included, before any of it is used on a device."""
import numpy as np
import pytest
import scipy.linalg as sla

from tests import dense64_bounds as DB

# (m, n, flags, alias, tb, k, dtype) -> what gemm.cu::gemm_t launches, worked out by hand from launch_dmma / launch_simt
TILE_TABLE = [
    ((1400, 1400, 0, None, 0, 16, np.float64), (128, 128)),        # 11 * 11 = 121 tiles of 128
    ((1270, 1270, 0, None, 0, 16, np.float64), (64, 128)),         # 10 * 10 = 100 tiles of 128; 20 * 10 of 64 x 128
    ((1000, 900, 0, None, 0, 16, np.float64), (64, 128)),          # 16 * 8 = 128 >= 100
    ((500, 300, 0, None, 0, 16, np.float64), (32, 128)),           # 8 * 3 = 24 < 100
    ((128, 6337, 0, None, 0, 16, np.float64), (128, 64)),          # m <= 128, 100 column tiles of 64
    ((128, 6336, 0, None, 0, 16, np.float64), (128, 32)),          # 99 column tiles of 64
    ((100, 15360, 0, None, 0, 16, np.float64), (128, 128)),        # 120 tiles of 128
    ((6337, 100, 0, None, 0, 16, np.float64), (64, 128)),          # n <= 128, 100 row tiles of 64
    ((6336, 100, 0, None, 0, 16, np.float64), (32, 128)),
    ((300, 16, 0, None, 0, 16, np.float64), "skinny"),
    ((300, 16, 0, None, 1, 16, np.float64), (32, 128)),            # transb: no skinny kernel
    ((300, 1, DB.GEMM_A_LOWER, None, 0, 16, np.float64), (32, 128)),  # flags: no skinny kernel
    ((300, 16, 0, "B", 0, 16, np.float64), (128, 32)),             # aliasing: no skinny kernel
    ((128, 300, 0, "B", 0, 16, np.float64), (128, 32)),
    ((128, 15500, 0, "B", 0, 16, np.float64), (128, 128)),         # the trsm leaf at nrhs = 15500
    ((128, 12000, 0, "B", 0, 16, np.float64), (128, 64)),
    ((300, 100, 0, "A", 0, 16, np.float64), (32, 128)),
    ((200, 128, 0, "A", 0, 16, np.float64), (32, 128)),            # alias A: the short-and-wide branch is skipped
    ((15400, 128, 0, "A", 0, 16, np.float64), (128, 128)),
    ((300, 300, DB.GEMM_COLSUMSQ, None, 0, 16, np.float64), (128, 128)),
    ((300, 300, DB.GEMM_LOWER_ONLY, None, 0, 16, np.float64), (32, 128)),
    ((128, 12208, 0, "B", 0, 128, np.float32), "tf32"),            # 128 * 12208 * 128 >= 2e8
    ((128, 12207, 0, "B", 0, 128, np.float32), (128, 64)),
    ((1000, 900, 0, None, 0, 63, np.float32), (64, 128)),          # k < 64: no tf32
    ((0, 5, 0, None, 0, 3, np.float64), None),
]


@pytest.mark.parametrize("args,want", TILE_TABLE)
def test_tile_mirror_matches_table(args, want):
    m, n, flags, alias, tb, k, dtype = args
    assert DB.dmma_tile(m, n, flags, alias, tb, k, dtype) == want


def test_lower_only_mask_skips_tiles_right_of_their_rows():
    mask = DB.tiles_written(300, 300, (32, 128), DB.GEMM_LOWER_ONLY)
    assert mask[:32, :128].all() and not mask[:32, 128:].any() and not mask[96:128, 128:].any()
    assert mask[128:160, :256].all() and not mask[128:160, 256:].any() and mask[256:, :].all()


def test_split_and_depth():
    assert [DB.split_point(n) for n in (129, 255, 256, 257, 383, 1000, 2500)] == [128, 128, 128, 128, 128, 512, 1280]
    assert [DB.depth(n) for n in (1, 128, 129, 384, 2048, 4099)] == [0, 0, 1, 2, 4, 6]
    # 383 = 128 + 255, 255 = 128 + 127: an odd second half
    assert DB.splits(383) == [(0, 128, 255), (128, 128, 127)]


def _factor(n, cond, seed):
    rng = np.random.default_rng(seed)
    return DB.factor_with_block_cond(n, rng, cond), rng


@pytest.mark.parametrize("n,cond", [(1, 1), (129, 1), (300, 1e3), (383, 1), (640, 1e6), (1000, 1e6)])
@pytest.mark.parametrize("trans", [0, 1])
def test_emulated_trsm_inside_bar(n, cond, trans):
    L, rng = _factor(n, cond, n)
    Xb = DB.leaf_inverses(L)
    B = rng.standard_normal((n, 17))
    X = DB.emu_trsm(trans, L, B, Xb)
    r, kap, _ = DB.trsm_check(L, B, X, Xb, trans, np.arange(17))
    assert r <= 1.0, r
    if cond > 1:
        assert kap > cond / 10  # the kappa term is exercised


@pytest.mark.parametrize("n,cond", [(129, 1), (257, 1), (383, 1), (1000, 1e6)])
def test_emulated_trtri_and_lauum_inside_bars(n, cond):
    L, rng = _factor(n, cond, n + 1)
    Xb = DB.leaf_inverses(L)
    X = DB.emu_trtri(L, Xb)
    assert DB.trtri_check(L, X, rng) <= 1.0
    np.testing.assert_allclose(np.tril(X), sla.solve_triangular(L, np.eye(n), lower=True),
                               rtol=0, atol=1e-6 * np.abs(X).max())
    C = DB.emu_lauum(X)
    rows, cols = DB.edge_indices(n, rng), DB.edge_indices(n, rng)
    assert DB.lauum_check(X, rows, cols)(C) <= 1.0


def test_emulated_chol_adjoint_inside_bar():
    n = 300
    L, rng = _factor(n, 1.0, 5)
    T = rng.standard_normal((n, n))
    Xb = DB.leaf_inverses(L)
    Phi = np.tril(T, -1) + 0.5 * np.diag(np.diag(T))
    Y = DB.emu_trsm(1, L, Phi, Xb)
    Z = DB.emu_trsm(1, L, Y.T.copy(), Xb)
    G = -0.5 * (Z + Z.T)
    kap, eta = DB.block_stats(L, Xb, 1)
    bar = DB.chol_adjoint_bar(L, T, kap.max(), eta.max())
    assert np.abs(G - DB.chol_adjoint_ref(L, T)).max() <= bar


def test_bars_catch_a_wrong_leaf_block():
    """The TRSM and trtri bars are not vacuous: using the neighbouring block's inverse in one leaf breaks both."""
    n = 383
    L, rng = _factor(n, 1.0, 9)
    Xb = DB.leaf_inverses(L)
    bad = list(Xb)
    bad[1] = Xb[0][: Xb[1].shape[0], : Xb[1].shape[0]]
    B = rng.standard_normal((n, 5))
    assert DB.trsm_check(L, B, DB.emu_trsm(1, L, B, bad), Xb, 1, np.arange(5))[0] > 1e3
    X = DB.emu_trtri(L, Xb)
    X[200, 31] += 1e-9 * abs(X[200, 31])
    assert DB.trtri_check(L, X, rng) > 1.0


def test_gemm_bar_holds_for_blas_and_catches_a_lost_chunk():
    rng = np.random.default_rng(3)
    m, n, k = 70, 90, 77
    A, B, C0 = rng.standard_normal((m, k)), rng.standard_normal((k, n)), rng.standard_normal((m, n))
    rows, cols = np.arange(m), np.arange(n)
    ref, bar = DB.gemm_ref(A, B, C0, -0.7, 1.0, 0, 0, rows, cols)
    got = -0.7 * (A @ B) + C0
    assert DB.ratio(np.abs(got - ref), bar) <= 1.0
    lost = -0.7 * (A[:, :64] @ B[:64]) + C0                         # last partial k-chunk (77 % 16 = 13) dropped
    assert DB.ratio(np.abs(lost - ref), bar) > 1e6
