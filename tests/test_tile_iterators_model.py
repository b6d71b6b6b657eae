"""Python mirrors of the persistent-kernel work iterators (TcTileIter in gemm_tc.cu, TfWork + tf_krange in
gemm_tf32.cu), checked exhaustively on the CPU: every needed output tile is produced by exactly one CTA, padding
tiles of a cluster unit are never stored, the CTAs of a cluster walk the same unit sequence (lock-step multicast), the
head tiles come first, and the k-ranges of the k-splits partition the needed K range."""
import itertools

import pytest

TC_BM, TC_BN = 128, 32
TF_BM, TF_BN, TF_KS, TF_SPP = 128, 128, 16, 4
TC_HEAD = 128 // TC_BN   # column tiles of the leading 128-column block


# ---- gemm_tc.cu::TcTileIter ------------------------------------------------------------------------------------
def tc_units(m, n, lower, cl, grid, block):
    ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
    rank, my, ncl = block % cl, block // cl, grid // cl
    head_w = cl if cl > TC_HEAD else TC_HEAD

    def ncols(t):
        return min((t + 1) * (TC_BM // TC_BN), ntn) if lower else ntn

    out = []
    pas, tm, tnb, idx = 0, 0, -cl, -1
    while True:
        tnb += cl
        while True:
            if pas == 0:
                lim = min(ncols(tm), head_w) if tm < ntm else 0
                if tm < ntm and tnb >= lim:
                    tm, tnb = tm + 1, 0
                    continue
                if tm >= ntm:
                    pas, tm, tnb = 1, 0, head_w
                    continue
            else:
                if tm < ntm and tnb >= ncols(tm):
                    tm, tnb = tm + 1, head_w
                    continue
                if tm >= ntm:
                    return out
            break
        idx += 1
        if idx % ncl == my:
            tn = tnb + rank
            out.append(dict(tm=tm, tnb=tnb, tn=tn, head=pas == 0, valid=tn < ncols(tm), idx=idx))


@pytest.mark.parametrize("cl", [1, 2, 4])
@pytest.mark.parametrize("lower", [0, 1])
def test_tc_tile_iterator_covers_every_tile_once(cl, lower):
    for m, n in [(128, 32), (128, 64), (128, 128), (256, 128), (384, 200), (1000, 1000), (1024, 320), (4096, 4096), (640, 64)]:
        if lower and n > m:
            continue
        for grid in {cl, 2 * cl, 6 * cl, (131 // cl) * cl}:
            ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
            need = {(tm, tn) for tm in range(ntm) for tn in range(min((tm + 1) * (TC_BM // TC_BN), ntn) if lower else ntn)}
            seen = []
            per_cta = [tc_units(m, n, lower, cl, grid, b) for b in range(grid)]
            for units in per_cta:
                seen += [(u["tm"], u["tn"]) for u in units if u["valid"]]
                heads = [u["head"] for u in units]
                assert heads == sorted(heads, reverse=True)            # head units first (look-ahead)
            assert sorted(seen) == sorted(need), (m, n, lower, cl, grid)
            for c in range(grid // cl):                                # lock-step inside a cluster
                seqs = [[(u["tm"], u["tnb"]) for u in per_cta[c * cl + r]] for r in range(cl)]
                assert all(s == seqs[0] for s in seqs)
            # head tiles (the first 128 columns) are all produced in pass 0
            for units in per_cta:
                for u in units:
                    if u["valid"] and u["tn"] < TC_HEAD:
                        assert u["head"]


# ---- gemm_tf32.cu::TfWork / tf_krange ----------------------------------------------------------------------------
def tf_units(m, n, nsplit, lower, cl, grid, block):
    ntm, ntn = -(-m // TF_BM), -(-n // TF_BN)
    rank, my, ncl = block % cl, block // cl, grid // cl

    def tile_skip(t, tn):
        return bool(lower) and tn * TF_BN > t * TF_BM + TF_BM - 1

    out = []
    idx, tm0, tn, ks = -1, 0, 0, -1
    while True:
        ks += 1
        if ks >= nsplit:
            ks, tm0 = 0, tm0 + cl
        while tn < ntn and (tm0 >= ntm or tile_skip(tm0 + cl - 1, tn)):
            if tm0 >= ntm:
                tm0, tn = 0, tn + 1
            else:
                tm0 += cl
        if tn >= ntn:
            return out
        idx += 1
        if idx % ncl == my:
            tm = tm0 + rank
            out.append(dict(tm0=tm0, tm=tm, tn=tn, ks=ks, valid=tm < ntm and not tile_skip(tm, tn)))


def tf_krange(tri, tm_first, tm_last, KB, nsplit, ks):
    lo, hi = 0, KB
    if tri == 2:
        lo = (tm_first * TF_BM // TF_KS) // TF_SPP * TF_SPP
    if tri == 1:
        hi = min(hi, ((tm_last + 1) * TF_BM + TF_KS - 1) // TF_KS)
    lo = min(lo, hi)
    per = (-(-(hi - lo) // nsplit) + TF_SPP - 1) // TF_SPP * TF_SPP
    kb0 = lo + ks * per
    kb1 = min(kb0 + per, hi)
    return min(kb0, kb1), kb1


@pytest.mark.parametrize("cl", [1, 2])
@pytest.mark.parametrize("lower", [0, 1])
def test_tf32_work_iterator_covers_every_tile_and_split_once(cl, lower):
    for (m, n), nsplit in itertools.product([(128, 256), (300, 1000), (1024, 1024), (1500, 1500), (1100, 2000), (2048, 4096)],
                                            [1, 2, 8]):
        ntm, ntn = -(-m // TF_BM), -(-n // TF_BN)
        if cl == 2 and ntm < 2:
            continue
        for grid in {cl, 4 * cl, (132 // cl) * cl}:
            need = {(tm, tn, ks) for tm in range(ntm) for tn in range(ntn) for ks in range(nsplit)
                    if not (lower and tn * TF_BN > tm * TF_BM + TF_BM - 1)}
            per_cta = [tf_units(m, n, nsplit, lower, cl, grid, b) for b in range(grid)]
            seen = [(u["tm"], u["tn"], u["ks"]) for units in per_cta for u in units if u["valid"]]
            assert sorted(seen) == sorted(need), (m, n, nsplit, lower, cl, grid)
            for c in range(grid // cl):
                seqs = [[(u["tm0"], u["tn"], u["ks"]) for u in per_cta[c * cl + r]] for r in range(cl)]
                assert all(s == seqs[0] for s in seqs)


@pytest.mark.parametrize("tri", [0, 1, 2])
def test_tf32_krange_splits_partition_the_needed_range(tri):
    for k, nsplit, cl in itertools.product([64, 900, 2048, 100000], [1, 2, 4, 64], [1, 2]):
        KB = -(-k // TF_KS)
        for tm_first in (0, 1, 2, 6, 15):
            tm_last = tm_first + cl - 1
            stages = []
            for ks in range(nsplit):
                kb0, kb1 = tf_krange(tri, tm_first, tm_last, KB, nsplit, ks)
                assert kb0 <= kb1 <= KB
                if kb0 < kb1:   # non-empty splits start on a whole promotion run
                    assert (kb0 - tf_krange(tri, tm_first, tm_last, KB, nsplit, 0)[0]) % TF_SPP == 0
                stages += list(range(kb0, kb1))
            assert stages == sorted(set(stages))                      # disjoint, ordered
            # every stage that can hold a non-zero of a triangular operand row tile is covered
            for tm in range(tm_first, tm_last + 1):
                for kb in range(KB):
                    k_lo, k_hi = kb * TF_KS, kb * TF_KS + TF_KS - 1
                    r_lo, r_hi = tm * TF_BM, tm * TF_BM + TF_BM - 1
                    nonzero = True if tri == 0 else (k_lo <= r_hi if tri == 1 else k_hi >= r_lo)
                    if nonzero:
                        assert kb in stages, (tri, k, nsplit, cl, tm, kb)


# ---- look-ahead progress counters (common.cuh::diag_units_total / diag_units_tile) ---------------------------------
def diag_units_total(m, n):
    a, b = min(m, 128), min(n, 128)
    return -(-a // 32) * -(-b // 32)


def diag_units_tile(m0, n0, bm, bn, m, n):
    if m0 >= 128 or n0 >= 128:
        return 0
    a, b = min(m, 128) - m0, min(n, 128) - n0
    ra, rb = min(a, bm), min(b, bn)
    if ra <= 0 or rb <= 0:
        return 0
    return -(-ra // 32) * -(-rb // 32)


@pytest.mark.parametrize("bm,bn", [(128, 128), (64, 128), (32, 128), (128, 64), (128, 32)])
def test_head_tiles_publish_exactly_the_units_the_next_leaf_waits_for(bm, bn):
    """Every GEMM tile shape (gemm.cu DMMA / SIMT shapes; 128x32 is also the wgmma int8 tile) must publish, over the
    tiles it actually computes under GPK_GEMM_LOWER_ONLY, exactly diag_units_total(m, n) units: fewer and the waiting
    leaf traps, more and it starts before its inputs are complete."""
    for m, n in [(128, 128), (200, 128), (1000, 128), (4096, 4096), (129, 1), (640, 100), (96, 96), (7000, 4096), (130, 130)]:
        published = 0
        for m0 in range(0, m, bm):
            for n0 in range(0, n, bn):
                if n0 > m0 + bm - 1:        # lower-only: tile strictly above the diagonal is skipped
                    continue
                if n0 < 128:                # kernels publish only for tiles in the first 128 columns
                    published += diag_units_tile(m0, n0, bm, bn, m, n)
        assert published == diag_units_total(m, n), (bm, bn, m, n)


# ---- pre-tiled operand layouts (canonical no-swizzle K-major wgmma operand images) ----------------------------------------------
def test_pretiled_plane_offsets_are_bijective_and_core_matrix_shaped():
    """tc_tile_off (gemm_tc.cu: int8, 128 rows x 32 B) and tf_tile_off (gemm_tf32.cu: tf32, RB rows x 16 k x 4 B):
    every (row, k) maps to a distinct offset inside the plane, the 8-row x 16-byte core matrices are contiguous
    128-byte blocks, and a 256-row B plane is the concatenation of two 128-row planes (what lets 2-CTA clusters and
    the A/B tile sizes share one layout)."""
    def tc_off(r, k):
        return (r >> 3) * 256 + (k >> 4) * 128 + (r & 7) * 16 + (k & 15)

    offs = {tc_off(r, k) for r in range(128) for k in range(32)}
    assert offs == set(range(128 * 32))
    for rg in range(16):
        for kc in range(2):
            blk = {tc_off(rg * 8 + r, kc * 16 + b) for r in range(8) for b in range(16)}
            assert blk == set(range(min(blk), min(blk) + 128))

    def tf_off(r, k):
        return (r >> 3) * 512 + (k >> 2) * 128 + (r & 7) * 16 + (k & 3) * 4

    for RB in (128, 256):
        offs = {tf_off(r, k) + b for r in range(RB) for k in range(16) for b in range(4)}
        assert offs == set(range(RB * 64))
    assert all(tf_off(128 + r, k) == 128 * 64 + tf_off(r, k) for r in range(128) for k in range(16))


def test_kbuild_lower_tile_decode_fp32_estimate():
    """kbuild_fast_kernel decodes t = by (by + 1) / 2 + bx from an fp32 square-root estimate plus fix-up loops; the
    estimate must stay within a step or two of the truth up to the 2^31 tile limit the host enforces."""
    import numpy as np

    rng = np.random.default_rng(0)
    ts = np.concatenate([np.arange(0, 5000), rng.integers(0, 2 ** 31 - 1, 20000), [2 ** 31 - 2]])
    for t in ts:
        t = int(t)
        by = int((np.sqrt(np.float32(8.0) * np.float32(t) + np.float32(1.0), dtype=np.float32) - np.float32(1.0)) * np.float32(0.5))
        steps = 0
        while by * (by + 1) // 2 > t:
            by -= 1
            steps += 1
        while (by + 1) * (by + 2) // 2 <= t:
            by += 1
            steps += 1
        bx = t - by * (by + 1) // 2
        assert 0 <= bx <= by and steps <= 3, (t, by, bx, steps)
