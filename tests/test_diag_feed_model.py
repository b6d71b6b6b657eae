"""Python mirror of which diagonal blocks the Cholesky feeds from the panel in front of them (potrf.cu: potrf_rec tags the
last block before an int8 trailing update with its k-range, potrf_block applies the diagonal feed when that K is at most
GPK_DIAG_FEED_MAX_K).  Checked on the CPU for C2 (N = 8192 with its Y row): the fed blocks are those behind the K = 256
updates (block index = 2 mod 4) and the K = 512 updates (= 4 mod 8)."""
import pytest

NB = 128


def split_point(n):
    return ((n // NB + 1) // 2) * NB


def preceding_update_k(n, rows, tc_min_k=256):
    """{block index: K of the trailing update directly in front of it, 128 for the fused K = 128 update}, and the set of
    blocks whose preceding update runs on the int8 tensor cores (the others take the fused panel or DMMA)."""
    before, int8 = {}, set()

    def rec(n_, col0):
        if n_ <= NB:
            return
        n1 = split_point(n_)
        if n_ <= 2 * NB:  # two diagonal blocks: the K = 128 update between them is fused into the first panel
            before[(col0 + n1) // NB] = n1
            rec(n_ - n1, col0 + n1)
            return
        rec(n1, col0)
        before[(col0 + n1) // NB] = n1
        if n1 >= tc_min_k and n1 % 32 == 0 and n_ - n1 <= rows - col0 - n1 and n1 * 7 * 16384 < 2 ** 31:
            int8.add((col0 + n1) // NB)
        rec(n_ - n1, col0 + n1)

    rec(n, 0)
    return before, int8


def fed_blocks(n, rows, max_k=512):
    """Blocks whose diagonal block the panel in front of them updates and publishes."""
    before, int8 = preceding_update_k(n, rows)
    return {b for b in int8 if NB < before[b] <= max_k and rows - (b - 1) * NB - NB >= NB}


def test_c2_fed_blocks():
    fed = fed_blocks(8192, 8193)
    assert fed == {b for b in range(1, 64) if b % 4 == 2 or b % 8 == 4}
    assert len(fed) == 24


@pytest.mark.parametrize("max_k,want", [(0, set()), (256, {2, 6}), (512, {2, 4, 6})])
def test_c2_fed_blocks_per_switch(max_k, want):
    assert {b % 8 for b in fed_blocks(8192, 8193, max_k)} == want


def test_c2_update_depth_per_block():
    """At N = 8192 the update in front of block b has K = 128 times the lowest set bit of b."""
    before, int8 = preceding_update_k(8192, 8193)
    assert before == {b: NB * (b & -b) for b in range(1, 64)}
    assert int8 == {b for b in range(1, 64) if b % 2 == 0}


@pytest.mark.parametrize("n,rows", [(1000, 1003), (4096, 4099), (2048, 2048), (513, 513)])
def test_fed_blocks_follow_an_int8_update(n, rows):
    before, int8 = preceding_update_k(n, rows)
    fed = fed_blocks(n, rows)
    assert fed <= int8
    assert all(256 <= before[b] <= 512 for b in fed)
