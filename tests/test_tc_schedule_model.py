"""Python mirror of the int8 trailing update's unit assignment (gemm_tc.cu::TcTileIter): the units keep the enumeration of
tests/test_tile_iterators_model.py::tc_units (head units of every row tile first, then the rest), but with units = q G + r
over G clusters, unit i < q G goes to cluster i % G and unit q G + j to cluster G - 1 - j, and the walk passes over other
clusters' units a row tile at a time.  Checked on the CPU for every launch shape of C2 (N = 8192), C5 (N = 4096) and
the M = 2048 factorisation, at cluster widths 1, 2, 4 and grids 64 .. 132."""
import pytest

from tests.test_tile_iterators_model import TC_BM, TC_BN, TC_HEAD, tc_units


def potrf_updates(n, rows, nb=128):
    """(m, n, K) of every trailing update of the recursive Cholesky of an n x n matrix with `rows` rows in all (potrf.cu's
    split rule, as scripts/tc_update_profile.py::c2_updates mirrors it)."""
    out = []

    def rec(n_, col0):
        if n_ <= 2 * nb:
            return
        n1 = ((n_ // nb + 1) // 2) * nb
        rec(n1, col0)
        out.append((rows - col0 - n1, n_ - n1, n1))
        rec(n_ - n1, col0 + n1)

    rec(n, 0)
    return out


def unit_count(m, n, lower, cl):
    ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
    return sum(-(-(min((t + 1) * (TC_BM // TC_BN), ntn) if lower else ntn) // cl) for t in range(ntm))


def tc_units_balanced(m, n, lower, cl, grid, block):
    """The units CTA `block` computes, as gemm_tc.cu::TcTileIter::next() walks them."""
    ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
    rank, c, G = block % cl, block // cl, grid // cl
    head_w = max(cl, TC_HEAD)
    units = unit_count(m, n, lower, cl)
    q, r = divmod(units, G)
    extra = c >= G - r
    left = q + (1 if extra else 0)
    last_gap = (2 * (G - 1 - c) if q > 0 else G - 1 - c) if extra else -1
    skip = c if q > 0 else last_gap

    def ncols(t):
        return min((t + 1) * (TC_BM // TC_BN), ntn) if lower else ntn

    def row_units(pas, t):
        lo, hi = (head_w, ncols(t)) if pas else (0, min(ncols(t), head_w))
        return -(-(hi - lo) // cl) if hi > lo else 0

    out = []
    pas, tm, u, nrow, idx = 0, 0, -1, row_units(0, 0), -1
    while left > 0:
        u += skip + 1
        idx += skip + 1
        steps = 0
        while u >= nrow:
            steps += 1
            if pas == 0 or not lower or ncols(tm) == ntn:
                rest = (ntm - tm) * nrow
                if u < rest:
                    tm, u = tm + u // nrow, u % nrow
                    break
                u -= rest
                tm = ntm
            else:
                u -= nrow
                tm += 1
            if tm >= ntm:
                assert pas == 0, "walked past the last unit"
                pas, tm = 1, 0
            nrow = row_units(pas, tm)
        left -= 1
        skip = last_gap if (left == 1 and last_gap >= 0) else G - 1
        tnb = (head_w if pas else 0) + u * cl
        tn = tnb + rank
        out.append(dict(tm=tm, tnb=tnb, tn=tn, head=pas == 0, valid=tn < ncols(tm), idx=idx, steps=steps))
    return out


def launch_shapes():
    shapes = set()
    for n, rows in [(8192, 8193), (4096, 4097), (2048, 2049), (8192, 8192), (4096, 4096), (2048, 2048)]:
        shapes.update(potrf_updates(n, rows))
    return sorted(shapes)


SHAPES = launch_shapes()


@pytest.mark.parametrize("cl", [1, 2, 4])
def test_balanced_units_cover_every_tile_once(cl):
    for m, n, K in SHAPES:
        old = {(u["tm"], u["tnb"], u["head"]) for u in tc_units(m, n, 1, cl, cl, 0)}  # the unit set of the round-robin walk
        for grid in sorted({64, 65, 96, 130, 131, 132}):
            grid = grid // cl * cl
            G = grid // cl
            per_cta = [tc_units_balanced(m, n, 1, cl, grid, b) for b in range(grid)]
            # the same units (head / rest classification included), each taken by exactly one cluster
            units = [(u["tm"], u["tnb"], u["head"]) for c in range(G) for u in per_cta[c * cl]]
            assert len(units) == len(set(units)) and set(units) == old, (m, n, cl, grid)
            # every lower tile stored exactly once; padding tiles never stored
            ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
            need = {(tm, tn) for tm in range(ntm) for tn in range(min((tm + 1) * (TC_BM // TC_BN), ntn))}
            seen = [(u["tm"], u["tn"]) for us in per_cta for u in us if u["valid"]]
            assert len(seen) == len(set(seen)) and set(seen) == need, (m, n, cl, grid)
            for us in per_cta:
                assert all(u["tn"] < ntn or not u["valid"] for u in us)
            # lock-step clusters, head units first, counts within one of each other
            counts = []
            for c in range(G):
                seqs = [[(u["tm"], u["tnb"]) for u in per_cta[c * cl + r]] for r in range(cl)]
                assert all(s == seqs[0] for s in seqs)
                heads = [u["head"] for u in per_cta[c * cl]]
                assert heads == sorted(heads, reverse=True)
                idx = [u["idx"] for u in per_cta[c * cl]]
                assert idx == sorted(idx)
                counts.append(len(heads))
            assert max(counts) - min(counts) <= 1, (m, n, cl, grid, counts)


@pytest.mark.parametrize("cl", [1, 2, 4])
def test_surplus_units_avoid_the_publishing_clusters(cl):
    """The units holding tiles of the next diagonal block (row tile 0, first 128 columns) are the first work of their
    clusters, and (in a launch with a unit for every cluster) those clusters get no surplus unit unless every cluster but
    fewer than their number has one."""
    for m, n, K in SHAPES:
        for grid in sorted({64, 96, 130, 132}):
            grid = grid // cl * cl
            G = grid // cl
            per = [tc_units_balanced(m, n, 1, cl, grid, c * cl) for c in range(G)]
            counts = [len(us) for us in per]
            pub = [c for c, us in enumerate(per) if any(u["tm"] == 0 and u["head"] for u in us)]
            for c in pub:
                first = per[c][0]
                assert first["tm"] == 0 and first["head"]
            q, r = divmod(sum(counts), G)
            if q and r and r <= G - len(pub):
                assert all(counts[c] == min(counts) for c in pub), (m, n, cl, grid)


def test_walk_steps_stay_few():
    """Passing over G - 1 units takes a few row-tile steps, not one step per unit (that cost ~9 us per tile on the H100)."""
    for m, n, K in SHAPES:
        for b in (0, 64, 129):
            us = tc_units_balanced(m, n, 1, 2, 130, b)
            ntm = -(-m // TC_BM)
            assert all(u["steps"] <= min(ntm, 12) + 2 for u in us), (m, n, b, max(u["steps"] for u in us))
