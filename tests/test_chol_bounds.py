"""CPU checks of tests/chol_bounds.py: the schedule mirror against launch tables written out from potrf.cu's rules, the
exact residual against long double, the NumPy emulation of the blocked factorisation inside every bar on every matrix
family, and named defects of the emulation outside the bar that is meant to catch them."""
import numpy as np
import pytest

from tests import chol_bounds as CB
from tests import dense64_bounds as DB


def sig(L):
    k = L["kind"]
    if k == "leaf":
        return f"leaf {L['c0']}+{L['nb']}"
    if k == "feed_old":
        return f"old {L['c0']} k{L['k0']}+{L['kold']}"
    if k == "panel":
        dyn = "" if L["dyn"] is None else " dyn%d+%d" % L["dyn"]
        return f"panel {L['c0']} {L['type']} {L['ctas']}{' event' if L['polled'] is False else ''}{dyn}"
    sl = f" slice-{L['slice'][2]}" if L["slice"] else ""
    return f"upd k{L['k0']}+{L['K']} {L['engine']} {L['m']}x{L['n']}{' skip' if L['row_skip'] else ''}{sl}"


# (n, rows) -> launches, from potrf_rec's rules: split_point, the fused first panel of n <= 256, int8 for K >= 256 with
# K % 32 == 0 and 128^2 K S < 2^31, the diagonal feed in front of int8 updates of K <= 512, ctas <= 132 - 8 polled
TABLE = {
    (129, 129): ["leaf 0+128", "panel 0 fused 1", "leaf 128+1"],
    (256, 256): ["leaf 0+128", "panel 0 fused 8", "leaf 128+128"],
    (257, 257): ["leaf 0+128", "panel 0 plain 3", "upd k0+128 dmma 129x129", "leaf 128+128", "panel 128 fused 1",
                 "leaf 256+1"],
    (257, 260): ["leaf 0+128", "panel 0 plain 3", "upd k0+128 dmma 132x129", "leaf 128+128", "panel 128 fused 1",
                 "leaf 256+1", "panel 256 plain 1"],
    (384, 384): ["leaf 0+128", "panel 0 fused 10", "leaf 128+128", "old 128 k0+128", "panel 128 feed 8",
                 "upd k0+256 int8 128x128 skip", "leaf 256+128"],
    (513, 513): ["leaf 0+128", "panel 0 fused 13", "leaf 128+128", "old 128 k0+128", "panel 128 feed 11",
                 "upd k0+256 int8 257x257 skip", "leaf 256+128", "panel 256 plain 3", "upd k256+128 dmma 129x129",
                 "leaf 384+128", "panel 384 fused 1", "leaf 512+1"],
    (1000, 1003): ["leaf 0+128", "panel 0 fused 20", "leaf 128+128", "old 128 k0+128", "panel 128 feed 18 dyn0+256",
                   "upd k0+256 int8 747x256 skip slice-panel", "leaf 256+128", "panel 256 fused 16", "leaf 384+128",
                   "old 384 k0+384", "panel 384 feed 14 dyn0+512", "upd k0+512 int8 491x488 skip slice-panel",
                   "leaf 512+128", "panel 512 fused 12", "leaf 640+128", "old 640 k512+128",
                   "panel 640 feed 10 dyn512+256", "upd k512+256 int8 235x232 skip slice-panel", "leaf 768+128",
                   "panel 768 fused 7", "leaf 896+104", "panel 896 plain 1"],
    (1152, 1152): ["leaf 0+128", "panel 0 fused 22", "leaf 128+128", "old 128 k0+128", "panel 128 feed 20",
                   "upd k0+256 int8 896x128 skip", "leaf 256+128", "old 256 k0+256", "panel 256 feed 18",
                   "upd k0+384 int8 768x256 skip", "leaf 384+128", "panel 384 fused 16", "leaf 512+128",
                   "panel 512 plain 8", "upd k0+640 int8 512x512", "leaf 640+128", "panel 640 fused 12",
                   "leaf 768+128", "old 768 k640+128", "panel 768 feed 10", "upd k640+256 int8 256x256 skip",
                   "leaf 896+128", "panel 896 fused 8", "leaf 1024+128"],
}
# the updates only, for the larger tables
UPDATES = {
    (2049, 2049): ["upd k0+256 int8 1793x256 skip", "upd k0+512 int8 1537x512 skip", "upd k512+256 int8 1281x256 skip",
                   "upd k0+1024 int8 1025x1025", "upd k1024+256 int8 769x256 skip", "upd k1024+512 int8 513x513 skip",
                   "upd k1536+256 int8 257x257 skip", "upd k1792+128 dmma 129x129"],
    (2049, 2052): ["upd k0+256 int8 1796x256 skip slice-panel", "upd k0+512 int8 1540x512 skip slice-panel",
                   "upd k512+256 int8 1284x256 skip slice-panel", "upd k0+1024 int8 1028x1025 slice-panel",
                   "upd k1024+256 int8 772x256 skip slice-panel", "upd k1024+512 int8 516x513 skip slice-panel",
                   "upd k1536+256 int8 260x257 skip slice-panel", "upd k1792+128 dmma 132x129"],
    (4096, 4096): ["upd k0+256 int8 3840x256 skip", "upd k0+512 int8 3584x512 skip", "upd k512+256 int8 3328x256 skip",
                   "upd k0+1024 int8 3072x1024", "upd k1024+256 int8 2816x256 skip", "upd k1024+512 int8 2560x512 skip",
                   "upd k1536+256 int8 2304x256 skip", "upd k0+2048 int8 2048x2048", "upd k2048+256 int8 1792x256 skip",
                   "upd k2048+512 int8 1536x512 skip", "upd k2560+256 int8 1280x256 skip",
                   "upd k2048+1024 int8 1024x1024", "upd k3072+256 int8 768x256 skip",
                   "upd k3072+512 int8 512x512 skip", "upd k3584+256 int8 256x256 skip"],
}


@pytest.mark.parametrize("key", list(TABLE))
def test_schedule_mirror_matches_the_launch_table(key):
    n, rows = key
    assert [sig(L) for L in CB.schedule(n, rows)] == TABLE[key]


@pytest.mark.parametrize("key", list(UPDATES))
def test_schedule_mirror_matches_the_update_table(key):
    n, rows = key
    ls = CB.schedule(n, rows)
    assert [sig(L) for L in ls if L["kind"] == "update"] == UPDATES[key]
    leaves = [L for L in ls if L["kind"] == "leaf"]
    assert [L["c0"] for L in leaves] == list(range(0, n, 128)) and all(L["slim"] for L in leaves)
    assert all(L["polled"] for L in ls if L["kind"] == "panel")


def test_schedule_mirror_event_orders_grids_beyond_the_sms():
    """The first panel (fused, 8 critical CTAs + ceil((n - 128) / 64)) polls while it leaves 8 SMs free."""
    for n, want in [(7552, True), (7553, False)]:
        first = next(L for L in CB.schedule(n, n) if L["kind"] == "panel")
        assert first["type"] == "fused" and first["ncrit"] == 8 and first["polled"] is want


def test_schedule_mirror_int32_headroom_and_engines():
    ls = CB.schedule(37504, 37504)
    top = next(L for L in ls if L["kind"] == "update" and L["k0"] == 0 and L["K"] == 18816)
    assert top["engine"] == "dmma" and top["headroom_dmma"]                  # 128^2 18816 7 >= 2^31
    assert all(L["engine"] == "int8" for L in ls if L["kind"] == "update" and 256 <= L["K"] <= 9408)
    dm = CB.schedule(1152, 1152, CB.Config(tc=False))
    assert all(L["engine"] == "dmma" and not L["row_skip"] for L in dm if L["kind"] == "update")
    assert not any(L["kind"] == "feed_old" for L in dm)
    dyn = CB.schedule(1000, 1003, CB.Config(static=False))
    assert all(L["slice"] == (L["r0"], 1003, "update") for L in dyn if L["kind"] == "update" and L["engine"] == "int8")
    f32 = CB.schedule(600, 605, CB.Config(f64=False))
    assert {L.get("type") for L in f32 if L["kind"] == "panel"} == {"gemm"}
    assert all(not L["slim"] for L in f32 if L["kind"] == "leaf")


@pytest.mark.parametrize("n", [1, 33, 300, 512])
def test_exact_residual_matches_long_double(n):
    rng = np.random.default_rng(n)
    A = CB.random_spd(n, rng)
    Y = rng.standard_normal((3, n))
    F = CB.emulate(A, n, Y)
    T = np.concatenate([A, Y])
    ri = np.arange(n + 3)
    R, M, trunc = CB.exact_residual(T, F, n, ri)
    Fl = F.astype(np.longdouble)
    ref = (T.astype(np.longdouble) - Fl @ Fl[:n].T).astype(np.float64)
    keep = CB.keep_mask(ri, n)
    err = np.abs(R - ref)[keep]
    assert np.all(err <= trunc[keep] + 2 * (n + 8) * CB.U_LD * M[keep] + 1e-300)
    assert np.median(err / (CB.U * M[keep])) < 1e-2            # far below the rounding the bars are about


def gpr_3_99(n, rng):
    """Clustered RBF gram matrix of variance 3.99: rows whose first entries reach 0.998 of their static scale."""
    return CB.gpr_matrix(n, rng, "rbf", 1e-6, variance=3.99)


FAMILIES = {
    "spd": CB.random_spd,
    "gpr_rbf": lambda n, r: CB.gpr_matrix(n, r, "rbf", 1e-6),
    "gpr_m52": lambda n, r: CB.gpr_matrix(n, r, "m52", 1e-6),
    "gpr_3_99": gpr_3_99,
    "dad": CB.dad,
    "block_cond": lambda n, r: (lambda L: L @ L.T)(DB.factor_with_block_cond(n, r, 1e3)),  # (1e4 from n = 1000 and 1e6:
    # cond(L L^T) ~ 1e16, LAPACK itself fails)
    "scale_m1060": lambda n, r: np.ldexp(CB.random_spd(n, r), -1060),
}
WORST = {}


@pytest.mark.parametrize("family", list(FAMILIES))
@pytest.mark.parametrize("n", [300, 513, 1152])
def test_emulation_inside_every_bar(family, n):
    rng = np.random.default_rng(n)
    A = FAMILIES[family](n, rng)
    Y = rng.standard_normal((3, n)) @ np.linalg.cholesky(A).T if n == 513 else None
    rows = n + (0 if Y is None else 3)
    T = A if Y is None else np.concatenate([A, Y])
    r = CB.check(T, CB.emulate(A, n, Y), n, rows, np.arange(rows), CB.schedule(n, rows), np.diag(A))
    for k, v in r.items():
        WORST[(k, family)] = max(WORST.get((k, family), 0.0), v)
    assert all(v <= 1.0 for v in r.values()), r


def growing_rows(n, rng, A):
    """Extra rows whose solution X grows by 2^12 from the first column to the last: a scale taken from an early k-range
    is too small for the later ones."""
    X = rng.standard_normal((4, n)) * np.exp2(np.linspace(0, 12, n))
    return X @ np.linalg.cholesky(A).T


# mutant -> (family, n, S, the bar that must catch it)
MUTANTS = {
    "drop_digit": ("gpr_3_99", 1000, 7, "rms"),       # the (0, S-1) digit product
    "drop33": ("spd", 1000, 6, "diag_mean"),           # the (3,3) square term at S = 6
    "tile_twice": ("spd", 513, 7, "worst"),            # one 128 x 32 tile of the first int8 update applied twice
    "tile_skip": ("spd", 513, 7, "worst"),             # ... or not at all
    "leaf_early": ("spd", 513, 7, "worst"),            # the leaf reads T before the last update of its last 32 x 32 unit
    "stale_dinv": ("spd", 513, 7, "worst"),            # the panel multiplies by the previous block's dinv64
    "exp_small": ("gpr_3_99", 1000, 7, "worst"),       # static row exponents one too small: the top digit wraps
    "newton1": ("spd", 513, 7, "diag_mean"),           # rsqrt with one Newton step (2^-44) instead of the 2^-66 step
    "extra_static": ("spd", 1000, 7, "worst"),         # the extra rows keep the scale of their first slicing
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_falls_outside_its_bar(mutant):
    family, n, S, bar = MUTANTS[mutant]
    rng = np.random.default_rng(3)
    A = FAMILIES[family](n, rng)
    Y = growing_rows(n, rng, A) if mutant == "extra_static" else None
    rows = n + (0 if Y is None else Y.shape[0])
    T = A if Y is None else np.concatenate([A, Y])
    cfg = CB.Config(S=S)
    ls = CB.schedule(n, rows, cfg)
    ri = np.arange(rows)
    clean = CB.check(T, CB.emulate(A, n, Y, cfg), n, rows, ri, ls, np.diag(A), S=S)
    assert all(v <= 1.0 for v in clean.values()), clean
    with np.errstate(all="ignore"):
        bad = CB.check(T, CB.emulate(A, n, Y, cfg, mutant=mutant), n, rows, ri, ls, np.diag(A), S=S)
    assert not bad[bar] <= 1.0, (mutant, bar, bad)


def test_report_worst_ratios():
    """Prints the worst ratio per bar and family of the emulation (run the file as a whole)."""
    print("\nemulation, worst ratio per bar and family:")
    for (k, fam), v in sorted(WORST.items()):
        print(f"  {k:10s} {fam:12s} {v:.3g}")
