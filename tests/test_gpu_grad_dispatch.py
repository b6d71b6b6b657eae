"""Every instantiation of the device gradient kernels (csrc/grad.cu) that its dispatch picks, through all four entries.

Which element kernel reduces sum G (.) dK/dtheta and dZ is chosen at launch time from the expression's staging: its
scalar slot count n_s, its per-dimension (ARD) slot count n_a and its staged column count n_cols (build_gradprog,
compile_kprog).  gpr_grad_launch runs gpr_grad_kernel<8 / 16 / 32> for a bare stationary leaf and
gpr_grad_expr_kernel<NS, NA> for everything else; gpr_lowrank_grad_launch (CGLB's N x N pass, its weight generated from
v and z) runs the same nine with LR = true; inducing_pass (SGPR, SVGP and CGLB: three passes, VGP: the square pass) runs
sgpr_grad_kernel<NS, NA, ND, SH>.  That is 25 kernels.  The case table below names, per row, the staging it produces and
the instantiation it must reach in each entry; a Python mirror of the slot and grouping rules checks those claims
against the library on the host, and the table as a whole must reach all 25.

Every row then runs GPR, SGPR, SVGP (the Gaussian route and a per-latent likelihood), VGP and CGLB (trainable v) against
the oracles (tests/grad_expr_oracle.py, sgpr_grad_oracle.py, svgp_grad_oracle.py, lik_oracle.py, vgp_grad_oracle.py,
cglb_grad_oracle.py) with a bar
that holds per slot, not per model; two checks need no oracle (a White leaf against the same amount of noise, and a
bare leaf against the same leaf under a one-child Sum); and the staging limits are accepted at the limit and refused
one step past it, the same way in all four entries."""
import functools

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from gpflow_b200.base import Parameter
from oracle import gp_oracle as O
from tests import cglb_grad_oracle as CGO
from tests import grad_check as GC
from tests import grad_expr_oracle as GO
from tests import lik_oracle as LO
from tests import sgpr_grad_oracle as SO
from tests import svgp_grad_oracle as SVO
from tests import vgp_grad_oracle as VO

K = gpf.kernels
gpu = pytest.mark.gpu

# ---- kernel specs: one description builds the device expression, the oracle expression and the staging mirror ------
_CLS = {"rbf": (K.SquaredExponential, O.SquaredExponential), "m12": (K.Matern12, O.Matern12),
        "m32": (K.Matern32, O.Matern32), "m52": (K.Matern52, O.Matern52), "exp": (K.Exponential, O.Exponential),
        "rq": (K.RationalQuadratic, O.RationalQuadratic), "lin": (K.Linear, O.Linear),
        "poly": (K.Polynomial, O.Polynomial), "white": (K.White, O.White), "const": (K.Constant, O.Constant)}
BARE = {"rbf", "m12", "m32", "m52", "exp"}          # the leaves gpr_grad_kernel takes on its own
STATIONARY = BARE | {"rq"}
LINEAR_LIKE = {"lin", "poly"}


def leaf(kind, **kw):
    return (kind, kw)


def add(*c):
    return ("sum", list(c))


def mul(*c):
    return ("prod", list(c))


def ard(n, base):
    """n distinct lengthscales (or Linear weights) around `base`, not monotone in the dimension."""
    return base * (0.7 + 0.8 * ((np.arange(n) * 7) % n) / n)


def build(spec):
    """(device kernel, oracle kernel) with the same values."""
    op, arg = spec
    if op in ("sum", "prod"):
        kids = [build(s) for s in arg]
        dc, oc = (K.Sum, O.Sum) if op == "sum" else (K.Product, O.Product)
        return dc([k for k, _ in kids]), oc([o for _, o in kids])
    dcls, ocls = _CLS[op]
    kw = {k: v for k, v in arg.items() if v is not None}
    return dcls(**kw), ocls(**kw)


def spec_leaves(spec):
    op, arg = spec
    return [lf for s in arg for lf in spec_leaves(s)] if op in ("sum", "prod") else [spec]


def staging(spec, D):
    """(n_s, n_a, n_cols, n_groups) by the rules of build_gradprog and compile_kprog.  Per leaf: stationary leaves
    take variance + (lengthscale, or one slot per ARD dim) + (RQ alpha); Linear / Polynomial take variance (or one slot
    per ARD dim) + (Polynomial offset); White / Constant take variance.  Gram groups: leaves on the same active dims
    share one when neither has ARD weights, or when both carry the same weights the same way (1 / lengthscale on both
    sides for stationary leaves, the variance on one side for Linear / Polynomial); the staged columns are the groups'
    dims laid end to end, so a column two groups read is staged twice."""
    groups = []
    n_s = n_a = 0
    for kind, kw in spec_leaves(spec):
        ar = False
        nd = 0
        if kind in STATIONARY | LINEAR_LIKE:
            dims = tuple(int(d) for d in (kw.get("active_dims") if kw.get("active_dims") is not None else range(D)))
            par = np.asarray(kw["lengthscales"] if kind in STATIONARY else kw.get("variance", 1.0), dtype=np.float64)
            ar = par.ndim > 0
            wmode = 0 if not ar else (1 if kind in LINEAR_LIKE else 2)
            w = () if not ar else tuple(par if kind in LINEAR_LIKE else 1.0 / par)
            if (dims, wmode, w) not in groups:
                groups.append((dims, wmode, w))
            nd = len(dims)
        if kind in STATIONARY:
            n_s += 1 + (0 if ar else 1) + (1 if kind == "rq" else 0)
        elif kind in LINEAR_LIKE:
            n_s += (0 if ar else 1) + (1 if kind == "poly" else 0)
        else:
            n_s += 1
        n_a += nd if ar else 0
    return n_s, n_a, sum(len(g[0]) for g in groups), len(groups)


def _bucket(n):
    return 8 if n <= 8 else (16 if n <= 16 else 36)


def dispatch(spec, D, lowrank=False):
    """(GPR kernel, inducing-pass kernel) as gpr_grad_launch and inducing_pass choose them; with `lowrank` the N x N
    kernel as gpr_lowrank_grad_launch (CGLB) chooses it, the same template with LR = true."""
    n_s, n_a, nc, _ = staging(spec, D)
    lr = ",true" if lowrank else ""
    if spec[0] in BARE:
        gpr = f"gpr_grad_kernel<{8 if nc <= 8 else (16 if nc <= 16 else 32)}{lr}>"
    else:
        gpr = f"gpr_grad_expr_kernel<{_bucket(n_s)},{32 if n_a else 0}{lr}>"
    nd = 16 if (n_a == 0 and n_s <= 8 and nc <= 16) else 32
    sh = "true" if (n_a > 0 and n_s > 16) else "false"
    return gpr, f"sgpr_grad_kernel<{_bucket(n_s)},{32 if n_a else 0},{nd},{sh}>"


ALL_KERNELS = {"gpr_grad_kernel<8>", "gpr_grad_kernel<16>", "gpr_grad_kernel<32>",
               "gpr_grad_expr_kernel<8,0>", "gpr_grad_expr_kernel<16,0>", "gpr_grad_expr_kernel<36,0>",
               "gpr_grad_expr_kernel<8,32>", "gpr_grad_expr_kernel<16,32>", "gpr_grad_expr_kernel<36,32>",
               "sgpr_grad_kernel<8,0,16,false>", "sgpr_grad_kernel<8,0,32,false>", "sgpr_grad_kernel<16,0,32,false>",
               "sgpr_grad_kernel<36,0,32,false>", "sgpr_grad_kernel<8,32,32,false>",
               "sgpr_grad_kernel<16,32,32,false>", "sgpr_grad_kernel<36,32,32,true>"}
LR_KERNELS = {k.replace(">", ",true>") for k in ALL_KERNELS if k.startswith("gpr_grad")}
INDUCING_KERNELS = {k for k in ALL_KERNELS if k.startswith("sgpr_grad")}
ALL_KERNELS = ALL_KERNELS | LR_KERNELS


# ---- the case table ------------------------------------------------------------------------------------------------
# The data seed of a row where the default one left a slot needlessly far below the largest in some entry (a gradient
# near one of its zero crossings by chance); see BAR.
SEEDS = {"d16_rbf_ard": 206, "d9_m12_ard": 215, "s9": 219, "s8": 226, "s8_ard": 223, "s17": 222, "s9_ard": 210,
         "d32_m32_ard": 225, "s17_ard_32_cols_4_groups": 215, "ard32_one_group": 221, "s35_ard_12_leaves": 224}


def _rows():
    r = {}

    def row(name, spec, D, stage, gpr, ind):
        r[name] = dict(spec=spec, D=D, stage=stage, gpr=gpr, ind=ind, seed=SEEDS.get(name, 100 + len(r)))

    s = np.sqrt
    # a bare stationary leaf: gpr_grad_kernel<ND> by its active dims, both sides of 8 | 9 and 16 | 17
    row("d8_rbf", leaf("rbf", variance=1.2, lengthscales=1.1 * s(8)), 8, (2, 0, 8, 1),
        "gpr_grad_kernel<8>", "sgpr_grad_kernel<8,0,16,false>")
    row("d9_m12_ard", leaf("m12", variance=0.9, lengthscales=ard(9, 1.6 * s(9))), 9, (1, 9, 9, 1),
        "gpr_grad_kernel<16>", "sgpr_grad_kernel<8,32,32,false>")
    row("d16_m32", leaf("m32", variance=1.1, lengthscales=1.2 * s(16)), 16, (2, 0, 16, 1),
        "gpr_grad_kernel<16>", "sgpr_grad_kernel<8,0,16,false>")
    row("d16_rbf_ard", leaf("rbf", variance=0.8, lengthscales=ard(16, 1.3 * s(16))), 16, (1, 16, 16, 1),
        "gpr_grad_kernel<16>", "sgpr_grad_kernel<8,32,32,false>")
    row("d17_m52", leaf("m52", variance=1.3, lengthscales=1.4 * s(17)), 17, (2, 0, 17, 1),
        "gpr_grad_kernel<32>", "sgpr_grad_kernel<8,0,32,false>")
    # 17 of 24 columns, in an order that is neither sorted nor contiguous
    perm = [int(c) for c in np.random.default_rng(17).permutation(24)[:17]]
    row("d17_of_24_exp_ard", leaf("exp", variance=0.7, lengthscales=ard(17, 1.5 * s(17)), active_dims=perm), 24,
        (1, 17, 17, 1), "gpr_grad_kernel<32>", "sgpr_grad_kernel<8,32,32,false>")
    row("d32_m12", leaf("m12", variance=1.0, lengthscales=1.5 * s(32)), 32, (2, 0, 32, 1),
        "gpr_grad_kernel<32>", "sgpr_grad_kernel<8,0,32,false>")
    row("d32_m32_ard", leaf("m32", variance=1.2, lengthscales=ard(32, 1.3 * s(32))), 32, (1, 32, 32, 1),
        "gpr_grad_kernel<32>", "sgpr_grad_kernel<8,32,32,false>")
    # expressions without ARD: n_s = 8 / 9 / 16 / 17 / 36
    row("s8", add(mul(add(leaf("rbf", variance=1.1, lengthscales=2.2), leaf("m32", variance=0.6, lengthscales=3.1)),
                      leaf("lin", variance=0.3)),
                  leaf("rq", variance=0.8, lengthscales=1.7, alpha=0.9)), 6, (8, 0, 6, 1),
        "gpr_grad_expr_kernel<8,0>", "sgpr_grad_kernel<8,0,16,false>")
    row("s9", add(leaf("rq", variance=0.9, lengthscales=1.2, alpha=1.5, active_dims=[0, 1, 2]),
                  leaf("rq", variance=0.6, lengthscales=1.8, alpha=0.7, active_dims=[3, 4, 5]),
                  leaf("m52", variance=0.5, lengthscales=2.9), leaf("white", variance=0.05)), 6, (9, 0, 12, 3),
        "gpr_grad_expr_kernel<16,0>", "sgpr_grad_kernel<16,0,32,false>")
    row("s16", add(mul(add(leaf("rq", variance=0.8, lengthscales=2.4, alpha=1.2),
                           leaf("rq", variance=0.5, lengthscales=1.3, alpha=2.0, active_dims=[0, 1, 2, 3])),
                       leaf("poly", degree=2.0, variance=0.1, offset=0.9)),
                   leaf("rq", variance=0.4, lengthscales=1.6, alpha=0.6, active_dims=[4, 5, 6]),
                   leaf("m12", variance=0.3, lengthscales=3.5), leaf("exp", variance=0.35, lengthscales=2.2,
                                                                     active_dims=[0, 1, 2, 3]),
                   leaf("const", variance=0.2)), 7, (16, 0, 14, 3),
        "gpr_grad_expr_kernel<16,0>", "sgpr_grad_kernel<16,0,32,false>")
    h1, h2 = list(range(6)), list(range(6, 12))
    row("s17", add(leaf("rq", variance=0.6, lengthscales=2.8, alpha=1.1), leaf("rq", variance=0.4, lengthscales=4.5,
                                                                            alpha=0.5),
                   leaf("rbf", variance=0.5, lengthscales=2.1, active_dims=h1),
                   leaf("m32", variance=0.45, lengthscales=2.6, active_dims=h2), leaf("lin", variance=0.05),
                   leaf("poly", degree=2.0, variance=0.08, offset=0.6, active_dims=h1),
                   leaf("exp", variance=0.3, lengthscales=3.0, active_dims=h2), leaf("white", variance=0.04),
                   leaf("const", variance=0.15)), 12, (17, 0, 24, 3),
        "gpr_grad_expr_kernel<36,0>", "sgpr_grad_kernel<36,0,32,false>")
    # the scalar limit: 12 Rational Quadratic leaves of 3 slots, in the 4-group limit, a flat Sum with two Products
    g4 = [None, [0, 1, 2, 3, 4], [5, 6, 7, 8, 9], [9, 0, 3]]
    rq12 = [leaf("rq", variance=0.25 + 0.05 * i, lengthscales=(1.2 + 0.25 * i) * (1.6 if g4[i % 4] is None else 1.0),
                 alpha=0.4 + 0.1 * i, active_dims=g4[i % 4]) for i in range(12)]
    row("s36_12_leaves_4_groups", add(mul(rq12[0], rq12[1]), *rq12[2:6], mul(rq12[6], rq12[7]), *rq12[8:]), 10,
        (36, 0, 23, 4), "gpr_grad_expr_kernel<36,0>", "sgpr_grad_kernel<36,0,32,false>")
    # with ARD: n_s = 8 / 9 / 16 / 17 / 35 (36 would need 12 scalar-lengthscale RQ leaves, which leave no ARD slot)
    row("s8_ard", add(leaf("rbf", variance=0.9, lengthscales=ard(5, 2.4)),
                      leaf("rq", variance=0.6, lengthscales=2.0, alpha=1.3), leaf("lin", variance=0.1),
                      leaf("poly", degree=2.0, variance=0.06, offset=0.8), leaf("white", variance=0.05)), 5,
        (8, 5, 10, 2), "gpr_grad_expr_kernel<8,32>", "sgpr_grad_kernel<8,32,32,false>")
    q4, r2 = [0, 1, 2, 3], [4, 5]
    row("s9_ard", add(mul(leaf("m52", variance=1.0, lengthscales=ard(4, 2.0), active_dims=q4),
                          leaf("lin", variance=ard(4, 0.4), active_dims=q4)),
                      leaf("rq", variance=0.5, lengthscales=2.3, alpha=0.8), leaf("m32", variance=0.4, lengthscales=3.3),
                      leaf("exp", variance=0.3, lengthscales=1.4, active_dims=r2), leaf("white", variance=0.05)), 6,
        (9, 8, 16, 4), "gpr_grad_expr_kernel<16,32>", "sgpr_grad_kernel<16,32,32,false>")
    lo4, hi4 = [0, 1, 2, 3], [4, 5, 6, 7]
    row("s16_ard", add(leaf("rq", variance=0.7, lengthscales=ard(8, 3.0), alpha=1.4),
                       leaf("rq", variance=0.5, lengthscales=2.6, alpha=0.7),
                       leaf("rq", variance=0.4, lengthscales=1.5, alpha=2.2, active_dims=lo4),
                       leaf("m12", variance=0.3, lengthscales=2.0, active_dims=hi4),
                       mul(leaf("poly", degree=2.0, variance=0.05, offset=1.0), leaf("lin", variance=0.2,
                                                                                    active_dims=lo4)),
                       leaf("const", variance=0.2), leaf("exp", variance=0.25, lengthscales=4.0)), 8, (16, 8, 24, 4),
        "gpr_grad_expr_kernel<16,32>", "sgpr_grad_kernel<16,32,32,false>")
    # 32 staged columns in 4 groups; columns 4..7 are staged by two of them (an ARD group and a scalar one), and 0, 5
    # by three: the dZ merge of sgpr_grad_kernel adds them into one atomicAdd per (row, column)
    ga, gb, gc, gd = list(range(8)), list(range(4, 16)), list(range(16, 22)), [22, 23, 0, 5, 9, 13]
    row("s17_ard_32_cols_4_groups", add(
        leaf("rbf", variance=0.8, lengthscales=ard(8, 3.2), active_dims=ga),
        leaf("rq", variance=0.5, lengthscales=3.4, alpha=1.2, active_dims=gb),
        mul(leaf("lin", variance=ard(6, 0.3), active_dims=gc), leaf("m32", variance=0.7, lengthscales=2.4,
                                                                     active_dims=gd)),
        leaf("rq", variance=0.3, lengthscales=5.0, alpha=0.6, active_dims=gb),
        leaf("m52", variance=0.35, lengthscales=1.9, active_dims=gd),
        leaf("poly", degree=2.0, variance=0.01, offset=0.7, active_dims=gb),
        leaf("white", variance=0.04), leaf("const", variance=0.1),
        leaf("exp", variance=0.2, lengthscales=4.1, active_dims=gb)), 24, (17, 14, 32, 4),
        "gpr_grad_expr_kernel<36,32>", "sgpr_grad_kernel<36,32,32,true>")
    rq11 = [leaf("rq", variance=0.2 + 0.04 * i, lengthscales=(1.3 + 0.2 * i) * (1.5 if i % 3 == 0 else 1.0),
                 alpha=0.4 + 0.1 * i, active_dims=[None, hi4, lo4][i % 3]) for i in range(11)]
    row("s35_ard_12_leaves", add(leaf("rq", variance=0.6, lengthscales=ard(4, 1.8), alpha=1.1, active_dims=lo4),
                                 mul(rq11[0], rq11[1]), *rq11[2:]), 8, (35, 4, 20, 4),
        "gpr_grad_expr_kernel<36,32>", "sgpr_grad_kernel<36,32,32,true>")
    # the ARD limit: two ARD leaves with the same lengthscales on the same 16 dims share one group and take 16 slots each
    ell16 = ard(16, 1.2 * s(16))
    row("ard32_one_group", add(leaf("rbf", variance=0.7, lengthscales=ell16),
                               leaf("m52", variance=0.6, lengthscales=ell16.copy())), 16, (2, 32, 16, 1),
        "gpr_grad_expr_kernel<8,32>", "sgpr_grad_kernel<8,32,32,false>")
    return r


ROWS = _rows()
NAMES = list(ROWS)
STRIP = dict(spec=add(leaf("rbf", variance=0.9, lengthscales=ard(3, 1.6)),
                      *[leaf("rq", variance=0.3 + 0.1 * i, lengthscales=1.0 + 0.4 * i, alpha=0.5 + 0.5 * i)
                        for i in range(5)],
                      leaf("m32", variance=0.4, lengthscales=2.5)), D=3, stage=(18, 3, 6, 2),
             gpr=None, ind="sgpr_grad_kernel<36,32,32,true>", seed=0)


# ---- host checks of the table: no device needed --------------------------------------------------------------------
def test_table_reaches_every_instantiation():
    reached = {}
    cglb = set()
    for name, r in ROWS.items():
        gpr, ind = dispatch(r["spec"], r["D"])
        assert (gpr, ind) == (r["gpr"], r["ind"]), name
        reached.setdefault(gpr, []).append(name)
        reached.setdefault(ind, []).append(name)
        lr, ind_lr = dispatch(r["spec"], r["D"], lowrank=True)
        assert lr == gpr.replace(">", ",true>") and ind_lr == ind, name
        cglb.update((lr, ind_lr))
        reached.setdefault(lr, []).append(name)
    assert set(reached) == ALL_KERNELS, sorted(ALL_KERNELS - set(reached))
    # the cglb entry alone: all nine low-rank N x N kernels and every inducing-pass kernel
    assert len(LR_KERNELS) == 9 and cglb == LR_KERNELS | INDUCING_KERNELS, sorted((LR_KERNELS | INDUCING_KERNELS) - cglb)
    # each dispatch boundary crossed from both sides
    stages = [r["stage"] for r in ROWS.values()]
    for n_s in (8, 9, 16, 17):
        assert any(st[0] == n_s and st[1] == 0 for st in stages) and any(st[0] == n_s and st[1] > 0 for st in stages)
    assert any(st[0] == 36 for st in stages) and any(st[0] == 35 and st[1] > 0 for st in stages)
    for nc in (16, 17, 32):
        assert any(st[2] == nc and st[1] == 0 for st in stages)
    bare = {(r["spec"][0], staging(r["spec"], r["D"])[2], r["stage"][1] > 0) for r in ROWS.values()
            if r["spec"][0] in BARE}
    assert {nc for _, nc, _ in bare} == {8, 9, 16, 17, 32}
    assert {k for k, _, _ in bare} == BARE and {a for _, _, a in bare} == {False, True}


@pytest.mark.parametrize("name", NAMES + ["strip"])
def test_staging_mirror_agrees_with_library(name):
    r = STRIP if name == "strip" else ROWS[name]
    kp, _ = build(r["spec"])
    D = r["D"]
    st = staging(r["spec"], D)
    assert st == r["stage"]
    nodes, n, dims, ar = gpf.kernels.compile_kernel(kp, D)
    assert _lib.load().gpk_gpr_lml_grad_slots(nodes, n, dims, ar, D) == st[0] + st[1]
    assert sum(c for _, _, c in gpf.kernels.gradient_slots(kp, D)) == st[0] + st[1]
    assert len(spec_leaves(r["spec"])) <= 12


def _past_limits():
    """One step past each staging limit: (name, device kernel factory, D, the library's message)."""
    ell17 = ard(17, 4.0)
    return {
        "13_leaves": (lambda: build(add(*spec_leaves(ROWS["s36_12_leaves_4_groups"]["spec"]),
                                        leaf("white", variance=0.1)))[0], 10, "more than 12 leaf kernels"),
        "34_ard_slots": (lambda: build(add(leaf("rbf", lengthscales=ell17), leaf("m52", lengthscales=ell17.copy())))[0],
                         17, "more than 32 per-dimension gradient slots"),
        "33_columns": (lambda: K.SquaredExponential(active_dims=list(range(17)))
                       + K.Matern52(active_dims=list(range(17, 33))), 33, "33 active columns, at most 32"),
        "5_groups": (lambda: build(add(*[leaf("rbf", lengthscales=1.0 + i, active_dims=[i]) for i in range(5)]))[0], 5,
                     "more than 4 distinct"),
    }


PAST = _past_limits()


def test_limits_are_accepted_and_one_step_past_refused_by_the_slot_query():
    lib = _lib.load()
    at = {"12 leaves": "s36_12_leaves_4_groups", "36 scalar slots": "s36_12_leaves_4_groups",
          "32 ARD slots": "ard32_one_group", "32 columns": "s17_ard_32_cols_4_groups", "4 groups": "s36_12_leaves_4_groups"}
    for what, name in at.items():
        r = ROWS[name]
        assert len(spec_leaves(r["spec"])) == 12 or what != "12 leaves"
        n_s, n_a, nc, ng = r["stage"]
        assert {"36 scalar slots": n_s == 36, "32 ARD slots": n_a == 32, "32 columns": nc == 32,
                "4 groups": ng == 4}.get(what, True), what
        nodes, n, dims, ar = gpf.kernels.compile_kernel(build(r["spec"])[0], r["D"])
        assert lib.gpk_gpr_lml_grad_slots(nodes, n, dims, ar, r["D"]) == n_s + n_a
    for name, (make, D, msg) in PAST.items():
        nodes, n, dims, ar = gpf.kernels.compile_kernel(make(), D)
        assert lib.gpk_gpr_lml_grad_slots(nodes, n, dims, ar, D) == -1, name
        assert msg in lib.gpk_last_error().decode(), name


# ---- data and oracles ----------------------------------------------------------------------------------------------
S2 = 0.15
ENTRIES = ("gpr", "sgpr", "svgp_gauss", "svgp_lik", "vgp", "cglb")


def _sizes(i):
    """Ragged sizes per row: GPR N < 512 (the factor on DMMA), inducing N and M off the 32 / 64 tile edges."""
    return dict(P=1 + i % 2, N_gpr=(333, 413, 479)[i % 3], N=(301, 389, 467)[i % 3], M=(45, 70)[i % 2],
                N_vgp=(173, 211)[i % 2], wq=[(True, False), (False, False), (True, True), (False, True)][i % 4],
                wq_lik=[(False, False), (True, True), (False, True), (True, False)][i % 4],
                lik="bernoulli" if i % 2 == 0 else "student_t", num_data=None if i % 2 == 0 else 4000)


def _lik(name):
    if name == "bernoulli":
        return gpf.likelihoods.Bernoulli(), LO.Bernoulli()
    return gpf.likelihoods.StudentT(scale=0.7, df=4.0), LO.StudentT(0.7, 4.0)


def _case(name):
    if name == "strip":
        # Kuf: ceil(M / 32) = 2 row strips, so about 2048 / 2 = 1024 CTAs per strip row and, with 1029 column tiles of
        # X, two tiles per CTA (the last CTA one): the dz of a row accumulates across tiles before its atomicAdd
        return STRIP, dict(P=2, N=32900, M=45, wq=(True, False), wq_lik=(False, True), lik="student_t",
                           num_data=None)
    i = NAMES.index(name)
    return ROWS[name], _sizes(i)


@functools.lru_cache(maxsize=None)
def _inputs(name, entry):
    r, sz = _case(name)
    D, P = r["D"], sz["P"]
    seed = r["seed"]
    N = sz["N_gpr"] if entry == "gpr" else (sz["N_vgp"] if entry == "vgp" else sz["N"])
    d = O.make_data(seed, N, D, P)
    X, Y = d["X"], d["Y"]
    out = dict(X=X, Y=Y, P=P)
    if entry in ("sgpr", "svgp_gauss", "svgp_lik", "cglb"):
        out["Z"] = GC.z(sz["M"], D, seed)
    if entry == "cglb":
        out["v"] = 0.3 * np.random.default_rng(seed + 1).standard_normal((P, N))
    if entry == "svgp_lik":
        out["Y"] = LO.targets(sz["lik"], np.sin(X[:, :1] @ np.ones((1, P))), np.random.default_rng(seed))
    if entry.startswith("svgp"):
        whiten, q_diag = sz["wq"] if entry == "svgp_gauss" else sz["wq_lik"]
        out.update(whiten=whiten, q_diag=q_diag, num_data=sz["num_data"], lik=sz["lik"])
        out["q_mu"], out["q_sqrt"] = GC.q(sz["M"], P, q_diag, seed, upper_noise=False)
    if entry == "vgp":
        out["q_mu"], out["q_sqrt"] = GC.q(N, P, False, seed, upper_noise=False)
    return out


@functools.lru_cache(maxsize=None)
def oracle(name, entry):
    """The oracle's value and gradient dict for one row and entry (cached: the bar check and the device check share)."""
    r, _ = _case(name)
    ko = build(r["spec"])[1]
    a = _inputs(name, entry)
    jit = gpf.config.default_jitter()
    if entry == "gpr":
        return GO.gpr_lml_and_grad_expr(a["X"], a["Y"], ko, S2, abs_sums=True)
    if entry == "sgpr":
        return SO.sgpr_elbo_and_grad_expr(a["X"], a["Y"], ko, a["Z"], S2, jitter=jit)
    if entry == "cglb":
        return CGO.cglb_elbo_and_grad_expr(a["X"], a["Y"], ko, a["Z"], S2, a["v"], jitter=jit, abs_sums=True)
    if entry.startswith("svgp"):
        lik = LO.Gaussian(S2) if entry == "svgp_gauss" else _lik(a["lik"])[1]
        return SVO.svgp_elbo_and_grad(a["X"], a["Y"], [ko], [a["Z"]], a["q_mu"], a["q_sqrt"], lik, whiten=a["whiten"],
                                      num_data=a["num_data"], jitter=jit)
    return VO.vgp_elbo_and_grad_expr(a["X"], a["Y"], ko, a["q_mu"], a["q_sqrt"], S2, jitter=jit)


def _flat_slots(g, entry):
    """The oracle's kernel slots (every leaf parameter entry) and its noise slot, as one vector."""
    v = [np.ravel(np.asarray(x, dtype=np.float64)) for gd in g["leaves"] for x in gd.values()]
    if entry == "svgp_gauss":
        v.append(np.array([g["lik"]]))
    elif entry != "svgp_lik":
        v.append(np.array([g["noise_variance"]]))
    return np.concatenate(v)


# The smallest slot of any row and entry relative to that entry's largest.  A gradient w.r.t. one of 32 ARD
# lengthscales, or w.r.t. one of 12 leaves' alphas, sits far below the largest slot for most data: the rows reach 4e-6
# at worst (the data seeds in SEEDS were picked to keep it there).
BAR = 1e-6


def _bar_ratio(name, entry):
    """min |slot| / max |slot| over the oracle's slots: a per-Parameter bar only bites on slots of a size it can see."""
    s = np.abs(_flat_slots(oracle(name, entry)[1], entry))
    return float(np.min(s) / np.max(s))


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("name", NAMES)
def test_rows_put_every_slot_within_reach_of_the_largest(name, entry):
    """The chosen hyperparameters and data keep every slot at least BAR of the largest in every entry, so that the
    per-Parameter bar of the inducing entries (1e-7 of the Parameter's largest entry) still resolves every slot."""
    assert _bar_ratio(name, entry) >= BAR


# ---- device against oracle -----------------------------------------------------------------------------------------
def _no_false_zeros(g, r, what):
    assert np.all(np.isfinite(g)), what
    assert not np.any((g == 0.0) & (r != 0.0)), f"{what}: a slot is exactly 0 where the oracle's is not"


# GPR: |device - oracle| <= C x S per slot, S = sum_ij |G_ij A_ij dK_ij/dtheta| (the oracle's abs_sums).
# The reduction itself is fp64 with at most ~32 sequential terms per thread, a 5-level shuffle tree, 4 warps and one
# atomicAdd per CTA (< 120 CTAs at N < 512): under 200 roundings, 2e-14 S.  What dominates is G: the device and the
# oracle each form K^-1 and alpha from their own Cholesky of K (DMMA at N < 512), which agree to about
# kappa(K) x u ~ (N var / s2) x 1.1e-16 ~ 5e-13 of |G|'s scale at these sizes, and an element's error relative to the
# sum of |terms| stays within that: C_GPR = 1e-11.  The sqrt-type leaves (Matern12, Exponential) add one more source:
# both forwards evaluate the diagonal through the norm expansion |x|^2 + |x|^2 - 2 x.x, whose rounding (a few
# u |x/l|^2) sits under the square root and moves k_ii by up to ~1e-8 var, differently in each; that is a change of the
# effective noise, which moves G by ~1e-8 / s2 of its diagonal: C_GPR_SQRT = 1e-8.  Measured with these rows on an
# H100 80GB HBM3 (700 W limit): at most 5e-13 S without a sqrt-type leaf, 1.7e-9 S with one.
C_GPR = 1e-11
C_GPR_SQRT = 1e-8
# SGPR / SVGP / VGP: per Parameter, relative to that Parameter's largest entry with a floor of 1e-3 x the model's
# largest gradient.  The same two sources, through more dense algebra (two Cholesky factors, triangular solves and
# inverses) on both sides: 1e-10 for rows of smooth leaves (measured at most 2.7e-12), and, where a sqrt-type leaf
# puts its ~1e-8 diagonal noise into Kuu and K(X, X), 2e-7 (measured at most 4.8e-8).
RTOL_INDUCING = 1e-10
RTOL_INDUCING_SQRT = 2e-7
# CGLB (trainable v): |device - oracle| <= C x S per slot and per element of Z and v, S the oracle's sum of |terms| over
# the N x N, Kuf, Kuu and Kdiag sources (abs_sums).  The reductions add ~1e-14 S as in GPR; what dominates is the
# forward on each side: L and LB (as in SGPR), r = e - K^ v through the matrix-free product, and z = Q^-1 r, whose
# rounding grows with the conditioning of Q = A'^T A' + s I, about (N var / s) u ~ 1e-13 here.  The sqrt-type leaves
# add their ~1e-8 var diagonal noise to K^ and Kuu, and Kuu's enters Guf and Guu amplified by its conditioning (about
# 40 for d32_m12): the elements of dZ move by ~1e-7 S (the oracle itself moves by 8e-8 S on d32_m12 under a random
# 1e-8 var diagonal).  Measured with these rows on an H100 80GB HBM3 (700 W limit): at most 1.1e-12 S without a
# sqrt-type leaf (s36_12_leaves_4_groups), 1.9e-7 S with one (d32_m12, on an element of dZ).
C_CGLB = 1e-11
C_CGLB_SQRT = 1e-6


def _has_sqrt_leaf(spec):
    return any(k in ("m12", "exp") for k, _ in spec_leaves(spec))


def gpr_error(name):
    """max over slots of |device - oracle| / (C x S); <= 1 passes."""
    r, _ = _case(name)
    a = _inputs(name, "gpr")
    kp, _ = build(r["spec"])
    m = gpf.models.GPR((a["X"], a["Y"]), kp, noise_variance=S2)
    lml, grads = m.log_marginal_likelihood_and_grad()
    ref_lml, g = oracle(name, "gpr")
    np.testing.assert_allclose(float(lml), ref_lml, rtol=1e-8)
    ref = GC.leaf_grads_by_param(kp, g["leaves"])
    sc = GC.leaf_grads_by_param(kp, g["leaves_abs"])
    ref[id(m.likelihood.variance)] = np.asarray(g["noise_variance"])
    sc[id(m.likelihood.variance)] = np.asarray(g["noise_abs"])
    assert {id(p) for p in grads} == set(ref)
    c = C_GPR_SQRT if _has_sqrt_leaf(r["spec"]) else C_GPR
    worst = 0.0
    for p, v in grads.items():
        v = np.asarray(v, dtype=np.float64).reshape(p.shape)
        _no_false_zeros(v, ref[id(p)], name)
        worst = max(worst, float(np.max(np.abs(v - ref[id(p)]) / (c * sc[id(p)]))))
    return worst


def _cglb_model(name):
    r, _ = _case(name)
    a = _inputs(name, "cglb")
    kp, _ = build(r["spec"])
    m = gpf.models.CGLB((a["X"], a["Y"]), kp, a["Z"].copy(), noise_variance=S2, v_grad_optimization=True)
    m.aux_vec.assign(a["v"].copy())
    return m, kp


def cglb_error(name):
    """max over the kernel slots, the noise and every element of Z and v of |device - oracle| / (C x S); <= 1 passes."""
    r, _ = _case(name)
    m, kp = _cglb_model(name)
    val, grads = m.elbo_and_grad()
    ref_val, g = oracle(name, "cglb")
    np.testing.assert_allclose(float(val), ref_val, rtol=1e-8)
    ref = GC.leaf_grads_by_param(kp, g["leaves"])
    sc = GC.leaf_grads_by_param(kp, g["leaves_abs"])
    for p, key in ((m.likelihood.variance, "noise"), (m.inducing_variable.Z, "Z"), (m.aux_vec, "v")):
        ref[id(p)] = np.asarray(g["noise_variance" if key == "noise" else key])
        sc[id(p)] = np.asarray(g[key + "_abs"])
    assert {id(p) for p in grads} == set(ref)
    c = C_CGLB_SQRT if _has_sqrt_leaf(r["spec"]) else C_CGLB
    worst = 0.0
    for p, v in grads.items():
        v = np.asarray(v, dtype=np.float64).reshape(p.shape)
        _no_false_zeros(v, ref[id(p)], (name, "cglb"))
        err, bar = np.abs(v - ref[id(p)]), c * sc[id(p)]
        # S = 0 (a column of Z no leaf reads): the entry must be exactly the oracle's 0
        worst = max(worst, float(np.max(np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err > 0, np.inf,
                                                                                                     0.0)))))
    return worst


def _model(name, entry):
    r, _ = _case(name)
    a = _inputs(name, entry)
    kp, _ = build(r["spec"])
    if entry == "sgpr":
        return gpf.models.SGPR((a["X"], a["Y"]), kp, a["Z"].copy(), noise_variance=S2), kp
    if entry.startswith("svgp"):
        lp = gpf.likelihoods.Gaussian(S2) if entry == "svgp_gauss" else _lik(a["lik"])[0]
        return gpf.models.SVGP(kp, lp, a["Z"].copy(), num_latent_gps=a["P"], q_mu=a["q_mu"].copy(),
                               q_sqrt=a["q_sqrt"].copy(), whiten=a["whiten"], q_diag=a["q_diag"],
                               num_data=a["num_data"]), kp
    m = gpf.models.VGP((a["X"], a["Y"]), kp, gpf.likelihoods.Gaussian(S2))
    m.q_mu.assign(a["q_mu"])
    m.q_sqrt.assign(a["q_sqrt"])
    return m, kp


def inducing_error(name, entry):
    """max over Parameters of max |device - oracle| / (rtol x max(|oracle|_max, 1e-3 x largest)); <= 1 passes."""
    r, _ = _case(name)
    rtol = RTOL_INDUCING_SQRT if _has_sqrt_leaf(r["spec"]) else RTOL_INDUCING
    a = _inputs(name, entry)
    m, kp = _model(name, entry)
    val, grads = m.elbo_and_grad((a["X"], a["Y"])) if entry.startswith("svgp") else m.elbo_and_grad()
    ref_val, g = oracle(name, entry)
    np.testing.assert_allclose(float(val), ref_val, rtol=1e-8)
    ref = GC.leaf_grads_by_param(kp, g["leaves"])
    if entry == "svgp_gauss":
        ref[id(m.likelihood.variance)] = np.asarray(g["lik"])
    elif entry != "svgp_lik":
        ref[id(m.likelihood.variance)] = np.asarray(g["noise_variance"])
    elif isinstance(m.likelihood, gpf.likelihoods.StudentT):
        ref[id(m.likelihood.scale)] = np.asarray(g["lik"])
    if entry != "vgp":
        ref[id(m.inducing_variable.Z)] = g["Z"]
    if entry != "sgpr":
        ref[id(m.q_mu)], ref[id(m.q_sqrt)] = g["q_mu"], g["q_sqrt"]
    assert {id(p) for p in grads} == set(ref)
    top = max(float(np.max(np.abs(v))) for v in ref.values())
    worst = 0.0
    for p, v in grads.items():
        v = np.asarray(v, dtype=np.float64).reshape(p.shape)
        rr = ref[id(p)]
        _no_false_zeros(v, rr, (name, entry))
        bound = rtol * max(float(np.max(np.abs(rr))), 1e-3 * top)
        worst = max(worst, float(np.max(np.abs(v - rr))) / bound)
    return worst


@gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpr_matches_oracle_per_slot(cuda_device, name):
    assert _bar_ratio(name, "gpr") >= BAR
    assert gpr_error(name) <= 1.0


@gpu
@pytest.mark.parametrize("entry", ["sgpr", "svgp_gauss", "svgp_lik", "vgp"])
@pytest.mark.parametrize("name", NAMES)
def test_inducing_entries_match_oracle_per_parameter(cuda_device, name, entry):
    assert _bar_ratio(name, entry) >= BAR
    assert inducing_error(name, entry) <= 1.0


@gpu
@pytest.mark.parametrize("name", NAMES)
def test_cglb_matches_oracle_per_slot(cuda_device, name):
    """Every row through CGLB with a fixed trainable v (no CG): the low-rank N x N kernel LR = true of the row's GPR
    instantiation, its inducing-pass kernel, and P = 2 on every other row."""
    assert _bar_ratio(name, "cglb") >= BAR
    err = cglb_error(name)
    print(f"cglb {name}: worst |device - oracle| / (C S) = {err:.3g}")
    assert err <= 1.0


@gpu
@pytest.mark.parametrize("entry", ["sgpr", "svgp_gauss", "svgp_lik"])
def test_kuf_strips_of_several_column_tiles(cuda_device, entry):
    """N = 32900 against M = 45: each Kuf CTA walks two column tiles of X (the last one), in the instantiation that keeps
    dz in shared memory."""
    assert dispatch(STRIP["spec"], STRIP["D"])[1] == STRIP["ind"]
    assert _bar_ratio("strip", entry) >= BAR
    assert inducing_error("strip", entry) <= 1.0


# ---- checks without the oracle -------------------------------------------------------------------------------------
def _slot_scale(kp, g):
    return GC.leaf_grads_by_param(kp, g["leaves_abs"])


@gpu
@pytest.mark.parametrize("name", ["s8", "s16"])
def test_white_leaf_matches_the_same_noise(cuda_device, name):
    """k + White(w) with noise s against k with noise s + w: the same K, so the same gradient for every leaf of k, and
    d/dw = d/d(noise).  The White slot moves n_s from 8 to 9 or 16 to 17: two instantiations compared directly."""
    r, _ = _case(name)
    a = _inputs(name, "gpr")
    w = 0.07
    k1, _ = build(r["spec"])
    k2, _ = build(add(r["spec"], leaf("white", variance=w)))
    n_s = r["stage"][0]
    assert dispatch(add(r["spec"], leaf("white", variance=w)), r["D"])[0] == \
        f"gpr_grad_expr_kernel<{_bucket(n_s + 1)},0>" != r["gpr"]
    m1 = gpf.models.GPR((a["X"], a["Y"]), k1, noise_variance=S2 + w)
    m2 = gpf.models.GPR((a["X"], a["Y"]), k2, noise_variance=S2)
    l1, g1 = m1.log_marginal_likelihood_and_grad()
    l2, g2 = m2.log_marginal_likelihood_and_grad()
    np.testing.assert_allclose(float(l2), float(l1), rtol=1e-12)
    sc = _slot_scale(k1, oracle(name, "gpr")[1])
    for p1, p2 in zip(_params(k1), _params(k2)):
        d = np.abs(np.asarray(g1[p1]) - np.asarray(g2[p2])).reshape(p1.shape)
        assert np.all(d <= 1e-12 * sc[id(p1)]), (name, d / sc[id(p1)])
    white = GC.py_leaves(k2)[-1].variance
    gn = float(g1[m1.likelihood.variance])
    np.testing.assert_allclose(float(g2[white]), gn, rtol=1e-11)
    np.testing.assert_allclose(float(g2[m2.likelihood.variance]), gn, rtol=1e-11)


def _params(k):
    return [getattr(lf, a) for lf in GC.py_leaves(k) for a in GC.ATTRS if isinstance(getattr(lf, a, None), Parameter)]


@gpu
@pytest.mark.parametrize("name", ["d9_m12_ard", "d16_m32", "d17_m52", "d17_of_24_exp_ard", "d32_m32_ard"])
def test_bare_leaf_matches_the_leaf_under_a_one_child_sum(cuda_device, name):
    """gpr_grad_kernel<16 / 32> on a bare leaf against gpr_grad_expr_kernel on the same leaf wrapped in a one-child Sum:
    the same K and G, two reductions."""
    r, _ = _case(name)
    a = _inputs(name, "gpr")
    kb, _ = build(r["spec"])
    ks, _ = build(r["spec"])
    ks = K.Sum([ks])
    assert r["gpr"].startswith("gpr_grad_kernel<") and dispatch(("sum", [r["spec"]]), r["D"])[0].startswith(
        "gpr_grad_expr_kernel<")
    mb = gpf.models.GPR((a["X"], a["Y"]), kb, noise_variance=S2)
    ms = gpf.models.GPR((a["X"], a["Y"]), ks, noise_variance=S2)
    lb, gb = mb.log_marginal_likelihood_and_grad()
    ls, gs = ms.log_marginal_likelihood_and_grad()
    assert float(lb) == float(ls)
    sc = _slot_scale(kb, oracle(name, "gpr")[1])
    for pb, ps in zip(_params(kb), _params(ks)):
        d = np.abs(np.asarray(gb[pb]) - np.asarray(gs[ps])).reshape(pb.shape)
        assert np.all(d <= 1e-12 * sc[id(pb)]), (name, d / sc[id(pb)])
    noise_abs = oracle(name, "gpr")[1]["noise_abs"]
    assert abs(float(gb[mb.likelihood.variance]) - float(gs[ms.likelihood.variance])) <= 1e-12 * noise_abs


@gpu
@pytest.mark.parametrize("case", list(PAST))
def test_one_step_past_each_limit_is_refused_by_every_entry(cuda_device, case):
    """The library's refusal, as the ValueError every entry raises, from the host-side slot query that runs before the
    fused call (so before any kernel of the gradient)."""
    make, D, msg = PAST[case]
    d = O.make_data(3, 100, D, 1)
    X, Y = d["X"], d["Y"]
    Z = GC.z(20, D, 3)
    q_mu, q_sqrt = GC.q(20, 1, False, 3, upper_noise=False)
    calls = {
        "gpr": lambda: gpf.models.GPR((X, Y), make(), noise_variance=S2).log_marginal_likelihood_and_grad(),
        "sgpr": lambda: gpf.models.SGPR((X, Y), make(), Z.copy(), noise_variance=S2).elbo_and_grad(),
        "svgp": lambda: gpf.models.SVGP(make(), gpf.likelihoods.Gaussian(S2), Z.copy(), num_latent_gps=1,
                                        q_mu=q_mu.copy(), q_sqrt=q_sqrt.copy()).elbo_and_grad((X, Y)),
        "vgp": lambda: gpf.models.VGP((X, Y), make(), gpf.likelihoods.Gaussian(S2)).elbo_and_grad(),
    }
    for entry, call in calls.items():
        with pytest.raises(ValueError, match=msg) as e:
            call()
        assert str(e.value).startswith("gpk_gpr_lml_grad_slots: "), (entry, str(e.value))
