"""The likelihood bars of tests/lik_bounds.py, on the CPU: the exact oracle agrees with the float64 oracles where those
are accurate, a float64 emulation of the kernels' operation order lands inside every bar of the case table (the worst
ratio is printed), and each mutant in MUTATIONS, a subtly wrong kernel, falls outside at least one bar."""
import functools

import numpy as np
import pytest

from tests import hetero_oracle as HO
from tests import lik_bounds as LB
from tests import lik_oracle as LO
from tests import multiclass_oracle as MO

EPS = 1e-3    # RobustMax epsilon
CS = 1.7      # the adjoints' scale


@functools.lru_cache(maxsize=None)
def _exact_scalar(i):
    kind, par = LB.scalar_cases()[i]
    return LB.exact_scalar(kind, par, *LB.scalar_elements(kind))


@functools.lru_cache(maxsize=None)
def _exact_predict(i):
    kind, par = LB.scalar_cases()[i]
    return LB.exact_scalar_predict(kind, par, *LB.predict_elements(kind))


@functools.lru_cache(maxsize=None)
def _exact_mc(C):
    return LB.exact_mc(C, EPS, *LB.mc_rows(C))


def _ratio(got, want, bar):
    """|got - want| / bar per element (0 where equal, inf where a bar of 0 is missed or the values are not finite)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.abs(got - want) / bar
    r = np.where(got == want, 0.0, r)
    return np.where(np.isnan(r), np.inf, r)


def _scalar_ratios(i, mutation=None, table=None):
    kind, par = LB.scalar_cases()[i]
    y, mu, v = LB.scalar_elements(kind)
    em = LB.scalar_ve(kind, par, y, mu, v, mutation=mutation, table=table)
    ex = _exact_scalar(i)
    return {k: _ratio(em[k].v, ex[k], LB.bar(em[k])) for k in ("ve", "dmu", "dv", "dpar")}


def _predict_ratios(i):
    kind, par = LB.scalar_cases()[i]
    y, mu, v = LB.predict_elements(kind)
    ex = _exact_predict(i)
    m, var = LB.scalar_predict_mv(kind, par, mu, v)
    ld = LB.scalar_predict_ld(kind, par, y, mu, v)
    out = {"ld": _ratio(ld.v, ex["ld"], LB.bar(ld))}
    if kind != "student_t" or par["df"] > 2:
        out.update(mean=_ratio(m.v, ex["mean"], LB.bar(m)), var=_ratio(var.v, ex["var"], LB.bar(var)))
    return out


def _mc_ratios(C, mutation=None):
    y, mu, v = LB.mc_rows(C)
    g = LB.mc_grad(C, EPS, y, mu, v, CS, mutation=mutation)
    ex = _exact_mc(C)
    return {"R": _ratio(g["R"].v, CS * ex["R"], LB.bar(g["R"])), "W": _ratio(g["W"].v, CS * ex["W"], LB.bar(g["W"])),
            "ve": _ratio(g["ve"].v, ex["ve"], LB.bar(g["ve"])),
            "deps": _ratio(g["deps"].v, ex["deps"], LB.bar(g["deps"]))}


SCALAR_IDS = [LB.case_name(*c) for c in LB.scalar_cases()]


# ---- the oracle ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(LB.scalar_cases())), ids=SCALAR_IDS)
def test_exact_oracle_agrees_with_lik_oracle(i):
    kind, par = LB.scalar_cases()[i]
    rng = np.random.default_rng(3 + i)
    mu, v = rng.uniform(-2, 2, 40), rng.uniform(0.01, 1.5, 40)
    y = LO.targets(kind, mu, rng)
    lo = LO.make(kind, **{"gaussian": {"variance": par.get("noise")}, "poisson": {"binsize": par.get("binsize")},
                          "student_t": {"scale": par.get("scale"), "df": par.get("df")}}.get(kind, {}))
    ex = LB.exact_scalar(kind, par, y, mu, v)
    a = [x[:, None] for x in (mu, v, y)]
    np.testing.assert_allclose(ex["ve"], lo.variational_expectations(*a)[:, 0], rtol=1e-12, atol=1e-13)
    for key, want in zip(("dmu", "dv", "dpar"), lo.ve_grads(*a)):
        np.testing.assert_allclose(ex[key], want[:, 0], rtol=1e-11, atol=1e-12)
    pr = LB.exact_scalar_predict(kind, par, y, mu, v)
    np.testing.assert_allclose(pr["ld"], lo.predict_log_density(*a), rtol=1e-12, atol=1e-13)
    if kind != "student_t" or par["df"] > 2:
        wm, wv = lo.predict_mean_and_var(a[0], a[1])
        np.testing.assert_allclose(pr["mean"], wm[:, 0], rtol=1e-12, atol=1e-14)
        np.testing.assert_allclose(pr["var"], wv[:, 0], rtol=1e-11, atol=1e-14)


def test_exact_oracle_agrees_with_hetero_oracle():
    """A constant log-scale g = log(sqrt s) with v_g = 0 makes the heteroskedastic likelihood the Gaussian(s)."""
    rng = np.random.default_rng(5)
    s = 0.3
    mu, v, y = rng.standard_normal(30), rng.uniform(0.0, 2.0, 30), rng.standard_normal(30)
    ex = LB.exact_scalar("gaussian", {"noise": s}, y, mu, v)
    M = np.c_[mu, np.full(30, 0.5 * np.log(s))]
    V = np.c_[v, np.zeros(30)]
    h = HO.Hetero()
    np.testing.assert_allclose(ex["ve"], h.grid_ve(M, V, y[:, None]), rtol=1e-12)
    dmu, dv, _ = h.ve_grads(M, V, y[:, None])
    np.testing.assert_allclose(ex["dmu"], dmu[:, 0], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(ex["dv"], dv[:, 0], rtol=1e-12)


@pytest.mark.parametrize("C", [3, 33])
def test_exact_oracle_agrees_with_multiclass_oracle(C):
    rng = np.random.default_rng(C)
    mu, v = 0.6 * rng.standard_normal((6, C)), rng.uniform(0.05, 1.0, (6, C))
    y = np.array([0.0, 1.0, C - 1.0, C + 1.0, 2.5, -0.5])
    ex = LB.exact_mc(C, EPS, y, mu, v)
    mo = MO.MultiClass(C, EPS)
    dmu, dv, deps = mo.ve_grads(mu, v, y[:, None])
    np.testing.assert_allclose(ex["p"], mo.prob_is_largest(y[:, None], mu, v), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(ex["ve"], mo.variational_expectations(mu, v, y[:, None]), rtol=1e-12)
    np.testing.assert_allclose(ex["ld"], mo.predict_log_density(mu, v, y[:, None]), rtol=1e-12)
    np.testing.assert_allclose(ex["deps"], deps, rtol=1e-12)
    for got, want in ((ex["R"], dmu), (ex["W"], dv)):
        np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-12 * np.max(np.abs(want)))


@pytest.mark.parametrize("C", LB.MC_CLASSES)
def test_float64_multiclass_oracle_is_inside_the_bars(C):
    """The GPU test holds the predictive class probabilities, which need p at every label, against the float64
    oracle within twice the bar; that oracle's p is inside one bar at every label of the case table."""
    y, mu, v = LB.mc_rows(C)
    mo = MO.MultiClass(C, EPS)
    p = LB.mc_prob(C, LB.mc_label(y, C), mu, v)["p"]
    r = _ratio(mo.prob_is_largest(y[:, None], mu, v), _exact_mc(C)["p"], LB.bar(p))
    assert r.max() <= 1.0, r.max()


# ---- soundness -----------------------------------------------------------------------------------------------------
def test_emulation_inside_every_bar():
    worst = {}
    for i, name in enumerate(SCALAR_IDS):
        for k, r in _scalar_ratios(i).items():
            worst[f"{name} {k}"] = r.max()
        for k, r in _predict_ratios(i).items():
            worst[f"{name} predict {k}"] = r.max()
    for C in LB.MC_CLASSES:
        for k, r in _mc_ratios(C).items():
            worst[f"multiclass C={C} {k}"] = r.max()
    print("\nworst |emulation - exact| / bar:")
    for k, r in worst.items():
        print(f"  {k:48s} {r:.3g}")
    bad = {k: r for k, r in worst.items() if not r <= 1.0}
    assert not bad, bad


# ---- sharpness -----------------------------------------------------------------------------------------------------
def _swap(a, i, j):
    a = a.copy()
    a[[i, j]] = a[[j, i]]
    return a


def _scalar_mutant(table=None, mutation=None, kinds=None, keys=("ve", "dmu", "dv", "dpar")):
    worst = 0.0
    for i, (kind, _) in enumerate(LB.scalar_cases()):
        if kinds and kind not in kinds:
            continue
        r = _scalar_ratios(i, mutation=mutation, table=table)
        worst = max(worst, max(r[k].max() for k in keys))
    return worst


def _wt_layout_mutant():
    """lik_grad_kernel writing Wt[b P + p] (the layout of R) instead of Wt[p B + b], read back as [P][B]."""
    worst = 0.0
    for i, (kind, par) in enumerate(LB.scalar_cases()):
        y, mu, v = LB.scalar_elements(kind)
        for P in (3, 7):
            B = len(y) // P
            em = LB.scalar_ve(kind, par, y[:B * P], mu[:B * P], v[:B * P])["dv"]
            ex = _exact_scalar(i)["dv"][:B * P]
            got = em.v.reshape(B, P).reshape(-1).reshape(P, B).T.reshape(-1)   # [B][P] memory read as [P][B]
            worst = max(worst, _ratio(got, ex, LB.bar(em)).max())
    return worst


def _fp32_arith_mutant():
    """The prediction operators with fp32 arithmetic, against the fp32 bar at fp32-rounded inputs."""
    worst = 0.0
    for i, (kind, par) in enumerate(LB.scalar_cases()):
        if kind == "student_t" and par["df"] <= 2:
            continue
        y, mu, v = (np.float32(a).astype(np.float64) for a in LB.predict_elements(kind))
        keep = np.abs(mu) + np.sqrt(v) * LB.GH_Z[-1] < 40.0
        y, mu, v = y[keep], mu[keep], v[keep]
        ex = LB.exact_scalar_predict(kind, par, y, mu, v)
        m64, v64 = LB.scalar_predict_mv(kind, par, mu, v)
        with LB.arithmetic(np.float32):
            m32, v32 = LB.scalar_predict_mv(kind, par, mu, v)
        for got, ref, key in ((m32, m64, "mean"), (v32, v64, "var")):
            worst = max(worst, _ratio(got.v, ex[key], LB.round32_bar(ex[key], LB.bar(ref))).max())
    return worst


MUTATIONS = {
    "node weight zeroed": lambda: _scalar_mutant(table=(LB.GH_Z, np.r_[0.0, LB.GH_W[1:]]),
                                                 kinds=("bernoulli", "student_t")),
    "two nodes swapped": lambda: _scalar_mutant(table=(_swap(LB.GH_Z, 8, 9), LB.GH_W), kinds=("bernoulli", "student_t")),
    "dv without the 1/2": lambda: _scalar_mutant(mutation="dv_no_half", keys=("dv",)),
    "v = 0 as 0/0": lambda: _scalar_mutant(mutation="no_v0_limit", keys=("dv",)),
    "Student-t dscale without -1/scale": lambda: _scalar_mutant(mutation="dscale_no_inv_scale", kinds=("student_t",),
                                                                keys=("dpar",)),
    "Wt stored [B][P]": _wt_layout_mutant,
    "after product missing the last chunk": lambda: max(_mc_ratios(C, "after_missing_last")["R"].max()
                                                        for C in LB.MC_CLASSES if C > 64),
    "E with its own cdf at lane 0": lambda: max(max(_mc_ratios(C, "own_cdf_lane0")[k].max() for k in ("R", "W"))
                                                for C in LB.MC_CLASSES),
    "E with its own cdf at lane 31": lambda: max(max(_mc_ratios(C, "own_cdf_lane31")[k].max() for k in ("R", "W"))
                                                 for C in LB.MC_CLASSES if C >= 32),
    "W_c clamp dropped": lambda: max(_mc_ratios(C, "no_w_clamp")["W"].max() for C in LB.MC_CLASSES),
    "s_y from v_y, not 2 v_y": lambda: max(_mc_ratios(C, "s_y_v")["ve"].max() for C in LB.MC_CLASSES),
    "fp32 predictions in fp32 arithmetic": _fp32_arith_mutant,
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_mutation_falls_outside_a_bar(name):
    worst = MUTATIONS[name]()
    print(f"\n{name}: worst |mutant - exact| / bar = {worst:.3g}")
    assert worst > 1.0, (name, worst)
