"""CPU self-checks of tests/kaux_bounds.py: the intervals of the materialised kernels and their compositions agree with
oracle/gp_oracle.py, a NumPy emulation of kaux_eval in the device's operation order lies inside every bar, and named
mutants of that emulation fall outside the bar meant to catch them."""
import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O
from tests import kaux_bounds as KA
from tests import kbuild_bounds as KB

f32, f64 = np.float32, np.float64
BASE_CLS = {_lib.K_RBF: "SquaredExponential", _lib.K_RQ: "RationalQuadratic", _lib.K_EXPONENTIAL: "Exponential",
            _lib.K_MATERN12: "Matern12", _lib.K_MATERN32: "Matern32", _lib.K_MATERN52: "Matern52"}


def inputs(D, dtype, seed, n=60, n2=45):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D)) * 1.5
    X[5] = X[4]                                   # coincident pair
    X[7] = X[6] + 1e-7 * rng.standard_normal(D)   # nearly coincident
    X[9] = -X[8]                                  # opposite directions (ArcCosine c near -1 for small bias)
    X[10] = 40.0 * X[3]                           # large |s| (Cosine), long arguments (Periodic)
    X2 = rng.standard_normal((n2, D)) * 1.5
    X2[0] = X[4]
    return X.astype(dtype), X2.astype(dtype)


def kaux_kernels(mod, D):
    """(name, kernel) of every materialised leaf configuration the tests use, in module `mod`."""
    ls = 0.7 + np.arange(D) * 0.3
    out = [("cosine", mod.Cosine(variance=1.2, lengthscales=ls)),
           ("cosine_iso", mod.Cosine(variance=0.8, lengthscales=2.3))]
    for b, cls in BASE_CLS.items():
        kw = {"alpha": 2.5} if b == _lib.K_RQ else {}
        base = getattr(mod, cls)(variance=1.1, lengthscales=ls * 0.9, **kw)
        out.append((f"periodic_{KB.FUSED_NAMES[b]}", mod.Periodic(base, period=1.0 + 0.5 * np.arange(D))))
    for order in (0, 1, 2):
        out.append((f"arccos{order}", mod.ArcCosine(order=order, variance=0.9, weight_variances=0.5 + 0.2 * np.arange(D),
                                                    bias_variance=0.3)))
    return out


def oracle_pair(D, dtype):
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        g = kaux_kernels(gpf.kernels, D)
    o = kaux_kernels(O, D)
    return [(n, kg, ko) for (n, kg), (_, ko) in zip(g, o)]


@pytest.mark.parametrize("dtype", [f64, f32], ids=["f64", "f32"])
def test_kaux_intervals_agree_with_oracle_and_hold_for_emulation(dtype):
    D = 3
    X, X2 = inputs(D, dtype, 1)
    worst = {}
    for name, kg, ko in oracle_pair(D, dtype):
        p = KA.params(kg, D)
        for Xb in (X2, None):
            cen, lo, hi = KA.kaux_interval(p, X, Xb, dtype)
            assert np.all(lo <= cen) and np.all(cen <= hi), name
            em = KA.emulate_kaux(p, X, Xb, dtype).astype(f64)
            ok = (em >= lo) & (em <= hi)
            assert ok.all(), (name, np.argwhere(~ok)[:3], float(KB.ratio(em, cen, lo, hi).max()))
            worst[name] = max(worst.get(name, 0.0), float(KB.ratio(em, cen, lo, hi).max()))
            if dtype == f64:
                # The oracle (fp64, its own operation order) lies inside the kernel's bar.  This is the independent
                # check that the descriptor's scales, periods, bias and variance are the oracle's hyperparameters: a
                # descriptor off by 1e-9 relative in one scale leaves the bar.
                orc = ko(X, Xb)
                assert np.all((orc >= lo) & (orc <= hi)), (name, float(KB.ratio(orc, cen, lo, hi).max()))
                off = KA.params(kg, D)
                off.scale = off.scale * np.array([1.0 + 1e-9] + [1.0] * (len(off.scale) - 1))
                oc, ol, oh = KA.kaux_interval(off, X, Xb, dtype)
                assert np.any((orc < ol) | (orc > oh)), name
        c, lo, hi = KA.kaux_diag_interval(p, X, dtype)
        em = KA.emulate_kaux(p, X, None, dtype)
        if dtype == f64:
            orc = ko(X, full_cov=False)
            assert np.all(np.abs(orc - c) <= (hi - lo) + 2 * KB.unit(dtype) * np.abs(c)), name
        if not name.startswith("arccos"):  # ArcCosine's K(x, x) carries the jitter, its K_diag does not (as in GPflow)
            kc = KA.kaux_interval(p, X, None, dtype)
            assert np.all(np.abs(np.diag(kc[0]) - c) <= np.diag(kc[2] - kc[1]) + (hi - lo) + 1e-300), name
            assert np.all((np.diag(em) >= lo) & (np.diag(em) <= hi)), name
    print(f"[emulation] kaux {np.dtype(dtype).name}: worst ratio " + " ".join(f"{k} {v:.3g}" for k, v in worst.items()))


def test_cosine_bar_grows_with_s():
    """The absolute half-width of Cosine grows with |s|: the far row 10 has a wider bar than row 3."""
    X, _ = inputs(3, f64, 1)
    with gpf.config.as_context(gpf.config.Config(float=f64)):
        p = KA.params(gpf.kernels.Cosine(variance=1.0, lengthscales=0.9), 3)
    cen, lo, hi = KA.kaux_interval(p, X, None, f64)
    assert (hi - lo)[10].max() > 10 * (hi - lo)[3].max()


def coregion_kernel(O_dim=4):
    k = gpf.kernels.Coregion(output_dim=O_dim, rank=2)
    k.W.assign(np.arange(O_dim * 2, dtype=np.float64).reshape(O_dim, 2) * 0.37 - 1.0)
    k.kappa.assign(0.5 + np.arange(O_dim, dtype=np.float64))
    return k


COREG_X = np.array([0.0, 1.0, 1.7, -0.5, 3.0, 3.99, -1.0, 4.0, np.nan, 2.2, 1e10, -0.999])


@pytest.mark.parametrize("dtype", [f64, f32], ids=["f64", "f32"])
def test_coregion_reference(dtype):
    """Indices truncate toward zero (1.7 -> 1, -0.5 -> 0); -1, 4 = O, NaN and 1e10 give NaN; the table entry is the fp64
    entry rounded once.  The oracle (tf.cast semantics) agrees on every valid index."""
    k = coregion_kernel()
    p = KA.params(k, 1)
    X = COREG_X[:, None].astype(dtype)
    v = KA.coregion_value(p, X, None, dtype)
    idx = KA.coregion_index(X[:, 0], 4)
    assert list(idx) == [0, 1, 1, 0, 3, 3, -1, -1, -1, 2, -1, 0]
    bad = idx < 0
    assert np.all(np.isnan(v[bad, :])) and np.all(np.isnan(v[:, bad]))
    ok = ~bad
    ko = O.Coregion(4, 2, W=k.W.numpy(), kappa=k.kappa.numpy())
    orc = ko(X[ok].astype(f64))
    assert np.array_equal(v[np.ix_(ok, ok)], orc.astype(dtype))
    d, _, _ = KA.kaux_diag_interval(p, X, dtype)
    assert np.array_equal(d[ok], ko(X[ok].astype(f64), full_cov=False).astype(dtype).astype(f64))
    assert np.all(np.isnan(d[bad]))


def changepoints(mod, dtype):
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        ks = [mod.SquaredExponential(variance=1.2, lengthscales=0.8), mod.Linear(variance=0.3),
              mod.Matern32(variance=0.7, lengthscales=1.5)]
        if mod is O:
            return O.ChangePoints(ks, locations=[-0.5, 1.0], steepness=np.array([4.0, 30.0]))
        return mod.ChangePoints(ks, locations=[-0.5, 1.0], steepness=[4.0, 30.0])


@pytest.mark.parametrize("dtype", [f64, f32], ids=["f64", "f32"])
def test_changepoints_interval(dtype):
    """ChangePoints through the weights' exact sigmoid form: the oracle (fp64) and the emulation lie in the interval;
    the weights cover each has_lo / has_hi combination, including 1 - sigma cancelling at steepness 30."""
    rng = np.random.default_rng(2)
    X = np.sort(rng.uniform(-3, 3, 50))[:, None].astype(dtype)
    X2 = rng.uniform(-3, 3, 31)[:, None].astype(dtype)
    kg, ko = changepoints(gpf.kernels, dtype), changepoints(O, dtype)
    for Xb in (X2, None):
        cen, lo, hi = KA.kernel_interval(kg, X, Xb, dtype)
        em = KA.emulate_changepoints(kg, X, Xb, dtype).astype(f64)
        assert np.all((em >= lo) & (em <= hi)), float(KB.ratio(em, cen, lo, hi).max())
        if dtype == f64:
            assert np.allclose(ko(X, Xb), cen, rtol=1e-12, atol=1e-14)
    c, lo, hi = KA.kernel_interval(kg, X, None, dtype, full_cov=False)
    assert np.all((lo <= c) & (c <= hi))
    if dtype == f64:
        assert np.allclose(ko(X, full_cov=False), c, rtol=1e-12, atol=1e-14)
    for has in ((0, 1), (1, 1), (1, 0), (0, 0)):
        a = KA.cp_weight_interval(X[:, 0], has[0], -0.5, 4.0, has[1], 1.0, 30.0, dtype)
        assert np.all((a[1] <= a[0]) & (a[0] <= a[2]))


def test_composition_intervals_agree_with_oracle():
    """Sum / Product with materialised children, including the coregionalisation pattern Coregion[1] * RBF[0]."""
    rng = np.random.default_rng(4)
    X = np.concatenate([rng.standard_normal((40, 1)), rng.integers(0, 3, (40, 1))], 1)
    X2 = np.concatenate([rng.standard_normal((25, 1)), rng.integers(0, 3, (25, 1))], 1)
    cg = coregion_kernel(3)
    cg.active_dims = [1]
    rbf = gpf.kernels.SquaredExponential(variance=1.3, lengthscales=0.7, active_dims=[0])
    per = gpf.kernels.Periodic(gpf.kernels.Matern52(variance=0.6, lengthscales=1.1, active_dims=[0]), period=2.0)
    co = O.Coregion(3, 2, W=cg.W.numpy(), kappa=cg.kappa.numpy(), active_dims=[1])
    ro = O.SquaredExponential(variance=1.3, lengthscales=0.7, active_dims=[0])
    po = O.Periodic(O.Matern52(variance=0.6, lengthscales=1.1, active_dims=[0]), period=2.0)
    for kg, ko in ((gpf.kernels.Product([cg, rbf]), O.Product([co, ro])),
                   (gpf.kernels.Sum([per, rbf, gpf.kernels.White(variance=0.1)]), O.Sum([po, ro, O.White(variance=0.1)]))):
        for Xb in (X2, None):
            cen, lo, hi = KA.kernel_interval(kg, X, Xb, f64)
            orc = ko(X, Xb)
            assert np.all((orc >= lo) & (orc <= hi)), float(KB.ratio(orc, cen, lo, hi).max())


# ---- mutants ---------------------------------------------------------------------------------------------------------
def _outside(em, cen, lo, hi):
    em = np.asarray(em, f64)
    return ~((em >= lo) & (em <= hi))


KAUX_MUTANTS = {
    # mutant: (kernel name, dtype)
    "periodic_sin2": ("periodic_m32", f64),
    "arccos_no_jitter": ("arccos0", f64),
    "in_float": ("cosine", f32),
    "cosine_no_2": ("cosine_iso", f64),
}


@pytest.mark.parametrize("mutant", list(KAUX_MUTANTS))
def test_kaux_mutants_fall_outside(mutant):
    name, dtype = KAUX_MUTANTS[mutant]
    D = 3
    X, X2 = inputs(D, dtype, 1)
    kg = dict((n, k) for n, k, _ in oracle_pair(D, dtype))[name]
    p = KA.params(kg, D)
    Xb = None if mutant == "arccos_no_jitter" else X2
    cen, lo, hi = KA.kaux_interval(p, X, Xb, dtype)
    em = KA.emulate_kaux(p, X, Xb, dtype, mutant=mutant)
    out = _outside(em, cen, lo, hi)
    print(f"[mutant] {mutant}: {int(out.sum())} elements outside")
    assert out.any()
    if mutant == "arccos_no_jitter":     # the jitter shows at the coincident points (the diagonal, rows 4 / 5)
        assert out[np.arange(X.shape[0]), np.arange(X.shape[0])].any()


def test_kaux_fp32_in_float_outside_for_every_op():
    """fp32 kaux computed in float instead of fp64 leaves every op's bar (Coregion has no arithmetic)."""
    D = 3
    X, X2 = inputs(D, f32, 1)
    for name in ("cosine", "periodic_rbf", "periodic_m52", "arccos1"):
        kg = dict((n, k) for n, k, _ in oracle_pair(D, f32))[name]
        p = KA.params(kg, D)
        cen, lo, hi = KA.kaux_interval(p, X, X2, f32)
        assert _outside(KA.emulate_kaux(p, X, X2, f32, mutant="in_float"), cen, lo, hi).any(), name


def test_coregion_round_to_nearest_falls_outside():
    k = coregion_kernel()
    p = KA.params(k, 1)
    X = COREG_X[:, None]
    good = KA.coregion_value(p, X, None, f64)
    bad = KA.emulate_kaux(p, X, None, f64, mutant="coregion_nearest")
    assert np.array_equal(KA.emulate_kaux(p, X, None, f64), good, equal_nan=True)
    assert not np.array_equal(bad, good, equal_nan=True)


def test_changepoints_x_weights_on_x2_columns_falls_outside():
    rng = np.random.default_rng(2)
    X = np.sort(rng.uniform(-3, 3, 50))[:, None]
    X2 = rng.uniform(-3, 3, 31)[:, None]
    kg = changepoints(gpf.kernels, f64)
    cen, lo, hi = KA.kernel_interval(kg, X, X2, f64)
    assert not _outside(KA.emulate_changepoints(kg, X, X2, f64), cen, lo, hi).any()
    out = _outside(KA.emulate_changepoints(kg, X, X2, f64, mutant="x_weights_on_cols"), cen, lo, hi)
    print(f"[mutant] changepoints x_weights_on_cols: {int(out.sum())} elements outside")
    assert out.any()
