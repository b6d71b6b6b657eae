"""Element-wise accuracy of the covariance functions beyond the stationary fast path, against the per-element intervals
of tests/kbuild_bounds.py (every fused leaf, K_diag) and tests/kaux_bounds.py (the materialised kernels and their
compositions).

1. The generic K-build (`kbuild_kernel<T, NG>`) in fp32 / fp64 x symmetric full / lower (with the diagonal shift),
   rectangular and rectangular with X2 = X, for RationalQuadratic (alpha 0.1 .. 1e3), Polynomial (degrees 1-4, ARD,
   offsets that cancel), Constant, White, ARD Linear, Sum / Product trees of depth 4 over 2-4 gram groups, expressions
   without a gram leaf, and 12 leaves.  Outputs are views with an odd (unaligned stores) or a 16-byte multiple
   (vector stores) leading dimension inside NaN-filled parents: the guards stay bit-unchanged.  Constant and White are
   bit-exact.  A second run is bit-identical.
2. K_diag (`kdiag_kernel<T>`) against its interval and against the diagonal of K(X).
3. The expression limits: 12 leaves and a four-entry evaluation stack are accepted, 13 leaves and a fifth level are
   refused.  A mirror of the dispatch checks that the table reaches every instantiation.
4. `gpk_kaux` / `gpk_kaux_diag` for Cosine, Periodic over all six bases, ArcCosine of orders 0-2 and Coregion
   (truncated, out-of-range and NaN indices), `gpk_changepoint_weights` for each has_lo / has_hi combination, and the
   compositions through the public K / K_diag (ChangePoints, Coregion[1] * RBF[0], Periodic + fused leaves).
5. `gpk_kmv` with RationalQuadratic, Polynomial, Constant and White leaves.
6. K(X, X2) with 4,194,241 rows in X (one more than 65535 tiles of 64 rows) for a generic expression and a Periodic."""
import functools

import numpy as np
import pytest

import gpflow_b200 as gpf
from gpflow_b200 import _lib, ops
from tests import kaux_bounds as KA
from tests import kbuild_bounds as B

pytestmark = pytest.mark.gpu

f32, f64 = np.float32, np.float64
DT = {"f64": f64, "f32": f32}
FORMS = ("full", "lower", "rect", "rect_xx")
WORST = {}


def _torch():
    import torch

    return torch


def tdt(dtype):
    return _torch().float64 if dtype == f64 else _torch().float32


def cfg(dtype):
    return gpf.config.as_context(gpf.config.Config(float=dtype))


# ---- expressions ---------------------------------------------------------------------------------------------------
def expr(name, dtype, D):
    """Fused kernel expressions of the case table (D >= 6)."""
    K = gpf.kernels
    rng = np.random.default_rng(sum(map(ord, name)))
    ard = 0.5 + rng.random(D)
    with cfg(dtype):
        if name == "rq_ard":
            return K.RationalQuadratic(variance=0.8, lengthscales=2.0 * ard, alpha=2.5)
        if name.startswith("rq_a"):
            return K.RationalQuadratic(variance=1.3, lengthscales=1.1 * np.sqrt(D), alpha=float(name[4:]))
        if name == "poly_ard":
            return K.Polynomial(degree=3.0, variance=0.3 * ard, offset=1.3)
        if name.startswith("poly_d"):
            return K.Polynomial(degree=float(name[6:]), variance=0.4, offset=0.7)
        if name == "lin_ard":
            return K.Linear(variance=0.3 * ard)
        if name == "const":
            return K.Constant(variance=0.9)
        if name == "white":
            return K.White(variance=0.45)
        if name == "const_white":      # no gram leaf at all: NG = 1 with zero groups
            return K.Sum([K.Constant(variance=0.9), K.White(variance=0.45)])
        if name == "white_x_lin":
            return K.Product([K.White(variance=0.6), K.Linear(variance=0.5)])
        if name == "rbf_white":        # an SGPR / SVGP Kuu with jitter as a White leaf
            return K.Sum([K.SquaredExponential(variance=1.1, lengthscales=1.4 * np.sqrt(D)), K.White(variance=1e-3)])
        if name.startswith("tree"):    # depth-4 Sum / Product trees over `g` gram groups
            g = int(name[4:])
            a = K.RationalQuadratic(variance=0.9, lengthscales=1.3 * np.sqrt(D), alpha=1.5, active_dims=list(range(D)))
            b = K.Polynomial(degree=2.0, variance=0.2, offset=1.0, active_dims=list(range(D)))
            c = K.Linear(variance=0.2 * ard)
            d = K.Matern32(variance=0.5, lengthscales=ard[:D - 2] * 2.0, active_dims=list(range(2, D)))
            e = K.Polynomial(degree=3.0, variance=0.1 * ard[:3], offset=0.5, active_dims=[0, 2, 4])
            w, k = K.White(variance=0.05), K.Constant(variance=0.3)
            leaves = [a, b, c, d, e][:{2: 3, 3: 4, 4: 5}[g]]
            inner = K.Product([K.Sum([leaves[0], k]), leaves[1]])
            rest = K.Sum([K.Product([inner, leaves[2]]), w] + ([K.Product([leaves[3], k])] if g >= 3 else []))
            return K.Sum([rest, leaves[4]]) if g == 4 else rest
        if name == "leaves12":         # KB_MAXL = 12 leaves, two gram groups
            ls = [K.RationalQuadratic(variance=0.1 * (i + 1), lengthscales=2.0 * np.sqrt(D), alpha=0.5 + i)
                  for i in range(4)]
            ps = [K.Polynomial(degree=1.0 + i % 3, variance=0.05, offset=0.5) for i in range(3)]
            st = [K.Constant(variance=0.2), K.White(variance=0.1), K.Linear(variance=0.1 * ard),
                  K.Constant(variance=0.05), K.White(variance=0.02)]
            return K.Sum([K.Product([ls[0], ps[0]]), K.Sum(ls[1:] + ps[1:]), K.Sum(st)])
    raise KeyError(name)


LEAF_EXPRS = (["rq_a0.1", "rq_a1", "rq_a2.5", "rq_a1000", "rq_ard", "poly_d1", "poly_d2", "poly_d3", "poly_d4",
               "poly_ard", "lin_ard", "const", "white", "const_white", "white_x_lin", "rbf_white"])
COMPOSITE_EXPRS = ["tree2", "tree3", "tree4", "leaves12"]
EXPRS = LEAF_EXPRS + COMPOSITE_EXPRS


def compiled(name, dtype, D):
    return gpf.kernels.compile_kernel(expr(name, dtype, D), D)


def n_groups(desc, D):
    """The gram groups compile_kprog forms: distinct (active dims, weight mode, weights) over the gram leaves."""
    nodes, n, dims, ard = desc
    seen = []
    for i in range(n):
        nd = nodes[i]
        if nd.op in (_lib.K_SUM, _lib.K_PRODUCT, _lib.K_WHITE, _lib.K_CONSTANT):
            continue
        cols, par = B._leaf_inputs(nd, dims, ard, D)
        lin = nd.op in (_lib.K_LINEAR, _lib.K_POLYNOMIAL)
        mode = 0 if nd.n_ard == 0 else (1 if lin else 2)
        w = tuple(par if nd.n_ard > 0 and lin else (1.0 / par if nd.n_ard > 0 else np.ones(len(cols))))
        key = (tuple(cols), mode, w)
        if key not in seen:
            seen.append(key)
    return len(seen)


def leaf_types(desc):
    nodes, n = desc[0], desc[1]
    return {nodes[i].op for i in range(n) if nodes[i].op not in (_lib.K_SUM, _lib.K_PRODUCT)}


def fast_path(desc):
    nodes, n = desc[0], desc[1]
    return n == 1 and nodes[0].op in B.STATIONARY


# ---- inputs and the guarded launch ---------------------------------------------------------------------------------
def case_inputs(name, dtype, N, N2, D, ldx):
    rng = np.random.default_rng(sum(map(ord, name)) + N)
    X = rng.standard_normal((N, D)) * 0.8 + 0.3
    X[5] = X[4]
    X[7] = X[6] + 1e-6 * rng.standard_normal(D)
    X2 = rng.standard_normal((N2, D)) * 0.8
    if name.startswith("poly"):  # var <x, x'> + offset cancels to near 0 against X2's row 3
        X[11] = -X2[3] * (0.7 / 0.4) / np.dot(X2[3], X2[3])
    Xp = np.full((N, ldx), np.nan)
    Xp[:, :D] = X
    return X.astype(dtype), X2.astype(dtype), Xp.astype(dtype)


SENT = float("nan")


def vec_ok(view):
    """kbuild_launch's test for the 16-byte vector stores: an aligned base and a leading dimension of 16-byte rows."""
    es = view.element_size()
    return view.data_ptr() % 16 == 0 and (view.stride(0) * es) % 16 == 0


def run_kbuild(desc, dtype, form, X, X2, Xp, odd, dvec=None, dsc=0.0):
    """K into a view of a NaN-filled parent: odd, an odd leading dimension starting at column 1 (element-wise stores);
    else a leading dimension of whole 16-byte units starting at column 0 of row 1 (vector stores).  Returns (K as fp64
    NumPy, guards kept, second run bit-identical)."""
    T = _torch()
    N, D = X.shape
    N2 = N if form in ("full", "lower", "rect_xx") else X2.shape[0]
    ld = N2 + (3 if N2 % 2 == 0 else 2) if odd else (N2 + 3) // 4 * 4 + 4
    parent = T.full((N + 2, ld), SENT, dtype=tdt(dtype), device="cuda")
    c0 = 1 if odd else 0
    view = parent[1:N + 1, c0:c0 + N2]
    assert vec_ok(view) == (not odd), "the view does not select the store path the case names"
    Xd = T.from_numpy(Xp).cuda()[:, :D]
    X2d = None if form in ("full", "lower") else (Xd if form == "rect_xx" else T.from_numpy(X2).cuda())
    uplo = _lib.GPK_LOWER if form == "lower" else _lib.GPK_FULL
    dv = None if dvec is None else T.from_numpy(dvec.astype(dtype)).cuda()
    with cfg(dtype):
        ops.kbuild(desc, Xd, X2d, uplo=uplo, diag_scalar=dsc, diag_vec=dv, out=view)
        first = parent.clone()
        ops.kbuild(desc, Xd, X2d, uplo=uplo, diag_scalar=dsc, diag_vec=dv, out=view)
    T.cuda.synchronize()
    rest = parent.clone()
    rest[1:N + 1, c0:c0 + N2] = 0
    guards = bool(T.all(T.isnan(rest) | (rest == 0)).item()) and int((rest == 0).sum()) == N * N2
    same = bool(T.equal(T.nan_to_num(first, nan=-7.0), T.nan_to_num(parent, nan=-7.0)))
    return view.cpu().numpy().astype(f64), guards, same


def fused_interval(desc, dtype, form, X, X2, dvec=None, dsc=0.0):
    Xb = {"full": None, "lower": None, "rect": X2, "rect_xx": X}[form]
    cen, lo, hi = B.expr_interval(desc, X, Xb, dtype=dtype, sym=form in ("full", "lower"))
    if form in ("full", "lower") and (dsc != 0.0 or dvec is not None):
        n = X.shape[0]
        shift = np.zeros(n) + dsc + (0.0 if dvec is None else dvec.astype(dtype).astype(f64))
        u = B.unit(dtype)
        I = np.arange(n)
        m = 2 * u * (np.maximum(np.abs(lo), np.abs(hi))[I, I] + shift)
        cen, lo, hi = cen.copy(), lo.copy(), hi.copy()
        cen[I, I] += shift
        lo[I, I] += shift - m
        hi[I, I] += shift + m
    return cen, lo, hi


def note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def worst_ratios():
    """After the module: the worst |device - reference| / bar per leaf / op and dtype over the tests that ran."""
    yield
    for (k, d), v in sorted(WORST.items(), key=lambda kv: (str(kv[0][0]), kv[0][1])):
        print(f"[worst] {k} {d}: {v:.3g}")


# ---- 1. the case table ---------------------------------------------------------------------------------------------
CASE_SHAPES = {  # (N, N2, D, ldx, odd output)
    "f64": (133, 70, 7, 9, True),
    "f32": (150, 67, 9, 9, False),
}


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("dname", ["f64", "f32"])
@pytest.mark.parametrize("name", EXPRS)
def test_fused_leaf_within_interval(cuda_device, name, dname, form):
    dtype = DT[dname]
    N, N2, D, ldx, odd = CASE_SHAPES[dname]
    if form in ("full", "rect_xx"):
        odd = not odd                    # both store paths in every dtype
    X, X2, Xp = case_inputs(name, dtype, N, N2, D, ldx + (2 if form == "lower" else 0))
    desc = compiled(name, dtype, D)
    assert not fast_path(desc)
    dvec = 0.1 + np.random.default_rng(1).random(N) if form == "lower" else None
    dsc = {"lower": 0.25, "full": 0.5}.get(form, 0.0)
    dev, guards, same = run_kbuild(desc, dtype, form, X, X2, Xp, odd, dvec, dsc)
    assert guards, "a store left the output view"
    assert same, "a second run is not bit-identical"
    cen, lo, hi = fused_interval(desc, dtype, form, X, X2, dvec, dsc)
    mask = np.tril(np.ones_like(dev, bool)) if form == "lower" else np.ones_like(dev, bool)
    ok = (dev >= lo) & (dev <= hi)
    bad = np.argwhere(mask & ~ok)
    assert len(bad) == 0, [(int(i), int(j), dev[i, j], lo[i, j], hi[i, j]) for i, j in bad[:4]]
    r = float(B.ratio(dev, cen, lo, hi)[mask].max())
    note((name, dname), r)
    if name in ("const", "white", "const_white"):
        # bit-exact: T(var) combined in the dtype, on the diagonal of the symmetric forms plus fl(T(dsc) + dvec_i)
        exact = KA.emulate_kbuild(desc, X, {"rect": X2, "rect_xx": X}.get(form), dtype, sym=form in ("full", "lower"))
        if form in ("full", "lower"):
            Tt = np.dtype(dtype).type
            shift = Tt(dsc) + (dvec.astype(dtype) if dvec is not None else np.zeros(N, dtype))
            I = np.arange(N)
            exact[I, I] = exact[I, I] + shift.astype(dtype)
        assert np.array_equal(dev[mask], exact.astype(f64)[mask]), "Constant / White must be bit-exact"
        if name == "white":
            off = mask & ~np.eye(N, dev.shape[1], dtype=bool)
            assert np.all(dev[off] == 0) and not np.signbit(dev[off]).any(), "White must be +0 off the diagonal"
    print(f"[fused] {name} {dname} {form}: max error / bar {r:.3g}")


@pytest.mark.parametrize("dname", ["f64", "f32"])
@pytest.mark.parametrize("name", EXPRS)
def test_kdiag_within_interval(cuda_device, name, dname):
    dtype = DT[dname]
    N, N2, D, ldx, _ = CASE_SHAPES[dname]
    X, X2, Xp = case_inputs(name, dtype, N, N2, D, ldx)
    desc = compiled(name, dtype, D)
    T = _torch()
    Xd = T.from_numpy(Xp).cuda()[:, :D]
    parent = T.full((N + 3,), SENT, dtype=tdt(dtype), device="cuda")
    with cfg(dtype):
        ops.kdiag(desc, Xd, out=parent[1:N + 1])
    p = parent.cpu().numpy().astype(f64)
    assert np.isnan(p[0]) and np.isnan(p[N + 1:]).all()
    dev = p[1:N + 1]
    c, lo, hi = B.kdiag_interval(desc, X, dtype)
    assert np.all((dev >= lo) & (dev <= hi)), float(B.ratio(dev, c, lo, hi).max())
    if not any(nd in leaf_types(desc) for nd in (_lib.K_LINEAR, _lib.K_POLYNOMIAL)):
        assert np.array_equal(dev, KA.emulate_kdiag(desc, X, dtype).astype(f64)), \
            "K_diag of stationary / static leaves is exactly T(var), combined in the dtype"
    kc, kl, kh = B.expr_interval(desc, X, None, dtype=dtype)
    d, dl, dh = np.diag(kc), np.diag(kl), np.diag(kh)
    assert np.all(np.abs(dev - d) <= (dh - dl) + (hi - lo) + 1e-300)
    r = float(B.ratio(dev, c, lo, hi).max())
    note(("kdiag", dname), r)
    print(f"[kdiag] {name} {dname}: max error / bar {r:.3g}")


# ---- 3. limits and the instantiation mirror ------------------------------------------------------------------------
def _try_kbuild(kern, D=3):
    T = _torch()
    X = T.zeros((4, D), dtype=T.float64, device="cuda")
    with cfg(f64):
        ops.kbuild(gpf.kernels.compile_kernel(kern, D), X)


def test_expression_limits(cuda_device):
    K = gpf.kernels
    with cfg(f64):
        _try_kbuild(K.Sum([K.Constant(variance=0.1 * (i + 1)) for i in range(12)]))
        with pytest.raises(ValueError, match="more than 12 leaf"):
            _try_kbuild(K.Sum([K.Constant(variance=0.1 * (i + 1)) for i in range(13)]))
        c = [K.Constant(variance=0.1 * (i + 1)) for i in range(5)]
        # postfix a b c d * * * needs four stack entries, one more level needs five
        _try_kbuild(K.Product([c[0], K.Sum([c[1], K.Product([c[2], c[3]])])]))
        deep = K.Product([c[0], K.Sum([c[1], K.Product([c[2], K.Sum([c[3], c[4]])])])])
        with pytest.raises(ValueError, match="4-entry evaluation stack"):
            _try_kbuild(deep)
    # the same limits reach the public K
    assert len(leaf_types(compiled("leaves12", f64, 7))) >= 5
    assert sum(compiled("leaves12", f64, 7)[0][i].op not in (_lib.K_SUM, _lib.K_PRODUCT)
               for i in range(compiled("leaves12", f64, 7)[1])) == 12


def test_instantiations_reached():
    """Mirror of kbuild_launch / kbuild_impl's dispatch over the case table: kbuild_kernel<float|double, NG = 1..4>
    each see RationalQuadratic, Polynomial, Constant, White and Linear leaves; ARD Linear / Polynomial reach NG >= 2;
    kdiag_kernel<float|double> run on every table expression (test_kdiag_within_interval)."""
    seen = {}
    for dname, dtype in DT.items():
        D = CASE_SHAPES[dname][2]
        for name in EXPRS:
            desc = compiled(name, dtype, D)
            assert not fast_path(desc)
            ng = min(max(n_groups(desc, D), 1), 4)
            seen.setdefault((dname, ng), set()).update(leaf_types(desc))
            nodes = desc[0]
            if any(nodes[i].n_ard > 0 and nodes[i].op in (_lib.K_LINEAR, _lib.K_POLYNOMIAL) for i in range(desc[1])):
                seen.setdefault((dname, "ard_lin"), set()).add(ng)
    want = {_lib.K_RQ, _lib.K_POLYNOMIAL, _lib.K_CONSTANT, _lib.K_WHITE, _lib.K_LINEAR}
    for dname in DT:
        for ng in (1, 2, 3, 4):
            assert want <= seen.get((dname, ng), set()), (dname, ng, seen.get((dname, ng)))
        assert any(g >= 2 for g in seen[(dname, "ard_lin")])


# ---- 4. the materialised kernels -----------------------------------------------------------------------------------
def kaux_kernel(name, dtype, D):
    K = gpf.kernels
    ls = 0.7 + np.arange(D) * 0.3
    with cfg(dtype):
        if name == "cosine":
            return K.Cosine(variance=1.2, lengthscales=ls)
        if name.startswith("periodic_"):
            cls = {"rbf": "SquaredExponential", "rq": "RationalQuadratic", "exp": "Exponential", "m12": "Matern12",
                   "m32": "Matern32", "m52": "Matern52"}[name[9:]]
            kw = {"alpha": 2.5} if cls == "RationalQuadratic" else {}
            return K.Periodic(getattr(K, cls)(variance=1.1, lengthscales=ls * 0.9, **kw), period=1.0 + 0.5 * np.arange(D))
        if name.startswith("arccos"):
            return K.ArcCosine(order=int(name[6:]), variance=0.9, weight_variances=0.5 + 0.2 * np.arange(D),
                               bias_variance=0.3)
    raise KeyError(name)


KAUX = ["cosine"] + [f"periodic_{b}" for b in ("rbf", "rq", "exp", "m12", "m32", "m52")] + ["arccos0", "arccos1",
                                                                                           "arccos2"]


def kaux_inputs(dtype, D=3, n=90, n2=70, seed=1):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, D)) * 1.5
    X[5] = X[4]
    X[7] = X[6] + 1e-7 * rng.standard_normal(D)
    X[9] = -X[8]
    X[10] = 40.0 * X[3]
    X2 = rng.standard_normal((n2, D)) * 1.5
    X2[0] = X[4]
    return X.astype(dtype), X2.astype(dtype)


def run_kaux(desc, dtype, X, X2, ld_pad=3):
    """gpk_kaux into a view of a NaN-filled parent (odd leading dimension); returns (K, guards kept, bit-identical)."""
    T = _torch()
    lib = _lib.load()
    N = X.shape[0]
    N2 = N if X2 is None else X2.shape[0]
    parent = T.full((N + 2, N2 + ld_pad), SENT, dtype=tdt(dtype), device="cuda")
    view = parent[1:N + 1, 1:N2 + 1]
    Xd = T.from_numpy(X).cuda()
    X2d = None if X2 is None else T.from_numpy(X2).cuda()
    dc = ops.dtype_code(Xd)
    outs = []
    for _ in range(2):
        _lib.check(lib.gpk_kaux(desc, ops._p(Xd), N, ops._ld(Xd), ops._p(X2d), N2, ops._ld(X2d) if X2d is not None else 0,
                                ops._p(view), ops._ld(view), dc, ops._stream()), "gpk_kaux")
        outs.append(parent.cpu().numpy().astype(f64))
    a, b = outs
    rest = a.copy()
    rest[1:N + 1, 1:N2 + 1] = 0.0
    guards = np.isnan(rest).sum() == rest.size - N * N2
    return a[1:N + 1, 1:N2 + 1], guards, np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("dname", ["f64", "f32"])
@pytest.mark.parametrize("name", KAUX)
def test_kaux_within_interval(cuda_device, name, dname):
    dtype = DT[dname]
    D = 3
    X, X2 = kaux_inputs(dtype, D)
    kern = kaux_kernel(name, dtype, D)
    p = KA.params(kern, D)
    desc = kern._desc(D)
    worst = 0.0
    for Xb in (X2, None):
        dev, guards, same = run_kaux(desc, dtype, X, Xb)
        assert guards and same
        cen, lo, hi = KA.kaux_interval(p, X, Xb, dtype)
        bad = np.argwhere(~((dev >= lo) & (dev <= hi)))
        assert len(bad) == 0, [(int(i), int(j), dev[i, j], lo[i, j], hi[i, j]) for i, j in bad[:4]]
        worst = max(worst, float(B.ratio(dev, cen, lo, hi).max()))
    with cfg(dtype):
        dd = kern(X, full_cov=False).cpu().numpy().astype(f64)
    c, lo, hi = KA.kaux_diag_interval(p, X, dtype)
    assert np.all((dd >= lo) & (dd <= hi)), float(B.ratio(dd, c, lo, hi).max())
    note((name.split("_")[0] if not name.startswith("periodic") else name, dname), worst)
    print(f"[kaux] {name} {dname}: max error / bar {worst:.3g}")


@pytest.mark.parametrize("dname", ["f64", "f32"])
def test_coregion_indices(cuda_device, dname):
    """Truncation toward zero, and NaN for indices that are negative beyond -1, >= O, NaN or beyond the int range; K
    is the fp64 table entry rounded once, bit for bit, and K_diag likewise."""
    from tests.test_kaux_bounds import COREG_X, coregion_kernel

    dtype = DT[dname]
    k = coregion_kernel()
    p = KA.params(k, 1)
    X = COREG_X[:, None].astype(dtype)
    X2 = COREG_X[::-1, None].astype(dtype)[:9]
    for Xb in (X2, None):
        dev, guards, same = run_kaux(k._desc(1), dtype, X, Xb)
        assert guards and same
        assert np.array_equal(dev, KA.coregion_value(p, X, Xb, dtype).astype(f64), equal_nan=True)
    with cfg(dtype):
        dd = k(X, full_cov=False).cpu().numpy().astype(f64)
    assert np.array_equal(dd, KA.kaux_diag_interval(p, X, dtype)[0], equal_nan=True)


@pytest.mark.parametrize("dname", ["f64", "f32"])
def test_changepoint_weights(cuda_device, dname):
    """cp_weights_kernel for each has_lo / has_hi combination, 1 - sigma cancelling at steepness 30, from a strided
    input column."""
    T = _torch()
    dtype = DT[dname]
    lib = _lib.load()
    x = np.linspace(-4, 4, 301)
    Xp = np.stack([np.full_like(x, np.nan), x, np.full_like(x, np.nan)], 1).astype(dtype)
    Xd = T.from_numpy(Xp).cuda()
    for has in ((0, 0), (1, 0), (0, 1), (1, 1)):
        out = T.full((len(x) + 2,), SENT, dtype=tdt(dtype), device="cuda")
        args = (has[0], -0.5, 4.0, has[1], 1.0, 30.0)
        _lib.check(lib.gpk_changepoint_weights(ops._p(Xd[:, 1:]), len(x), 3, 0, *args, ops._p(out[1:]),
                                               ops.dtype_code(Xd), ops._stream()), "gpk_changepoint_weights")
        o = out.cpu().numpy().astype(f64)
        assert np.isnan(o[0]) and np.isnan(o[-1])
        c, lo, hi = KA.cp_weight_interval(Xp[:, 1], *args, dtype)
        dev = o[1:-1]
        assert np.all((dev >= lo) & (dev <= hi)), (has, float(B.ratio(dev, c, lo, hi).max()))
        note(("cp_weights", dname), float(B.ratio(dev, c, lo, hi).max()))


def compositions(dtype):
    from tests.test_kaux_bounds import changepoints, coregion_kernel

    K = gpf.kernels
    with cfg(dtype):
        cg = coregion_kernel(3)
        cg.active_dims = [1]
        rbf = K.SquaredExponential(variance=1.3, lengthscales=0.7, active_dims=[0])
        per = K.Periodic(K.Matern52(variance=0.6, lengthscales=1.1, active_dims=[0]), period=2.0)
        return {"coreg_x_rbf": (K.Product([cg, rbf]), 2),
                "periodic_plus_fused": (K.Sum([per, rbf, K.White(variance=0.1), K.Polynomial(degree=2.0)]), 2),
                "cosine_x_rq": (K.Product([K.Cosine(variance=0.7, lengthscales=3.0, active_dims=[0]),
                                           K.RationalQuadratic(variance=1.1, alpha=0.5, active_dims=[0])]), 2),
                "changepoints": (changepoints(K, dtype), 1)}


@pytest.mark.parametrize("dname", ["f64", "f32"])
@pytest.mark.parametrize("name", ["coreg_x_rbf", "periodic_plus_fused", "cosine_x_rq", "changepoints"])
def test_compositions_through_public_K(cuda_device, name, dname):
    dtype = DT[dname]
    kern, D = compositions(dtype)[name]
    rng = np.random.default_rng(4)
    X = np.concatenate([np.sort(rng.uniform(-3, 3, (70, 1)), 0), rng.integers(0, 3, (70, 1))], 1)[:, :D].astype(dtype)
    X2 = np.concatenate([rng.uniform(-3, 3, (45, 1)), rng.integers(0, 3, (45, 1))], 1)[:, :D].astype(dtype)
    worst = 0.0
    for Xb in (X2, None):
        with cfg(dtype):
            dev = kern(X, Xb).cpu().numpy().astype(f64)
            again = kern(X, Xb).cpu().numpy().astype(f64)
        assert np.array_equal(dev, again)
        cen, lo, hi = KA.kernel_interval(kern, X, Xb, dtype)
        bad = np.argwhere(~((dev >= lo) & (dev <= hi)))
        assert len(bad) == 0, [(int(i), int(j), dev[i, j], lo[i, j], hi[i, j]) for i, j in bad[:4]]
        worst = max(worst, float(B.ratio(dev, cen, lo, hi).max()))
    with cfg(dtype):
        dd = kern(X, full_cov=False).cpu().numpy().astype(f64)
    c, lo, hi = KA.kernel_interval(kern, X, None, dtype, full_cov=False)
    assert np.all((dd >= lo) & (dd <= hi)), float(B.ratio(dd, c, lo, hi).max())
    note((name, dname), worst)
    print(f"[composition] {name} {dname}: max error / bar {worst:.3g}")


# ---- 5. gpk_kmv with the other leaves ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["rq_a2.5", "poly_d3", "const_white", "tree3"])
@pytest.mark.parametrize("shape", [(200, None, 2), (150, 333, 3)])
def test_kmv_other_leaves(cuda_device, name, shape):
    from tests.test_gpu_cglb import _kmv, _kmv_bar

    N, N2, P = shape
    D = 7
    rng = np.random.default_rng(N + P)
    X = rng.standard_normal((N, D)) * 0.8
    X2 = None if N2 is None else rng.standard_normal((N2, D)) * 0.8
    V = rng.standard_normal((N if N2 is None else N2, P))
    desc = compiled(name, f64, D)
    diag = 0.37 if N2 is None else 0.0
    dev = _kmv(desc, X, X2, V, diag)
    ref, bar = _kmv_bar(desc, X, X2, V, diag)
    ratio = float(np.max(np.abs(dev - ref) / bar))
    print(f"[kmv] {name} {shape}: max error / bar {ratio:.3g}")
    assert ratio <= 1.0
    assert np.array_equal(dev, _kmv(desc, X, X2, V, diag))


# ---- 6. K(X, X2) taller than 65535 tile rows -----------------------------------------------------------------------
WIDE_N = 65535 * 64 + 1


@functools.lru_cache(maxsize=None)
def wide_inputs():
    rng = np.random.default_rng(9)
    X = rng.uniform(-3, 3, (WIDE_N, 1)).astype(f32)
    X2 = np.array([[-1.0], [0.25], [2.0]], f32)
    return X, X2


@pytest.mark.parametrize("name", ["rbf_white", "periodic"])
def test_wide_rectangular(cuda_device, name):
    """4,194,241 rows against 3 columns (fp32): the launch runs as two row chunks; every element checked at the chunk
    boundary, the ends and a sample in between."""
    T = _torch()
    X, X2 = wide_inputs()
    K = gpf.kernels
    with cfg(f32):
        kern = (K.Sum([K.SquaredExponential(variance=1.1, lengthscales=0.8), K.White(variance=1e-3)])
                if name == "rbf_white" else K.Periodic(K.SquaredExponential(variance=0.9, lengthscales=0.6), period=1.5))
        dev = kern(T.from_numpy(X).cuda(), T.from_numpy(X2).cuda()).cpu().numpy().astype(f64)
    assert dev.shape == (WIDE_N, 3) and np.isfinite(dev).all()
    b = 65535 * 64
    rows = np.unique(np.concatenate([np.arange(2048), np.arange(b - 2048, WIDE_N),
                                     np.random.default_rng(1).choice(WIDE_N, 20000, replace=False)]))
    cen, lo, hi = KA.kernel_interval(kern, X[rows], X2, f32)
    d = dev[rows]
    assert np.all((d >= lo) & (d <= hi)), float(B.ratio(d, cen, lo, hi).max())
    r = float(B.ratio(d, cen, lo, hi).max())
    note(("wide_" + name, "f32"), r)
    print(f"[wide] {name}: max error / bar {r:.3g}")


