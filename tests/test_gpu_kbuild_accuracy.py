"""Element-wise accuracy of the K-build (csrc/kbuild.cu), above all its single-stationary-leaf fast path.

1. Device exp / sqrt to the ulp: axis-aligned inputs whose x the device evaluates is known bit for bit, about 10^6
   points per kernel type over u in [0, 750] (fp32: [0, 110]), against long-double references, with the bars
   (a + b u) eps derived in tests/kbuild_bounds.py.
2. Realistic matrices (D up to 64, ARD, active dims, every mode, ragged edges, an output view with an odd leading
   dimension, sizes that give every persistent CTA several tiles) against the per-element intervals of
   tests/kbuild_bounds.py.
3. Bitwise invariants: GPK_FULL is bit-symmetric, GPK_LOWER equals GPK_FULL's lower triangle, the rectangular K(X, X)
   equals the symmetric K(X).
4. Every K-build switch in its own process (tests/_kbuild_worker.py).
5. The generic kernel with several dimension chunks, gram groups and tiles, composed through Sum / Product."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from gpflow_b200 import _lib
from tests import _kbuild_worker as W
from tests import kbuild_bounds as B

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32, f64 = np.float32, np.float64
LN2_64 = 64 / np.log(2.0)


def sweep_errors(s, op, dtype, bar=None):
    """Checks one sweep against the function bar; returns (max error in units of eps where the result is normal,
    max ratio to the bar)."""
    dev, x = s["dev"].astype(f64), s["x"].astype(f64)
    var = float(np.dtype(dtype).type(s["var"]))         # the kernel evaluates with T(var)
    coinc = x <= B.clip_of(op) if op != _lib.K_RBF else x == 0
    assert coinc.any()
    assert np.all(s["dev"][coinc] == np.dtype(dtype).type(var)), "coincident points must give exactly the variance"
    u = B.u_of_x(op, x)
    refl = B.k_of_x(op, np.maximum(x, B.clip_of(op)), var)
    ref = np.asarray(refl, f64)
    a, b = bar or B.fast_bar(op, dtype)
    eps = B.unit(dtype)
    allowed = (a + b * u) * eps * ref + B.atol_fn(dtype, var, u)
    err = np.asarray(np.abs(dev.astype(np.longdouble) - refl), f64)   # against the unrounded reference
    bad = np.argwhere(err > allowed)
    assert len(bad) == 0, (f"{len(bad)} elements outside (a + b u) eps, a={a:.2f} b={b:.2f}; first (i, j, x, dev, ref): "
                           f"{[(int(i), int(j), x[i, j], dev[i, j], ref[i, j]) for i, j in bad[:4]]}")
    tiny = np.finfo(dtype).tiny
    normal = (ref > tiny) & ((u <= 708.0) if dtype == f64 else (np.exp(-u) * 2.0 ** 125 >= 1))
    units = err / np.where(normal, ref * eps, np.inf)
    return float(units.max()), float(units[u <= 1].max()), float((err / allowed).max())


@pytest.mark.parametrize("dtype", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("op", W.TYPES, ids=[B.NAMES[t] for t in W.TYPES])
def test_fast_path_function_ulps(cuda_device, op, dtype):
    s = W.sweep(op, dtype)
    units, small, r = sweep_errors(s, op, dtype)
    a, b = B.fast_bar(op, dtype)
    print(f"[part1] {B.NAMES[op]} {np.dtype(dtype).name}: max {units:.2f} eps, {small:.2f} eps for u <= 1 "
          f"(bar {a:.2f} + {b:.2f} u), max error / bar {r:.3f}")
    if dtype == f64:  # the sweep reaches both branches of the 2^n scaling, small u in the slow one included
        u = B.u_of_x(op, s["x"])
        k = np.rint(-u * LN2_64)
        n, n2 = k.shape
        grp = k.reshape(n, n2 // 64, 2, 16, 2).min(axis=(2, 4))          # kmin of each thread's 4-column group
        slow = np.broadcast_to(grp[:, :, None, :, None] < -57600, (n, n2 // 64, 2, 16, 2)).reshape(n, n2)
        assert np.any(slow & (u < 1)) and np.any(~slow & (u > 1)) and np.any(u > 708)


@pytest.mark.parametrize("var_key", ["tiny", "huge"])
@pytest.mark.parametrize("op", W.TYPES, ids=[B.NAMES[t] for t in W.TYPES])
def test_fast_path_extreme_variance(cuda_device, op, var_key):
    """Variance below 2^-100 (the exponent-field shortcut is off) and above 1e300 (fp64)."""
    s = W.sweep(op, f64, var_key, n=500, n2=512)
    units, small, r = sweep_errors(s, op, f64)
    print(f"[part1] {B.NAMES[op]} var={s['var']:.3g}: max {units:.2f} eps, {small:.2f} eps for u <= 1, "
          f"max error / bar {r:.3f}")


def test_fast_path_known_points(cuda_device):
    """Integer inputs with a unit weight (Matern12, lengthscale 1): x = v^2 + t^2 exactly, and the values are exp(-u)
    for integer u to the function bar."""
    kern = W.leaf_kernel(_lib.K_MATERN12, 2, f64, variance=1.0, ell=1.0)
    desc = W.compiled(kern, 2)
    assert desc[0][0].lengthscale == 1.0 and desc[0][0].variance == 1.0 and B.fast_weight(_lib.K_MATERN12, 1.0) == 1.0
    v, t = np.array([3.0, 5.0, 0.0, 8.0, 20.0]), np.array([4.0, 12.0, 0.0, 15.0, 21.0])
    X, X2 = np.stack([v, 0 * v], 1), np.stack([0 * t, t], 1)
    x = B.fast_x(v, t, 1.0, f64)
    assert np.array_equal(x, v[:, None] ** 2 + t[None, :] ** 2)
    dev = W.kbuild(desc, f64, X, X2).cpu().numpy()
    assert dev[0, 0] != 0 and dev[2, 2] == 1.0
    sweep_errors(dict(dev=dev, x=x, var=1.0), _lib.K_MATERN12, f64)


# ---- part 2 / 3 ----------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def matrix(name, op):
    return W.run_matrix(name, op)


_REF_CACHE = {}


def interval_ratio(name, op, res):
    worst = 0.0
    for part in ("rows", "cols"):
        dev = res[part]
        if dev.size == 0:
            continue
        cen, lo, hi, mask = W.case_interval(name, W.case_desc(name, op), part, _REF_CACHE.setdefault((name, part), {}))
        d = dev.astype(f64)
        bad = np.argwhere(mask & ~((d >= lo) & (d <= hi)))
        assert len(bad) == 0, (f"{name} {B.NAMES[op]} {part}: {len(bad)} outside the interval; first (i, j, dev, lo, hi):"
                               f" {[(int(i), int(j), d[i, j], lo[i, j], hi[i, j]) for i, j in bad[:4]]}")
        worst = max(worst, float(B.ratio(d, cen, lo, hi)[mask].max()))
    return worst


def resident_ctas(dtype):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * (2 if dtype == f64 else 3)


@pytest.mark.parametrize("name", list(W.CASES))
def test_fast_path_matrix_within_interval(cuda_device, name):
    dtype, D, mode, N, N2, ard, active, odd = W.CASES[name]
    if name.startswith("p_"):
        nty, ntx = -(-N // 64), -(-(N2 or N) // 64)
        ntiles = nty * ntx if mode == "rect" else nty * (nty + 1) // 2
        assert ntiles >= 3 * resident_ctas(dtype), (name, ntiles)
    assert N % 64 != 0 or (N2 or N) % 64 != 0
    worst = {B.NAMES[op]: interval_ratio(name, op, matrix(name, op)) for op in W.TYPES}
    print(f"[part2] {name}: max error / bound " + " ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("name", list(W.CASES))
def test_fast_path_stores_stay_inside_the_view(cuda_device, name):
    """Everything of the sentinel-filled parent outside the output view keeps its sentinel; in lower mode so do the
    tiles strictly above the diagonal."""
    for op in W.TYPES:
        res = matrix(name, op)
        assert res["outside_kept"], (name, B.NAMES[op])
        if W.CASES[name][2] == "lower":
            assert res["upper_tiles_kept"], (name, B.NAMES[op])


SYM_CASES = [n for n, c in W.CASES.items() if c[2] != "rect"]


@pytest.mark.parametrize("name", SYM_CASES)
def test_fast_path_bitwise_invariants(cuda_device, name):
    for op in W.TYPES:
        res = matrix(name, op)
        for key in ("bit_symmetric", "lower_equals_full", "rect_equals_sym"):
            assert res.get(key, True), (name, B.NAMES[op], key)


# ---- part 5: the generic kernel with chunks, groups and tiles ------------------------------------------------------
def generic_expr(groups, dtype):
    import gpflow_b200 as gpf

    rng = np.random.default_rng(groups)
    K = gpf.kernels
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        rbf = K.SquaredExponential(variance=1.2, lengthscales=5.0 * (0.5 + rng.random(40)), active_dims=list(range(40)))
        lin = K.Linear(variance=0.3, active_dims=list(range(40, 46)))
        if groups == 2:
            return K.Product([rbf, lin])
        m52 = K.Matern52(variance=0.7, lengthscales=5.0 * (0.5 + rng.random(36)), active_dims=list(range(5, 41)))
        if groups == 3:
            return K.Sum([K.Product([rbf, lin]), m52])
        m12 = K.Matern12(variance=0.4, lengthscales=4.0, active_dims=list(range(10, 44)))
        return K.Sum([rbf, K.Product([lin, m12]), m52])


@pytest.mark.parametrize("dtype", [f64, f32], ids=["f64", "f32"])
@pytest.mark.parametrize("groups", [2, 3, 4])
def test_generic_kernel_groups_chunks_tiles(cuda_device, groups, dtype):
    """ARD over more than KB_KC = 32 dims per group, 2-4 gram groups (the NG templates), N x N2 over several tiles."""
    D, N, N2 = 50, 200, 150
    rng = np.random.default_rng(10 + groups)
    X, X2 = (rng.standard_normal((N, D)) + 0.5).astype(dtype), (rng.standard_normal((N2, D)) + 0.5).astype(dtype)
    desc = W.compiled(generic_expr(groups, dtype), D)
    nodes, n = desc[0], desc[1]
    assert sum(nodes[i].op not in (_lib.K_SUM, _lib.K_PRODUCT) for i in range(n)) == min(groups, 3) + (groups == 4)
    worst = 0.0
    for Xb in (X2, None):
        dev = W.kbuild(desc, dtype, X, Xb).cpu().numpy().astype(f64)
        cen, lo, hi = B.expr_interval(desc, X, Xb, dtype=dtype)
        bad = np.argwhere(~((dev >= lo) & (dev <= hi)))
        assert len(bad) == 0, [(int(i), int(j), dev[i, j], lo[i, j], hi[i, j]) for i, j in bad[:4]]
        worst = max(worst, float(B.ratio(dev, cen, lo, hi).max()))
    print(f"[part5] groups={groups} {np.dtype(dtype).name}: max error / bound {worst:.3g}")


# ---- part 4: every switch of the K-build, one process each ---------------------------------------------------------
SWITCHES = {
    "default": {},
    "minb2": {"GPK_KF_MINB": "2"},
    "minb3": {"GPK_KF_MINB": "3"},
    "generic": {"GPK_KBUILD_GENERIC": "1"},
}


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("kbuild_switches"))


@functools.lru_cache(maxsize=None)
def run_switch(name, tmpdir):
    env = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    env.update(SWITCHES[name])
    out = os.path.join(tmpdir, f"{name}.npz")
    r = subprocess.run([sys.executable, "-m", "tests._kbuild_worker", out], cwd=ROOT, env=env, timeout=600,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, f"{name}: worker failed\n{r.stdout[-4000:]}"
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


@functools.lru_cache(maxsize=None)
def worker_sweep(op, dtype):
    return W.sweep_inputs(op, dtype, **W.WORKER_SWEEP)


@pytest.mark.parametrize("name", list(SWITCHES))
def test_kbuild_switch(cuda_device, tmp, name):
    """Under each switch: the part-2 intervals everywhere, the part-1 ulp bars where the fast path runs (the generic
    path's x is not reproducible bit for bit, so its sweeps get the part-2 interval instead)."""
    res = run_switch(name, tmp)
    fast = name != "generic"
    for dtype in (f64, f32):
        for op in W.TYPES:
            dev = res[f"sweep_{dtype.__name__}_{op}"]
            desc = W.compiled(W.leaf_kernel(op, 2, dtype), 2)
            var, ell = desc[0][0].variance, desc[0][0].lengthscale
            w = B.fast_weight(op, ell)
            p, q = worker_sweep(op, dtype)
            v, t = (np.sqrt(p) / w).astype(dtype), (np.sqrt(q) / w).astype(dtype)
            if fast:
                sweep_errors(dict(dev=dev, x=B.fast_x(v, t, w, dtype), var=var), op, dtype)
            else:
                X, X2 = np.stack([v, 0 * v], 1), np.stack([0 * t, t], 1)
                cen, lo, hi = B.expr_interval(desc, X, X2, dtype=dtype)
                d = dev.astype(f64)
                assert np.all((d >= lo) & (d <= hi)), (name, B.NAMES[op], np.dtype(dtype).name)
    for case in W.WORKER_CASES:
        for op in W.TYPES:
            r = {k: res[f"{case}_{op}_{k}"] for k in ("rows", "cols")}
            interval_ratio(case, op, r)
            for key in ("outside_kept", "upper_tiles_kept", "bit_symmetric", "lower_equals_full", "rect_equals_sym"):
                k = f"{case}_{op}_{key}"
                if k in res:
                    assert bool(res[k]), (name, k)


def test_fast_path_bit_identical_across_minb(cuda_device, tmp):
    """The two instantiations of the fast path (2 and 3 resident CTAs per SM) do the same arithmetic: register
    allocation must not change a bit.  The default run is one of the two."""
    a, b, d = run_switch("minb2", tmp), run_switch("minb3", tmp), run_switch("default", tmp)
    assert set(a) == set(b)
    for k in a:
        assert np.array_equal(a[k], b[k]), k
        assert np.array_equal(a[k], d[k]), k
