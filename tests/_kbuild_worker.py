"""Workloads of tests/test_gpu_kbuild_accuracy.py.  The functions run in the test process; `main` runs a fixed subset in a
fresh process, so that the K-build switches (GPK_KF_MINB, GPK_KBUILD_GENERIC, read once per process) take effect, and
saves the device results.  Usage: python -m tests._kbuild_worker OUT.npz"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from gpflow_b200 import _lib  # noqa: E402
from tests import kbuild_bounds as B  # noqa: E402

f32, f64 = np.float32, np.float64
TYPES = list(B.STATIONARY)
CLASSES = {_lib.K_RBF: "SquaredExponential", _lib.K_MATERN12: "Matern12", _lib.K_MATERN32: "Matern32",
           _lib.K_MATERN52: "Matern52", _lib.K_EXPONENTIAL: "Exponential"}
SENT = -7.25      # sentinel: no kernel value is negative
TILE = 64

# name: (dtype, D, mode, N, N2, ARD lengthscales, active dims (None: all D), odd leading dimension of the output view)
# "p_" cases give every resident CTA of the persistent grid at least three tiles on an H100.
CASES = {
    "d1_rect": (f64, 1, "rect", 333, 190, False, None, True),
    "d8_lower": (f32, 8, "lower", 333, None, False, None, False),
    "d9_full": (f64, 9, "full", 333, None, False, None, True),
    "d64_rect_ard": (f32, 64, "rect", 200, 270, True, None, True),
    "d16_lower_active": (f64, 24, "lower", 300, None, False, [1, 2, 3, 5, 7, 8, 9, 11, 12, 14, 15, 17, 19, 20, 22, 23],
                         True),
    "d33_full_ard": (f32, 33, "full", 260, None, True, None, True),
    "p_f64_rect_d17": (f64, 17, "rect", 1000, 3300, True, None, True),
    "p_f64_lower_d8": (f64, 8, "lower", 2600, None, False, None, True),
    "p_f64_full_d64": (f64, 64, "full", 2600, None, False, None, False),
    "p_f32_rect_d9": (f32, 9, "rect", 1100, 4500, False, None, True),
    "p_f32_lower_d16": (f32, 16, "lower", 3100, None, True, None, False),
    "p_f32_full_d33": (f32, 40, "full", 3100, None, False, list(range(3, 36)), True),
}
DIAG_SCALAR = {"lower": 0.25, "full": 0.5, "rect": 0.0}


def _gpf():
    import gpflow_b200 as gpf

    return gpf


def leaf_kernel(op, D, dtype, variance=1.3, ell=1.7, active=None):
    gpf = _gpf()
    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        kw = {} if active is None else {"active_dims": active}
        return getattr(gpf.kernels, CLASSES[op])(variance=variance, lengthscales=ell, **kw)


def compiled(kern, D, variance=None):
    """compile_kernel(kern, D); `variance` overrides the leaf's variance in the compiled node."""
    desc = _gpf().kernels.compile_kernel(kern, D)
    if variance is not None:
        desc[0][0].variance = float(variance)
    return desc


def kbuild(desc, dtype, X, X2=None, **kw):
    gpf = _gpf()
    from gpflow_b200 import ops

    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Xd = ops.to_device(X)
        X2d = None if X2 is None else ops.to_device(X2)
        return ops.kbuild(desc, Xd, X2d, **kw)


# ---- part 1: axis-aligned sweeps --------------------------------------------------------------------------------
SWEEP_VARS = {"default": None, "tiny": 2.0 ** -110, "huge": 3e300}


def sweep_inputs(op, dtype, n=1000, n2=1024):
    """Rows (v_i, 0) and (0, t_j): x_ij = p_i + q_j over u in [0, 750] (fp64; [0, 110] fp32), dense near zero.  In the
    second half of the columns every column 32 + 2m of a 64-column tile (one of the four columns of each thread's row
    group in kbuild_fast_kernel) has u in [630, 700]: its k < -57600 sends the whole group, small u included, through
    the slow branch of the 2^n scaling."""
    umax = 750.0 if dtype == f64 else 110.0
    p = B.sweep_targets(op, n, umax)
    q = B.sweep_targets(op, n2 // 2, umax)
    q2 = q.copy()
    j = np.arange(n2 // 2)
    big = (j % TILE >= 32) & (j % 2 == 0)
    ub = np.linspace(630.0, 700.0, big.sum()) if dtype == f64 else np.linspace(95.0, 105.0, big.sum())
    q2[big] = ub if op == _lib.K_RBF else ub * ub
    q = np.concatenate([q, q2])
    return p, q


def sweep(op, dtype, var_key="default", n=1000, n2=1024):
    """Device K of the sweep, with the exact x it evaluated and the variance / lengthscale read back from the node."""
    desc = compiled(leaf_kernel(op, 2, dtype), 2, SWEEP_VARS[var_key])
    var, ell = desc[0][0].variance, desc[0][0].lengthscale
    w = B.fast_weight(op, ell)
    p, q = sweep_inputs(op, dtype, n, n2)
    v, t = (np.sqrt(p) / w).astype(dtype), (np.sqrt(q) / w).astype(dtype)
    X = np.stack([v, np.zeros_like(v)], 1)
    X2 = np.stack([np.zeros_like(t), t], 1)
    dev = kbuild(desc, dtype, X, X2).cpu().numpy()
    return dict(dev=dev, x=B.fast_x(v, t, w, dtype), var=var, X=X, X2=X2, desc=desc)


# ---- part 2 / 3: realistic matrices -----------------------------------------------------------------------------
def case_inputs(name):
    dtype, D, mode, N, N2, ard, active, odd = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    nd = D if active is None else len(active)
    X = rng.standard_normal((N, D)) + 1.5                   # offset: the norm expansion cancels more
    X[5] = X[4]                                              # coincident pair
    X[7] = X[6] + 1e-6 * rng.standard_normal(D)              # nearly coincident pair
    X[9] = X[8] * 9.0                                         # far-apart rows
    X2 = None if N2 is None else rng.standard_normal((N2, D)) + 1.0
    ell = np.sqrt(nd) * (0.4 + rng.random(nd)) if ard else float(np.sqrt(nd) * 0.7)
    dvec = 0.1 + rng.random(N) if mode == "lower" else None
    return X.astype(dtype), None if X2 is None else X2.astype(dtype), ell, dvec


def case_desc(name, op):
    dtype, D, mode, N, N2, ard, active, odd = CASES[name]
    return compiled(leaf_kernel(op, D, dtype, ell=case_inputs(name)[2], active=active), D)


def check_rows(N, rng_seed=0):
    """All rows of the first and last tile rows, plus a random sample (all rows for small N)."""
    if N <= 400:
        return np.arange(N)
    last = (N - 1) // TILE * TILE
    rs = np.random.default_rng(rng_seed).choice(np.arange(TILE, last), 48, replace=False)
    return np.unique(np.concatenate([np.arange(TILE), np.arange(last, N), rs]))


def check_cols(N2):
    if N2 <= 400:
        return np.arange(0)
    last = (N2 - 1) // TILE * TILE
    return np.concatenate([np.arange(TILE), np.arange(last, N2)])


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def run_matrix(name, op):
    """One case and one kernel type: K into a sentinel-filled parent, the checked rows / columns, the sentinel checks,
    and the bitwise invariants of part 3 (symmetric modes)."""
    import torch

    dtype, D, mode, N, N2, ard, active, odd = CASES[name]
    X, X2, ell, dvec = case_inputs(name)
    desc = case_desc(name, op)
    M2 = N if N2 is None else N2
    ld = M2 + (3 if M2 % 2 == 0 else 2) if odd else (M2 + 3) // 4 * 4 + 4
    c0 = 1 if odd else 0
    tdt = torch.float64 if dtype == f64 else torch.float32
    parent = torch.full((N + 2, ld), SENT, dtype=tdt, device="cuda")
    view = parent[1:N + 1, c0:c0 + M2]
    s = DIAG_SCALAR[mode]
    gpf = _gpf()
    from gpflow_b200 import ops

    with gpf.config.as_context(gpf.config.Config(float=dtype)):
        Xd = ops.to_device(X)
        X2d = None if X2 is None else ops.to_device(X2)
        dv = None if dvec is None else ops.to_device(dvec.astype(dtype))
        uplo = _lib.GPK_LOWER if mode == "lower" else _lib.GPK_FULL
        ops.kbuild(desc, Xd, X2d, uplo=uplo, diag_scalar=s, diag_vec=dv, out=view)
        res = {}
        rest = parent.clone()
        rest[1:N + 1, c0:c0 + M2] = SENT
        res["outside_kept"] = bool(torch.all(rest == SENT))
        if mode == "lower":
            ti = torch.arange(N, device="cuda") // TILE
            res["upper_tiles_kept"] = bool(torch.all(view[(ti[None, :] > ti[:, None])] == SENT))
            full = ops.kbuild(desc, Xd, None, uplo=_lib.GPK_FULL, diag_scalar=s, diag_vec=dv)
            res["lower_equals_full"] = bool(torch.equal(torch.tril(view), torch.tril(full)))
        if mode == "full":
            res["bit_symmetric"] = bool(torch.equal(view, view.T))
        if mode != "rect":
            sym = ops.kbuild(desc, Xd, None)
            res["rect_equals_sym"] = bool(torch.equal(ops.kbuild(desc, Xd, Xd), sym))
        rows, cols = check_rows(N), check_cols(M2)
        res["rows"] = view[torch.as_tensor(rows, device="cuda")].cpu().numpy()
        res["cols"] = view[:, torch.as_tensor(cols, device="cuda", dtype=torch.long)].cpu().numpy()
        res["digest"] = digest(view.cpu().numpy())
    res["desc"] = desc
    return res


def case_interval(name, desc, part, cache=None):
    """(center, lo, hi, mask) of the checked rows ("rows") or columns ("cols") of a case, diagonal shift included;
    `cache` keeps the reference distances across kernel types."""
    dtype, D, mode, N, N2, ard, active, odd = CASES[name]
    X, X2, ell, dvec = case_inputs(name)
    M2 = N if N2 is None else N2
    Xo = X if X2 is None else X2
    if part == "rows":
        ri = check_rows(N)
        cen, lo, hi = B.expr_interval(desc, X, Xo, rows=ri, dtype=dtype, cache=cache)
        I, J = np.meshgrid(ri, np.arange(M2), indexing="ij")
    else:
        ci = check_cols(M2)
        cen, lo, hi = B.expr_interval(desc, X, Xo[ci], dtype=dtype, cache=cache)
        I, J = np.meshgrid(np.arange(N), ci, indexing="ij")
    if mode != "rect":
        shift = DIAG_SCALAR[mode] + (0.0 if dvec is None else dvec.astype(dtype).astype(f64)[I])
        on = I == J
        u = B.unit(dtype)
        m = 2 * u * (np.abs(hi) + shift)
        cen, lo, hi = (np.where(on, cen + shift, cen), np.where(on, lo + shift - m, lo),
                       np.where(on, hi + shift + m, hi))
    mask = (J <= I) if mode == "lower" else np.ones_like(I, bool)
    return cen, lo, hi, mask


# ---- the subset run under each K-build switch ------------------------------------------------------------------
WORKER_SWEEP = dict(n=500, n2=512)
WORKER_CASES = ["d9_full", "d64_rect_ard", "p_f64_lower_d8", "p_f32_rect_d9"]


def main(out):
    import torch

    torch.cuda.set_device(0)
    res = {}
    for dtype in (f64, f32):
        for op in TYPES:
            res[f"sweep_{dtype.__name__}_{op}"] = sweep(op, dtype, **WORKER_SWEEP)["dev"]
    for name in WORKER_CASES:
        for op in TYPES:
            r = run_matrix(name, op)
            for k, v in r.items():
                if k != "desc":
                    res[f"{name}_{op}_{k}"] = np.array(v)
    torch.cuda.synchronize()
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
