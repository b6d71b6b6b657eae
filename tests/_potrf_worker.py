"""gpk_potrf through the C ABI on views inside NaN-filled parents, for tests/test_gpu_potrf_elements.py; run as
`python -m tests._potrf_worker OUT.npz` it factors the engine-configuration cases in a fresh process (the GPK_* switches
are read once per process) and saves the factors."""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

F64, F32 = 1, 0
LDPAD, GUARD = 5, 3          # leading dimension n + LDPAD, GUARD NaN rows below the last row
# (n, extra rows, family, seed) factored under every engine configuration
CONFIG_CASES = [(1000, 3, "spd", 11), (2049, 129, "spd", 12), (1000, 0, "gpr", 13)]


def _t():
    import torch
    return torch


def lib():
    from gpflow_b200 import _lib
    return _lib.load()


def ptr(x, off=0):
    return ctypes.c_void_p(x.data_ptr() + off * x.element_size())


def parent_of(T, n, rows, dtype=np.float64):
    """NaN parent [rows + GUARD, n + LDPAD] with T's lower triangle in the square part and T's extra rows below it."""
    P = np.full((rows + GUARD, n + LDPAD), np.nan, dtype=dtype)
    P[:n, :n] = np.where(np.tri(n, dtype=bool), T[:n, :n], np.nan)
    P[n:rows, :n] = T[n:rows, :n]
    return P


def run_parent(dP, n, rows, dtype=np.float64):
    """gpk_potrf on the view [rows, n] at the head of the device parent dP (ld = its width); returns info."""
    torch = _t()
    dc = F64 if dtype == np.float64 else F32
    ws = torch.empty(int(lib().gpk_potrf_ws(n, rows, dc)), dtype=torch.uint8, device="cuda")
    info = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    rc = lib().gpk_potrf(ptr(dP), n, rows, dP.shape[1], dc, ptr(info), ptr(ws), None)
    assert rc == 0, lib().gpk_last_error().decode()
    torch.cuda.synchronize()
    return int(info.item()), ws


def factor(T, n, rows=None, dtype=np.float64):
    """Factor T (lower triangle of A in rows < n, Y below) on the device.  Returns (F [rows, n] lower-trapezoidal as
    float64, parent after, parent before, info, digit planes the factorisation used)."""
    torch = _t()
    rows = n if rows is None else rows
    P = parent_of(T, n, rows, dtype)
    dP = torch.from_numpy(P).cuda()
    info, _ = run_parent(dP, n, rows, dtype)
    out = dP.cpu().numpy()
    F = np.where(np.tri(rows, n, dtype=bool), out[:rows, :n], 0.0).astype(np.float64)
    return F, out, P, info, int(lib().gpk_potrf_last_slices())


def target(A, Y=None):
    return A if Y is None else np.concatenate([A, Y])


def config_case(n, p, family, seed):
    from tests import chol_bounds as CB
    rng = np.random.default_rng(seed)
    A = CB.random_spd(n, rng) if family == "spd" else CB.gpr_matrix(n, rng, "m52")
    Y = rng.standard_normal((p, n)) if p else None
    return A, Y


def main(out):
    _t().cuda.set_device(0)
    res = {}
    for n, p, fam, seed in CONFIG_CASES:
        A, Y = config_case(n, p, fam, seed)
        F, _, _, info, S = factor(target(A, Y), n, n + p)
        res[f"F_{n}_{p}_{fam}"] = F
        res[f"info_{n}_{p}_{fam}"] = np.array(info)
        res[f"S_{n}_{p}_{fam}"] = np.array(S)
    np.savez(out, **res)


if __name__ == "__main__":
    main(sys.argv[1])
