"""Phase cycles (clock64) of one fp64 128x128 leaf, gpk_debug_leaf: the full-inverse leaf and the slim leaf of factorisations
with n > 128 (inverses of the two 64x64 diagonal sub-blocks only; the phases up to its done flag, after which it stores the
part of L that the panel kernel does not read).

    python scripts/leaf_timing.py
"""
import ctypes, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from gpflow_b200 import _lib, ops
lib = _lib.load()
rng = np.random.default_rng(0)
A = rng.standard_normal((128, 140)); K = A @ A.T / 128 + 0.5 * np.eye(128)
L = np.linalg.cholesky(K)
for slim in (0, 1):
    print("slim leaf" if slim else "full-inverse leaf")
    for rep in range(3):
        Kd = ops.to_device(K.copy()); dinv = ops.empty((128, 128), like=Kd)
        dbg = torch.zeros(16, dtype=torch.int64, device="cuda")
        lib.gpk_debug_leaf(ctypes.c_void_p(Kd.data_ptr()), 128, 128, ctypes.c_void_p(dinv.data_ptr()), ctypes.c_void_p(dbg.data_ptr()),
                           slim, None)
        torch.cuda.synchronize()
        t = dbg.cpu().numpy()
        tail = ["inv32 | store C", "level 32", "write dinv64"] if slim else ["store L", "inverses", "write dinv"]
        names = ["load", "chol32(J0)", "-", "panel(J0)", "trailing(J0)", "rest J1-3"] + tail
        d = np.diff(t[:10])
        print("  total cycles", t[9] - t[0], {n: int(v) for n, v in zip(names, d) if n != "-"})
        print("     J0 detail: pair0 update", t[10] - t[4], "chol32(block 1)", t[11] - t[10], "wait for the other warps", t[5] - t[11])
    Ld = np.tril(Kd.cpu().numpy())
    if slim:
        Dv = dinv.cpu().numpy().reshape(-1)[: 2 * 4096].reshape(2, 64, 64)
        err_inv = max(np.abs(Dv[b] - np.linalg.inv(L[64 * b:64 * b + 64, 64 * b:64 * b + 64])).max() for b in (0, 1))
    else:
        err_inv = np.abs(dinv.cpu().numpy() - np.linalg.inv(L)).max()
    print("  err L", np.abs(Ld - L).max(), "err inv", err_inv)
