"""Device timeline of one C2-shaped GPR evaluation (gpk_debug_trace): %globaltimer stamps of the leaf / panel / int8 tensor-core update
kernels, written to a CSV and summarised as the dependent chain (who waited for whom, how long the hops between kernels are).

    python scripts/trace_chain.py [N] [out.csv]
"""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import gpflow_b200 as gpf
from gpflow_b200 import _lib
from oracle import gp_oracle as O

N = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
out = sys.argv[2] if len(sys.argv) > 2 else "gpurun_out/trace_c2.csv"
lib = _lib.load()
d = O.make_data(2, N, 8, 1)
m = gpf.models.GPR((d["X"], d["Y"]), gpf.kernels.Matern52(lengthscales=np.sqrt(8.0)), noise_variance=0.1)
for _ in range(3):
    m.log_marginal_likelihood()
torch.cuda.synchronize()
cap = 4096
buf = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
pos = torch.zeros(1, dtype=torch.int32, device="cuda")
assert lib.gpk_debug_trace(ctypes.c_void_p(buf.data_ptr()), ctypes.c_void_p(pos.data_ptr()), cap) == 0
m.log_marginal_likelihood()
torch.cuda.synchronize()
lib.gpk_debug_trace(None, None, 0)
n = min(int(pos.item()), cap)
b = buf.cpu().numpy().astype(np.uint64)[: 2 * n].reshape(n, 2)
t = b[:, 0].astype(np.int64)
kid = (b[:, 1] >> np.uint64(8)).astype(np.int64)
ph = (b[:, 1] & np.uint64(255)).astype(np.int64)
order = np.argsort(t, kind="stable")
t, kid, ph = t[order], kid[order], ph[order]
t0 = t[0]
names = {1: "leaf", 2: "fused_panel", 3: "panel", 4: "syrk_i8"}
phn = {0: "start", 1: "ready/published", 2: "cta0_done", 3: "last_cta_done", 10: "p10", 11: "p11", 12: "p12", 13: "p13", 14: "p14", 15: "p15", 16: "p16", 17: "p17"}
os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
with open(out, "w") as f:
    f.write("t_us,kernel,phase\n")
    for a, k, p in zip(t, kid, ph):
        f.write(f"{(a - t0) / 1e3:.3f},{names.get(int(k), k)},{phn.get(int(p), p)}\n")
print(f"{n} marks, span {(t[-1] - t0) / 1e3:.1f} us -> {out}")
# summary: leaf spin (start -> ready), leaf run (ready -> done), and the gap from the end of a leaf to the next kernel start
ev = [((a - t0) / 1e3, int(k), int(p)) for a, k, p in zip(t, kid, ph)]
spin, run = [], []
ls = lr = None
for a, k, p in ev:
    if k == 1 and p == 0: ls = a
    if k == 1 and p == 1: lr = a; spin.append(a - ls)
    if k == 1 and p == 2: run.append(a - lr)
print(f"leaves {len(run)}: spin mean {np.mean(spin):.1f} us (sum {np.sum(spin):.0f}), run mean {np.mean(run):.1f} us (sum {np.sum(run):.0f})")
# hop: leaf done -> next panel start (fused or plain)
hops = {"leaf->fused_panel": [], "leaf->panel": [], "panel_last->syrk_start": [], "syrk_start->first_publish": [],
        "fused_start->publish": [], "publish->leaf_ready": []}
last_leaf_done = last_panel_done = syrk_start = fused_start = last_publish = None
for a, k, p in ev:
    if k == 1 and p == 2: last_leaf_done = a
    if k == 2 and p == 0:
        fused_start = a
        if last_leaf_done is not None: hops["leaf->fused_panel"].append(a - last_leaf_done)
    if k == 3 and p == 0 and last_leaf_done is not None: hops["leaf->panel"].append(a - last_leaf_done)
    if k == 3 and p in (2, 3): last_panel_done = a
    if k == 4 and p == 0:
        syrk_start = a
        if last_panel_done is not None: hops["panel_last->syrk_start"].append(a - last_panel_done)
    if k == 4 and p == 1 and syrk_start is not None:
        hops["syrk_start->first_publish"].append(a - syrk_start); syrk_start = None
    if k == 2 and p == 1 and fused_start is not None:
        hops["fused_start->publish"].append(a - fused_start); fused_start = None
    if (k == 2 and p == 1) or (k == 4 and p == 1): last_publish = a
    if k == 1 and p == 1 and last_publish is not None:
        hops["publish->leaf_ready"].append(a - last_publish)
for k2, v in hops.items():
    if v: print(f"{k2}: n={len(v)} mean {np.mean(v):.1f} median {np.median(v):.1f} min {np.min(v):.1f} max {np.max(v):.1f} sum {np.sum(v):.0f} us")
