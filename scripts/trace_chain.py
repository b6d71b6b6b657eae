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
cap = 1 << 16  # (the int8 update marks every tile of two CTAs per launch)
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
        "fused_start->publish": [], "feed_start->publish": [], "publish->leaf_ready": []}
last_leaf_done = last_panel_done = syrk_start = fused_start = last_publish = None
for a, k, p in ev:
    if k == 1 and p == 2: last_leaf_done = a
    if k in (2, 3) and p == 0: fused_start = a  # (a plain panel that publishes is one with the diagonal feed)
    if k == 2 and p == 0 and last_leaf_done is not None: hops["leaf->fused_panel"].append(a - last_leaf_done)
    if k == 3 and p == 0 and last_leaf_done is not None: hops["leaf->panel"].append(a - last_leaf_done)
    if k == 3 and p in (2, 3): last_panel_done = a
    if k == 4 and p == 0:
        syrk_start = a
        if last_panel_done is not None: hops["panel_last->syrk_start"].append(a - last_panel_done)
    if k == 4 and p == 1 and syrk_start is not None:
        hops["syrk_start->first_publish"].append(a - syrk_start); syrk_start = None
    if k in (2, 3) and p == 1 and fused_start is not None:
        hops["fused_start->publish" if k == 2 else "feed_start->publish"].append(a - fused_start); fused_start = None
    if k in (2, 3, 4) and p == 1: last_publish = a
    if k == 1 and p == 1 and last_publish is not None:
        hops["publish->leaf_ready"].append(a - last_publish)
for k2, v in hops.items():
    if v: print(f"{k2}: n={len(v)} mean {np.mean(v):.1f} median {np.median(v):.1f} min {np.min(v):.1f} max {np.max(v):.1f} sum {np.sum(v):.0f} us")
# chain budget per diagonal block: leaf k pairs with the k-th panel (every C2 block has rows below it: the (Y - m)^T row)
leaves, panels, updates = [], [], []
for a, k, p in ev:
    if k == 1 and p == 1: leaves.append({"ready": a})
    if k == 1 and p == 2 and leaves: leaves[-1]["done"] = a
    if k in (2, 3) and p == 0: panels.append({"start": a, "fused": k == 2})
    if k in (2, 3) and p in (10, 11, 1) and panels: panels[-1].setdefault({10: "ops", 11: "solved", 1: "publish"}[p], a)
    if k == 4 and p == 0: updates.append({"start": a})
    if k == 4 and p == 1 and updates: updates[-1].setdefault("publish", a)


def stat(name, v):
    if v: print(f"  {name}: n={len(v)} mean {np.mean(v):.1f} median {np.median(v):.1f} sum {np.sum(v):.0f} us")


print("chain budget per block:")
stat("leaf ready -> done", [l["done"] - l["ready"] for l in leaves if "done" in l])
stat("panel start -> operands staged (CTA 0)", [p["ops"] - p["start"] for p in panels if "ops" in p])
stat("panel phase-1 start -> solved rows stored (CTA 0)", [p["solved"] - p["ops"] for p in panels if "solved" in p])
stat("fused panel start -> critical CTA publish", [p["publish"] - p["start"] for p in panels if p["fused"] and "publish" in p])
stat("update start -> head publish", [u["publish"] - u["start"] for u in updates if "publish" in u])
pairs = [(l, p) for l, p in zip(leaves, panels) if "done" in l and "ops" in p]
stat("panel phase-1 start before its leaf's done mark (us earlier)", [l["done"] - p["ops"] for l, p in pairs])
stat("leaf done -> panel solved rows stored (CTA 0)", [p["solved"] - l["done"] for l, p in pairs if "solved" in p])


def update_k_before(n, nb=128):
    """K of the trailing update directly in front of each diagonal block (potrf.cu's split rule; 128 = the fused update)."""
    out = {}

    def rec(n_, col0):
        if n_ <= nb:
            return
        n1 = ((n_ // nb + 1) // 2) * nb
        if n_ > 2 * nb:
            rec(n1, col0)
        out[(col0 + n1) // nb] = n1
        rec(n_ - n1, col0 + n1)

    rec(n, 0)
    return out


# leaf b done -> leaf b + 1 ready, by the K of the update in front of block b + 1: K = 128 blocks come from the fused panel,
# K = 256 / 512 from the diagonal feed (GPK_DIAG_FEED_MAX_K=0: from the int8 update's head tiles), K >= 1024 from the update
kb = update_k_before(N)
by_k = {}
for b in range(len(leaves) - 1):
    if "done" in leaves[b] and b + 1 in kb:
        k = kb[b + 1]
        by_k.setdefault(f"K={k}" if k <= 512 else "K>=1024", []).append(leaves[b + 1]["ready"] - leaves[b]["done"])
print("leaf done -> next leaf ready, by the K of the update in front of the next block:")
for k in sorted(by_k, key=lambda s: int(s.split("=")[-1])):
    stat(k, by_k[k])
