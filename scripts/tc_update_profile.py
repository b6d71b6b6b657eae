"""Per-launch breakdown of the int8 digit-sliced trailing update (gemm_tc.cu::syrk_i8_kernel) in one C2 evaluation.

    python scripts/tc_update_profile.py [--evals 3] [--out DIR]
    python scripts/tc_update_profile.py --phases [--evals 3] [--out DIR]

Runs C2 (GPR Matern52 fp64, N = 8192) under torch.profiler with CUDA activities, joins every syrk_i8_kernel launch with the
int8 `update` entries of the launch-schedule mirror (tests/test_host_logic_r2.py::_potrf_schedule) and prints each launch's
duration, the int8 operations it issues (the count of the ProfScope in syrk_tc_planes: every tile of every cluster unit x
k-steps x digit products x 2 ops per MAC) and the rate, then the same grouped by K.  It then times a standalone update at
m = n = K = 4096 through gpk_debug_syrk_i8 for cluster widths 1, 2 and 4.

--phases instead records the gpk_debug_trace timeline of C2 evaluations and splits every syrk_i8_kernel launch into the
phases its %globaltimer marks bound (median over the launches of each K): the prologue (barrier set-up, cluster sync), the
main loop and the epilogue of CTA 0's first tile (a head tile), the wait until that tile's update is complete in global
memory and may be published (phase 16; absent from builds without it), and the time from the start to the end of CTA 0 and
of the launch's last CTA (the highest index; CTA 0 publishes more head tiles and often finishes later).  It then prints,
per K, the per-tile timeline of CTA 0 and of the last CTA (marks 20-23 / 30-33, written by the kernel instantiations
launched while a trace buffer is installed): when each tile starts, the wait for its first full pipeline stage, its main
loop, its epilogue, and the time from its reductions to the next tile's start (or to the CTA's end), with the number of
tiles those launches gave the CTA.

A measurement tool: nothing depends on it.  Needs a GPU; profile in a process of its own (tracing slows the host).
GPFLOW_B200_LIB points it at another build of the library (to compare two kernels in one run)."""
from __future__ import annotations

import argparse
import collections
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TC_BM, TC_BN, TC_KB = 128, 32, 32


def n_products(S: int) -> int:
    return S * (S + 1) // 2 + (1 if S == 6 else 0)


def issued_ops(m: int, n: int, K: int, S: int, cl: int, lower: bool = True) -> float:
    """int8 operations one syrk_i8_kernel launch issues (padding tiles of partly empty cluster units included)."""
    ntm, ntn = -(-m // TC_BM), -(-n // TC_BN)
    units = 0
    for t in range(ntm):
        nc = min((t + 1) * (TC_BM // TC_BN), ntn) if lower else ntn
        units += -(-nc // cl)
    return 2.0 * units * cl * (K // TC_KB) * n_products(S) * TC_BM * TC_BN * TC_KB


def kernel_events(prof, needle: str):
    """(start_us, duration_us) of every device kernel whose name contains `needle`, in start order."""
    import torch

    out = [(e.time_range.start, e.time_range.elapsed_us()) for e in prof.events()
           if e.device_type == torch.autograd.DeviceType.CUDA and needle in e.name]
    return sorted(out)


def c2_updates(n: int, rows: int, nb: int = 128):
    """(m, n, K) of every update that runs on the int8 tensor cores, in launch order.  The schedule mirror lists an update
    as (col0, K); its C block is the rest of the sub-problem it splits, so the sub-problem sizes are recomputed here with the
    mirror's split rule and the two enumerations are checked against each other."""
    from tests.test_host_logic_r2 import _potrf_schedule

    dims = []

    def rec(n_, col0):
        if n_ <= 2 * nb:
            return
        n1 = ((n_ // nb + 1) // 2) * nb
        rec(n1, col0)
        dims.append((col0, n1, n_ - n1))
        rec(n_ - n1, col0 + n1)

    rec(n, 0)
    sched = [e for e in _potrf_schedule(n, rows, nb) if e[0] == "update"]
    assert [(e[1], e[2]) for e in sched] == [(c, k) for c, k, _ in dims]
    return [(rows - col0 - K, nn, K) for (col0, K, nn), e in zip(dims, sched) if e[3]]


def profile_c2(evals: int, S: int, cl: int):
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench

    hp = bench.host_problem("gpr_c2", 0)
    arm = bench.OurArm("gpr_c2", hp, 0, 1)
    arm.build_resident()
    for _ in range(3):
        arm.eval_resident()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(evals):
            arm.eval_resident()
        torch.cuda.synchronize()
    n = hp["X"].shape[0]
    ups = c2_updates(n, n + 1)
    ev = kernel_events(prof, "syrk_i8_kernel")
    assert len(ev) == evals * len(ups), f"{len(ev)} syrk_i8_kernel launches, expected {evals} x {len(ups)}"
    rows = []
    for i, (m, nn, K) in enumerate(ups):
        us = statistics.median(ev[j * len(ups) + i][1] for j in range(evals))
        ops = issued_ops(m, nn, K, S, cl)
        rows.append({"i": i, "m": m, "n": nn, "K": K, "us": us, "ops": ops, "tops": ops / us * 1e-6})
    return rows


# syrk_i8_kernel's trace marks (id 4, gemm_tc.cu): 0 start, 10 prologue done, 13 accumulators complete, 15 update stored or
# its reductions issued, 16 update complete in global memory (head tiles), 2 / 3 CTA 0 / the last CTA done
PHASES = [("prologue", 0, 10), ("main loop", 10, 13), ("epilogue", 13, 15), ("to complete", 15, 16), ("CTA 0 done", 0, 2),
          ("last CTA done", 0, 3)]


def trace_phases(evals: int):
    """Per syrk_i8_kernel launch of `evals` traced C2 evaluations: (K, {phase name: us or None})."""
    import ctypes

    import numpy as np
    import torch

    import bench
    from gpflow_b200 import _lib

    lib = _lib.load()
    hp = bench.host_problem("gpr_c2", 0)
    arm = bench.OurArm("gpr_c2", hp, 0, 1)
    arm.build_resident()
    for _ in range(3):
        arm.eval_resident()
    torch.cuda.synchronize()
    cap = 1 << 18
    buf = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.gpk_debug_trace(ctypes.c_void_p(buf.data_ptr()), ctypes.c_void_p(pos.data_ptr()), cap) == 0
    try:
        for _ in range(evals):
            arm.eval_resident()
        torch.cuda.synchronize()
    finally:
        lib.gpk_debug_trace(None, None, 0)
    nm = int(pos.item())
    assert nm <= cap, f"{nm} trace marks overflow the buffer of {cap}"
    b = buf.cpu().numpy()[: 2 * nm].reshape(nm, 2)
    b = b[np.argsort(b[:, 0], kind="stable")]
    launches = []  # one {phase: [times in ns]} per launch; a launch's marks lie between its start mark and the next one
    for t, tag in b:
        if tag >> 8 != 4:
            continue
        ph = int(tag & 255)
        if ph == 0:
            launches.append({})
        if launches:
            launches[-1].setdefault(ph, []).append(int(t))
    ups = c2_updates(hp["X"].shape[0], hp["X"].shape[0] + 1)
    assert len(launches) == evals * len(ups), f"{len(launches)} traced syrk_i8_kernel launches, expected {evals} x {len(ups)}"
    out = []
    for j, marks in enumerate(launches):
        first = {ph: ts[0] for ph, ts in marks.items()}
        phases = {name: (first[b_] - first[a]) * 1e-3 if a in first and b_ in first else None for name, a, b_ in PHASES}
        out.append((ups[j % len(ups)][2], phases, {who: tile_timeline(marks, base) for who, base in TILE_MARKS}))
    return out


# per-tile marks of CTA 0 (20-23) and of the launch's last CTA (30-33): tile start, first stage full, accumulators complete,
# update stored or its reductions issued
TILE_MARKS = [("CTA 0", 20), ("last CTA", 30)]
TILE_PHASES = ["start", "stage wait", "main loop", "epilogue", "to next tile"]


def tile_timeline(marks, base):
    """[{phase: us}] for every tile one CTA computed in a launch: its start after the launch's start mark, the wait for the
    producer's first full stage, the main loop, the epilogue and the time from its reductions to the next tile's start
    (the CTA's end for its last tile: mark 2 / 3)."""
    t0 = marks[0][0]
    starts, full, acc, done = (marks.get(base + i, []) for i in range(4))
    assert len(starts) == len(full) == len(acc) == len(done), "incomplete per-tile marks"
    end = marks.get(2 if base == 20 else 3, [None])[0]
    tiles = []
    for i in range(len(starts)):
        nxt = starts[i + 1] if i + 1 < len(starts) else end
        tiles.append({"start": (starts[i] - t0) * 1e-3, "stage wait": (full[i] - starts[i]) * 1e-3,
                      "main loop": (acc[i] - full[i]) * 1e-3, "epilogue": (done[i] - acc[i]) * 1e-3,
                      "to next tile": (nxt - done[i]) * 1e-3 if nxt is not None else None})
    return tiles


def tile_table(launches):
    """Per K and traced CTA: the median of every per-tile phase over the launches of that K, tile by tile, with the tile
    counts those launches gave the CTA."""
    by_k = collections.OrderedDict()
    for K, _, tl in sorted(launches, key=lambda r: -r[0]):
        by_k.setdefault(K, []).append(tl)
    table = collections.OrderedDict()
    for K, rows in by_k.items():
        table[K] = {}
        for who, _ in TILE_MARKS:
            runs = [r[who] for r in rows]
            ntile = max(len(r) for r in runs)
            med = []
            for i in range(ntile):
                have = [r[i] for r in runs if i < len(r)]
                med.append({"launches": len(have), **{p: (statistics.median(v) if v else None) for p in TILE_PHASES
                                                          for v in [[h[p] for h in have if h[p] is not None]]}})
            table[K][who] = {"tiles": sorted(collections.Counter(len(r) for r in runs).items()), "per_tile": med}
    return table


def phase_table(launches):
    """Median of every phase over the launches of each K, largest K first."""
    by_k = collections.OrderedDict()
    for K, ph, _ in sorted(launches, key=lambda r: -r[0]):
        by_k.setdefault(K, []).append(ph)
    table = collections.OrderedDict()
    for K, rows in by_k.items():
        med = {}
        for name, _, _ in PHASES:
            v = [r[name] for r in rows if r[name] is not None]
            med[name] = statistics.median(v) if v else None
        table[K] = {"launches": len(rows), "us": med}
    return table


def debug_update(size: int, S: int, cl: int, reps: int):
    """Median duration (us) of syrk_i8_kernel in gpk_debug_syrk_i8 at m = n = K = size, row-maximum scales."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from gpflow_b200 import _lib

    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(0)
    r0 = size
    A = torch.randn((size, r0), dtype=torch.float64, device="cuda", generator=g)
    C = torch.zeros((size, size), dtype=torch.float64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(lib.gpk_debug_syrk_i8(A.data_ptr(), r0, r0, 0, size, C.data_ptr(), size, size, size, 1, S, cl, None, None,
                                         st), "gpk_debug_syrk_i8")

    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            run()
        torch.cuda.synchronize()
    ev = kernel_events(prof, "syrk_i8_kernel")
    assert len(ev) == reps, (len(ev), reps)
    return statistics.median(d for _, d in ev)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--evals", type=int, default=3, help="profiled C2 evaluations (per-launch median over them)")
    ap.add_argument("--reps", type=int, default=5, help="standalone updates per cluster width")
    ap.add_argument("--out", default=None, help="directory for a JSON copy of the tables")
    ap.add_argument("--phases", action="store_true", help="per-K phase timeline of the launches (gpk_debug_trace) instead")
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "tc_update_profile.py needs a CUDA device"
    # C2's conditioning hint ((1 + 0.1) / 0.1 <= 1e4) selects S = 6 (potrf.cu::pick_slices); GPK_TC_SLICES pins it
    S = int(os.environ.get("GPK_TC_SLICES", "0") or 0) or 6
    e = os.environ.get("GPK_TC_CLUSTER", "")
    cl = 1 if e.startswith("1") else 4 if e.startswith("4") else 2
    print(f"device {torch.cuda.get_device_name(0)}; S = {S}, cluster width {cl}")
    if args.phases:
        launches = trace_phases(args.evals)
        table = phase_table(launches)
        print(f"\nC2 syrk_i8_kernel phases, us (median over the launches of each K in {args.evals} evaluations; "
              "main loop / epilogue / to complete: CTA 0's first tile)")
        print(f"{'K':>5} {'launches':>8}" + "".join(f" {name:>13}" for name, _, _ in PHASES))
        for K, g in table.items():
            cells = "".join(f" {g['us'][name]:>13.1f}" if g["us"][name] is not None else f" {'-':>13}" for name, _, _ in PHASES)
            print(f"{K:>5} {g['launches']:>8}{cells}")
        tiles = tile_table(launches)
        print("\nper-tile timeline, us (median over the launches of each K that gave the CTA that tile; start: from the "
              "launch's start mark; to next tile: from its reductions to the next tile's start, or to the CTA's end)")
        for K, g in tiles.items():
            for who, _ in TILE_MARKS:
                cnt = ", ".join(f"{c} tiles x {k}" for c, k in g[who]["tiles"])
                print(f"K = {K}, {who} ({cnt} launches)")
                print(f"  {'tile':>4} {'launches':>8}" + "".join(f" {p:>12}" for p in TILE_PHASES))
                for i, r in enumerate(g[who]["per_tile"]):
                    cells = "".join(f" {r[p]:>12.1f}" if r[p] is not None else f" {'-':>12}" for p in TILE_PHASES)
                    print(f"  {i:>4} {r['launches']:>8}{cells}")
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "tc_update_phases.json"), "w") as f:
                json.dump({"device": torch.cuda.get_device_name(0), "S": S, "cluster": cl, "by_k": table, "tiles": tiles},
                          f, indent=1)
        return
    rows = profile_c2(args.evals, S, cl)
    print(f"\nC2 syrk_i8_kernel launches (median of {args.evals} evaluations)")
    print(f"{'#':>3} {'m':>5} {'n':>5} {'K':>5} {'us':>9} {'T op/s':>8}")
    for r in rows:
        print(f"{r['i']:>3} {r['m']:>5} {r['n']:>5} {r['K']:>5} {r['us']:>9.1f} {r['tops']:>8.0f}")
    by_k = collections.OrderedDict()
    for r in sorted(rows, key=lambda r: -r["K"]):
        g = by_k.setdefault(r["K"], {"launches": 0, "us": 0.0, "ops": 0.0})
        g["launches"] += 1
        g["us"] += r["us"]
        g["ops"] += r["ops"]
    tot_us, tot_ops = sum(r["us"] for r in rows), sum(r["ops"] for r in rows)
    print(f"\n{'K':>5} {'launches':>8} {'ms':>8} {'share':>6} {'T op/s':>8}")
    for K, g in by_k.items():
        print(f"{K:>5} {g['launches']:>8} {g['us'] * 1e-3:>8.3f} {g['us'] / tot_us:>6.1%} {g['ops'] / g['us'] * 1e-6:>8.0f}")
    print(f"{'all':>5} {len(rows):>8} {tot_us * 1e-3:>8.3f} {1:>6.1%} {tot_ops / tot_us * 1e-6:>8.0f}")
    solo = {}
    print("\nstandalone update m = n = K = 4096 (gpk_debug_syrk_i8, lower tiles)")
    for c in (1, 2, 4):
        us = debug_update(4096, S, c, args.reps)
        ops = issued_ops(4096, 4096, 4096, S, c)
        solo[c] = {"us": us, "tops": ops / us * 1e-6}
        print(f"cluster {c}: {us:9.1f} us  {ops / us * 1e-6:6.0f} T op/s")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tc_update_profile.json"), "w") as f:
            json.dump({"device": torch.cuda.get_device_name(0), "S": S, "cluster": cl, "launches": rows,
                       "by_k": by_k, "standalone_4096": solo}, f, indent=1)


if __name__ == "__main__":
    main()
