"""Time one SVGP training iteration at the C4 shape, three ways, and profile the Adam step.

    python scripts/train_step_time.py [--rounds 4] [--per-round 5] [--warmup 3]

SVGP in float64 at the C4 shape (B = 4096, M = 2048, D = 16, P = 8; RBF + White, whiten=True, dense q_sqrt, Gaussian
likelihood), every parameter trainable unless stated:
  (g) the fused value + gradient call alone, gradients of Z, q_mu and q_sqrt left on the device;
  (a) the loop a user writes by hand on `training_loss_closure(data).value_and_gradients`: gradients copied to the host,
      the Adam update in NumPy, `assign_unconstrained` (the next evaluation uploads the values again);
  (b) `optimizers.Adam.minimize` over all trainable parameters;
  (c) `NaturalGradient.minimize` on (q_mu, q_sqrt), made untrainable, then `Adam.minimize` on the rest.
ms per iteration = host wall clock around one iteration that ends in a device synchronise.  (g), (a), (b) and (c)
alternate in rounds of `per-round` iterations after `warmup` iterations each; the median and the range over all timed
iterations are printed.  A separate `torch.profiler` run of (b) gives the time of `adam_step_kernel`, the bytes it
moves (56 B per element of Z, q_mu and q_sqrt: value, gradient and two moments read, value and moments written) over
that time against the 3.35 TB/s of the H100 SXM data sheet, and the bytes of every memory copy per iteration.  The card
name, power limit and maximum SM clock are read in the same run and printed with the numbers.  Needs a CUDA device;
there is no CPU fallback."""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from scripts.natgrad_time import card  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM data sheet, a card allowed 700 W


def model(gpf, X, Z, P: int):
    K = gpf.kernels
    M = Z.shape[0]
    rng = np.random.default_rng(1)
    q_mu = 0.1 * rng.standard_normal((M, P))
    q_sqrt = np.stack([np.tril(0.02 * rng.standard_normal((M, M)), -1) + np.eye(M) for _ in range(P)])
    return gpf.models.SVGP(K.SquaredExponential(lengthscales=4.0) + K.White(variance=0.01),
                           gpf.likelihoods.Gaussian(0.1), Z.copy(), num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt,
                           whiten=True, num_data=10 * X.shape[0])


def host_adam_loop(m, closure, lr=1e-3, beta_1=0.9, beta_2=0.999, epsilon=1e-7):
    """(a): one iteration per call, everything but the gradient evaluation on the host."""
    variables = m.trainable_variables
    state = [(np.zeros(p.shape), np.zeros(p.shape)) for p in variables]
    t = [0]

    def step():
        t[0] += 1
        _, grads = closure.value_and_gradients(variables)
        lr_t = lr * np.sqrt(1.0 - beta_2 ** t[0]) / (1.0 - beta_1 ** t[0])
        for p, g, (mm, vv) in zip(variables, grads, state):
            g = np.asarray(g).reshape(p.shape)
            mm += (1.0 - beta_1) * (g - mm)
            vv += (1.0 - beta_2) * (g * g - vv)
            p.assign_unconstrained(p.unconstrained_variable - lr_t * mm / (np.sqrt(vv) + epsilon))

    return step


def timed(fn) -> float:
    import torch

    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def profile_adam(step, iters: int, step_bytes: int) -> None:
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(iters):
                step()
            torch.cuda.synchronize()
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    adam = [e["dur"] for e in events if e.get("cat") == "kernel" and "adam_step_kernel" in e.get("name", "")]
    if len(adam) != iters:
        raise SystemExit(f"expected {iters} adam_step_kernel launches in the profile, found {len(adam)}")
    us = float(np.median(adam))
    rate = step_bytes / (us * 1e-6)
    print(f"  adam_step_kernel: {us / 1e3:.3f} ms median of {iters} ({min(adam) / 1e3:.3f} .. {max(adam) / 1e3:.3f}), "
          f"{step_bytes / 1e9:.3f} GB moved, {rate / 1e12:.2f} TB/s = {100 * rate / PEAK_BYTES_PER_S:.0f}% of the "
          "3.35 TB/s data-sheet bandwidth")
    copies = {}
    for e in events:
        if e.get("cat") == "gpu_memcpy":
            n, b = copies.get(e["name"], (0, 0))
            copies[e["name"]] = (n + 1, b + int(e.get("args", {}).get("bytes", 0)))
    print(f"  memory copies per iteration of Adam.minimize (profile of {iters} iterations):")
    for name, (n, b) in sorted(copies.items()):
        print(f"    {name}: {n / iters:.1f} copies, {b / iters:.0f} B")
    if not copies:
        print("    none recorded")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--per-round", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    import gpflow_b200 as gpf
    from gpflow_b200 import ops

    if not torch.cuda.is_available():
        raise SystemExit("train_step_time.py needs a CUDA device")
    print(f"card: {card()}")
    rng = np.random.default_rng(0)
    B, M, D, P = 4096, 2048, 16, 8
    X = rng.standard_normal((B, D))
    Z = rng.standard_normal((M, D))
    Y = np.sin(X[:, :P]) + 0.1 * rng.standard_normal((B, P))
    data = (ops.to_device(X), ops.to_device(Y))
    OPT = gpf.optimizers

    mg = model(gpf, X, Z, P)
    ma = model(gpf, X, Z, P)
    mb = model(gpf, X, Z, P)
    mc = model(gpf, X, Z, P)
    gpf.utilities.set_trainable([mc.q_mu, mc.q_sqrt], False)
    adam_b, adam_c, natgrad = OPT.Adam(), OPT.Adam(), OPT.NaturalGradient(1e-3)
    closure_b, closure_c = mb.training_loss_closure(data), mc.training_loss_closure(data)

    def step_c():
        natgrad.minimize(closure_c, [(mc.q_mu, mc.q_sqrt)])
        adam_c.minimize(closure_c, mc.trainable_variables)

    ways = [("(g) value + gradient alone", lambda: mg.elbo_and_grad(data, device_arrays=True)),
            ("(a) hand-written host loop", host_adam_loop(ma, ma.training_loss_closure(data))),
            ("(b) Adam.minimize, all parameters", lambda: adam_b.minimize(closure_b, mb.trainable_variables)),
            ("(c) NaturalGradient + Adam", step_c)]
    for _, fn in ways:
        for _ in range(a.warmup):
            timed(fn)
    times = {name: [] for name, _ in ways}
    for _ in range(a.rounds):
        for name, fn in ways:
            times[name] += [timed(fn) for _ in range(a.per_round)]
    print(f"SVGP Gaussian (C4): B = {B}, M = {M}, D = {D}, P = {P}, float64; ms per iteration, median (min .. max) of "
          f"{a.rounds * a.per_round} in {a.rounds} alternating rounds")
    for name, _ in ways:
        t = times[name]
        print(f"  {name:36s}: {np.median(t):8.2f}  ({min(t):.2f} .. {max(t):.2f})")
    n = sum(int(np.prod(p.shape)) for p in (mb.inducing_variable.Z, mb.q_mu, mb.q_sqrt))
    profile_adam(ways[2][1], 5, 56 * n)
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
