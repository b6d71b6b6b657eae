"""Time one natural-gradient step at the C4 shape and its parts.

    python scripts/natgrad_time.py [--reps 10] [--warmup 2]

SVGP in float64 at the C4 shape (B = 4096, M = 2048, D = 16, P = 8; RBF + White, whiten=True, dense q_sqrt, Gaussian
likelihood), then the same with the MultiClass likelihood at C = P = 10 classes and random labels.  For each:
  * the fused value + gradient call (SVGP.elbo_and_grad with the q gradients left on the device);
  * gpk_natgrad_step alone for XiNat and XiSqrtMeanVar, with CUDA events around the call;
  * the device-to-host refresh of q_mu and q_sqrt (Parameter.assign_device of the step's outputs);
  * one whole NaturalGradient.minimize call, for each transform.
ms = host wall clock over `reps` calls ending in a device synchronise, except the step alone (CUDA events).  The step's
operation count comes from the shapes: per latent XiNat issues S^T gS (lower triangle, M^3 / 3 multiply-adds), the
Cholesky of J B J (M^3 / 6) and the triangular solve of M right-hand sides (M^3 / 2), 2 M^3 flops in all; XiSqrtMeanVar
issues S^T gS and the lower product S Phi(T) (M^3 / 6), M^3 flops.  The card name, power limit and maximum SM clock are
read in the same run and printed with the numbers.  Needs a CUDA device; there is no CPU fallback."""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        import torch
        return f"{torch.cuda.get_device_name(0)}, power limit unknown"


def wall(fn, reps: int, warmup: int) -> float:
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def events(fn, reps: int, warmup: int) -> float:
    import torch

    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def run(gpf, name: str, lik, P: int, Y, X, Z, reps: int, warmup: int) -> None:
    import torch

    from gpflow_b200 import _lib, ops

    K = gpf.kernels
    M = Z.shape[0]
    rng = np.random.default_rng(1)
    q_mu = 0.1 * rng.standard_normal((M, P))
    q_sqrt = np.stack([np.tril(0.02 * rng.standard_normal((M, M)), -1) + np.eye(M) for _ in range(P)])
    m = gpf.models.SVGP(K.SquaredExponential(lengthscales=4.0) + K.White(variance=0.01), lik, Z.copy(),
                        num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt, whiten=True, num_data=10 * X.shape[0])
    data = (ops.to_device(X), ops.to_device(Y))
    t_grad = wall(lambda: m.elbo_and_grad(data, device_arrays=True), reps, warmup)
    _, g = m.elbo_and_grad(data, device_arrays=True)
    gm, gS = g[m.q_mu], g[m.q_sqrt]
    lib = _lib.load()
    qm, qs = ops.to_device(m.q_mu), ops.to_device(m.q_sqrt)
    m_out, S_out = torch.empty_like(qm), torch.empty_like(qs)
    info = torch.empty((P,), dtype=torch.int32, device=qm.device)
    print(f"{name}: B = {X.shape[0]}, M = {M}, D = {X.shape[1]}, P = {P}, float64")
    print(f"  fused value + gradient (q gradients on the device): {t_grad:8.2f} ms")
    for xi, label, flops in ((_lib.GPK_XI_NAT, "XiNat", 2.0), (_lib.GPK_XI_SQRT_MEAN_VAR, "XiSqrtMeanVar", 1.0)):
        ws = ops.scratch_bytes(lib.gpk_natgrad_step_ws(M, P, xi, _lib.GPK_F64))

        def step():
            _lib.check(lib.gpk_natgrad_step(xi, M, P, ops._p(qm), ops._p(qs), ops._p(gm), ops._p(gS), 1e-3,
                                            _lib.GPK_F64, ops._p(m_out), ops._p(S_out), ops._p(info), ops._p(ws),
                                            ops._stream()), "gpk_natgrad_step")

        t = events(step, reps, warmup)
        if int(info.abs().sum()):
            print(f"  gpk_natgrad_step {label}: the step failed, info = {info.tolist()}")
        op = flops * P * M ** 3
        print(f"  gpk_natgrad_step {label:14s}: {t:8.2f} ms  ({op / 1e9:.1f} GFLOP, {op / t / 1e9:.2f} TFLOP/s)")
    probe_mu, probe_sq = gpf.base.Parameter(q_mu), gpf.base.Parameter(q_sqrt)
    t_d2h = wall(lambda: (probe_mu.assign_device(m_out), probe_sq.assign_device(S_out)), reps, warmup)
    print(f"  device-to-host refresh of q_mu and q_sqrt: {t_d2h:8.2f} ms  ({(m_out.numel() + S_out.numel()) * 8 / 1e6:.0f} MB)")
    for xi, label in ((gpf.optimizers.XiNat(), "XiNat"), (gpf.optimizers.XiSqrtMeanVar(), "XiSqrtMeanVar")):
        opt = gpf.optimizers.NaturalGradient(1e-3, xi_transform=xi)
        closure = m.training_loss_closure(data)
        t = wall(lambda: opt.minimize(closure, [(m.q_mu, m.q_sqrt)]), reps, warmup)
        print(f"  NaturalGradient.minimize {label:14s}: {t:8.2f} ms")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    import gpflow_b200 as gpf

    if not torch.cuda.is_available():
        raise SystemExit("natgrad_time.py needs a CUDA device")
    print(f"card: {card()}")
    rng = np.random.default_rng(0)
    B, M, D = 4096, 2048, 16
    X = rng.standard_normal((B, D))
    Z = rng.standard_normal((M, D))
    P = 8
    Y = np.sin(X[:, :P]) + 0.1 * rng.standard_normal((B, P))
    run(gpf, "SVGP Gaussian (C4)", gpf.likelihoods.Gaussian(0.1), P, Y, X, Z, a.reps, a.warmup)
    C = 10
    labels = rng.integers(0, C, (B, 1)).astype(np.float64)
    run(gpf, "SVGP MultiClass C = 10", gpf.likelihoods.MultiClass(C), C, labels, X, Z, a.reps, a.warmup)
    print(f"card: {card()}")


if __name__ == "__main__":
    main()
