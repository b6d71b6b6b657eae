"""Time the GPR value and value + gradient per evaluation, and the two gradient reductions' kernel times.

    python scripts/grad_time.py [--reps 20] [--warmup 3] [--out DIR] [--only-svgp] [--only-vgp] [--only-svgp-lik]
                                [--only-svgp-multiclass]

  * C5 (BASELINE configs[4]: (RBF + Matern32) * Linear, N = 4096, D = 32, four outputs on four CUDA streams as bench.py
    runs them): value only (gpk_gpr_lml) and value + gradient (gpk_gpr_lml_grad_expr).
  * C2 (Matern52, N = 8192, D = 8): value only, and value + gradient through gpk_gpr_lml_grad_expr twice: on the bare
    leaf (gpr_grad_kernel) and on the leaf under a one-child Sum node (gpr_grad_expr_kernel).
  * Then, in a torch.profiler run of its own, the device time of gpr_grad_kernel and gpr_grad_expr_kernel per launch.
  * SGPR at the C3 shape in float64 (BASELINE configs[2]: RBF, N = 100000, M = 1024, D = 16): value only
    (gpk_sgpr_elbo) and value + gradient (gpk_sgpr_elbo_grad, inducing points included), then in profiler runs of their
    own the kernel times of the G_uf GEMM (the longest GEMM launch after the forward's launches) and of the Kuf, Kuu
    and Kdiag passes of sgpr_grad_kernel.
  * SVGP at the C4 shape in float64 (B = 4096, M = 2048, P = 8, D = 16; RBF + White, whiten=True, dense q_sqrt): value
    only (gpk_svgp_elbo) and value + gradient (gpk_svgp_elbo_grad), then in a profiler run of its own the backward's
    GEMM and pass times.
  * VGP in float64 (N = 4096, D = 8, P = 1; RBF): VGP.elbo() and value + gradient (gpk_vgp_elbo_grad), then in a
    profiler run of its own the grad call's GEMM and square-pass times.
  * SVGP with non-Gaussian likelihoods at the C4 shape in float64 (B = 4096, M = 2048, D = 16; RBF + White, whitened,
    dense q_sqrt): Bernoulli at P = 1 and Student-t at P = 8, value (SVGP.elbo, the unfused route) and value + gradient
    (gpk_svgp_elbo_grad), then in a profiler run of its own the grad call's GEMM, element-pass and likelihood
    kernel times.
  * SVGP with the MultiClass (RobustMax) likelihood at the C4 shape in float64 with C = P = 10 classes and random
    labels: value (SVGP.elbo) and value + gradient, then in a profiler run of its own the grad call's GEMM,
    element-pass and MultiClass kernel times.
ms per evaluation = host wall clock over `reps` evaluations ending in a device synchronise.  The card name, power limit
and maximum SM clock are read with the numbers and printed with them.  Needs a CUDA device; there is no CPU fallback."""
from __future__ import annotations

import argparse
import ctypes
import json
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


class Enq:
    """Enqueues one fused call of a model on the current stream from the model's own workspace (no host read): fn =
    "value" (gpk_gpr_lml), "single" (gpk_gpr_lml_grad_expr) or "expr" (the same, the kernel under a one-child Sum node,
    which takes a single stationary leaf from gpr_grad_kernel to gpr_grad_expr_kernel)."""

    def __init__(self, gpf, m, fn: str):
        from gpflow_b200 import _lib, ops

        self.lib, self.ops, self.fn = _lib.load(), ops, fn
        X, Y = m.data
        self.X, self.Y = X, Y.contiguous()
        self.N, self.D = X.shape
        self.P = Y.shape[1]
        self.desc = gpf.kernels.compile_kernel(m.kernel, self.D)
        if fn == "expr" and self.desc[1] == 1:
            nodes = (_lib.KNode * 2)(self.desc[0][0])
            nodes[1].op, nodes[1].n_children, nodes[1].child[0] = _lib.K_SUM, 1, 0
            self.desc = (nodes, 2) + tuple(self.desc[2:])
        self.s2 = m.likelihood._variance_value()
        T = ops.torch()
        if fn == "value":
            self.ws = ops.scratch_bytes(self.lib.gpk_gpr_lml_ws(self.N, self.P, _lib.GPK_F64))
            self.out = T.empty((4,), dtype=T.float64, device=X.device)
        else:
            self.ws = ops.scratch_bytes(self.lib.gpk_gpr_lml_grad_ws(self.N, self.P, _lib.GPK_F64))
            n = self.lib.gpk_gpr_lml_grad_slots(*self.desc, self.D) + 5
            self.n_out = n
            self.out = T.empty((n,), dtype=T.float64, device=X.device)

    def __call__(self):
        from gpflow_b200 import _lib

        o, L = self.ops, self.lib
        nodes, n, dims, ard = self.desc
        if self.fn == "value":
            st = L.gpk_gpr_lml(nodes, n, dims, ard, o._p(self.X), self.N, o._ld(self.X), self.D, o._p(self.Y), self.P,
                               self.s2, None, _lib.GPK_F64, o._p(self.out), o._p(self.ws), o._stream())
        else:
            st = L.gpk_gpr_lml_grad_expr(nodes, n, dims, ard, o._p(self.X), self.N, o._ld(self.X), self.D, o._p(self.Y),
                                         self.P, self.s2, _lib.GPK_F64, o._p(self.out), self.n_out, o._p(self.ws),
                                         o._stream())
        _lib.check(st, self.fn)


class SgprEnq:
    """Enqueues one gpk_sgpr_elbo (fn="value") or gpk_sgpr_elbo_grad (fn="grad") call of an SGPR model."""

    def __init__(self, gpf, m, fn: str):
        from gpflow_b200 import _lib, ops

        self.lib, self.ops, self.fn = _lib.load(), ops, fn
        X, Y = m.data
        self.X, self.Y = X, Y.contiguous()
        self.Z = ops.to_device(m.inducing_variable.Z)
        self.N, self.D = X.shape
        self.P = Y.shape[1]
        self.M = self.Z.shape[0]
        self.desc = gpf.kernels.compile_kernel(m.kernel, self.D)
        self.s2 = m.likelihood._variance_value()
        T = ops.torch()
        if fn == "value":
            self.ws = ops.scratch_bytes(self.lib.gpk_sgpr_elbo_ws(self.N, self.M, self.P, _lib.GPK_F64))
            self.out = T.empty((8,), dtype=T.float64, device=X.device)
        else:
            self.ws = ops.scratch_bytes(self.lib.gpk_sgpr_elbo_grad_ws(self.N, self.M, self.P, _lib.GPK_F64))
            self.n_out = 9 + self.lib.gpk_gpr_lml_grad_slots(*self.desc, self.D)
            self.out = T.empty((self.n_out,), dtype=T.float64, device=X.device)
            self.dZ = T.empty((self.M, self.D), dtype=T.float64, device=X.device)

    def __call__(self):
        from gpflow_b200 import _lib

        o, L = self.ops, self.lib
        nodes, n, dims, ard = self.desc
        args = (nodes, n, dims, ard, o._p(self.X), self.N, o._ld(self.X), self.D, o._p(self.Y), self.P, o._p(self.Z),
                self.M, o._ld(self.Z), self.s2, 1e-6, _lib.GPK_F64, o._p(self.out))
        if self.fn == "value":
            st = L.gpk_sgpr_elbo(*args, None, None, None, o._p(self.ws), o._stream())
        else:
            st = L.gpk_sgpr_elbo_grad(*args, self.n_out, o._p(self.dZ), o._p(self.ws), o._stream())
        _lib.check(st, "sgpr_" + self.fn)


class SvgpEnq:
    """Enqueues one gpk_svgp_elbo call of an SVGP model with a Gaussian likelihood on a batch (no host read)."""

    def __init__(self, gpf, m, data):
        from gpflow_b200 import _lib, ops

        self.lib, self.ops, self.m = _lib.load(), ops, m
        self.X, self.Y = (ops.to_device(t).contiguous() for t in data)
        self.Z = ops.to_device(m.inducing_variable.Z)
        self.q_mu, self.q_sqrt = ops.to_device(m.q_mu), ops.to_device(m.q_sqrt)
        self.B, self.D = self.X.shape
        self.P = self.Y.shape[1]
        self.M = self.Z.shape[0]
        self.desc = gpf.kernels.compile_kernel(m.kernel, self.D)
        self.lik = m.likelihood._lik_desc()
        self.scale = float(m.num_data) / self.B if m.num_data else 1.0
        self.ws = ops.scratch_bytes(self.lib.gpk_svgp_elbo_ws(self.B, self.M, self.P, _lib.GPK_F64))
        self.out = ops.torch().empty((4,), dtype=ops.torch().float64, device=self.X.device)

    def __call__(self):
        from gpflow_b200 import _lib, config

        o, m = self.ops, self.m
        _lib.check(self.lib.gpk_svgp_elbo(*self.desc, o._p(self.X), self.B, o._ld(self.X), self.D, o._p(self.Y), None,
                                          self.P, o._p(self.Z), self.M, o._ld(self.Z), o._p(self.q_mu),
                                          o._p(self.q_sqrt), int(m.q_diag), int(m.whiten), ctypes.byref(self.lik),
                                          self.scale, config.default_jitter(), 0, self.P, _lib.GPK_F64, o._p(self.out),
                                          o._p(self.ws), o._stream()),
                   "svgp_value")


class SvgpGradEnq:
    """Enqueues one gpk_svgp_elbo_grad call of an SVGP model (zero mean) on a batch with the likelihood descriptor
    `lik` (default: the model's), from its own workspace (no host read)."""

    def __init__(self, gpf, m, data, lik=None):
        from gpflow_b200 import _lib, config, ops

        self.lib, self.ops = _lib.load(), ops
        self.X, self.Y = (ops.to_device(a).contiguous() for a in data)
        self.B, self.D = self.X.shape
        self.Z = ops.to_device(m.inducing_variable.Z)
        self.M, self.P = self.Z.shape[0], m.num_latent_gps
        self.q_mu, self.q_sqrt = ops.to_device(m.q_mu), ops.to_device(m.q_sqrt)
        self.m = m
        self.kdesc = gpf.kernels.compile_kernel(m.kernel, self.D)
        self.lik = m.likelihood._lik_desc() if lik is None else lik
        self.scale = m._scale(data, None)
        self.jitter = config.default_jitter()
        T = ops.torch()
        self.n_out = 5 + self.lib.gpk_gpr_lml_grad_slots(*self.kdesc, self.D)
        self.out = T.empty((self.n_out,), dtype=T.float64, device=self.X.device)
        self.dZ = T.empty((self.M, self.D), dtype=T.float64, device=self.X.device)
        self.dq_mu = T.empty(tuple(self.q_mu.shape), dtype=T.float64, device=self.X.device)
        self.dq_sqrt = T.empty(tuple(self.q_sqrt.shape), dtype=T.float64, device=self.X.device)
        self.ws = ops.scratch_bytes(self.lib.gpk_svgp_elbo_grad_ws(self.B, self.M, self.P, ctypes.byref(self.lik),
                                                                   _lib.GPK_F64))

    def __call__(self):
        from gpflow_b200 import _lib

        o, L, m = self.ops, self.lib, self.m
        _lib.check(L.gpk_svgp_elbo_grad(*self.kdesc, o._p(self.X), self.B, o._ld(self.X), self.D, o._p(self.Y), None,
                                        self.P, o._p(self.Z), self.M, o._ld(self.Z), o._p(self.q_mu), o._p(self.q_sqrt),
                                        int(m.q_diag), int(m.whiten), ctypes.byref(self.lik), self.scale, self.jitter,
                                        _lib.GPK_F64, o._p(self.out), self.n_out, o._p(self.dZ), o._p(self.dq_mu),
                                        o._p(self.dq_sqrt), o._p(self.ws), o._stream()), "svgp_grad")


def svgp_leg(T, gpf, O, reps: int, warmup: int) -> dict:
    """SVGP at the C4 shape in float64 (B = 4096, M = 2048, P = 8, D = 16, num_data = 1e6; RBF + White, whitened, dense
    q_sqrt): ms per evaluation of the value and of value + gradient, then from a profiler run of its own the backward's
    kernels (the grad call's launches after the forward's): all GEMM launches (the triangular solves included, which
    run on the same GEMM kernels), the three element passes, and the twelve longest kernels by name."""
    B, M, P, D = 4096, 2048, 8, 16
    d = O.make_data(4, B, D, P, M=M)
    q_mu, q_sqrt = O.make_q(4, M, P)
    res = {}
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
        K = gpf.kernels
        m = gpf.models.SVGP(K.SquaredExponential(variance=1.0, lengthscales=4.0) + K.White(variance=0.01),
                            gpf.likelihoods.Gaussian(0.1), d["Z"], num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt,
                            whiten=True, num_data=1000000)
        data = (d["X"], d["Y"])
        sv = {"value": SvgpEnq(gpf, m, data), "grad": SvgpGradEnq(gpf, m, data)}
        for fn in ("value", "grad"):
            res[f"c4_svgp_{fn}_ms"] = ms_per_eval(T, sv[fn], reps, warmup)
        v4, g4 = sv["value"].out.cpu().numpy(), sv["grad"].out.cpu().numpy()[:4]
        res["c4_svgp_value_vs_grad_entry_max_rel_diff"] = float(np.max(np.abs(v4 - g4) /
                                                                       np.maximum(np.abs(v4), 1e-300)))
        fwd = cuda_kernels(T, sv["value"])
        bwd = cuda_kernels(T, sv["grad"])[len(fwd):]
    by_name: dict = {}
    for n, t in bwd:
        key = n.split("(")[0][:60]
        by_name[key] = by_name.get(key, 0.0) + float(t)
    passes = [float(t) for n, t in bwd if "sgpr_grad_kernel" in n]
    res["c4_svgp_backward_us"] = {
        "total": float(sum(t for _, t in bwd)),
        "gemm": float(sum(t for n, t in bwd if "gemm" in n.lower())),
        "Kuf pass": passes[0] if len(passes) == 3 else float("nan"),
        "Kuu pass": passes[1] if len(passes) == 3 else float("nan"),
        "Kdiag pass": passes[2] if len(passes) == 3 else float("nan"),
        "by kernel": dict(sorted(by_name.items(), key=lambda e: -e[1])[:12]),
    }
    return res


class VgpEnq:
    """Enqueues one gpk_vgp_elbo_grad call of a VGP model from its own workspace (no host read)."""

    def __init__(self, gpf, m):
        from gpflow_b200 import _lib, ops

        self.lib, self.ops, self.m = _lib.load(), ops, m
        self.X, self.Y = (ops.to_device(t).contiguous() for t in m.data)
        self.q_mu, self.q_sqrt = ops.to_device(m.q_mu), ops.to_device(m.q_sqrt)
        self.N, self.D = self.X.shape
        self.P = self.Y.shape[1]
        self.desc = gpf.kernels.compile_kernel(m.kernel, self.D)
        T = ops.torch()
        dev = self.X.device
        self.ws = ops.scratch_bytes(self.lib.gpk_vgp_elbo_grad_ws(self.N, self.P, _lib.GPK_F64))
        self.n_out = 5 + self.lib.gpk_gpr_lml_grad_slots(*self.desc, self.D)
        self.out = T.empty((self.n_out,), dtype=T.float64, device=dev)
        self.dq_mu, self.dq_sqrt = T.empty_like(self.q_mu), T.empty_like(self.q_sqrt)

    def __call__(self):
        from gpflow_b200 import _lib, config

        o = self.ops
        _lib.check(self.lib.gpk_vgp_elbo_grad(*self.desc, o._p(self.X), self.N, o._ld(self.X), self.D, o._p(self.Y),
                                              self.P, o._p(self.q_mu), o._p(self.q_sqrt),
                                              self.m.likelihood._variance_value(), config.default_jitter(),
                                              _lib.GPK_F64, o._p(self.out), self.n_out, o._p(self.dq_mu),
                                              o._p(self.dq_sqrt), o._p(self.ws), o._stream()), "vgp_grad")


def vgp_leg(T, gpf, O, reps: int, warmup: int) -> dict:
    """VGP in float64 (N = 4096, D = 8, P = 1; RBF): ms per evaluation of VGP.elbo() (the operator-by-operator value)
    and of gpk_vgp_elbo_grad (value + gradient in one call), then from a profiler run of its own the grad call's kernels:
    all GEMM launches (the triangular solves and the lauum included, which run on the same GEMM kernels), the square
    element pass, and the twelve longest kernels by name."""
    N, D, P = 4096, 8, 1
    d = O.make_data(9, N, D, P)
    rng = np.random.default_rng(9)
    q_mu = 0.3 * rng.standard_normal((N, P))
    q_sqrt = (np.tril(0.01 * rng.standard_normal((N, N)), -1) + np.diag(0.5 + 0.5 * rng.random(N)))[None]
    res = {}
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-6)):
        m = gpf.models.VGP((d["X"], d["Y"]), gpf.kernels.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))),
                           gpf.likelihoods.Gaussian(0.1))
        m.q_mu.assign(q_mu)
        m.q_sqrt.assign(q_sqrt)
        grad = VgpEnq(gpf, m)
        res["vgp_value_ms"] = ms_per_eval(T, m.elbo, reps, warmup)
        res["vgp_grad_ms"] = ms_per_eval(T, grad, reps, warmup)
        v, g = float(m.elbo()), float(grad.out[0].cpu())
        res["vgp_value_vs_grad_entry_rel_diff"] = abs(v - g) / abs(v)
        ks = cuda_kernels(T, grad)
    by_name: dict = {}
    for n, t in ks:
        key = n.split("(")[0][:60]
        by_name[key] = by_name.get(key, 0.0) + float(t)
    res["vgp_grad_us"] = {
        "total": float(sum(t for _, t in ks)),
        "gemm": float(sum(t for n, t in ks if "gemm" in n.lower())),
        "square pass": float(sum(t for n, t in ks if "sgpr_grad_kernel" in n)),
        "by kernel": dict(sorted(by_name.items(), key=lambda e: -e[1])[:12]),
    }
    return res


def svgp_lik_leg(T, gpf, O, reps: int, warmup: int) -> dict:
    """SVGP at the C4 shape in float64 with a Bernoulli likelihood (P = 1) and a Student-t likelihood (P = 8): ms per
    evaluation of SVGP.elbo (the unfused route: prior_kl, predict_f, the likelihood's variational expectations) and of
    gpk_svgp_elbo_grad, then from a profiler run of its own the grad call's GEMM, element-pass (sgpr_grad_kernel)
    and likelihood (lik_*) kernel times."""
    B, M, D = 4096, 2048, 16
    res = {}
    for name, P in (("bernoulli", 1), ("student_t", 8)):
        d = O.make_data(4, B, D, P, M=M)
        q_mu, q_sqrt = O.make_q(4, M, P)
        rng = np.random.default_rng(4)
        if name == "bernoulli":
            Y = (d["Y"] > np.median(d["Y"])).astype(np.float64)
            lik = gpf.likelihoods.Bernoulli()
        else:
            Y = d["Y"] + 0.3 * rng.standard_t(3.0, d["Y"].shape)
            lik = gpf.likelihoods.StudentT(scale=0.5)
        with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
            k = gpf.kernels.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) \
                + gpf.kernels.White(variance=0.01)
            m = gpf.models.SVGP(k, lik, d["Z"], num_latent_gps=P, q_mu=q_mu, q_sqrt=q_sqrt, whiten=True,
                                num_data=1000000)
            data = (gpf.ops.to_device(d["X"]), gpf.ops.to_device(Y))
            grad = SvgpGradEnq(gpf, m, data)
            key = f"c4_{name}_p{P}"
            res[f"{key}_value_ms"] = ms_per_eval(T, lambda: m.elbo(data), reps, warmup)
            res[f"{key}_grad_ms"] = ms_per_eval(T, grad, reps, warmup)
            v, g = float(m.elbo(data)), float(grad.out[0].cpu())
            res[f"{key}_value_vs_grad_entry_rel_diff"] = abs(v - g) / abs(v)
            ks = cuda_kernels(T, grad)
        res[f"{key}_grad_us"] = {
            "total": float(sum(t for _, t in ks)),
            "gemm": float(sum(t for n, t in ks if "gemm" in n.lower())),
            "element passes": float(sum(t for n, t in ks if "sgpr_grad_kernel" in n)),
            "likelihood kernels": float(sum(t for n, t in ks if "lik_" in n)),
        }
    return res


def svgp_multiclass_leg(T, gpf, O, reps: int, warmup: int) -> dict:
    """SVGP at the C4 shape in float64 with MultiClass(10) and random labels: ms per evaluation of SVGP.elbo (the
    unfused route) and of gpk_svgp_elbo_grad, then from a profiler run of its own the grad call's GEMM, element-pass
    (sgpr_grad_kernel) and MultiClass (mc_*) kernel times."""
    B, M, D, C = 4096, 2048, 16, 10
    d = O.make_data(4, B, D, 1, M=M)
    q_mu, q_sqrt = O.make_q(4, M, C)
    Y = np.random.default_rng(4).integers(0, C, (B, 1)).astype(np.float64)
    with gpf.config.as_context(gpf.config.Config(float=np.float64, jitter=1e-4)):
        k = gpf.kernels.SquaredExponential(variance=1.0, lengthscales=float(np.sqrt(D))) + gpf.kernels.White(variance=0.01)
        m = gpf.models.SVGP(k, gpf.likelihoods.MultiClass(C), d["Z"], num_latent_gps=C, q_mu=q_mu, q_sqrt=q_sqrt,
                            whiten=True, num_data=1000000)
        data = (gpf.ops.to_device(d["X"]), gpf.ops.to_device(Y))
        grad = SvgpGradEnq(gpf, m, data)
        key = f"c4_multiclass_c{C}"
        res = {f"{key}_value_ms": ms_per_eval(T, lambda: m.elbo(data), reps, warmup),
               f"{key}_grad_ms": ms_per_eval(T, grad, reps, warmup)}
        v, g = float(m.elbo(data)), float(grad.out[0].cpu())
        res[f"{key}_value_vs_grad_entry_rel_diff"] = abs(v - g) / abs(v)
        ks = cuda_kernels(T, grad)
        kv = cuda_kernels(T, lambda: m.elbo(data))
    res[f"{key}_grad_us"] = {
        "total": float(sum(t for _, t in ks)),
        "gemm": float(sum(t for n, t in ks if "gemm" in n.lower())),
        "element passes": float(sum(t for n, t in ks if "sgpr_grad_kernel" in n)),
        "multiclass kernels": float(sum(t for n, t in ks if "mc_" in n)),
    }
    res[f"{key}_value_us"] = {"total": float(sum(t for _, t in kv)),
                              "multiclass kernels": float(sum(t for n, t in kv if "mc_" in n))}
    return res


def cuda_kernels(T, call):
    """[(name, device us)] of the kernels of one call (memsets and copies left out), in start order, from a profiler run
    of its own."""
    from torch.profiler import ProfilerActivity, profile

    T.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        T.cuda.synchronize()
    evs = [ev for ev in prof.events() if ev.device_type.name == "CUDA" and not ev.name.startswith(("Memset", "Memcpy"))]
    evs.sort(key=lambda ev: ev.time_range.start)
    return [(ev.name, ev.device_time if hasattr(ev, "device_time") else ev.cuda_time) for ev in evs]


def run_streams(T, calls, streams):
    cur = T.cuda.current_stream()
    for c, s in zip(calls, streams):
        s.wait_stream(cur)
        with T.cuda.stream(s):
            c()
    for s in streams:
        cur.wait_stream(s)


def ms_per_eval(T, step, reps: int, warmup: int) -> float:
    for _ in range(warmup):
        step()
    T.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    T.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only-svgp", action="store_true", help="time the SVGP leg alone")
    ap.add_argument("--only-vgp", action="store_true", help="time the VGP leg alone")
    ap.add_argument("--only-svgp-lik", action="store_true",
                    help="time the SVGP leg with Bernoulli and Student-t likelihoods alone")
    ap.add_argument("--only-svgp-multiclass", action="store_true",
                    help="time the SVGP leg with the MultiClass likelihood alone")
    a = ap.parse_args()
    import torch as T

    import gpflow_b200 as gpf
    from oracle import gp_oracle as O

    if not T.cuda.is_available():
        raise SystemExit("grad_time.py needs a CUDA device")
    K = gpf.kernels
    res = {"card": card()}
    if a.only_svgp:
        res.update(svgp_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
        emit(res, a.out)
        return
    if a.only_vgp:
        res.update(vgp_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
        emit(res, a.out)
        return
    if a.only_svgp_lik:
        res.update(svgp_lik_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
        emit(res, a.out)
        return
    if a.only_svgp_multiclass:
        res.update(svgp_multiclass_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
        emit(res, a.out)
        return
    # C5: four outputs, four streams
    d = O.make_data(5, 4096, 32, 4)
    Xd = gpf.ops.to_device(d["X"])
    s = float(np.sqrt(32))
    c5 = [gpf.models.GPR((Xd, d["Y"][:, p:p + 1].copy()),
                         (K.SquaredExponential(variance=1.0 + 0.1 * p, lengthscales=s * (1 + 0.05 * p))
                          + K.Matern32(variance=1.0, lengthscales=2 * s)) * K.Linear(variance=1.0 / (1 + p)),
                         noise_variance=0.1) for p in range(4)]
    streams = [T.cuda.Stream() for _ in c5]
    for fn in ("value", "expr"):
        calls = [Enq(gpf, m, fn) for m in c5]
        res[f"c5_{fn}_ms"] = ms_per_eval(T, lambda: run_streams(T, calls, streams), a.reps, a.warmup)
    # C2: one model
    d2 = O.make_data(2, 8192, 8, 1)
    c2 = gpf.models.GPR((d2["X"], d2["Y"]), K.Matern52(variance=1.0, lengthscales=float(np.sqrt(8))), noise_variance=0.1)
    c2_calls = {}
    for fn in ("value", "single", "expr"):
        c2_calls[fn] = Enq(gpf, c2, fn)
        res[f"c2_{fn}_ms"] = ms_per_eval(T, c2_calls[fn], a.reps, a.warmup)
    g1, g2 = c2_calls["single"].out.cpu().numpy(), c2_calls["expr"].out.cpu().numpy()
    res["c2_single_vs_expr_max_rel_diff"] = float(np.max(np.abs(g1[4:7] - g2[4:7])) / np.max(np.abs(g2[4:7])))
    # kernel times, profiler on, in a run of their own
    from torch.profiler import ProfilerActivity, profile

    T.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            c2_calls["single"]()
            c2_calls["expr"]()
        calls = [Enq(gpf, m, "expr") for m in c5]
        for _ in range(5):
            run_streams(T, calls, streams)
        T.cuda.synchronize()
    kt = {}
    for ev in sorted(prof.events(), key=lambda ev: ev.time_range.start):
        name = ev.name
        for key in ("gpr_grad_expr_kernel", "gpr_grad_kernel"):
            if key + "<" in name and ev.device_type.name == "CUDA":
                kt.setdefault(key, []).append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
    # gpr_grad_expr_kernel ran 5x on C2 first, then 20x on C5 (4 per evaluation)
    e = kt.get("gpr_grad_expr_kernel", [])
    res["kernel_us"] = {
        "gpr_grad_kernel C2": float(np.median(kt.get("gpr_grad_kernel", [float("nan")]))),
        "gpr_grad_expr_kernel C2": float(np.median(e[:5])) if len(e) >= 5 else float("nan"),
        "gpr_grad_expr_kernel C5 (one output)": float(np.median(e[5:])) if len(e) > 5 else float("nan"),
    }
    # SGPR at the C3 shape, float64
    d3 = O.make_data(3, 100000, 16, 1, M=1024)
    c3 = gpf.models.SGPR((d3["X"], d3["Y"]), K.SquaredExponential(variance=1.0, lengthscales=4.0), d3["Z"],
                         noise_variance=0.1)
    sg = {fn: SgprEnq(gpf, c3, fn) for fn in ("value", "grad")}
    for fn in ("value", "grad"):
        res[f"c3_sgpr_{fn}_ms"] = ms_per_eval(T, sg[fn], max(a.reps // 2, 3), a.warmup)
    v8, g8 = sg["value"].out.cpu().numpy(), sg["grad"].out.cpu().numpy()[:8]
    res["c3_sgpr_value_vs_grad_entry_max_rel_diff"] = float(np.max(np.abs(v8 - g8) / np.maximum(np.abs(v8), 1e-300)))
    fwd = cuda_kernels(T, sg["value"])
    bwd = cuda_kernels(T, sg["grad"])[len(fwd):]
    gemms = [(n, t) for n, t in bwd if "gemm" in n.lower()]
    passes = [t for n, t in bwd if "sgpr_grad_kernel" in n]
    res["c3_sgpr_kernel_us"] = {
        "G_uf GEMM": float(max(t for _, t in gemms)) if gemms else float("nan"),
        "G_uf GEMM kernel": max(gemms, key=lambda e: e[1])[0][:80] if gemms else "",
        "Kuf pass": float(passes[0]) if len(passes) == 3 else float("nan"),
        "Kuu pass": float(passes[1]) if len(passes) == 3 else float("nan"),
        "Kdiag pass": float(passes[2]) if len(passes) == 3 else float("nan"),
        "backward total": float(sum(t for _, t in bwd)),
    }
    res.update(svgp_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
    res.update(vgp_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
    res.update(svgp_lik_leg(T, gpf, O, max(a.reps // 2, 3), a.warmup))
    emit(res, a.out)


def emit(res: dict, out) -> None:
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "grad_time.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
