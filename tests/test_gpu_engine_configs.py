"""Every documented engine configuration of the Cholesky / GEMM path, one process each.

The engine switches (GPK_TC_SLICES, GPK_TC_CLUSTER, GPK_FP64_ENGINE, GPK_LOOKAHEAD, ...) are read once per process, so a
test process by itself only ever sees the default configuration.  Each configuration here runs tests/_engine_worker.py in
its own subprocess on the same fixed matrices; the results are compared with LAPACK / the NumPy oracle, with the default
configuration and -- for the int8 tensor-core engine -- with the DMMA engine (GPK_FP64_ENGINE=dmma), in units of the row
scales sqrt(A_ii) of the factorised matrix, which is what the digit model of csrc/planes.cuh bounds."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg as sla

from tests import _engine_worker as W

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = {
    "default": {},
    "slices6": {"GPK_TC_SLICES": "6"},
    "slices7": {"GPK_TC_SLICES": "7"},
    "slices8": {"GPK_TC_SLICES": "8"},
    "cluster1": {"GPK_TC_CLUSTER": "1"},
    "cluster4": {"GPK_TC_CLUSTER": "4"},
    "dynamic_scales": {"GPK_TC_STATIC": "0"},
    "dmma": {"GPK_FP64_ENGINE": "dmma"},
    "no_lookahead": {"GPK_LOOKAHEAD": "0"},
    "no_flag_hops": {"GPK_FLAG_HOPS": "0"},
    "no_panel_fuse": {"GPK_PANEL_FUSE": "0"},
    "no_slim_leaf": {"GPK_SLIM_LEAF": "0"},
    "f32_native": {"GPK_F32_VIA_F64": "0"},
    "fp32_simt": {"GPK_FP32_ENGINE": "simt"},
    "tf32_cluster1": {"GPK_TF32_CLUSTER": "1"},
}


@functools.lru_cache(maxsize=None)
def run_config(name, tmpdir):
    """Runs the worker under CONFIGS[name] (every other GPK_* switch unset) and returns its results."""
    env = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    env.update(CONFIGS[name])
    out = os.path.join(tmpdir, f"{name}.npz")
    r = subprocess.run([sys.executable, "-m", "tests._engine_worker", out], cwd=ROOT, env=env, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, f"{name}: worker failed\n{r.stdout[-4000:]}"
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


@functools.lru_cache(maxsize=None)
def references():
    """LAPACK / fp64 NumPy / oracle values of the worker's workloads (computed once)."""
    from oracle import gp_oracle as O

    ref = {}
    for n in W.POTRF_N:
        A = W.spd(n, n)
        ref[f"potrf{n}"] = np.linalg.cholesky(A)
        ref[f"scale{n}"] = np.sqrt(np.diag(A))
    n, p = W.EXTRA
    A = W.spd(n, n + 1)
    L = np.linalg.cholesky(A)
    ref["extra"] = np.concatenate([L, sla.solve_triangular(L, W.extra_rows(n, p, 5).T, lower=True).T])
    ref["scale_extra"] = np.concatenate([np.sqrt(np.diag(A)), np.abs(ref["extra"][n:]).max(axis=1)])
    B = np.random.default_rng(3).standard_normal(W.TRSM)
    ref["trsm"] = sla.solve_triangular(ref[f"potrf{W.TRSM[0]}"], B, lower=True)
    d = O.make_data(2, W.GPR_N, 8, 1)
    ref["lml"] = O.gpr_log_marginal_likelihood(d["X"], d["Y"], O.Matern52(lengthscales=np.sqrt(8.0)), 0.1)
    A32 = W.spd(1000, 1000).astype(np.float32).astype(np.float64)
    ref["potrf32"] = np.linalg.cholesky(A32)
    ref["scale32"] = np.sqrt(np.diag(A32))
    Ag, Bg = W.gemm32_operands()
    ref["gemm32"] = Ag.astype(np.float64) @ Bg.astype(np.float64)
    ref["gemm32_scale"] = np.abs(Ag).astype(np.float64) @ np.abs(Bg).astype(np.float64)
    return ref


def factor_diff(a, b, ref):
    """max |a - b| over the fp64 factors, relative to the row scales sqrt(A_ii) (extra rows: their maxima)."""
    d = [np.abs(a[f"potrf{n}"] - b[f"potrf{n}"]).max(axis=1) / ref[f"scale{n}"] for n in W.POTRF_N]
    d.append(np.abs(a["extra"] - b["extra"]).max(axis=1) / ref["scale_extra"])
    return float(max(x.max() for x in d))


def metrics(res, ref):
    """Errors of one configuration's results against the references."""
    return dict(
        factor=factor_diff(res, ref, ref),
        trsm=float(np.abs(res["trsm"] - ref["trsm"]).max() / np.abs(ref["trsm"]).max()),
        lml=float(abs(res["lml"] - ref["lml"]) / abs(ref["lml"])),
        potrf32=float((np.abs(res["potrf32"] - ref["potrf32"]).max(axis=1) / ref["scale32"]).max()),
        gemm32=float((np.abs(res["gemm32"] - ref["gemm32"]) / ref["gemm32_scale"]).max()),
    )


# Bars against LAPACK / the oracle, about 10x the largest value measured over the configurations on an H100 (80 GB HBM3,
# 700 W): factor 4.7e-14 (S = 7, n = 4096), trsm 1.0e-13, lml 8.1e-13, potrf32 2.2e-7 (GPK_F32_VIA_F64=0), gemm32 3.3e-7
# (GPK_FP32_ENGINE=simt).  S = 6 digit planes resolve 2^-46 of the row scale: factor 1.1e-11, trsm 2.2e-11.
LAPACK_BARS = dict(factor=5e-13, trsm=1e-12, lml=1e-11, potrf32=2e-6, gemm32=3e-6)
LAPACK_BARS_S6 = dict(LAPACK_BARS, factor=1e-10, trsm=2e-10)


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("engine_configs"))


@pytest.mark.parametrize("name", list(CONFIGS))
def test_engine_configuration_matches_lapack(cuda_device, tmp, name):
    res = run_config(name, tmp)
    got = metrics(res, references())
    bars = LAPACK_BARS_S6 if name == "slices6" else LAPACK_BARS
    bad = {k: (v, bars[k]) for k, v in got.items() if not v <= bars[k]}
    assert not bad, f"{name}: {bad}"
    for n in W.POTRF_N:
        want = {"dmma": 0, "no_slim_leaf": 0, "slices6": 6, "slices8": 8}.get(name, 7)
        assert int(res[f"slices{n}"]) == want, (name, n, int(res[f"slices{n}"]))


# int8 engine vs DMMA engine on the same matrices, max over every factor of the worker relative to the row scales.  Measured
# on an H100 (80 GB HBM3, 700 W), largest at n = 4096: S = 6 1.1e-11, S = 7 4.7e-14, S = 8 1.3e-15 with the static row scales
# sqrt(A_ii) of the panel kernel, and 6.5e-16 at S = 7 with row-maximum scales (GPK_TC_STATIC=0: no leading digit bits
# unused).  The digit model's a-priori bound is K (S + 1) 2^(-8S+2) per dot product (2e-10 / 9e-13 / 4e-15 at K = 2048).
INT8_VS_DMMA_BARS = {"slices6": 1e-10, "default": 4e-13, "cluster1": 4e-13, "cluster4": 4e-13, "slices8": 1.3e-14,
                     "dynamic_scales": 6e-15}


@pytest.mark.parametrize("name", list(INT8_VS_DMMA_BARS))
def test_int8_factor_vs_dmma_factor(cuda_device, tmp, name):
    d = factor_diff(run_config(name, tmp), run_config("dmma", tmp), references())
    assert d <= INT8_VS_DMMA_BARS[name], (name, d)


# Values reduced with fp64 atomics (the LML sums alpha^2 and log diag L over CTAs): their last bits follow the order in
# which the atomics land, which changes from launch to launch, so they are compared to rounding, not bit for bit.
ATOMIC_OUTPUTS = {"lml": 1e-14}


@pytest.mark.parametrize("name", ["cluster1", "cluster4", "no_flag_hops", "tf32_cluster1"])
def test_schedule_switches_give_the_default_result(cuda_device, tmp, name):
    """Cluster widths and flag hops change who computes what when, not the arithmetic: the factors, solves and products
    equal the default bit for bit (the atomically reduced LML to rounding).  (GPK_LOOKAHEAD=0 also switches the panel fusion
    off, which applies one update in a different kernel.)"""
    a, b = run_config(name, tmp), run_config("default", tmp)
    assert set(a) == set(b)
    for k in a:
        if k in ATOMIC_OUTPUTS:
            np.testing.assert_allclose(a[k], b[k], rtol=ATOMIC_OUTPUTS[k], atol=0, err_msg=f"{name}: {k}")
        else:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{name}: {k}")


# The fused GPR LML, int8 engine (S = 6) vs DMMA engine: measured 6.9e-13 relative on an H100 (80 GB HBM3, 700 W).
LML_TC_VS_DMMA = 5e-12


def test_gpr_lml_tc_vs_dmma_engines(cuda_device, tmp):
    """The fused GPR LML (N = 2048, S = 6 digit planes from the conditioning hint) agrees between the int8 tensor-core
    engine and the DMMA engine (measured 6.9e-13 relative on an H100), and both with the oracle."""
    a, b, ref = run_config("default", tmp), run_config("dmma", tmp), references()
    assert int(a["lml_slices"]) == 6 and int(b["lml_slices"]) == 0
    np.testing.assert_allclose(a["lml"], b["lml"], rtol=LML_TC_VS_DMMA)
    np.testing.assert_allclose(a["lml"], ref["lml"], rtol=1e-9)
    np.testing.assert_allclose(b["lml"], ref["lml"], rtol=1e-9)

