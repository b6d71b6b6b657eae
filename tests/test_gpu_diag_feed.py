"""The diagonal feed (potrf.cu: diag_feed_old_kernel, PanelFuse::feed): in front of an int8 trailing update of
K <= GPK_DIAG_FEED_MAX_K the next diagonal block gets that update on DMMA and the panel kernel publishes it, and the int8 update leaves that block out.  Each switch setting
runs tests/_diag_feed_worker.py in its own process; the factors (n = 1000 and 4096 with extra rows, and the C2 matrix with
its Y row) are compared with LAPACK and with the DMMA engine in units of the row scales, and the default is deterministic."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg as sla

from tests import _diag_feed_worker as W
from tests.test_gpu_engine_configs import INT8_VS_DMMA_BARS, LAPACK_BARS, LML_TC_VS_DMMA

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CONFIGS = {
    "default": {},
    "feed0": {"GPK_DIAG_FEED_MAX_K": "0"},
    "feed256": {"GPK_DIAG_FEED_MAX_K": "256"},
    "feed512": {"GPK_DIAG_FEED_MAX_K": "512"},
    "no_flag_hops": {"GPK_FLAG_HOPS": "0"},
    "dmma": {"GPK_FP64_ENGINE": "dmma"},
}
FACTORS = [f"extra{n}" for n, _ in W.EXTRA] + ["c2"]
# The n = 1000 / 4096 inputs take the bars of tests/test_gpu_engine_configs.py (measured on an H100 80GB HBM3 at 700 W: at most
# 2.6e-13 against LAPACK and the DMMA engine, with or without the feed).  The C2 matrix (bare factorisation: S = 7) is far less
# well conditioned: int8 factor 3.1e-12 from LAPACK and from the DMMA engine with every switch setting, DMMA engine 4.2e-13
# from LAPACK; the bar is about 10x that.
BARS = {"extra1000": (LAPACK_BARS["factor"], INT8_VS_DMMA_BARS["default"]),
        "extra4096": (LAPACK_BARS["factor"], INT8_VS_DMMA_BARS["default"]),
        "c2": (3e-11, 3e-11)}


@pytest.fixture(scope="module")
def tmp(tmp_path_factory):
    return str(tmp_path_factory.mktemp("diag_feed"))


@functools.lru_cache(maxsize=None)
def run_config(name, tmpdir):
    env = {k: v for k, v in os.environ.items() if not k.startswith("GPK_")}
    env.update(CONFIGS[name])
    out = os.path.join(tmpdir, f"{name}.npz")
    r = subprocess.run([sys.executable, "-m", "tests._diag_feed_worker", out], cwd=ROOT, env=env, timeout=900,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, f"{name}: worker failed\n{r.stdout[-4000:]}"
    with np.load(out) as z:
        return {k: z[k] for k in z.files}


@functools.lru_cache(maxsize=None)
def references():
    """LAPACK factors (extra rows solved against them) and the row scales of every input."""
    ref = {}
    inputs = {f"extra{n}": (W.extra_input(n, p), n) for n, p in W.EXTRA}
    inputs["c2"] = (W.c2_input()[0], W.C2_N)
    for k, (A, n) in inputs.items():
        S = np.tril(A[:n]) + np.tril(A[:n], -1).T
        L = np.linalg.cholesky(S)
        X = sla.solve_triangular(L, A[n:].T, lower=True).T
        ref[k] = np.concatenate([L, X])
        ref[f"scale_{k}"] = np.concatenate([np.sqrt(np.diag(S)), np.abs(X).max(axis=1)])
    return ref


def factor_diff(a, b, ref, k):
    return float((np.abs(a[k] - b[k]).max(axis=1) / ref[f"scale_{k}"]).max())


@pytest.mark.parametrize("name", [n for n in CONFIGS if n != "dmma"])
def test_diag_feed_factor_matches_lapack_and_dmma(cuda_device, tmp, name):
    res, dmma, ref = run_config(name, tmp), run_config("dmma", tmp), references()
    got = {k: (factor_diff(res, ref, ref, k), factor_diff(res, dmma, ref, k)) for k in FACTORS}
    bad = {k: (v, BARS[k]) for k, v in got.items() if not (v[0] <= BARS[k][0] and v[1] <= BARS[k][1])}
    assert not bad, f"{name}: {bad}"


def test_diag_feed_default_is_512_and_deterministic(cuda_device, tmp):
    a, b = run_config("default", tmp), run_config("feed512", tmp)
    assert str(a["c2_sha"]) == str(a["c2_again_sha"])
    for k in FACTORS:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_diag_feed_is_independent_of_flag_hops(cuda_device, tmp):
    a, b = run_config("default", tmp), run_config("no_flag_hops", tmp)
    for k in FACTORS:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_diag_feed_moves_the_c2_objective_towards_the_dmma_engine(cuda_device, tmp):
    """The fed diagonal blocks get fp64 DMMA products instead of int8 digit products (S = 6 for the GPR LML): the C2 LML moves
    by less than the int8 engine's distance from the DMMA engine, and towards the DMMA value (measured on an H100: 1.6e-12
    relative between the two settings; 5.3e-12 from the DMMA engine without the feed, 3.7e-12 with it)."""
    on, off, dmma = run_config("default", tmp), run_config("feed0", tmp), run_config("dmma", tmp)
    assert not np.array_equal(on["c2"], off["c2"])  # the switch does reach the factorisation
    np.testing.assert_allclose(on["c2_lml"], off["c2_lml"], rtol=LML_TC_VS_DMMA)
    assert abs(on["c2_lml"] - dmma["c2_lml"]) < abs(off["c2_lml"] - dmma["c2_lml"])
