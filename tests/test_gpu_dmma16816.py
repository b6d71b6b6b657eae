"""The fragment map of dmma16816 (common.cuh: mma.sync.m16n8k16.row.col.f64), which every fp64 DMMA kernel of the Cholesky
chain loads its operands by.  gpk_debug_dmma16816 runs one instruction per warp, D = A B + C with A 16 x 16, B 16 x 8; each lane
loads its registers by the documented map, so a wrong map puts elements in the wrong place.

Integer inputs pin the map exactly (every product and partial sum is exact).  Seeded inputs with denormals, signed zeros
and values near 1e+-150 are checked against a long double reference at the bar of a 16-term dot product whatever its order
(Higham (3.5)): |D - (A B + C)| <= gamma_17 (|A| |B| + |C|), plus one half-unit of the denormal grid per rounding for results
that underflow."""
import ctypes

import numpy as np
import pytest

from tests.dense64_bounds import gamma

pytestmark = pytest.mark.gpu

TINY = 2.0 ** -1074  # the smallest denormal


def run(A, B, C):
    import torch

    from gpflow_b200 import _lib

    lib = _lib.load()
    d = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (A, B, C)]
    D = torch.empty_like(d[2])
    assert lib.gpk_debug_dmma16816(*(ctypes.c_void_p(x.data_ptr()) for x in (*d, D)), A.shape[0], None) == 0
    torch.cuda.synchronize()
    return D.cpu().numpy()


def ref(A, B, C):
    Al, Bl = A.astype(np.longdouble), B.astype(np.longdouble)
    return np.matmul(Al, Bl) + C.astype(np.longdouble), np.matmul(np.abs(Al), np.abs(Bl)) + np.abs(C).astype(np.longdouble)


def test_dmma16816_map_exact_on_integers(cuda_device):
    rng = np.random.default_rng(16816)
    w = 64
    A = rng.integers(-1000, 1000, (w, 16, 16)).astype(np.float64)
    B = rng.integers(-1000, 1000, (w, 16, 8)).astype(np.float64)
    C = rng.integers(-10 ** 6, 10 ** 6, (w, 16, 8)).astype(np.float64)
    A[0] = np.arange(256).reshape(16, 16)  # distinct entries: any swapped row, column or k shows in warp 0
    B[0] = 1000.0 ** (np.arange(128).reshape(16, 8) % 3)
    want, _ = ref(A, B, C)
    np.testing.assert_array_equal(run(A, B, C), want.astype(np.float64))


def special_inputs(rng, w):
    def draw(shape):
        x = rng.standard_normal(shape)
        kind = rng.integers(0, 6, shape)
        x = np.where(kind == 1, x * 1e150, x)                          # +-large (products near 1e300, still finite)
        x = np.where(kind == 2, x * 1e-155, x)                         # tiny: products of two underflow to denormals
        x = np.where(kind == 3, rng.integers(1, 2 ** 20, shape) * TINY * np.sign(x), x)  # denormals
        x = np.where(kind == 4, np.where(x > 0, 0.0, -0.0), x)         # signed zeros
        return x
    return draw((w, 16, 16)), draw((w, 16, 8)), draw((w, 16, 8))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_dmma16816_within_the_dot_product_bar(cuda_device, seed):
    rng = np.random.default_rng(seed)
    A, B, C = special_inputs(rng, 512)
    got = run(A, B, C)
    want, mag = ref(A, B, C)
    assert np.isfinite(got).all()
    bar = gamma(17) * mag + 17 * TINY + 2.0 ** -64 * mag
    err = np.abs(got.astype(np.longdouble) - want)
    bad = err > bar
    assert not bad.any(), (int(bad.sum()), float((err / bar).max()))
