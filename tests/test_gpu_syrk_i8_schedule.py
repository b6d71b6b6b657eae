"""The int8 trailing update under its unit assignment (gemm_tc.cu::TcTileIter, mirrored in tests/test_tc_schedule_model.py),
bit for bit against the NumPy emulation of its arithmetic: launches thinner than one unit per cluster, launches of several
rounds with a partial last round, S = 6 / 7 / 8, cluster widths 1 and 2 and the factorisation's own width (cluster = 0)."""
import numpy as np
import pytest

from tests.test_digit_slicing_model import syrk_i8_accumulators, syrk_i8_epilogue
from tests.test_gpu_syrk_i8 import check, dev_matmul, mixed_rows, sentinel_c
from tests.test_tile_iterators_model import diag_units_total, tc_units

pytestmark = pytest.mark.gpu

# (m, n, K): C2's thinnest K = 256 launches (m = 257: 10 units of 2 tiles for 65 clusters; m = 769: 26), one with a
# partial second round (m = 2305: 74 units) and a ragged several-round one
SHAPES = [(257, 256, 256), (769, 256, 256), (2305, 256, 64), (1500, 700, 96)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "m%d_n%d_K%d" % s)
@pytest.mark.parametrize("cl", [0, 1, 2])
@pytest.mark.parametrize("S", [6, 7, 8])
def test_syrk_i8_schedule_bit_exact(cuda_device, S, cl, shape):
    m, n, K = shape
    rng = np.random.default_rng(m + n + K + S)
    P = mixed_rows(m, K, rng)
    C0 = sentinel_c(m, n, rng)
    acc, rs = syrk_i8_accumulators(P, n, S, matmul=dev_matmul)
    want = syrk_i8_epilogue(acc, rs, C0)
    r0 = -(-K // 128) * 128
    check(P, n, S, cl, 1, C0, want=want, r0=r0)
    check(P, n, S, cl, 0, C0, want=want, r0=r0)


@pytest.mark.parametrize("m,n", [(257, 256), (2305, 256), (1000, 130)])
def test_syrk_i8_schedule_head_flag_counts(cuda_device, m, n):
    """At the factorisation's own width the look-ahead counters stay what the 2-CTA unit set gives."""
    rng = np.random.default_rng(m + n)
    P = rng.standard_normal((m, 64))
    C0 = sentinel_c(m, n, rng)
    flag = check(P, n, 6, 0, 1, C0, head_flag=True)
    heads = sum(u["head"] for b in range(2) for u in tc_units(m, n, 1, 2, 2, b))
    assert flag.tolist() == [heads, diag_units_total(m, n)]
