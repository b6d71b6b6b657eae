"""NumPy model of the 3xTF32 operand split of gpflow_b200/csrc/gemm_tf32.cu (split_tiles_kernel: hi = rna_tf32(x),
lo = rna_tf32(x - hi); products hi*hi + hi*lo + lo*hi): checks without a GPU that the compensated product carries
fp32-level accuracy where a plain TF32 product would lose 13 bits.  The split itself lives in tests/dense32_bounds.py
with the rest of the model."""
import numpy as np

from tests.dense32_bounds import split


def test_split_reconstructs_to_21_bits():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(100000) * np.exp2(rng.integers(-30, 30, 100000))).astype(np.float32)
    hi, lo = split(x)
    assert np.all(np.abs((hi.astype(np.float64) + lo) - x) <= np.abs(x) * 2.0 ** -21)
    assert np.all((hi.view(np.uint32) & 0x1FFF) == 0) and np.all((lo.view(np.uint32) & 0x1FFF) == 0)   # TF32-representable


def test_three_term_product_has_fp32_accuracy():
    rng = np.random.default_rng(1)
    m, n, k = 64, 48, 2048
    A = rng.standard_normal((m, k)).astype(np.float32)
    B = rng.standard_normal((n, k)).astype(np.float32)
    ah, al = split(A)
    bh, bl = split(B)
    exact = A.astype(np.float64) @ B.astype(np.float64).T
    three = (al.astype(np.float64) @ bh.T.astype(np.float64) + ah.astype(np.float64) @ bl.T.astype(np.float64)
             + ah.astype(np.float64) @ bh.T.astype(np.float64))
    one = ah.astype(np.float64) @ bh.T.astype(np.float64)
    absdot = np.abs(A).astype(np.float64) @ np.abs(B).astype(np.float64).T
    assert np.all(np.abs(three - exact) <= 2.0 ** -20 * absdot)          # dropped lo*lo term and split rounding
    assert np.abs(one - exact).max() > 50 * np.abs(three - exact).max()   # plain TF32 is orders of magnitude worse
