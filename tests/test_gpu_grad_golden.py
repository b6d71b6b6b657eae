"""Loss and gradients of `training_loss_and_gradients` for GPR, SGPR, SVGP (Gaussian, Student-t and Bernoulli, across
whiten x q_diag) and VGP against tests/golden/grad_golden.npz (tests/golden/make_grad_golden.py).  The device
reductions add through atomics, so the outputs are reproduced to rounding, not bit for bit."""
import os

import numpy as np
import pytest

from tests.golden import make_grad_golden as G

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "grad_golden.npz")


def test_device_gradients_reproduce_the_golden_record(cuda_device):
    ref = np.load(GOLDEN)
    got = G.record()
    assert set(got) == set(ref.files)
    for key in sorted(ref.files):
        r = ref[key]
        np.testing.assert_allclose(got[key], r, rtol=0, atol=1e-12 * max(1.0, float(np.max(np.abs(r)))), err_msg=key)
