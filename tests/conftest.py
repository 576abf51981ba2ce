import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, 'tests', 'golden')

# Convolution precision modes every whole-network / whole-step GPU golden is run under (fixture params, so the
# mode shows up in the test id): the exact-fp32 FFMA kernels and the fp32-grade wgmma modes that bench.py times.
TEST_PRECISIONS = [p for p in os.environ.get('PXL_TEST_PRECISIONS', 'fp32,tf32x3,f16x3').split(',') if p]


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100; run with -m gpu)')
    config.addinivalue_line('markers', 'slow: CPU test that takes more than a few seconds')


@pytest.fixture(scope='session')
def golden_dir():
    return GOLDEN


# ---- noise yardstick shared by the whole-step GPU goldens -------------------------------------------------------------
# tests/golden/fp64_truth*.npz hold the oracle evaluated in fp64 on the golden inputs.  The engine must be within
# the north_star's 1e-3 of the exact value OR within FACTOR x the deviation the reference's own fp32 evaluation
# (the *_step_*.npz fixtures) shows from it - whichever is larger (deep random-init nets amplify rounding ~1e3 x).
FACTOR = 3.0


def assert_loss_yardstick(got, ref32, truth, what, rel_floor=1e-3):
    tol = max(FACTOR * abs(ref32 - truth), rel_floor * abs(truth))
    assert abs(got - truth) <= tol, '%s: engine %.8g truth %.8g (reference fp32 %.8g, tol %.2e)' % (what, got, truth, ref32, tol)


def assert_energy_yardstick(got_sq, ref32, truth, what, keep=None, floor_med=3e-4, floor_max=3e-3):
    """Per-tensor gradient energies (sum of squares): engine-vs-truth deviation against reference-fp32-vs-truth over
    the parameter tensors: median and 95th percentile within FACTOR x the reference's, the worst tensor within
    2 FACTOR x the reference's worst (plus small floors).
    Why the worst tensor gets the wider bound: it is always the same ill-conditioned tensor (a first-layer weight whose
    gradient sums rounding noise of the whole net), and its deviation moves between 2.9e-2 and 6.3e-2 (reference fp32:
    1.9e-2) for arithmetic-equivalent variants of the SAME kernels - statistics by register butterfly or shared-memory
    walk, the order of the tests in the process (fp32 atomics / split-K order).  A wrong gradient shows up as O(1)."""
    import numpy as np
    den = np.maximum(np.abs(truth[:, 1]), 1e-300)
    e, r = np.abs(got_sq - truth[:, 1]) / den, np.abs(ref32[:, 1] - truth[:, 1]) / den
    if keep is not None:
        e, r = e[keep], r[keep]
    msg = '%s: engine median %.2e q95 %.2e max %.2e | reference fp32 median %.2e q95 %.2e max %.2e' % (
        what, np.median(e), np.quantile(e, 0.95), e.max(), np.median(r), np.quantile(r, 0.95), r.max())
    assert np.median(e) <= FACTOR * np.median(r) + floor_med, msg
    assert np.quantile(e, 0.95) <= FACTOR * np.quantile(r, 0.95) + floor_max, msg
    assert e.max() <= 2.0 * FACTOR * r.max() + floor_max, msg
    return msg
