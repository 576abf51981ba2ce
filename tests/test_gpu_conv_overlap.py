"""fp16-pair wgmma convolutions (csrc/conv_tc.cu): the main loops drop the MMA waits that order nothing, and must
still compute bit for bit what the loop that waited for every MMA group computed.
* bit-identity: f16x3 and f16 forward, BatchNorm sums and wgrad of a few small launches against the stored fixture
  tests/golden/conv_f16_launches.npz, written by that earlier loop (regenerate with
  ``python tests/test_gpu_conv_overlap.py --write-golden`` only when results are meant to change);
* accuracy: f16x3 forward, dgrad and wgrad of the longest reductions of DeepLab-v2-R101 at 513x513, batch 16, against
  a float64 torch reference on the device, within the fp32-grade tolerances of test_gpu_conv_tc.py (2e-5 for outputs
  and input gradients, 5e-5 for weight gradients);
* reproducibility: two launches on the same inputs give bit-identical outputs, BatchNorm sums and weight gradients.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
CL = torch.channels_last
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_f16_launches.npz')


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    return _ops


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def taps_of(k, dil):
    r = k // 2
    return [v for i in range(k) for j in range(k) for v in ((i - r) * dil, (j - r) * dil)]


# name, N, Cin, H, W, Cout, k, dil: the longest forward / dgrad reductions (K = Cin * taps) and the longest wgrad
# reduction (K = N * H * W pixels) of the benchmark step
LONG_CASES = [
    ('l3.conv2 3x3 256>256 @33', 16, 256, 33, 33, 256, 3, 1),
    ('l4.conv1 1x1 2048>512 @33', 16, 2048, 33, 33, 512, 1, 1),
    ('l4.conv2 3x3 512>512 d2 @33', 16, 512, 33, 33, 512, 3, 2),
    ('l1.conv2 3x3 64>64 @129', 16, 64, 129, 129, 64, 3, 1),
]


def _bound(K, s_abs_max, ref_max):
    """Worst-case bound of the loop's own fp32 sums, relative to max|reference| as the measured error is: at most
    three round-to-nearest adds per 64 of K at 2^-24 sum|products| each, and about 2^-33 sum|products| of truncation
    per correction MMA (lo < 2^-11 |hi|, one fresh eight-MMA chain per stage), K / 8 of them.  The fp16-pair operand
    split is not included."""
    return (3 * K / 64 * 2.0 ** -24 + K / 8 * 2.0 ** -33) * s_abs_max / ref_max


def _fp64(x, w, gy, pad, dil):
    """float64 torch: (y, dx, dW)."""
    xd, wd = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yd = F.conv2d(xd, wd, None, 1, pad, dil)
    yd.backward(gy.double())
    return yd.detach(), xd.grad, wd.grad


@pytest.mark.parametrize('case', LONG_CASES, ids=[c[0] for c in LONG_CASES])
def test_f16x3_long_reductions_against_fp64(ops, case):
    name, N, Cin, H, W, Cout, k, dil = case
    g = torch.Generator().manual_seed(Cin * 7 + Cout + H)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda().contiguous(memory_format=CL)
    gy = (torch.randn(N, Cout, H, W, generator=g) * 1e-3).cuda().contiguous(memory_format=CL)
    pad = dil * (k // 2)
    ops._conv_precision = ops.PRECISION['f16x3']
    try:
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        y = ops.conv2d(xg, wg, None, 1, pad, dil)
        y.backward(gy)
        torch.cuda.synchronize()
    finally:
        ops._conv_precision = 0
    assert ops.conv_tc_status() == 0, 'mbarrier watchdog fired: role %d' % ops.conv_tc_status()
    assert ops.h16_status() == 0, 'an fp16 pair saturated'
    got = (y.detach(), xg.grad, wg.grad)
    del y, xg, wg
    ref = _fp64(x, w, gy, pad, dil)
    s_abs = _fp64(x.abs(), w.abs(), gy.abs(), pad, dil)        # sum|products| of every output
    Ks = (Cin * k * k, Cout * k * k, N * H * W)
    errs = []
    for what, a, b, sa, K, tol in zip(('fwd', 'dgrad', 'wgrad'), got, ref, s_abs, Ks, (2e-5, 2e-5, 5e-5)):
        e = rel(a, b)
        print('%s %-5s K=%6d: max rel err %.2e (tol %.0e), accumulation bound %.2e'
              % (name, what, K, e, tol, _bound(K, float(sa.max()), float(b.abs().max()))))
        errs.append((what, e, tol))
    assert all(e <= tol for _, e, tol in errs), errs


@pytest.mark.parametrize('precision', ['f16x3', 'f16'])
@pytest.mark.parametrize('case', [LONG_CASES[0], LONG_CASES[3]], ids=[LONG_CASES[0][0], LONG_CASES[3][0]])
def test_repeat_launches_are_bit_identical(ops, case, precision):
    name, N, Cin, H, W, Cout, k, dil = case
    prec = ops.PRECISION[precision]
    taps = taps_of(k, dil)
    g = torch.Generator().manual_seed(H + Cout)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = torch.randn(Cout * k * k * Cin, generator=g).cuda() * 0.05
    dy = (torch.randn(N, Cout, H, W, generator=g) * 1e-4).cuda().contiguous(memory_format=CL)
    outs = []
    for _ in range(2):
        y = torch.empty(N, Cout, H, W, device='cuda').contiguous(memory_format=CL)
        st = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda')
        ops.conv_raw(x, w, None, taps, N, H, W, Cin, H, W, Cout, Cout, 1, 1, out=y, precision=prec, bn_stats=st)
        dw = torch.zeros(Cout * k * k * Cin, device='cuda')
        ops.conv_wgrad_raw(x, dy, dw, taps, N, H, W, Cin, H, W, Cout, Cout, 1, 1, precision=prec)
        outs.append((y, st, dw))
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0
    for what, a, b in zip(('output', 'bn sums', 'dW'), outs[0], outs[1]):
        assert torch.equal(a, b), '%s %s: %s differs between two launches' % (name, precision, what)


# ---- both fp16 modes against the stored fixture --------------------------------------------------------------------
# name, N, Cin, H, W, Cout, k, dil.  Forward: BN = 128, 64 and 32 channel tiles, 2-D and flat pixel tiles; wgrad
# (MMAs per stage in f16x3 / f16): 4 / 8, 3 / 7 and, flat, 4 / 8.
PAIR_FWD = [
    ('fwd 3x3 128>128 @17x19', 2, 128, 17, 19, 128, 3, 1),
    ('fwd 1x1 256>64 @33', 2, 256, 33, 33, 64, 1, 1),
    ('fwd 3x3 d2 256>21 @17', 1, 256, 17, 17, 21, 3, 2),
]
PAIR_WGRAD = [
    ('wgrad 3x3 64>64 @33', 2, 64, 33, 33, 64, 3, 1),
    ('wgrad 3x3 64>128 @65', 1, 64, 65, 65, 128, 3, 1),
    ('wgrad 1x1 128>256 @17', 2, 128, 17, 17, 256, 1, 1),
]
SAMPLES = 1024


def pair_launches(ops):
    """{key: array} for every PAIR_FWD / PAIR_WGRAD launch in f16x3 and f16: the SHA-256 of each result tensor and a
    seeded sample of its entries (the sample says where a mismatch lies; the digest decides)."""
    res = {}

    def put(key, t):
        a = t.detach().cpu().contiguous().numpy()
        res[key + ':sha256'] = np.array(hashlib.sha256(a.tobytes()).hexdigest())
        idx = torch.randint(0, a.size, (SAMPLES,), generator=torch.Generator().manual_seed(a.size)).numpy()
        res[key + ':sample'] = a.reshape(-1)[idx]

    for mode in ('f16x3', 'f16'):
        prec = ops.PRECISION[mode]
        for name, N, Cin, H, W, Cout, k, dil in PAIR_FWD:
            g = torch.Generator().manual_seed(Cin + Cout + H)
            x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
            w = (torch.randn(Cout * k * k * Cin, generator=g) / (Cin * k * k) ** 0.5).cuda()
            b = torch.randn(Cout, generator=g).cuda()
            y = torch.empty(N, Cout, H, W, device='cuda').contiguous(memory_format=CL)
            st = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda')
            ops.conv_raw(x, w, b, taps_of(k, dil), N, H, W, Cin, H, W, Cout, Cout, 1, 1, out=y, precision=prec,
                         bn_stats=st)
            put('%s %s:out' % (mode, name), y.permute(0, 2, 3, 1))
            put('%s %s:bn' % (mode, name), st)
        for name, N, Cin, H, W, Cout, k, dil in PAIR_WGRAD:
            g = torch.Generator().manual_seed(Cin + Cout + H)
            x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
            dy = (torch.randn(N, Cout, H, W, generator=g) * 1e-4).cuda().contiguous(memory_format=CL)
            dw = torch.zeros(Cout * k * k * Cin, device='cuda')
            ops.conv_wgrad_raw(x, dy, dw, taps_of(k, dil), N, H, W, Cin, H, W, Cout, Cout, 1, 1, precision=prec)
            put('%s %s:dw' % (mode, name), dw)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0
    return res


def test_launches_match_the_stored_fixture(ops):
    want = np.load(GOLDEN)
    got = pair_launches(ops)
    assert sorted(got) == sorted(want.files)
    bad = []
    for key in sorted(k for k in got if k.endswith(':sha256')):
        if str(got[key]) != str(want[key]):
            base = key[:-len(':sha256')]
            d = np.abs(got[base + ':sample'].astype(np.float64) - want[base + ':sample'].astype(np.float64))
            bad.append('%s (sampled entries differ by up to %.3g)' % (base, float(d.max())))
    assert not bad, 'results changed: ' + ', '.join(bad)


if __name__ == '__main__':
    if not sys.argv[1:2] == ['--write-golden'] or len(sys.argv) > 3:
        sys.exit('usage: python tests/test_gpu_conv_overlap.py --write-golden [PATH]')
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pixelssl_b200 import ops as _ops
    path = sys.argv[2] if len(sys.argv) == 3 else GOLDEN
    np.savez(path, **pair_launches(_ops))
    print('wrote', path)
