"""fp16-pair forward/dgrad convolution (csrc/conv_tc.cu) at launches of the size the benchmark step runs: several waves
of the persistent grid, where each CTA walks over many tiles and keeps its BatchNorm partial sums across the tiles of
one channel block.  A change to the kernel's schedule (which CTA takes which tile, how stages are loaded or shared) that
keeps the MMA chains, the adds and the per-CTA partials must leave every result bit for bit as it was.

The stored fixture tests/golden/conv_f16_multiwave_launches.npz holds, for f16x3 and f16, the SHA-256 of each output
and BatchNorm-sum tensor and a seeded sample of its entries (regenerate with
``python tests/test_gpu_conv_multiwave.py --write-golden`` only when results are meant to change).  The launches cover
an odd number of pixel tiles (consecutive tiles then straddle a channel block), 3x3 and stride-2 tiles, the dgrad of a
stride-2 convolution (one launch per output parity class, output stored at every second pixel), an odd number of
tiles below one wave and BN = 64 / 32 channel tiles.
"""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
CL = torch.channels_last
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_f16_multiwave_launches.npz')
SAMPLES = 1024

# name, N, Cin, H, W, Cout, k, dil, stride, dgrad.  A dgrad launch runs over dY (Cin channels at H x W) into an
# output of (2H - 1) x (2W - 1), one launch per output parity class.
CASES = [
    ('flat 1x1 256>1024 @33 (137 pixel tiles)', 16, 256, 33, 33, 1024, 1, 1, 1, False),
    ('3x3 256>256 @33', 16, 256, 33, 33, 256, 3, 1, 1, False),
    ('stride-2 3x3 128>128 @65', 8, 128, 65, 65, 128, 3, 1, 2, False),
    ('stride-2 dgrad 3x3 128>128 @33', 8, 128, 33, 33, 128, 3, 1, 1, True),
    ('27 tiles 1x1 256>384 @33', 1, 256, 33, 33, 384, 1, 1, 1, False),
    ('BN 64 1x1 256>64 @65 (133 tiles)', 4, 256, 65, 65, 64, 1, 1, 1, False),
    ('BN 32 3x3 d2 256>21 @33', 4, 256, 33, 33, 21, 3, 2, 1, False),
]


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    return _ops


def taps_of(k, dil):
    r = k // 2
    return [v for i in range(k) for j in range(k) for v in ((i - r) * dil, (j - r) * dil)]


def multiwave_launches(ops):
    """{key: array}: digest and sample of the output and the BatchNorm sums of every CASES launch in f16x3 and f16."""
    res = {}

    def put(key, t):
        a = t.detach().cpu().contiguous().numpy()
        res[key + ':sha256'] = np.array(hashlib.sha256(a.tobytes()).hexdigest())
        idx = torch.randint(0, a.size, (SAMPLES,), generator=torch.Generator().manual_seed(a.size)).numpy()
        res[key + ':sample'] = a.reshape(-1)[idx]

    for mode in ('f16x3', 'f16'):
        prec = ops.PRECISION[mode]
        for name, N, Cin, H, W, Cout, k, dil, stride, dgrad in CASES:
            g = torch.Generator().manual_seed(Cin + Cout + H + stride)
            x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
            w = (torch.randn(Cout * k * k * Cin, generator=g) / (Cin * k * k) ** 0.5).cuda()
            taps = taps_of(k, dil)
            if dgrad:
                OH, OW = 2 * H - 1, 2 * W - 1
                y = torch.zeros(N, Cout, OH, OW, device='cuda').contiguous(memory_format=CL)
                ops.conv_raw(x, w, None, [-v for v in taps], N, H, W, Cin, OH, OW, Cout, Cout, 1, 2, out=y,
                             precision=prec)
                put('%s %s:out' % (mode, name), y.permute(0, 2, 3, 1))
                continue
            OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
            b = torch.randn(Cout, generator=g).cuda()
            y = torch.empty(N, Cout, OH, OW, device='cuda').contiguous(memory_format=CL)
            st = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda')
            ops.conv_raw(x, w, b, taps, N, H, W, Cin, OH, OW, Cout, Cout, stride, 1, out=y, precision=prec,
                         bn_stats=st)
            put('%s %s:out' % (mode, name), y.permute(0, 2, 3, 1))
            put('%s %s:bn' % (mode, name), st)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0, 'mbarrier watchdog fired: role %d' % ops.conv_tc_status()
    return res


def test_multiwave_launches_match_the_stored_fixture(ops):
    want = np.load(GOLDEN)
    got = multiwave_launches(ops)
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
        sys.exit('usage: python tests/test_gpu_conv_multiwave.py --write-golden [PATH]')
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from pixelssl_b200 import ops as _ops
    path = sys.argv[2] if len(sys.argv) == 3 else GOLDEN
    np.savez(path, **multiwave_launches(_ops))
    print('wrote', path)
