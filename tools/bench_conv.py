"""Per-shape device timing of the wgmma convolution kernels (forward/dgrad kernel and wgrad kernel) on the
ResNet-101 @ 513x513, batch 16 shapes that dominate the MT step.

    python tools/bench_conv.py tf32|tf32x3|f16x3|f16 [fwd|wgrad|both]

In the fp16-pair modes the operands are split outside the timed region: in the engine the pairs are written by the
producing BatchNorm launches (ops._ConvBnAct), not by a separate pass.
"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pixelssl_b200 import ops

CL = torch.channels_last
# name, N, H, W, Cin, Cout, k, dil, launches per MT step (fwd+fwd+dgrad)
SHAPES = [
    ('l3.conv2 3x3 256>256 @33', 16, 33, 33, 256, 256, 3, 1, 69),
    ('l3.conv3 1x1 256>1024 @33', 16, 33, 33, 256, 1024, 1, 1, 69),
    ('l3.conv1 1x1 1024>256 @33', 16, 33, 33, 1024, 256, 1, 1, 69),
    ('l4.conv2 3x3 512>512 d2 @33', 16, 33, 33, 512, 512, 3, 2, 9),
    ('l4.conv3 1x1 512>2048 @33', 16, 33, 33, 512, 2048, 1, 1, 9),
    ('l4.conv1 1x1 2048>512 @33', 16, 33, 33, 2048, 512, 1, 1, 9),
    ('l2.conv2 3x3 128>128 @65', 16, 65, 65, 128, 128, 3, 1, 12),
    ('l2.conv3 1x1 128>512 @65', 16, 65, 65, 128, 512, 1, 1, 12),
    ('l2.conv1 1x1 512>128 @65', 16, 65, 65, 512, 128, 1, 1, 12),
    ('l1.conv2 3x3 64>64 @129', 16, 129, 129, 64, 64, 3, 1, 9),
    ('l1.conv3 1x1 64>256 @129', 16, 129, 129, 64, 256, 1, 1, 9),
    ('l1.conv1 1x1 256>64 @129', 16, 129, 129, 256, 64, 1, 1, 9),
]


def taps_of(k, dil):
    r = k // 2
    t = []
    for i in range(k):
        for j in range(k):
            t += [(i - r) * dil, (j - r) * dil]
    return t


def time_fn(fn, iters=8, warmup=3, reps=12):
    """Median device time of one launch: `reps` back-to-back launches between two events (a single launch between
    events would mostly measure the host-side launch latency of these 30-100 us kernels)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(200000)           # ~100 us of GPU idle spin so the queue fills behind it
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    prec_name = sys.argv[1] if len(sys.argv) > 1 else 'tf32'
    what = sys.argv[2] if len(sys.argv) > 2 else 'both'
    prec = ops.PRECISION[prec_name]
    tot_f = tot_w = 0.0
    print('precision %s' % prec_name)
    for name, N, H, W, Cin, Cout, k, dil, mult in SHAPES:
        taps = taps_of(k, dil)
        nt = k * k
        xs = [torch.randn(N, Cin, H, W, device='cuda').contiguous(memory_format=CL) for _ in range(3)]
        w = torch.randn(Cout * nt * Cin, device='cuda') * 0.05
        out = torch.empty(N, Cout, H, W, device='cuda').contiguous(memory_format=CL)
        if prec >= 3:
            xs = [ops.h16_split(t, ops.H16_ACT_SCALE, prec == 3) for t in xs]
            w = ops.h16_split(w, ops.H16_W_SCALE, prec == 3)
        flop = 2.0 * N * H * W * Cin * Cout * nt
        line = '%-30s' % name
        if what in ('fwd', 'both', 'fwdstats'):
            it = [0]
            st = torch.zeros(2 * Cout, dtype=torch.float64, device='cuda') if what == 'fwdstats' else None

            def f():
                it[0] += 1
                ops.conv_raw(xs[it[0] % 3], w, None, taps, N, H, W, Cin, H, W, Cout, Cout, 1, 1, out=out, precision=prec, bn_stats=st)
            us = time_fn(f)
            tot_f += us * mult
            line += '  fwd %8.1f us %7.1f TF/s' % (us, flop / us / 1e6)
        if what in ('wgrad', 'both'):
            dw = torch.zeros(Cout * nt * Cin, device='cuda')
            dy = torch.randn(N, Cout, H, W, device='cuda').contiguous(memory_format=CL)
            if prec >= 3:
                dy = ops.h16_split(dy * 1e-6, None, prec == 3)

            def g():
                ops.conv_wgrad_raw(xs[0], dy, dw, taps, N, H, W, Cin, H, W, Cout, Cout, 1, 1, precision=prec)
            us = time_fn(g)
            tot_w += us * mult / 3.0
            line += '  wgrad %8.1f us %7.1f TF/s' % (us, flop / us / 1e6)
        print(line)
        del xs, w, out
    print('weighted per-step estimate: fwd/dgrad %.2f ms, wgrad %.2f ms   (tc status %d)' %
          (tot_f / 1e3, tot_w / 1e3, ops.conv_tc_status()))


if __name__ == '__main__':
    main()
