"""Per-kernel device timings (CUDA events on the launching stream, L2 flushed between timed
iterations) for the HBM-bound tail kernels.  Scratch tool; bench.py is the contract."""
import json
import sys
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pixelssl_b200 import ops


def timeit(fn, iters=20, warmup=5, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def main():
    dev = 'cuda'
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)    # 256 MB > 50 MB L2
    out = {}
    for rows in (8, 16):
        n = rows * 21 * 513 * 513
        s = torch.randn(n, device=dev)
        t = torch.randn(n, device=dev)
        med, best = timeit(lambda: ops.mse_consistency_raw(s, t, 1.0, True), flush=flush)
        out['mse_fused_%drows' % rows] = {'ms_median': med, 'ms_best': best, 'GBps_median': 12 * n / med / 1e6, 'GBps_best': 12 * n / best / 1e6}
        med, best = timeit(lambda: ops.mse_consistency_raw(s, t, 1.0, False), flush=flush)
        out['mse_fwd_%drows' % rows] = {'ms_median': med, 'ms_best': best, 'GBps_median': 8 * n / med / 1e6, 'GBps_best': 8 * n / best / 1e6}
        # stock torch for context
        def torch_mse():
            sr = s.detach().requires_grad_(True)
            l = torch.nn.functional.mse_loss(sr, t)
            l.backward()
        med, best = timeit(torch_mse, flush=flush)
        out['torch_mse_fwd_bwd_%drows' % rows] = {'ms_median': med, 'GBps_at_12B': 12 * n / med / 1e6}
        del s, t
    x = torch.randn(8, 21, 513, 513, device=dev)
    lab = torch.randint(0, 21, (8, 1, 513, 513), device=dev).float()
    med, best = timeit(lambda: ops._CrossEntropy2d.apply(x.requires_grad_(True), lab, 255, 0.125), flush=flush)
    px = 8 * 513 * 513
    out['ce_fused'] = {'ms_median': med, 'GBps': (4 * 21 * 2 + 4) * px / med / 1e6}
    med, best = timeit(lambda: ops.softmax_planar(x.detach()), flush=flush)
    out['softmax'] = {'ms_median': med, 'GBps': 8 * 21 * px / med / 1e6}
    low = torch.randn(16, 32, 33, 33, device=dev).contiguous(memory_format=torch.channels_last)
    med, best = timeit(lambda: ops.bilinear(low, (513, 513), True, channels=21, nhwc=True), flush=flush)
    out['bilinear_fwd_16'] = {'ms_median': med, 'GBps': 4 * 21 * 16 * 513 * 513 / med / 1e6}
    gl = torch.randn(16, 21, 513, 513, device=dev)
    gin = torch.zeros_like(low)
    from pixelssl_b200.ops import call, _p, _stream
    med, best = timeit(lambda: call('pxl_bilinear_bwd', _p(gl), _p(gin), 16, 21, 33, 33, 513, 513, 1, 1, 32, _stream()), flush=flush)
    out['bilinear_bwd_16'] = {'ms_median': med, 'GBps_1read': 4 * 21 * 16 * 513 * 513 / med / 1e6}
    n = 44048532
    p, g, b, tt = (torch.randn(n, device=dev) for _ in range(4))
    med, best = timeit(lambda: ops.sgd_ema_(p, g, b, tt, 1e-3, 0.9, 5e-4, 0.99, False), flush=flush)
    out['sgd_ema_44M'] = {'ms_median': med, 'GBps': 28 * n / med / 1e6}
    a = torch.randn(16, 256, 129, 129, device=dev).contiguous(memory_format=torch.channels_last)
    gm, bt, rm, rv = torch.ones(256, device=dev), torch.zeros(256, device=dev), torch.zeros(256, device=dev), torch.ones(256, device=dev)
    med, best = timeit(lambda: ops.bn_act(a, gm, bt, rm, rv, True, relu=True), flush=flush)
    out['bn_relu_fwd_layer1'] = {'ms_median': med, 'GBps_12B': 12 * a.numel() / med / 1e6}
    # fp32 conv kernels
    for (N, C, HW, Co, k, d) in ((16, 256, 129, 64, 1, 1), (16, 64, 129, 64, 3, 1), (16, 1024, 33, 256, 1, 1), (16, 256, 33, 256, 3, 1), (16, 512, 33, 512, 3, 2)):
        xx = torch.randn(N, C, HW, HW, device=dev).contiguous(memory_format=torch.channels_last)
        ww = torch.randn(Co, C, k, k, device=dev).contiguous(memory_format=torch.channels_last)
        med, best = timeit(lambda: ops.conv2d(xx, ww, None, 1, d * (k // 2), d), iters=5, warmup=2)
        fl = 2.0 * N * HW * HW * C * Co * k * k
        out['conv_fp32_%d_%d_%d_k%d' % (C, HW, Co, k)] = {'ms': med, 'TFLOPs': fl / med / 1e9}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
