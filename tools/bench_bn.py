"""Device timing of the BN kernels on the ResNet-101 @513, batch-16 shapes (achieved GB/s against algorithmic bytes)."""
import ctypes
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pixelssl_b200._lib import call

P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
SHAPES = [('l1 mid 64 @129', 16 * 129 * 129, 64), ('l1 out 256 @129', 16 * 129 * 129, 256), ('l2 out 512 @65', 16 * 65 * 65, 512),
          ('l3 mid 256 @33', 16 * 33 * 33, 256), ('l3 out 1024 @33', 16 * 33 * 33, 1024), ('l4 out 2048 @33', 16 * 33 * 33, 2048)]


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
for name, rows, C in SHAPES:
    n = rows * C
    x, y, dy, res = (torch.randn(rows, C, device='cuda') for _ in range(4))
    dx, dres = torch.empty_like(x), torch.empty_like(x)
    coeff = torch.rand(4, C, device='cuda') + 0.5
    gamma = torch.rand(C, device='cuda')
    sums = torch.zeros(2 * C, dtype=torch.float64, device='cuda')
    t_apply = timeit(lambda: call('pxl_bn_apply', P(x), P(coeff[2]), P(coeff[3]), P(res), 1, P(y), rows, C, P(None), P(None), 1.0, P(None), st))
    t_red = timeit(lambda: call('pxl_bn_bwd_reduce', P(x), P(y), P(dy), P(coeff[0]), P(coeff[1]), 1, rows, C, P(sums), P(None), P(None), P(None), P(None), st))
    t_dx = timeit(lambda: call('pxl_bn_bwd_dx', P(x), P(y), P(dy), P(coeff[0]), P(coeff[1]), P(gamma), P(sums), float(rows), 1,
                               P(dx), P(dres), rows, C, P(None), P(None), P(None), P(None), P(None), P(None), P(None), 0, P(None), st))
    rm, rv = torch.zeros(C, device='cuda'), torch.ones(C, device='cuda')
    beta = torch.rand(C, device='cuda')
    sums2 = torch.cat((x.double().sum(0), (x.double() ** 2).sum(0)))
    t_fa = timeit(lambda: call('pxl_bn_finalize_apply', P(x), P(sums2), float(rows), P(gamma), P(beta), P(rm), P(rv), 0.1, 1e-5, 0,
                               P(coeff[0]), P(coeff[1]), P(coeff[2]), P(coeff[3]), P(res), 1, P(y), rows, C, P(None), P(None), 1.0,
                               P(None), st))
    t_st = timeit(lambda: call('pxl_bn_stats', P(x), rows, C, P(sums), st))
    print('%-18s %6.1f MB  apply(+res,relu) %6.1f us %5.0f GB/s | fused fin+apply %6.1f us | bwd_reduce %6.1f us %5.0f GB/s | bwd_dx(+dres) %6.1f us %5.0f GB/s | stats %6.1f us %5.0f GB/s'
          % (name, n * 4 / 1e6, t_apply, 16 * n / t_apply / 1e3, t_fa, t_red, 12 * n / t_red / 1e3, t_dx, 20 * n / t_dx / 1e3, t_st, 4 * n / t_st / 1e3))
