"""Mean-Teacher training step with DeepLabV3+ on the aligned Xception-65 backbone at output stride 16 (two timed runs
after a warm-up), plus the same step written with stock torch ops (the CPU oracle, oracle/xception_oracle.py, on the
same GPU: cuDNN grouped convolutions, TF32 allowed).  Prints one JSON line: images/s, ms/step and peak memory of both,
per depthwise kernel family the launches, CUDA-event time, algorithmic bytes from shapes, TB/s and share of the H100
SXM's 3.35 TB/s in one step, the depthwise kernels' share of that step, and the card's name and power limit.

    python tools/bench_xception.py [--steps 10] [--warmup 3] [--precision f16x3] [--size 513] [--lbs 8] [--ubs 8]
"""
import argparse
import json
import os
import random
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_deepstem import card, run_steps, timed

FAMILIES = ('pxl_dw_conv_fwd', 'pxl_dw_conv_dgrad', 'pxl_dw_conv_wgrad')
HBM_TBPS = 3.35


def build_engine(args):
    from pixelssl_b200 import runner
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    cfg = {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 3,
           'ema_decay': 0.99, 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9,
           'batch_size': args.lbs + args.ubs, 'unlabeled_batch_size': args.ubs, 'backbone': 'xception65',
           'pretrained_backbone': 'none', 'output_stride': 16, 'models': {'model': 'deeplabv3plus'}}
    return runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=662))


def depthwise_kernels(alg, args, batches):
    """One step with CUDA events around every depthwise launch.  Bytes per launch: the activation read once and the
    activation written once (wgrad: x and dY read), 4 B per lane, from the shapes (the weights are negligible).
    Launches on the 33x33 middle-flow maps (16 x 33 x 33 x 768 x 4 B = 54 MB per map) work on operands that fit the
    50 MB L2 about as well as not, so their rate is not bounded by HBM alone."""
    from pixelssl_b200 import ops
    for k in FAMILIES:
        ops.kernel_timer_start(k)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run_steps(alg, batches, 1, 2)
    e1.record()
    out, total = {}, 0.0
    per = {k: ops.kernel_timer_stop(k, with_meta=True) for k in FAMILIES}
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1)
    for k, rec in per.items():
        ms, byts = sum(t for t, _ in rec), sum(m[0] for _, m in rec)
        mid = [(t, m) for t, m in rec if ' 33x33 ' in m[1]]
        out[k] = {'launches': len(rec), 'ms': ms, 'gbytes': byts / 1e9, 'tb_per_s': byts / (ms / 1e3) / 1e12 if ms else None,
                  'share_of_hbm_peak': byts / (ms / 1e3) / 1e12 / HBM_TBPS if ms else None,
                  'middle_flow_33x33': {'launches': len(mid), 'ms': sum(t for t, _ in mid),
                                        'tb_per_s': (sum(m[0] for _, m in mid) / (sum(t for t, _ in mid) / 1e3) / 1e12)
                                        if mid else None}}
        total += ms
    out['depthwise_ms_total'] = total
    out['step_ms_with_event_timers'] = step_ms
    out['depthwise_share_of_step'] = total / step_ms
    return out


def stock_torch(args, batches):
    from oracle import xception_oracle as X
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    dev = torch.device('cuda:0')
    s = {k: v.to(dev) for k, v in X.init(0).items()}
    t = {k: v.to(dev) for k, v in X.init(1).items()}
    mt = X.MTOracle(s, t, lr=0.00025, momentum=0.9, weight_decay=0.0005, max_iters=20 * 662, cons_scale=1.0,
                    rampup_steps=3 * 662, ema_decay=0.99, cons_for_labeled=False)

    def one(i):
        img, lab = batches[i % len(batches)]
        return mt.step(img, lab, args.lbs)

    for i in range(args.warmup):
        one(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    runs = []
    for _ in range(2):
        t0 = time.perf_counter()
        for i in range(args.steps):
            one(i)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        runs.append({'images_per_s': (args.lbs + args.ubs) * args.steps / dt, 'ms_per_step': dt * 1e3 / args.steps})
    return {'runs': runs, 'images_per_s_median': float(np.median([r['images_per_s'] for r in runs])),
            'peak_mem_gib': torch.cuda.max_memory_allocated() / 2 ** 30,
            'torch_conv': 'cuDNN, TF32 allowed=%s' % torch.backends.cudnn.allow_tf32}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--precision', default='f16x3')
    p.add_argument('--size', type=int, default=513)
    p.add_argument('--lbs', type=int, default=8)
    p.add_argument('--ubs', type=int, default=8)
    p.add_argument('--skip-torch', action='store_true')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_xception: needs a CUDA device')
    torch.cuda.set_device(0)
    from oracle import sseg_oracle as O
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, args.lbs + args.ubs, args.lbs, args.size, args.size))
               for i in range(2)]
    res = {'metric': 'DeepLabV3+-Xception65 OS16 Mean-Teacher step, %d+%d x %dx%d, %s' % (
        args.lbs, args.ubs, args.size, args.size, args.precision), 'steps': args.steps, 'warmup': args.warmup,
        'card': card()}
    if not args.skip_torch:         # first, so that its peak memory does not include the engine's caches
        try:
            res['stock_torch'] = stock_torch(args, batches)
        except torch.cuda.OutOfMemoryError as e:
            res['stock_torch'] = {'error': 'out of memory: %s' % str(e).splitlines()[0]}
        torch.cuda.empty_cache()
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    ops.set_conv_precision(args.precision)
    alg = build_engine(args)
    run_steps(alg, batches, args.warmup, 0)
    runs = [timed(alg, args, batches) for _ in range(2)]
    res['engine'] = {'runs': runs, 'images_per_s_median': float(np.median([r['images_per_s'] for r in runs]))}
    if 'images_per_s_median' in res.get('stock_torch', {}):
        res['engine_vs_stock_torch'] = res['engine']['images_per_s_median'] / res['stock_torch']['images_per_s_median']
    res['depthwise_kernels_one_step'] = depthwise_kernels(alg, args, batches)
    res['status'] = (ops.conv_tc_status(), ops.h16_status())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
