"""Mean-Teacher training step with the DeepLabV3+-R101 task model (output stride 16): engine kernels against the same
step written with stock torch ops (the CPU oracle, oracle/deeplabv3plus_oracle.py, run on the same GPU with cuDNN's
defaults).  Prints one JSON line: images/s and peak memory of both, per-launch CUDA-event times of the head's
concatenation / spatial-mean kernels, and the card's name and power limit.

    python tools/bench_deeplabv3plus.py [--steps 10] [--warmup 3] [--precision f16x3] [--size 513] [--lbs 8] [--ubs 8]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

NEW_KERNELS = ('pxl_lane_concat_nhwc', 'pxl_lane_concat_bwd_nhwc', 'pxl_spatial_mean_nhwc')


def card():
    info = {'name': torch.cuda.get_device_name(0), 'power_limit_w': None}
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info['power_limit_w'] = float(out.splitlines()[0])
    except Exception as e:          # the figure is reported as unknown, never guessed
        info['power_limit_error'] = str(e)
    return info


def engine(args, batches):
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import runner, ops
    ops.set_conv_precision(args.precision)
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    cfg = {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 3,
           'ema_decay': 0.99, 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9,
           'batch_size': args.lbs + args.ubs, 'unlabeled_batch_size': args.ubs, 'backbone': 'resnet101',
           'output_stride': 16, 'models': {'model': 'deeplabv3plus'}}
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=662))

    def steps(count, epoch):
        alg._train([((batches[i % len(batches)][0],), (batches[i % len(batches)][1],)) for i in range(count)], epoch)

    steps(args.warmup, 0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    steps(args.steps, 1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    peak = torch.cuda.max_memory_allocated()
    loss = float(alg.meters['s_task_loss'].val)
    # one more step with CUDA events around every launch of the new kernels (outside the timed window)
    for k in NEW_KERNELS:
        ops.kernel_timer_start(k)
    steps(1, 2)
    kern = {}
    for k in NEW_KERNELS:
        t = ops.kernel_timer_stop(k)
        kern[k] = {'launches': len(t), 'ms_total': sum(t), 'ms_each': [round(v, 4) for v in t]}
    status = (ops.conv_tc_status(), ops.h16_status())
    del alg
    torch.cuda.empty_cache()
    return {'value': (args.lbs + args.ubs) * args.steps / (ms / 1e3), 'unit': 'images/s', 'ms_per_step': ms / args.steps,
            'peak_mem_gib': peak / 2 ** 30, 's_task_loss': loss, 'conv_precision': args.precision,
            'kernels_one_step': kern, 'status': status}


def stock_torch(args, batches):
    from oracle import deeplabv3plus_oracle as D
    dev = torch.device('cuda:0')
    s = {k: v.to(dev) for k, v in D.init(0).items()}
    t = {k: v.to(dev) for k, v in D.init(1).items()}
    mt = D.MTOracle(s, t, lr=0.00025, momentum=0.9, weight_decay=0.0005, max_iters=20 * 662, cons_scale=1.0,
                    rampup_steps=3 * 662, ema_decay=0.99, cons_for_labeled=False)

    def one(i):
        img, lab = batches[i % len(batches)]
        return mt.step(img, lab, args.lbs)

    for i in range(args.warmup):
        one(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for i in range(args.steps):
        out = one(i)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated()
    return {'value': (args.lbs + args.ubs) * args.steps / dt, 'unit': 'images/s', 'ms_per_step': dt * 1e3 / args.steps,
            'peak_mem_gib': peak / 2 ** 30, 's_task_loss': float(out['s_task_loss']),
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
        raise SystemExit('bench_deeplabv3plus: needs a CUDA device')
    torch.cuda.set_device(0)
    from oracle import sseg_oracle as O
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, args.lbs + args.ubs, args.lbs, args.size, args.size))
               for i in range(2)]
    res = {'metric': 'DeepLabV3+-R101 OS16 Mean-Teacher step, %d+%d x %dx%d' % (args.lbs, args.ubs, args.size, args.size),
           'steps': args.steps, 'warmup': args.warmup, 'card': card()}
    if not args.skip_torch:         # first, so that its peak memory does not include the engine's caches
        res['stock_torch'] = stock_torch(args, batches)
        torch.cuda.empty_cache()
    res['engine'] = engine(args, batches)
    if not args.skip_torch:
        res['speedup'] = res['engine']['value'] / res['stock_torch']['value']
    print(json.dumps(res))


if __name__ == '__main__':
    main()
