"""Mean-Teacher training step with DeepLabV3+ at output stride 16 on the deep-stem ResNet-101 (resnet101-deepstem) and on
the 7x7-stem ResNet-101, alternating in one process (two timed runs each after a warm-up), plus the deep-stem step
written with stock torch ops (the CPU oracle, oracle/deepstem_oracle.py, on the same GPU, cuDNN with TF32 allowed).
Prints one JSON line: images/s, ms/step and peak memory per backbone, CUDA-event times of the 3x3 unfold and of every
convolution launch at the stem's resolution in one step with their FLOPs and algorithmic bytes from shapes, and the
card's name and power limit.

    python tools/bench_deepstem.py [--steps 10] [--warmup 3] [--precision f16x3] [--size 513] [--lbs 8] [--ubs 8]
"""
import argparse
import json
import os
import random
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

CONV_LAUNCHES = ('pxl_conv_h16_launch', 'pxl_conv_wgrad_h16_launch', 'pxl_conv_tc_launch_ex', 'pxl_conv_wgrad_tc_launch')
UNFOLDS = ('pxl_stem3x3s2_im2col_h16', 'pxl_stem3x3s2_im2col')


def card():
    info = {'name': torch.cuda.get_device_name(0), 'power_limit_w': None}
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info['power_limit_w'] = float(out.splitlines()[0])
    except Exception as e:          # the figure is reported as unknown, never guessed
        info['power_limit_error'] = str(e)
    return info


def build_engine(args, backbone):
    from pixelssl_b200 import runner
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    cfg = {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 3,
           'ema_decay': 0.99, 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9,
           'batch_size': args.lbs + args.ubs, 'unlabeled_batch_size': args.ubs, 'backbone': backbone,
           'output_stride': 16, 'models': {'model': 'deeplabv3plus'}}
    return runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=662))


def run_steps(alg, batches, count, epoch):
    alg._train([((batches[i % len(batches)][0],), (batches[i % len(batches)][1],)) for i in range(count)], epoch)


def timed(alg, args, batches):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run_steps(alg, batches, args.steps, 1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    # peak memory: both engines' parameters and optimizer state stay resident, only this backbone's step runs
    return {'images_per_s': (args.lbs + args.ubs) * args.steps / (ms / 1e3), 'ms_per_step': ms / args.steps,
            'peak_mem_gib': torch.cuda.max_memory_allocated() / 2 ** 30}


def stem_kernels(alg, args, batches):
    """One step with CUDA events around the unfold and every convolution launch; keeps the launches at the stem's
    output resolution (the stem's three convolutions: forward, dgrad of the two that have one, wgrad)."""
    from pixelssl_b200 import ops
    oh = (args.size - 1) // 2 + 1
    for k in UNFOLDS + CONV_LAUNCHES:
        ops.kernel_timer_start(k)
    run_steps(alg, batches, 1, 2)
    n = args.lbs + args.ubs
    out = {}
    for k in UNFOLDS:
        t = ops.kernel_timer_stop(k)
        if t:
            lanes = 64 if k.endswith('h16') else 32
            per = n * (3 * args.size * args.size * 4 + oh * oh * lanes * 4)      # image read, matrix written (4 B/lane)
            out[k] = {'launches': len(t), 'ms_total': sum(t), 'bytes_each': per,
                      'gb_per_s': per * len(t) / (sum(t) / 1e3) / 1e9}
    convs = []
    for k in CONV_LAUNCHES:
        for ms, meta in ops.kernel_timer_stop(k, with_meta=True):
            if meta is None or (' %dx%d ' % (oh, oh)) not in meta[1]:
                continue
            toks = {k: int(v) for k, v in re.findall(r'\b(N|Cin|Cout|taps)(\d+)', meta[1])}
            px = toks['N'] * oh * oh
            # algorithmic bytes: the operands as the kernel reads them (fp16 pairs, 4 B per value) once, the fp32 output
            # written once; weights are negligible
            byts = px * (toks['Cin'] + toks['Cout']) * 4
            convs.append({'launch': meta[1], 'ms': ms, 'gflop': meta[0] / 1e9, 'tflop_per_s': meta[0] / (ms / 1e3) / 1e12,
                          'bytes': byts})
    out['stem_resolution_convs'] = convs
    out['stem_resolution_convs_ms_total'] = sum(c['ms'] for c in convs)
    return out


def stock_torch(args, batches):
    from oracle import deeplabv3plus_oracle as D
    from oracle import deepstem_oracle as S
    torch.backends.cudnn.allow_tf32 = True
    dev = torch.device('cuda:0')
    with S.deep_stem():
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
            one(i)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    return {'images_per_s': (args.lbs + args.ubs) * args.steps / dt, 'ms_per_step': dt * 1e3 / args.steps,
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
        raise SystemExit('bench_deepstem: needs a CUDA device')
    torch.cuda.set_device(0)
    from oracle import sseg_oracle as O
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, args.lbs + args.ubs, args.lbs, args.size, args.size))
               for i in range(2)]
    res = {'metric': 'DeepLabV3+-R101 OS16 Mean-Teacher step, %d+%d x %dx%d, %s' % (args.lbs, args.ubs, args.size,
                                                                                  args.size, args.precision),
           'steps': args.steps, 'warmup': args.warmup, 'card': card()}
    if not args.skip_torch:         # first, so that its peak memory does not include the engine's caches
        try:
            res['stock_torch_deepstem'] = stock_torch(args, batches)
        except torch.cuda.OutOfMemoryError as e:
            res['stock_torch_deepstem'] = {'error': 'out of memory: %s' % str(e).splitlines()[0]}
        torch.cuda.empty_cache()
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    ops.set_conv_precision(args.precision)
    names = ('resnet101-deepstem', 'resnet101')
    algs = {b: build_engine(args, b) for b in names}
    for b in names:
        run_steps(algs[b], batches, args.warmup, 0)
    runs = {b: [] for b in names}
    for _ in range(2):
        for b in names:
            runs[b].append(timed(algs[b], args, batches))
    res['engine'] = {b: {'runs': runs[b], 'images_per_s_median': float(np.median([r['images_per_s'] for r in runs[b]]))}
                     for b in names}
    res['deepstem_vs_7x7'] = res['engine'][names[0]]['images_per_s_median'] / res['engine'][names[1]]['images_per_s_median']
    res['deepstem_kernels_one_step'] = stem_kernels(algs[names[0]], args, batches)
    res['status'] = (ops.conv_tc_status(), ops.h16_status())
    print(json.dumps(res))


if __name__ == '__main__':
    main()
