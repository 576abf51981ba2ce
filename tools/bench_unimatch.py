"""UniMatch training step (ssl_unimatch): one DeepLabV3+-R101 (or --model deeplabv2) task model, output stride 16,
engine kernels against the same step written with stock torch ops (the CPU oracle, oracle/unimatch_oracle.py, run on
the same GPU with cuDNN's defaults and torchvision's augmentation).  Prints one JSON line: images/s and peak memory of
both, the CUDA-event time of every pxl_unimatch_ce and pxl_strong_aug launch of one extra step with its bytes, GB/s
and share of the H100 SXM data-sheet bandwidth, and the card's name and power limit.

The networks start from random weights.  Their BatchNorm running statistics are first set to the batch statistics of
one training-mode forward (as a trained network's are), so the step's eval-mode forward stays in the range of the
fp16-pair convolutions.  The default threshold 0 supervises every pixel, so the loss kernel moves all the bytes its
timer metadata counts (a random-init network is never confident enough for UniMatch's 0.95).

    python tools/bench_unimatch.py [--model deeplabv3plus] [--steps 10] [--warmup 3] [--precision f16x3]
                                   [--size 513] [--lbs 8] [--ubs 8] [--threshold 0] [--skip-torch]
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

from tools.bench_deeplabv3plus import card

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
TIMED = ('pxl_unimatch_ce', 'pxl_strong_aug')
LOSSES = ('task_loss', 's1_loss', 's2_loss', 'fp_loss')


def engine(args, batches):
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import runner, ops
    ops.set_conv_precision(args.precision)
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    cfg = {'ssl_algorithm': 'ssl_unimatch', 'uni_threshold': args.threshold, 'uni_scale': 1.0, 'uni_rampup_epochs': 0,
           'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9,
           'batch_size': args.lbs + args.ubs, 'unlabeled_batch_size': args.ubs, 'backbone': 'resnet101',
           'output_stride': 16, 'models': {'model': args.model}}
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=662))
    from pixelssl_b200.nn.modules import BatchNorm2d
    bns = [m for m in alg.model.modules() if isinstance(m, BatchNorm2d)]
    saved = [m.momentum for m in bns]
    for m in bns:
        m.momentum = 1.0
    alg.model.train()
    with torch.no_grad():
        alg.model.forward((batches[0][0],))
    for m, mom in zip(bns, saved):
        m.momentum = mom

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
    losses = {k: float(alg.meters[k].val) for k in LOSSES + ('mask_ratio',)}
    # one more step with CUDA events around every timed launch (outside the timed window)
    for name in TIMED:
        ops.kernel_timer_start(name)
    steps(1, 2)
    launches = {}
    for name in TIMED:
        launches[name] = []
        for t_ms, nbytes in ops.kernel_timer_stop(name, with_meta=True):
            gbs = nbytes / (t_ms * 1e-3) / 1e9
            launches[name].append({'ms': round(t_ms, 4), 'bytes': nbytes, 'GB_per_s': round(gbs, 1),
                                   'share_of_3.35TB_per_s': round(gbs * 1e9 / HBM_BYTES_PER_S, 3)})
    status = (ops.conv_tc_status(), ops.h16_status())
    del alg
    torch.cuda.empty_cache()
    return {'value': (args.lbs + args.ubs) * args.steps / (ms / 1e3), 'unit': 'images/s', 'ms_per_step': ms / args.steps,
            'peak_mem_gib': peak / 2 ** 30, 'losses': losses, 'conv_precision': args.precision,
            'launches_one_step': launches, 'status': status}


def stock_torch(args, batches):
    from oracle import unimatch_oracle as U
    from oracle import deeplabv3plus_oracle as D
    from oracle import sseg_oracle as O
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params, draw_fp_scales
    init = D.init if args.model == 'deeplabv3plus' else O.init_deeplabv2
    chans = (256, 2048) if args.model == 'deeplabv3plus' else (2048,)
    dev = torch.device('cuda:0')
    state = {k: v.to(dev) for k, v in init(0).items()}
    saved = O.batch_norm.__defaults__
    O.batch_norm.__defaults__ = (1.0,) + saved[1:]
    try:
        with torch.no_grad():
            (D.forward if args.model == 'deeplabv3plus' else O.deeplabv2_forward)(batches[0][0], state, True)
    finally:
        O.batch_norm.__defaults__ = saved
    orc = U.UniMatchOracle(state, model=args.model, lr=0.00025, momentum=0.9, weight_decay=0.0005,
                           max_iters=20 * 662, threshold=args.threshold, scale=1.0, rampup_steps=0)
    rng = np.random.RandomState(0)

    def one(i):
        img, lab = batches[i % len(batches)]
        table, boxes = draw_strong_params(args.ubs, args.size, args.size, 0.5, rng=rng)
        scales = [s.to(dev) for s in draw_fp_scales(args.lbs + args.ubs, chans, 0.5)]
        return orc.step(img, lab, args.lbs, table, boxes, scales)

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
            'peak_mem_gib': peak / 2 ** 30, 'losses': {k: float(out[k]) for k in LOSSES},
            'torch_conv': 'cuDNN, TF32 allowed=%s' % torch.backends.cudnn.allow_tf32}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--model', default='deeplabv3plus', choices=['deeplabv2', 'deeplabv3plus'])
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--precision', default='f16x3')
    p.add_argument('--size', type=int, default=513)
    p.add_argument('--lbs', type=int, default=8)
    p.add_argument('--ubs', type=int, default=8)
    p.add_argument('--threshold', type=float, default=0.0)
    p.add_argument('--skip-torch', action='store_true')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_unimatch: needs a CUDA device')
    torch.cuda.set_device(0)
    from oracle import sseg_oracle as O
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, args.lbs + args.ubs, args.lbs, args.size, args.size))
               for i in range(2)]
    name = {'deeplabv2': 'DeepLab-v2-R101', 'deeplabv3plus': 'DeepLabV3+-R101'}[args.model]
    res = {'metric': '%s OS16 UniMatch step, %d+%d x %dx%d' % (name, args.lbs, args.ubs, args.size, args.size),
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
