"""Cross Pseudo Supervision training step (ssl_cps): two DeepLab-v2-R101 (or --model deeplabv3plus) task models, output
stride 16, engine kernels against the same step written with stock torch ops (the CPU oracle, oracle/cps_oracle.py,
run on the same GPU with cuDNN's defaults).  --cutmix times the CutMix variant.  Prints one JSON line: images/s and
peak memory of both, the CUDA-event time of every pxl_cps_ce launch of one extra step with its algorithmic bytes,
GB/s and share of the H100 SXM data-sheet bandwidth, and the card's name and power limit.

    python tools/bench_cps.py [--model deeplabv2] [--cutmix] [--steps 10] [--warmup 3] [--precision f16x3]
                              [--size 513] [--lbs 8] [--ubs 8]
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


def engine(args, batches):
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import runner, ops
    ops.set_conv_precision(args.precision)
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    cfg = {'ssl_algorithm': 'ssl_cps', 'cps_scale': 1.5, 'cps_rampup_epochs': 0, 'cps_cutmix': args.cutmix,
           'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9,
           'batch_size': args.lbs + args.ubs, 'unlabeled_batch_size': args.ubs, 'backbone': 'resnet101',
           'output_stride': 16, 'models': {'model': args.model}}
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
    losses = {k: float(alg.meters[k].val) for k in ('l_task_loss', 'r_task_loss', 'l_cps_loss', 'r_cps_loss')}
    # one more step with CUDA events around every pxl_cps_ce launch (outside the timed window)
    ops.kernel_timer_start('pxl_cps_ce')
    steps(1, 2)
    launches = []
    for t_ms, nbytes in ops.kernel_timer_stop('pxl_cps_ce', with_meta=True):
        gbs = nbytes / (t_ms * 1e-3) / 1e9
        launches.append({'ms': round(t_ms, 4), 'bytes': nbytes, 'GB_per_s': round(gbs, 1),
                         'share_of_3.35TB_per_s': round(gbs * 1e9 / HBM_BYTES_PER_S, 3)})
    status = (ops.conv_tc_status(), ops.h16_status())
    del alg
    torch.cuda.empty_cache()
    return {'value': (args.lbs + args.ubs) * args.steps / (ms / 1e3), 'unit': 'images/s', 'ms_per_step': ms / args.steps,
            'peak_mem_gib': peak / 2 ** 30, 'losses': losses, 'conv_precision': args.precision,
            'cps_ce_launches_one_step': launches, 'status': status}


def stock_torch(args, batches):
    from oracle import cps_oracle as C
    from oracle import deeplabv3plus_oracle as D
    from oracle import sseg_oracle as O
    init = D.init if args.model == 'deeplabv3plus' else O.init_deeplabv2
    dev = torch.device('cuda:0')
    l_state = {k: v.to(dev) for k, v in init(0).items()}
    r_state = {k: v.to(dev) for k, v in init(1).items()}
    cps = C.CPSOracle(l_state, r_state, model=args.model, lr=0.00025, momentum=0.9, weight_decay=0.0005,
                      max_iters=20 * 662, cps_scale=1.5, rampup_steps=0, cutmix=args.cutmix)
    rng = np.random.RandomState(0)

    def one(i):
        img, lab = batches[i % len(batches)]
        return cps.step(img, lab, args.lbs, rng)

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
            'peak_mem_gib': peak / 2 ** 30,
            'losses': {k: float(out[k]) for k in ('l_task_loss', 'r_task_loss', 'l_cps_loss', 'r_cps_loss')},
            'torch_conv': 'cuDNN, TF32 allowed=%s' % torch.backends.cudnn.allow_tf32}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--model', default='deeplabv2', choices=['deeplabv2', 'deeplabv3plus'])
    p.add_argument('--cutmix', action='store_true')
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--precision', default='f16x3')
    p.add_argument('--size', type=int, default=513)
    p.add_argument('--lbs', type=int, default=8)
    p.add_argument('--ubs', type=int, default=8)
    p.add_argument('--skip-torch', action='store_true')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_cps: needs a CUDA device')
    torch.cuda.set_device(0)
    from oracle import sseg_oracle as O
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, args.lbs + args.ubs, args.lbs, args.size, args.size))
               for i in range(2)]
    name = {'deeplabv2': 'DeepLab-v2-R101', 'deeplabv3plus': 'DeepLabV3+-R101'}[args.model]
    res = {'metric': '%s OS16 CPS%s step, %d+%d x %dx%d' % (name, ' (CutMix)' if args.cutmix else '', args.lbs, args.ubs,
                                                            args.size, args.size),
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
