"""OHEM cross-entropy (ohem_sseg_criterion): the criterion alone, forward plus fused gradient, against the stock torch
restatement (the oracle, oracle/ohem_oracle.py, on the same GPU), and a Mean-Teacher DeepLab-v2-R101 step with
ohem_sseg_criterion against the same step with sseg_criterion.  Prints one JSON line with the card's name and power
limit.

Criterion shapes: 8 x 21 x 513^2 with k = 100 000, and 8 x 19 x 801^2 (UniMatch's Cityscapes crop) with k = 200 000.
For each, tau is taken from the q distribution of the map: once at the q of rank 2k (at least k pixels have q <= tau:
the early exit, T = tau) and once at the q of rank k/2 (fewer than k: the radix selection runs, T = t_k).  Kernel times
are CUDA events around each pxl_ohem_ce call; bytes are the call's algorithmic traffic, ``ops.ohem_bytes`` with the
K and the path the call's stats report (the logits are read for the kept pixels only; the refinement passes read q
when the selection runs), shown against the H100 SXM data sheet's 3.35 TB/s.  The step runs 8 labeled + 8 unlabeled
513x513 images; the criteria alternate in one session, ``--windows`` windows of ``--steps`` steps each, and the
fp16-pair saturation count is reset before and read after every window.  A random-init network's q is near 1/21, so
the default tau = 0.7 takes the early exit; the step also runs with tau = 0 (the selection every step).  Trained on
its hardest pixels only, a random-init network diverges at the usual learning rate and its fp16 pairs saturate, so
the step uses a small one (``--step-lr``); the kernels and their launches do not depend on its value.

    python tools/bench_ohem.py [--reps 20] [--steps 6] [--warmup 2] [--windows 4] [--step-lr 2.5e-6]
                               [--precision f16x3] [--skip-step]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.bench_deeplabv3plus import card

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
SHAPES = [(8, 21, 513, 513, 100000), (8, 19, 801, 801, 200000)]


def _maps(n, c, h, w):
    g = torch.Generator(device='cuda').manual_seed(0)
    logits = torch.randn(n, c, h, w, device='cuda', generator=g) * 3
    labels = torch.randint(0, c, (n, 1, h, w), device='cuda', generator=g).float()
    labels[torch.rand(n, 1, h, w, device='cuda', generator=g) < 0.1] = 255
    return logits, labels


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def criterion_alone(ops, reps):
    from oracle import ohem_oracle as H
    out = []
    for n, c, h, w, k in SHAPES:
        logits, labels = _maps(n, c, h, w)
        q = ops.ohem_raw(logits, labels, 255, -1.0, 1)[2]
        qs = torch.sort(q[labels[:, 0] != 255])[0]
        for path, tau in (('early_exit', float(qs[2 * k - 1])), ('selection', float(qs[k // 2 - 1]))):
            stats = ops.ohem_raw(logits, labels, 255, tau, k, upstream_const=1.0 / n)[3].cpu().tolist()
            ops.kernel_timer_start('pxl_ohem_ce')
            for _ in range(reps):
                ops.ohem_raw(logits, labels, 255, tau, k, upstream_const=1.0 / n)
            rec = ops.kernel_timer_stop('pxl_ohem_ce', with_meta=True)
            ms = float(np.median([t for t, _ in rec]))
            # every call of the loop has the inputs, and so the K and the path, of the call above
            nbytes = ops.ohem_bytes(n, c, h * w, int(stats[1]), not np.isnan(stats[3]), True)
            x = logits.clone().requires_grad_(True)

            def torch_step():
                x.grad = None
                H.ohem_criterion(x, labels, 255, tau, k).mean().backward()
            torch_ms = _time(torch_step, max(reps // 4, 3))
            gbs = nbytes / (ms * 1e-3) / 1e9
            assert (path == 'selection') == (not np.isnan(stats[3])), (path, stats)
            out.append({'shape': [n, c, h, w], 'k': k, 'tau': tau, 'path': path, 'V': int(stats[0]), 'K': int(stats[1]),
                        'T': stats[2], 'engine_ms': round(ms, 4), 'bytes': nbytes, 'GB_per_s': round(gbs, 1),
                        'share_of_3.35TB_per_s': round(gbs * 1e9 / HBM_BYTES_PER_S, 3),
                        'stock_torch_ms': round(torch_ms, 3), 'speedup': round(torch_ms / ms, 1)})
            del x
        del logits, labels, q, qs
        torch.cuda.empty_cache()
    return out


def mt_step(ops, args):
    from pixelssl_b200 import runner
    from pixelssl_b200._lib import call
    from oracle import sseg_oracle as O
    lbs, ubs, size = 8, 8, 513
    batches = [tuple(t.cuda() for t in O.synthetic_batch(1234 + i, lbs + ubs, lbs, size, size)) for i in range(2)]
    variants = {'sseg_criterion': {}, 'ohem_tau0.7': {'ohem_thresh': 0.7}, 'ohem_tau0': {'ohem_thresh': 0.0}}
    algs = {}
    for name, extra in variants.items():
        cfg = dict(ssl_algorithm='ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=1, ema_decay=0.99,
                   lr=args.step_lr, momentum=0.9, weight_decay=0.0005, epochs=20, log_freq=10 ** 9, batch_size=lbs + ubs,
                   unlabeled_batch_size=ubs, output_stride=16, backbone='resnet101',
                   criterions={'model': 'sseg_criterion' if not extra else 'ohem_sseg_criterion'}, **extra)
        if extra:
            cfg['ohem_min_kept'] = 100000
        torch.manual_seed(0)
        algs[name] = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=662))

    def steps(alg, count, epoch):
        alg._train([((batches[i % 2][0],), (batches[i % 2][1],)) for i in range(count)], epoch)

    for alg in algs.values():
        steps(alg, args.warmup, 0)
    times = {name: [] for name in algs}
    saturated = {name: [] for name in algs}
    for rnd in range(args.windows):      # alternate the criteria
        for name, alg in algs.items():
            torch.cuda.synchronize()
            call('pxl_h16_reset_status')
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            steps(alg, args.steps, 1 + rnd)
            e1.record()
            torch.cuda.synchronize()
            times[name].append((lbs + ubs) * args.steps / (e0.elapsed_time(e1) / 1e3))
            saturated[name].append(ops.h16_status())
    res = {'metric': 'MT DeepLab-v2-R101 OS16 step, %d+%d x %dx%d, images/s per window' % (lbs, ubs, size, size),
           'conv_precision': args.precision, 'lr': args.step_lr,
           'images_per_s': {k: [round(v, 1) for v in t] for k, t in times.items()},
           'median_images_per_s': {k: round(float(np.median(t)), 1) for k, t in times.items()},
           'h16_saturations_per_window': saturated,
           's_task_loss': {k: float(a.meters['s_task_loss'].val) for k, a in algs.items()},
           'conv_tc_status': ops.conv_tc_status()}
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--reps', type=int, default=20)
    p.add_argument('--steps', type=int, default=6)
    p.add_argument('--warmup', type=int, default=2)
    p.add_argument('--precision', default='f16x3')
    p.add_argument('--windows', type=int, default=4)
    p.add_argument('--step-lr', type=float, default=2.5e-6)
    p.add_argument('--skip-step', action='store_true')
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ohem: needs a CUDA device')
    torch.cuda.set_device(0)
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    ops.set_conv_precision(args.precision)
    res = {'card': card(), 'criterion': criterion_alone(ops, args.reps)}
    if not args.skip_step:
        res['mt_step'] = mt_step(ops, args)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
