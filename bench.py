#!/usr/bin/env python
"""Benchmark of the PixelSSL sseg SSL-training hot path on H100.

    python bench.py --gpus N --steps K --warmup W [--config mt|cutmix|gct|cct] [--precision f16x3|f16|tf32x3|tf32|fp32]
                    [--dump-outputs DIR]
    python bench.py --impl reference --gpus N --steps K --warmup W          (torchrun for N > 1)

Default workload (BASELINE.json configs[1]): Mean-Teacher, DeepLab-v2-ResNet101 OS16, per-GPU batch 16
(8 labeled + 8 unlabeled) of 513x513 synthetic images, 21 classes, cons_for_labeled=False, cons_scale 1,
ema_decay .99, SGD(2.5e-4, .9, 5e-4) + PolynomialLR - weak scaling over GPUs.  ``--config`` selects the other
BASELINE configurations (cutmix = configs[2]; gct = configs[3]: PSPNet-R50 713x713, 1+1 per GPU, meant for N=4;
cct = configs[4]: 11 perturbation decoders, 2+2 per GPU, meant for N=8).  A "step" is one full iteration of the
algorithm's ``_train`` loop body: zero_grad, forward(s), losses, backward, gradient all-reduce (N>1), fused
optimiser (+EMA) step, LR step.

Printed JSON line (rank 0), keys as in the task statement:
  value      steps timed with the batches already in HBM (``algorithm._train`` on device batches, log_freq off)
  e2e        ``algorithm.train(data_loader, epoch)`` - the plugin API a PixelSSL user calls - on pinned HOST batches
             with log_freq = 1: H2D of every batch and a D2H read of every step's losses inside the timed region
  roofline   the DOMINANT kernel: the wgmma forward/dgrad convolution.  achieved = algorithmic FLOPs (2*M*K*N per
             launch) / CUDA-event time of its launches, measured live in an instrumented pass right after the timed
             region (events around ~300 launches per step would perturb ``value``); peak = the measured dense 16-bit
             tensor throughput of MEASURED_PEAKS.json when present, else the H100 SXM data-sheet figures (989 TFLOP/s
             dense 16-bit, 3.35 TB/s HBM3)
  roofline_wgrad / roofline_hbm   the same for the wgrad kernel and for the metric kernel of BASELINE.json (fused MSE
             consistency fwd+bwd, 12 B/element, HBM-bound; timed inside the timed steps)
  step_tensor_frac   whole-step algorithmic TFLOP/s over the same tensor peak
  alt_precision      ``value`` again with the single-pass mode of the same kernel family (TF32-grade numerics, what
             cuDNN gives the reference on a GPU); the headline is the fp32-grade mode
  gpu_torch_baseline the reference step written with stock PyTorch ops (oracle port on cuda:0: NCHW, cuDNN TF32
             default, eager) on this GPU - the "reference's 1-GPU PyTorch images/sec" of the north_star target
  cpu_baseline / ``--impl reference``   the CPU oracle port of the reference step (torch CPU fp32, up to 32 host
             threads) on a bounded sample.
  --dump-outputs DIR   after the timed steps: what the last timed step computed, as DIR/<name>.npy (losses of the
             step, a fixed seeded sample of each trained model's updated parameters and BN buffers); the inputs are
             seeded, so two builds can be compared output for output."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

H = W = 513
LBS, UBS = 8, 8
NUM_CLASSES = 21
MT_FLOP_PER_IMG = 451e9          # SURVEY.md 8(d): student fwd+bwd 338.4 + teacher fwd 112.8 GFLOP
_BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 9}


def mt_config():
    return dict(_BASE, ssl_algorithm='ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=3,
                ema_decay=0.99, batch_size=LBS + UBS, unlabeled_batch_size=UBS, output_stride=16, backbone='resnet101')


# name -> (algorithm config, labeled per GPU, unlabeled per GPU, image size, description); flag values from the
# reference's scripts (task/sseg/script/*_sslcutmix.py:22-28, *_sslgct.py:23-33, *_sslcct.py:23-33)
CONFIGS = {
    'mt': (mt_config, 8, 8, 513,
           'MT (ssl_mt) DeepLab-v2-ResNet101 OS16, per-GPU batch 16 = 8 labeled + 8 unlabeled, 513x513x3 synthetic, '
           '21 classes, cons_for_labeled=False (BASELINE.json configs[1])'),
    'cutmix': (lambda: dict(_BASE, ssl_algorithm='ssl_cutmix', cons_scale=20.0, cons_rampup_epochs=0, cons_threshold=0.97,
                            ema_decay=0.99, mask_prop_range=(0.5, 0.5), batch_size=16, unlabeled_batch_size=8,
                            output_stride=16, backbone='resnet101'), 8, 8, 513,
               'CutMix (ssl_cutmix) DeepLab-v2-ResNet101 OS16, per-GPU batch 16 = 8 labeled + 8 unlabeled, 513x513x3 '
               'synthetic, 21 classes (BASELINE.json configs[2])'),
    'gct': (lambda: dict(_BASE, ssl_algorithm='ssl_gct', models={'model': 'pspnet'}, backbone='resnet50', ssl_mode='gct',
                         fc_ssl_scale=1.0, dc_ssl_scale=100.0, dc_threshold=0.6, dc_rampup_epochs=5, fd_lr=1e-4,
                         fd_scale=10.0, mu=0.5, nu=1, im_size=713, batch_size=2, unlabeled_batch_size=1), 1, 1, 713,
            'GCT (ssl_gct) two PSPNet-ResNet50 task models + flaw detector, per-GPU batch 2 = 1 labeled + 1 unlabeled '
            '(global 8 at N=4), 713x713x3 synthetic (BASELINE.json configs[3])'),
    'cct': (lambda: dict(_BASE, ssl_algorithm='ssl_cct', cons_scale=30.0, cons_rampup_epochs=5, ad_lr_scale=10.0,
                         vat_dec_num=1, drop_dec_num=2, cut_dec_num=2, context_dec_num=1, object_dec_num=1,
                         fd_dec_num=2, fn_dec_num=2, batch_size=4, unlabeled_batch_size=2, output_stride=16,
                         backbone='resnet101'), 2, 2, 513,
            'CCT (ssl_cct) DeepLab-v2-ResNet101 shared encoder + 11 perturbation decoders, per-GPU batch 4 = 2 labeled '
            '+ 2 unlabeled (global 32 at N=8), 513x513x3 synthetic (BASELINE.json configs[4])'),
}


def measured_peaks():
    path = os.path.join(ROOT, 'MEASURED_PEAKS.json')
    if os.path.exists(path):
        d = json.load(open(path))
        return d.get('hbm_gbs', 3350.0), d.get('bf16_tflops_sustained', 989.0), 'measured'
    return 3350.0, 989.0, 'H100 SXM data sheet'


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = 'index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,' \
        'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,' \
        'clocks_event_reasons.sw_power_cap'

    def __init__(self, gpu_index):
        self.idx, self.proc, self.lines = gpu_index, None, []

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', '-i', str(self.idx), '--query-gpu=' + self.Q,
                                          '--format=csv,noheader,nounits', '-lms', '100'],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for line in self.lines:
            f = [x.strip() for x in line.split(',')]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(('hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap'), f[4:8]):
                if v.lower().startswith('active'):
                    reasons.add(name)
        sm.sort()
        return {'sm_mhz': sm[len(sm) // 2] if sm else None, 'sm_max_mhz': mx, 'reasons': sorted(reasons),
                'samples': len(sm)}


def synthetic_host_batches(count, rank, pin, lbs=None, ubs=None, size=None):
    import torch
    lbs = LBS if lbs is None else lbs
    ubs = UBS if ubs is None else ubs
    size = H if size is None else size
    g = torch.Generator().manual_seed(1234 + rank)
    out = []
    for _ in range(count):
        img = torch.randn(lbs + ubs, 3, size, size, generator=g)
        lab = torch.randint(0, NUM_CLASSES, (lbs + ubs, 1, size, size), generator=g).float()
        ign = torch.rand(lbs + ubs, 1, size, size, generator=g) < 0.05
        lab[ign] = 255.0
        lab[lbs:] = -1.0
        if pin:
            img, lab = img.pin_memory(), lab.pin_memory()
        out.append((img, lab))
    return out


def _roofline_from(records, peak, src, kernel, bound='tensor', traffic=None):
    """records: [(ms, flop)] of one entry point's launches -> roofline block (TFLOP/s against the measured 16-bit peak)."""
    records = [(ms, fl[0] if isinstance(fl, tuple) else fl) for ms, fl in records if fl]
    if not records:
        return None
    ms, fl = sum(r[0] for r in records), sum(r[1] for r in records)
    ach = fl / (ms * 1e-3) / 1e12
    return {'kernel': kernel, 'bound': bound, 'achieved': ach, 'peak': peak, 'unit': 'TFLOP/s', 'frac': ach / peak,
            'traffic': traffic, 'launches_timed': len(records), 'avg_launch_ms': ms / len(records),
            'algorithmic_flop_per_launch': fl / len(records), 'peak_source': src}


def ddp_check(world, rank, precision):
    """N > 1 only, before the timed region: (a) a 65x65 Mean-Teacher step run data-parallel (1 labeled + 1 unlabeled
    image per rank) against the SAME global batch run by rank 0 alone as one big batch - gradients, updated
    parameters and BN running statistics must agree (the reference synchronises BN statistics across replicas,
    sync_batchnorm/batchnorm.py:55-78, and averages gradients); (b) every rank must hold bit-identical parameters
    and BN buffers after the step.  Differences between (a)'s two runs come from the order of the fp32 partial sums
    inside the BN statistics (row -> tile assignment differs between a 2*world-image batch and 2-image shards),
    amplified by the 101-layer random-init net on 5x5 feature maps (DESIGN.md section 2); they are reported, and
    bounded by the same limits as tests/test_gpu_ddp.py."""
    import torch
    import torch.distributed as dist
    from pixelssl_b200 import runner, ops
    from pixelssl_b200.nn import arena as arena_mod
    from pixelssl_b200.nn.modules import BatchNorm2d
    size = 65
    prev = {v: k for k, v in ops.PRECISION.items()}[ops.get_conv_precision()]
    ops.set_conv_precision(precision)

    def cfg(bs, ubs):
        return dict(_BASE, ssl_algorithm='ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=0,
                    ema_decay=0.99, batch_size=bs, unlabeled_batch_size=ubs, output_stride=16, backbone='resnet101')

    def flat(alg):
        sp = list(alg.s_model.module.model.parameters())
        grads = torch.cat([p.grad.contiguous().reshape(-1) for p in sp]).double()
        params = alg.s_model.arena.data.double().clone()
        bufs = torch.cat([b.reshape(-1).double() for n, b in alg.s_model.named_buffers() if 'num_batches' not in n])
        return grads, params, bufs

    g = torch.Generator().manual_seed(4242)
    img = torch.randn(2 * world, 3, size, size, generator=g)
    lab = torch.randint(0, NUM_CLASSES, (2 * world, 1, size, size), generator=g).float()
    lab[world:] = -1.0
    torch.manual_seed(7)
    alg = runner.build_algorithm(runner.build_args(cfg(2, 1), iters_per_epoch=5))      # parameters broadcast from rank 0
    state = {k: v.clone() for k, v in alg.s_model.state_dict().items()}
    alg.t_model.load_state_dict(state)
    idx = [rank, world + rank]
    alg._train([((img[idx].cuda(),), (lab[idx].cuda(),))], 0)
    gd, pd, bd = flat(alg)
    # (b) cross-rank equality of the updated parameters and BN running statistics
    sums = torch.stack([pd.sum(), (pd * pd).sum(), bd.sum(), (bd * bd).sum()])
    allsums = [torch.empty_like(sums) for _ in range(world)]
    dist.all_gather(allsums, sums)
    equal = all(torch.equal(allsums[0], t) for t in allsums)
    res = {'ranks_hold_identical_params_and_bn_buffers': bool(equal)}
    if rank == 0:
        def big_batch(perm):
            arena_mod.DISTRIBUTED = False
            try:
                big = runner.build_algorithm(runner.build_args(cfg(2 * world, world), iters_per_epoch=5))
            finally:
                arena_mod.DISTRIBUTED = True
            big.s_model.load_state_dict(state)
            big.t_model.load_state_dict(state)
            for m in list(big.s_model.modules()) + list(big.t_model.modules()):
                if isinstance(m, BatchNorm2d):
                    m.multi_replica_formula = True       # batchnorm.py:125: the multi-replica path clamps var instead of adding eps
            big._train([((img[perm].cuda(),), (lab[perm].cuda(),))], 0)
            return flat(big)
        ident = list(range(2 * world))
        g1, p1, b1 = big_batch(ident)
        # yardstick: the SAME big batch with its labeled and its unlabeled samples reversed - identical loss, different
        # order of the fp32 partial sums; what a data-parallel run may differ by (tests/test_gpu_ddp.py)
        gp, pp, bp = big_batch(ident[:world][::-1] + ident[world:][::-1])
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))
        noise = {'grad': rel(gp, g1), 'param': rel(pp, p1), 'bn_buffer': rel(bp, b1)}
        res.update({'size': size, 'per_rank_batch': '1 labeled + 1 unlabeled', 'conv_precision': precision,
                    'grad_max_rel_vs_big_batch': rel(gd, g1), 'param_max_rel_vs_big_batch': rel(pd, p1),
                    'bn_buffer_max_rel_vs_big_batch': rel(bd, b1), 'batch_permutation_noise_of_the_big_batch': noise})
        res['ok'] = bool(equal and res['grad_max_rel_vs_big_batch'] <= 3 * noise['grad'] + 1e-3
                         and res['param_max_rel_vs_big_batch'] <= 3 * noise['param'] + 1e-5
                         and res['bn_buffer_max_rel_vs_big_batch'] <= 3 * noise['bn_buffer'] + 1e-5)
    dist.barrier()
    del alg
    torch.cuda.empty_cache()
    ops.set_conv_precision(prev)
    return res


def run_engine(args):
    import random
    import numpy as np
    import torch
    import torch.distributed as dist
    rank = int(os.environ.get('RANK', 0))
    world = int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    import __graft_entry__ as ge
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    import pixelssl_b200
    from pixelssl_b200 import runner, ops
    ops.set_conv_precision(args.precision)
    import logging
    logging.getLogger('PixelSSL').setLevel(logging.ERROR)
    ddp = ddp_check(world, rank, 'fp32') if (world > 1 and not args.no_ddp_check) else None
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    make_cfg, lbs, ubs, size, workload = CONFIGS[args.config]
    nb = 4
    host = synthetic_host_batches(nb, rank, True, lbs, ubs, size)
    dev = [(i.cuda(), l.cuda()) for i, l in host]
    st = {'alg': None, 'a': None, 'epoch': 0}

    def fresh_algorithm():
        """Every timed phase starts from the same freshly initialised models / optimiser state: on random-label
        synthetic batches the reference algorithm itself drifts upwards in loss within tens of steps (the CPU oracle
        does the same, DESIGN.md section 7), so phases run back to back would not time the same regime."""
        if st['alg'] is not None:
            st['alg'] = None
            torch.cuda.empty_cache()
        torch.manual_seed(0); random.seed(0); np.random.seed(0)
        st['a'] = runner.build_args(make_cfg(), iters_per_epoch=662)
        st['alg'] = runner.build_algorithm(st['a'])
        st['epoch'] = 0

    def run_steps(batches, count, api):
        """``count`` iterations through the algorithm's own loop (``_train`` / the public ``train``)."""
        alg = st['alg']
        loader = [((batches[i % nb][0],), (batches[i % nb][1],)) for i in range(count)]
        (alg.train if api else alg._train)(loader, st['epoch'])
        st['epoch'] += 1

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        t = torch.tensor([ms], device='cuda')
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t)

    losses = {}
    clock_rec = []
    sampler = ClockSampler(local) if rank == 0 else None

    def first_loss():
        vals = st['alg'].meters.values()
        return float(next(v for k, v in sorted(vals.items()) if 'task_loss' in k))

    def timed(batches, api=False, tag=None):
        fresh_algorithm()
        st['a'].log_freq = 1 if api else 10 ** 9   # api: every step's losses are read back for its log line
        run_steps(batches, args.warmup, api)
        barrier()
        if tag == 'value' and sampler:
            sampler.start()                   # clocks / throttle reasons DURING the timed region
        ops.reset_launch_count()
        ops.kernel_timer_start('pxl_mse_consistency')
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run_steps(batches, args.steps, api)
        last = first_loss() if api else None                             # the last step's loss is on the host
        e1.record()
        barrier()
        if tag == 'value' and sampler:
            clock_rec.append(sampler.stop())
        ms = e0.elapsed_time(e1)
        ktimes = ops.kernel_timer_stop('pxl_mse_consistency')
        if tag:
            losses[tag] = {'task_loss_after_%d_steps' % (args.warmup + args.steps): last if last is not None else first_loss()}
        return max_over_ranks(ms), ktimes, ops.launch_count()

    sat_log = {}
    ms_dev, ktimes, launches = timed(dev, tag='value')
    if args.dump_outputs and rank == 0:
        dump_outputs(st['alg'], args.dump_outputs)
    sat_log['after_value'] = ops.h16_status_sites()
    clocks = clock_rec[0] if clock_rec else None
    ms_e2e, _, _ = timed(host, api=True, tag='e2e')
    sat_log['after_e2e'] = ops.h16_status_sites()

    # instrumented pass: CUDA events around every convolution launch (outside the timed region on purpose)
    h16 = args.precision in ('f16x3', 'f16')
    fwd_name = 'pxl_conv_h16_launch' if h16 else 'pxl_conv_tc_launch_ex'
    wg_name = 'pxl_conv_wgrad_h16_launch' if h16 else 'pxl_conv_wgrad_tc_launch'
    conv_rec = wg_rec = []
    if args.precision != 'fp32':
        fresh_algorithm()
        st['a'].log_freq = 10 ** 9
        run_steps(dev, 1, False)
        barrier()
        ops.kernel_timer_start(fwd_name); ops.kernel_timer_start(wg_name)
        run_steps(dev, min(args.steps, 3), False)
        conv_rec = ops.kernel_timer_stop(fwd_name, with_meta=True)
        wg_rec = ops.kernel_timer_stop(wg_name, with_meta=True)

    alt = None
    alt_name = {'tf32x3': 'tf32', 'f16x3': 'f16'}.get(args.precision)
    if alt_name and not args.no_alt:
        # secondary figure: the same step with the single-pass mode of the same kernels (11-bit significands: what
        # cuDNN's TF32 default gives the reference on a GPU); not the headline because it is outside the 1e-3
        # tolerance against the CPU reference
        ops.set_conv_precision(alt_name)
        sat_log['before_alt'] = ops.h16_status_sites()
        ms_alt, _, _ = timed(dev, tag='alt')
        ops.set_conv_precision(args.precision)
        alt = {'conv_precision': alt_name, 'value': (lbs + ubs) * world * args.steps / (ms_alt / 1e3), 'unit': 'images/s',
               'ms_per_step': ms_alt / args.steps}
    status = (ops.conv_tc_status(), ops.h16_status())

    imgs = (lbs + ubs) * world * args.steps
    value = imgs / (ms_dev / 1e3)
    e2e = imgs / (ms_e2e / 1e3)
    hbm_peak, tf_peak, peak_src = measured_peaks()
    traffic = {}
    tpath = os.path.join(ROOT, 'profiles', 'kernel_traffic.json')
    if os.path.exists(tpath):
        traffic = json.load(open(tpath))
    kname = {'f16x3': 'conv_wg_kernel, wgmma f16 x3 (fp16 pairs)', 'f16': 'conv_wg_kernel, wgmma f16',
             'tf32x3': 'conv_wg_kernel, wgmma tf32 x3', 'tf32': 'conv_wg_kernel, wgmma tf32'}
    roof = _roofline_from(conv_rec, tf_peak, peak_src, 'forward/dgrad convolution: ' + kname.get(args.precision, ''),
                          traffic=traffic.get('conv_fwd_dram_bytes_per_launch'))
    roof_wg = _roofline_from(wg_rec, tf_peak, peak_src, 'conv_wgrad_wg_kernel (' + args.precision + ')',
                             traffic=traffic.get('conv_wgrad_dram_bytes_per_launch'))
    mma_per_product = 3 if args.precision in ('f16x3', 'tf32x3') else 1
    for r in (roof, roof_wg):
        if r:
            r['mma_rate_frac'] = r['frac'] * mma_per_product * (2.0 if args.precision in ('tf32', 'tf32x3') else 1.0)
            r['note'] = ('achieved counts each product once; the fp32-grade modes issue 3 MMAs per product, tf32 '
                         'runs at half the 16-bit rate: mma_rate_frac = tensor-pipe rate over the same peak')
    n_elem = ubs * NUM_CLASSES * size * size
    k_ms = sum(ktimes) / max(len(ktimes), 1) if ktimes else float('nan')
    achieved = 12.0 * n_elem / (k_ms * 1e-3) / 1e9 if ktimes else None
    roof_hbm = {'kernel': 'mse_vec_kernel<true> (pxl_mse_consistency, fused fwd+bwd)', 'bound': 'hbm',
                'achieved': achieved, 'peak': hbm_peak, 'unit': 'GB/s',
                'frac': (achieved / hbm_peak) if achieved else None,
                'traffic': traffic.get('mse_dram_bytes_per_launch'),
                'algorithmic_bytes_per_launch': 12.0 * n_elem, 'avg_launch_ms': k_ms,
                'launches_timed': len(ktimes), 'peak_source': peak_src} if ktimes else None
    out = {
        'metric': 'images/sec DeepLab-v2-R101 MT 513x513 bs16' if args.config == 'mt' else 'images/sec ' + args.config,
        'value': value, 'unit': 'images/s',
        'n_gpus': world, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': ms_dev / args.steps,
        'higher_is_better': True, 'scaling': 'weak', 'vs_baseline': None,
        'dtype': {'fp32': 'f32', 'tf32': 'tf32', 'tf32x3': 'tf32x3', 'f16x3': 'f16x3 (fp16 pairs, fp32 accumulate)',
                  'f16': 'f16 (fp32 accumulate)'}[args.precision], 'data': 'synthetic',
        'config': {'workload': workload, 'name': args.config,
                   'global_batch': (lbs + ubs) * world, 'parallelism': 'dp%d' % world,
                   'conv_precision': args.precision, 'weights': 'random init (reference initialisers)',
                   'l2': 'inputs and activations (>20 GB/step) far exceed the 50 MB L2; no explicit flush'},
        'e2e': {'value': e2e, 'unit': 'images/s',
                'h2d_bytes_per_step': (lbs + ubs) * (3 + 1) * size * size * 4, 'd2h_bytes_per_step': 24,
                'api': 'algorithm.train(data_loader, epoch) on pinned host batches, log_freq=1 (losses read back every step)'},
        'gpu_launches': launches,
        'clocks': clocks,
        'roofline': roof if roof else roof_hbm,
        'roofline_wgrad': roof_wg,
        'roofline_hbm': roof_hbm,
        'losses': losses,
        'pipeline_status': {'conv_watchdog': status[0], 'fp16_pair_saturations': status[1],
                            'saturations_by_site_split_fixed_dyn_bnapply_bndx': ops.h16_status_sites(), 'phases': sat_log},
    }
    if args.config == 'mt':
        ach = MT_FLOP_PER_IMG * (lbs + ubs) / (ms_dev / args.steps / 1e3) / 1e12
        out['step_tflops'] = {'algorithmic_flop_per_step_per_gpu': MT_FLOP_PER_IMG * (lbs + ubs),
                              'achieved_tflops_per_gpu': ach, 'tensor_peak_tflops': tf_peak, 'peak_source': peak_src}
        out['step_tensor_frac'] = ach / tf_peak
    if alt is not None:
        out['alt_precision'] = alt
    if ddp is not None:
        out['ddp_check'] = ddp
    if rank == 0:
        if world == 1 and args.config == 'mt':
            st['alg'] = None
            del dev
            torch.cuda.empty_cache()
            if not args.no_gpu_torch_baseline:
                r = stock_torch_gpu_reference(steps=50, warmup=10, lbs=LBS, ubs=UBS)
                out['gpu_torch_baseline'] = {'value': r['value'], 'unit': 'images/s', 'ms_per_step': r['seconds'] / 50 * 1e3,
                                             'steps': 50, 'warmup': 10, 'dtype': 'tf32 (cuDNN default)', 'what': r['sample'],
                                             'engine_over_baseline': value / r['value'],
                                             'engine_alt_over_baseline': (alt['value'] / r['value']) if alt else None}
                torch.cuda.empty_cache()
            if not args.no_cpu_baseline:
                out['cpu_baseline'] = cpu_reference(steps=2, warmup=1, lbs=1, ubs=1)     # ~15-30 s of CPU work
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def dump_outputs(alg, out_dir):
    """What the last timed step handed back to the caller of ``_train``: its losses and the updated models.  The
    parameter vectors are large, so a fixed seeded sample of 2^20 entries of each model's state is stored."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    losses = {k: float(v) for k, v in alg.meters.values().items() if 'loss' in k}
    np.save(os.path.join(out_dir, 'losses.npy'), np.array([losses[k] for k in sorted(losses)], dtype=np.float64))
    with open(os.path.join(out_dir, 'losses.json'), 'w') as f:
        json.dump(sorted(losses), f)
    g = torch.Generator().manual_seed(2024)
    # every model the algorithm trains (MT / CutMix: s_model, t_model; GCT: l_model, r_model, fd_model; CCT: model,
    # which holds the main network and all auxiliary decoders)
    for name, model in sorted(alg.models.items()):
        state = model.state_dict()
        flat = torch.cat([state[k].detach().reshape(-1).float().cpu() for k in sorted(state)
                          if state[k].is_floating_point()])
        idx = torch.randint(0, flat.numel(), (1 << 20,), generator=g)
        np.save(os.path.join(out_dir, '%s_state_sample.npy' % name), flat[idx].numpy().astype(np.float32))


def cpu_reference(steps, warmup, lbs, ubs):
    """The reference's CPU path restated by the oracle (torch CPU fp32; the Python reference itself
    cannot travel to the GPU box), all host threads, on a bounded sample of the workload."""
    import torch
    from oracle import sseg_oracle as O
    # all host cores up to 32: torch's CPU conv/BN kernels at batch 2 get SLOWER beyond that
    # (measured on the 128-core GPU box: 112 s/step with 128 threads vs ~5 s/step with 8-32)
    cores = min(os.cpu_count() or 1, 32)
    torch.set_num_threads(cores)
    s, t = O.init_deeplabv2(0), O.init_deeplabv2(1)
    mt = O.MTOracle(s, t, lr=0.00025, momentum=0.9, weight_decay=0.0005, max_iters=20 * 662, cons_scale=1.0,
                    rampup_steps=3 * 662, ema_decay=0.99, cons_for_labeled=False)
    batches = [O.synthetic_batch(1234 + i, lbs + ubs, lbs, H, W) for i in range(2)]
    for i in range(warmup):
        mt.step(batches[i % 2][0], batches[i % 2][1], lbs)
    t0 = time.perf_counter()
    for i in range(steps):
        mt.step(batches[i % 2][0], batches[i % 2][1], lbs)
    dt = time.perf_counter() - t0
    return {'value': (lbs + ubs) * steps / dt, 'unit': 'images/s', 'cores': cores, 'kind': 'port',
            'sample': '%d MT steps (after %d warm-up) of DeepLab-v2-R101 at batch %d+%d (labeled+unlabeled), '
                      '513x513, torch CPU fp32, %d threads' % (steps, warmup, lbs, ubs, cores),
            'seconds': dt}


def stock_torch_gpu_reference(steps, warmup, lbs, ubs):
    """Informational only (``--impl reference --ref-device cuda``): the SAME oracle port of the reference
    step run with stock PyTorch/cuDNN ops on cuda:0 (NCHW fp32 storage, cuDNN TF32 convolutions = torch's
    default, no cudnn.benchmark - the reference sets none), full batch.  This is the "reference's 1-GPU
    PyTorch images/sec" that BASELINE.json's >=5x target is phrased against; none of this repo's kernels
    run here."""
    import torch
    from oracle import sseg_oracle as O
    dev = torch.device('cuda:0')
    s = {k: v.to(dev) for k, v in O.init_deeplabv2(0).items()}
    t = {k: v.to(dev) for k, v in O.init_deeplabv2(1).items()}
    mt = O.MTOracle(s, t, lr=0.00025, momentum=0.9, weight_decay=0.0005, max_iters=20 * 662, cons_scale=1.0,
                    rampup_steps=3 * 662, ema_decay=0.99, cons_for_labeled=False)
    batches = [O.synthetic_batch(1234 + i, lbs + ubs, lbs, H, W) for i in range(2)]
    batches = [(a.pin_memory(), b.pin_memory()) for a, b in batches]

    def one(i):
        img, lab = batches[i % 2]
        out = mt.step(img.to(dev, non_blocking=True), lab.to(dev, non_blocking=True), lbs)
        return float(out['s_task_loss'])

    for i in range(warmup):
        one(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        one(i)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {'value': (lbs + ubs) * steps / dt, 'unit': 'images/s', 'seconds': dt,
            'sample': '%d MT steps of DeepLab-v2-R101 at batch %d+%d, 513x513, stock PyTorch ops on cuda:0 '
                      '(oracle port, cuDNN TF32 default)' % (steps, lbs, ubs)}


def run_reference(args):
    rank = int(os.environ.get('RANK', 0))
    if rank != 0:
        return
    if args.ref_device == 'cuda':
        r = stock_torch_gpu_reference(args.steps, args.warmup, 8, 8)
        print(json.dumps({'impl': 'reference', 'ref_device': 'cuda', 'metric': 'images/sec DeepLab-v2-R101 MT 513x513 bs16',
                          'value': r['value'], 'unit': 'images/s', 'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup,
                          'ms_per_step': r['seconds'] / args.steps * 1e3, 'higher_is_better': True, 'dtype': 'tf32 (cuDNN default)',
                          'data': 'synthetic', 'config': {'workload': r['sample'], 'global_batch': 16}, 'gpu_launches': 0,
                          'note': 'informational: stock PyTorch on the GPU, not the CPU reference arm'}))
        return
    cb = cpu_reference(steps=args.steps, warmup=min(args.warmup, 1) if args.steps > 3 else args.warmup, lbs=1, ubs=1)
    out = {'impl': 'reference', 'metric': 'images/sec DeepLab-v2-R101 MT 513x513 bs16', 'value': cb['value'],
           'unit': 'images/s', 'n_gpus': int(os.environ.get('WORLD_SIZE', args.gpus)), 'steps': args.steps,
           'warmup': args.warmup, 'ms_per_step': cb['seconds'] / args.steps * 1e3, 'higher_is_better': True,
           'scaling': 'weak', 'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
           'config': {'workload': 'MT (ssl_mt) DeepLab-v2-ResNet101 OS16 513x513 synthetic, CPU oracle port of the '
                                  'reference step; bounded sample: batch 1 labeled + 1 unlabeled per step',
                      'global_batch': 2, 'parallelism': 'cpu'},
           'cpu_baseline': cb,
           'e2e': {'value': cb['value'], 'unit': 'images/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
           'gpu_launches': 0}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', type=str, default='engine', choices=['engine', 'reference'])
    ap.add_argument('--precision', type=str, default=os.environ.get('PXL_CONV_PRECISION', 'f16x3'),
                    choices=['fp32', 'tf32', 'tf32x3', 'f16x3', 'f16'])
    ap.add_argument('--config', type=str, default='mt', choices=sorted(CONFIGS))
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--no-gpu-torch-baseline', action='store_true')
    ap.add_argument('--no-alt', action='store_true', help='skip the alt_precision pass')
    ap.add_argument('--no-ddp-check', action='store_true', help='N > 1: skip the data-parallel parity check')
    ap.add_argument('--dump-outputs', type=str, default=None, metavar='DIR',
                    help='write what the last timed step computed to DIR/<name>.npy')
    ap.add_argument('--ref-device', type=str, default='cpu', choices=['cpu', 'cuda'],
                    help='--impl reference only: cuda = the oracle port with stock PyTorch ops on cuda:0 (informational)')
    args = ap.parse_args()
    if args.warmup < 3 and args.impl == 'engine':
        args.warmup = 3
    if args.impl == 'reference':
        run_reference(args)
    else:
        run_engine(args)


if __name__ == '__main__':
    main()
