"""Multi-view evaluation (task/sseg/evaluation.py) on Cityscapes-shaped input: synthetic 1024 x 2048 images, 19
classes, DeepLabV3+-R101 at output stride 16, eval mode, in ``--precision`` (f16x3).  Prints one JSON line with the
card's name and power limit.

Configurations: the whole image (the default protocol: the plain forward and its softmax), UniMatch's sliding window
(crop 801), and the sliding window over scales (0.75, 1.0, 1.25) with flips.  For each:
  * images/s from CUDA events around ``--steps`` batches, after a warm-up batch that runs every tile shape;
  * the peak memory allocated by torch during the timed batches;
  * the protocol kernels' own time (CUDA events around each pxl_eval_* call) and their algorithmic bytes (every
    value written once, every value read once; ops.eval_* timer metadata), against the H100 SXM data sheet's
    3.35 TB/s;
  * the same protocol as the oracle's torch loop (oracle/eval_oracle.py) around the engine's plain forward, one tile
    at a time, in the same run.

    python tools/bench_eval.py [--steps 3] [--warmup 1] [--batch 1] [--precision f16x3] [--skip-oracle]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.bench_deeplabv3plus import card

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
KERNELS = ('pxl_eval_tiles', 'pxl_eval_merge', 'pxl_eval_view_add', 'pxl_eval_finish')
CONFIGS = {
    'whole': {},
    'sliding_801': {'val_protocol': 'sliding', 'val_crop_size': 801},
    'sliding_801_ms_flip': {'val_protocol': 'sliding', 'val_crop_size': 801, 'val_scales': [0.75, 1.0, 1.25],
                            'val_flip': True},
}


def _build(proto):
    from pixelssl_b200 import runner
    cfg = {'ssl_algorithm': 'ssl_null', 'lr': 0.01, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 1,
           'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True, 'num_classes': 19,
           'output_stride': 16, 'backbone': 'resnet101', 'models': {'model': 'deeplabv3plus'}}
    cfg.update(proto)
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=1))
    alg.model.eval()
    return alg


def _timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.reset_peak_memory_stats()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps, torch.cuda.max_memory_allocated()


def run(args):
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    from pixelssl_b200.task.sseg import evaluation
    from oracle import eval_oracle as E
    ops.set_conv_precision(args.precision)
    g = torch.Generator(device='cuda').manual_seed(0)
    img = torch.randn(args.batch, 3, 1024, 2048, device='cuda', generator=g)
    results = {}
    for name, proto in CONFIGS.items():
        alg = _build(proto)
        plain = alg.model.module.model

        def engine():
            with torch.no_grad(), evaluation.validating():
                res, _ = alg.model.forward((img,))
                return res['activated_pred'][0]
        for _ in range(args.warmup):
            engine()
        torch.cuda.synchronize()
        ops.reset_launch_count()
        ms, peak = _timed(engine, args.steps)
        launches = ops.launch_count() // args.steps
        for k in KERNELS:
            ops.kernel_timer_start(k)
        engine()
        kern = {k: ops.kernel_timer_stop(k, with_meta=True) for k in KERNELS}
        kms = sum(t for v in kern.values() for t, _ in v)
        kbytes = sum(m for v in kern.values() for _, m in v)
        r = {'ms_per_batch': ms, 'images_per_s': args.batch * 1000.0 / ms, 'peak_mem_gb': peak / 1e9,
             'launches_per_batch': launches,
             'protocol_kernels': {'ms': kms, 'bytes': kbytes,
                                  'tb_per_s': kbytes / (kms * 1e-3) / 1e12 if kms else None,
                                  'share_of_3_35_tb_s': kbytes / (kms * 1e-3) / HBM_BYTES_PER_S if kms else None,
                                  'calls': {k: len(v) for k, v in kern.items()}}}
        if not args.skip_oracle:
            protocol, crop, scales, flip = evaluation.settings(alg.args)

            def oracle():
                with torch.no_grad():
                    return E.evaluate(lambda t: plain(t)[0], img, protocol, crop, scales, flip)[0]
            oracle()
            torch.cuda.synchronize()
            oms, opeak = _timed(oracle, args.steps)
            with torch.no_grad():
                diff = float((engine() - oracle()).abs().max())
            r['oracle_loop'] = {'ms_per_batch': oms, 'images_per_s': args.batch * 1000.0 / oms,
                                'peak_mem_gb': opeak / 1e9, 'max_abs_diff_vs_engine': diff}
        results[name] = r
        del alg, plain
        torch.cuda.empty_cache()
    ops.set_conv_precision('fp32')
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--batch', type=int, default=1)
    ap.add_argument('--precision', default='f16x3')
    ap.add_argument('--skip-oracle', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval.py measures on a GPU; none is visible')
    info = card()
    out = {'bench': 'eval_views', 'card': info, 'shape': [args.batch, 3, 1024, 2048], 'classes': 19,
           'model': 'deeplabv3plus-r101-os16', 'precision': args.precision, 'steps': args.steps,
           'results': run(args)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
