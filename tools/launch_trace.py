"""Every library call of one training step, one line each: two versions of the host code that issue the same launches
in the same order with the same arguments print the same text.

    python tools/launch_trace.py CONFIGS PRECISIONS [WARMUP]

CONFIGS: comma list of bench.CONFIGS names, or 'mt_v3plus' (Mean-Teacher with the DeepLabV3+ task model); PRECISIONS:
comma list of ops.PRECISION names.  Per pair: WARMUP (default 2) untraced steps, then one traced step.  Pointer arguments
print as null / ptr (addresses differ between runs), scalars by value, ConvGeom / ConvTcExt fields expanded, host arrays
of pointers as lists of null / ptr and other host arrays (taps, weight indices) by value."""
import ctypes
import logging
import os
import random
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import bench
from pixelssl_b200 import _lib, ops, runner

CONFIGS = dict(bench.CONFIGS, mt_v3plus=(lambda: dict(bench.mt_config(), models={'model': 'deeplabv3plus'}),) + bench.CONFIGS['mt'][1:])


def _ptr(a):
    if isinstance(a, ctypes.Array):
        return [_ptr(v) for v in a]
    if isinstance(a, ctypes.c_void_p):
        a = a.value
    return 'ptr' if a else 'null'


def fmt(name, args):
    args = [a._obj if type(a).__name__ == 'CArgObject' else a for a in args]     # ctypes.byref(struct)
    ntaps = next((a.ntaps for a in args if isinstance(a, _lib.ConvGeom)), 0)
    parts = []
    for a, t in zip(args, _lib.SIGNATURES[name][1]):
        if isinstance(a, ctypes.Structure):
            fields = []
            for f, ft in a._fields_:
                v = getattr(a, f)
                if ft is ctypes.c_void_p:
                    v = _ptr(v)
                elif f == 'widx_host':
                    v = list(v[:ntaps]) if v else 'null'
                fields.append('%s=%s' % (f, v))
            parts.append('{%s}' % ' '.join(fields))
        elif isinstance(a, ctypes.Array):
            parts.append(str(_ptr(a) if a._type_ is ctypes.c_void_p else list(a)))
        elif t is ctypes.c_void_p:
            parts.append(_ptr(a))
        else:
            parts.append(repr(a))
    return '%s(%s)' % (name, ', '.join(parts))


def trace(config, precision, warmup):
    make_cfg, lbs, ubs, size, _ = CONFIGS[config]
    ops.set_conv_precision(precision)
    torch.manual_seed(0); random.seed(0); np.random.seed(0)
    alg = runner.build_algorithm(runner.build_args(make_cfg(), iters_per_epoch=662))
    img, lab = bench.synthetic_host_batches(1, 0, False, lbs, ubs, size)[0]
    batch = [((img.cuda(),), (lab.cuda(),))]
    for i in range(warmup):
        alg._train(batch, i)
    torch.cuda.synchronize()
    lines, orig = [], _lib.call

    def spy(name, *args):
        lines.append(fmt(name, args))
        return orig(name, *args)

    patched = [m for m in list(sys.modules.values()) if getattr(m, 'call', None) is orig]     # every `from _lib import call`
    for m in patched:
        m.call = spy
    try:
        alg._train(batch, warmup)
        torch.cuda.synchronize()
    finally:
        for m in patched:
            m.call = orig
    del alg
    torch.cuda.empty_cache()
    return lines


if __name__ == '__main__':
    logging.getLogger('PixelSSL').setLevel(logging.ERROR)
    warmup = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    for config in sys.argv[1].split(','):
        for precision in sys.argv[2].split(','):
            lines = trace(config, precision, warmup)
            print('== %s %s: %d calls' % (config, precision, len(lines)))
            print('\n'.join(lines), flush=True)
