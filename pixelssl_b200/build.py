"""Builds libpixelssl_b200.so (sm_90a only) in-tree with nvcc.  No torch headers involved: the
library is a plain C-ABI shared object (include/pixelssl_b200.h)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libpixelssl_b200.so')
SOURCES = ['loss_kernels.cu', 'norm_pool_optim.cu', 'resample.cu', 'conv_fp32.cu', 'conv_tc.cu',
           'h16_prep.cu', 'conv_api.cu', 'gct_kernels.cu', 'metrics_noise.cu', 'peer_exchange.cu', 'input_pipeline.cu', 'aspp_gather.cu', 's4l_kernels.cu',
           'lane_concat.cu', 'strong_aug.cu', 'ohem.cu', 'eval_views.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
              '-Xcompiler', '-fPIC', '--use_fast_math=false']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return 'nvcc'


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + \
           [os.path.join(os.path.dirname(HERE), 'include', 'pixelssl_b200.h'), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=True):
    os.makedirs(LIBDIR, exist_ok=True)
    if not force and not needs_build():
        return LIB
    objs = []
    flags = [f for f in NVCC_FLAGS if not f.startswith('--use_fast_math')]
    procs = []
    for src in SOURCES:
        path = os.path.join(CSRC, src)
        if not os.path.exists(path):
            continue
        obj = os.path.join(LIBDIR, src.replace('.cu', '.o'))
        objs.append(obj)
        cmd = [_nvcc()] + flags + ['-c', path, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (src, out.decode()))
        if verbose and out.strip():
            print(out.decode())
    cmd = [_nvcc(), '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv))
