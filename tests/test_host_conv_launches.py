"""Every library call of the convolution nodes, forward and backward, in the order they are issued, in every precision
mode (CPU only: the calls are recorded, not made): nn.modules.Conv2d over strides, dilations, a zero-padded output and
a 21-channel input, with and without a parameter arena (whose arena-wide transposed, tf32-split and fp16-pair weights
the launches then read), with and without the input gradient and the conv-epilogue BatchNorm sums; the ASPP head on
its tap and GEMM paths; the stride-2 stem in both kernel sizes.  Arguments print as tools/launch_trace.py prints them.
Also checks which outputs carry ``_pxl_bn_sums`` and which weights got their gradient in place.  The expected calls
(tests/golden/conv_launches.json) were recorded from the previous version of the convolution nodes."""
import itertools
import json
import os

import pytest
import torch

from pixelssl_b200 import ops
from pixelssl_b200.nn import ParamArena
from pixelssl_b200.nn.modules import Conv2d
from tools.launch_trace import fmt

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'conv_launches.json')
PRECISIONS = list(ops.PRECISION)

# name -> (Cin, Cout, kernel, stride, dilation, bias, out_lanes); padding keeps the size at stride 1
CONVS = {
    'c64-64-k3': (64, 64, 3, 1, 1, False, 0),
    'c96-128-k3s2': (96, 128, 3, 2, 1, False, 0),
    'c128-64-k3d2': (128, 64, 3, 1, 2, False, 0),
    'c64-21-k1-bias-lanes32': (64, 21, 1, 1, 1, True, 32),
    'c21-64-k3-bias': (21, 64, 3, 1, 1, True, 0),
}
CONV_CASES = list(itertools.product(CONVS, PRECISIONS, (False, True), (False, True), (False, True)))


def conv_id(name, precision, arena, dx, bn):
    return '%s-%s-arena%d-dx%d-bn%d' % (name, precision, arena, dx, bn)


def _record(monkeypatch, precision):
    rec = []
    monkeypatch.setattr(ops, 'call', lambda name, *args: rec.append(fmt(name, args)) or 0)
    monkeypatch.setattr(ops, '_stream', lambda: 0)
    monkeypatch.setattr(ops, '_chk', lambda *a, **k: None)
    monkeypatch.setattr(ops, '_conv_precision', ops.PRECISION[precision])
    ops.new_step()
    return rec


def _grad_seen(t):
    """A list that gets an entry when autograd hands ``t`` a gradient (not when a kernel added it into t.grad)."""
    seen = []
    t.register_hook(lambda g: seen.append(1) if g is not None else None)
    return seen


def _cl(*shape, grad=False):
    return torch.zeros(shape).contiguous(memory_format=ops.CL).requires_grad_(grad)


def run_conv(monkeypatch, name, precision, arena, dx, bn):
    cin, cout, k, stride, dil, bias, lanes = CONVS[name]
    rec = _record(monkeypatch, precision)
    conv = Conv2d(cin, cout, k, stride=stride, padding=dil * (k // 2), dilation=dil, bias=bias, out_lanes=lanes)
    conv.feeds_bn = bn
    keep = ParamArena(conv) if arena else None
    seen = _grad_seen(conv.weight)
    out = conv(_cl(2, cin, 6, 6, grad=dx))
    sums = hasattr(out, '_pxl_bn_sums')
    out.backward(torch.ones_like(out))
    del keep
    return {'calls': rec, 'bn_sums': sums, 'weight_grad_in_place': not seen}


def run_aspp(monkeypatch, precision, dx):
    rec = _record(monkeypatch, precision)
    weights = [_cl(21, 2048, 3, 3, grad=True) for _ in range(4)]
    biases = [torch.zeros(21, requires_grad=True) for _ in range(4)]
    seen = [_grad_seen(w) for w in weights]
    out = ops.aspp(_cl(1, 2048, 4, 4, grad=dx), weights, biases)
    out.backward(torch.ones_like(out))
    return {'calls': rec, 'weight_grad_in_place': [not s for s in seen]}


def run_stem(monkeypatch, precision, ks, bn):
    rec = _record(monkeypatch, precision)
    weight = _cl(64, 3, ks, ks, grad=True)
    seen = _grad_seen(weight)
    out = ops.stem_conv(torch.zeros(1, 3, 9, 9), weight, want_bn_stats=bn)
    sums = hasattr(out, '_pxl_bn_sums')
    out.backward(torch.ones_like(out))
    return {'calls': rec, 'bn_sums': sums, 'weight_grad_in_place': not seen}


@pytest.fixture(scope='module')
def expected():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize('name,precision,arena,dx,bn', CONV_CASES, ids=[conv_id(*c) for c in CONV_CASES])
def test_conv2d(monkeypatch, expected, name, precision, arena, dx, bn):
    assert run_conv(monkeypatch, name, precision, arena, dx, bn) == expected['conv2d-' + conv_id(name, precision, arena, dx, bn)]


@pytest.mark.parametrize('dx', [False, True])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_aspp(monkeypatch, expected, precision, dx):
    """2048 -> 21: the 36-tap convolution below the fp16 modes, the fp16-pair GEMM + gather in them."""
    assert run_aspp(monkeypatch, precision, dx) == expected['aspp-%s-dx%d' % (precision, dx)]


@pytest.mark.parametrize('bn', [False, True])
@pytest.mark.parametrize('ks', [7, 3])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_stem_conv(monkeypatch, expected, precision, ks, bn):
    assert run_stem(monkeypatch, precision, ks, bn) == expected['stem-%s-k%d-bn%d' % (precision, ks, bn)]
