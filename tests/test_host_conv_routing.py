"""Which convolution kernel family serves a shape, in every precision mode (CPU only: library calls are recorded, not
made).  The table below is the rule set of the wgmma kernels (csrc/conv_tc.cu): the fp16-pair kernels take channel
counts that are multiples of 64, the tf32 kernels multiples of 32, both only stride 1 and 2 forward and the dgrad of a
stride-2 convolution; everything else runs on the FFMA kernels.  Shapes the fp16 kernels do not cover fall back to the
tf32 kernels of the same grade."""
import itertools
import types

import pytest
import torch

from pixelssl_b200 import ops

PRECISIONS = ('fp32', 'tf32', 'tf32x3', 'f16x3', 'f16')
CHANNELS = (128, 96, 21)                      # multiple of 64, of 32 only, of neither
STRIDES = ((1, 1), (2, 1), (1, 2))            # (mul, div): stride 1, stride 2, dgrad of a stride-2 convolution
FAMILY = {'pxl_conv_h16_launch': 'h16', 'pxl_conv_tc_launch_ex': 'tc', 'pxl_conv_nhwc': 'ffma',
          'pxl_conv_wgrad_h16_launch': 'h16', 'pxl_conv_wgrad_tc_launch': 'tc', 'pxl_conv_wgrad_nhwc': 'ffma'}


def expected(direction, cin, cout, mul, div, prec):
    """-> (family, precision the launch runs at)."""
    if direction == 'wgrad':
        fits = lambda a: div == 1 and mul in (1, 2) and cin % a == 0 and cout % a == 0
    else:
        fits = lambda a: cin % a == 0 and (mul, div) in ((1, 1), (2, 1), (1, 2))
    if prec >= 3:
        if fits(64):
            return 'h16', prec
        prec = {3: 2, 4: 1}[prec]
    if prec and fits(32):
        return 'tc', prec
    return 'ffma', 0


CASES = list(itertools.product(('fwd', 'dgrad', 'wgrad'), CHANNELS, CHANNELS, STRIDES, PRECISIONS))


@pytest.mark.parametrize('direction,cin,cout,stride,precision', CASES)
def test_route_table(direction, cin, cout, stride, precision):
    prec = ops.PRECISION[precision]
    assert ops.conv_route(direction, cin, cout, stride[0], stride[1], prec) == expected(direction, cin, cout, *stride, prec)


@pytest.fixture
def recorded(monkeypatch):
    """Library calls as [(family, geom.precision)] of the convolution launches; nothing reaches the library."""
    launches = []

    def fake_call(name, *args):
        if name in FAMILY:
            launches.append((FAMILY[name], args[0]._obj.precision))
        return 0

    monkeypatch.setattr(ops, 'call', fake_call)
    monkeypatch.setattr(ops, '_stream', lambda: 0)
    return launches


@pytest.mark.parametrize('direction,cin,cout,stride,precision', [c for c in CASES if c[0] != 'dgrad'])
def test_launchers_follow_the_table(recorded, direction, cin, cout, stride, precision):
    """conv_raw (forward and dgrad launches) and conv_wgrad_raw pick the family and precision of the table."""
    prec = ops.PRECISION[precision]
    mul, div = stride
    N, H, W, taps = 1, 4, 4, ops._taps(3, 3, 1, 1)
    T = len(taps) // 2
    x = torch.zeros((N, cin, H, W)).contiguous(memory_format=ops.CL)
    dy = torch.zeros((N, cout, H, W)).contiguous(memory_format=ops.CL)
    w = torch.zeros((cout, T, cin))
    if direction == 'fwd':
        ops.conv_raw(x, w, None, taps, N, H, W, cin, H, W, cout, cout, mul, div, precision=prec)
        want = expected('fwd', cin, cout, mul, div, prec)
    else:
        ops.conv_wgrad_raw(x, dy, torch.zeros_like(w), taps, N, H, W, cin, H, W, cout, cout, mul, div, precision=prec)
        want = expected('wgrad', cin, cout, mul, div, prec)
    assert recorded and set(recorded) == {want}


@pytest.mark.parametrize('cin,cout,stride', list(itertools.product(CHANNELS, CHANNELS, (1, 2, 3))))
@pytest.mark.parametrize('precision', PRECISIONS)
def test_conv_bn_unit_and_aspp(monkeypatch, cin, cout, stride, precision):
    """conv -> BN runs as one fp16-pair node exactly when all three directions of the convolution run on the fp16
    kernels; the ASPP runs as one fp16 GEMM when its forward does."""
    prec = ops.PRECISION[precision]
    monkeypatch.setattr(ops, '_conv_precision', prec)
    conv = types.SimpleNamespace(in_channels=cin, out_channels=cout, stride=stride, bias=None, out_lanes=0)
    bn = types.SimpleNamespace(training=True)
    h16 = all(expected(d, a, b, m, v, prec)[0] == 'h16' for d, a, b, m, v in
              (('fwd', cin, cout, stride, 1), ('dgrad', cout, cin, 1, stride), ('wgrad', cin, cout, stride, 1)))
    assert ops.conv_bn_unit_ok(conv, bn) == h16
    assert not ops.conv_bn_unit_ok(types.SimpleNamespace(**dict(vars(conv), bias=object())), bn)
    assert not ops.conv_bn_unit_ok(conv, types.SimpleNamespace(training=False))

    chosen = []
    monkeypatch.setattr(ops._AsppGemm, 'apply', lambda *a: chosen.append('gemm'))
    monkeypatch.setattr(ops._Aspp, 'apply', lambda *a: chosen.append('taps'))
    ops.aspp(torch.zeros((1, cin, 4, 4)), [torch.zeros(21, cin, 3, 3)] * 4, [torch.zeros(21)] * 4)
    assert chosen == ['gemm' if expected('fwd', cin, 21, 1, 1, prec)[0] == 'h16' else 'taps']
