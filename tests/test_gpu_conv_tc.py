"""wgmma convolution (csrc/conv_tc.cu) against the FFMA fp32 kernel and the torch-CPU oracle op.

precision 2 (3xTF32: hi/lo operand split, fp32 accumulation) must agree with fp32 to 5e-5 relative (the
tensor core's fp32 accumulator is not an IEEE round-to-nearest adder, so the error grows with K); precision 1
(single TF32 pass, what cuDNN does by default for the reference on GPU) to 2e-3.  The mbarrier watchdog must stay silent."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
CL = torch.channels_last


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    return _ops


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


# (pxl_conv_geom.precision, tolerance vs the FFMA kernel): 2 = 3xTF32 and 3 = fp16-pair x3 are fp32-grade,
# 1 = single TF32 and 4 = single fp16 carry 11-bit operands (what cuDNN gives the reference on a GPU)
PRECS = [(2, 5e-5), (1, 2e-3), (3, 5e-5), (4, 2e-3)]

CASES = [
    # N, Cin, H, W, Cout, k, dil
    (2, 64, 17, 19, 64, 1, 1),
    (1, 32, 8, 16, 32, 1, 1),         # exactly one 128-row tile
    (2, 256, 33, 33, 64, 1, 1),
    (2, 64, 33, 33, 256, 1, 1),
    (1, 1024, 9, 9, 256, 1, 1),
    (2, 64, 13, 13, 64, 3, 1),
    (2, 64, 33, 33, 64, 3, 1),
    (1, 128, 65, 65, 128, 3, 1),
    (2, 256, 33, 33, 256, 3, 1),
    (1, 512, 17, 17, 512, 3, 2),      # layer4 dilation 2
    (1, 512, 17, 17, 512, 3, 4),
    (1, 96, 20, 24, 160, 3, 1),       # Cin = 3 chunks, Cout not a power of two
    (2, 64, 129, 129, 64, 3, 1),      # layer1 conv2 shape (many tiles)
    (1, 2048, 17, 17, 512, 1, 1),     # layer4 conv1: the longest 1x1 reduction
    (2, 192, 21, 23, 320, 3, 1),      # 3 fp16 K chunks, Cout = 2.5 x 128
]


@pytest.mark.parametrize('precision,tol', PRECS)
@pytest.mark.parametrize('case', CASES)
def test_conv_tc_forward_and_dgrad(ops, case, precision, tol):
    N, Cin, H, W, Cout, k, dil = case
    g = torch.Generator().manual_seed(Cin + Cout + H)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda().contiguous(memory_format=CL)
    b = torch.randn(Cout, generator=g).cuda()
    pad = dil * (k // 2)
    outs = {}
    for prec in (0, precision):
        ops._conv_precision = prec
        xg = x.clone().requires_grad_(True)
        wg = w.clone().requires_grad_(True)
        y = ops.conv2d(xg, wg, b, 1, pad, dil)
        y.backward(torch.ones_like(y) * 0.5 + y.detach() * 0.1)
        outs[prec] = (y.detach(), xg.grad, wg.grad)
    ops._conv_precision = 0
    assert ops.conv_tc_status() == 0, 'mbarrier watchdog fired: role %d' % ops.conv_tc_status()
    assert ops.h16_status() == 0, 'an fp16 pair saturated' 
    ef, eb = rel(outs[precision][0], outs[0][0]), rel(outs[precision][1], outs[0][1])
    ew = rel(outs[precision][2], outs[0][2])
    print('case %s precision %d: fwd %.2e dgrad %.2e wgrad %.2e' % (case, precision, ef, eb, ew))
    assert ef <= tol and eb <= tol and ew <= tol, (ef, eb, ew)
    # and against torch CPU for one anchor per kernel size
    if (N, Cin, H) in ((2, 64, 17), (2, 64, 13)):
        yc = F.conv2d(x.cpu().contiguous(), w.cpu().contiguous(), b.cpu(), padding=pad, dilation=dil)
        assert rel(outs[precision][0].cpu(), yc) <= tol


@pytest.mark.parametrize('precision,tol', PRECS)
@pytest.mark.parametrize('case', [(2, 128, 33, 35, 128, 3), (2, 256, 17, 17, 512, 1), (1, 64, 65, 65, 64, 3),
                                  (2, 128, 32, 36, 128, 3), (1, 64, 64, 64, 128, 1)])      # even input sizes too
def test_conv_tc_stride2(ops, case, precision, tol):
    """stride-2 convolutions: forward and wgrad use the TMA traversal stride, dgrad is decomposed by
    output parity into four stride-1 launches."""
    N, Cin, H, W, Cout, k = case
    g = torch.Generator().manual_seed(H + Cout)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda().contiguous(memory_format=CL)
    res = {}
    for prec in (0, precision):
        ops._conv_precision = prec
        wg = w.clone().requires_grad_(True)
        xg = x.clone().requires_grad_(True)
        y = ops.conv2d(xg, wg, None, 2, k // 2, 1)
        y.backward(torch.ones_like(y) * 0.5 + y.detach() * 0.1)
        res[prec] = (y.detach(), xg.grad, wg.grad)
    ops._conv_precision = 0
    assert ops.conv_tc_status() == 0
    ef, eb, ew = (rel(res[precision][i], res[0][i]) for i in range(3))
    print('stride-2 case %s precision %d: fwd %.2e dgrad %.2e wgrad %.2e' % (case, precision, ef, eb, ew))
    assert ef <= tol and eb <= tol and ew <= tol, (ef, eb, ew)


@pytest.mark.parametrize('precision,tol', PRECS)
@pytest.mark.parametrize('case', [(2, 64, 65, 65, 128, 2), (3, 128, 33, 33, 128, 1), (2, 256, 17, 19, 512, 2), (2, 512, 9, 9, 512, 1),
                                  (3, 64, 64, 64, 128, 2), (3, 128, 32, 32, 128, 1), (3, 128, 31, 31, 256, 2), (3, 256, 14, 14, 512, 2),
                                  (3, 512, 7, 7, 512, 1)])        # the FlawDetector's sizes at 129x129 (even and odd)
def test_conv_tc_4x4_pad1(ops, case, precision, tol):
    """The 4x4 / padding 1 convolutions (stride 2 and 1, with bias) of the FlawDetector (ssl_gct.py:539-585) and the
    FC discriminator (ssl_adv.py:466-503): even kernel, so the stride-2 dgrad parity classes are asymmetric."""
    N, Cin, H, W, Cout, stride = case
    g = torch.Generator().manual_seed(H + Cout + stride)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = (torch.randn(Cout, Cin, 4, 4, generator=g) / (Cin * 16) ** 0.5).cuda().contiguous(memory_format=CL)
    b = torch.randn(Cout, generator=g).cuda()
    res = {}
    for prec in (0, precision):
        ops._conv_precision = prec
        wg, xg, bg = w.clone().requires_grad_(True), x.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = ops.conv2d(xg, wg, bg, stride, 1, 1)
        y.backward(torch.ones_like(y) * 0.5 + y.detach() * 0.1)
        res[prec] = (y.detach(), xg.grad, wg.grad, bg.grad)
    ops._conv_precision = 0
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    errs = [rel(res[precision][i], res[0][i]) for i in range(4)]
    print('4x4 case %s precision %d: fwd %.2e dgrad %.2e wgrad %.2e dbias %.2e' % ((case, precision) + tuple(errs)))
    assert max(errs) <= tol, errs
    xc, wc = x.cpu().contiguous().requires_grad_(True), w.cpu().contiguous()
    yc = F.conv2d(xc, wc, b.cpu(), stride=stride, padding=1)
    (yc * (0.5 + 0.1 * yc.detach())).sum().backward()
    assert rel(res[precision][0].cpu(), yc) <= tol and rel(res[precision][1].cpu(), xc.grad) <= tol


@pytest.mark.parametrize('precision,tol', PRECS)
def test_aspp_head_tc(ops, precision, tol):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 2048, 33, 33, generator=g).cuda().contiguous(memory_format=CL)
    ws = [(torch.randn(21, 2048, 3, 3, generator=g) * 0.01).cuda().contiguous(memory_format=CL) for _ in range(4)]
    bs = [(torch.randn(21, generator=g) * 0.1).cuda() for _ in range(4)]
    res = {}
    for prec in (0, precision):
        ops._conv_precision = prec
        xg = x.clone().requires_grad_(True)
        wl = [t.clone().requires_grad_(True) for t in ws]
        y = ops.aspp(xg, wl, bs)
        gy = torch.zeros_like(y)
        gy[:, :21] = 0.3 + 0.1 * y.detach()[:, :21]
        y.backward(gy)
        res[prec] = (y.detach(), xg.grad, torch.stack([t.grad for t in wl]))
    ops._conv_precision = 0
    assert ops.conv_tc_status() == 0
    atol = max(tol, 1e-4)        # K = 36 taps x 2048 = 73,728: the longest reduction on the path
    assert rel(res[precision][0][:, :21], res[0][0][:, :21]) <= atol
    assert float(res[precision][0][:, 21:].abs().max()) == 0.0
    assert rel(res[precision][1], res[0][1]) <= tol
    assert rel(res[precision][2], res[0][2]) <= tol


def test_h16_pair_split_is_exact_to_22_bits(ops):
    """x * s == hi + lo to 2^-22 relative (or 2^-25 absolute in scaled units); dynamic scale puts absmax in (2^13, 2^14]."""
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(1 << 16, generator=g) * torch.logspace(-6, 2, 1 << 16)).cuda()
    h = ops.h16_split(x, 16.0)
    rec = (h.hi.double() + h.lo.double()) / 16.0
    err = (rec - x.double()).abs()
    bound = torch.maximum(x.double().abs() * 2.0 ** -21, torch.full_like(err, 2.0 ** -24 / 16.0))
    assert bool((err <= bound).all()), float((err / bound).max())
    gsmall = x * 1e-9
    hd = ops.h16_split(gsmall, None)
    s, inv = float(hd.slot[0]), float(hd.slot[1])
    assert s * inv == 1.0 and 2.0 ** 13 < float(gsmall.abs().max()) * s <= 2.0 ** 14
    rec = (hd.hi.double() + hd.lo.double()) * inv
    err = (rec - gsmall.double()).abs()
    assert float(err.max()) <= float(gsmall.abs().max()) * 2.0 ** -21
    assert ops.h16_status() == 0
    big = torch.full((64,), 1e6).cuda()
    ops.h16_split(big, 16.0)
    assert ops.h16_status() > 0                      # saturation is counted, not silent
    ops._lib.load().pxl_h16_reset_status()


def test_tf32_operand_rounding_probe(ops):
    """Documents what tf32 wgmma does with the low 13 mantissa bits of raw fp32 operands."""
    x = torch.full((1, 32, 8, 16), 1.0 + 2.0 ** -11 + 2.0 ** -12).cuda().contiguous(memory_format=CL)   # low bits set
    w = torch.zeros(32, 32, 1, 1).cuda().contiguous(memory_format=CL)
    w[0, 0] = 1.0
    ops._conv_precision = 1
    y = ops.conv2d(x, w, None, 1, 0, 1)
    ops._conv_precision = 0
    v = float(y[0, 0, 0, 0])
    print('tf32 probe: 1 + 2^-11 + 2^-12 ->', v, '(truncation gives 1.0, round-to-nearest gives 1 + 2^-10)')
    assert v in (1.0, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -11 + 2.0 ** -12)


@pytest.mark.parametrize('precision', [1, 2, 3, 4])
@pytest.mark.parametrize('shape', [(2, 64, 33, 33, 256, 1), (2, 128, 17, 19, 64, 3), (1, 64, 129, 129, 64, 3),
                                   (4, 256, 40, 40, 512, 1), (16, 256, 33, 33, 256, 3)])
def test_bn_statistics_fused_in_epilogue(ops, shape, precision):
    """The conv epilogue's per-channel sum / sum-of-squares equal those of the tensor it stored."""
    N, Cin, H, W, Cout, k = shape
    g = torch.Generator().manual_seed(Cout + H)
    x = torch.randn(N, Cin, H, W, generator=g).cuda().contiguous(memory_format=CL)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).cuda().contiguous(memory_format=CL)
    ops._conv_precision = precision
    y = ops.conv2d(x, w, None, 1, k // 2, 1, want_bn_stats=True)
    ops._conv_precision = 0
    sums = getattr(y, '_pxl_bn_sums', None)
    assert sums is not None and ops.conv_tc_status() == 0
    yd = y.double()
    ref = torch.cat((yd.sum(dim=(0, 2, 3)), (yd * yd).sum(dim=(0, 2, 3))))
    assert rel(sums, ref) <= 1e-5
    # and bn_act consumes them: identical output with and without the fused statistics
    gm, bt = torch.ones(Cout).cuda(), torch.zeros(Cout).cuda()
    a = ops.bn_act(y, gm, bt, torch.zeros(Cout).cuda(), torch.ones(Cout).cuda(), training=True, relu=True)
    y2 = y.clone(memory_format=torch.preserve_format)
    b = ops.bn_act(y2, gm, bt, torch.zeros(Cout).cuda(), torch.ones(Cout).cuda(), training=True, relu=True)
    assert rel(a, b) <= 1e-5


@pytest.mark.parametrize('precision,tol_y,tol_w', [('tf32x3', 2e-5, 5e-5), ('tf32', 3e-3, 3e-3), ('f16x3', 2e-5, 5e-5), ('f16', 3e-3, 3e-3)])
@pytest.mark.parametrize('N,H,W', [(2, 65, 65), (1, 97, 129), (2, 40, 36)])
def test_stem_tensor_core_path(ops, N, H, W, precision, tol_y, tol_w):
    """7x7/2 stem as im2col (pxl_stem_im2col) + flat 1x1 wgmma convolution, forward, weight gradient and the
    fused BatchNorm sums, against torch CPU fp32 (resnet.py:69,121)."""
    gs = torch.Generator().manual_seed(H * 7 + W)
    img = torch.randn(N, 3, H, W, generator=gs)
    w = torch.randn(64, 3, 7, 7, generator=gs) * 0.1
    wc = w.clone().requires_grad_(True)
    yc = F.conv2d(img, wc, stride=2, padding=3)
    wt = torch.randn(yc.shape, generator=gs)
    (yc * wt).sum().backward()
    ops.set_conv_precision(precision)
    try:
        wg = w.cuda().contiguous(memory_format=CL).requires_grad_(True)
        yg = ops.stem_conv(img.cuda(), wg, want_bn_stats=True)
        (yg * wt.cuda()).sum().backward()
        sums = yg._pxl_bn_sums.cpu()
    finally:
        ops.set_conv_precision('fp32')
    assert rel(yg.cpu(), yc) <= tol_y
    assert rel(wg.grad.cpu(), wc.grad) <= tol_w
    ref = torch.cat((yc.double().sum(dim=(0, 2, 3)), (yc.double() ** 2).sum(dim=(0, 2, 3))))
    assert rel(sums, ref) <= max(tol_y * 10, 1e-4)
    assert ops.conv_tc_status() == 0
