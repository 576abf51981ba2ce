"""GPU parity of every C-ABI kernel against the CPU oracle (oracle/sseg_oracle.py restates the
reference call sites with torch CPU fp32 ops) and the reference-generated goldens.

Tolerances (north_star: 1e-3 relative fp32; bit-exact for CutMix mask/mix):
  rel(a, b) = max|a - b| / max|b|   must be <= the value written next to each check."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sseg_oracle as O

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')
CL = torch.channels_last


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    _ops.set_conv_precision('fp32')
    return _ops


def rel(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def cuda(t):
    return t.detach().clone().cuda()


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------------------------

def test_mse_golden(ops):
    g = np.load(os.path.join(G, 'ops.npz'))
    s = torch.tensor(g['mse_s']).cuda().requires_grad_(True)
    t = torch.tensor(g['mse_t']).cuda()
    loss = ops.mse_consistency(s, t, loss_scale=float(g['mse_grad_scale']), unit_upstream=True)
    loss.backward()
    assert abs(float(loss) / float(g['mse_grad_scale']) - float(g['mse_loss'])) <= 1e-6 * float(g['mse_loss'])
    assert rel(s.grad, torch.tensor(g['mse_grad'])) <= 1e-6


@pytest.mark.parametrize('n,off', [(1, 0), (3, 1), (1023, 0), (1024 * 7 + 5, 3), (2 * 21 * 129 * 129, 0),
                                   (4 * 21 * 257 * 257 + 1, 2)])
def test_mse_sizes_and_alignment(ops, n, off):
    gs = gen(n)
    base_s = torch.randn(n + 8, generator=gs)
    base_t = torch.randn(n + 8, generator=gs)
    s_c, t_c = base_s[off:off + n], base_t[off:off + n]
    s = base_s.cuda()[off:off + n].requires_grad_(True)
    t = base_t.cuda()[off:off + n]
    # general (device upstream) path and fused path
    loss = ops.mse_consistency(s, t, loss_scale=0.5, unit_upstream=False)
    (loss * 3.0).backward()
    sc = s_c.clone().requires_grad_(True)
    ref = 0.5 * O.mse_consistency(sc, t_c)
    (ref * 3.0).backward()
    assert abs(float(loss) - float(ref)) <= 2e-6 * abs(float(ref))
    assert rel(s.grad, sc.grad) <= 2e-6
    l2, g2 = ops.mse_consistency_raw(s.detach(), t, 0.5, want_grad=True)
    assert abs(float(l2) - float(ref)) <= 2e-6 * abs(float(ref))
    assert rel(g2 * 3.0, sc.grad) <= 2e-6
    # misaligned student vs aligned teacher -> scalar path
    if n > 16:
        l3, _ = ops.mse_consistency_raw(s.detach(), t.clone(), 0.5, want_grad=False)
        assert abs(float(l3) - float(ref)) <= 2e-6 * abs(float(ref))
    # determinism: identical bits on a second launch
    l4, g4 = ops.mse_consistency_raw(s.detach(), t, 0.5, want_grad=True)
    assert float(l4) == float(l2) and torch.equal(g4, g2)


def test_ce_golden(ops):
    g = np.load(os.path.join(G, 'ops.npz'))
    logits = torch.tensor(g['ce_logits']).cuda().requires_grad_(True)
    lab = torch.tensor(g['ce_labels']).cuda()
    per = ops.cross_entropy2d(logits, lab, 255)
    per.mean().backward()
    assert rel(per, torch.tensor(g['ce_loss'])) <= 1e-5
    assert rel(logits.grad, torch.tensor(g['ce_grad'])) <= 1e-5
    # fused-gradient variant (upstream known on the host)
    l2 = torch.tensor(g['ce_logits']).cuda().requires_grad_(True)
    per2 = ops.cross_entropy2d(l2, lab, 255, upstream_const=1.0 / per.numel())
    per2.mean().backward()
    assert rel(per2, per) <= 1e-6 and rel(l2.grad, torch.tensor(g["ce_grad"])) <= 1e-5   # fp32 atomics: order-dependent last bit


@pytest.mark.parametrize('n,c,h,w', [(1, 21, 1, 1), (2, 21, 65, 65), (2, 2, 31, 17), (1, 32, 40, 40)])
def test_ce_shapes_all_ignored_and_unlabeled(ops, n, c, h, w):
    gs = gen(5)
    logits = torch.randn(n, c, h, w, generator=gs) * 5
    lab = torch.randint(0, c, (n, 1, h, w), generator=gs).float()
    lab[0, 0, 0, :] = 255.0
    if n > 1:
        lab[1] = 255.0           # a fully ignored sample -> loss 0, grad 0
    lc = logits.clone().requires_grad_(True)
    ref = O.sseg_criterion(lc, lab, 255)
    ref.sum().backward()
    lg = logits.cuda().requires_grad_(True)
    per = ops.cross_entropy2d(lg, lab.cuda(), 255)
    per.sum().backward()
    assert rel(per, ref) <= 1e-5
    assert rel(lg.grad, lc.grad) <= 1e-5


def test_softmax_fwd_bwd_and_fused_mse(ops):
    gs = gen(9)
    x = torch.randn(3, 21, 37, 29, generator=gs) * 4
    tp = torch.softmax(torch.randn(3, 21, 37, 29, generator=gs), 1)
    xc = x.clone().requires_grad_(True)
    pc = O.channel_softmax(xc)
    w = torch.randn(3, 21, 37, 29, generator=gs)
    (pc * w).sum().backward()
    xg = x.cuda().requires_grad_(True)
    pg = ops.softmax_planar(xg)
    (pg * w.cuda()).sum().backward()
    assert rel(pg, pc) <= 1e-6 and rel(xg.grad, xc.grad) <= 1e-5
    xc2 = x.clone().requires_grad_(True)
    ref = 20.0 * F.mse_loss(O.channel_softmax(xc2), tp)
    (ref * 0.7).backward()
    xg2 = x.cuda().requires_grad_(True)
    loss = ops.softmax_mse(xg2, tp.cuda(), 20.0)
    (loss * 0.7).backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert rel(xg2.grad, xc2.grad) <= 1e-5


def test_cutmix_bit_exact(ops):
    g = np.load(os.path.join(G, 'ops.npz'))
    mixed = ops.cutmix_mix(torch.tensor(g['cutmix_masks']).cuda(), torch.tensor(g['cutmix_a']).cuda(),
                           torch.tensor(g['cutmix_b']).cuda()).cpu().numpy()
    ref = g['cutmix_mixed']
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(mixed), nan)
    assert np.array_equal(mixed.view(np.uint32)[~nan], ref.view(np.uint32)[~nan])
    conf = ops.cutmix_confidence(torch.tensor(g['conf_prob']).cuda(), 0.97)
    assert float(conf) == float(g['conf_value'])
    # full-size property: mask in {0,1} -> output is exactly a or b element-wise
    rng = np.random.RandomState(3)
    masks, _ = O.box_masks(rng, 2, (513, 513))
    a = torch.randn(2, 3, 513, 513, generator=gen(1)).cuda()
    b = torch.randn(2, 3, 513, 513, generator=gen(2)).cuda()
    m = torch.tensor(masks).cuda()
    out = ops.cutmix_mix(m, a, b)
    assert torch.equal(out, torch.where(m.bool().expand_as(a), a, b))
    assert torch.equal(out, m * a + (1 - m) * b)


# ---------------------------------------------------------------------------------------------
# bilinear
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('h,w,H,W,ac', [(33, 33, 513, 513, True), (9, 9, 129, 129, True), (5, 7, 97, 65, True),
                                        (33, 33, 65, 65, False), (20, 20, 39, 39, False), (1, 1, 8, 8, True),
                                        (6, 6, 45, 45, False), (45, 45, 90, 90, True),
                                        (65, 65, 33, 33, True), (40, 40, 17, 23, False), (3, 300, 7, 601, True),
                                        (17, 17, 17, 17, False), (2, 2, 64, 64, False)])
def test_bilinear_planar(ops, h, w, H, W, ac):
    gs = gen(h * 100 + H)
    x = torch.randn(2, 5, h, w, generator=gs)
    wt = torch.randn(2, 5, H, W, generator=gs)
    xc = x.clone().requires_grad_(True)
    yc = F.interpolate(xc, size=(H, W), mode='bilinear', align_corners=ac)
    (yc * wt).sum().backward()
    xg = x.cuda().requires_grad_(True)
    yg = ops.bilinear(xg, (H, W), align_corners=ac)
    (yg * wt.cuda()).sum().backward()
    assert rel(yg, yc) <= 2e-6
    assert rel(xg.grad, xc.grad) <= 2e-5


def test_bilinear_nhwc_padded_input(ops):
    gs = gen(77)
    x = torch.randn(2, 21, 33, 33, generator=gs)
    wt = torch.randn(2, 21, 257, 257, generator=gs)
    xc = x.clone().requires_grad_(True)
    yc = O.bilinear_align_corners(xc, (257, 257))
    (yc * wt).sum().backward()
    xp = torch.zeros(2, 32, 33, 33)
    xp[:, :21] = x
    xg = xp.cuda().contiguous(memory_format=CL).requires_grad_(True)
    yg = ops.bilinear(xg, (257, 257), align_corners=True, channels=21, nhwc=True)
    (yg * wt.cuda()).sum().backward()
    assert rel(yg, yc) <= 2e-6
    assert rel(xg.grad[:, :21], xc.grad) <= 2e-5
    assert float(xg.grad[:, 21:].abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------
# batch norm, max pool
# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize('N,C,H,W,relu,res', [(2, 64, 17, 19, True, False), (3, 256, 9, 9, True, True),
                                              (2, 2048, 5, 5, False, False), (1, 8, 33, 33, True, True),
                                              (4, 128, 1, 1, False, True)])
def test_bn_act_train(ops, N, C, H, W, relu, res):
    gs = gen(C + H)
    x = torch.randn(N, C, H, W, generator=gs) * 2 + 0.5
    r = torch.randn(N, C, H, W, generator=gs) if res else None
    gamma = 1 + 0.3 * torch.randn(C, generator=gs)
    beta = 0.2 * torch.randn(C, generator=gs)
    wt = torch.randn(N, C, H, W, generator=gs)
    st = {'bn.weight': gamma.clone().requires_grad_(True), 'bn.bias': beta.clone().requires_grad_(True),
          'bn.running_mean': torch.zeros(C), 'bn.running_var': torch.ones(C)}
    xc = x.clone().requires_grad_(True)
    rc = r.clone().requires_grad_(True) if res else None
    yc = O.batch_norm(xc, st, 'bn', True)
    if res:
        yc = yc + rc
    if relu:
        yc = F.relu(yc)
    (yc * wt).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    rg = r.cuda().contiguous(memory_format=CL).requires_grad_(True) if res else None
    gg, bg = gamma.cuda().requires_grad_(True), beta.cuda().requires_grad_(True)
    rm, rv = torch.zeros(C).cuda(), torch.ones(C).cuda()
    yg = ops.bn_act(xg, gg, bg, rm, rv, training=True, relu=relu, residual=rg)
    (yg * wt.cuda()).sum().backward()
    assert rel(yg, yc) <= 1e-5
    assert rel(rm, st['bn.running_mean']) <= 1e-5 and rel(rv, st['bn.running_var']) <= 1e-5
    assert rel(xg.grad, xc.grad) <= 2e-4
    assert rel(gg.grad, st['bn.weight'].grad) <= 1e-4 and rel(bg.grad, st['bn.bias'].grad) <= 1e-4
    if res:
        assert rel(rg.grad, rc.grad) <= 1e-6

@pytest.mark.parametrize('rows,C', [(1000, 64), (33 * 33 * 2, 256), (77, 2048)])
def test_bn_relu_byte_mask_equals_the_fp32_result_mask(ops, rows, C):
    """Block outputs record sign bits (1 byte per 4 values) in the forward apply; the backward launches that read
    them must produce bit-identical sums, dX pair and residual gradient to the launches that re-read the fp32 result."""
    from pixelssl_b200._lib import call
    P = ops._p
    g = gen(rows + C)
    dev = 'cuda'
    x = (torch.randn(rows, C, generator=g) * 2).to(dev)
    res = torch.randn(rows, C, generator=g).to(dev)
    dy = (torch.randn(rows, C, generator=g) * 1e-3).to(dev)
    gamma = (1 + 0.3 * torch.randn(C, generator=g)).to(dev)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev)
    sums = torch.cat((x.double().sum(0), (x.double() ** 2).sum(0)))
    coeff = torch.empty(4, C, device=dev)
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    y = torch.empty_like(x)
    pair = torch.empty(2, rows * C, dtype=torch.float16, device=dev)
    mask = torch.zeros(rows * C // 4, dtype=torch.uint8, device=dev)
    st = ops._stream()
    call('pxl_bn_finalize_apply', P(x), P(sums), float(rows), P(gamma), P(beta), P(rm), P(rv), 0.1, 1e-5, 0,
         P(coeff[0]), P(coeff[1]), P(coeff[2]), P(coeff[3]), P(res), 1, P(y), rows, C, P(pair[0]), P(pair[1]), 16.0, P(mask), st)
    bits = (y.view(-1, 4) > 0).to(torch.uint8)
    want = bits[:, 0] | (bits[:, 1] << 1) | (bits[:, 2] << 2) | (bits[:, 3] << 3)
    assert torch.equal(mask, want)
    outs = []
    ds_ref = None
    for use_mask in (False, True):
        dsums = torch.zeros(2 * C, dtype=torch.float64, device=dev)
        slot = torch.zeros(4, device=dev)
        call('pxl_bn_bwd_reduce', P(x), P(None if use_mask else y), P(dy), P(coeff[0]), P(coeff[1]), 1, rows, C, P(dsums),
             P(coeff[2]), P(coeff[3]), P(slot), P(mask if use_mask else None), st)
        if ds_ref is None:
            ds_ref = dsums.clone()
        # the fp64 atomics of the reduction commute only up to rounding: same sums to 1e-12, and the dx launches of
        # both variants then get the SAME sums so that their outputs can be compared bit for bit
        assert rel(dsums, ds_ref) <= 1e-12
        dpair = torch.empty(2, rows * C, dtype=torch.float16, device=dev)
        dres = torch.empty_like(x)
        dx = torch.empty_like(x)
        call('pxl_bn_bwd_dx', P(x), P(None if use_mask else y), P(dy), P(coeff[0]), P(coeff[1]), P(gamma), P(ds_ref), float(rows), 1,
             P(dx), P(dres), rows, C, P(coeff[2]), P(coeff[3]), P(None), P(None), P(dpair[0]), P(dpair[1]), P(slot), 12,
             P(mask if use_mask else None), st)
        torch.cuda.synchronize()
        outs.append((dx, dres, dpair, slot))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert ops.h16_status() == 0


def test_bn_eval(ops):
    gs = gen(4)
    C = 64
    x = torch.randn(2, C, 7, 7, generator=gs)
    st = {'bn.weight': torch.rand(C, generator=gs) + 0.5, 'bn.bias': torch.randn(C, generator=gs),
          'bn.running_mean': torch.randn(C, generator=gs), 'bn.running_var': torch.rand(C, generator=gs) + 0.5}
    yc = F.relu(O.batch_norm(x, st, 'bn', False))
    yg = ops.bn_act(x.cuda().contiguous(memory_format=CL), st['bn.weight'].cuda(), st['bn.bias'].cuda(),
                    st['bn.running_mean'].cuda(), st['bn.running_var'].cuda(), training=False, relu=True)
    assert rel(yg, yc) <= 1e-5


def test_maxpool_with_ties(ops):
    gs = gen(6)
    x = F.relu(torch.randn(2, 64, 33, 35, generator=gs))      # many exact-zero ties
    wt = torch.randn(2, 64, 17, 18, generator=gs)
    xc = x.clone().requires_grad_(True)
    yc = F.max_pool2d(xc, 3, 2, 1)
    (yc * wt).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    yg = ops.maxpool3x3s2(xg)
    (yg * wt.cuda()).sum().backward()
    assert torch.equal(yg.cpu(), yc.detach())
    assert rel(xg.grad, xc.grad) <= 1e-6


# ---------------------------------------------------------------------------------------------
# convolutions
# ---------------------------------------------------------------------------------------------

CONV_CASES = [
    # N, Cin, H, W, Cout, k, stride, pad, dil, bias
    (2, 64, 17, 19, 64, 1, 1, 0, 1, False),
    (2, 64, 17, 19, 256, 1, 1, 0, 1, False),
    (2, 64, 13, 13, 64, 3, 1, 1, 1, False),
    (1, 128, 21, 23, 128, 3, 2, 1, 1, False),     # layer2.0.conv2
    (2, 256, 17, 17, 512, 1, 2, 0, 1, False),     # downsample
    (2, 32, 11, 11, 48, 3, 1, 2, 2, False),       # dilation 2
    (1, 16, 15, 15, 16, 3, 1, 4, 4, True),        # dilation 4 + bias
    (2, 21, 9, 9, 84, 1, 1, 0, 1, True),          # Cin % 16 != 0 (generic gather path)
    (2, 24, 18, 18, 64, 4, 2, 1, 1, True),        # FlawDetector-like 4x4 / 2
    (1, 512, 9, 9, 21, 1, 1, 0, 1, False),        # skinny N
]


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv2d_fwd_dgrad_wgrad(ops, case):
    N, Cin, H, W, Cout, k, stride, pad, dil, has_bias = case
    gs = gen(Cin * 7 + Cout + k)
    x = torch.randn(N, Cin, H, W, generator=gs)
    w = torch.randn(Cout, Cin, k, k, generator=gs) / (Cin * k * k) ** 0.5
    b = torch.randn(Cout, generator=gs) if has_bias else None
    xc, wc = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    bc = b.clone().requires_grad_(True) if has_bias else None
    yc = F.conv2d(xc, wc, bc, stride=stride, padding=pad, dilation=dil)
    wt = torch.randn(yc.shape, generator=gs)
    (yc * wt).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    wg = w.cuda().contiguous(memory_format=CL).requires_grad_(True)
    bg = b.cuda().requires_grad_(True) if has_bias else None
    yg = ops.conv2d(xg, wg, bg, stride=stride, padding=pad, dilation=dil)
    assert tuple(yg.shape) == tuple(yc.shape)
    (yg * wt.cuda()).sum().backward()
    assert rel(yg, yc) <= 1e-5
    assert rel(xg.grad, xc.grad) <= 1e-5
    assert rel(wg.grad, wc.grad) <= 1e-4
    if has_bias:
        assert rel(bg.grad, bc.grad) <= 1e-5


@pytest.mark.parametrize('N,hw', [(2, 33), (1, 9), (2, 45)])
def test_aspp_head(ops, N, hw):
    gs = gen(hw)
    Cin, C = 2048, 21
    x = torch.randn(N, Cin, hw, hw, generator=gs)
    st = {}
    for i in range(4):
        st['classifier.conv2d_list.%d.weight' % i] = (torch.randn(C, Cin, 3, 3, generator=gs) * 0.01).requires_grad_(True)
        st['classifier.conv2d_list.%d.bias' % i] = (torch.randn(C, generator=gs) * 0.1).requires_grad_(True)
    xc = x.clone().requires_grad_(True)
    yc = O.aspp_classifier(xc, st)
    wt = torch.randn(yc.shape, generator=gs)
    (yc * wt).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    ws = [st['classifier.conv2d_list.%d.weight' % i].detach().cuda().contiguous(memory_format=CL).requires_grad_(True) for i in range(4)]
    bs = [st['classifier.conv2d_list.%d.bias' % i].detach().cuda().requires_grad_(True) for i in range(4)]
    yg = ops.aspp(xg, ws, bs)
    assert yg.shape[1] == 32
    wpad = torch.zeros(N, 32, hw, hw)
    wpad[:, :C] = wt
    (yg * wpad.cuda()).sum().backward()
    assert rel(yg[:, :C], yc) <= 1e-5
    assert float(yg[:, C:].abs().max()) == 0.0
    assert rel(xg.grad, xc.grad) <= 1e-5
    for i in range(4):
        assert rel(ws[i].grad, st['classifier.conv2d_list.%d.weight' % i].grad) <= 1e-4
        assert rel(bs[i].grad, st['classifier.conv2d_list.%d.bias' % i].grad) <= 1e-5


@pytest.mark.parametrize('N,H,W', [(2, 65, 65), (1, 97, 129), (2, 40, 36)])
def test_stem(ops, N, H, W):
    gs = gen(H)
    img = torch.randn(N, 3, H, W, generator=gs)
    w = torch.randn(64, 3, 7, 7, generator=gs) * 0.1
    wc = w.clone().requires_grad_(True)
    yc = F.conv2d(img, wc, stride=2, padding=3)
    wt = torch.randn(yc.shape, generator=gs)
    (yc * wt).sum().backward()
    wg = w.cuda().contiguous(memory_format=CL).requires_grad_(True)
    yg = ops.stem_conv(img.cuda(), wg)
    (yg * wt.cuda()).sum().backward()
    assert rel(yg, yc) <= 1e-5
    assert rel(wg.grad, wc.grad) <= 1e-4


# ---------------------------------------------------------------------------------------------
# optimiser + EMA
# ---------------------------------------------------------------------------------------------

def test_sgd_ema_matches_torch_and_oracle(ops):
    gs = gen(12)
    n = 100003
    p = torch.randn(n, generator=gs)
    t = torch.randn(n, generator=gs)
    pc, tc = p.clone(), t.clone()
    bufc = torch.zeros(n)
    pg, tg, bufg = p.cuda(), t.cuda(), torch.zeros(n).cuda()
    for step in range(3):
        g = torch.randn(n, generator=gs)
        O.sgd_momentum_step([pc], [g], [bufc], [0.01], 0.9, 5e-4, first_step=(step == 0))
        d = O.ema_update([tc], [pc], 0.99, step)
        ops.sgd_ema_(pg, g.cuda(), bufg, tg, 0.01, 0.9, 5e-4, d, step == 0)
        assert rel(pg, pc) <= 1e-6 and rel(bufg, bufc) <= 1e-6 and rel(tg, tc) <= 1e-6
    # against torch.optim.SGD itself
    q = torch.nn.Parameter(p.clone())
    opt = torch.optim.SGD([q], lr=0.01, momentum=0.9, weight_decay=5e-4)
    q2, b2 = p.cuda(), torch.zeros(n).cuda()
    gs2 = gen(13)
    for step in range(2):
        g = torch.randn(n, generator=gs2)
        q.grad = g.clone()
        opt.step()
        ops.sgd_ema_(q2, g.cuda(), b2, None, 0.01, 0.9, 5e-4, 0.0, step == 0)
    assert rel(q2, q.data) <= 1e-6
    t2 = t.cuda()
    ops.ema_(t2, q2, 0.5)
    assert rel(t2, t * 0.5 + 0.5 * q.data) <= 1e-6
