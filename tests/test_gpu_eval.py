"""Multi-view evaluation on the engine: the four protocol kernels against torch (fp64; the resizes against fp32
F.interpolate, whose source-index arithmetic they share), the driver against the oracle
(oracle/eval_oracle.py) around a stub network, around the engine's own network and against the CPU fp64 oracle
networks, every algorithm validating with the protocol, no change to default validation or to training, and the
launches and synchronisations per batch."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import deeplabv3plus_oracle as D
from oracle import eval_oracle as E
from oracle import sseg_oracle as O

from conftest import TEST_PRECISIONS

pytestmark = pytest.mark.gpu
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000}
PROTO = {'val_protocol': 'sliding', 'val_crop_size': 45, 'val_scales': [0.75, 1.0, 1.25], 'val_flip': True}


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    return ops


@pytest.fixture(scope='module', params=TEST_PRECISIONS)
def ops(request, eng):
    eng.set_conv_precision(request.param)
    yield eng
    eng.set_conv_precision('fp32')


@pytest.fixture(autouse=True)
def _no_fp16_pair_saturation(eng):
    """The fp16-pair saturation count is process-wide and sticky: a test here that saturates fails here, instead of
    leaving the count for a later test to find."""
    before = eng.h16_status()
    yield
    torch.cuda.synchronize()
    assert eng.h16_status() == before, 'an fp16 pair saturated in this test: %s' % (eng.h16_status_sites(),)


@contextlib.contextmanager
def _precision(eng, name):
    """Run a block in one convolution precision mode and restore the mode the module's fixture set."""
    before = {v: k for k, v in eng.PRECISION.items()}[eng.get_conv_precision()]
    eng.set_conv_precision(name)
    try:
        yield
    finally:
        eng.set_conv_precision(before)


def _ev():
    from pixelssl_b200.task.sseg import evaluation
    return evaluation


def _absmax(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max())


# ---- kernels ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('s', [1.0, 0.5, 0.75, 1.25, 2.0])
@pytest.mark.parametrize('flip', [False, True])
def test_tiles_match_interpolate(eng, s, flip):
    g = torch.Generator().manual_seed(int(s * 100) + flip)
    x = torch.randn(2, 3, 37, 53, generator=g).cuda()
    ev = _ev()
    hv, wv = ev.view_size(37, 53, s)
    # F.interpolate in fp32 on the device: the kernel shares ATen's fp32 source-index arithmetic, so what remains is
    # the rounding of the four-tap blend (in fp64 the source positions themselves differ by ~dst * 2^-24)
    want = E.view_image(x, s, flip)
    for r0, nr, c0, nc, th, tw in ev.tile_groups(hv, wv, 'sliding', 17)[4]:
        sh = sw = int(17 * 2 / 3)
        got = eng.eval_tiles(x, hv, wv, flip, r0, nr, c0, nc, sh, sw, th, tw)
        assert tuple(got.shape) == (nr * nc * 2, 3, th, tw)
        for t in range(nr * nc):
            r, c = r0 + (t // nc) * sh, c0 + (t % nc) * sw
            ref = want[:, :, r:r + th, c:c + tw]
            if s == 1.0:
                assert torch.equal(got[t * 2:t * 2 + 2], ref)           # a copy, bit for bit
            else:
                assert _absmax(got[t * 2:t * 2 + 2], ref) <= 2e-6
        assert torch.equal(got, eng.eval_tiles(x, hv, wv, flip, r0, nr, c0, nc, sh, sw, th, tw))


def _merge_ref(groups_logits, groups, n, hv, wv, sh, sw, flip):
    """The sequential softmax-add loop in fp64, tiles in row-major order."""
    tiles = []
    for lg, (r0, nr, c0, nc, th, tw) in zip(groups_logits, groups):
        for t in range(nr * nc):
            tiles.append((r0 + (t // nc) * sh, c0 + (t % nc) * sw, th, tw, lg[t * n:(t + 1) * n]))
    tiles.sort(key=lambda z: (z[0], z[1]))
    C = groups_logits[0].shape[1]
    P = torch.zeros(n, C, hv, wv, dtype=torch.float64)
    for r, c, th, tw, lg in tiles:
        P[:, :, r:r + th, c:c + tw] += torch.softmax(lg.double().cpu(), 1)
    return torch.flip(P, (3,)) if flip else P


MERGE_CASES = [(2, 37, 53, 17), (19, 33, 41, 16), (21, 9, 13, 6), (32, 9, 9, 6), (19, 5, 7, 8), (21, 12, 1, 6),
               (19, 16, 21, None)]       # (C, hv, wv, g): odd sizes, hv < g, 1-pixel tails (9 = 4 + 4 + 1), whole


@pytest.mark.parametrize('C,hv,wv,g', MERGE_CASES)
@pytest.mark.parametrize('flip', [False, True])
def test_merge_matches_the_sequential_loop(eng, C, hv, wv, g, flip):
    ev = _ev()
    n = 2
    protocol = 'whole' if g is None else 'sliding'
    gh, gw, sh, sw, groups = ev.tile_groups(hv, wv, protocol, g)
    gen = torch.Generator().manual_seed(C * 1000 + hv * 10 + wv + flip)
    logits = [(torch.randn(nr * nc * n, C, th, tw, generator=gen) * 4).cuda() for _, nr, _, nc, th, tw in groups]
    want = _merge_ref(logits, groups, n, hv, wv, sh, sw, flip)
    got = eng.eval_merge(logits, n, hv, wv, gh, gw, sh, sw, flip)
    assert _absmax(got, want) <= 1e-6
    assert torch.equal(got, eng.eval_merge(logits, n, hv, wv, gh, gw, sh, sw, flip))
    base = torch.randn(n, C, hv, wv, generator=gen).cuda()
    acc = eng.eval_merge(logits, n, hv, wv, gh, gw, sh, sw, flip, out=base.clone(), accumulate=True)
    assert _absmax(acc, want + base.double().cpu()) <= 2e-6


@pytest.mark.parametrize('size', [(37, 53, 28, 40), (20, 30, 41, 59), (16, 16, 16, 16), (1, 5, 3, 9)])
def test_view_add_and_finish(eng, size):
    hv, wv, H, W = size
    gen = torch.Generator().manual_seed(hv * wv)
    P = torch.rand(2, 19, hv, wv, generator=gen).cuda()
    S0 = torch.rand(2, 19, H, W, generator=gen).cuda()
    want = F.interpolate(P, (H, W), mode='bilinear', align_corners=True).double()     # fp32 source indices, as above
    got = eng.eval_view_add(P, torch.empty_like(S0), accumulate=False)
    assert _absmax(got, want) <= 1e-6
    got = eng.eval_view_add(P, S0.clone(), accumulate=True)
    assert _absmax(got, want + S0.double()) <= 1e-6
    assert torch.equal(got, eng.eval_view_add(P, S0.clone(), accumulate=True))
    S = torch.rand(2, 19, H, W, generator=gen).cuda() * 3
    S[0, 0, 0, 0] = 0.0
    mean, logmean = eng.eval_finish(S, 3)
    assert _absmax(mean, S.double() / 3) <= 1e-6
    ref = torch.log(torch.clamp(mean.double(), min=E.FLT_MIN))
    assert float(((logmean.double() - ref).abs() / ref.abs().clamp_min(1.0)).max()) <= 1e-6
    assert abs(float(logmean[0, 0, 0, 0]) - float(np.log(E.FLT_MIN))) <= 1e-5
    m2, l2 = eng.eval_finish(S, 3)
    assert torch.equal(mean, m2) and torch.equal(logmean, l2)


def test_unsupported_input_is_rejected(eng):
    from pixelssl_b200._lib import PxlError
    ev = _ev()
    gh, gw, sh, sw, groups = ev.tile_groups(9, 9, 'sliding', 6)
    big = [torch.zeros(nr * nc, 33, th, tw, device='cuda') for _, nr, _, nc, th, tw in groups]
    with pytest.raises(PxlError):
        eng.eval_merge(big, 1, 9, 9, gh, gw, sh, sw, False)
    with pytest.raises(PxlError):
        eng.eval_view_add(torch.zeros(1, 33, 4, 4, device='cuda'), torch.zeros(1, 33, 8, 8, device='cuda'))
    ok = [torch.zeros(nr * nc, 4, th, tw, device='cuda') for _, nr, _, nc, th, tw in groups]
    with pytest.raises(ValueError):
        eng.eval_merge([t.transpose(2, 3) for t in ok], 1, 9, 9, gh, gw, sh, sw, False)
    with pytest.raises(TypeError):
        eng.eval_merge([t.double() for t in ok], 1, 9, 9, gh, gw, sh, sw, False)
    with pytest.raises(PxlError):
        eng.eval_merge(ok[:-1], 1, 9, 9, gh, gw, sh, sw, False)                # a group missing
    x = torch.zeros(1, 3, 9, 9, device='cuda')
    with pytest.raises(ValueError):
        eng.eval_tiles(x.transpose(2, 3), 9, 9, False, 0, 1, 0, 1, 6, 6, 6, 6)
    with pytest.raises(TypeError):
        eng.eval_tiles(x.half(), 9, 9, False, 0, 1, 0, 1, 6, 6, 6, 6)
    with pytest.raises(PxlError):
        eng.eval_tiles(x, 9, 9, False, 0, 2, 0, 1, 6, 6, 6, 6)                # tiles past the view
    with pytest.raises(TypeError):
        eng.eval_finish(torch.zeros(4, device='cuda', dtype=torch.float64), 2)


# ---- the driver around a stub network --------------------------------------------------------------------------------

def _stub_weights(dtype, device):
    gen = torch.Generator().manual_seed(5)
    w1, w2 = torch.randn(8, 3, 3, 3, generator=gen) * 0.5, torch.randn(5, 8, 3, 3, generator=gen) * 0.5
    return w1.to(device=device, dtype=dtype), w2.to(device=device, dtype=dtype)


def _stub(dtype, device):
    """Two zero-padded 3x3 convolutions: position dependent, so tile borders change the logits."""
    w1, w2 = _stub_weights(dtype, device)
    return lambda t: F.conv2d(torch.tanh(F.conv2d(t, w1, padding=1)), w2, padding=1) * 2


STUB_CASES = {'whole': ('whole', None, [1.0], True), 'sliding': ('sliding', 20, [1.0], False),
              'sliding_scales_flip': ('sliding', 20, [0.75, 1.25], True)}


@pytest.mark.parametrize('case', sorted(STUB_CASES))
def test_driver_matches_the_oracle_around_a_stub(eng, case):
    protocol, crop, scales, flip = STUB_CASES[case]
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 3, 37, 53, generator=g)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        mean, logmean = _ev().evaluate_views(_stub(torch.float32, 'cuda'), x.cuda(), protocol, crop, scales, flip)
        want, _ = E.evaluate(_stub(torch.float32, 'cuda'), x.cuda(), protocol, crop, scales, flip)
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    assert _absmax(mean, want) <= 1e-6
    assert _absmax(torch.exp(logmean), mean) <= 1e-6


def test_launches_per_batch_and_no_synchronisation(eng):
    ev = _ev()
    x = torch.randn(2, 3, 37, 53, generator=torch.Generator().manual_seed(3)).cuda()
    fn = _stub(torch.float32, 'cuda')
    protocol, crop, scales, flip = 'sliding', 20, [0.75, 1.0, 1.25], True
    steps = ev.plan(37, 53, protocol, crop, scales, flip)
    ev.evaluate_views(fn, x, protocol, crop, scales, flip)               # warm-up
    torch.cuda.synchronize()
    seen = []
    real = eng.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)
    eng.call = spy
    torch.cuda.set_sync_debug_mode('error')
    try:
        ev.evaluate_views(fn, x, protocol, crop, scales, flip)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        eng.call = real
    torch.cuda.synchronize()
    assert seen.count('pxl_eval_tiles') == sum(len(st[4][4]) for st in steps)
    assert seen.count('pxl_eval_merge') == len(steps) == 6
    assert seen.count('pxl_eval_view_add') == sum(1 for st in steps if st[0] != 1.0) == 4
    assert seen.count('pxl_eval_finish') == 1


# ---- the driver around the engine's networks -------------------------------------------------------------------------

NETS = {'deeplabv2': {'models': {'model': 'deeplabv2'}},
        'deeplabv3plus': {'models': {'model': 'deeplabv3plus'}},
        'pspnet': {'models': {'model': 'pspnet'}, 'backbone': 'resnet50'}}


def _net_state(net, seed, img):
    """A random-init state whose BatchNorm running statistics are the batch statistics of one training-mode forward
    of ``img`` (momentum 1), as a trained network's are: with mean 0, variance 1 the eval-mode activations of a
    random-init ResNet grow past what the fp16-pair convolutions hold."""
    if net == 'deeplabv2':
        st, fwd = O.randomize_bn_affine(O.init_deeplabv2(seed, cls_bias_std=0.01), seed + 1), O.deeplabv2_forward
    elif net == 'deeplabv3plus':
        st, fwd = O.randomize_bn_affine(D.init(seed, cls_bias_std=0.01), seed + 1), D.forward
    else:
        st, fwd = O.randomize_bn_affine(O.init_pspnet(seed), seed + 1), O.pspnet_forward
    saved = O.batch_norm.__defaults__
    O.batch_norm.__defaults__ = (1.0,) + saved[1:]
    try:
        with torch.no_grad():
            fwd(img, st, True)
    finally:
        O.batch_norm.__defaults__ = saved
    return st, fwd


def _build(net, **proto):
    from pixelssl_b200 import runner
    cfg = dict(BASE, ssl_algorithm='ssl_null', batch_size=2, unlabeled_batch_size=0, ignore_unlabeled=True,
               **NETS[net], **proto)
    return runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))


def _engine_ensemble(alg, img):
    alg.model.eval()
    with torch.no_grad(), _ev().validating():
        res, _ = alg.model.forward((img.cuda(),))
    assert 'sslcct_ad_inp' not in res and res['ssls4l_rc_inp'] is res['pred'][0]
    return res


NET_CASES = [('deeplabv2', 'sliding', 65, [1.0], False), ('deeplabv3plus', 'sliding', 65, [1.0], False),
             ('pspnet', 'sliding', 65, [1.0], False), ('deeplabv2', 'sliding', 65, [0.75, 1.25], True)]


@pytest.mark.parametrize('net,protocol,crop,scales,flip', NET_CASES)
def test_driver_matches_the_tile_loop_around_the_engine_network(ops, net, protocol, crop, scales, flip):
    """The oracle loop calling the engine model's plain forward one tile at a time on the GPU: the protocol alone.
    Within 1e-5, or within FACTOR x the loop's own run-to-run spread where the network's forward is not reproducible
    bit for bit: PSPNet's pyramid pooling adds with fp32 atomics, so two identical per-tile loops differ by up to
    ~1e-5 in P (measured on an H100: 4e-6 .. 1.0e-5 between the ensemble and the loop).  DeepLab-v2 and DeepLabV3+
    repeat bit for bit, so for them the bound is 1e-5 (measured: 0)."""
    from conftest import FACTOR
    img, _ = O.synthetic_batch(21, 2, 2, 97, 129)
    st, _ = _net_state(net, 23, img)
    alg = _build(net, val_protocol=protocol, val_crop_size=crop, val_scales=scales, val_flip=flip)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    res = _engine_ensemble(alg, img)
    plain = alg.model.module.model
    with torch.no_grad():
        loops = [E.evaluate(lambda t: plain(t)[0], img.cuda(), protocol, crop, scales, flip)[0] for _ in range(3)]
    own = max(_absmax(loops[0], loops[1]), _absmax(loops[0], loops[2]))
    err = _absmax(res['activated_pred'][0], loops[0])
    print('%s %s: ensemble vs per-tile loop %.2e (loop vs itself %.2e)' % (net, scales, err, own))
    if net != 'pspnet':
        assert own == 0.0
    assert err <= max(1e-5, FACTOR * own)


_NET_ORACLE = {}


def _oracle_ensemble(net, protocol, crop, scales, flip):
    key = (net, protocol, crop, tuple(scales), flip)
    if key not in _NET_ORACLE:
        img, _ = O.synthetic_batch(31, 2, 2, 97, 129)
        st, fwd = _net_state(net, 33, img)
        out = []
        for dt in (torch.float32, torch.float64):
            s = O.to_dtype(O.to_dtype(st, torch.float64), dt)
            with torch.no_grad():
                out.append(E.evaluate(lambda t: fwd(t, s, False)[0], img.to(dt), protocol, crop, scales, flip)[0])
        _NET_ORACLE[key] = (img, st, out[0], out[1])
    return _NET_ORACLE[key]


@pytest.mark.parametrize('net,protocol,crop,scales,flip', NET_CASES)
def test_whole_network_matches_the_fp64_oracle(ops, net, protocol, crop, scales, flip):
    img, st, p32, p64 = _oracle_ensemble(net, protocol, crop, scales, flip)
    alg = _build(net, val_protocol=protocol, val_crop_size=crop, val_scales=scales, val_flip=flip)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    res = _engine_ensemble(alg, img)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0
    got = res['activated_pred'][0].double().cpu()
    own = _absmax(p32, p64)
    bound = max(1e-3, 3.0 * own)
    err = _absmax(got, p64)
    print('%s %s flip=%s: P vs fp64 %.2e (oracle fp32 %.2e, bound %.2e)' % (net, scales, flip, err, own, bound))
    assert err <= bound
    top2 = torch.topk(p64, 2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 2 * bound
    assert bool(clear.any())
    assert torch.equal(got.argmax(1)[clear], p64.argmax(1)[clear])
    assert _absmax(torch.exp(res['pred'][0]), got) <= 1e-6


# ---- the algorithms --------------------------------------------------------------------------------------------------

ALGS = {
    'ssl_null': {},
    'ssl_mt': {'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1, 'ema_decay': 0.99},
    'ssl_adv': {'adv_for_labeled': True, 'labeled_adv_scale': 0.01, 'unlabeled_adv_scale': 0.001,
                'discriminator_scale': 1.0, 'discriminator_lr': 1e-4, 'unlabeled_for_discriminator': True},
    'ssl_s4l': {'rotated_sup_scale': 0.5, 'rotation_scale': 1.0},
    'ssl_gct': {'ssl_mode': 'gct', 'fc_ssl_scale': 1.0, 'dc_ssl_scale': 100.0, 'dc_threshold': 0.6,
                'dc_rampup_epochs': 1, 'fd_lr': 1e-4, 'fd_scale': 10.0, 'mu': 0.5, 'nu': 1, 'im_size': 65,
                'models': {'lmodel': 'deeplabv2', 'rmodel': 'deeplabv2'}, 'optimizers': {'lmodel': 'sgd', 'rmodel': 'sgd'},
                'lrers': {'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
                'criterions': {'lmodel': 'sseg_criterion', 'rmodel': 'sseg_criterion'}},
    'ssl_cct': {'cons_scale': 30.0, 'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0, 'vat_dec_num': 1, 'drop_dec_num': 1,
                'cut_dec_num': 1, 'context_dec_num': 1, 'object_dec_num': 1, 'fd_dec_num': 1, 'fn_dec_num': 1},
    'ssl_cutmix': {'cons_scale': 20.0, 'cons_rampup_epochs': 0, 'cons_threshold': 0.97, 'ema_decay': 0.99,
                   'batch_size': 6, 'unlabeled_batch_size': 4},      # CutMix mixes pairs of unlabeled rows
    'ssl_cps': {'cps_scale': 1.5, 'cps_rampup_epochs': 0,
                'models': {'lmodel': 'deeplabv2', 'rmodel': 'deeplabv2'}, 'optimizers': {'lmodel': 'sgd', 'rmodel': 'sgd'},
                'lrers': {'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
                'criterions': {'lmodel': 'sseg_criterion', 'rmodel': 'sseg_criterion'}},
    'ssl_unimatch': {'uni_threshold': 0.95, 'uni_scale': 1.0, 'uni_rampup_epochs': 0},
}


def _alg(name, **extra):
    from pixelssl_b200 import runner
    cfg = dict(BASE, ssl_algorithm=name, batch_size=4, unlabeled_batch_size=2)
    cfg.update(ALGS[name])
    cfg.update(extra)
    return runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))


def test_every_algorithm_is_listed():
    from pixelssl_b200 import ALL_SSL_ALGORITHMS
    assert sorted(ALGS) == sorted(ALL_SSL_ALGORITHMS)


@pytest.mark.parametrize('name', sorted(ALGS))
def test_every_algorithm_validates_with_the_protocol(eng, name):
    """Random-init networks in eval mode (running statistics 0 / 1): their activations grow past what the fp16-pair
    convolutions hold, so these run on the exact-fp32 convolutions whatever mode an earlier test left set."""
    torch.manual_seed(0)
    vimg, vlab = O.synthetic_batch(72, 2, 2, 65, 65)
    seen = []
    real = eng.call

    def spy(fn, *args):
        seen.append(fn)
        return real(fn, *args)
    with _precision(eng, 'fp32'):
        alg = _alg(name, **PROTO)
        eng.call = spy
        try:
            alg.validate([((vimg,), (vlab,))], 0)
            torch.cuda.synchronize()
        finally:
            eng.call = real
    values = {k: float(alg.meters[k].val) for k in alg.meters.keys() if '_metric_' in k or 'loss' in k}
    assert any('_metric_' in k for k in values) and all(np.isfinite(v) for v in values.values()), values
    assert seen.count('pxl_eval_finish') >= 1


def _bits(v):
    """The meter value's fp64 bit pattern (NaN compares equal to the same NaN)."""
    return np.ascontiguousarray(np.asarray(v.detach().cpu() if torch.is_tensor(v) else v,
                                           dtype=np.float64)).view(np.uint64)


# meters that do not repeat bit for bit between two identical runs: S4L's rotation head pools with
# ops.adaptive_avg_pool, which adds with fp32 atomics (measured on an H100: the two runs' rotation_loss differ in the
# last bits of the fp32 value in some runs and agree in others); the task meters of every algorithm repeat exactly
NOT_REPRODUCIBLE = {'ssl_s4l': ('rotation_loss',)}


@pytest.mark.parametrize('name', ['ssl_mt', 'ssl_cps', 'ssl_s4l'])
def test_default_protocol_changes_nothing(eng, name):
    """Validation meters with the flags at their defaults are bit-identical to a run without the flags (the few meters
    in NOT_REPRODUCIBLE: within 1e-6 relative), with the same launches."""
    import random
    vimg, vlab = O.synthetic_batch(74, 2, 2, 65, 65)
    meters, launches = [], []
    for extra in ({}, {'val_protocol': 'whole', 'val_scales': [1.0], 'val_flip': False}):
        random.seed(0)
        np.random.seed(0)
        torch.manual_seed(0)
        with _precision(eng, 'fp32'):          # random-init networks in eval mode, as above
            alg = _alg(name, **extra)
            eng.reset_launch_count()
            alg.validate([((vimg,), (vlab,))], 0)
            torch.cuda.synchronize()
            launches.append(eng.launch_count())
        meters.append({k: _bits(alg.meters[k].val) for k in alg.meters.keys()})
        del alg
    assert sorted(meters[0]) == sorted(meters[1]) and launches[0] == launches[1]
    loose = NOT_REPRODUCIBLE.get(name, ())
    for k in meters[0]:
        if k in loose:
            x, y = meters[0][k].view(np.float64), meters[1][k].view(np.float64)
            assert np.all(np.abs(x - y) <= 1e-6 * np.abs(x)), (k, x, y)
        else:
            assert np.array_equal(meters[0][k], meters[1][k]), k
    assert 'task_loss' in meters[0] or 's_task_loss' in meters[0] or 'l_task_loss' in meters[0]


@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_unimatch_training_is_unchanged_by_the_flags(eng, model):
    """The eval-mode pseudo-label forward inside the training step stays the plain forward."""
    img, lab = O.synthetic_batch(91, 4, 2, 65, 65)
    st, _ = _net_state(model, 93, img)
    after = []
    with _precision(eng, 'f16x3'):
        for extra in ({}, PROTO):
            alg = _alg('ssl_unimatch', models={'model': model}, **extra)
            alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
            np.random.seed(3)
            torch.manual_seed(4)
            alg.train([((img,), (lab,))], 0)
            torch.cuda.synchronize()
            after.append(alg.model.arena.data.clone())
            del alg
    assert torch.equal(after[0], after[1])
