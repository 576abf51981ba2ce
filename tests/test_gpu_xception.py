"""DeepLabV3+ on the aligned Xception-65 backbone, on the engine: the depthwise kernels (forward, dgrad, wgrad) against
fp64 F.conv2d(groups=C), the whole forward and SupOnly / Mean-Teacher steps against the fp64 oracle
(oracle/xception_oracle.py) in every test precision, the tensor-core coverage of a step, every SSL algorithm end to end,
and run-to-run determinism."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sseg_oracle as O
from oracle import xception_oracle as X

from conftest import FACTOR, TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
CL = torch.channels_last
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000, 'backbone': 'xception65',
        'pretrained_backbone': 'none'}
_NULL = {'ssl_algorithm': 'ssl_null', 'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True}
_MT = {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1,
       'ema_decay': 0.99, 'batch_size': 4, 'unlabeled_batch_size': 2}
DW_ENTRIES = ('pxl_dw_conv_fwd', 'pxl_dw_conv_dgrad', 'pxl_dw_conv_wgrad')


@pytest.fixture(scope='module', params=TEST_PRECISIONS)
def ops(request):
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    _ops.set_conv_precision(request.param)
    yield _ops
    _ops.set_conv_precision('fp32')


@pytest.fixture
def eng():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    yield _ops
    _ops.set_conv_precision('fp32')


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ---- depthwise kernels -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('N,H,W', [(1, 17, 17), (3, 16, 22), (1, 33, 20)])
@pytest.mark.parametrize('stride,dilation', [(1, 1), (1, 2), (1, 4), (2, 1)])
@pytest.mark.parametrize('C,ld', [(64, 64), (128, 128), (256, 256), (728, 768), (1024, 1024), (1536, 1536)])
def test_depthwise_matches_fp64(eng, C, ld, stride, dilation, N, H, W):
    """Against fp64 on the same fp32 inputs: forward and dgrad sum 9 products per value (bound 1e-6 of the largest),
    wgrad sums N*OH*OW up to ~1000 products (bound 1e-5).  The input's pad lanes hold NaN: they are never read, and
    every output pad lane is an exact zero.  Two calls are bit-identical."""
    g = torch.Generator().manual_seed(C * 131 + H * 7 + W + N * 3 + stride * 17 + dilation)
    x = torch.randn(N, C, H, W, generator=g, dtype=torch.float64).float().double()
    w = (torch.randn(C, 1, 3, 3, generator=g, dtype=torch.float64) * 0.3).float().double()
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    dy = torch.randn(N, C, OH, OW, generator=g, dtype=torch.float64).float().double()
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yr = F.conv2d(F.pad(xr, (dilation,) * 4), wr, stride=stride, dilation=dilation, groups=C)
    assert yr.shape == dy.shape
    (yr * dy).sum().backward()

    def padded(t):
        out = torch.full((t.shape[0], ld) + tuple(t.shape[2:]), float('nan'), device='cuda').contiguous(memory_format=CL)
        out[:, :C] = t.float().cuda()
        return out

    xg, dyg, wg = padded(x), padded(dy), w.float().cuda().contiguous()
    runs = []
    for _ in range(2):
        wl = wg.clone().requires_grad_(True)
        xl = xg.clone().requires_grad_(True)
        y = eng.depthwise_conv(xl, wl, stride, dilation)
        y.backward(dyg)
        torch.cuda.synchronize()
        runs.append((y.detach(), xl.grad, wl.grad))
    y, dx, dw = runs[0]
    assert y.shape == (N, ld, OH, OW) and y.is_contiguous(memory_format=CL)
    assert rel(y[:, :C], yr) <= 1e-6
    assert rel(dx[:, :C], xr.grad) <= 1e-6
    assert rel(dw, wr.grad) <= 1e-5
    if ld > C:
        assert torch.equal(y[:, C:], torch.zeros_like(y[:, C:]))
        assert torch.equal(dx[:, C:], torch.zeros_like(dx[:, C:]))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)


def test_depthwise_rejects_what_it_does_not_cover(eng):
    from pixelssl_b200._lib import PxlError
    x = torch.zeros(1, 64, 9, 9, device='cuda').contiguous(memory_format=CL)
    with pytest.raises(PxlError):
        eng.depthwise_conv(x, torch.zeros(64, 1, 3, 3, device='cuda'), 2, 2)
    with pytest.raises(ValueError):
        eng.depthwise_conv(x, torch.zeros(128, 1, 3, 3, device='cuda'), 1, 1)


# ---- the network --------------------------------------------------------------------------------------------------------

def _build(cfg, **over):
    from pixelssl_b200 import runner
    return runner.build_algorithm(runner.build_args(dict(BASE, models={'model': 'deeplabv3plus'}, **dict(cfg, **over)),
                                                    iters_per_epoch=5))


def _init(seed, bn_seed):
    return O.randomize_bn_affine(X.init(seed, cls_bias_std=0.01), bn_seed)


@pytest.mark.parametrize('h,w', [(97, 97), (75, 97)])
def test_forward_matches_oracle_train_and_eval(ops, h, w):
    """Logits against the oracle in fp64, within 1e-3 or 2 FACTOR x the oracle's own fp32 deviation from it (as for the
    ResNet backbones).  Train mode first; its running-statistics update is what eval mode then reads, on every side."""
    alg = _build(_NULL)
    st = _init(31, 32)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    img, _ = O.synthetic_batch(33, 2, 2, h, w)
    st32, st64 = O.to_dtype(O.to_dtype(st, torch.float64), torch.float32), O.to_dtype(st, torch.float64)
    for training in (True, False):
        alg.model.train(training)
        with torch.no_grad():
            res, _ = alg.model.forward((img.cuda(),))
        ref32, latent = X.forward(img, st32, training)
        truth, _ = X.forward(img.double(), st64, training)
        got, own = rel(res['pred'][0], truth), rel(ref32, truth)
        print('xception65 %s logits vs fp64: engine %.2e, oracle fp32 %.2e' % ('train' if training else 'eval', got, own))
        assert got <= max(1e-3, 2.0 * FACTOR * own)
        assert tuple(res['sslcct_ad_inp'].shape) == tuple(latent.shape)
    sd = alg.model.state_dict()
    for k, v in st64.items():
        if k.endswith('running_var') or k.endswith('running_mean'):
            assert rel(sd['module.model.' + k], v) <= 1e-2, k
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0


def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


_ORACLE_CACHE = {}


def _oracle_step(kind, size):
    key = (kind, size)
    if key not in _ORACLE_CACHE:
        lbs = 2 if kind == 'mt' else 4
        n = lbs + (2 if kind == 'mt' else 0)
        img, lab = O.synthetic_batch(41, n, lbs, size, size)
        s0 = _init(43, 44)
        t0 = _init(45, 46) if kind == 'mt' else None
        out = []
        for dt in (torch.float32, torch.float64):
            s = O.to_dtype(O.to_dtype(s0, torch.float64), dt)
            t = O.to_dtype(O.to_dtype(t0, torch.float64), dt) if t0 is not None else None
            mt = X.MTOracle(s, t, lr=0.00025, max_iters=10, cons_scale=1.0, rampup_steps=1, ema_decay=0.99,
                            cons_for_labeled=False)
            r = mt.step(img.to(dt), lab.to(dt), lbs)
            out.append({'loss': {k: float(v) for k, v in r.items() if k.endswith('_loss')},
                        'energy': _energies(r['grads'], mt.names), 'names': mt.names})
        _ORACLE_CACHE[key] = (img, lab, s0, t0, out[0], out[1])
    return _ORACLE_CACHE[key]


@pytest.mark.parametrize('kind,size', [('null', 65), ('mt', 81)])
def test_step_matches_oracle(ops, kind, size):
    img, lab, s0, t0, r32, r64 = _oracle_step(kind, size)
    if kind == 'null':
        alg = _build(_NULL, batch_size=4)
        alg.model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        net, keys = alg.model, {'task_loss': 's_task_loss'}
    else:
        alg = _build(_MT)
        alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
        net, keys = alg.s_model, {'s_task_loss': 's_task_loss', 't_task_loss': 't_task_loss', 'cons_loss': 'cons_loss'}
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    for mk, ok in keys.items():
        assert_loss_yardstick(float(alg.meters[mk].val), r32['loss'][ok], r64['loss'][ok], 'xception65 %s %s' % (kind, mk))
    sp = dict(net.module.model.named_parameters())
    assert [n for n in sp] == r64['names']
    got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in r64['names']])
    print(assert_energy_yardstick(got, r32['energy'], r64['energy'], 'xception65 %s grad energies' % kind))


@pytest.mark.parametrize('precision', ['f16x3', 'tf32x3'])
def test_step_runs_on_tensor_cores(eng, precision):
    """One Mean-Teacher step: no FFMA dense-convolution launch (forward, dgrad or wgrad); the depthwise kernels run."""
    eng.set_conv_precision(precision)
    seen = []
    real = eng.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)

    alg = _build(_MT)
    img, lab = O.synthetic_batch(61, 4, 2, 97, 97)
    eng.call = spy
    try:
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
    finally:
        eng.call = real
    assert not {'pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc'} & set(seen)
    assert set(DW_ENTRIES) <= set(seen)
    assert eng.conv_tc_status() == 0 and eng.h16_status() == 0


_ALGS = {
    'ssl_null': dict(_NULL),
    'ssl_mt': {'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1, 'ema_decay': 0.99},
    'ssl_cutmix': {'cons_scale': 20.0, 'cons_rampup_epochs': 0, 'cons_threshold': 0.97, 'ema_decay': 0.99,
                   'unlabeled_batch_size': 4, 'batch_size': 6},
    'ssl_adv': {'adv_for_labeled': True, 'labeled_adv_scale': 0.01, 'unlabeled_adv_scale': 0.001,
                'discriminator_scale': 1.0, 'discriminator_lr': 1e-4, 'unlabeled_for_discriminator': True},
    'ssl_gct': {'ssl_mode': 'gct', 'fc_ssl_scale': 1.0, 'dc_ssl_scale': 100.0, 'dc_threshold': 0.6, 'dc_rampup_epochs': 1,
                'fd_lr': 1e-4, 'fd_scale': 10.0, 'mu': 0.5, 'nu': 1, 'im_size': 65,
                'models': {'lmodel': 'deeplabv3plus', 'rmodel': 'deeplabv3plus'},
                'optimizers': {'lmodel': 'sgd', 'rmodel': 'sgd'},
                'lrers': {'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
                'criterions': {'lmodel': 'sseg_criterion', 'rmodel': 'sseg_criterion'}},
    'ssl_cct': {'cons_scale': 30.0, 'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0, 'vat_dec_num': 1, 'drop_dec_num': 1,
                'cut_dec_num': 1, 'context_dec_num': 1, 'object_dec_num': 1, 'fd_dec_num': 1, 'fn_dec_num': 1},
    'ssl_s4l': {'rotated_sup_scale': 0.5, 'rotation_scale': 1.0},
    'ssl_cps': {'cps_scale': 1.5, 'cps_rampup_epochs': 0,
                'models': {'lmodel': 'deeplabv3plus', 'rmodel': 'deeplabv3plus'},
                'optimizers': {'lmodel': 'sgd', 'rmodel': 'sgd'},
                'lrers': {'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
                'criterions': {'lmodel': 'sseg_criterion', 'rmodel': 'sseg_criterion'}},
    'ssl_unimatch': {'uni_threshold': 0.0, 'uni_scale': 1.0, 'uni_rampup_epochs': 0},
}


def _running_stats_of_one_batch(model, img):
    """BatchNorm running statistics := the batch statistics of one training-mode forward (momentum 1), as a trained
    network's are, before UniMatch's eval-mode pseudo-label forward."""
    from pixelssl_b200.nn.modules import BatchNorm2d
    bns = [m for m in model.modules() if isinstance(m, BatchNorm2d)]
    for m in bns:
        m.momentum = 1.0
    model.train()
    with torch.no_grad():
        model.forward((img.cuda(),))
    for m in bns:
        m.momentum = 0.1


@pytest.mark.parametrize('name', sorted(_ALGS))
def test_every_algorithm_trains(eng, name):
    from pixelssl_b200 import runner
    eng.set_conv_precision('f16x3')
    cfg = dict(BASE, models={'model': 'deeplabv3plus'}, ssl_algorithm=name, batch_size=4, unlabeled_batch_size=2)
    cfg.update(_ALGS[name])
    torch.manual_seed(0)
    np.random.seed(0)
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
    if name == 'ssl_unimatch':
        assert alg.model.module.fp_channels == (128, 2048)
    img, lab = O.synthetic_batch(71, cfg['batch_size'], cfg['batch_size'] - cfg['unlabeled_batch_size'], 65, 65)
    if name == 'ssl_unimatch':
        _running_stats_of_one_batch(alg.model, img)
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
    losses = {k: float(alg.meters[k].val) for k in alg.meters.keys() if 'loss' in k}
    assert losses and all(np.isfinite(v) for v in losses.values()), losses


def test_mean_teacher_step_is_deterministic(eng):
    eng.set_conv_precision('f16x3')
    s0, t0 = _init(81, 82), _init(83, 84)
    img, lab = O.synthetic_batch(85, 4, 2, 65, 65)
    runs = []
    for _ in range(2):
        alg = _build(_MT)
        alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        runs.append(({k: float(alg.meters[k].val) for k in ('s_task_loss', 't_task_loss', 'cons_loss')},
                     {k: v.detach().cpu().clone() for k, v in alg.s_model.state_dict().items()}))
    assert runs[0][0] == runs[1][0]
    for k, v in runs[0][1].items():
        assert torch.equal(v, runs[1][1][k]), k
