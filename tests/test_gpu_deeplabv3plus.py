"""DeepLabV3+ on the engine: the head's concatenation and spatial-mean kernels against torch in fp64, the whole network
against the CPU oracle (oracle/deeplabv3plus_oracle.py), SupOnly / Mean-Teacher steps against the oracle's fp32 and fp64
evaluations, every SSL algorithm end to end, and the tensor-core coverage of the head."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import deeplabv3plus_oracle as D
from oracle import sseg_oracle as O

from conftest import TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
CL = torch.channels_last
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000,
        'models': {'model': 'deeplabv3plus'}}


@pytest.fixture(scope='module', params=TEST_PRECISIONS)
def ops(request):
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    _ops.set_conv_precision(request.param)
    yield _ops
    _ops.set_conv_precision('fp32')


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# sources as (h, w, lanes, channels used), output size, output lanes (None = sum of the used channels)
CONCAT_CASES = {
    'decoder_33to129_320': ([(33, 33, 256, 256), (129, 129, 64, 48)], (129, 129), 320),
    'aspp_broadcast_1to33': ([(33, 33, 16, 16), (33, 33, 8, 8), (1, 1, 24, 24)], (33, 33), None),
    'nonsquare_32x24to125x94': ([(32, 24, 12, 12), (125, 94, 4, 4)], (125, 94), 20),
    'odd_5x7to17x25': ([(5, 7, 7, 5)], (17, 25), None),
    'tiny_2x2to3x3': ([(2, 2, 4, 4), (3, 3, 4, 4)], (3, 3), 12),
    'lines_1x5_4x1to6x9': ([(1, 5, 4, 4), (4, 1, 4, 4), (6, 9, 4, 4)], (6, 9), None),
    'to_one_row_4x4to1x6': ([(4, 4, 4, 4)], (1, 6), None),
}


def _ref_concat(srcs, chans, size, ld):
    parts = [s[:, :c] if tuple(s.shape[2:]) == tuple(size) else
             F.interpolate(s[:, :c], size=size, mode='bilinear', align_corners=True) for s, c in zip(srcs, chans)]
    out = torch.cat(parts, 1)
    return F.pad(out, (0, 0, 0, 0, 0, ld - out.shape[1]))


@pytest.mark.parametrize('case', sorted(CONCAT_CASES))
def test_lane_concat_forward_backward(ops, case):
    spec, size, ld = CONCAT_CASES[case]
    chans = [c for _, _, _, c in spec]
    ld = ld or sum(chans)
    g = torch.Generator().manual_seed(len(case))
    n = 2
    xs = [torch.randn(n, lanes, h, w, generator=g) for h, w, lanes, _ in spec]
    wgt = torch.randn(n, ld, *size, generator=g)
    xd = [x.double().requires_grad_(True) for x in xs]
    ref = _ref_concat(xd, chans, size, ld)
    ref_grads = torch.autograd.grad(ref, xd, wgt.double())
    xg = [x.cuda().contiguous(memory_format=CL).requires_grad_(True) for x in xs]
    out = ops.lane_concat(list(zip(xg, chans)), size, ld)
    assert out.shape == (n, ld, *size) and out.is_contiguous(memory_format=CL)
    assert rel(out, ref) <= 1e-6
    assert torch.count_nonzero(out[:, sum(chans):]) == 0                    # pad lanes are exact zeros
    grads = torch.autograd.grad(out, xg, wgt.cuda(), retain_graph=True)
    again = torch.autograd.grad(out, xg, wgt.cuda())
    for gr, gr2, rg, c in zip(grads, again, ref_grads, chans):
        assert rel(gr, rg) <= 1e-5
        assert torch.count_nonzero(gr[:, c:]) == 0
        assert torch.equal(gr, gr2)                                          # gathered in a fixed order


def test_lane_concat_rejects_bad_windows(ops):
    from pixelssl_b200 import _lib
    x = torch.randn(1, 8, 3, 3, device='cuda').contiguous(memory_format=CL)
    with pytest.raises(_lib.PxlError):
        ops.lane_concat([(x, 8)], (3, 3), 4)                                 # window beyond the output lanes
    with pytest.raises(_lib.PxlError):
        ops.lane_concat([(x, 9)], (3, 3))                                    # more channels than the source has


@pytest.mark.parametrize('shape', [(16, 2048, 33, 33), (2, 64, 7, 5), (3, 40, 1, 9), (2, 33, 1, 1)])
def test_spatial_mean(ops, shape):
    g = torch.Generator(device='cuda').manual_seed(7)
    x = torch.randn(*shape, device='cuda', generator=g).contiguous(memory_format=CL) + 0.5
    y = ops.spatial_mean(x)
    assert rel(y, x.double().mean((2, 3), keepdim=True)) <= 1e-6
    assert torch.equal(y, ops.spatial_mean(x))
    xs = x[:1, :16].contiguous(memory_format=CL).requires_grad_(True)
    w = torch.randn(1, 16, 1, 1, device='cuda', generator=g)
    (gx,) = torch.autograd.grad(ops.spatial_mean(xs), xs, w)
    assert rel(gx, w.double().expand(xs.shape) / (shape[2] * shape[3])) <= 1e-6


def _build(cfg, **over):
    from pixelssl_b200 import runner
    return runner.build_algorithm(runner.build_args(dict(BASE, **dict(cfg, **over)), iters_per_epoch=5))


_NULL = {'ssl_algorithm': 'ssl_null', 'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True}


@pytest.mark.parametrize('h,w', [(97, 97), (75, 97)])
def test_forward_matches_oracle_train_and_eval(ops, h, w):
    """Logits against the oracle evaluated in fp64, within 1e-3 or 2 FACTOR x the oracle's own fp32 deviation from it
    (tests/conftest.py: a deep randomly initialised net amplifies rounding), whichever is larger.  Train mode first; its
    running-statistics update is then what eval mode reads, on every side.
    Measured on an H100 (engine / oracle fp32, relative to the largest logit): train mode 1.1e-3 .. 2.1e-3 / 7.5e-4 in
    fp32, 1.1e-3 .. 2.7e-3 / 6.2e-4 in the tensor-core modes; eval mode 1.3e-4 .. 3.1e-4 / 5.6e-5.  The training-mode
    BatchNorm of the five head layers at batch 2 amplifies rounding more than DeepLab-v2's linear head does; the worst
    case gets the same 2 FACTOR allowance as the worst tensor of assert_energy_yardstick."""
    from conftest import FACTOR
    alg = _build(_NULL)
    st = O.randomize_bn_affine(D.init(31, cls_bias_std=0.01), 32)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    img, _ = O.synthetic_batch(33, 2, 2, h, w)
    st32, st64 = O.to_dtype(O.to_dtype(st, torch.float64), torch.float32), O.to_dtype(st, torch.float64)
    for training in (True, False):
        alg.model.train(training)
        with torch.no_grad():
            res, _ = alg.model.forward((img.cuda(),))
        ref32, latent = D.forward(img, st32, training)
        truth, _ = D.forward(img.double(), st64, training)
        got, own = rel(res['pred'][0], truth), rel(ref32, truth)
        print('deeplabv3+ %s logits vs fp64: engine %.2e, oracle fp32 %.2e' % ('train' if training else 'eval', got, own))
        assert got <= max(1e-3, 2.0 * FACTOR * own)
        assert tuple(res['sslcct_ad_inp'].shape) == tuple(latent.shape)


def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


_ORACLE_CACHE = {}


def _oracle_step(kind, size):
    """The oracle step evaluated in fp32 and fp64 (cached across the precision modes)."""
    key = (kind, size)
    if key not in _ORACLE_CACHE:
        lbs = 2
        n = lbs + (2 if kind == 'mt' else 0)
        img, lab = O.synthetic_batch(41, n, lbs, size, size)
        s0 = O.randomize_bn_affine(D.init(43, cls_bias_std=0.01), 44)
        t0 = O.randomize_bn_affine(D.init(45, cls_bias_std=0.01), 46) if kind == 'mt' else None
        out = []
        for dt in (torch.float32, torch.float64):
            # the oracle steps its states in place: each run gets its own copy
            s = O.to_dtype(O.to_dtype(s0, torch.float64), dt)
            t = O.to_dtype(O.to_dtype(t0, torch.float64), dt) if t0 is not None else None
            mt = D.MTOracle(s, t, lr=0.00025, max_iters=10,
                            cons_scale=1.0, rampup_steps=1, ema_decay=0.99, cons_for_labeled=False)
            r = mt.step(img.to(dt), lab.to(dt), lbs)
            out.append({'loss': {k: float(v) for k, v in r.items() if k.endswith('_loss')},
                        'energy': _energies(r['grads'], mt.names), 'names': mt.names})
        _ORACLE_CACHE[key] = (img, lab, s0, t0, out[0], out[1])
    return _ORACLE_CACHE[key]


@pytest.mark.parametrize('kind,size', [('null', 65), ('mt', 81)])
def test_step_matches_oracle(ops, kind, size):
    img, lab, s0, t0, r32, r64 = _oracle_step(kind, size)
    if kind == 'null':
        alg = _build(_NULL)
        alg.model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        model, keys = alg.model, {'task_loss': 's_task_loss'}
    else:
        alg = _build({'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1,
                      'ema_decay': 0.99, 'batch_size': 4, 'unlabeled_batch_size': 2})
        alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
        model, keys = alg.s_model, {'s_task_loss': 's_task_loss', 't_task_loss': 't_task_loss', 'cons_loss': 'cons_loss'}
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    for mk, ok in keys.items():
        assert_loss_yardstick(float(alg.meters[mk].val), r32['loss'][ok], r64['loss'][ok], '%s %s' % (kind, mk))
    sp = dict(model.module.model.named_parameters())
    got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in r64['names']])
    print(assert_energy_yardstick(got, r32['energy'], r64['energy'], '%s grad energies' % kind))


def test_single_sample_training_forward_raises(ops):
    alg = _build(_NULL)
    img, _ = O.synthetic_batch(51, 1, 1, 65, 65)
    m = alg.model.module.model.aspp.convs[4][2]
    before = (m.running_mean.clone(), m.running_var.clone())
    alg.model.train()
    with pytest.raises(ValueError, match='more than 1 value per channel'):
        alg.model.forward((img.cuda(),))
    assert torch.equal(m.running_mean, before[0]) and torch.equal(m.running_var, before[1])
    alg.model.eval()
    with torch.no_grad():
        res, _ = alg.model.forward((img.cuda(),))
    assert res['pred'][0].shape == (1, 21, 65, 65) and bool(torch.isfinite(res['pred'][0]).all())


@pytest.mark.parametrize('precision', ['f16x3', 'tf32x3'])
def test_head_runs_on_tensor_cores(precision):
    """One Mean-Teacher step: no FFMA convolution launch (forward, dgrad or wgrad) at all, and the head's new kernels
    run."""
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops
    ops.set_conv_precision(precision)
    seen = []
    real = ops.call

    def spy(name, *args):
        if name in ('pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc'):
            gm = args[0]._obj
            seen.append((name, gm.N, gm.H, gm.W, gm.Cin, gm.OH, gm.OW, gm.Cout, gm.ntaps))
        else:
            seen.append((name,))
        return real(name, *args)

    try:
        alg = _build({'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1,
                      'ema_decay': 0.99, 'batch_size': 4, 'unlabeled_batch_size': 2})
        img, lab = O.synthetic_batch(61, 4, 2, 97, 97)
        ops.call = spy
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
    finally:
        ops.call = real
        ops.set_conv_precision('fp32')
    ffma = [s for s in seen if s[0] in ('pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc')]
    assert not ffma, ffma
    names = {s[0] for s in seen}
    assert {'pxl_lane_concat_nhwc', 'pxl_lane_concat_bwd_nhwc', 'pxl_spatial_mean_nhwc'} <= names
    assert names & {'pxl_conv_h16_launch', 'pxl_conv_tc_launch_ex'}


_ALGS = {
    'ssl_null': dict(_NULL),
    'ssl_mt': {'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1, 'ema_decay': 0.99},
    'ssl_cutmix': {'cons_scale': 20.0, 'cons_rampup_epochs': 0, 'cons_threshold': 0.97, 'ema_decay': 0.99,
                   'unlabeled_batch_size': 4, 'batch_size': 6},       # the mixed half of the unlabeled rows is a batch of 2
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
}


@pytest.mark.parametrize('name', sorted(_ALGS))
def test_every_algorithm_trains_validates_and_checkpoints(name, tmp_path):
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops, runner
    ops.set_conv_precision('f16x3')
    try:
        cfg = dict(BASE, ssl_algorithm=name, batch_size=4, unlabeled_batch_size=2)
        cfg.update(_ALGS[name])
        args = runner.build_args(cfg, iters_per_epoch=5)
        args.checkpoint_path = str(tmp_path)
        torch.manual_seed(0)
        alg = runner.build_algorithm(args)
        img, lab = O.synthetic_batch(71, cfg['batch_size'], cfg['batch_size'] - cfg['unlabeled_batch_size'], 65, 65)
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
        losses = {k: float(alg.meters[k].val) for k in alg.meters.keys() if 'loss' in k}
        assert losses and all(np.isfinite(v) for v in losses.values()), losses
        vimg, vlab = O.synthetic_batch(72, 2, 2, 65, 65)
        alg._validate([((vimg,), (vlab,))], 0)
        metrics = {k: float(alg.meters[k].val) for k in alg.meters.keys() if '_metric_' in k}
        assert metrics and all(np.isfinite(v) for v in metrics.values()), metrics
        alg.save_checkpoint(1)
        path = os.path.join(str(tmp_path), 'checkpoint_1.ckpt')
        alg2 = runner.build_algorithm(args)
        args.resume = path
        assert alg2.load_checkpoint() == 1
        for key, mod in alg.models.items():
            a, b = mod.state_dict(), alg2.models[key].state_dict()
            assert list(a) == list(b) and all(k.startswith('module.') for k in a)
            for k in a:
                assert torch.equal(a[k].cpu(), b[k].cpu()), (key, k)
    finally:
        ops.set_conv_precision('fp32')
