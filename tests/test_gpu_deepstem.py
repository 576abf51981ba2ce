"""Deep-stem ResNet backbones on the engine: the 3x3/2 stem unfold (fp32 and fp16 pair) bit for bit against torch, the
stem convolution against fp64 torch in every precision mode, DeepLab-v2 / DeepLabV3+ with resnet101-deepstem against
the fp64 oracle (oracle/deepstem_oracle.py), SupOnly / Mean-Teacher steps against the oracle's fp32 and fp64
evaluations, the tensor-core coverage of a step, every SSL algorithm end to end, and run-to-run determinism."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import deeplabv3plus_oracle as D
from oracle import deepstem_oracle as S
from oracle import sseg_oracle as O

from conftest import FACTOR, TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
CL = torch.channels_last
BB = 'resnet101-deepstem'
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000, 'backbone': BB}
_NULL = {'ssl_algorithm': 'ssl_null', 'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True}
_MT = {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1,
       'ema_decay': 0.99, 'batch_size': 4, 'unlabeled_batch_size': 2}
_ORACLES = {'deeplabv2': (O.init_deeplabv2, O.deeplabv2_forward, O.MTOracle),
            'deeplabv3plus': (D.init, D.forward, D.MTOracle)}


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


def _unfold_ref(img, lanes):
    """[N*OH*OW, lanes] with k = (r*3 + s)*3 + c for k < 27 and zeros above, from F.unfold ((c, r, s) order)."""
    N = img.shape[0]
    u = F.unfold(img, 3, padding=1, stride=2)                          # [N, 27, L], row c*9 + r*3 + s
    u = u.view(N, 3, 9, -1).permute(0, 3, 2, 1).reshape(-1, 27)        # [N*L, (r, s, c)]
    return F.pad(u, (0, lanes - 27))


@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('H,W', [(65, 65), (97, 97), (75, 97), (513, 513)])
def test_unfold_is_exact(eng, N, H, W):
    from pixelssl_b200.ops import _p, H16_ACT_SCALE
    g = torch.Generator().manual_seed(H * 31 + W + N)
    img = torch.randn(N, 3, H, W, generator=g).cuda()
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    cols = torch.full((N * OH * OW, 32), float('nan'), device='cuda')
    eng.call('pxl_stem3x3s2_im2col', _p(img), _p(cols), N, H, W, OH, OW, eng._stream())
    ref = _unfold_ref(img, 32)
    assert torch.equal(cols, ref)
    before = eng.h16_status()
    buf = torch.full((2, N * OH * OW * 64), float('nan'), dtype=torch.float16, device='cuda')
    eng.call('pxl_stem3x3s2_im2col_h16', _p(img), _p(buf[0]), _p(buf[1]), float(H16_ACT_SCALE), N, H, W, OH, OW, eng._stream())
    torch.cuda.synchronize()
    v = _unfold_ref(img, 64).reshape(-1) * H16_ACT_SCALE                # exact: power-of-two scale
    hi = v.half()
    assert torch.equal(buf[0], hi)
    assert torch.equal(buf[1], (v - hi.float()).half())
    assert float((buf[0].float() + buf[1].float() - v).abs().max()) <= float(v.abs().max()) * 2.0 ** -21
    assert eng.h16_status() == before


@pytest.mark.parametrize('precision,tol_y,tol_w', [('fp32', 1e-5, 1e-4), ('tf32x3', 2e-5, 5e-5), ('tf32', 3e-3, 3e-3),
                                                   ('f16x3', 2e-5, 5e-5), ('f16', 3e-3, 3e-3)])
@pytest.mark.parametrize('N,H,W', [(2, 65, 65), (1, 97, 129), (2, 40, 36)])
def test_stem_conv_matches_fp64(eng, N, H, W, precision, tol_y, tol_w):
    """3x3/2 pad 1 stem convolution: forward, weight gradient and (tensor-core modes) the fused BatchNorm sums."""
    gs = torch.Generator().manual_seed(H * 7 + W)
    img = torch.randn(N, 3, H, W, generator=gs, dtype=torch.float64)
    w = torch.randn(64, 3, 3, 3, generator=gs, dtype=torch.float64) * 0.3
    wc = w.clone().requires_grad_(True)
    yc = F.conv2d(img, wc, stride=2, padding=1)
    wt = torch.randn(yc.shape, generator=gs, dtype=torch.float64)
    (yc * wt).sum().backward()
    eng.set_conv_precision(precision)
    wg = w.float().cuda().contiguous(memory_format=CL).requires_grad_(True)
    yg = eng.stem_conv(img.float().cuda(), wg, want_bn_stats=True)
    (yg * wt.float().cuda()).sum().backward()
    torch.cuda.synchronize()
    assert yg.shape == yc.shape and yg.is_contiguous(memory_format=CL)
    assert rel(yg, yc) <= tol_y
    assert rel(wg.grad, wc.grad) <= tol_w
    if precision != 'fp32':
        ref = torch.cat((yc.sum(dim=(0, 2, 3)), (yc ** 2).sum(dim=(0, 2, 3))))
        assert rel(yg._pxl_bn_sums, ref) <= max(tol_y * 10, 1e-4)
    assert eng.conv_tc_status() == 0 and eng.h16_status() == 0


def _build(cfg, model, **over):
    from pixelssl_b200 import runner
    return runner.build_algorithm(runner.build_args(dict(BASE, models={'model': model}, **dict(cfg, **over)),
                                                    iters_per_epoch=5))


def _init(model, seed, bn_seed, **k):
    with S.deep_stem():
        return O.randomize_bn_affine(_ORACLES[model][0](seed, cls_bias_std=0.01, **k), bn_seed)


@pytest.mark.parametrize('h,w', [(97, 97), (75, 97)])
@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_forward_matches_oracle_train_and_eval(ops, model, h, w):
    """Logits against the oracle evaluated in fp64, within 1e-3 or 2 FACTOR x the oracle's own fp32 deviation from it,
    as for DeepLabV3+ (tests/test_gpu_deeplabv3plus.py).  Train mode first; its running-statistics update is then what
    eval mode reads, on every side."""
    alg = _build(_NULL, model)
    st = _init(model, 31, 32)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    img, _ = O.synthetic_batch(33, 2, 2, h, w)
    st32, st64 = O.to_dtype(O.to_dtype(st, torch.float64), torch.float32), O.to_dtype(st, torch.float64)
    fwd = _ORACLES[model][1]
    for training in (True, False):
        alg.model.train(training)
        with torch.no_grad():
            res, _ = alg.model.forward((img.cuda(),))
        with S.deep_stem():
            ref32, latent = fwd(img, st32, training)
            truth, _ = fwd(img.double(), st64, training)
        got, own = rel(res['pred'][0], truth), rel(ref32, truth)
        print('%s deep stem %s logits vs fp64: engine %.2e, oracle fp32 %.2e' % (model, 'train' if training else 'eval', got, own))
        assert got <= max(1e-3, 2.0 * FACTOR * own)
        assert tuple(res['sslcct_ad_inp'].shape) == tuple(latent.shape)
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0


def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


_ORACLE_CACHE = {}


def _oracle_step(model, kind, size):
    key = (model, kind, size)
    if key not in _ORACLE_CACHE:
        # SupOnly on 4 labeled images: with 2, DeepLabV3+'s image-pooling BatchNorm normalises 2 values per channel and
        # the gradient energies of a random-init net become chaotic in rounding (the oracle's own fp32 evaluation is
        # then 3e-2 from fp64 at the median, 15x the other cases)
        lbs = 2 if kind == 'mt' else 4
        n = lbs + (2 if kind == 'mt' else 0)
        img, lab = O.synthetic_batch(41, n, lbs, size, size)
        s0 = _init(model, 43, 44)
        t0 = _init(model, 45, 46) if kind == 'mt' else None
        out = []
        for dt in (torch.float32, torch.float64):
            s = O.to_dtype(O.to_dtype(s0, torch.float64), dt)
            t = O.to_dtype(O.to_dtype(t0, torch.float64), dt) if t0 is not None else None
            with S.deep_stem():
                mt = _ORACLES[model][2](s, t, lr=0.00025, max_iters=10, cons_scale=1.0, rampup_steps=1, ema_decay=0.99,
                                        cons_for_labeled=False)
                r = mt.step(img.to(dt), lab.to(dt), lbs)
            out.append({'loss': {k: float(v) for k, v in r.items() if k.endswith('_loss')},
                        'energy': _energies(r['grads'], mt.names), 'names': mt.names})
        _ORACLE_CACHE[key] = (img, lab, s0, t0, out[0], out[1])
    return _ORACLE_CACHE[key]


@pytest.mark.parametrize('kind,size', [('null', 65), ('mt', 81)])
@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_step_matches_oracle(ops, model, kind, size):
    img, lab, s0, t0, r32, r64 = _oracle_step(model, kind, size)
    if kind == 'null':
        alg = _build(_NULL, model, batch_size=4)
        alg.model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        net, keys = alg.model, {'task_loss': 's_task_loss'}
    else:
        alg = _build(_MT, model)
        alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
        net, keys = alg.s_model, {'s_task_loss': 's_task_loss', 't_task_loss': 't_task_loss', 'cons_loss': 'cons_loss'}
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    for mk, ok in keys.items():
        assert_loss_yardstick(float(alg.meters[mk].val), r32['loss'][ok], r64['loss'][ok], '%s %s %s' % (model, kind, mk))
    sp = dict(net.module.model.named_parameters())
    assert [n for n in sp] == r64['names']
    got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in r64['names']])
    print(assert_energy_yardstick(got, r32['energy'], r64['energy'], '%s %s grad energies' % (model, kind)))


@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
@pytest.mark.parametrize('precision', ['f16x3', 'tf32x3'])
def test_step_runs_on_tensor_cores(eng, precision, model):
    """One Mean-Teacher step: no FFMA convolution launch (forward, dgrad or wgrad) at all, and the 3x3 unfold runs."""
    eng.set_conv_precision(precision)
    seen = []
    real = eng.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)

    alg = _build(_MT, model)
    img, lab = O.synthetic_batch(61, 4, 2, 97, 97)
    eng.call = spy
    try:
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
    finally:
        eng.call = real
    assert not {'pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc'} & set(seen)
    unfold = 'pxl_stem3x3s2_im2col_h16' if precision == 'f16x3' else 'pxl_stem3x3s2_im2col'
    assert unfold in seen
    assert not {'pxl_stem_im2col', 'pxl_stem_im2col_h16', 'pxl_stem_conv7x7s2'} & set(seen)
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
    network's are.  UniMatch's step runs an eval-mode forward; with the initial running statistics (mean 0, variance 1)
    a random-init ResNet's activations grow past what the fp16-pair convolutions hold (tests/test_gpu_unimatch.py)."""
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
def test_every_algorithm_trains_validates_and_checkpoints(eng, name, tmp_path):
    from pixelssl_b200 import runner
    eng.set_conv_precision('f16x3')
    cfg = dict(BASE, models={'model': 'deeplabv3plus'}, ssl_algorithm=name, batch_size=4, unlabeled_batch_size=2)
    cfg.update(_ALGS[name])
    args = runner.build_args(cfg, iters_per_epoch=5)
    args.checkpoint_path = str(tmp_path)
    torch.manual_seed(0)
    np.random.seed(0)
    alg = runner.build_algorithm(args)
    img, lab = O.synthetic_batch(71, cfg['batch_size'], cfg['batch_size'] - cfg['unlabeled_batch_size'], 65, 65)
    if name == 'ssl_unimatch':
        _running_stats_of_one_batch(alg.model, img)
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
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
        assert list(a) == list(b)
        for k in a:
            assert torch.equal(a[k].cpu(), b[k].cpu()), (key, k)
    assert any(k.endswith('backbone.conv1.6.weight') for mod in alg.models.values() for k in mod.state_dict())


@pytest.mark.parametrize('precision', ['f16x3', 'tf32x3'])
def test_mean_teacher_step_is_deterministic(eng, precision):
    eng.set_conv_precision(precision)
    s0, t0 = _init('deeplabv3plus', 81, 82), _init('deeplabv3plus', 83, 84)
    img, lab = O.synthetic_batch(85, 4, 2, 65, 65)
    runs = []
    for _ in range(2):
        alg = _build(_MT, 'deeplabv3plus')
        alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
        alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        runs.append(({k: float(alg.meters[k].val) for k in ('s_task_loss', 't_task_loss', 'cons_loss')},
                     {k: v.detach().cpu().clone() for k, v in alg.s_model.state_dict().items()}))
    assert runs[0][0] == runs[1][0]
    for k, v in runs[0][1].items():
        assert torch.equal(v, runs[1][1][k]), k
