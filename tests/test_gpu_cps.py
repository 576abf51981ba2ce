"""Cross Pseudo Supervision on the engine: the fused pxl_cps_ce kernel against torch in fp64, the plain and CutMix steps
against the CPU oracle (oracle/cps_oracle.py) evaluated in fp32 and fp64, ssl_cps end to end with every task model,
its launches, and the step's determinism."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cps_oracle as C
from oracle import sseg_oracle as O

from conftest import TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
BASE = {'ssl_algorithm': 'ssl_cps', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'log_freq': 1000, 'cps_scale': 1.5, 'cps_rampup_epochs': 0}
PAIR = {'models': {'lmodel': 'deeplabv2', 'rmodel': 'deeplabv2'}, 'optimizers': {'lmodel': 'sgd', 'rmodel': 'sgd'},
        'lrers': {'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
        'criterions': {'lmodel': 'sseg_criterion', 'rmodel': 'sseg_criterion'}}
MASK_SEED = 2024


@pytest.fixture(scope='module')
def eng():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import __graft_entry__ as ge
    ge.build()
    from pixelssl_b200 import ops
    return ops


@pytest.fixture(params=TEST_PRECISIONS)
def ops(request, eng):
    eng.set_conv_precision(request.param)
    yield eng
    eng.set_conv_precision('fp32')


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


# ---- the kernel ------------------------------------------------------------------------------------------------------

def _logits(g, n, c, h, w):
    """randn logits, with every other pixel replaced by values on a coarse grid: many exact ties in the argmax"""
    x = torch.randn(n, c, h, w, generator=g)
    q = torch.randint(-2, 3, (n, c, h, w), generator=g).float() * 0.75
    tied = (torch.arange(h * w).reshape(h, w) % 2 == 0)
    return torch.where(tied, q, x)


def _reference(s_l, s_r, t_l, t_r, scale, w_l=1.0, w_r=1.0):
    """fp64 torch: per-sample losses, the two scaled means, and the gradients of w_l * loss_l + w_r * loss_r"""
    sl, sr = s_l.double().requires_grad_(True), s_r.double().requires_grad_(True)
    y_r, y_l = t_r.double().argmax(1), t_l.double().argmax(1)
    per_l = F.cross_entropy(sl, y_r, reduction='none').mean((1, 2))
    per_r = F.cross_entropy(sr, y_l, reduction='none').mean((1, 2))
    ll, lr = scale * per_l.mean(), scale * per_r.mean()
    gl, gr = torch.autograd.grad(w_l * ll + w_r * lr, (sl, sr))
    return torch.cat([per_l, per_r]).detach(), ll.detach(), lr.detach(), gl, gr, y_l, y_r


def _labels_from_grad(grad):
    """the pseudo-label each pixel was trained towards: the one channel with a negative gradient (p_y - 1 < 0)"""
    neg = grad < 0
    assert bool((neg.sum(1) == 1).all())
    return neg.float().argmax(1).cpu()


KERNEL_CASES = [(n, c, hw, alias) for n in (1, 3) for c in (2, 21, 32) for hw in ((65, 65), (1, 1), (33, 47))
                for alias in (True, False)] + [(2, 21, (513, 513), True), (2, 21, (513, 513), False)]


@pytest.mark.parametrize('n,c,hw,alias', KERNEL_CASES)
def test_cps_kernel_matches_torch_fp64(eng, n, c, hw, alias):
    h, w = hw
    g = torch.Generator().manual_seed(n * 1000 + c * 10 + h)
    s_l, s_r = _logits(g, n, c, h, w), _logits(g, n, c, h, w)
    t_l, t_r = (s_l, s_r) if alias else (_logits(g, n, c, h, w), _logits(g, n, c, h, w))
    scale = 1.7
    per_ref, ll_ref, lr_ref, gl_ref, gr_ref, y_l, y_r = _reference(s_l, s_r, t_l, t_r, scale)
    dl, dr = s_l.cuda().requires_grad_(True), s_r.cuda().requires_grad_(True)
    tl, tr = (None, None) if alias else (t_l.cuda(), t_r.cuda())
    ll, lr = eng.cps_cross_entropy(dl, dr, tl, tr, loss_scale=scale, unit_upstream=True)
    assert ll.dim() == 0 and lr.dim() == 0
    assert rel(ll, ll_ref) <= 1e-6 and rel(lr, lr_ref) <= 1e-6
    gl, gr = torch.autograd.grad(ll + lr, (dl, dr))
    assert rel(gl, gl_ref) <= 1e-6 and rel(gr, gr_ref) <= 1e-6
    # exact pseudo-labels (first maximal index on ties): l learns towards argmax t_r, r towards argmax t_l
    assert torch.equal(_labels_from_grad(gl), y_r) and torch.equal(_labels_from_grad(gr), y_l)
    # per-sample rows of the raw launch, and bit-identical repeats
    tl_, tr_ = (dl.detach(), dr.detach()) if alias else (tl, tr)
    per, g1, g2 = eng.cps_raw(dl.detach(), dr.detach(), tl_, tr_, scale / n, True)
    assert rel(per, per_ref) <= 1e-6
    per2, g1b, g2b = eng.cps_raw(dl.detach(), dr.detach(), tl_, tr_, scale / n, True)
    assert torch.equal(per, per2) and torch.equal(g1, g1b) and torch.equal(g2, g2b)
    assert torch.equal(g1, gl) and torch.equal(g2, gr)
    # loss only: same losses, no gradient buffers
    per3, none_l, none_r = eng.cps_raw(dl.detach(), dr.detach(), tl_, tr_, scale / n, False)
    assert none_l is None and none_r is None and torch.equal(per, per3)


@pytest.mark.parametrize('alias', [True, False])
def test_cps_backward_scales_by_the_upstream_gradients(eng, alias):
    g = torch.Generator().manual_seed(5)
    s_l, s_r = _logits(g, 3, 21, 33, 47), _logits(g, 3, 21, 33, 47)
    t_l, t_r = (s_l, s_r) if alias else (_logits(g, 3, 21, 33, 47), _logits(g, 3, 21, 33, 47))
    _, ll_ref, lr_ref, gl_ref, gr_ref, _, _ = _reference(s_l, s_r, t_l, t_r, 0.8, w_l=2.5, w_r=-0.25)
    dl, dr = s_l.cuda().requires_grad_(True), s_r.cuda().requires_grad_(True)
    tl, tr = (None, None) if alias else (t_l.cuda(), t_r.cuda())
    ll, lr = eng.cps_cross_entropy(dl, dr, tl, tr, loss_scale=0.8)
    gl, gr = torch.autograd.grad(2.5 * ll - 0.25 * lr, (dl, dr))
    assert rel(ll, ll_ref) <= 1e-6 and rel(lr, lr_ref) <= 1e-6
    assert rel(gl, gl_ref) <= 1e-6 and rel(gr, gr_ref) <= 1e-6
    with torch.no_grad():
        a, b = eng.cps_cross_entropy(dl, dr, tl, tr, loss_scale=0.8)
    assert torch.equal(a, ll) and torch.equal(b, lr)


def test_cps_rejects_unsupported_inputs(eng):
    from pixelssl_b200 import _lib
    x = torch.randn(2, 33, 5, 5, device='cuda')
    with pytest.raises(_lib.PxlError):
        eng.cps_cross_entropy(x, x.clone())                                # C = 33 > 32
    y = torch.randn(2, 21, 5, 6, device='cuda')
    with pytest.raises(ValueError):
        eng.cps_cross_entropy(y[..., :5], y[..., 1:])                      # not contiguous
    with pytest.raises(ValueError):
        eng.cps_cross_entropy(y, y.clone(), t_l=torch.randn(2, 21, 6, 5, device='cuda'), t_r=y)   # shape mismatch
    with pytest.raises(TypeError):
        eng.cps_cross_entropy(y, y.double())                              # not fp32


# ---- whole steps against the oracle ----------------------------------------------------------------------------------

def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


_ORACLE_CACHE = {}


def _oracle_step(kind):
    """The CPS oracle step (DeepLab-v2-R101, 65x65) in fp32 and fp64, cached across the precision modes."""
    if kind not in _ORACLE_CACHE:
        lbs, ubs = 2, (2 if kind == 'plain' else 4)
        img, lab = O.synthetic_batch(81, lbs + ubs, lbs, 65, 65)
        l0 = O.randomize_bn_affine(O.init_deeplabv2(83, cls_bias_std=0.01), 84)
        r0 = O.randomize_bn_affine(O.init_deeplabv2(85, cls_bias_std=0.01), 86)
        out = []
        for dt in (torch.float32, torch.float64):
            l, r = (O.to_dtype(O.to_dtype(s, torch.float64), dt) for s in (l0, r0))
            cps = C.CPSOracle(l, r, lr=0.00025, max_iters=10, cps_scale=1.5, rampup_steps=0, cutmix=(kind == 'cutmix'))
            res = cps.step(img.to(dt), lab.to(dt), lbs, np.random.RandomState(MASK_SEED))
            out.append({'loss': {k: float(v) for k, v in res.items() if k.endswith('_loss')},
                        'energy': {s: _energies(res[s + '_grads'], cps.names) for s in 'lr'}, 'names': cps.names})
        _ORACLE_CACHE[kind] = (img, lab, l0, r0, lbs, ubs, out[0], out[1])
    return _ORACLE_CACHE[kind]


def _build(cfg):
    from pixelssl_b200 import runner
    return runner.build_algorithm(runner.build_args(dict(BASE, **cfg), iters_per_epoch=5))


def _load(model, state):
    model.load_state_dict({'module.model.' + k: v for k, v in state.items()}, strict=True)


@pytest.mark.parametrize('kind', ['plain', 'cutmix'])
def test_step_matches_oracle(ops, kind):
    img, lab, l0, r0, lbs, ubs, r32, r64 = _oracle_step(kind)
    alg = _build(dict(PAIR, batch_size=lbs + ubs, unlabeled_batch_size=ubs, cps_cutmix=(kind == 'cutmix')))
    _load(alg.l_model, l0)
    _load(alg.r_model, r0)
    np.random.seed(MASK_SEED)
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    for key in ('l_task_loss', 'r_task_loss', 'l_cps_loss', 'r_cps_loss'):
        got = float(alg.meters[key].val)
        print('%s %s: engine %.8g oracle fp32 %.8g fp64 %.8g' % (kind, key, got, r32['loss'][key], r64['loss'][key]))
        assert_loss_yardstick(got, r32['loss'][key], r64['loss'][key], '%s %s' % (kind, key))
    for side, model in (('l', alg.l_model), ('r', alg.r_model)):
        sp = dict(model.module.model.named_parameters())
        got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in r64['names']])
        print(assert_energy_yardstick(got, r32['energy'][side], r64['energy'][side], '%s %s grad energies' % (kind, side)))


# ---- end to end ------------------------------------------------------------------------------------------------------

def _cfg(model, cutmix):
    cfg = dict(BASE, models={'model': model}, cps_cutmix=cutmix)
    if cutmix:
        cfg.update(batch_size=6, unlabeled_batch_size=4)      # the mixed half of the unlabeled rows is a batch of 2
    else:
        cfg.update(batch_size=4, unlabeled_batch_size=2)
    return cfg


@pytest.mark.parametrize('model', ['deeplabv2', 'pspnet', 'deeplabv3plus'])
@pytest.mark.parametrize('cutmix', [False, True])
def test_trains_validates_and_checkpoints(eng, model, cutmix, tmp_path):
    from pixelssl_b200 import runner
    eng.set_conv_precision('f16x3')
    try:
        cfg = _cfg(model, cutmix)
        args = runner.build_args(cfg, iters_per_epoch=5)
        args.checkpoint_path = str(tmp_path)
        torch.manual_seed(0)
        np.random.seed(0)
        alg = runner.build_algorithm(args)
        assert set(alg.models) == {'l_model', 'r_model'}
        assert not torch.equal(alg.l_model.arena.data, alg.r_model.arena.data)      # independent initialisations
        img, lab = O.synthetic_batch(71, cfg['batch_size'], cfg['batch_size'] - cfg['unlabeled_batch_size'], 65, 65)
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
        losses = {k: float(alg.meters[k].val) for k in ('l_task_loss', 'r_task_loss', 'l_cps_loss', 'r_cps_loss')}
        assert all(np.isfinite(v) for v in losses.values()) and losses['l_cps_loss'] > 0, losses
        vimg, vlab = O.synthetic_batch(72, 2, 2, 65, 65)
        alg._validate([((vimg,), (vlab,))], 0)
        metrics = {k: float(alg.meters[k].val) for k in alg.meters.keys() if '_metric_' in k}
        assert metrics and all(np.isfinite(v) for v in metrics.values()), metrics
        assert any(k.startswith('l_') for k in metrics) and any(k.startswith('r_') for k in metrics)
        alg.save_checkpoint(1)
        path = os.path.join(str(tmp_path), 'checkpoint_1.ckpt')
        ck = torch.load(path, weights_only=False)
        assert set(ck) == {'algorithm', 'epoch', 'l_model', 'r_model', 'l_optimizer', 'r_optimizer', 'l_lrer', 'r_lrer'}
        alg2 = runner.build_algorithm(args)
        args.resume = path
        assert alg2.load_checkpoint() == 1
        for key, mod in alg.models.items():
            a, b = mod.state_dict(), alg2.models[key].state_dict()
            assert list(a) == list(b) and all(k.startswith('module.') for k in a)
            for k in a:
                assert torch.equal(a[k].cpu(), b[k].cpu()), (key, k)
        for key in ('l_optimizer', 'r_optimizer'):
            sa, sb = getattr(alg, key).state_dict(), getattr(alg2, key).state_dict()
            assert sa['param_groups'] == sb['param_groups']
            for i, st in sa['state'].items():
                assert torch.equal(st['momentum_buffer'].cpu(), sb['state'][i]['momentum_buffer'].cpu()), (key, i)
        for key in ('l_lrer', 'r_lrer'):
            assert getattr(alg, key).state_dict() == getattr(alg2, key).state_dict()
    finally:
        eng.set_conv_precision('fp32')


@pytest.mark.parametrize('cutmix', [False, True])
def test_one_cps_launch_per_step_and_no_ffma_convolutions(eng, cutmix):
    """A spy on ops.call (as in test_gpu_deeplabv3plus.test_head_runs_on_tensor_cores): one fused CPS launch per step
    and, in f16x3, no FFMA convolution launch."""
    seen = []
    real = eng.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)

    eng.set_conv_precision('f16x3')
    try:
        cfg = _cfg('deeplabv3plus', cutmix)
        alg = _build(cfg)
        img, lab = O.synthetic_batch(61, cfg['batch_size'], cfg['batch_size'] - cfg['unlabeled_batch_size'], 97, 97)
        eng.call = spy
        alg._train([((img,), (lab,)), ((img,), (lab,))], 0)
        torch.cuda.synchronize()
    finally:
        eng.call = real
        eng.set_conv_precision('fp32')
    assert seen.count('pxl_cps_ce') == 2
    assert not [s for s in seen if s in ('pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc')]
    assert set(seen) & {'pxl_conv_h16_launch', 'pxl_conv_tc_launch_ex'}


def test_plain_steps_are_bit_identical(eng):
    """Two plain steps from the same states on the same batch leave bit-identical parameters in both arenas."""
    img, lab = O.synthetic_batch(91, 4, 2, 65, 65)
    l0 = O.randomize_bn_affine(O.init_deeplabv2(93, cls_bias_std=0.01), 94)
    r0 = O.randomize_bn_affine(O.init_deeplabv2(95, cls_bias_std=0.01), 96)
    eng.set_conv_precision('f16x3')
    try:
        after = []
        for _ in range(2):
            alg = _build(dict(PAIR, batch_size=4, unlabeled_batch_size=2))
            _load(alg.l_model, l0)
            _load(alg.r_model, r0)
            alg._train([((img,), (lab,))], 0)
            torch.cuda.synchronize()
            after.append((alg.l_model.arena.data.clone(), alg.r_model.arena.data.clone()))
            del alg
    finally:
        eng.set_conv_precision('fp32')
    assert torch.equal(after[0][0], after[1][0]) and torch.equal(after[0][1], after[1][1])
    assert not torch.equal(after[0][0], after[0][1])
