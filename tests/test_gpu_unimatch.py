"""UniMatch on the engine: the strong augmentation (pxl_strong_aug) against torchvision in fp64, the feature
perturbation op (fp_dup), the fused loss (pxl_unimatch_ce) against torch in fp64, the whole step against the CPU
oracle (oracle/unimatch_oracle.py) evaluated in fp32 and fp64, ssl_unimatch end to end with each supported task
model, its launches, and the step's determinism."""
import os

import numpy as np
import pytest
import torch

from oracle import sseg_oracle as O
from oracle import deeplabv3plus_oracle as D
from oracle import unimatch_oracle as U

from conftest import TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
BASE = {'ssl_algorithm': 'ssl_unimatch', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'log_freq': 1000, 'uni_threshold': 0.5, 'uni_scale': 1.0, 'uni_rampup_epochs': 0}
MEAN = torch.tensor(U.MEAN, dtype=torch.float64).view(1, 3, 1, 1)
STD = torch.tensor(U.STD, dtype=torch.float64).view(1, 3, 1, 1)


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


# ---- the strong augmentation -----------------------------------------------------------------------------------------

def _weak(seed, ubs, h, w):
    """normalised images whose [0, 1] values reach slightly past both ends (the clamp) and hold gray pixels"""
    g = torch.Generator().manual_seed(seed)
    x01 = torch.rand(ubs, 3, h, w, generator=g, dtype=torch.float64) * 1.1 - 0.05
    x01[:, :, ::7, ::5] = x01[:, :1, ::7, ::5]                      # r == g == b: hue's degenerate branch
    return ((x01 - MEAN) / STD).float()


def _row(jitter=None, order=(0, 1, 2, 3), gray=False, sigma=None, box=None):
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import gaussian_weights
    r = np.zeros(32, dtype=np.float64)
    r[5:9] = order
    if jitter is not None:
        r[0] = 1.0
        r[1:5] = jitter
    r[9] = float(gray)
    if sigma is not None:
        wts = gaussian_weights(sigma)
        r[10], r[11] = (len(wts) - 1) // 2, sigma
        r[16:16 + len(wts)] = wts
    if box is not None:
        r[12:16] = box
    return r


AUG_ROWS = {
    'identity': _row(),
    'brightness': _row((1.4, 1.0, 1.0, 0.0), order=(0, 1, 2, 3)),
    'contrast': _row((1.0, 0.6, 1.0, 0.0), order=(1, 0, 2, 3)),
    'saturation': _row((1.0, 1.0, 1.45, 0.0), order=(2, 0, 1, 3)),
    'hue': _row((1.0, 1.0, 1.0, -0.22), order=(3, 0, 1, 2)),
    'order_bcsh': _row((0.7, 1.3, 0.6, 0.17), order=(0, 1, 2, 3)),
    'order_hscb': _row((1.2, 0.55, 1.4, -0.09), order=(3, 2, 1, 0)),
    'order_shbc': _row((0.9, 1.45, 0.5, 0.24), order=(2, 3, 0, 1)),
    'grayscale': _row(gray=True),
    'jitter_gray': _row((1.1, 0.8, 1.2, 0.1), order=(1, 3, 0, 2), gray=True),
    'blur_0.1': _row(sigma=0.1),
    'blur_2.0': _row(sigma=2.0),
    'all': _row((0.8, 1.2, 1.3, -0.2), order=(2, 1, 3, 0), gray=False, sigma=1.3),
}


def _to01(x):
    return x.double().cpu() * STD + MEAN


def _check_views(eng, weak, table, what):
    got, _ = eng.strong_aug(weak.cuda(), torch.from_numpy(table))
    want = U.strong_views(weak.double(), table)
    err = float((_to01(got) - _to01(want)).abs().max())
    print('%s: max |engine - torchvision fp64| in [0, 1] space = %.2e' % (what, err))
    assert err <= 3e-6, (what, err)
    return got


@pytest.mark.parametrize('name', sorted(AUG_ROWS))
def test_strong_aug_single_ops_match_torchvision(eng, name):
    """Each op alone or in a drawn order, on view 1 of image 0; the other views are identities, no boxes."""
    ubs = 2
    table = np.stack([AUG_ROWS['identity']] * (2 * ubs))
    table[0] = AUG_ROWS[name]
    table[3] = AUG_ROWS[name]
    _check_views(eng, _weak(1, ubs, 37, 45), table.astype(np.float32), name)


def test_strong_aug_drawn_tables_boxes_and_repeats(eng):
    """Drawn tables (every box coin, including boxes that touch an edge or are missing) on a 4-image batch; box
    pixels are bit-exact copies of the partner's view without boxes; repeated calls are bit-identical."""
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params
    ubs, h, w = 4, 65, 71
    weak = _weak(2, ubs, h, w)
    table, boxes = draw_strong_params(ubs, h, w, 1.0, rng=np.random.RandomState(11))
    boxes[1] = (0, 0, 20, 15)              # corner box
    boxes[2] = (40, 50, h, w)              # box to the bottom-right edges
    boxes[5] = (0, 0, 0, 0)                # missing
    table[:, 12:16] = boxes
    got = _check_views(eng, weak, table, 'drawn table')
    again, _ = eng.strong_aug(weak.cuda(), torch.from_numpy(table))
    assert torch.equal(got, again)
    plain = table.copy()
    plain[:, 12:16] = 0
    unpasted, _ = eng.strong_aug(weak.cuda(), torch.from_numpy(plain))
    for v in range(2 * ubs):
        k, i = divmod(v, ubs)
        y0, x0, y1, x1 = boxes[v]
        inside = torch.zeros(h, w, dtype=torch.bool, device='cuda')
        inside[y0:y1, x0:x1] = True
        src = unpasted[k * ubs + (i + ubs // 2) % ubs]
        assert torch.equal(got[v][:, inside], src[:, inside])
        assert torch.equal(got[v][:, ~inside], unpasted[v][:, ~inside])


def test_strong_aug_full_size_batch(eng):
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params
    ubs, h, w = 8, 513, 513
    weak = _weak(3, ubs, h, w)
    table, _ = draw_strong_params(ubs, h, w, 0.5, rng=np.random.RandomState(5))
    got = _check_views(eng, weak, table, '513x513 batch of 8')
    again, _ = eng.strong_aug(weak.cuda(), torch.from_numpy(table))
    assert torch.equal(got, again)


# ---- feature perturbation --------------------------------------------------------------------------------------------

@pytest.mark.parametrize('shape', [(2, 256, 17, 17), (3, 2048, 5, 5), (4, 64, 1, 3)])
def test_fp_dup_forward_is_bit_exact_and_backward_matches_torch(eng, shape):
    n, c, h, w = shape
    g = torch.Generator().manual_seed(c + h)
    x = torch.randn(shape, generator=g).cuda().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    scale = ((torch.rand(n, c, generator=g) > 0.5).float() / 0.5).cuda()
    out = eng.fp_dup(x, scale)
    assert out.shape == (2 * n, c, h, w) and out.is_contiguous(memory_format=torch.channels_last)
    ref = torch.cat([x.detach(), x.detach() * scale[:, :, None, None]])
    assert torch.equal(out, ref)
    up = torch.randn(2 * n, c, h, w, generator=g).cuda()
    (dx,) = torch.autograd.grad(out, x, grad_outputs=up)
    want = up[:n] + up[n:] * scale[:, :, None, None]
    assert torch.allclose(dx, want, rtol=0, atol=0), float((dx - want).abs().max())
    with pytest.raises(ValueError):
        eng.fp_dup(x.detach(), scale[:, :c // 2])


# ---- the fused loss --------------------------------------------------------------------------------------------------

def _logits(g, n, c, h, w, spread=1.0):
    x = torch.randn(n, c, h, w, generator=g) * spread
    q = torch.randint(-2, 3, (n, c, h, w), generator=g).float() * 0.75
    tied = (torch.arange(h * w).reshape(h, w) % 3 == 0)
    return torch.where(tied, q, x)


def _reference(w, mix, s, fp_all, lbs, boxes, tau, weights):
    """fp64 torch: the three losses, the count and the gradients of sum(weights * losses)."""
    sd, fd = s.double().requires_grad_(True), fp_all.double().requires_grad_(True)
    l1, l2, lf, cnt = U.unimatch_terms(w.double(), mix.double(), sd, fd[lbs:], boxes, tau)
    gs, gf = torch.autograd.grad(weights[0] * l1 + weights[1] * l2 + weights[2] * lf, (sd, fd), allow_unused=True)
    gs = torch.zeros_like(sd) if gs is None else gs
    gf = torch.zeros_like(fd) if gf is None else gf
    return (l1.detach(), l2.detach(), lf.detach()), int(cnt), gs, gf


def _gap_threshold(conf, others=None):
    """A threshold in the widest gap, between the 40 % and 60 % quantiles of ``conf``, of the values of ``conf`` and
    ``others`` together (no value of either lies in the gap) -> (threshold, gap width)."""
    conf = conf.flatten().double().numpy()
    lo, hi = np.quantile(conf, [0.4, 0.6])
    v = np.sort(conf if others is None else np.concatenate([conf, others.flatten().double().numpy()]))
    gaps, mids = np.diff(v), (v[1:] + v[:-1]) / 2
    k = int(np.argmax(np.where((mids >= lo) & (mids <= hi), gaps, -1.0)))
    return float(mids[k]), float(gaps[k])


BOX_KINDS = {'empty': [(0, 0, 0, 0)] * 4, 'partial': [(3, 5, 20, 17), (0, 0, 9, 9), (10, 30, 33, 47), (0, 0, 0, 0)],
             'whole': [(0, 0, 33, 47)] * 4}
CE_CASES = [(c, kind, tau) for c in (2, 21, 32) for kind in sorted(BOX_KINDS) for tau in ('zero', 'gap', 'above_one')]


@pytest.mark.parametrize('c,kind,tau', CE_CASES)
def test_unimatch_kernel_matches_torch_fp64(eng, c, kind, tau):
    ubs, lbs, h, w = 2, 3, 33, 47
    g = torch.Generator().manual_seed(c * 100 + len(kind))
    wk = _logits(g, ubs, c, h, w, spread=3.0 / c ** 0.5)
    mix = _logits(g, ubs, c, h, w, spread=3.0 / c ** 0.5)
    s = _logits(g, 2 * ubs, c, h, w)
    fp_all = _logits(g, lbs + ubs, c, h, w)
    boxes = torch.tensor(BOX_KINDS[kind], dtype=torch.int32)
    if tau == 'zero':
        t = 0.0
    elif tau == 'above_one':
        t = 1.01
    else:
        conf = torch.cat([U.pseudo_labels(wk.double())[1], U.pseudo_labels(mix.double())[1]])
        t, gap = _gap_threshold(conf)
        assert gap > 1e-6, gap
    weights = (0.3, 0.45, 0.7)
    (r1, r2, rf), rcnt, gs_ref, gf_ref = _reference(wk, mix, s, fp_all, lbs, boxes, t, weights)
    ds, dfp = s.cuda().requires_grad_(True), fp_all.cuda().requires_grad_(True)
    l1, l2, lf, cnt = eng.unimatch_cross_entropy(ds, dfp, wk.cuda(), mix.cuda(), boxes, t, weights=weights,
                                                 fp_offset=lbs, unit_upstream=True)
    assert int(cnt) == rcnt
    if tau == 'zero':
        assert rcnt == ubs * h * w
    if tau == 'above_one':
        assert rcnt == 0 and float(l1) == float(l2) == float(lf) == 0.0
    for a, b in ((l1, r1), (l2, r2), (lf, rf)):
        assert abs(float(a) - float(b)) <= 1e-6 * max(abs(float(b)), 1e-30) or float(b) == float(a) == 0.0
    gs, gf = torch.autograd.grad(weights[0] * l1 + weights[1] * l2 + weights[2] * lf, (ds, dfp))
    assert float((gs.double().cpu() - gs_ref).abs().max()) <= 1e-6 * max(float(gs_ref.abs().max()), 1e-30)
    assert float((gf.double().cpu() - gf_ref).abs().max()) <= 1e-6 * max(float(gf_ref.abs().max()), 1e-30)
    assert not gf[:lbs].any()
    # bit-identical repeats of the raw launch, and the same gradients as the autograd path
    out, g1, g2 = eng.unimatch_raw(wk.cuda(), mix.cuda(), ds.detach(), dfp.detach(), lbs, boxes, t, weights, ubs // 2)
    out2, g1b, g2b = eng.unimatch_raw(wk.cuda(), mix.cuda(), ds.detach(), dfp.detach(), lbs, boxes, t, weights, ubs // 2)
    assert torch.equal(out, out2) and torch.equal(g1, g1b) and torch.equal(g2, g2b)
    assert torch.equal(g1, gs) and torch.equal(g2, gf)


@pytest.mark.parametrize('c', [2, 32])
def test_unimatch_threshold_edge_counts_equal_confidences(eng, c):
    """All channels tied: the confidence is exactly 1/C and a threshold of exactly 1/C keeps every pixel."""
    ubs, h, w = 2, 5, 9
    wk = torch.full((ubs, c, h, w), 0.25)
    s = torch.randn(2 * ubs, c, h, w).cuda()
    fp_all = torch.randn(ubs, c, h, w).cuda()
    boxes = torch.zeros(2 * ubs, 4, dtype=torch.int32)
    for t, want in ((1.0 / c, ubs * h * w), (np.nextafter(np.float32(1.0 / c), np.float32(1)), 0)):
        l1, l2, lf, cnt = eng.unimatch_cross_entropy(s, fp_all, wk.cuda(), wk.cuda(), boxes, float(t))
        assert int(cnt) == want, (t, int(cnt))


def test_unimatch_non_unit_upstream_scales_by_the_upstream_gradients(eng):
    ubs, lbs, c, h, w = 2, 1, 21, 17, 19
    g = torch.Generator().manual_seed(9)
    wk, mix = _logits(g, ubs, c, h, w, 0.6), _logits(g, ubs, c, h, w, 0.6)
    s, fp_all = _logits(g, 2 * ubs, c, h, w), _logits(g, lbs + ubs, c, h, w)
    boxes = torch.tensor(BOX_KINDS['partial'], dtype=torch.int32)
    weights = (2.5, -0.25, 0.75)
    _, _, gs_ref, gf_ref = _reference(wk, mix, s, fp_all, lbs, boxes, 0.0, weights)
    ds, dfp = s.cuda().requires_grad_(True), fp_all.cuda().requires_grad_(True)
    l1, l2, lf, _ = eng.unimatch_cross_entropy(ds, dfp, wk.cuda(), mix.cuda(), boxes, 0.0)
    gs, gf = torch.autograd.grad(weights[0] * l1 + weights[1] * l2 + weights[2] * lf, (ds, dfp))
    assert rel(gs, gs_ref) <= 1e-6 and rel(gf, gf_ref) <= 1e-6


def test_unimatch_rejects_unsupported_inputs(eng):
    from pixelssl_b200 import _lib
    boxes = torch.zeros(4, 4, dtype=torch.int32)
    x = torch.randn(2, 33, 5, 5, device='cuda')
    with pytest.raises(_lib.PxlError):                                  # C = 33 > 32
        eng.unimatch_cross_entropy(torch.randn(4, 33, 5, 5, device='cuda'), x.clone(), x, x, boxes, 0.5)
    y = torch.randn(2, 21, 5, 6, device='cuda')
    s = torch.randn(4, 21, 5, 5, device='cuda')
    with pytest.raises(ValueError):                                     # not contiguous
        eng.unimatch_cross_entropy(s, y[..., :5], y[..., 1:], y[..., 1:].contiguous(), boxes, 0.5)
    with pytest.raises(ValueError):                                     # shape mismatch
        eng.unimatch_cross_entropy(s, y, y, y, boxes, 0.5)
    z = torch.randn(2, 21, 5, 5, device='cuda')
    with pytest.raises(TypeError):                                      # not fp32
        eng.unimatch_cross_entropy(s.double(), z, z, z, boxes, 0.5)
    with pytest.raises(TypeError):                                      # not on the GPU
        eng.unimatch_cross_entropy(s.cpu(), z.cpu(), z.cpu(), z.cpu(), boxes, 0.5)
    with pytest.raises(ValueError):                                     # one box per strong view
        eng.unimatch_cross_entropy(s, z, z, z, boxes[:3], 0.5)


# ---- the whole step against the oracle -------------------------------------------------------------------------------

def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


DRAW_SEED, TORCH_SEED = 2024, 77
_ORACLE_CACHE = {}


def _init(model, seed, img):
    """A random-init state whose BatchNorm running statistics are the batch statistics of one training-mode forward
    of ``img`` (momentum 1), as a trained network's are.  The step's eval-mode forward then stays in range; with the
    initial running statistics (mean 0, variance 1) the activations of a random-init ResNet grow past what the
    fp16-pair convolutions hold, which no pretrained network does."""
    if model == 'deeplabv2':
        st, fwd = O.randomize_bn_affine(O.init_deeplabv2(seed, cls_bias_std=0.01), seed + 1), O.deeplabv2_forward
    else:
        st, fwd = O.randomize_bn_affine(D.init(seed, cls_bias_std=0.01), seed + 1), D.forward
    saved = O.batch_norm.__defaults__
    O.batch_norm.__defaults__ = (1.0,) + saved[1:]
    try:
        with torch.no_grad():
            fwd(img, st, True)
    finally:
        O.batch_norm.__defaults__ = saved
    return st


def _draws(model, lbs, ubs, h, w):
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params, draw_fp_scales
    table, boxes = draw_strong_params(ubs, h, w, 0.5, rng=np.random.RandomState(DRAW_SEED))
    torch.manual_seed(TORCH_SEED)
    chans = (2048,) if model == 'deeplabv2' else (256, 2048)
    return table, boxes, draw_fp_scales(lbs + ubs, chans, 0.5)


def _oracle_step(eng, model):
    """The UniMatch oracle step (R101, 65x65, 2 + 2 images) in fp32 and fp64 on the engine's strong views, with the
    threshold in the widest gap of the middle of the fp64 confidences."""
    if model not in _ORACLE_CACHE:
        lbs, ubs, h, w = 2, 2, 65, 65
        img, lab = O.synthetic_batch(81, lbs + ubs, lbs, h, w)
        st0 = _init(model, 83, img)
        table, boxes, scales = _draws(model, lbs, ubs, h, w)
        strong = eng.strong_aug(img[lbs:].contiguous().cuda(), torch.from_numpy(table))[0].cpu()
        probe = U.UniMatchOracle(O.to_dtype(O.to_dtype(st0, torch.float64), torch.float64), model=model, max_iters=10,
                                 threshold=0.5)
        mix = probe.mix_source(img[lbs:].double())
        res = probe.step(img.double(), lab.double(), lbs, table, boxes, [s.double() for s in scales], strong)
        tau, gap = _gap_threshold(U.pseudo_labels(res['pred_u'])[1], U.pseudo_labels(mix)[1])
        out = []
        for dt in (torch.float32, torch.float64):
            orc = U.UniMatchOracle(O.to_dtype(O.to_dtype(st0, torch.float64), dt), model=model, max_iters=10,
                                   threshold=tau)
            r = orc.step(img.to(dt), lab.to(dt), lbs, table, boxes, [s.to(dt) for s in scales], strong)
            out.append({'loss': {k: float(r[k]) for k in ('task_loss', 's1_loss', 's2_loss', 'fp_loss')},
                        'ratio': r['mask_ratio'], 'energy': _energies(r['grads'], orc.names), 'names': orc.names})
        _ORACLE_CACHE[model] = (img, lab, st0, lbs, ubs, tau, gap, out[0], out[1])
    return _ORACLE_CACHE[model]


def _build(cfg):
    from pixelssl_b200 import runner
    return runner.build_algorithm(runner.build_args(dict(BASE, **cfg), iters_per_epoch=5))


def _load(model, state):
    model.load_state_dict({'module.model.' + k: v for k, v in state.items()}, strict=True)


@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_step_matches_oracle(ops, model):
    img, lab, st0, lbs, ubs, tau, gap, r32, r64 = _oracle_step(ops, model)
    alg = _build(dict(models={'model': model}, batch_size=lbs + ubs, unlabeled_batch_size=ubs, uni_threshold=tau))
    _load(alg.model, st0)
    np.random.seed(DRAW_SEED)
    torch.manual_seed(TORCH_SEED)
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    print('%s: tau %.9f in a gap of %.2e; mask ratio engine %.6f oracle fp64 %.6f' % (
        model, tau, gap, float(alg.meters['mask_ratio'].val), r64['ratio']))
    assert 0.3 <= r64['ratio'] <= 0.7
    assert abs(float(alg.meters['mask_ratio'].val) - r64['ratio']) <= 2e-3
    for key in ('task_loss', 's1_loss', 's2_loss', 'fp_loss'):
        got = float(alg.meters[key].val)
        print('%s %s: engine %.8g oracle fp32 %.8g fp64 %.8g' % (model, key, got, r32['loss'][key], r64['loss'][key]))
        assert_loss_yardstick(got, r32['loss'][key], r64['loss'][key], '%s %s' % (model, key))
    sp = dict(alg.model.module.model.named_parameters())
    got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in r64['names']])
    print(assert_energy_yardstick(got, r32['energy'], r64['energy'], '%s grad energies' % model))


# ---- end to end ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_trains_validates_checkpoints_and_resumes(eng, model, tmp_path):
    from pixelssl_b200 import runner
    eng.set_conv_precision('f16x3')
    try:
        cfg = dict(BASE, models={'model': model}, batch_size=4, unlabeled_batch_size=2, uni_threshold=0.0)
        args = runner.build_args(cfg, iters_per_epoch=5)
        args.checkpoint_path = str(tmp_path)
        torch.manual_seed(0)
        np.random.seed(0)
        alg = runner.build_algorithm(args)
        assert set(alg.models) == {'model'}
        img, lab = O.synthetic_batch(71, 4, 2, 65, 65)
        _load(alg.model, _init(model, 73, img))
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
        losses = {k: float(alg.meters[k].val) for k in ('task_loss', 's1_loss', 's2_loss', 'fp_loss', 'mask_ratio')}
        assert all(np.isfinite(v) for v in losses.values()) and losses['s1_loss'] > 0, losses
        assert losses['mask_ratio'] == 1.0                     # threshold 0: every pixel
        vimg, vlab = O.synthetic_batch(72, 2, 2, 65, 65)
        alg._validate([((vimg,), (vlab,))], 0)
        metrics = {k: float(alg.meters[k].val) for k in alg.meters.keys() if '_metric_' in k}
        assert metrics and all(np.isfinite(v) for v in metrics.values()), metrics
        alg.save_checkpoint(1)
        path = os.path.join(str(tmp_path), 'checkpoint_1.ckpt')
        ck = torch.load(path, weights_only=False)
        assert set(ck) == {'algorithm', 'epoch', 'model', 'optimizer', 'lrer'}
        alg2 = runner.build_algorithm(args)
        args.resume = path
        assert alg2.load_checkpoint() == 1
        a, b = alg.model.state_dict(), alg2.model.state_dict()
        assert list(a) == list(b)
        for k in a:
            assert torch.equal(a[k].cpu(), b[k].cpu()), k
        sa, sb = alg.optimizer.state_dict(), alg2.optimizer.state_dict()
        assert sa['param_groups'] == sb['param_groups']
        for i, st in sa['state'].items():
            assert torch.equal(st['momentum_buffer'].cpu(), sb['state'][i]['momentum_buffer'].cpu()), i
        assert alg.lrer.state_dict() == alg2.lrer.state_dict()
        alg2._train([((img,), (lab,))], 1)                     # the resumed run trains on
        torch.cuda.synchronize()
        assert np.isfinite(float(alg2.meters['s1_loss'].val))
    finally:
        eng.set_conv_precision('fp32')


def test_one_unimatch_launch_per_step_and_no_ffma_convolutions(eng):
    seen = []
    real = eng.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)

    eng.set_conv_precision('f16x3')
    try:
        alg = _build(dict(models={'model': 'deeplabv3plus'}, batch_size=4, unlabeled_batch_size=2))
        img, lab = O.synthetic_batch(61, 4, 2, 97, 97)
        _load(alg.model, _init('deeplabv3plus', 63, img))
        eng.call = spy
        alg._train([((img,), (lab,)), ((img,), (lab,))], 0)
        torch.cuda.synchronize()
    finally:
        eng.call = real
        eng.set_conv_precision('fp32')
    assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
    assert seen.count('pxl_unimatch_ce') == 2
    assert seen.count('pxl_strong_aug') == 2
    assert not [s for s in seen if s in ('pxl_conv_nhwc', 'pxl_conv_wgrad_nhwc')]
    assert set(seen) & {'pxl_conv_h16_launch', 'pxl_conv_tc_launch_ex'}


@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus'])
def test_steps_are_bit_identical(eng, model):
    """Two steps from the same state on the same batch with the same seeds leave bit-identical parameters."""
    img, lab = O.synthetic_batch(91, 4, 2, 65, 65)
    st0 = _init(model, 93, img)
    eng.set_conv_precision('f16x3')
    try:
        after = []
        for _ in range(2):
            alg = _build(dict(models={'model': model}, batch_size=4, unlabeled_batch_size=2))
            _load(alg.model, st0)
            np.random.seed(3)
            torch.manual_seed(4)
            alg._train([((img,), (lab,))], 0)
            torch.cuda.synchronize()
            after.append(alg.model.arena.data.clone())
            del alg
    finally:
        eng.set_conv_precision('fp32')
    assert torch.equal(after[0], after[1])
