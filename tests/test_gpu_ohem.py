"""OHEM cross-entropy on the engine: the q map and the exact device-side selection of pxl_ohem_ce against torch, the
loss and both gradient paths against the fp64 oracle (oracle/ohem_oracle.py), determinism, no host synchronisation,
and whole Mean-Teacher, CPS and UniMatch steps with ohem_sseg_criterion against the step oracles in fp32 and fp64."""
import math

import numpy as np
import pytest
import torch

from oracle import cps_oracle as C
from oracle import deeplabv3plus_oracle as D
from oracle import ohem_oracle as H
from oracle import sseg_oracle as O
from oracle import unimatch_oracle as U

from conftest import TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

pytestmark = pytest.mark.gpu
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000}


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


def _maps(seed, n, c, h, w, spread=2.0, ignore_frac=0.1):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, c, h, w, generator=g) * spread
    labels = torch.randint(0, c, (n, 1, h, w), generator=g).float()
    labels[torch.rand(n, 1, h, w, generator=g) < ignore_frac] = 255
    return logits.cuda(), labels.cuda()


def _ulps(a, b):
    a, b = a.float().cpu().view(torch.int32).long(), b.float().cpu().view(torch.int32).long()
    return int((a - b).abs().max())


def _check_selection(eng, logits, labels, k, thresh=-1.0):
    """The kernel's stats against torch.sort / the oracle's rule on the kernel's own q map -> (q, stats, sel)."""
    per, grad, q, stats = eng.ohem_raw(logits, labels, 255, thresh, k)
    stats = stats.cpu().tolist()
    valid = H.q_map(logits.double(), labels.double())[1]
    sel = H.select(q.double(), valid, thresh, k)
    V = int(valid.sum())
    assert stats[0] == V
    if 0 < k <= V:
        want = torch.sort(q.flatten())[0][k - 1]
        if math.isnan(float(want)):
            assert math.isnan(stats[3]) or bool(want.cpu() <= thresh)
        elif not bool(want <= thresh):                 # not an early exit: t_k was selected
            assert torch.tensor(stats[3], dtype=torch.float32).view(torch.int32) == want.cpu().view(torch.int32), (
                stats[3], float(want))
    assert (stats[1], stats[2]) == (sel['K'], sel['T']), (stats, sel['K'], sel['T'])
    return q, stats, sel


# ---- the q map and the selection -------------------------------------------------------------------------------------

def test_q_map_matches_torch_softmax_gather(eng):
    logits, labels = _maps(1, 4, 21, 97, 83)
    q = eng.ohem_raw(logits, labels, 255, 0.7, 100)[2]
    y = labels[:, 0].long()
    valid = (y != 255)
    want = torch.softmax(logits, 1).gather(1, torch.where(valid, y, 0)[:, None])[:, 0]
    want = torch.where(valid, want, torch.ones_like(want))
    assert _ulps(q, want) <= 2


SIZES = [(1, 3, 1, 1), (2, 2, 7, 5), (3, 21, 65, 65), (2, 32, 33, 129), (8, 21, 513, 513), (8, 19, 801, 801)]


@pytest.mark.parametrize('n,c,h,w', SIZES)
def test_selection_is_exact_for_k_1_v_and_all(eng, n, c, h, w):
    logits, labels = _maps(2, n, c, h, w)
    V = int(((labels != 255)).sum())
    for k in sorted({1, max(V // 2, 1), V, n * h * w}):
        _check_selection(eng, logits, labels, k)


@pytest.mark.parametrize('kind', ['all_equal', 'heavy_ties', 'straddle', 'nan_logits', 'tiny_q'])
def test_selection_ties_bins_and_nan(eng, kind):
    n, c, h, w = 2, 5, 61, 67
    logits, labels = _maps(3, n, c, h, w)
    if kind == 'all_equal':
        logits.zero_()
    elif kind == 'heavy_ties':
        logits = (logits * 2).round() / 2              # few distinct q values
    elif kind == 'straddle':
        # target probabilities just below and above powers of two and level-2 bin edges of the keys
        g = torch.Generator().manual_seed(4)
        base = torch.tensor([0.25, 0.5, 0.125, 0.0625, 1 / 3])
        qs = base[torch.randint(0, 5, (n, h, w), generator=g)] * (1 + (torch.randint(-3, 4, (n, h, w), generator=g)
                                                                       * 2.0 ** -21))
        logits = torch.zeros(n, c, h, w)
        y = torch.randint(0, c, (n, h, w), generator=g)
        # q = e^a / (e^a + c - 1)  =>  a = log(q (c - 1) / (1 - q))
        logits.scatter_(1, y[:, None], torch.log(qs * (c - 1) / (1 - qs))[:, None])
        logits, labels = logits.cuda(), y[:, None].float().cuda()
    elif kind == 'nan_logits':
        logits[0, :, :5, :] = float('nan')
    elif kind == 'tiny_q':
        logits = logits * 40                            # q underflows to 0 and saturates to 1
    V = int((labels != 255).sum())
    for k in (1, 2, V // 3, V - 1, V, n * h * w):
        _check_selection(eng, logits, labels, k)


def test_branches_v0_k0_and_early_exit(eng):
    logits, labels = _maps(5, 2, 7, 31, 29)
    _, stats, _ = _check_selection(eng, logits, torch.full_like(labels, 255), 10, 0.7)
    assert stats[0] == 0 and stats[1] == 0
    per = eng.ohem_raw(logits, torch.full_like(labels, 255), 255, 0.7, 10)[0]
    assert torch.isnan(per).all()
    V = int((labels != 255).sum())
    for k, thresh in ((0, 0.3), (V + 1, 0.3)):
        _, stats, _ = _check_selection(eng, logits, labels, k, thresh)
        assert stats[1] == V and math.isinf(stats[2]) and math.isnan(stats[3])
    q = eng.ohem_raw(logits, labels, 255, -1.0, 1)[2]
    qs = torch.sort(q[labels[:, 0] != 255])[0]
    tau = float(qs[V // 2])
    _, stats, _ = _check_selection(eng, logits, labels, V // 4, tau)        # early exit: T = tau, t_k not selected
    assert stats[2] == tau and math.isnan(stats[3])
    _, stats, _ = _check_selection(eng, logits, labels, 3 * V // 4, tau)    # t_k > tau: T = t_k
    assert stats[2] == stats[3] > tau
    _, stats, _ = _check_selection(eng, logits, labels, V // 2, 1.5)        # tau >= 1: every valid pixel
    assert stats[2] == 1.5 and stats[1] == V


# ---- loss and gradients ----------------------------------------------------------------------------------------------

def _gap_k(q, valid, lo=0.3, hi=0.7):
    """A k in the middle of the valid q's whose k-th and (k+1)-th smallest q are furthest apart -> (k, gap)."""
    s = torch.sort(q[valid].double().flatten().cpu())[0]
    V = s.numel()
    ks = torch.arange(max(int(lo * V), 1), int(hi * V))
    gaps = s[ks] - s[ks - 1]
    j = int(torch.argmax(gaps))
    return int(ks[j]), float(gaps[j])


@pytest.mark.parametrize('c', [2, 19, 21, 32])
@pytest.mark.parametrize('branch', ['t_k', 'tau', 'keep_all'])
def test_loss_and_gradients_match_the_fp64_oracle(eng, c, branch):
    n, h, w = 3, 47, 53
    logits, labels = _maps(6 + c, n, c, h, w, spread=1.5)
    q64, valid, _ = H.q_map(logits.double(), labels.double())
    k, gap = _gap_k(q64, valid)
    assert gap > 1e-6, gap
    s = torch.sort(q64[valid])[0]
    thresh = {'t_k': 0.0, 'tau': float(s[k - 1] + s[k]) / 2, 'keep_all': 0.5}[branch]
    if branch == 'tau':
        k = k // 2
    if branch == 'keep_all':
        k = 0
    x64 = logits.double().requires_grad_(True)
    per64, _, sel = H.ohem_criterion(x64, labels.double(), 255, thresh, k, return_selection=True)
    per64.mean().backward()
    per, grad, q, stats = eng.ohem_raw(logits, labels, 255, thresh, k, upstream_const=1.0 / n)
    assert stats[1].item() == sel['K']
    assert float((per.double() - per64.detach()).abs().max() / per64.detach().abs().max()) <= 1e-6
    assert float((grad.double() - x64.grad).abs().max() / x64.grad.abs().max()) <= 1e-6
    # unfused: backward of the per-sample values with a non-uniform upstream
    x = logits.clone().requires_grad_(True)
    up = torch.tensor([0.3, -1.2, 2.0][:n], device='cuda')
    out = eng.ohem_cross_entropy2d(x, labels, 255, thresh, k)
    (out * up).sum().backward()
    x64.grad = None
    (H.ohem_criterion(x64, labels.double(), 255, thresh, k) * up.double()).sum().backward()
    assert float((x.grad.double() - x64.grad).abs().max() / x64.grad.abs().max()) <= 1e-6
    assert float((out.double() - per64.detach()).abs().max() / per64.detach().abs().max()) <= 1e-6


def test_repeated_calls_are_bit_identical_and_never_synchronise(eng):
    logits, labels = _maps(9, 4, 21, 129, 129)
    V = int((labels != 255).sum())
    outs = []
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(2):
            for k, thresh in ((V // 3, 0.0), (V // 3, 0.7), (0, 0.7)):
                x = logits.clone().requires_grad_(True)
                per = eng.ohem_cross_entropy2d(x, labels, 255, thresh, k, upstream_const=1.0 / 4)
                torch.mean(per).backward()
                y = logits.clone().requires_grad_(True)
                (eng.ohem_cross_entropy2d(y, labels, 255, thresh, k) * 0.5).sum().backward()
                outs.append((per.detach(), x.grad, y.grad))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    half = len(outs) // 2
    for a, b in zip(outs[:half], outs[half:]):
        for u, v in zip(a, b):
            assert torch.equal(u, v)


def test_rejects_unsupported_inputs(eng):
    logits, labels = _maps(10, 1, 33, 5, 5)
    with pytest.raises(RuntimeError):
        eng.ohem_raw(logits, labels, 255, 0.7, 3)
    logits, labels = _maps(10, 1, 4, 5, 5)
    for thresh, k in ((float('nan'), 3), (float('inf'), 3), (0.7, -1)):
        with pytest.raises(ValueError):
            eng.ohem_raw(logits, labels, 255, thresh, k)


# ---- whole steps -----------------------------------------------------------------------------------------------------

def _energies(grads, names):
    return np.array([[float(grads[n].double().sum()), float((grads[n].double() ** 2).sum())] for n in names])


DRAW_SEED, TORCH_SEED = 2024, 77
LBS, UBS, SIZE = 2, 2, 65


def _init_state(model, seed, img):
    """Random-init state with BatchNorm running statistics from one training-mode forward (see test_gpu_unimatch)."""
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


def _unimatch_draws(eng, img):
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params, draw_fp_scales
    table, boxes = draw_strong_params(UBS, SIZE, SIZE, 0.5, rng=np.random.RandomState(DRAW_SEED))
    torch.manual_seed(TORCH_SEED)
    scales = draw_fp_scales(LBS + UBS, (256, 2048), 0.5)
    strong = eng.strong_aug(img[LBS:].contiguous().cuda(), torch.from_numpy(table))[0].cpu()
    return table, boxes, scales, strong


def _run_oracle(alg, dt, states, img, lab, crit, draws):
    st = [O.to_dtype(O.to_dtype(s, torch.float64), dt) for s in states]
    with H.supervised_criterion(crit):
        if alg == 'ssl_mt':
            orc = O.MTOracle(st[0], st[1], lr=0.00025, max_iters=10, cons_scale=1.0, rampup_steps=1, ema_decay=0.99)
            r = orc.step(img.to(dt), lab.to(dt), LBS)
            return {k: float(r[k]) for k in ('s_task_loss', 't_task_loss', 'cons_loss')}, {'s': r['grads']}, orc.names
        if alg == 'ssl_cps':
            orc = C.CPSOracle(st[0], st[1], lr=0.00025, max_iters=10, cps_scale=1.5, rampup_steps=0)
            r = orc.step(img.to(dt), lab.to(dt), LBS)
            return ({k: float(v) for k, v in r.items() if k.endswith('_loss')},
                    {'l': r['l_grads'], 'r': r['r_grads']}, orc.names)
        table, boxes, scales, strong = draws
        orc = U.UniMatchOracle(st[0], model='deeplabv3plus', max_iters=10, threshold=0.95)
        r = orc.step(img.to(dt), lab.to(dt), LBS, table, boxes, [s.to(dt) for s in scales], strong)
        return ({k: float(r[k]) for k in ('task_loss', 's1_loss', 's2_loss', 'fp_loss')}, {'m': r['grads']},
                orc.names)


STEP_CASES = [(a, b) for a in ('ssl_mt', 'ssl_cps', 'ssl_unimatch') for b in ('t_k', 'tau')]
_STEP_CACHE = {}


def _oracle_steps(eng, alg, branch):
    """fp32 and fp64 oracle steps with k and tau chosen so that T lies in the widest gap of the fp64 q values of every
    criterion call of the step (T = t_k: the k-th and (k+1)-th smallest q are furthest apart, tau = 0; T = tau: tau
    in the widest gap of the middle q values, k = 1)."""
    key = (alg, branch)
    if key not in _STEP_CACHE:
        img, lab = O.synthetic_batch(91, LBS + UBS, LBS, SIZE, SIZE)
        model = 'deeplabv3plus' if alg == 'ssl_unimatch' else 'deeplabv2'
        n_states = 1 if alg == 'ssl_unimatch' else 2
        states = [_init_state(model, 93 + 2 * i, img) for i in range(n_states)]
        draws = _unimatch_draws(eng, img) if alg == 'ssl_unimatch' else None
        seen = []

        def probe(logits, gt, ignore_index=255):
            q, valid, _ = H.q_map(logits.detach(), gt, ignore_index)
            seen.append((q, valid))
            return H.ohem_criterion(logits, gt, ignore_index, 0.5, 0)
        _run_oracle(alg, torch.float64, states, img, lab, probe, draws)
        if branch == 't_k':
            sorted_q = [torch.sort(q[v])[0] for q, v in seen]
            V = min(s.numel() for s in sorted_q)
            ks = torch.arange(int(0.3 * V), int(0.7 * V))
            gaps = torch.stack([s[ks] - s[ks - 1] for s in sorted_q]).min(0)[0]
            j = int(torch.argmax(gaps))
            k, thresh, gap = int(ks[j]), 0.0, float(gaps[j])
        else:
            allq = torch.sort(torch.cat([q[v] for q, v in seen]))[0]
            lo, hi = int(0.4 * allq.numel()), int(0.6 * allq.numel())
            d = allq[lo + 1:hi] - allq[lo:hi - 1]
            j = int(torch.argmax(d))
            k, thresh, gap = 1, float(allq[lo + j] + allq[lo + j + 1]) / 2, float(d[j])
        crit = H.criterion(thresh, k)
        out = [_run_oracle(alg, dt, states, img, lab, crit, draws) for dt in (torch.float32, torch.float64)]
        _STEP_CACHE[key] = (img, lab, states, draws, k, thresh, gap, out)
    return _STEP_CACHE[key]


def _engine_step(alg, k, thresh, states, img, lab):
    from pixelssl_b200 import runner
    cfg = dict(BASE, ssl_algorithm=alg, batch_size=LBS + UBS, unlabeled_batch_size=UBS, ohem_thresh=thresh,
               ohem_min_kept=k)
    if alg == 'ssl_mt':
        cfg.update(cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=1, ema_decay=0.99,
                   criterions={'model': 'ohem_sseg_criterion'})
    elif alg == 'ssl_cps':
        cfg.update(cps_scale=1.5, cps_rampup_epochs=0, models={'lmodel': 'deeplabv2', 'rmodel': 'deeplabv2'},
                   optimizers={'lmodel': 'sgd', 'rmodel': 'sgd'},
                   lrers={'lmodel': 'polynomiallr', 'rmodel': 'polynomiallr'},
                   criterions={'lmodel': 'ohem_sseg_criterion', 'rmodel': 'ohem_sseg_criterion'})
    else:
        cfg.update(uni_threshold=0.95, uni_scale=1.0, uni_rampup_epochs=0, models={'model': 'deeplabv3plus'},
                   criterions={'model': 'ohem_sseg_criterion'})
    a = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
    if alg == 'ssl_mt':
        mods = {'s': a.s_model}
        pairs = [(a.s_model, states[0]), (a.t_model, states[1])]
    elif alg == 'ssl_cps':
        mods = {'l': a.l_model, 'r': a.r_model}
        pairs = [(a.l_model, states[0]), (a.r_model, states[1])]
    else:
        mods = {'m': a.model}
        pairs = [(a.model, states[0])]
    for m, st in pairs:
        m.load_state_dict({'module.model.' + kk: v for kk, v in st.items()}, strict=True)
    np.random.seed(DRAW_SEED)
    torch.manual_seed(TORCH_SEED)
    a._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    return a, mods


@pytest.mark.parametrize('alg,branch', STEP_CASES)
def test_step_with_ohem_matches_oracle(ops, alg, branch):
    img, lab, states, draws, k, thresh, gap, (r32, r64) = _oracle_steps(ops, alg, branch)
    print('%s %s: k %d tau %.9g in a gap of %.2e' % (alg, branch, k, thresh, gap))
    a, mods = _engine_step(alg, k, thresh, states, img, lab)
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    loss32, g32, names = r32
    loss64, g64, _ = r64
    for key in loss64:
        got = float(a.meters[key].val)
        print('%s %s %s: engine %.8g oracle fp32 %.8g fp64 %.8g' % (alg, branch, key, got, loss32[key], loss64[key]))
        assert_loss_yardstick(got, loss32[key], loss64[key], '%s %s %s' % (alg, branch, key))
    for side, m in mods.items():
        sp = dict(m.module.model.named_parameters())
        got = np.array([float((sp[n].grad.double() ** 2).sum()) for n in names])
        print(assert_energy_yardstick(got, _energies(g32[side], names), _energies(g64[side], names),
                                      '%s %s %s grad energies' % (alg, branch, side)))


ALGS = {
    'ssl_null': {'unlabeled_batch_size': 0, 'batch_size': 2, 'ignore_unlabeled': True},
    'ssl_mt': {'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 1, 'ema_decay': 0.99},
    'ssl_adv': {'adv_for_labeled': True, 'labeled_adv_scale': 0.01, 'unlabeled_adv_scale': 0.001,
                'discriminator_scale': 1.0, 'discriminator_lr': 1e-4, 'unlabeled_for_discriminator': True},
    'ssl_s4l': {'rotated_sup_scale': 0.5, 'rotation_scale': 1.0},
    'ssl_gct': {'ssl_mode': 'gct', 'fc_ssl_scale': 1.0, 'dc_ssl_scale': 100.0, 'dc_threshold': 0.6,
                'dc_rampup_epochs': 1, 'fd_lr': 1e-4, 'fd_scale': 10.0, 'mu': 0.5, 'nu': 1, 'im_size': 65},
    'ssl_cct': {'cons_scale': 30.0, 'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0, 'vat_dec_num': 1, 'drop_dec_num': 1,
                'cut_dec_num': 1, 'context_dec_num': 1, 'object_dec_num': 1, 'fd_dec_num': 1, 'fn_dec_num': 1},
    'ssl_cutmix': {'cons_scale': 20.0, 'cons_rampup_epochs': 0, 'cons_threshold': 0.97, 'ema_decay': 0.99,
                   'batch_size': 6, 'unlabeled_batch_size': 4},
    'ssl_cps': {'cps_scale': 1.5, 'cps_rampup_epochs': 0},
    'ssl_unimatch': {'uni_threshold': 0.95, 'uni_scale': 1.0, 'uni_rampup_epochs': 0},
}


@pytest.mark.parametrize('name', sorted(ALGS))
def test_every_algorithm_trains_with_the_ohem_criterion(eng, name):
    from pixelssl_b200 import runner
    # UniMatch's eval-mode forward of a random-init network with the initial BatchNorm running statistics leaves the
    # fp16-pair range (see test_gpu_unimatch._init): it runs on the exact-fp32 convolutions here
    eng.set_conv_precision('fp32' if name == 'ssl_unimatch' else 'f16x3')
    try:
        keys = ['lmodel', 'rmodel'] if name in ('ssl_gct', 'ssl_cps') else ['model']
        cfg = dict(BASE, ssl_algorithm=name, batch_size=4, unlabeled_batch_size=2, ohem_min_kept=3000)
        cfg.update(ALGS[name])
        cfg.update(models={k: 'deeplabv2' for k in keys}, optimizers={k: 'sgd' for k in keys},
                   lrers={k: 'polynomiallr' for k in keys}, criterions={k: 'ohem_sseg_criterion' for k in keys})
        torch.manual_seed(0)
        alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
        lbs = cfg['batch_size'] - cfg['unlabeled_batch_size']
        img, lab = O.synthetic_batch(71, cfg['batch_size'], lbs, 65, 65)
        alg._train([((img,), (lab,))], 0)
        torch.cuda.synchronize()
        assert eng.conv_tc_status() == 0 and eng.h16_status() == 0
        losses = {k: float(alg.meters[k].val) for k in alg.meters.keys() if 'loss' in k}
        assert losses and all(np.isfinite(v) for v in losses.values()), losses
    finally:
        eng.set_conv_precision('fp32')
