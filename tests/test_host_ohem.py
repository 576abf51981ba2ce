"""ohem_sseg_criterion without a GPU: its flags (absent by default, added by build_args and by register_into_pixelssl
on request), its validation, every algorithm built with it, and the OHEM oracle against a by-hand fp64 evaluation of
each branch of the selection."""
import math
import types

import pytest
import torch

from oracle import ohem_oracle as H
from oracle import sseg_oracle as O

BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'batch_size': 4,
        'unlabeled_batch_size': 2}
ALGS = {
    'ssl_null': {},
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
PAIRED = ('ssl_gct', 'ssl_cps')


def _cfg(name, crit='ohem_sseg_criterion', **extra):
    keys = ['lmodel', 'rmodel'] if name in PAIRED else ['model']
    cfg = dict(BASE, ssl_algorithm=name, **ALGS[name])
    cfg.update(models={k: 'deeplabv2' for k in keys}, optimizers={k: 'sgd' for k in keys},
               lrers={k: 'polynomiallr' for k in keys}, criterions={k: crit for k in keys}, **extra)
    return cfg


# ---- flags and registration ------------------------------------------------------------------------------------------

def test_flags_absent_from_the_default_parser():
    from pixelssl_b200 import runner
    args = runner.build_args(_cfg('ssl_mt', crit='sseg_criterion'))
    assert not hasattr(args, 'ohem_thresh') and not hasattr(args, 'ohem_min_kept')
    with pytest.raises(SystemExit):
        runner.build_args(_cfg('ssl_mt', crit='sseg_criterion', ohem_thresh=0.5))


def test_build_args_adds_the_flags_for_an_ohem_criterion():
    from pixelssl_b200 import runner
    args = runner.build_args(_cfg('ssl_mt'))
    assert args.ohem_thresh == 0.7 and args.ohem_min_kept == 200000
    args = runner.build_args(_cfg('ssl_cps', ohem_thresh=0.6, ohem_min_kept=1000))
    assert args.ohem_thresh == 0.6 and args.ohem_min_kept == 1000


def _fake_pixelssl():
    pkg = types.ModuleType('pixelssl')
    pkg.ssl_algorithm = types.ModuleType('pixelssl.ssl_algorithm')
    pkg.nn = types.ModuleType('pixelssl.nn')
    pkg.nn.data = types.ModuleType('pixelssl.nn.data')
    return pkg


@pytest.mark.parametrize('with_parser_hook', [True, False])
def test_register_into_pixelssl_installs_the_criterion_on_request(with_parser_hook):
    import argparse
    import pixelssl_b200
    from pixelssl_b200.task.sseg import criterion as eng_criterion
    seen = []
    pkg, task_model, task_criterion = _fake_pixelssl(), types.ModuleType('model'), types.ModuleType('criterion')
    if with_parser_hook:
        task_criterion.add_parser_arguments = lambda parser: seen.append(parser)
    # the default installs what it installed before
    pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion))
    assert not hasattr(task_criterion, 'ohem_sseg_criterion')
    if with_parser_hook:
        p = argparse.ArgumentParser()
        task_criterion.add_parser_arguments(p)
        assert seen == [p] and not hasattr(p.parse_args([]), 'ohem_thresh')
    # on request: installed, and the module's parser hook adds the flags once however often it is registered
    for _ in range(2):
        pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion),
                                             extra_criterions=['ohem_sseg_criterion'])
    assert task_criterion.ohem_sseg_criterion is eng_criterion.ohem_sseg_criterion
    assert task_criterion.sseg_criterion is eng_criterion.sseg_criterion
    p = argparse.ArgumentParser()
    task_criterion.add_parser_arguments(p)
    a = p.parse_args(['--ohem-thresh', '0.6'])
    assert a.ohem_thresh == 0.6 and a.ohem_min_kept == 200000
    if with_parser_hook:
        assert seen[-1] is p
    with pytest.raises(ValueError):
        pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion), extra_criterions=['ohem2'])
    with pytest.raises(ValueError):
        pixelssl_b200.register_into_pixelssl(pkg, extra_criterions=['ohem_sseg_criterion'])


@pytest.mark.parametrize('bad', [{'ohem_thresh': float('nan')}, {'ohem_thresh': float('inf')},
                                 {'ohem_min_kept': -1}])
def test_invalid_hyper_parameters_fail_when_built(bad):
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import criterion as eng_criterion
    args = runner.build_args(_cfg('ssl_mt', **bad))
    with pytest.raises(SystemExit):
        eng_criterion.ohem_sseg_criterion()(args)
    ok = runner.build_args(_cfg('ssl_mt'))
    crit = eng_criterion.ohem_sseg_criterion()(ok)
    assert crit.thresh == 0.7 and crit.min_kept == 200000
    with pytest.raises(SystemExit):
        crit.forward([None, None], [None], [None])


@pytest.mark.slow
@pytest.mark.parametrize('name', sorted(ALGS))
def test_every_algorithm_builds_with_the_ohem_criterion(name, monkeypatch):
    """Built on the CPU (the modules stay where they are); the training step with it runs in test_gpu_ohem.py."""
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg.criterion import OHEMSSEGCriterion
    monkeypatch.setattr(torch.nn.Module, 'cuda', lambda self, device=None: self)
    alg = runner.build_algorithm(runner.build_args(_cfg(name, ohem_min_kept=1000)))
    crits = [c for c in vars(alg).values() if isinstance(c, OHEMSSEGCriterion)]
    assert len(crits) == (2 if name in PAIRED else 1)
    assert all(c.min_kept == 1000 and c.thresh == 0.7 for c in crits)


# ---- the oracle against a by-hand evaluation -------------------------------------------------------------------------

def _by_hand(logits, labels, ignore, thresh, k):
    """Plain Python over every pixel, in fp64: -> (loss, V, K, T)."""
    n, c, h, w = logits.shape
    pix = []
    for i in range(n):
        for yy in range(h):
            for xx in range(w):
                v = [float(logits[i, j, yy, xx]) for j in range(c)]
                lab = int(float(labels[i, yy, xx]))
                ok = lab != ignore and 0 <= lab < c
                m = max(v)
                se = sum(math.exp(t - m) for t in v)
                q = math.exp(v[lab] - m) / se if ok else 1.0
                nll = (math.log(se) + m - v[lab]) if ok else 0.0
                pix.append((i, ok, q, nll))
    V = sum(ok for _, ok, _, _ in pix)
    if V == 0 or k == 0 or k > V:
        T, kept = math.inf, [ok for _, ok, _, _ in pix]
    else:
        t_k = sorted(q for _, _, q, _ in pix)[k - 1]
        T = t_k if t_k > thresh else thresh
        kept = [ok and q <= T for _, ok, q, _ in pix]
    K = sum(kept)
    tot = sum(nll for (_, _, _, nll), kp in zip(pix, kept) if kp)
    per = [n * sum(nll for (i, _, _, nll), kp in zip(pix, kept) if kp and i == b) / K if K else math.nan
           for b in range(n)]
    return (tot / K if K else math.nan), V, K, T, per


def _maps(seed, n=2, c=4, h=3, w=5):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, c, h, w, generator=g, dtype=torch.float64) * 2
    labels = torch.randint(0, c, (n, h, w), generator=g).double()
    return logits, labels


def _sorted_q(logits, labels):
    return torch.sort(H.q_map(logits, labels)[0].flatten())[0]


CASES = ['v0', 'k_gt_v', 'k0', 'tk_above', 'tk_below', 'tau_ge_1', 'ties', 'invalid_labels']


@pytest.mark.parametrize('case', CASES)
def test_oracle_matches_a_by_hand_evaluation(case):
    logits, labels = _maps(3)
    thresh, k = 0.3, 7
    if case == 'v0':
        labels[:] = 255
    elif case == 'k_gt_v':
        labels[0, 0, :3] = 255
        k = 28                                        # V = 27
    elif case == 'k0':
        k = 0
    elif case == 'tk_above':
        q = _sorted_q(logits, labels)
        thresh = float(q[k - 1]) / 2                  # t_k > thresh: T = t_k
    elif case == 'tk_below':
        q = _sorted_q(logits, labels)
        thresh = float(q[k - 1] + q[k]) / 2           # t_k <= thresh: T = thresh
        k = 3
    elif case == 'tau_ge_1':
        thresh = 1.5
    elif case == 'ties':
        logits = 3.0 * torch.nn.functional.one_hot(labels.long(), 4).permute(0, 3, 1, 2).double()
        logits[:, :, :, :2] = 0.0                     # 12 pixels with q = 1/4 exactly, the others q = 0.87
        thresh, k = 0.01, 2
    elif case == 'invalid_labels':
        labels[0, 0, 0], labels[0, 1, 1], labels[1, 2, 2], labels[1, 0, 4] = -1, 255, 4, 3.7   # 3.7 -> 3, valid
        labels[0, 2, 0] = -0.5                        # truncates to 0: valid
    loss, V, K, T, per = _by_hand(logits, labels, 255, thresh, k)
    got, q, sel = H.ohem_criterion(logits, labels[:, None], 255, thresh, k, return_selection=True)
    assert (sel['V'], sel['K']) == (V, K)
    assert sel['T'] == T if math.isinf(T) else abs(sel['T'] - T) <= 1e-12 * T     # by-hand q: within an ulp
    if case == 'v0':
        assert V == 0 and torch.isnan(got).all()
        return
    assert abs(float(got.mean()) - loss) <= 1e-12 * abs(loss)
    assert torch.allclose(got, torch.tensor(per, dtype=torch.float64), rtol=1e-12, atol=0)
    if case == 'ties':
        assert K == 12 and sel['t_k'] == 0.25
    if case == 'tk_above':
        assert sel['T'] == sel['t_k'] > thresh
    if case in ('tk_below', 'tau_ge_1'):
        assert sel['T'] == thresh
    if case in ('k_gt_v', 'k0'):
        assert K == V and math.isinf(sel['T'])


def test_oracle_per_sample_contract_and_gradient():
    """mean(per) is the OHEM loss, and its gradient is (softmax - onehot) / K on the kept pixels."""
    logits, labels = _maps(5, n=3, c=5, h=4, w=4)
    logits.requires_grad_(True)
    per, q, sel = H.ohem_criterion(logits, labels, 255, 0.2, 10, return_selection=True)
    per.mean().backward()
    y = labels.long()
    want = (torch.softmax(logits.detach(), 1) - torch.nn.functional.one_hot(y, 5).permute(0, 3, 1, 2)) / sel['K']
    want = want * sel['kept'][:, None]
    assert torch.allclose(logits.grad, want, rtol=1e-12, atol=1e-15)


def test_supervised_criterion_swaps_the_step_oracles_criterion():
    crit = H.criterion(0.5, 3)
    with H.supervised_criterion(crit):
        assert O.sseg_criterion is crit
    assert O.sseg_criterion is not crit and O.sseg_criterion.__module__ == 'oracle.sseg_oracle'
