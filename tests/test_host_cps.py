"""Cross Pseudo Supervision (ssl_cps) on the host: arguments, constructor and element-dict validation, plugin
registration, and the CPU oracle's CPS term against its per-pixel definition."""
import types

import numpy as np
import pytest
import torch

from oracle import cps_oracle as C

BASE = {'ssl_algorithm': 'ssl_cps', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20,
        'log_freq': 10 ** 6, 'batch_size': 16, 'unlabeled_batch_size': 8, 'cps_scale': 1.5, 'cps_rampup_epochs': 0}


def test_parser_defaults_and_options():
    from pixelssl_b200 import runner
    ns = runner.create_parser('ssl_cps').parse_args([])
    assert (ns.cps_scale, ns.cps_rampup_epochs, ns.cps_cutmix) == (-1, -1, False)
    assert list(ns.mask_prop_range) == [0.5, 0.5]
    ns = runner.create_parser('ssl_cps').parse_args(['--cps-scale', '1.5', '--cps-rampup-epochs', '3', '--cps-cutmix',
                                                     'true', '--mask-prop-range', '(0.25, 0.5)'])
    assert (ns.cps_scale, ns.cps_rampup_epochs, ns.cps_cutmix) == (1.5, 3, True)
    assert list(ns.mask_prop_range) == [0.25, 0.5]


def _construct(**over):
    from pixelssl_b200 import runner
    from pixelssl_b200.ssl_algorithm import ssl_cps
    return ssl_cps.SSLCPS(runner.build_args(dict(BASE, **over), iters_per_epoch=5))


@pytest.mark.parametrize('override,rejected', [
    ({}, False),
    ({'cps_cutmix': True}, False),
    ({'cps_cutmix': True, 'batch_size': 12, 'unlabeled_batch_size': 4}, False),
    ({'cps_scale': -1.0}, True),
    ({'cps_rampup_epochs': -1}, True),
    ({'cps_scale': -1.0, 'cps_rampup_epochs': -1, 'batch_size': 4, 'unlabeled_batch_size': 0}, False),
    ({'cps_cutmix': True, 'batch_size': 4, 'unlabeled_batch_size': 2}, True),
    ({'cps_cutmix': True, 'batch_size': 8, 'unlabeled_batch_size': 5}, True),
    ({'batch_size': 4, 'unlabeled_batch_size': 2}, False),
    ({'batch_size': 8, 'unlabeled_batch_size': 5}, False),
])
def test_constructor_validates_arguments(override, rejected, capsys):
    try:
        _construct(**override)
        got = False
    except SystemExit:
        got = True
    capsys.readouterr()
    assert got == rejected


@pytest.mark.parametrize('keys', [('model', 'lmodel', 'rmodel'), ('model', 'rmodel'), ('lmodel', 'other'), ('other',)])
def test_export_rejects_bad_element_dicts_before_building(keys, caplog):
    from pixelssl_b200 import runner
    from pixelssl_b200.ssl_algorithm import ssl_cps
    args = runner.build_args(dict(BASE), iters_per_epoch=5)
    d = {k: object() for k in keys}
    with pytest.raises(SystemExit):
        ssl_cps.ssl_cps(args, d, dict(d), dict(d), dict(d), None)
    assert 'SSL_CPS' in caplog.text


def test_element_dict_messages_name_the_algorithm(caplog):
    """GCT and CPS share one element-dict check; each message names its own algorithm."""
    from pixelssl_b200.ssl_algorithm import ssl_base
    for name in ('ssl_gct', 'ssl_cps'):
        with pytest.raises(SystemExit):
            ssl_base.pair_picker(name, {'a': 1, 'b': 2, 'c': 3}, {}, {}, {})
        assert 'The len(element_dict) of %s should be the same' % name.upper() in caplog.text
        caplog.clear()
        with pytest.raises(SystemExit):
            ssl_base.pair_picker(name, {'a': 1, 'b': 2, 'c': 3}, {'a': 1, 'b': 2, 'c': 3}, {'a': 1, 'b': 2, 'c': 3},
                                 {'a': 1, 'b': 2, 'c': 3})
        assert 'The %s algorithm supports element_dict with 1 or 2 elements, but given 3 elements' % name.upper() in \
            caplog.text
        caplog.clear()
    pick = ssl_base.pair_picker('ssl_cps', {'model': 1}, {'model': 2}, {'model': 3}, {'model': 4})
    assert pick({'model': 7}) == [7, 7]
    pick = ssl_base.pair_picker('ssl_cps', {'lmodel': 1, 'rmodel': 2}, {'lmodel': 1, 'rmodel': 2},
                                {'lmodel': 1, 'rmodel': 2}, {'lmodel': 1, 'rmodel': 2})
    assert pick({'lmodel': 'l', 'rmodel': 'r'}) == ['l', 'r']


def _fake_pixelssl(with_list):
    pkg = types.ModuleType('pixelssl')
    pkg.ssl_algorithm = types.ModuleType('pixelssl.ssl_algorithm')
    reference = ['ssl_null', 'ssl_mt', 'ssl_adv', 'ssl_s4l', 'ssl_gct', 'ssl_cct', 'ssl_cutmix']
    if with_list:
        pkg.ssl_algorithm.SSL_ALGORITHMS = list(reference)
    pkg.nn = types.ModuleType('pixelssl.nn')
    pkg.nn.data = types.ModuleType('pixelssl.nn.data')
    return pkg, reference


@pytest.mark.parametrize('with_list', [True, False])
def test_register_into_pixelssl_adds_ssl_cps(with_list):
    import pixelssl_b200
    pkg, reference = _fake_pixelssl(with_list)
    kept = pkg.ssl_algorithm.SSL_ALGORITHMS if with_list else None
    pixelssl_b200.register_into_pixelssl(pkg)
    names = pkg.ssl_algorithm.SSL_ALGORITHMS
    if with_list:
        assert names is kept and names == reference + ['ssl_cps']
    else:
        assert sorted(names) == sorted(pixelssl_b200.SSL_ALGORITHMS)
    assert pixelssl_b200.SSL_CPS == 'ssl_cps'
    for name in reference + ['ssl_cps']:
        mod = pkg.ssl_algorithm.__dict__[name]
        assert mod.__name__ == 'pixelssl_b200.ssl_algorithm.' + name
        assert callable(getattr(mod, name)) and callable(mod.add_parser_arguments)
    pixelssl_b200.register_into_pixelssl(pkg)                  # idempotent
    assert pkg.ssl_algorithm.SSL_ALGORITHMS.count('ssl_cps') == 1


def _by_hand(s, t):
    """mean over samples and pixels of logsumexp(s[:, :, p]) - s[y, p], y the first maximal index of t[:, :, p]"""
    n, c, h, w = s.shape
    total = 0.0
    for b in range(n):
        for i in range(h):
            for j in range(w):
                tv = [float(t[b, k, i, j]) for k in range(c)]
                y = tv.index(max(tv))
                sv = [float(s[b, k, i, j]) for k in range(c)]
                m = max(sv)
                total += m + np.log(sum(np.exp(v - m) for v in sv)) - sv[y]
    return total / (n * h * w)


def test_oracle_cps_term_matches_the_per_pixel_definition_with_ties():
    g = torch.Generator().manual_seed(3)
    s = torch.randn(2, 5, 4, 3, generator=g, dtype=torch.float64)
    t = torch.randint(0, 3, (2, 5, 4, 3), generator=g).double()     # values in {0, 1, 2}: many exact ties
    t[0, :, 0, 0] = 2.0                                              # all classes tied: index 0 wins
    t[1, :, 1, 2] = torch.tensor([0.0, 1.0, 0.0, 1.0, 1.0])          # first of three maxima: index 1
    assert int(t.argmax(1)[0, 0, 0]) == 0 and int(t.argmax(1)[1, 1, 2]) == 1
    assert abs(float(C.cps_term(s, t)) - _by_hand(s, t)) <= 1e-12
    # the plain step's form (each side's own logits as the other's target)
    assert abs(float(C.cps_term(s, s)) - _by_hand(s, s)) <= 1e-12
