"""UniMatch (ssl_unimatch) on the host: arguments, constructor validation, the refusal of PSPNet, plugin registration,
the seeded draws of the strong-view tables, and the CPU oracle's loss against its per-pixel definition."""
import math
import types

import numpy as np
import pytest
import torch

from oracle import unimatch_oracle as U

BASE = {'ssl_algorithm': 'ssl_unimatch', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20,
        'log_freq': 10 ** 6, 'batch_size': 16, 'unlabeled_batch_size': 8, 'uni_threshold': 0.95, 'uni_scale': 1.0,
        'uni_rampup_epochs': 0}


def test_parser_defaults_and_options():
    from pixelssl_b200 import runner
    ns = runner.create_parser('ssl_unimatch').parse_args([])
    assert (ns.uni_threshold, ns.uni_scale, ns.uni_rampup_epochs) == (-1, -1, -1)
    assert (ns.uni_fp_drop, ns.uni_cutmix_prob) == (0.5, 0.5)
    ns = runner.create_parser('ssl_unimatch').parse_args(['--uni-threshold', '0.9', '--uni-scale', '2', '--uni-rampup-epochs',
                                                          '3', '--uni-fp-drop', '0.25', '--uni-cutmix-prob', '1'])
    assert (ns.uni_threshold, ns.uni_scale, ns.uni_rampup_epochs, ns.uni_fp_drop, ns.uni_cutmix_prob) == \
        (0.9, 2.0, 3, 0.25, 1.0)


def _construct(**over):
    from pixelssl_b200 import runner
    from pixelssl_b200.ssl_algorithm import ssl_unimatch
    return ssl_unimatch.SSLUNIMATCH(runner.build_args(dict(BASE, **over), iters_per_epoch=5))


@pytest.mark.parametrize('override,rejected', [
    ({}, False),
    ({'uni_threshold': 0.0}, False),
    ({'uni_threshold': 1.0}, False),
    ({'uni_rampup_epochs': 5, 'uni_fp_drop': 0.0, 'uni_cutmix_prob': 0.0}, False),
    ({'batch_size': 4, 'unlabeled_batch_size': 2}, False),
    ({'uni_threshold': -1.0}, True),                # missing
    ({'uni_threshold': 1.5}, True),
    ({'uni_threshold': -0.1}, True),
    ({'uni_scale': -1.0}, True),                    # missing
    ({'uni_rampup_epochs': -1}, True),              # missing
    ({'uni_fp_drop': 1.0}, True),
    ({'uni_cutmix_prob': 1.5}, True),
    ({'batch_size': 8, 'unlabeled_batch_size': 5}, True),     # odd
    ({'batch_size': 4, 'unlabeled_batch_size': 0}, True),     # zero
    ({'batch_size': 4, 'unlabeled_batch_size': 1}, True),
])
def test_constructor_validates_arguments(override, rejected, capsys):
    try:
        _construct(**override)
        got = False
    except SystemExit:
        got = True
    capsys.readouterr()
    assert got == rejected


def test_pspnet_is_refused_at_build_time(caplog):
    from pixelssl_b200.task.sseg import model
    alg = _construct()
    with pytest.raises(SystemExit):
        alg.build([model.pspnet()], [None], [None], [None], None)
    assert 'forward_fp' in caplog.text and 'PSPNet' in caplog.text
    assert getattr(model.deeplabv2(), 'forward_fp', None) is not None
    assert getattr(model.deeplabv3plus(), 'forward_fp', None) is not None


def test_export_rejects_bad_element_dicts(caplog):
    from pixelssl_b200 import runner
    from pixelssl_b200.ssl_algorithm import ssl_unimatch
    args = runner.build_args(dict(BASE), iters_per_epoch=5)
    d = {'lmodel': object(), 'rmodel': object()}
    with pytest.raises(SystemExit):
        ssl_unimatch.ssl_unimatch(args, d, dict(d), dict(d), dict(d), None)
    assert 'SSL_UNIMATCH' in caplog.text


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
def test_register_into_pixelssl_installs_ssl_unimatch_on_request(with_list):
    import pixelssl_b200
    from pixelssl_b200 import runner
    assert pixelssl_b200.SSL_UNIMATCH == 'ssl_unimatch'
    assert pixelssl_b200.EXTRA_SSL_ALGORITHMS == ['ssl_unimatch']
    assert pixelssl_b200.ALL_SSL_ALGORITHMS == pixelssl_b200.SSL_ALGORITHMS + ['ssl_unimatch']
    # the default installs what it installed before UniMatch existed
    pkg, reference = _fake_pixelssl(with_list)
    pixelssl_b200.register_into_pixelssl(pkg)
    assert 'ssl_unimatch' not in pkg.ssl_algorithm.SSL_ALGORITHMS and 'ssl_unimatch' not in pkg.ssl_algorithm.__dict__
    # on request: installed and listed after ssl_cps
    pkg, reference = _fake_pixelssl(with_list)
    kept = pkg.ssl_algorithm.SSL_ALGORITHMS if with_list else None
    pixelssl_b200.register_into_pixelssl(pkg, extra_algorithms=['ssl_unimatch'])
    names = pkg.ssl_algorithm.SSL_ALGORITHMS
    if with_list:
        assert names is kept and names == reference + ['ssl_cps', 'ssl_unimatch']
    else:
        assert sorted(names) == sorted(pixelssl_b200.ALL_SSL_ALGORITHMS)
    mod = pkg.ssl_algorithm.__dict__['ssl_unimatch']
    assert mod.__name__ == 'pixelssl_b200.ssl_algorithm.ssl_unimatch'
    assert callable(mod.ssl_unimatch) and callable(mod.add_parser_arguments)
    pixelssl_b200.register_into_pixelssl(pkg, extra_algorithms=['ssl_unimatch'])     # idempotent
    assert names.count('ssl_unimatch') == 1 and names.count('ssl_cps') == 1
    with pytest.raises(ValueError):
        pixelssl_b200.register_into_pixelssl(pkg, extra_algorithms=['ssl_fixmatch'])
    # the engine's own runner accepts it either way
    assert runner.create_parser('ssl_unimatch').parse_args([]).uni_fp_drop == 0.5


# ---- the host draws --------------------------------------------------------------------------------------------------

def _by_hand_draws(rng, ubs, h, w, p_box):
    """The documented draw order, restated: per image, view 1 then view 2."""
    rows = {}
    for i in range(ubs):
        for k in range(2):
            d = {'jitter': rng.random_sample() < 0.8}
            if d['jitter']:
                d['order'] = list(rng.permutation(4))
                d['f'] = [rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5), rng.uniform(-0.25, 0.25)]
            d['gray'] = rng.random_sample() < 0.2
            d['sigma'] = rng.uniform(0.1, 2.0) if rng.random_sample() < 0.5 else None
            d['box'] = None
            if not rng.random_sample() > p_box:
                size = rng.uniform(0.02, 0.4) * h * w
                while True:
                    ratio = rng.uniform(0.3, 1 / 0.3)
                    cw, ch = int(np.sqrt(size / ratio)), int(np.sqrt(size * ratio))
                    x, y = rng.randint(0, w), rng.randint(0, h)
                    if x + cw <= w and y + ch <= h:
                        break
                d['box'] = (y, x, y + ch, x + cw)
            rows[k * ubs + i] = d
    return rows, rng.random_sample()


@pytest.mark.parametrize('ubs,h,w,p_box', [(2, 65, 65, 0.5), (4, 33, 47, 1.0), (8, 513, 513, 0.5), (4, 65, 65, 0.0)])
def test_strong_param_draws_are_seeded_and_follow_the_documented_order(ubs, h, w, p_box):
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_strong_params, gaussian_weights
    np.random.seed(123)
    table, boxes = draw_strong_params(ubs, h, w, p_box)
    after = np.random.random_sample()
    np.random.seed(123)
    table2, boxes2 = draw_strong_params(ubs, h, w, p_box)
    assert np.array_equal(table, table2) and np.array_equal(boxes, boxes2)
    rows, after_ref = _by_hand_draws(np.random.RandomState(123), ubs, h, w, p_box)
    assert after == after_ref                            # the same number of draws from the global stream
    assert table.shape == (2 * ubs, 32) and table.dtype == np.float32 and boxes.dtype == np.int32
    for v, d in rows.items():
        r = table[v]
        assert r[0] == float(d['jitter'])
        if d['jitter']:
            assert list(r[5:9]) == d['order'] and np.allclose(r[1:5], d['f'], rtol=1e-7, atol=0)
        else:
            assert list(r[5:9]) == [0, 1, 2, 3]
        assert r[9] == float(d['gray'])
        if d['sigma'] is None:
            assert r[10] == 0 and not r[16:].any()
        else:
            k = math.ceil(3 * d['sigma'])
            assert r[10] == k and np.float32(d['sigma']) == r[11]
            wts = gaussian_weights(d['sigma'])
            assert len(wts) == 2 * k + 1 and abs(wts.sum() - 1) < 1e-12
            assert np.array_equal(r[16:16 + 2 * k + 1], wts.astype(np.float32)) and not r[17 + 2 * k:].any()
        box = (0, 0, 0, 0) if d['box'] is None else d['box']
        assert tuple(boxes[v]) == box and tuple(r[12:16]) == box
        if d['box'] is not None:
            y0, x0, y1, x1 = box
            assert 0 <= y0 <= y1 <= h and 0 <= x0 <= x1 <= w
    if p_box == 0.0:
        assert not boxes.any()


def test_gaussian_weights_match_torchvision():
    import torchvision.transforms.v2.functional as TF
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import gaussian_weights
    for sigma in (0.1, 0.5, 1.37, 2.0):
        wts = gaussian_weights(sigma)
        k = len(wts)
        impulse = torch.zeros(1, 1, 2 * k + 1, 2 * k + 1, dtype=torch.float64)
        impulse[0, 0, k, k] = 1.0
        got = TF.gaussian_blur(impulse, kernel_size=[k, k], sigma=[sigma, sigma])[0, 0]
        want = torch.outer(torch.from_numpy(wts), torch.from_numpy(wts))
        assert torch.allclose(got[k - k // 2:k + k // 2 + 1, k - k // 2:k + k // 2 + 1], want, rtol=0, atol=1e-15)


def test_fp_scales_are_dropout2d_draws():
    from pixelssl_b200.ssl_algorithm.ssl_unimatch import draw_fp_scales
    torch.manual_seed(7)
    a = draw_fp_scales(6, (256, 2048), 0.5)
    torch.manual_seed(7)
    ref = [(torch.empty(6, c, 1, 1).bernoulli_(0.5) / 0.5).view(6, c) for c in (256, 2048)]
    assert [t.shape for t in a] == [(6, 256), (6, 2048)]
    assert all(torch.equal(x, y) for x, y in zip(a, ref))
    assert set(torch.cat([t.flatten() for t in a]).tolist()) == {0.0, 2.0}


# ---- the oracle's loss -----------------------------------------------------------------------------------------------

def _by_hand(w, mix, s, fp, boxes, tau):
    """fp64 loops over every pixel: the definition in the issue, first maximal index, confidence = max softmax."""
    ubs, c, h, wd = w.shape

    def label(v):
        vals = [float(x) for x in v]
        m = max(vals)
        return vals.index(m), 1.0 / sum(math.exp(x - m) for x in vals)

    def ce(v, y):
        vals = [float(x) for x in v]
        m = max(vals)
        return m + math.log(sum(math.exp(x - m) for x in vals)) - vals[y]

    tot = [0.0, 0.0, 0.0]
    count = 0
    for i in range(ubs):
        src = (i + ubs // 2) % ubs
        for py in range(h):
            for px in range(wd):
                y, conf = label(w[i, :, py, px])
                if conf >= tau:
                    count += 1
                    tot[2] += ce(fp[i, :, py, px], y)
                for k in range(2):
                    y0, x0, y1, x1 = boxes[k * ubs + i]
                    yk, ck = (label(mix[src, :, py, px]) if y0 <= py < y1 and x0 <= px < x1 else (y, conf))
                    if ck >= tau:
                        tot[k] += ce(s[k * ubs + i, :, py, px], yk)
    n = ubs * h * wd
    return tot[0] / n, tot[1] / n, tot[2] / n, count


def _case(seed, ubs=2, c=5, h=4, wd=6):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(ubs, c, h, wd, generator=g, dtype=torch.float64)
    w[0, :, 0, 0] = 1.5                                                # all tied: label 0, confidence 1/c
    w[1, :, 1, 2] = torch.tensor([0.0, 2.0, 0.0, 2.0, 2.0], dtype=torch.float64)[:c]   # first of three maxima: 1
    mix = torch.randint(0, 3, (ubs, c, h, wd), generator=g).double()  # many exact ties
    s = torch.randn(2 * ubs, c, h, wd, generator=g, dtype=torch.float64)
    fp = torch.randn(ubs, c, h, wd, generator=g, dtype=torch.float64)
    boxes = [(1, 2, 3, 5), (0, 0, 0, 0), (0, 0, h, wd), (2, 1, 4, 2)][:2 * ubs]
    return w, mix, s, fp, boxes


@pytest.mark.parametrize('tau', [0.0, 0.2, 0.35, 0.6, 1.01])
def test_oracle_loss_matches_the_per_pixel_definition(tau):
    w, mix, s, fp, boxes = _case(3)
    assert int(w.argmax(1)[0, 0, 0]) == 0 and int(w.argmax(1)[1, 1, 2]) == 1
    got = U.unimatch_terms(w, mix, s, fp, torch.tensor(boxes), tau)
    want = _by_hand(w, mix, s, fp, boxes, tau)
    for a, b in zip(got[:3], want[:3]):
        assert abs(float(a) - b) <= 1e-12
    assert int(got[3]) == want[3]
    n = w.shape[0] * w.shape[2] * w.shape[3]
    if tau == 0.0:
        assert int(got[3]) == n                          # every pixel
    if tau > 1.0:
        assert int(got[3]) == 0 and all(float(x) == 0.0 for x in got[:3])


def test_oracle_loss_gradient_vanishes_above_one():
    w, mix, s, fp, boxes = _case(4)
    s, fp = s.requires_grad_(True), fp.requires_grad_(True)
    l1, l2, lf, _ = U.unimatch_terms(w, mix, s, fp, torch.tensor(boxes), 1.01)
    gs, gf = torch.autograd.grad(l1 + l2 + lf, (s, fp))
    assert not gs.any() and not gf.any()
