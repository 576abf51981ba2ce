"""Multi-view evaluation without a GPU: its flags (absent by default, added by build_args and by register_into_pixelssl
on request), their validation when an algorithm is built, the tile enumeration of the driver, and the oracle
(oracle/eval_oracle.py) against a by-hand fp64 evaluation."""
import argparse
import math
import types

import pytest
import torch

from oracle import eval_oracle as E

BASE = {'ssl_algorithm': 'ssl_null', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'batch_size': 2, 'unlabeled_batch_size': 0}


# ---- flags and registration ------------------------------------------------------------------------------------------

def test_flags_absent_from_the_default_parser():
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import evaluation
    args = runner.build_args(dict(BASE))
    assert not any(hasattr(args, f) for f in evaluation.FLAGS)
    assert evaluation.is_default(args) and evaluation.settings(args) == ('whole', None, [1.0], False)
    parser = runner.create_parser('ssl_null')
    runner.add_proxy_arguments(parser)
    with pytest.raises(SystemExit):
        parser.parse_args(['--val-protocol', 'sliding'])


@pytest.mark.parametrize('flag', ['val_protocol', 'val_crop_size', 'val_scales', 'val_flip'])
def test_build_args_adds_the_flags_when_configured(flag):
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import evaluation
    value = {'val_protocol': 'whole', 'val_crop_size': 801, 'val_scales': [1.0], 'val_flip': False}[flag]
    args = runner.build_args(dict(BASE, **{flag: value}))
    assert {f: getattr(args, f) for f in evaluation.FLAGS} == dict(evaluation.DEFAULTS, **{flag: value})
    args = runner.build_args(dict(BASE, val_protocol='sliding', val_crop_size=801, val_scales=[0.75, 1.0, 1.25],
                                  val_flip=True))
    assert evaluation.settings(args) == ('sliding', 801, [0.75, 1.0, 1.25], True)
    assert not evaluation.is_default(args)


def _fake_pixelssl():
    pkg = types.ModuleType('pixelssl')
    pkg.ssl_algorithm = types.ModuleType('pixelssl.ssl_algorithm')
    pkg.nn = types.ModuleType('pixelssl.nn')
    pkg.nn.data = types.ModuleType('pixelssl.nn.data')
    return pkg


@pytest.mark.parametrize('with_parser_hook', [True, False])
def test_register_into_pixelssl_adds_the_flags_on_request(with_parser_hook):
    import pixelssl_b200
    seen = []
    pkg, task_model, task_criterion = _fake_pixelssl(), types.ModuleType('model'), types.ModuleType('criterion')
    if with_parser_hook:
        task_model.add_parser_arguments = lambda parser: seen.append(parser)
    pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion))
    if with_parser_hook:
        p = argparse.ArgumentParser()
        task_model.add_parser_arguments(p)
        assert seen == [p] and not hasattr(p.parse_args([]), 'val_protocol')
    else:
        assert not hasattr(task_model, 'add_parser_arguments')
    for _ in range(2):          # idempotent: the flags are added once however often it is registered
        pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion), val_protocol=True)
    p = argparse.ArgumentParser()
    task_model.add_parser_arguments(p)
    a = p.parse_args(['--val-protocol', 'sliding', '--val-crop-size', '801', '--val-scales', '[0.5,1.5]'])
    assert (a.val_protocol, a.val_crop_size, a.val_scales, a.val_flip) == ('sliding', 801, [0.5, 1.5], False)
    if with_parser_hook:
        assert seen[-1] is p
    with pytest.raises(ValueError):
        pixelssl_b200.register_into_pixelssl(pkg, val_protocol=True)


@pytest.mark.parametrize('bad', [{'val_protocol': 'sliding'}, {'val_protocol': 'sliding', 'val_crop_size': 1},
                                 {'val_crop_size': 0}, {'val_scales': [1.0, 0.0]}, {'val_scales': [-0.5]},
                                 {'val_scales': [float('nan')]}])
def test_invalid_values_fail_when_the_algorithm_is_built(bad):
    from pixelssl_b200 import runner
    args = runner.build_args(dict(BASE, **bad))
    with pytest.raises(SystemExit):
        runner.build_algorithm(args)


def test_invalid_values_fail_in_the_shared_build():
    """The check sits in _SSLBase.build, which every algorithm's build runs before it makes any model."""
    from pixelssl_b200.ssl_algorithm import ssl_base
    from pixelssl_b200.task.sseg import evaluation
    called = []

    class Probe(ssl_base._SSLBase):
        def _build(self, *a):
            called.append(a)
    with pytest.raises(SystemExit):
        Probe(argparse.Namespace(val_protocol='sliding', val_crop_size=None)).build(None, None, None, None, None)
    assert not called
    Probe(argparse.Namespace(val_protocol='sliding', val_crop_size=2)).build(None, None, None, None, None)
    assert len(called) == 1
    with pytest.raises(SystemExit):
        evaluation.check_args(argparse.Namespace(val_scales=[]))


def test_validating_scope_and_multi_view_condition():
    from pixelssl_b200.task.sseg import evaluation
    m = types.SimpleNamespace(training=False, args=argparse.Namespace(val_flip=True))
    assert not evaluation.multi_view(m)
    with evaluation.validating():
        assert evaluation.multi_view(m)
        m.training = True
        assert not evaluation.multi_view(m)                    # train mode: the plain forward
        m.training = False
        assert not evaluation.multi_view(types.SimpleNamespace(training=False, args=argparse.Namespace()))
    assert not evaluation.multi_view(m)


# ---- views and tiles -------------------------------------------------------------------------------------------------

def test_cityscapes_tiles():
    from pixelssl_b200.task.sseg import evaluation
    tiles = evaluation.tiles(1024, 2048, 'sliding', 801)
    assert sorted({t[0] for t in tiles}) == [0, 534] and sorted({t[2] for t in tiles}) == [490, 801]
    assert sorted({t[1] for t in tiles}) == [0, 534, 1068, 1602]
    assert [t[3] for t in tiles[:4]] == [801, 801, 801, 446]
    assert len(tiles) == 8
    gh, gw, sh, sw, groups = evaluation.tile_groups(1024, 2048, 'sliding', 801)
    assert (gh, gw, sh, sw) == (801, 801, 534, 534)
    assert groups == [(0, 1, 0, 3, 801, 801), (0, 1, 1602, 1, 801, 446),
                      (534, 1, 0, 3, 490, 801), (534, 1, 1602, 1, 490, 446)]


def test_small_tiles_keep_the_covered_tail():
    from pixelssl_b200.task.sseg import evaluation
    tiles = evaluation.tiles(97, 129, 'sliding', 65)
    assert len(tiles) == 9
    assert [t[0] for t in tiles[::3]] == [0, 43, 86] and [t[2] for t in tiles[::3]] == [65, 54, 11]
    assert [t[1] for t in tiles[:3]] == [0, 43, 86] and [t[3] for t in tiles[:3]] == [65, 65, 43]
    # the row-86 tail tile lies inside the row-43 tile, and is kept
    assert (86, 0, 11, 65) in tiles and (43, 0, 54, 65) in tiles and 86 + 11 == 43 + 54
    assert len(evaluation.tile_groups(97, 129, 'sliding', 65)[4]) == 6


@pytest.mark.parametrize('h,w,g', [(97, 129, 65), (1024, 2048, 801), (60, 70, 65), (9, 9, 6), (5, 3, 2), (3, 4, 3),
                                   (801, 801, 801), (1, 1, 2), (1280, 2560, 801), (2048, 4096, 801)])
def test_tiles_cover_every_pixel_and_match_the_groups_and_the_oracle(h, w, g):
    from pixelssl_b200.task.sseg import evaluation
    tiles = evaluation.tiles(h, w, 'sliding', g)
    assert tiles == E.sliding_tiles(h, w, g)
    cover = torch.zeros(h, w, dtype=torch.int32)
    for r, c, th, tw in tiles:
        assert th >= 1 and tw >= 1 and r + th <= h and c + tw <= w
        cover[r:r + th, c:c + tw] += 1
    assert int(cover.min()) >= 1
    gh, gw, sh, sw, groups = evaluation.tile_groups(h, w, 'sliding', g)
    assert len(groups) <= 9
    from_groups = sorted((r0 + i * sh, c0 + j * sw, th, tw) for r0, nr, c0, nc, th, tw in groups
                         for i in range(nr) for j in range(nc))
    assert from_groups == sorted(tiles)
    shapes = [(th, tw) for *_, th, tw in groups]
    assert len(set(shapes)) == len(shapes)
    assert evaluation.tiles(h, w, 'whole', None) == [(0, 0, h, w)]


def test_views_and_view_sizes():
    from pixelssl_b200.task.sseg import evaluation
    assert evaluation.views([0.75, 1.0], True) == [(0.75, False), (0.75, True), (1.0, False), (1.0, True)]
    assert evaluation.views([1.25, 0.5], False) == E.views([1.25, 0.5], False)
    assert evaluation.view_size(1024, 2048, 0.75) == (768, 1536)
    assert evaluation.view_size(97, 129, 1.25) == (int(97 * 1.25 + 0.5), int(129 * 1.25 + 0.5)) == (121, 161)
    assert evaluation.view_size(97, 129, 1.0) == (97, 129)
    with pytest.raises(ValueError):
        evaluation.view_size(3, 3, 0.1)


# ---- the oracle against a by-hand evaluation -------------------------------------------------------------------------

def _stub(x):
    """A position-dependent stub network: a 3x3 zero-padded box sum of the channels, mixed into 3 classes."""
    w = torch.tensor([[1.0, -0.5, 0.25], [-0.3, 0.8, 0.1], [0.2, 0.1, -0.9]], dtype=x.dtype)
    k = torch.ones(3, 1, 3, 3, dtype=x.dtype) / 9
    box = torch.nn.functional.conv2d(x, k, padding=1, groups=3)
    return torch.einsum('kc,nchw->nkhw', w, box)


def _hand_resize(img, H, W):
    """Bilinear, align_corners=True, by hand: img [C][h][w] lists -> [C][H][W]."""
    C, h, w = len(img), len(img[0]), len(img[0][0])
    sy = (h - 1) / (H - 1) if H > 1 else 0.0
    sx = (w - 1) / (W - 1) if W > 1 else 0.0
    out = [[[0.0] * W for _ in range(H)] for _ in range(C)]
    for c in range(C):
        for y in range(H):
            fy = sy * y
            y0 = int(fy)
            y1 = min(y0 + 1, h - 1)
            ly = fy - y0
            for x in range(W):
                fx = sx * x
                x0 = int(fx)
                x1 = min(x0 + 1, w - 1)
                lx = fx - x0
                out[c][y][x] = ((1 - ly) * ((1 - lx) * img[c][y0][x0] + lx * img[c][y0][x1]) +
                                ly * ((1 - lx) * img[c][y1][x0] + lx * img[c][y1][x1]))
    return out


def _hand_softmax(v):
    m = max(v)
    e = [math.exp(t - m) for t in v]
    s = sum(e)
    return [t / s for t in e]


def _by_hand(x, protocol, crop, scales, flip):
    n, _, H, W = x.shape
    res = []
    for b in range(n):
        img = x[b].tolist()
        S = None
        vs = [(s, f) for s in scales for f in ((False, True) if flip else (False,))]
        for s, f in vs:
            hv, wv = (H, W) if s == 1.0 else (int(H * s + 0.5), int(W * s + 0.5))
            v = img if s == 1.0 else _hand_resize(img, hv, wv)
            if f:
                v = [[row[::-1] for row in ch] for ch in v]
            if protocol == 'whole':
                boxes = [(0, 0, hv, wv)]
            else:
                st = int(crop * 2 / 3)
                boxes = [(r, c, min(crop, hv - r), min(crop, wv - c)) for r in range(0, hv, st) for c in range(0, wv, st)]
            P = None
            for r, c, th, tw in boxes:
                tile = torch.tensor([[row[c:c + tw] for row in ch[r:r + th]] for ch in v], dtype=torch.float64)
                logits = _stub(tile[None])[0].tolist()
                K = len(logits)
                if P is None:
                    P = [[[0.0] * wv for _ in range(hv)] for _ in range(K)]
                for yy in range(th):
                    for xx in range(tw):
                        p = _hand_softmax([logits[k][yy][xx] for k in range(K)])
                        for k in range(K):
                            P[k][r + yy][c + xx] += p[k]
            if f:
                P = [[row[::-1] for row in ch] for ch in P]
            if s != 1.0:
                P = _hand_resize(P, H, W)
            S = P if S is None else [[[a + b_ for a, b_ in zip(ra, rb)] for ra, rb in zip(ca, cb)] for ca, cb in zip(S, P)]
        res.append([[[t / len(vs) for t in row] for row in ch] for ch in S])
    return torch.tensor(res, dtype=torch.float64)


@pytest.mark.parametrize('protocol,crop,scales,flip', [('whole', None, [1.0], True), ('sliding', 4, [1.0], False),
                                                       ('sliding', 4, [0.75, 1.25], True), ('whole', None, [0.5, 2.0], False),
                                                       ('sliding', 2, [1.0, 0.6], True)])
def test_oracle_matches_a_by_hand_evaluation(protocol, crop, scales, flip):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 3, 7, 10, generator=g, dtype=torch.float64)
    want = _by_hand(x, protocol, crop, scales, flip)
    mean, logmean = E.evaluate(_stub, x, protocol, crop, scales, flip)
    assert mean.dtype == torch.float64
    assert float((mean - want).abs().max()) <= 1e-12
    if protocol == 'whole':         # overlapping sliding tiles add up: only the whole views sum to 1 per pixel
        assert torch.allclose(mean.sum(1), torch.ones(2, 7, 10, dtype=torch.float64), atol=1e-12)
    assert torch.equal(logmean, torch.log(torch.clamp(mean, min=E.FLT_MIN)))


def test_oracle_clamps_the_log():
    x = torch.zeros(1, 3, 2, 2, dtype=torch.float64)
    mean, logmean = E.evaluate(lambda t: torch.cat([t[:, :1] * 0 + 1e4, t[:, :1] * 0], 1), x)
    assert float(mean[0, 1].max()) == 0.0 and float(logmean[0, 1].max()) == math.log(E.FLT_MIN)
