"""PSPNet on the engine: pyramid-pooling kernels against torch CPU, whole-network forward against the
reference-generated golden (tests/golden/pspnet_forward_97.npz) and forward+backward against the oracle."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sseg_oracle as O

from conftest import TEST_PRECISIONS

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')
CL = torch.channels_last


@pytest.fixture(scope='module', params=TEST_PRECISIONS)
def ops(request):
    """Every test of this module runs once per convolution precision mode (tests/conftest.py): the exact FFMA
    path and the wgmma paths bench.py measures are held to the same goldens."""
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    _ops.set_conv_precision(request.param)
    yield _ops
    _ops.set_conv_precision('fp32')


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize('hw,bin_size', [(7, 1), (7, 2), (7, 3), (7, 6), (45, 6), (33, 3)])
def test_adaptive_avg_pool(ops, hw, bin_size):
    g = torch.Generator().manual_seed(hw + bin_size)
    x = torch.randn(2, 64, hw, hw, generator=g)
    xc = x.clone().requires_grad_(True)
    ref = F.adaptive_avg_pool2d(xc, bin_size)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    out = ops.adaptive_avg_pool(xg, bin_size)
    (out * w.cuda()).sum().backward()
    assert rel(out, ref) <= 1e-6 and rel(xg.grad, xc.grad) <= 1e-6


def test_pyramid_concat(ops):
    g = torch.Generator().manual_seed(3)
    f = torch.randn(2, 64, 9, 11, generator=g)
    bs = [torch.randn(2, 16, b, b, generator=g) for b in (1, 2, 3, 6)]
    fc = f.clone().requires_grad_(True)
    bc = [b.clone().requires_grad_(True) for b in bs]
    ref = torch.cat([fc] + [F.interpolate(b, size=(9, 11), mode='bilinear', align_corners=False) for b in bc], 1)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    fg = f.cuda().contiguous(memory_format=CL).requires_grad_(True)
    bg = [b.cuda().contiguous(memory_format=CL).requires_grad_(True) for b in bs]
    out = ops.pyramid_concat(fg, bg)
    (out * w.cuda()).sum().backward()
    assert rel(out, ref) <= 1e-6 and rel(fg.grad, fc.grad) <= 1e-6
    for a, b in zip(bg, bc):
        assert rel(a.grad, b.grad) <= 1e-5


def _build(ops):
    from pixelssl_b200 import runner
    cfg = {'ssl_algorithm': 'ssl_null', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000,
           'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True, 'backbone': 'resnet50',
           'models': {'model': 'pspnet'}}
    return runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))


def test_pspnet_forward_golden_and_state_dict(ops):
    g = np.load(os.path.join(G, 'pspnet_forward_97.npz'))
    alg = _build(ops)
    st = O.randomize_bn_affine(O.init_pspnet(111), 112)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)      # same keys / shapes as the reference
    alg.model.train()
    img, _ = O.synthetic_batch(900, int(g['batch']), int(g['batch']), int(g['size']), int(g['size']))
    with torch.no_grad():
        resulter, _ = alg.model.forward((img.cuda(),))
    ref = torch.tensor(g['logits'])
    err = float((resulter['pred'][0].cpu() - ref).abs().max() / ref.abs().max())
    print('pspnet logits rel err vs reference:', err)
    assert err <= 1e-3
    px = resulter['sslcct_ad_inp']
    assert tuple(px.shape) == (2, 512, 7, 7)
    np.testing.assert_allclose(float((px.double() ** 2).sum()), g['latent_checksum'][0][1], rtol=2e-3)


def test_pspnet_supervised_step_vs_oracle(ops):
    """SSLNULL step with the PSPNet task model against the CPU oracle (loss, gradient energies)."""
    alg = _build(ops)
    st = O.randomize_bn_affine(O.init_pspnet(121), 122)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()}, strict=True)
    img, lab = O.synthetic_batch(901, 2, 2, 97, 97)
    alg._train([((img,), (lab,))], 0)
    names = [n for n, _, _ in O.pspnet_param_shapes()]
    stc = {k: (v.clone().requires_grad_(True) if k in names else v.clone()) for k, v in st.items()}
    logits, _ = O.pspnet_forward(img, stc, True)
    loss = O.sseg_criterion(logits, lab).mean()
    loss.backward()
    assert abs(float(alg.meters['task_loss'].val) - float(loss)) <= 1e-3 * float(loss)
    sp = dict(alg.model.module.model.named_parameters())
    e = np.array([float((sp[n].grad.double() ** 2).sum()) for n in names])
    r = np.array([float((stc[n].grad.double() ** 2).sum()) for n in names])
    relg = np.abs(e - r) / np.maximum(r, 1e-30)
    head = np.array([not n.startswith('backbone.') for n in names])
    print('pspnet grad energy rel: head median %.2e max %.2e | backbone median %.2e' % (
        np.median(relg[head]), relg[head].max(), np.median(relg[~head])))
    # measured over repeated runs (the pyramid's pooling / resize backward use fp32 atomics, and a few ReLU kinks take
    # either branch): head median 3.5e-4 .. 9.4e-4, max 2e-3 .. 3e-2 in every precision mode
    assert np.median(relg[head]) <= 3e-3 and relg[head].max() <= 5e-2
    assert np.median(relg[~head]) <= 2e-2
