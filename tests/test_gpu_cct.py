"""CCT on the engine: decoder kernels (pixel shuffle, perturbations, masks) and every auxiliary decoder
against the CPU oracle with identical random draws; a whole SSLCCT step against the reference-generated
golden (tests/golden/cct_step_65.npz)."""
import os
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sseg_oracle as O
from oracle import cct_oracle as C

from conftest import TEST_PRECISIONS, assert_loss_yardstick, assert_energy_yardstick

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


def rel_q(a, b, frac=2e-3):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    err = (a - b).abs() / b.abs().max().clamp_min(1e-30)
    return float(err.kthvalue(max(1, int(err.numel() * (1 - frac)))).values)


def test_pixel_shuffle_and_perturb_kernels(ops):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 84, 5, 7, generator=g)
    xc = x.clone().requires_grad_(True)
    ref = F.pixel_shuffle(xc, 2)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    out = ops.pixel_shuffle2(xg, 21)
    assert out.shape == (2, 32, 10, 14) and torch.equal(out[:, :21].cpu(), ref.detach())
    assert float(out[:, 21:].abs().max()) == 0.0
    wp = torch.zeros(2, 32, 10, 14)
    wp[:, :21] = w
    (out * wp.cuda()).sum().backward()
    assert torch.equal(xg.grad.cpu(), xc.grad)
    # perturbations
    x = torch.randn(2, 64, 9, 11, generator=g)
    pm = (torch.rand(2, 1, 9, 11, generator=g) > 0.4).float()
    cs = torch.rand(2, 64, generator=g)
    nz = torch.rand(64, 9, 11, generator=g) - 0.5
    xc = x.clone().requires_grad_(True)
    ref = (xc * pm * cs.view(2, 64, 1, 1))
    ref = ref * nz.unsqueeze(0) + ref
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    out = ops.perturb(xg, pm.cuda(), cs.cuda(), nz.cuda())
    (out * w.cuda()).sum().backward()
    assert rel(out, ref) <= 1e-6 and rel(xg.grad, xc.grad) <= 1e-6
    assert rel(ops.channel_mean(x.cuda().contiguous(memory_format=CL)), x.mean(1, keepdim=True)) <= 1e-6
    lg = torch.randn(2, 21, 33, 35, generator=g)
    lg[0, :, 0, 0] = 1.0                               # an all-tie pixel: argmax = 0
    assert torch.equal(ops.argmax_nonzero_mask(lg.cuda()).cpu()[:, 0], (lg.argmax(1) > 0).float())


@pytest.mark.parametrize('kind', C.KINDS)
def test_auxiliary_decoder_matches_oracle(ops, kind):
    from pixelssl_b200.ssl_algorithm import ssl_cct as E
    g = torch.Generator().manual_seed(3)
    cin, nc = 256, 21
    st = C.init_decoders(5, 1, in_channels=cin)
    cls = {'vat': lambda: E.VATDecoder(8, cin, nc, xi=1e-6, eps=2.0), 'drop': lambda: E.DropOutDecoder(8, cin, nc, 0.5, True),
           'cut': lambda: E.CutOutDecoder(8, cin, nc, erase=0.4), 'context': lambda: E.ContextMaskingDecoder(8, cin, nc),
           'object': lambda: E.ObjectMaskingDecoder(8, cin, nc), 'fd': lambda: E.FeatureDropDecoder(8, cin, nc),
           'fn': lambda: E.FeatureNoiseDecoder(8, cin, nc, 0.3)}[kind]
    dec = cls().cuda()
    dec.load_state_dict({k.replace('auxiliary_decoders.0.', ''): v for k, v in st.items()})
    dec.train()
    x = torch.randn(2, cin, 9, 9, generator=g)
    main = torch.randn(2, nc, 65, 65, generator=g)
    main[:, 0] += 0.8                                  # some background so the masks are not trivial
    cfg = {'xi': 1e-6, 'eps': 2.0, 'drop_rate': 0.5, 'erase': 0.4, 'uniform': 0.3}
    stc = {k: v.clone().requires_grad_(True) for k, v in st.items()}
    xc = x.clone().requires_grad_(True)
    random.seed(1); np.random.seed(2); torch.manual_seed(3)
    ref = C.decoder_forward(stc, 0, kind, xc, main, cfg)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    random.seed(1); np.random.seed(2); torch.manual_seed(3)
    out = dec(xg, pred_of_main_decoder=main.cuda())
    assert out.shape[1] == 32 and float(out[:, nc:].abs().max()) == 0.0
    wp = torch.zeros(2, 32, 72, 72)
    wp[:, :nc] = w
    (out * wp.cuda()).sum().backward()
    tol = 5e-3 if kind == 'vat' else 2e-5             # VAT: direction of a normalised gradient (amplifies round-off)
    # The decoders are ReLU networks: an activation within round-off of zero takes either branch, and ONE such flip
    # moves isolated gradient entries by percents of the maximum (measured: the same single element, 3e-2, in the cut /
    # context / fd cases whenever the accumulation order of the first convolution changes; VAT's normalised
    # adversarial direction flips a few more).  So gradients are compared on all
    # but the worst 0.2 % of the entries (1 % for VAT) and the outputs, which are continuous, on every entry.
    cmp = (lambda a, b: rel_q(a, b, 1e-2)) if kind == 'vat' else rel_q
    e_out, e_in = rel(out[:, :nc], ref), cmp(xg.grad, xc.grad)
    print('%s: out %.2e d/dx %.2e (max %.2e)' % (kind, e_out, e_in, rel(xg.grad, xc.grad)))
    assert e_out <= tol and e_in <= tol * 5
    for n, p in dec.named_parameters():
        assert cmp(p.grad, stc['auxiliary_decoders.0.' + n].grad) <= tol * 10, n


def test_cct_step_golden(ops):
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, 'cct_step_65.npz'))
    size = int(g['size'])
    cfg = {'ssl_algorithm': 'ssl_cct', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1000,
           'cons_scale': 30.0, 'cons_rampup_epochs': 0, 'ad_lr_scale': 10.0, 'vat_dec_num': 1, 'drop_dec_num': 1,
           'cut_dec_num': 1, 'context_dec_num': 1, 'object_dec_num': 1, 'fd_dec_num': 1, 'fn_dec_num': 1,
           'batch_size': 4, 'unlabeled_batch_size': 2, 'models': {'model': 'deeplabv2'}}
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
    st = O.randomize_bn_affine(O.init_deeplabv2(101, cls_bias_std=0.01), 102)
    sd = {'module.main_model.model.' + k: v for k, v in st.items()}
    sd.update({'module.' + k: v for k, v in C.init_decoders(103, 7).items()})
    alg.model.load_state_dict(sd, strict=True)
    img, lab = O.synthetic_batch(800, 4, 2, size, size)
    random.seed(7); np.random.seed(8); torch.manual_seed(9)
    alg._train([((img,), (lab,))], 0)
    t, c = float(alg.meters['task_loss'].val), float(alg.meters['cons_loss'].val)
    print('cct losses', t, float(g['task_loss']), c, float(g['cons_loss']))
    t64 = np.load(os.path.join(G, 'fp64_truth_algs.npz'))        # the oracle in fp64 on the same step (make_golden.py)
    assert_loss_yardstick(t, float(g['task_loss']), float(t64['cct_task_loss']), 'task_loss')
    assert_loss_yardstick(c, float(g['cons_loss']), float(t64['cct_cons_loss']), 'cons_loss')
    np.testing.assert_allclose([grp['lr'] for grp in alg.optimizer.param_groups], g['lrs'], rtol=1e-12)
    dnames = [n for i in range(7) for n, _ in C.decoder_param_shapes(i)]
    dp = dict(alg.model.module.named_parameters())
    sq = np.array([float((dp[n].grad.double() ** 2).sum()) for n in dnames])
    print(assert_energy_yardstick(sq, g['dec_grad_checksum'], t64['cct_dec_grad_checksum'], 'cct decoder grads',
                                  floor_med=1e-3, floor_max=1e-2))
    names = [n for n, _, _ in O.deeplabv2_param_shapes()]
    sp = dict(alg.model.module.main_model.model.named_parameters())
    sq = np.array([float((sp[n].grad.double() ** 2).sum()) for n in names])
    print(assert_energy_yardstick(sq, g['grad_checksum'], t64['cct_grad_checksum'], 'cct encoder grads'))
