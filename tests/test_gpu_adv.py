"""AdvSSL on the engine: kernel-level parity of the discriminator tail against the CPU oracle, and a
whole SSLADV step against the reference-generated golden (tests/golden/adv_step_65.npz)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sseg_oracle as O
from oracle import adv_oracle as A

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
    """Like rel() but ignoring the worst `frac` of the elements: a LeakyReLU pre-activation that is
    exactly 0.0 on the CPU and 1e-8 on the GPU flips one derivative (1 vs 0.2), which perturbs the
    4x4x21 input-gradient patch under it - a kink of the function, not a kernel error."""
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    err = (a - b).abs() / b.abs().max().clamp_min(1e-30)
    k = max(1, int(err.numel() * (1 - frac)))
    return float(err.kthvalue(k).values)


def test_layout_and_onehot_kernels(ops):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 21, 37, 41, generator=g)
    y = ops.planar_to_nhwc(x.cuda())
    assert y.shape == (2, 32, 37, 41) and y.is_contiguous(memory_format=CL)
    assert torch.equal(y[:, :21].cpu(), x) and float(y[:, 21:].abs().max()) == 0.0
    xg = x.cuda().requires_grad_(True)
    w = torch.randn(2, 32, 37, 41, generator=g).cuda()
    (ops.planar_to_nhwc(xg) * w).sum().backward()
    assert torch.equal(xg.grad, w[:, :21].contiguous())
    a, b = torch.randn(2, 3, 9, 9, generator=g), torch.randn(2, 21, 9, 9, generator=g)
    c = ops.cat_planar_to_nhwc([a.cuda(), b.cuda()])
    assert torch.equal(c[:, :24].cpu(), torch.cat((a, b), 1)) and float(c[:, 24:].abs().max()) == 0.0
    _, lab = O.synthetic_batch(3, 2, 2, 19, 23)
    oh = ops.onehot_nhwc(lab.cuda(), 21)
    assert torch.equal(oh[:, :21].cpu(), A.onehot_gt(lab)) and float(oh[:, 21:].abs().max()) == 0.0


def test_leaky_relu_and_masked_bce(ops):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 64, 9, 11, generator=g)
    xc = x.clone().requires_grad_(True)
    w = torch.randn(2, 64, 9, 11, generator=g)
    (F.leaky_relu(xc, 0.2) * w).sum().backward()
    xg = x.cuda().contiguous(memory_format=CL).requires_grad_(True)
    yg = ops.leaky_relu(xg, 0.2)
    (yg * w.cuda()).sum().backward()
    assert rel(yg, F.leaky_relu(x, 0.2)) == 0.0 and rel(xg.grad, xc.grad) == 0.0
    pred = torch.randn(3, 1, 33, 35, generator=g) * 3
    _, lab = O.synthetic_batch(4, 3, 3, 33, 35)
    for is_real in (True, False):
        for labels in (lab, None):
            pc = pred.clone().requires_grad_(True)
            p, t = A.fcd_preprocess(pc, labels, is_real)
            ref = A.fcd_criterion(p, t)
            (ref * torch.tensor([1.0, 2.0, 3.0])).sum().backward()
            pg = pred.cuda().requires_grad_(True)
            out = ops.bce_logits_masked(pg, None if labels is None else labels.cuda(), 1.0 if is_real else 0.0)
            (out * torch.tensor([1.0, 2.0, 3.0]).cuda()).sum().backward()
            assert rel(out, ref) <= 1e-6 and rel(pg.grad, pc.grad) <= 1e-5


def test_fc_discriminator_forward_backward(ops):
    from pixelssl_b200.ssl_algorithm.ssl_adv import FCDiscriminator
    st = A.init_fcd(5)
    d = FCDiscriminator(21).cuda()
    d.load_state_dict({k: v for k, v in st.items()})
    g = torch.Generator().manual_seed(3)
    prob = torch.softmax(torch.randn(2, 21, 65, 65, generator=g), 1)
    pc = prob.clone().requires_grad_(True)
    stc = {k: v.clone().requires_grad_(True) for k, v in st.items()}
    ref = A.fcd_forward(stc, pc)
    w = torch.randn(ref.shape, generator=g)
    (ref * w).sum().backward()
    pg = prob.cuda().requires_grad_(True)
    conf = d(pg)[0]['confidence']
    (conf * w.cuda()).sum().backward()
    assert rel(conf, ref) <= 2e-5
    assert rel_q(pg.grad, pc.grad) <= 2e-5 and rel(pg.grad, pc.grad) <= 5e-2
    for n, p in d.named_parameters():
        assert rel_q(p.grad, stc[n].grad) <= 1e-2 and rel(p.grad, stc[n].grad) <= 5e-2, n   # one kink flip touches a whole filter


def test_adam_resume_continues_moments_and_step(ops):
    """Checkpoint resume of the arena Adam (discriminator / flaw detector optimisers, ssl_adv.py:101-102,
    ssl_gct.py:153-154): optimizer.load_state_dict + arena.adopt_optimizer_state must continue exp_avg, exp_avg_sq and
    the bias-correction step exactly like torch.optim.Adam does on resume."""
    from pixelssl_b200.nn.arena import ParamArena
    g = torch.Generator().manual_seed(5)
    w0 = [torch.randn(7, 5, generator=g), torch.randn(12, generator=g)]
    grads = [[torch.randn(7, 5, generator=g), torch.randn(12, generator=g)] for _ in range(4)]
    # torch reference: 4 uninterrupted steps on CPU
    ref = [w.clone().requires_grad_(True) for w in w0]
    opt_ref = torch.optim.Adam(ref, lr=1e-2, betas=(0.9, 0.99))
    for gs in grads:
        for p, gr in zip(ref, gs):
            p.grad = gr.clone()
        opt_ref.step()

    def make():
        m = torch.nn.ParameterList([torch.nn.Parameter(w.clone().cuda()) for w in w0])
        arena = ParamArena(m)
        return m, arena, torch.optim.Adam(list(m), lr=1e-2, betas=(0.9, 0.99))

    m1, a1, o1 = make()
    for gs in grads[:2]:
        for p, gr in zip(m1, gs):
            p.grad.copy_(gr.cuda())
        a1.adam_step(o1)
    state = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in m1.state_dict().items()}
    ostate = o1.state_dict()
    m2, a2, o2 = make()
    m2.load_state_dict(state)
    o2.load_state_dict(ostate)
    a2.adopt_optimizer_state(o2)
    assert a2.steps == 2
    for gs in grads[2:]:
        for p, gr in zip(m2, gs):
            p.grad.copy_(gr.cuda())
        a2.adam_step(o2)
    for p, q in zip(m2, ref):
        assert rel(p, q) <= 1e-6
    st = o2.state_dict()['state']
    assert all(float(v['step']) == 4.0 for v in st.values())


def test_adam_matches_torch(ops):
    g = torch.Generator().manual_seed(4)
    n = 10007
    p0 = torch.randn(n, generator=g)
    q = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([q], lr=1e-3, betas=(0.9, 0.99))
    p, m, v = p0.cuda(), torch.zeros(n).cuda(), torch.zeros(n).cuda()
    for step in range(1, 4):
        gr = torch.randn(n, generator=g)
        q.grad = gr.clone()
        opt.step()
        ops.adam_(p, gr.cuda(), m, v, 1e-3, 0.9, 0.99, 1e-8, 0.0, step)
        assert rel(p, q.data) <= 1e-6


def test_adv_step_golden(ops):
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, 'adv_step_65.npz'))
    size = int(g['size'])
    cfg = {'ssl_algorithm': 'ssl_adv', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
           'log_freq': 1000, 'adv_for_labeled': True, 'labeled_adv_scale': 0.01, 'unlabeled_adv_scale': 0.001,
           'discriminator_lr': 1e-4, 'discriminator_scale': 1.0, 'unlabeled_for_discriminator': True,
           'batch_size': 4, 'unlabeled_batch_size': 2}
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
    st = O.randomize_bn_affine(O.init_deeplabv2(81, cls_bias_std=0.01), 82)
    alg.model.load_state_dict({'module.model.' + k: v for k, v in st.items()})
    alg.d_model.load_state_dict({'module.' + k: v for k, v in A.init_fcd(83).items()})
    img, lab = O.synthetic_batch(600, 4, 2, size, size)
    alg._train([((img,), (lab,))], 0)
    t64 = np.load(os.path.join(G, 'fp64_truth_algs.npz'))        # the oracle in fp64 on the same step (make_golden.py)
    for k in ('task_loss', 'labeled_adv_loss', 'unlabeled_adv_loss', 'fake_d_loss', 'real_d_loss'):
        assert_loss_yardstick(float(alg.meters[k].val), float(g[k]), float(t64['adv_' + k]), k)
    dn = [n for n, _ in A.fcd_shapes()]
    dp = dict(alg.d_model.module.named_parameters())
    sq = np.array([float((dp[n].grad.double() ** 2).sum()) for n in dn])
    print(assert_energy_yardstick(sq, g['d_grad_checksum'], t64['adv_d_grad_checksum'], 'discriminator grads'))
    cs = np.array([[float(dp[n].double().sum()), float((dp[n].double() ** 2).sum())] for n in dn])
    np.testing.assert_allclose(cs[:, 1], g['d_param_checksum'][:, 1], rtol=1e-4)
    assert abs(alg.d_optimizer.param_groups[0]['lr'] - float(g['d_lr'])) <= 1e-12
    names = [n for n, _, _ in O.deeplabv2_param_shapes()]
    sp = dict(alg.model.module.model.named_parameters())
    sq = np.array([float((sp[n].grad.double() ** 2).sum()) for n in names])
    print(assert_energy_yardstick(sq, g['grad_checksum'], t64['adv_grad_checksum'], 'adv task-model grads'))
