"""BASELINE.json's configurations at their FULL sizes on the wgmma path bench.py measures (fp16-pair x3): every algorithm must step with
finite losses and a silent pipeline watchdog, and the size-independent properties of the hot kernels must hold on
full-size tensors (the oracle cannot run these sizes in seconds; small-size parity is in the other test files).

  C2 MT        DeepLab-v2-R101, 8+8 x 513x513           C3 CutMix  DeepLab-v2-R101, 8+8 x 513x513
  C4 GCT       PSPNet-R50, per GPU 1+1 x 713x713        C5 CCT     DeepLab-v2-R101, per GPU 2+2 x 513x513, 11 decoders
  AdvSSL       DeepLab-v2-R101, 2+2 x 513x513"""
import random

import numpy as np
import pytest
import torch

from oracle import sseg_oracle as O

pytestmark = pytest.mark.gpu
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 20, 'log_freq': 10 ** 6}


@pytest.fixture(scope='module')
def ops():
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    from pixelssl_b200 import ops as _ops
    _ops.set_conv_precision('f16x3')
    yield _ops
    _ops.set_conv_precision('fp32')


def _step(ops, cfg, lbs, ubs, size, steps=2):
    from pixelssl_b200 import runner
    random.seed(1); np.random.seed(2); torch.manual_seed(3)
    alg = runner.build_algorithm(runner.build_args(dict(BASE, batch_size=lbs + ubs, unlabeled_batch_size=ubs, **cfg),
                                                   iters_per_epoch=662))
    batches = [tuple((t,) for t in O.synthetic_batch(40 + i, lbs + ubs, lbs, size, size)) for i in range(steps)]
    alg._train(batches, 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    vals = {k: float(alg.meters[k].val) for k in alg.meters.keys() if 'loss' in k}
    assert vals and all(np.isfinite(v) for v in vals.values()), vals
    del alg
    torch.cuda.empty_cache()
    return vals


def test_c2_mean_teacher_full_size(ops):
    v = _step(ops, {'ssl_algorithm': 'ssl_mt', 'cons_for_labeled': False, 'cons_scale': 1.0, 'cons_rampup_epochs': 3,
                    'ema_decay': 0.99}, 8, 8, 513)
    assert 1.0 < v['s_task_loss'] < 20.0         # ln(21) = 3.04 plus random-init spread


def test_c2_full_size_step_matches_the_cpu_oracle(ops):
    """Parity at the benchmark's image size (513x513, the tile-edge cases 513 -> 257 -> 129 -> 65 -> 33 of every
    kernel): one Mean-Teacher step at batch 2+2 on the fp16-pair tensor-core path against the CPU oracle (the
    restatement of ssl_mt.py:124-224 pinned to the reference at 97x97 and 257x257).  Losses within the north_star's
    1e-3; per-tensor gradient energies within the reference's own fp32 noise level measured at the smaller sizes
    (median 1.5e-3, tail 3e-2; tests/test_gpu_model.py) times a small factor."""
    from pixelssl_b200 import runner
    size, lbs, ubs = 513, 2, 2
    cfg = dict(BASE, ssl_algorithm='ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=1, ema_decay=0.99,
               batch_size=lbs + ubs, unlabeled_batch_size=ubs, epochs=2)
    alg = runner.build_algorithm(runner.build_args(cfg, iters_per_epoch=5))
    s0 = O.randomize_bn_affine(O.init_deeplabv2(11, cls_bias_std=0.01), 12)
    t0 = O.randomize_bn_affine(O.init_deeplabv2(21, cls_bias_std=0.01), 22)
    alg.s_model.load_state_dict({'module.model.' + k: v for k, v in s0.items()})
    alg.t_model.load_state_dict({'module.model.' + k: v for k, v in t0.items()})
    img, lab = O.synthetic_batch(100, lbs + ubs, lbs, size, size)
    alg._train([((img,), (lab,))], 0)
    torch.cuda.synchronize()
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0
    mt = O.MTOracle(s0, t0, lr=0.00025, momentum=0.9, weight_decay=0.0005, max_iters=10, cons_scale=1.0,
                    rampup_steps=1, ema_decay=0.99, cons_for_labeled=False)
    ref = mt.step(img, lab, lbs)
    for key in ('s_task_loss', 't_task_loss', 'cons_loss'):
        got, want = float(alg.meters[key].val), float(ref[key])
        assert abs(got - want) <= 1e-3 * max(abs(want), 1e-2), (key, got, want)
    names = mt.names
    sp = dict(alg.s_model.module.model.named_parameters())
    e = np.array([abs(float((sp[n].grad.double() ** 2).sum()) - float((ref['grads'][n].double() ** 2).sum())) /
                  max(float((ref['grads'][n].double() ** 2).sum()), 1e-300) for n in names])
    print('513x513 step vs CPU oracle: grad energy rel median %.2e p95 %.2e max %.2e (%s)' % (
        np.median(e), np.percentile(e, 95), e.max(), names[int(e.argmax())]))
    assert np.median(e) <= 1e-2 and np.percentile(e, 95) <= 5e-2 and e.max() <= 2e-1
    del alg
    torch.cuda.empty_cache()


def test_c3_cutmix_full_size(ops):
    v = _step(ops, {'ssl_algorithm': 'ssl_cutmix', 'cons_scale': 20.0, 'cons_rampup_epochs': 0, 'cons_threshold': 0.97,
                    'ema_decay': 0.99, 'mask_prop_range': (0.5, 0.5)}, 8, 8, 513)
    assert 1.0 < v['task_loss'] < 20.0 and v['cons_loss'] >= 0.0


def test_c4_gct_pspnet_full_size(ops):
    v = _step(ops, {'ssl_algorithm': 'ssl_gct', 'models': {'model': 'pspnet'}, 'backbone': 'resnet50',
                    'ssl_mode': 'gct', 'fc_ssl_scale': 1.0, 'dc_ssl_scale': 100.0, 'dc_threshold': 0.6, 'dc_rampup_epochs': 5,
                    'fd_lr': 1e-4, 'fd_scale': 10.0, 'mu': 0.5, 'nu': 1, 'im_size': 713}, 2, 2, 713, steps=1)
    assert 1.0 < v['l_task_loss'] < 20.0 and 1.0 < v['r_task_loss'] < 20.0


def test_c5_cct_full_size(ops):
    v = _step(ops, {'ssl_algorithm': 'ssl_cct', 'cons_scale': 30.0, 'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0,
                    'vat_dec_num': 1, 'drop_dec_num': 2, 'cut_dec_num': 2, 'context_dec_num': 1, 'object_dec_num': 1,
                    'fd_dec_num': 2, 'fn_dec_num': 2}, 2, 2, 513, steps=1)
    assert 1.0 < v['task_loss'] < 20.0


def test_advssl_full_size(ops):
    v = _step(ops, {'ssl_algorithm': 'ssl_adv', 'adv_for_labeled': True, 'labeled_adv_scale': 0.01,
                    'unlabeled_adv_scale': 0.001, 'discriminator_lr': 1e-4, 'discriminator_scale': 1.0,
                    'unlabeled_for_discriminator': True}, 2, 2, 513, steps=1)
    assert 1.0 < v['task_loss'] < 20.0


def test_full_size_kernel_properties(ops):
    g = torch.Generator(device='cuda').manual_seed(5)
    n, c, h, w = 8, 21, 513, 513
    s = torch.randn(n, c, h, w, device='cuda', generator=g)
    t = torch.randn(n, c, h, w, device='cuda', generator=g)
    # MSE consistency: linear in the scale, gradient = 2*scale*(s - t)/N exactly the elementwise formula
    l1, g1 = ops.mse_consistency_raw(s, t, 1.0, True)
    l3, g3 = ops.mse_consistency_raw(s, t, 3.0, True)
    assert abs(float(l3) - 3.0 * float(l1)) <= 1e-6 * abs(float(l3))
    ref = (s - t) * (2.0 / s.numel())
    assert float((g1 - ref).abs().max()) <= 1e-6 * float(ref.abs().max())
    assert abs(float(l1) - float(((s - t).double() ** 2).mean())) <= 1e-6 * float(l1)
    # CutMix mix with a {0,1} mask picks exactly one operand: mix(a,b,m) + mix(b,a,m) == a + b bit for bit
    a = torch.randn(4, 3, h, w, device='cuda', generator=g)
    b = torch.randn(4, 3, h, w, device='cuda', generator=g)
    m = (torch.rand(4, 1, h, w, device='cuda', generator=g) < 0.5).float()
    ab, ba = ops.cutmix_mix(m, a, b), ops.cutmix_mix(m, b, a)
    assert torch.equal(torch.where(m.bool().expand_as(a), a, b), ab)
    assert torch.equal(ab + ba, a + b)
    # softmax rows sum to one; confusion matrix counts every valid pixel once
    p = ops.softmax_planar(s)
    assert float((p.sum(1) - 1.0).abs().max()) <= 2e-6
    gt = torch.randint(0, c, (n, 1, h, w), device='cuda', generator=g).float()
    gt[torch.rand(n, 1, h, w, device='cuda', generator=g) < 0.05] = 255.0
    cm = torch.zeros(c, c, dtype=torch.int64, device='cuda')
    ops.confusion_matrix_(cm, p, gt)
    assert int(cm.sum()) == int((gt < c).sum())
    assert torch.equal(cm.sum(1), torch.bincount(gt[gt < c].long(), minlength=c))
    # separable Gaussian blur is a partition of unity (reflection padding): constants stay constant, mass of a
    # centred impulse is preserved
    x = torch.full((2, 1, 713, 713), 0.37, device='cuda')
    for k in (45, 89, 179):
        y = ops.gaussian_blur(x, k)
        assert float((y - 0.37).abs().max()) <= 2e-6
    imp = torch.zeros(1, 1, 713, 713, device='cuda')
    imp[0, 0, 356, 356] = 1.0
    assert abs(float(ops.gaussian_blur(imp, 179).double().sum()) - 1.0) <= 1e-5
