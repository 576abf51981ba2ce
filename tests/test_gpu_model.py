"""GPU parity of the whole DeepLab-v2 forward and of complete training steps (SupOnly, Mean
Teacher, CutMix) against vectors produced by the UNMODIFIED reference (tests/golden/*.npz, see
oracle/make_golden.py) and against the CPU oracle.

Tolerances.  Per-kernel parity is held to 1e-5..1e-4 in tests/test_gpu_ops.py.  For the WHOLE
101-layer random-init network with train-mode BN on small maps the function itself is
ill-conditioned: a 1e-7 relative input perturbation moves the logits by 9e-5, and the
reference's own fp32 evaluation is 3.5e-4 (logits) / median 1.5e-3, max 2.9e-2 (step-0 per-tensor
gradient energy) away from exact arithmetic, growing to median 8e-2 by the second step
(tests/golden/fp64_truth.npz = the oracle evaluated in fp64, oracle/make_golden.py:golden_fp64).
So whole-network checks use that measured noise as the yardstick: the engine's deviation from
the fp64 truth must stay within FACTOR x the reference-fp32's deviation from the same truth
(plus small floors), and logits within the north_star 1e-3."""
import os

import numpy as np
import pytest
import torch

from oracle import sseg_oracle as O

from conftest import TEST_PRECISIONS

pytestmark = pytest.mark.gpu
FACTOR = 3.0
G = os.path.join(os.path.dirname(__file__), 'golden')


@pytest.fixture(scope='module', params=TEST_PRECISIONS)
def eng(request):
    """Every whole-network / whole-step golden runs once per convolution precision mode (tests/conftest.py):
    the exact FFMA path AND the wgmma paths that bench.py measures are held to the same reference vectors."""
    if not torch.cuda.is_available():
        pytest.skip('needs a GPU')
    import pixelssl_b200
    from pixelssl_b200 import ops
    ops.set_conv_precision(request.param)
    yield pixelssl_b200
    ops.set_conv_precision('fp32')


def _state(seeds):
    return O.randomize_bn_affine(O.init_deeplabv2(int(seeds[0]), cls_bias_std=0.01), int(seeds[1]))


def _load(model, state):
    model.load_state_dict({'module.model.' + k: v for k, v in state.items()}, strict=True)


def _checks(tensors):
    return np.array([[float(t.double().sum()), float((t.double() ** 2).sum())] for t in tensors])


def _cfg(alg, **kw):
    cfg = {'ssl_algorithm': alg, 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005,
           'output_stride': 16, 'backbone': 'resnet101', 'epochs': 2, 'log_freq': 1000}
    cfg.update(kw)
    return cfg


def test_state_dict_keys_match_reference_layout(eng):
    from pixelssl_b200 import runner
    args = runner.build_args(_cfg('ssl_null', batch_size=2, unlabeled_batch_size=0), iters_per_epoch=5)
    alg = runner.build_algorithm(args)
    keys = list(alg.model.state_dict().keys())
    want = ['module.model.' + n for n, _, _ in O.deeplabv2_param_shapes()]
    assert [k for k in keys if not any(s in k for s in ('running_', 'num_batches'))] == want
    for n, shape, _ in O.deeplabv2_param_shapes():
        assert tuple(alg.model.state_dict()['module.model.' + n].shape) == tuple(shape)
    assert sum(p.numel() for p in alg.model.parameters()) == 44048532


def test_deeplabv2_forward_golden(eng):
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, 'deeplabv2_forward_129.npz'))
    args = runner.build_args(_cfg('ssl_null', batch_size=2, unlabeled_batch_size=0), iters_per_epoch=5)
    alg = runner.build_algorithm(args)
    _load(alg.model, _state(g['seed']))
    alg.model.train()
    size, batch = int(g['size']), int(g['batch'])
    img, _ = O.synthetic_batch(int(g['data_seed']), batch, batch, size, size)
    with torch.no_grad():
        resulter, _ = alg.model.forward((img.cuda(),))
    logits = resulter['pred'][0]
    ref = torch.tensor(g['logits'])
    truth = torch.tensor(np.load(os.path.join(G, 'fp64_truth.npz'))['fwd_logits'])
    err_ref = float((logits.cpu() - ref).abs().max() / ref.abs().max())
    err_truth = float((logits.cpu() - truth).abs().max() / truth.abs().max())
    ref_truth = float((ref - truth).abs().max() / truth.abs().max())
    assert err_ref <= 1e-3 and err_truth <= 1e-3, (err_ref, err_truth, ref_truth)       # north_star tolerance
    assert err_truth <= FACTOR * ref_truth, (err_truth, ref_truth)                      # fp32 noise yardstick
    lat = resulter['sslcct_ad_inp']
    cs = np.array([float(lat.double().sum()), float((lat.double() ** 2).sum())])
    np.testing.assert_allclose(cs[1], g['latent_checksum'][0][1], rtol=2e-3)
    # lazily activated prediction == softmax of the engine's own logits (kernel check)
    act = resulter['activated_pred'][0]
    assert float((act - torch.softmax(logits, 1)).abs().max()) <= 1e-6
    # BN running buffers after one training forward
    bufs = [b for n, b in alg.model.named_buffers() if 'num_batches' not in n]
    got = _checks(bufs)
    np.testing.assert_allclose(got[:, 1], g['running_checksum'][:, 1], rtol=2e-3)


def _rel_energy(a, truth):
    return np.abs(a[:, 1] - truth[:, 1]) / np.maximum(truth[:, 1], 1e-300)


def _assert_within_yardstick(names, got, ref32, truth, what, floor_med=3e-4, floor_max=3e-3):
    """got / ref32 / truth: [n_tensors, 2] (sum, sum of squares).  Engine-vs-truth deviation of the
    per-tensor energy must be within FACTOR x the reference-fp32-vs-truth deviation."""
    e, r = _rel_energy(got, truth), _rel_energy(ref32, truth)
    msg = '%s: engine median %.2e p95 %.2e max %.2e (worst %s) | reference fp32 median %.2e p95 %.2e max %.2e' % (
        what, np.median(e), np.percentile(e, 95), e.max(), names[int(e.argmax())],
        np.median(r), np.percentile(r, 95), r.max())
    assert np.median(e) <= FACTOR * np.median(r) + floor_med, msg
    assert np.percentile(e, 95) <= FACTOR * np.percentile(r, 95) + floor_max, msg
    assert e.max() <= FACTOR * r.max() + floor_max, msg
    return msg


def _assert_loss(got, ref32, truth, what, later_step=False):
    """later_step: after the first SGD update the fp32 and exact trajectories have already diverged
    chaotically (reference fp32 itself is 1e-3..2e-2 off), so the factor is doubled and a 1e-2 floor added."""
    tol = FACTOR * abs(ref32 - truth) + 1e-4 * max(abs(truth), 1e-2)
    if later_step:
        tol = 2 * tol + 1e-2 * max(abs(truth), 1e-2)
    assert abs(got - truth) <= tol, (what, got, ref32, truth)


def test_null_step_golden(eng):
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, 'null_step_65.npz'))
    size = int(g['size'])
    args = runner.build_args(_cfg('ssl_null', batch_size=2, unlabeled_batch_size=0, ignore_unlabeled=True), iters_per_epoch=5)
    alg = runner.build_algorithm(args)
    _load(alg.model, _state((41, 42)))
    img, lab = O.synthetic_batch(300, 2, 2, size, size)
    alg._train([((img,), (lab,))], 0)
    names = [n for n, _, _ in O.deeplabv2_param_shapes()]
    sp = dict(alg.model.module.model.named_parameters())
    t = np.load(os.path.join(G, 'fp64_truth.npz'))
    _assert_loss(float(alg.meters['task_loss'].val), float(g['task_loss']), float(t['null_task_loss']), 'task_loss')
    print(_assert_within_yardstick(names, _checks([sp[n].grad for n in names]), g['grad_checksum'],
                                   t['null_grad_checksum'], 'SupOnly grads'))
    _assert_within_yardstick(names, _checks([sp[n] for n in names]), g['param_checksum'], t['null_param_checksum'],
                             'SupOnly params', floor_med=1e-6, floor_max=1e-4)


def _run_mt_golden(golden, truth):
    """SSLMT steps on the seeds / batches of oracle/make_golden.py:golden_mt, held to the reference-generated fixture
    ``golden`` with the fp64 oracle evaluation ``truth`` as the noise yardstick."""
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, golden))
    size, lbs, ubs = int(g['size']), int(g['lbs']), int(g['ubs'])
    args = runner.build_args(_cfg('ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=1,
                                  ema_decay=0.99, batch_size=lbs + ubs, unlabeled_batch_size=ubs), iters_per_epoch=5)
    alg = runner.build_algorithm(args)
    _load(alg.s_model, _state(g['s_seed']))
    _load(alg.t_model, _state(g['t_seed']))
    names = [str(n) for n in g['names']]
    t64 = np.load(os.path.join(G, truth))
    for k in range(int(g['steps'])):
        img, lab = O.synthetic_batch(int(g['data_seed']) + k, lbs + ubs, lbs, size, size)
        alg._train([((img,), (lab,))], k)
        sp = dict(alg.s_model.module.model.named_parameters())
        tp = dict(alg.t_model.module.model.named_parameters())
        for key in ('s_task_loss', 't_task_loss', 'cons_loss'):
            _assert_loss(float(alg.meters[key].val), float(g['%s_%d' % (key, k)]), float(t64['mt_%s_%d' % (key, k)]),
                         '%s step %d' % (key, k), later_step=k > 0)
        print(_assert_within_yardstick(names, _checks([sp[n].grad for n in names]), g['grad_checksum_%d' % k],
                                       t64['mt_grad_checksum_%d' % k], 'MT grads step %d' % k))
        _assert_within_yardstick(names, _checks([sp[n] for n in names]), g['s_param_checksum_%d' % k],
                                 t64['mt_s_param_checksum_%d' % k], 'MT student params step %d' % k, 1e-6, 1e-4)
        _assert_within_yardstick(names, _checks([tp[n] for n in names]), g['t_param_checksum_%d' % k],
                                 t64['mt_t_param_checksum_%d' % k], 'MT teacher params step %d' % k, 1e-6, 1e-4)
        lrs = np.array([grp['lr'] for grp in alg.s_optimizer.param_groups])
        np.testing.assert_allclose(lrs, g['lr_%d' % k], rtol=1e-12)
        if k == 0:
            # element-wise check on a few step-0 gradients (step 0 is the well-conditioned one)
            for n in ('backbone.conv1.weight', 'classifier.conv2d_list.0.bias', 'backbone.layer4.2.conv3.weight'):
                f = sp[n].grad.contiguous().reshape(-1).cpu()
                stride = max(1, f.numel() // 4096)
                mine = f[::stride][:4096].numpy()
                ref, tru = g['grad_0/%s' % n], t64['mt_grad_0/%s' % n]
                yard = np.abs(ref - tru).max()
                assert np.abs(mine - tru).max() <= FACTOR * yard + 1e-3 * np.abs(tru).max(), (n, np.abs(mine - tru).max(), yard)
    from pixelssl_b200 import ops
    assert ops.conv_tc_status() == 0 and ops.h16_status() == 0


def test_mt_steps_golden(eng):
    """Three SSLMT steps at 97x97 (ssl_mt.py:124-224)."""
    _run_mt_golden('mt_steps_97.npz', 'fp64_truth.npz')


def test_mt_step_golden_257(eng):
    """One SSLMT step at 257x257, batch 2+2: feature maps 129 -> 65 -> 33 -> 17 -> 17, i.e. odd edges on every level
    and several 128-pixel tiles per row, the tile-edge cases the 513x513 benchmark configuration hits."""
    _run_mt_golden('mt_steps_257.npz', 'fp64_truth_257.npz')


def test_cutmix_step_golden(eng):
    from pixelssl_b200 import runner
    g = np.load(os.path.join(G, 'cutmix_step_65.npz'))
    size = int(g['size'])
    args = runner.build_args(_cfg('ssl_cutmix', cons_scale=20.0, cons_rampup_epochs=0, ema_decay=0.99,
                                  cons_threshold=float(g['cons_threshold']), batch_size=6, unlabeled_batch_size=4,
                                  mask_prop_range='(0.5, 0.5)'), iters_per_epoch=5)
    alg = runner.build_algorithm(args)
    _load(alg.s_model, _state((51, 52)))
    _load(alg.t_model, _state((61, 62)))
    img, lab = O.synthetic_batch(400, 6, 2, size, size)
    np.random.seed(int(g['mask_seed']))
    alg._train([((img,), (lab,))], 0)
    names = [n for n, _, _ in O.deeplabv2_param_shapes()]
    sp = dict(alg.s_model.module.model.named_parameters())
    tp = dict(alg.t_model.module.model.named_parameters())
    t = np.load(os.path.join(G, 'fp64_truth.npz'))
    for key in ('task_loss', 'cons_loss'):
        _assert_loss(float(alg.meters[key].val), float(g[key]), float(t['cutmix_' + key]), key)
    print(_assert_within_yardstick(names, _checks([sp[n].grad for n in names]), g['grad_checksum'],
                                   t['cutmix_grad_checksum'], 'CutMix grads'))
    _assert_within_yardstick(names, _checks([sp[n] for n in names]), g['s_param_checksum'], t['cutmix_s_param_checksum'],
                             'CutMix student params', 1e-6, 1e-4)
    _assert_within_yardstick(names, _checks([tp[n] for n in names]), g['t_param_checksum'], t['cutmix_t_param_checksum'],
                             'CutMix teacher params', 1e-6, 1e-4)


def test_checkpoint_roundtrip(eng, tmp_path):
    """Checkpoint dict layout of ssl_mt.py:296-322 (keys, 'module.' prefix) and resume."""
    from pixelssl_b200 import runner
    args = runner.build_args(_cfg('ssl_mt', cons_for_labeled=False, cons_scale=1.0, cons_rampup_epochs=1,
                                  batch_size=2, unlabeled_batch_size=1), iters_per_epoch=5)
    args.checkpoint_path = str(tmp_path)
    alg = runner.build_algorithm(args)
    img, lab = O.synthetic_batch(1, 2, 1, 33, 33)
    alg._train([((img,), (lab,))], 0)
    alg.save_checkpoint(3)
    ck = torch.load(os.path.join(str(tmp_path), 'checkpoint_3.ckpt'), weights_only=False)
    assert set(ck.keys()) == {'algorithm', 'epoch', 's_model', 't_model', 's_optimizer', 's_lrer'}
    assert ck['algorithm'] == 'ssl_mt' and all(k.startswith('module.model.') for k in ck['s_model'])
    assert 'momentum_buffer' in ck['s_optimizer']['state'][0]
    alg2 = runner.build_algorithm(args)
    args.resume = os.path.join(str(tmp_path), 'checkpoint_3.ckpt')
    assert alg2.load_checkpoint() == 3
    for (n1, p1), (n2, p2) in zip(alg.s_model.named_parameters(), alg2.s_model.named_parameters()):
        assert torch.equal(p1, p2), n1
