"""The plumbing every SSL algorithm shares through ``_SSLBase``, on the host: all nine algorithms are built on the CPU
with their parameter arenas in host memory, then their checkpoints are saved and resumed, and their epoch and
validation loops run with stubbed per-batch steps.  Nothing here launches a kernel."""
import collections
import gzip
import itertools
import json
import os
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = {'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2, 'log_freq': 1, 'batch_size': 4,
        'unlabeled_batch_size': 2, 'backbone': 'resnet50'}
ALGS = {
    'ssl_null': {'unlabeled_batch_size': 0, 'ignore_unlabeled': True},
    'ssl_mt': {'cons_scale': 1.0, 'cons_rampup_epochs': 3},
    'ssl_cutmix': {'cons_scale': 20.0, 'cons_rampup_epochs': 1, 'cons_threshold': 0.97, 'batch_size': 6,
                   'unlabeled_batch_size': 4},
    'ssl_adv': {'adv_for_labeled': True, 'labeled_adv_scale': 0.01, 'unlabeled_adv_scale': 0.001},
    'ssl_gct': {'fc_ssl_scale': 1.0, 'dc_ssl_scale': 100.0, 'dc_threshold': 0.6, 'dc_rampup_epochs': 5, 'mu': 0.5,
                'nu': 1, 'im_size': 65},
    'ssl_cct': {'cons_scale': 30.0, 'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0},
    'ssl_s4l': {'rotation_scale': 1.0, 'rotated_sup_scale': 1.0},
    'ssl_cps': {'cps_scale': 1.5, 'cps_rampup_epochs': 2},
    'ssl_unimatch': {'uni_threshold': 0.95, 'uni_scale': 1.0, 'uni_rampup_epochs': 4},
}
# checkpoint layouts of the algorithms tests/golden/host_reference.json.gz does not record
CHECKPOINT_KEYS = {
    'ssl_s4l': {'algorithm', 'epoch', 'model', 'optimizer', 'lrer'},
    'ssl_cps': {'algorithm', 'epoch', 'l_model', 'r_model', 'l_optimizer', 'r_optimizer', 'l_lrer', 'r_lrer'},
    'ssl_unimatch': {'algorithm', 'epoch', 'model', 'optimizer', 'lrer'},
}
RAMPUP_EPOCHS = {'ssl_null': 0, 'ssl_mt': 3, 'ssl_cutmix': 1, 'ssl_adv': 0, 'ssl_gct': 5, 'ssl_cct': 5, 'ssl_s4l': 0,
                 'ssl_cps': 2, 'ssl_unimatch': 4}
ITER_LRERS = {'ssl_adv': {'d_lrer'}, 'ssl_gct': {'fd_lrer'}}          # stepped every iteration in any case
VALIDATION_IDS = {'ssl_mt': ('student', 'teacher'), 'ssl_cutmix': ('student', 'teacher'), 'ssl_gct': ('l', 'r'),
                  'ssl_cps': ('l', 'r')}
METERS = ['task_loss', 'cons_loss', 's_task_loss', 't_task_loss', 'labeled_adv_loss', 'unlabeled_adv_loss',
          'fake_d_loss', 'real_d_loss', 'l_task_loss', 'r_task_loss', 'l_dc_loss', 'r_dc_loss', 'l_fc_loss', 'r_fc_loss',
          'l_fd_loss', 'r_fd_loss', 'l_cps_loss', 'r_cps_loss', 'unrotated_task_loss', 'rotated_task_loss',
          'rotation_loss', 'rotation_acc', 's1_loss', 's2_loss', 'fp_loss', 'mask_ratio']
# the step log line after 'step: [..][../..]\tbatch-time: ...\n' with meter k at 0.125 (k + 1)
STEP_LOG = {
    'ssl_null': '  task-sseg\t=>\ttask-loss: 0.125000 (0.125000)\t',
    'ssl_mt': '  student-sseg\t=>\ts-task-loss: 0.375000 (0.375000)\ts-cons-loss: 0.250000 (0.250000)\n'
              '  teacher-sseg\t=>\tt-task-loss: 0.500000 (0.500000)\n',
    'ssl_cutmix': '  student-sseg\t=>\ts-task-loss: 0.125000 (0.125000)\ts-cons-loss: 0.250000 (0.250000)\n',
    'ssl_adv': '  task-sseg\t=>\ttask-loss: 0.125000 (0.125000)\tlabeled-adv-loss: 0.625000 (0.625000)\t'
               'unlabeled-adv-loss: 0.750000 (0.750000)\n'
               '  fc-discriminator\t=>\tfake-d-loss: 0.875000 (0.875000)\treal-d-loss: 1.000000 (1.000000)\n',
    'ssl_gct': '  l-sseg\t=>\tl-task-loss: 1.125000 (1.125000)\tl-dc-loss: 1.375000 (1.375000)\t'
               'l-fc-loss: 1.625000 (1.625000)\n'
               '  r-sseg\t=>\tr-task-loss: 1.250000 (1.250000)\tr-dc-loss: 1.500000 (1.500000)\t'
               'r-fc-loss: 1.750000 (1.750000)\n'
               '  fd\t=>\tl-fd-loss: 1.875000 (1.875000)\tr-fd-loss: 2.000000 (2.000000)\n',
    'ssl_cct': '  task-sseg\t=>\ttask-loss: 0.125000 (0.125000)\tcons-loss: 0.250000 (0.250000)\n',
    'ssl_s4l': '  task-sseg\t=>\tunrotated-task-loss: 2.375000 (2.375000)\trotated-task-loss: 2.500000 (2.500000)\n'
               '  rotation-sseg\t=>\trotation-loss: 2.625000 (2.625000)\trotation-acc: 2.750000 (2.750000)\n',
    'ssl_cps': '  l-sseg\t=>\tl-task-loss: 1.125000 (1.125000)\tl-cps-loss: 2.125000 (2.125000)\n'
               '  r-sseg\t=>\tr-task-loss: 1.250000 (1.250000)\tr-cps-loss: 2.250000 (2.250000)\n',
    'ssl_unimatch': '  task-sseg\t=>\ttask-loss: 0.125000 (0.125000)\ts1-loss: 2.875000 (2.875000)\t'
                    's2-loss: 3.000000 (3.000000)\tfp-loss: 3.125000 (3.125000)\tmask-ratio: 3.2500 (3.2500)\n',
}


@pytest.fixture
def build(monkeypatch):
    """Builds an algorithm through runner.build_algorithm with every parameter arena in host memory."""
    from pixelssl_b200 import runner
    from pixelssl_b200.nn.arena import EngineParallel, ParamArena

    def host_cuda(self, device=None):
        self.arena = ParamArena(self.module)
        return self
    monkeypatch.setattr(EngineParallel, 'cuda', host_cuda)
    return lambda name: runner.build_algorithm(runner.build_args(dict(BASE, ssl_algorithm=name, **ALGS[name]),
                                                                 iters_per_epoch=3))


def _reference_checkpoint_keys():
    with gzip.open(os.path.join(ROOT, 'tests', 'golden', 'host_reference.json.gz'), 'rt') as f:
        return json.load(f)['checkpoint_keys']


def _stub_optimizer_step(optimizer, step):
    """The state torch's SGD / Adam keep after ``step`` steps: momentum buffers, or moments and the step count."""
    g = torch.Generator().manual_seed(step)
    for group in optimizer.param_groups:
        for p in group['params']:
            if isinstance(optimizer, torch.optim.Adam):
                optimizer.state[p] = {'step': torch.tensor(float(step)), 'exp_avg': torch.randn(p.shape, generator=g),
                                      'exp_avg_sq': torch.rand(p.shape, generator=g)}
            else:
                optimizer.state[p] = {'momentum_buffer': torch.randn(p.shape, generator=g)}


def _params(optimizer):
    return [p for group in optimizer.param_groups for p in group['params']]


@pytest.mark.slow
@pytest.mark.parametrize('name', list(ALGS))
def test_checkpoint_round_trip(name, build, tmp_path, caplog):
    """save_checkpoint writes the reference's top-level keys with every state dict; load_checkpoint into a fresh
    instance restores models, schedulers and optimizers, moves the optimizer state into the parameter arenas, and
    refuses a checkpoint of another algorithm."""
    src = build(name)
    src.args.checkpoint_path = str(tmp_path)
    with torch.no_grad():
        for model in src.models.values():
            for v in model.state_dict().values():
                if v.is_floating_point():
                    v.add_(torch.rand_like(v))
    for optimizer in src.optimizers.values():
        _stub_optimizer_step(optimizer, 7)
    for lrer in src.lrers.values():
        lrer.step()
        lrer.step()
    src.save_checkpoint(3)
    path = tmp_path / 'checkpoint_3.ckpt'

    checkpoint = torch.load(path, weights_only=False)
    if name in CHECKPOINT_KEYS:
        assert set(checkpoint) == CHECKPOINT_KEYS[name]
    else:
        assert sorted(checkpoint) == _reference_checkpoint_keys()[name]
    assert checkpoint['algorithm'] == name and checkpoint['epoch'] == 3
    for elements in (src.models, src.optimizers, src.lrers):
        for key, element in elements.items():
            assert checkpoint[key].keys() == element.state_dict().keys(), key
    del checkpoint

    dst = build(name)
    dst.args.resume = str(path)
    assert dst.load_checkpoint() == 3
    for key, model in src.models.items():
        got = dst.models[key].state_dict()
        for k, v in model.state_dict().items():
            assert torch.equal(got[k], v), (key, k)
    for key, lrer in src.lrers.items():
        assert dst.lrers[key].state_dict() == lrer.state_dict(), key
    for key, optimizer in dst.optimizers.items():
        params = _params(optimizer)
        arena = next(m.arena for m in dst.models.values() if id(params[0]) in m.arena._index)
        adam = isinstance(optimizer, torch.optim.Adam)
        assert arena.steps == (7 if adam else 1), key
        fields = (('exp_avg', arena.exp_avg), ('exp_avg_sq', arena.exp_avg_sq)) if adam else (('momentum_buffer', arena.mom),)
        for p, sp in zip(params, _params(src.optimizers[key])):
            offset = arena._index[id(p)][0]
            for field, flat in fields:
                view = arena._view_like(flat, offset, p)
                assert optimizer.state[p][field].data_ptr() == view.data_ptr(), (key, field)
                assert torch.equal(view, src.optimizers[key].state[sp][field]), (key, field)
    if name == 'ssl_s4l':
        assert dst.task_model is dst.model.module.task_model
        assert dst.rotation_classifier is dst.model.module.rotation_classifier
    path.unlink()

    other = tmp_path / 'other.ckpt'
    torch.save({'algorithm': 'ssl_other', 'epoch': 3}, other)
    dst.args.resume = str(other)
    with pytest.raises(SystemExit):
        dst.load_checkpoint()
    assert 'Unmatched SSL algorithm format in checkpoint => required: %s - given: ssl_other' % name in caplog.text


@pytest.mark.slow
@pytest.mark.parametrize('name', list(ALGS))
def test_epoch_and_validation_loops(name, build, monkeypatch):
    """_train: train mode, train_step per batch with (cur_step, total_steps), the step log line, the schedulers per
    iteration or per epoch; _validate: eval mode, validate_step per batch, the metrics of the algorithm's ids."""
    from pixelssl_b200.ssl_algorithm import ssl_base
    from pixelssl_b200.utils import logger
    alg = build(name)
    steps, lrer_steps, validated, emitted = [], [], [], []

    def train_step(inp, gt, cur_step, total_steps):
        steps.append((inp, gt, cur_step, total_steps))
        for k, meter in enumerate(METERS):
            alg.meters.update(meter, 0.125 * (k + 1))
    monkeypatch.setattr(alg, 'train_step', train_step)
    monkeypatch.setattr(alg, 'validate_step', lambda inp, gt: validated.append((inp, gt)))
    for key, lrer in alg.lrers.items():
        monkeypatch.setattr(lrer, 'step', lambda key=key: lrer_steps.append(key))
    monkeypatch.setattr(ssl_base, 'time', types.SimpleNamespace(time=itertools.cycle([0.0, 0.25]).__next__))
    monkeypatch.setattr(logger, 'log_info', emitted.append)
    batches = [((torch.full((2, 3), float(i)),), (torch.full((2, 1), -float(i)),)) for i in range(3)]

    for is_epoch_lrer in (False, True):
        alg.args.is_epoch_lrer = is_epoch_lrer
        for model in alg.models.values():
            model.eval()
        del steps[:], lrer_steps[:], emitted[:]
        alg.train(batches, 2)
        assert [(cur, total) for _, _, cur, total in steps] == [(6 + i, 3 * RAMPUP_EPOCHS[name]) for i in range(3)]
        if not torch.cuda.is_available():           # with CUDA, device_prefetch hands over device copies
            assert all(s[0] is b[0] and s[1] is b[1] for s, b in zip(steps, batches))
        want = {key: 3 if key in ITER_LRERS.get(name, ()) or not is_epoch_lrer else 1 for key in alg.lrers}
        assert collections.Counter(lrer_steps) == want
        assert all(m.training for model in alg.models.values() for m in model.modules())
        assert emitted == ['step: [3][%d/3]\tbatch-time: 0.250 (0.250)\n' % i + STEP_LOG[name] for i in range(3)]

    del emitted[:]
    alg.validate(batches, 2)
    assert len(validated) == 3 and all(v[0] is b[0] and v[1] is b[1] for v, b in zip(validated, batches))
    assert not any(m.training for model in alg.models.values() for m in model.modules())
    ids = VALIDATION_IDS.get(name, ('task',))
    assert emitted == ['Validation metrics:\n' + ''.join('  %s-metrics\t=>\t\n' % i for i in ids)]


def test_s4l_warns_about_several_ground_truths_on_the_first_batch_of_every_epoch(build, monkeypatch):
    alg = build('ssl_s4l')

    class Stop(Exception):
        pass

    def prehandle(inp, gt, is_train):
        raise Stop
    warnings = []
    monkeypatch.setattr(alg, '_inp_warn', lambda: warnings.append(True))
    monkeypatch.setattr(alg, '_batch_prehandle', prehandle)
    two_gts = ((torch.zeros(2, 3, 4, 4),), (torch.zeros(2, 1, 4, 4), torch.zeros(2, 1, 4, 4)))
    for epoch in range(2):
        with pytest.raises(Stop):
            alg._train([two_gts, two_gts], epoch)
        assert len(warnings) == epoch + 1
        with pytest.raises(Stop):
            alg.train_step(*two_gts, 1, 0)              # a later batch of the same epoch
        assert len(warnings) == epoch + 1
    with pytest.raises(Stop):
        alg._train([((torch.zeros(2, 3, 4, 4),), (torch.zeros(2, 1, 4, 4),))], 2)
    assert len(warnings) == 2
