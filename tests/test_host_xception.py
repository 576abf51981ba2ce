"""DeepLabV3+ on the aligned Xception-65 backbone (xception65), host side (-m "not gpu"): the module tree, unpadded
checkpoint shapes and LR groups against the CPU oracle (oracle/xception_oracle.py), initialisation and --freeze-bn,
the per-model backbone rule, the pretrained-checkpoint rule, and the oracle against an nn.Module restatement."""
import types

import pytest
import torch
import torch.nn as nn

from oracle import xception_oracle as X

_CFG = {'ssl_algorithm': 'ssl_null', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True, 'pretrained_backbone': 'none'}


def _task_model(model='deeplabv3plus', **over):
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import model as eng_model
    args = runner.build_args(dict(_CFG, models={'model': model}, **dict({'backbone': 'xception65'}, **over)),
                             iters_per_epoch=5)
    return getattr(eng_model, model)()(args), args


@pytest.mark.parametrize('output_stride', [8, 16])
def test_state_dict_and_param_groups_match_the_oracle(output_stride):
    eng, args = _task_model(output_stride=output_stride)
    params = [(n, tuple(s)) for n, s, _ in X.param_shapes(21, output_stride)]
    assert [(n, tuple(p.shape)) for n, p in eng.model.named_parameters()] == params
    state = {k: tuple(v.shape) for k, v in X.init(0, 21, output_stride).items()}
    got = {k: tuple(v.shape) for k, v in eng.model.state_dict().items()}
    assert got == state and list(got) == list(state)
    for k, s in (('backbone.block1.rep.0.conv1.weight', (64, 1, 3, 3)), ('backbone.block1.rep.0.bn.running_var', (64,)),
                 ('backbone.block1.rep.0.pointwise.weight', (128, 64, 1, 1)), ('backbone.block1.rep.1.weight', (128,)),
                 ('backbone.block4.rep.1.conv1.weight', (728, 1, 3, 3)), ('backbone.block1.skipbn.bias', (128,)),
                 ('backbone.conv3.pointwise.weight', (1536, 1024, 1, 1)), ('decoder.reduce.0.weight', (48, 128, 1, 1))):
        assert got[k] == s, k
    assert 'backbone.block4.skip.weight' not in got and 'backbone.block20.skip.weight' in got
    names = {id(p): n for n, p in eng.model.named_parameters()}
    groups = [[names[id(p)] for p in g['params']] for g in eng.param_groups]
    assert groups[0] == [n for n, _ in params if n.startswith('backbone.')]
    assert all(not n.startswith('backbone.') for g in groups[1:] for n in g)
    assert eng.param_groups[0]['lr'] == args.lr
    assert eng.fp_channels == (128, 2048)


def test_resnet_models_keep_their_fp_channels():
    eng, _ = _task_model(backbone='resnet50')
    assert eng.fp_channels == (256, 2048)


@pytest.mark.parametrize('output_stride', [8, 16])
def test_dilation_plan(output_stride):
    from pixelssl_b200.task.sseg.module.xception import SeparableConv2d
    eng, _ = _task_model(output_stride=output_stride)
    bb = eng.model.backbone
    plan, exit_dil = X.block_plan(output_stride)
    for name, cin, cout, reps, stride, dil, swr, gf, last in plan:
        ref = X.block_rep(cin, cout, reps, stride, dil, swr, gf, last)
        rep = getattr(bb, name).rep
        assert len(rep) == len(ref)
        for m, e in zip(rep, ref):
            if e[0] == 'relu':
                assert isinstance(m, nn.ReLU) and m.inplace
            elif e[0] == 'sep':
                assert isinstance(m, SeparableConv2d)
                assert (m.conv1.in_channels, m.pointwise.out_channels, m.conv1.stride, m.conv1.dilation) == e[1:]
    assert [bb.conv3.conv1.dilation, bb.conv4.conv1.dilation, bb.conv5.conv1.dilation] == [exit_dil] * 3
    assert bb.block3.rep[-2].conv1.stride == (2 if output_stride == 16 else 1)
    assert bb.block3.rep[-2].conv1.dilation == 1


def test_init_and_freeze_bn_cover_every_layer():
    from pixelssl_b200.nn.modules import BatchNorm2d, Conv2d, DepthwiseConv2d
    eng, _ = _task_model(freeze_bn=True)
    bb = eng.model.backbone
    for conv in (bb.conv1, bb.conv2, bb.block4.rep[1].pointwise, bb.block20.skip, bb.conv5.pointwise):
        assert isinstance(conv, Conv2d) and conv.bias is None
        k, cout = conv.kernel_size[0], conv.out_channels
        assert abs(float(conv.weight.detach().std()) / (2.0 / (k * k * cout)) ** 0.5 - 1) < 0.15
    for dw in (bb.block1.rep[0].conv1, bb.block4.rep[1].conv1, bb.conv5.conv1):
        assert isinstance(dw, DepthwiseConv2d)
        assert abs(float(dw.weight.detach().std()) / (2.0 / (9 * dw.in_channels)) ** 0.5 - 1) < 0.15
    bns = [m for m in eng.model.modules() if isinstance(m, BatchNorm2d)]
    assert len(bns) == len([n for n, _, k in X.param_shapes() if k == 'bn_w'])
    for bn in bns:
        assert not bn.training
    for bn in [m for m in bb.modules() if isinstance(m, BatchNorm2d)]:
        assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))


# ---- backbone rule and pretrained weights --------------------------------------------------------------------------------

class _Refused(Exception):
    pass


@pytest.fixture
def refuse(monkeypatch):
    """logger.log_err prints and exits; here it raises with its message."""
    from pixelssl_b200.utils import logger

    def log_err(message):
        raise _Refused(message)
    monkeypatch.setattr(logger, 'log_err', log_err)


@pytest.mark.parametrize('model,name', [('deeplabv2', 'DeepLabV2'), ('pspnet', 'PSPNet')])
def test_other_models_refuse_xception(refuse, model, name):
    with pytest.raises(_Refused, match='%s.*xception65' % name):
        _task_model(model)


def test_auto_is_refused(refuse):
    from pixelssl_b200.task.sseg import model as eng_model
    with pytest.raises(_Refused, match='none'):
        eng_model.pretrained_backbone_url(types.SimpleNamespace(backbone='xception65', pretrained_backbone='auto'))
    assert eng_model.pretrained_backbone_url(types.SimpleNamespace(backbone='xception65', pretrained_backbone='none')) is None


def _xception_file(tmp_path, edit=None):
    """A checkpoint in the tree's own key layout with an fc head, under a module. prefix."""
    from pixelssl_b200.task.sseg.module.xception import AlignedXception
    src = AlignedXception(16)
    g = torch.Generator().manual_seed(7)
    sd = {}
    for k, v in src.state_dict().items():
        v = v.contiguous().clone()
        if v.is_floating_point():
            v = torch.randn(v.shape, generator=g) if not k.endswith('running_var') else torch.rand(v.shape, generator=g) + 0.5
        sd[k] = v
    sd['fc.weight'], sd['fc.bias'] = torch.randn(1000, 2048, generator=g), torch.randn(1000, generator=g)
    if edit is not None:
        edit(sd)
    path = tmp_path / 'xception65.pth'
    torch.save({'module.' + k: v for k, v in sd.items()}, str(path))
    return str(path), sd


def test_checkpoint_loads_bit_equal(tmp_path):
    path, sd = _xception_file(tmp_path)
    eng, _ = _task_model(pretrained_backbone=path)
    got = eng.model.backbone.state_dict()
    assert set(got) == set(sd) - {'fc.weight', 'fc.bias'}
    for k, v in got.items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize('case,key', [('missing', 'block7.rep.4.bn.running_var'), ('misshapen', 'block4.rep.1.conv1.weight'),
                                      ('missing', 'conv5.pointwise.weight'), ('misshapen', 'block12.rep.5.weight')])
def test_incomplete_checkpoint_is_refused(tmp_path, refuse, case, key):
    from pixelssl_b200.task.sseg.module.xception import AlignedXception

    def edit(sd):
        if case == 'missing':
            del sd[key]
        else:
            sd[key] = torch.cat([sd[key], sd[key][:40]])         # 728 -> 768: a padded shape is not accepted either
    path, _ = _xception_file(tmp_path, edit)
    with pytest.raises(_Refused, match=key.replace('.', r'\.')):
        AlignedXception(16, path)


# ---- the oracle against an nn.Module restatement --------------------------------------------------------------------------

class _Sep(nn.Module):
    def __init__(self, cin, cout, stride, dilation):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cin, 3, stride, 0, dilation, groups=cin, bias=False)
        self.bn = nn.BatchNorm2d(cin)
        self.pointwise = nn.Conv2d(cin, cout, 1, bias=False)

    def forward(self, x):
        d = self.conv1.dilation[0]
        return self.pointwise(self.bn(self.conv1(nn.functional.pad(x, (d, d, d, d)))))


class _Block(nn.Module):
    def __init__(self, cin, cout, reps, stride, dilation, start_with_relu, grow_first, is_last):
        super().__init__()
        if cout != cin or stride != 1:
            self.skip = nn.Conv2d(cin, cout, 1, stride=stride, bias=False)
            self.skipbn = nn.BatchNorm2d(cout)
        else:
            self.skip = None
        relu = nn.ReLU(inplace=True)
        rep, f = [], cin
        if grow_first:
            rep += [relu, _Sep(cin, cout, 1, dilation), nn.BatchNorm2d(cout)]
            f = cout
        for _ in range(reps - 1):
            rep += [relu, _Sep(f, f, 1, dilation), nn.BatchNorm2d(f)]
        if not grow_first:
            rep += [relu, _Sep(cin, cout, 1, dilation), nn.BatchNorm2d(cout)]
        if stride != 1:
            rep += [relu, _Sep(cout, cout, 2, 1), nn.BatchNorm2d(cout)]
        if stride == 1 and is_last:
            rep += [relu, _Sep(cout, cout, 1, 1), nn.BatchNorm2d(cout)]
        if not start_with_relu:
            rep = rep[1:]
        self.rep = nn.Sequential(*rep)

    def forward(self, inp):
        x = self.rep(inp)            # an in-place leading ReLU rectifies inp, which the skip then reads
        skip = self.skipbn(self.skip(inp)) if self.skip is not None else inp
        return x + skip


class _Xception(nn.Module):
    def __init__(self, output_stride):
        super().__init__()
        s3, md, ed = {16: (2, 1, (1, 2)), 8: (1, 2, (2, 4))}[output_stride]
        self.conv1 = nn.Conv2d(3, 32, 3, 2, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(32)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(32, 64, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(64)
        self.block1 = _Block(64, 128, 2, 2, 1, False, True, False)
        self.block2 = _Block(128, 256, 2, 2, 1, False, True, False)
        self.block3 = _Block(256, 728, 2, s3, 1, True, True, True)
        for i in range(4, 20):
            setattr(self, 'block%d' % i, _Block(728, 728, 3, 1, md, True, True, False))
        self.block20 = _Block(728, 1024, 2, 1, ed[0], True, False, True)
        self.conv3, self.bn3 = _Sep(1024, 1536, 1, ed[1]), nn.BatchNorm2d(1536)
        self.conv4, self.bn4 = _Sep(1536, 1536, 1, ed[1]), nn.BatchNorm2d(1536)
        self.conv5, self.bn5 = _Sep(1536, 2048, 1, ed[1]), nn.BatchNorm2d(2048)

    def forward(self, x):
        x = self.relu(self.bn2(self.conv2(self.relu(self.bn1(self.conv1(x))))))
        x = self.relu(self.block1(x))
        low = x
        for i in range(2, 21):
            x = getattr(self, 'block%d' % i)(x)
        x = self.relu(x)
        for i in (3, 4, 5):
            x = self.relu(getattr(self, 'bn%d' % i)(getattr(self, 'conv%d' % i)(x)))
        return low, x


@pytest.mark.parametrize('training', [True, False])
@pytest.mark.parametrize('output_stride', [8, 16])
def test_oracle_equals_module_restatement(output_stride, training):
    ref = _Xception(output_stride).double()
    g = torch.Generator().manual_seed(11 + output_stride)
    st = {}
    for k, v in ref.state_dict().items():
        if k.endswith('num_batches_tracked'):
            st['backbone.' + k] = v.clone()
        elif k.endswith('running_var'):
            st['backbone.' + k] = 0.5 + torch.rand(v.shape, generator=g, dtype=torch.float64)
        elif v.dim() == 1:
            st['backbone.' + k] = 0.3 * torch.randn(v.shape, generator=g, dtype=torch.float64) + (1.0 if k.endswith('weight') else 0.0)
        else:
            st['backbone.' + k] = torch.randn(v.shape, generator=g, dtype=torch.float64) * (2.0 / v[0].numel()) ** 0.5
    assert set(st) == {k for k in X.init(0, 21, output_stride) if k.startswith('backbone.')}
    ref.load_state_dict({k[len('backbone.'):]: v.clone() for k, v in st.items()})
    ref.train(training)
    x = torch.randn(2, 3, 49, 41, generator=g, dtype=torch.float64)
    with torch.no_grad():
        low_r, out_r = ref(x)
        low, out = X.backbone_forward(x, st, training, output_stride)
    assert low.shape == low_r.shape == (2, 128, 13, 11)
    assert out.shape == out_r.shape and out.shape[1] == 2048
    assert float((low - low_r).abs().max() / low_r.abs().max()) < 1e-12
    assert float((out - out_r).abs().max() / out_r.abs().max()) < 1e-12
    if training:
        for k, v in ref.state_dict().items():
            if k.endswith('running_mean') or k.endswith('running_var'):
                assert float((st['backbone.' + k] - v).abs().max()) < 1e-12, k


def test_new_entry_points_are_declared():
    import os
    import re
    from pixelssl_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, 'include', 'pixelssl_b200.h')).read()
    for name in ('pxl_dw_conv_fwd', 'pxl_dw_conv_dgrad', 'pxl_dw_conv_wgrad'):
        assert re.search(r'\b%s\s*\(' % name, header) and name in _lib.SIGNATURES
