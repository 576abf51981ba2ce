"""Deep-stem ResNet backbones (resnet50-deepstem / resnet101-deepstem), host side (-m "not gpu"): the module tree and LR
groups of every task model against the CPU oracle (oracle/deepstem_oracle.py), the dilation plan and the layer1-4
arithmetic against torchvision's ResNet, and the pretrained-checkpoint rule."""
import pytest
import torch

from oracle import deeplabv3plus_oracle as D
from oracle import deepstem_oracle as S
from oracle import sseg_oracle as O

_CFG = {'ssl_algorithm': 'ssl_null', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True}
_BLOCKS = {'resnet50-deepstem': O.R50_BLOCKS, 'resnet101-deepstem': O.R101_BLOCKS}


def _task_model(model, **over):
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import model as eng_model
    args = runner.build_args(dict(_CFG, models={'model': model}, **over), iters_per_epoch=5)
    return getattr(eng_model, model)()(args), args


def _oracle_params(model, output_stride, blocks):
    """-> (parameter (name, shape) list in order, {state key: shape}) of the oracle with the deep stem."""
    with S.deep_stem():
        if model == 'deeplabv2':
            shapes, st = O.deeplabv2_param_shapes(21, output_stride, blocks), O.init_deeplabv2(0, 21, output_stride, blocks)
        elif model == 'deeplabv3plus':
            shapes, st = D.param_shapes(21, output_stride, blocks), D.init(0, 21, output_stride, blocks)
        else:
            shapes, st = O.pspnet_param_shapes(21, output_stride, blocks), O.init_pspnet(0, 21, output_stride, blocks)
    return [(n, tuple(s)) for n, s, _ in shapes], {k: tuple(v.shape) for k, v in st.items()}


@pytest.mark.parametrize('output_stride', [8, 16])
@pytest.mark.parametrize('backbone', ['resnet50-deepstem', 'resnet101-deepstem'])
@pytest.mark.parametrize('model', ['deeplabv2', 'deeplabv3plus', 'pspnet'])
def test_state_dict_and_param_groups_match_the_oracle(model, backbone, output_stride):
    eng, args = _task_model(model, backbone=backbone, output_stride=output_stride)
    params, state = _oracle_params(model, output_stride, _BLOCKS[backbone])
    assert [(n, tuple(p.shape)) for n, p in eng.model.named_parameters()] == params
    assert {k: tuple(v.shape) for k, v in eng.model.state_dict().items()} == state
    keys = [k for k in eng.model.state_dict() if k.startswith('backbone.')]
    assert keys[:14] == ['backbone.conv1.%d.%s' % (i, s) for i, ss in ((0, ('weight',)),
                         (1, ('weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked')), (3, ('weight',)),
                         (4, ('weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked')), (6, ('weight',)))
                         for s in ss] + ['backbone.bn1.weight']
    names = {id(p): n for n, p in eng.model.named_parameters()}
    groups = [[names[id(p)] for p in g['params']] for g in eng.param_groups]
    assert groups[0] == [n for n, _ in params if n.startswith('backbone.')]
    assert all(not n.startswith('backbone.') for g in groups[1:] for n in g)
    assert [g['lr'] for g in eng.param_groups][0] == args.lr
    bb = eng.model.backbone
    assert bb.layer1[0].conv1.in_channels == 128 and bb.layer1[0].downsample[0].in_channels == 128


def test_init_and_freeze_bn_cover_the_stem():
    eng, _ = _task_model('deeplabv2', backbone='resnet101-deepstem', freeze_bn=True)
    stem = eng.model.backbone.conv1
    for conv in (stem[0], stem[3], stem[6]):
        k, cout = conv.kernel_size[0], conv.out_channels
        assert conv.bias is None
        assert abs(float(conv.weight.detach().std()) / (2.0 / (k * k * cout)) ** 0.5 - 1) < 0.15
    for bn in (stem[1], stem[4], eng.model.backbone.bn1):
        assert not bn.training
        assert torch.equal(bn.weight, torch.ones_like(bn.weight)) and torch.equal(bn.bias, torch.zeros_like(bn.bias))


def _torchvision_deep_layers(depth, output_stride):
    """torchvision's ResNet layer1..4 built by its own _make_layer with the deep stem's 128 input channels."""
    import torchvision
    rswd = [False, False, True] if output_stride == 16 else [False, True, True]
    tv = getattr(torchvision.models, 'resnet%d' % depth)(weights=None, replace_stride_with_dilation=rswd)
    block = torchvision.models.resnet.Bottleneck
    tv.inplanes, tv.dilation = 128, 1
    n = {50: O.R50_BLOCKS, 101: O.R101_BLOCKS}[depth]
    tv.layer1 = tv._make_layer(block, 64, n[0])
    tv.layer2 = tv._make_layer(block, 128, n[1], stride=2, dilate=rswd[0])
    tv.layer3 = tv._make_layer(block, 256, n[2], stride=2, dilate=rswd[1])
    tv.layer4 = tv._make_layer(block, 512, n[3], stride=2, dilate=rswd[2])
    return tv, rswd


@pytest.mark.parametrize('output_stride', [8, 16])
@pytest.mark.parametrize('depth', [50, 101])
def test_dilation_plan_matches_torchvision(depth, output_stride):
    import torchvision
    from pixelssl_b200.task.sseg.module.resnet import build_backbone
    rswd = [False, False, True] if output_stride == 16 else [False, True, True]
    tv = getattr(torchvision.models, 'resnet%d' % depth)(weights=None, replace_stride_with_dilation=rswd)
    eng = build_backbone('resnet%d-deepstem' % depth, output_stride)
    plan = S.resnet_plan(output_stride, {50: O.R50_BLOCKS, 101: O.R101_BLOCKS}[depth])
    i = 0
    for li in range(1, 5):
        for tb, eb in zip(getattr(tv, 'layer%d' % li), getattr(eng, 'layer%d' % li)):
            assert (eb.conv2.stride, eb.conv2.dilation, eb.conv2.padding) == \
                (tb.conv2.stride[0], tb.conv2.dilation[0], tb.conv2.padding[0])
            assert (tb.downsample is None) == (eb.downsample is None)
            if tb.downsample is not None:
                assert eb.downsample[0].stride == tb.downsample[0].stride[0]
            _, _, _, stride, dil, down = plan[i]
            assert (stride, dil, down) == (eb.conv2.stride, eb.conv2.dilation, eb.downsample is not None)
            i += 1
    assert i == len(plan)


@pytest.mark.parametrize('output_stride', [8, 16])
def test_oracle_layers_equal_torchvision_in_eval_mode(output_stride):
    tv, _ = _torchvision_deep_layers(50, output_stride)
    tv = tv.double().eval()
    g = torch.Generator().manual_seed(5)
    st = {}
    for k, v in tv.state_dict().items():
        if not k.startswith('layer'):
            continue
        if k.endswith('num_batches_tracked'):
            st['backbone.' + k] = v.clone()
        elif k.endswith('running_var'):
            st['backbone.' + k] = 0.5 + torch.rand(v.shape, generator=g, dtype=torch.float64)
        elif v.dim() == 1:
            st['backbone.' + k] = 0.5 * torch.randn(v.shape, generator=g, dtype=torch.float64) + (1.0 if k.endswith('weight') else 0.0)
        else:
            st['backbone.' + k] = torch.randn(v.shape, generator=g, dtype=torch.float64) * (2.0 / v[0].numel()) ** 0.5
    tv.load_state_dict({k[len('backbone.'):]: v for k, v in st.items()}, strict=False)
    x = torch.randn(1, 128, 33, 33, generator=g, dtype=torch.float64)
    with torch.no_grad():
        ref = tv.layer4(tv.layer3(tv.layer2(tv.layer1(x))))
        low, got = S.layers_forward(x, st, False, output_stride, O.R50_BLOCKS)
    assert got.shape == ref.shape and low.shape[1] == 256
    assert float((got - ref).abs().max() / ref.abs().max()) < 1e-12


# ---- pretrained weights ----------------------------------------------------------------------------------------------

class _Refused(Exception):
    pass


@pytest.fixture
def refuse(monkeypatch):
    """logger.log_err prints and exits; here it raises with its message."""
    from pixelssl_b200.utils import logger

    def log_err(message):
        raise _Refused(message)
    monkeypatch.setattr(logger, 'log_err', log_err)


def _cps_layout_file(tmp_path, backbone='resnet50-deepstem', seed=3, edit=None):
    """A checkpoint in the CPS / UniMatch layout: the backbone's own keys plus an fc head, under a module. prefix."""
    from pixelssl_b200.task.sseg.module.resnet import build_backbone
    torch.manual_seed(seed)
    src = build_backbone(backbone, 16)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in src.state_dict().items():
        v = v.contiguous().clone()
        if v.is_floating_point():
            v = torch.randn(v.shape, generator=g) if not k.endswith('running_var') else torch.rand(v.shape, generator=g) + 0.5
        sd[k] = v
    sd['fc.weight'], sd['fc.bias'] = torch.randn(1000, 2048, generator=g), torch.randn(1000, generator=g)
    if edit is not None:
        edit(sd)
    path = tmp_path / 'resnet_deepstem.pth'
    torch.save({'module.' + k: v for k, v in sd.items()}, str(path))
    return str(path), sd


def test_cps_layout_checkpoint_loads_bit_equal(tmp_path):
    from pixelssl_b200.task.sseg.module.resnet import build_backbone
    path, sd = _cps_layout_file(tmp_path)
    eng = build_backbone('resnet50-deepstem', 16, path)
    got = eng.state_dict()
    assert set(got) == set(sd) - {'fc.weight', 'fc.bias'}
    for k, v in got.items():
        assert torch.equal(v, sd[k]), k


def test_task_model_loads_the_file(tmp_path):
    path, sd = _cps_layout_file(tmp_path, 'resnet50-deepstem')
    eng, _ = _task_model('deeplabv3plus', backbone='resnet50-deepstem', pretrained_backbone=path)
    assert torch.equal(eng.model.backbone.conv1[0].weight, sd['conv1.0.weight'])
    assert torch.equal(eng.model.backbone.layer4[2].bn3.running_var, sd['layer4.2.bn3.running_var'])


@pytest.mark.parametrize('case,key', [('missing', 'conv1.4.running_var'), ('misshapen', 'conv1.6.weight'),
                                      ('missing', 'layer3.5.conv2.weight')])
def test_incomplete_checkpoint_is_refused(tmp_path, refuse, case, key):
    from pixelssl_b200.task.sseg.module.resnet import build_backbone

    def edit(sd):
        if case == 'missing':
            del sd[key]
        else:
            sd[key] = sd[key][:, :32]
    path, _ = _cps_layout_file(tmp_path, edit=edit)
    with pytest.raises(_Refused, match=key.replace('.', r'\.')):
        build_backbone('resnet50-deepstem', 16, path)


def test_torchvision_7x7_checkpoint_is_refused(tmp_path, refuse):
    import torchvision
    from pixelssl_b200.task.sseg.module.resnet import build_backbone
    path = tmp_path / 'resnet50_torchvision.pth'
    torch.save(torchvision.models.resnet50(weights=None).state_dict(), str(path))
    with pytest.raises(_Refused, match=r'conv1\.0\.weight'):
        build_backbone('resnet50-deepstem', 16, str(path))


@pytest.mark.parametrize('backbone', ['resnet50-deepstem', 'resnet101-deepstem'])
def test_auto_is_refused(refuse, backbone):
    import types
    from pixelssl_b200.task.sseg import model as eng_model
    with pytest.raises(_Refused, match='none'):
        eng_model.pretrained_backbone_url(types.SimpleNamespace(backbone=backbone, pretrained_backbone='auto'))
    assert eng_model.pretrained_backbone_url(types.SimpleNamespace(backbone=backbone, pretrained_backbone='none')) is None
    assert eng_model.pretrained_backbone_url(types.SimpleNamespace(backbone='resnet101', pretrained_backbone='auto')) == \
        eng_model.PRETRAINED_BACKBONE_URLS['resnet101']


def test_new_entry_points_are_declared():
    import os
    import re
    from pixelssl_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, 'include', 'pixelssl_b200.h')).read()
    for name in ('pxl_stem3x3s2_im2col', 'pxl_stem3x3s2_im2col_h16'):
        assert re.search(r'\b%s\s*\(' % name, header) and name in _lib.SIGNATURES
