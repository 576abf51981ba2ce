"""DeepLabV3+ task model, host side (-m "not gpu"): module tree and LR groups against the CPU oracle, the ASPP layout and
arithmetic against torchvision's, plugin registration and the CCT shape hooks."""
import types

import pytest
import torch

from oracle import deeplabv3plus_oracle as D

_CFG = {'ssl_algorithm': 'ssl_null', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005, 'epochs': 2,
        'batch_size': 2, 'unlabeled_batch_size': 0, 'ignore_unlabeled': True, 'models': {'model': 'deeplabv3plus'}}


def _task_model(**over):
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import model as eng_model
    args = runner.build_args(dict(_CFG, **over), iters_per_epoch=5)
    return eng_model.deeplabv3plus()(args), args


@pytest.mark.parametrize('backbone,output_stride', [('resnet101', 16), ('resnet50', 8)])
def test_state_dict_and_param_groups_match_the_oracle(backbone, output_stride):
    eng, args = _task_model(backbone=backbone, output_stride=output_stride)
    blocks = D.O.R101_BLOCKS if backbone == 'resnet101' else D.O.R50_BLOCKS
    ref = D.init(0, output_stride=output_stride, blocks=blocks)
    assert [(k, tuple(v.shape), v.dtype) for k, v in eng.model.state_dict().items()] == \
        [(k, tuple(v.shape), v.dtype) for k, v in ref.items()]
    names = {id(p): n for n, p in eng.model.named_parameters()}
    assert [n for n, _, _ in D.param_shapes(21, output_stride, blocks)] == list(names.values())
    assert [g['lr'] for g in eng.param_groups] == [args.lr, args.lr * 10]
    groups = [[names[id(p)] for p in g['params']] for g in eng.param_groups]
    assert groups[0] == [n for n in names.values() if n.startswith('backbone.')]
    assert groups[1] == [n for n in names.values() if not n.startswith('backbone.')]
    assert eng.model.aspp.convs[1][0].dilation == D.ASPP_RATES[output_stride][0]
    # checkpoints load into the module tree with the usual prefix
    wrapped = torch.nn.Module()
    wrapped.module = eng
    wrapped.load_state_dict({'module.model.' + k: v for k, v in ref.items()}, strict=True)


def test_init_distributions():
    eng, _ = _task_model()
    m = eng.model
    for conv in (m.aspp.convs[1][0], m.aspp.project[0], m.decoder.fuse[0]):
        k, cout = conv.kernel_size[0], conv.out_channels
        assert abs(float(conv.weight.detach().std()) / (2.0 / (k * k * cout)) ** 0.5 - 1) < 0.05
    assert abs(float(m.classifier.weight.detach().std()) / 0.01 - 1) < 0.1 and float(m.classifier.bias.detach().abs().max()) == 0.0
    bn = m.decoder.fuse[4]
    assert torch.equal(bn.weight, torch.ones(256)) and torch.equal(bn.bias, torch.zeros(256))


def test_aspp_loads_torchvision_state_dict():
    from torchvision.models.segmentation.deeplabv3 import ASPP
    tv = ASPP(2048, [6, 12, 18], 256)
    eng, _ = _task_model()
    eng.model.aspp.load_state_dict(tv.state_dict(), strict=True)
    assert torch.equal(eng.model.aspp.project[0].weight, tv.project[0].weight)


def test_oracle_aspp_equals_torchvision_in_eval_mode():
    from torchvision.models.segmentation.deeplabv3 import ASPP
    torch.manual_seed(0)
    tv = ASPP(64, [2, 3, 5], 32).eval()
    with torch.no_grad():
        for m in tv.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
                m.running_mean.uniform_(-0.1, 0.1)
                m.running_var.uniform_(0.5, 2.0)
    state = {'aspp.' + k: v.clone() for k, v in tv.state_dict().items()}
    x = torch.randn(2, 64, 11, 9)
    with torch.no_grad():
        want = tv(x)
        got = D.aspp(x, state, False, rates=(2, 3, 5))
    assert float((got - want).abs().max() / want.abs().max()) <= 1e-6


def test_register_into_pixelssl_adds_deeplabv3plus():
    import pixelssl_b200
    from pixelssl_b200.task.sseg import model as eng_model
    pkg = types.ModuleType('pixelssl')
    pkg.ssl_algorithm = types.ModuleType('pixelssl.ssl_algorithm')
    pkg.nn = types.ModuleType('pixelssl.nn')
    pkg.nn.data = types.ModuleType('pixelssl.nn.data')
    task_model, task_criterion = types.ModuleType('model'), types.ModuleType('criterion')
    pixelssl_b200.register_into_pixelssl(pkg, (task_model, task_criterion))
    assert task_model.deeplabv3plus is eng_model.deeplabv3plus
    assert task_model.deeplabv2 is eng_model.deeplabv2 and task_model.pspnet is eng_model.pspnet
    assert eng_model.deeplabv3plus() is eng_model.DeepLabV3Plus


def test_cct_hooks_for_deeplabv3plus():
    from pixelssl_b200 import runner
    from pixelssl_b200.task.sseg import func as eng_func
    args = runner.build_args({'ssl_algorithm': 'ssl_cct', 'lr': 0.00025, 'momentum': 0.9, 'weight_decay': 0.0005,
                              'epochs': 20, 'batch_size': 16, 'unlabeled_batch_size': 8, 'cons_scale': 30.0,
                              'cons_rampup_epochs': 5, 'ad_lr_scale': 10.0, 'models': {'model': 'deeplabv3plus'}},
                             iters_per_epoch=5)
    f = eng_func.task_func()(args)
    assert f.sslcct_ad_in_channels() == 2048 and f.sslcct_ad_upsample_scale() == 8
