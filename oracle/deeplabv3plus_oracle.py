"""CPU oracle for the DeepLabV3+ task model (pixelssl_b200/task/sseg/module/deeplab_v3plus.py).  TEST INFRASTRUCTURE ONLY.

A functional torch-CPU restatement in the style of ``sseg_oracle``: the dilated ResNet and BatchNorm are
``sseg_oracle``'s, the head follows DeepLabV3+ (Chen et al., ECCV 2018) as torchvision lays out its ASPP
(``torchvision.models.segmentation.deeplabv3.ASPP``) but without the projection's dropout.  PixelSSL ships no
DeepLabV3+, so there is no reference run to pin this file to; ``tests/test_host_deeplabv3plus.py`` pins its ASPP to
torchvision's in eval mode instead."""
import contextlib
import math

import torch
import torch.nn.functional as F

from . import sseg_oracle as O

ASPP_RATES = {16: (6, 12, 18), 8: (12, 24, 36)}
_DEEPLABV2_PARAM_SHAPES = O.deeplabv2_param_shapes


def _head_shapes(num_classes):
    """(name, shape, kind) of the head in ``parameters()`` order: aspp, decoder, classifier."""
    out = [('aspp.convs.0.0.weight', (256, 2048, 1, 1), 'conv'),
           ('aspp.convs.0.1.weight', (256,), 'bn_w'), ('aspp.convs.0.1.bias', (256,), 'bn_b')]
    for i in (1, 2, 3):
        out += [('aspp.convs.%d.0.weight' % i, (256, 2048, 3, 3), 'conv'),
                ('aspp.convs.%d.1.weight' % i, (256,), 'bn_w'), ('aspp.convs.%d.1.bias' % i, (256,), 'bn_b')]
    out += [('aspp.convs.4.1.weight', (256, 2048, 1, 1), 'conv'),
            ('aspp.convs.4.2.weight', (256,), 'bn_w'), ('aspp.convs.4.2.bias', (256,), 'bn_b'),
            ('aspp.project.0.weight', (256, 1280, 1, 1), 'conv'),
            ('aspp.project.1.weight', (256,), 'bn_w'), ('aspp.project.1.bias', (256,), 'bn_b'),
            ('decoder.reduce.0.weight', (48, 256, 1, 1), 'conv'),
            ('decoder.reduce.1.weight', (48,), 'bn_w'), ('decoder.reduce.1.bias', (48,), 'bn_b'),
            ('decoder.fuse.0.weight', (256, 304, 3, 3), 'conv'),
            ('decoder.fuse.1.weight', (256,), 'bn_w'), ('decoder.fuse.1.bias', (256,), 'bn_b'),
            ('decoder.fuse.3.weight', (256, 256, 3, 3), 'conv'),
            ('decoder.fuse.4.weight', (256,), 'bn_w'), ('decoder.fuse.4.bias', (256,), 'bn_b'),
            ('classifier.weight', (num_classes, 256, 1, 1), 'cls_w'),
            ('classifier.bias', (num_classes,), 'cls_b')]
    return out


def param_shapes(num_classes=21, output_stride=16, blocks=O.R101_BLOCKS):
    """Ordered (name, shape, kind) list in ``parameters()`` order; names relative to the model (checkpoint key
    ``module.model.<name>``)."""
    backbone = [t for t in _DEEPLABV2_PARAM_SHAPES(num_classes, output_stride, blocks) if t[0].startswith('backbone.')]
    return backbone + _head_shapes(num_classes)


def buffer_shapes(output_stride=16, blocks=O.R101_BLOCKS):
    """(BN prefix, channels) per BatchNorm layer, in module order."""
    return O.deeplabv2_buffer_shapes(output_stride, blocks) + \
        [(n[:-len('.weight')], s[0]) for n, s, k in _head_shapes(21) if k == 'bn_w']


def init(seed, num_classes=21, output_stride=16, blocks=O.R101_BLOCKS, cls_bias_std=0.0):
    """Deterministic state with the model's initial distributions: every conv ~ N(0, sqrt(2/(k*k*Cout))), BN gamma=1
    beta=0, classifier weight ~ N(0, 0.01) and bias ~ N(0, cls_bias_std) (the model starts at 0).  One generator draws
    in parameter order; the dict is in ``state_dict`` order (each BN's buffers follow its bias)."""
    g = torch.Generator().manual_seed(seed)
    state = {}
    for name, shape, kind in param_shapes(num_classes, output_stride, blocks):
        if kind == 'conv':
            state[name] = torch.randn(shape, generator=g) * math.sqrt(2.0 / (shape[2] * shape[3] * shape[0]))
        elif kind == 'cls_w':
            state[name] = torch.randn(shape, generator=g) * 0.01
        elif kind == 'cls_b':
            state[name] = torch.randn(shape, generator=g) * cls_bias_std
        elif kind == 'bn_w':
            state[name] = torch.ones(shape)
        else:
            state[name] = torch.zeros(shape)
            bn = name[:-len('.bias')]
            state[bn + '.running_mean'] = torch.zeros(shape)
            state[bn + '.running_var'] = torch.ones(shape)
            state[bn + '.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)
    return state


def _cbr(x, state, conv, bn, training, padding=0, dilation=1):
    return F.relu(O.batch_norm(F.conv2d(x, state[conv + '.weight'], padding=padding, dilation=dilation), state, bn, training))


def aspp(x, state, training, rates=ASPP_RATES[16], prefix='aspp.'):
    """torchvision ASPP.forward without the projection's dropout: 1x1, three dilated 3x3 and image pooling branches,
    concatenated, 1x1 projection; every conv bias-free and followed by BN + ReLU."""
    h, w = x.shape[2:]
    res = [_cbr(x, state, prefix + 'convs.0.0', prefix + 'convs.0.1', training)]
    for i, r in enumerate(rates, 1):
        res.append(_cbr(x, state, prefix + 'convs.%d.0' % i, prefix + 'convs.%d.1' % i, training, padding=r, dilation=r))
    p = _cbr(F.adaptive_avg_pool2d(x, 1), state, prefix + 'convs.4.1', prefix + 'convs.4.2', training)
    res.append(F.interpolate(p, size=(h, w), mode='bilinear', align_corners=False))
    return _cbr(torch.cat(res, dim=1), state, prefix + 'project.0', prefix + 'project.1', training)


def backbone_forward(img, state, training, output_stride=16, blocks=O.R101_BLOCKS):
    """sseg_oracle.resnet_forward, also returning the layer1 output."""
    x = F.conv2d(img, state['backbone.conv1.weight'], stride=2, padding=3)
    x = F.relu(O.batch_norm(x, state, 'backbone.bn1', training))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    low = None
    for bp, inpl, pl, stride, dil, down in O.resnet_plan(output_stride, blocks):
        x = O.bottleneck(x, state, 'backbone.' + bp, stride, dil, down, training)
        if bp.startswith('layer1.'):
            low = x
    return low, x


def forward(img, state, training=True, output_stride=16, blocks=O.R101_BLOCKS):
    """-> (logits at the input size, layer4 latent)."""
    low, latent = backbone_forward(img, state, training, output_stride, blocks)
    a = aspp(latent, state, training, ASPP_RATES[output_stride])
    r = _cbr(low, state, 'decoder.reduce.0', 'decoder.reduce.1', training)
    x = torch.cat([F.interpolate(a, size=low.shape[2:], mode='bilinear', align_corners=True), r], dim=1)
    x = _cbr(x, state, 'decoder.fuse.0', 'decoder.fuse.1', training, padding=1)
    x = _cbr(x, state, 'decoder.fuse.3', 'decoder.fuse.4', training, padding=1)
    x = F.conv2d(x, state['classifier.weight'], state['classifier.bias'])
    return F.interpolate(x, size=img.shape[2:], mode='bilinear', align_corners=True), latent


def lr_multipliers(names):
    """backbone at 1x, ASPP / decoder / classifier at 10x."""
    return [1.0 if n.startswith('backbone.') else 10.0 for n in names]


@contextlib.contextmanager
def _as_task_model():
    """Point the names sseg_oracle.MTOracle looks up in its module (the forward, the parameter list and the LR
    multipliers) at this model's for the duration of the block."""
    saved = O.deeplabv2_forward, O.deeplabv2_param_shapes, O.lr_multipliers
    O.deeplabv2_forward, O.deeplabv2_param_shapes, O.lr_multipliers = forward, param_shapes, lr_multipliers
    try:
        yield
    finally:
        O.deeplabv2_forward, O.deeplabv2_param_shapes, O.lr_multipliers = saved


class MTOracle(O.MTOracle):
    """sseg_oracle.MTOracle (Mean Teacher; SupOnly with t_state=None) with DeepLabV3+ as the task model."""

    def __init__(self, *a, **k):
        with _as_task_model():
            super().__init__(*a, **k)

    def step(self, *a, **k):
        with _as_task_model():
            return super().step(*a, **k)
