"""CPU oracle for the deep-stem ResNet backbones (``resnet50-deepstem`` / ``resnet101-deepstem``).  TEST INFRASTRUCTURE
ONLY.

The deep-stem ResNet of CPS (Chen et al., CVPR 2021) and UniMatch (Yang et al., CVPR 2023), PSPNet's "deep base": the
7x7/2 stem is three 3x3 convolutions 3->64 (stride 2), 64->64, 64->128, each followed by BN and ReLU (the last BN is
``bn1``), layer1 starts from 128 channels, and the layers are dilated the torchvision way
(``replace_stride_with_dilation``).  PixelSSL has no such backbone, so there is no reference run to pin this file to;
``tests/test_host_deepstem.py`` pins its dilation plan and its layer1-4 forward to torchvision's ResNet.

The functions restate the backbone in the style of ``sseg_oracle``; ``deep_stem()`` points the names the DeepLab-v2,
DeepLabV3+ and PSPNet oracles (and their step oracles) look up at them for the duration of a ``with`` block, so every
existing oracle runs with the deep stem without changing."""
import contextlib

import torch.nn.functional as F

from . import deeplabv3plus_oracle as D
from . import sseg_oracle as O

_PLAIN_DEEPLABV2_PARAM_SHAPES = O.deeplabv2_param_shapes


def resnet_plan(output_stride=16, blocks=O.R101_BLOCKS):
    """(prefix, inplanes, planes, stride, dilation, has_downsample) per bottleneck, like ``sseg_oracle.resnet_plan``:
    torchvision's ``_make_layer`` with replace_stride_with_dilation [F, F, T] (OS16) or [F, T, T] (OS8) - a dilated
    layer has stride 1 and its first block keeps the previous dilation - and layer1 from 128 channels."""
    if output_stride == 16:
        dilate = (False, False, False, True)
    elif output_stride == 8:
        dilate = (False, False, True, True)
    else:
        raise NotImplementedError
    plan, inplanes, dilation = [], 128, 1
    for li, planes in enumerate((64, 128, 256, 512)):
        stride, prev = (1 if li == 0 else 2), dilation
        if dilate[li]:
            dilation *= stride
            stride = 1
        for bi in range(blocks[li]):
            s, d = (stride, prev) if bi == 0 else (1, dilation)
            down = bi == 0 and (s != 1 or inplanes != planes * 4)
            plan.append(('layer%d.%d' % (li + 1, bi), inplanes, planes, s, d, down))
            inplanes = planes * 4
    return plan


def stem_param_shapes():
    """(name, shape, kind) of the stem in ``parameters()`` order: conv1.{0,1,3,4,6}, then bn1."""
    return [('backbone.conv1.0.weight', (64, 3, 3, 3), 'conv'),
            ('backbone.conv1.1.weight', (64,), 'bn_w'), ('backbone.conv1.1.bias', (64,), 'bn_b'),
            ('backbone.conv1.3.weight', (64, 64, 3, 3), 'conv'),
            ('backbone.conv1.4.weight', (64,), 'bn_w'), ('backbone.conv1.4.bias', (64,), 'bn_b'),
            ('backbone.conv1.6.weight', (128, 64, 3, 3), 'conv'),
            ('backbone.bn1.weight', (128,), 'bn_w'), ('backbone.bn1.bias', (128,), 'bn_b')]


def backbone_param_shapes(output_stride=16, blocks=O.R101_BLOCKS):
    """(name, shape, kind) of the backbone in ``parameters()`` order: the stem, then the bottlenecks of this plan."""
    out = stem_param_shapes()
    for prefix, inpl, pl, stride, dil, down in resnet_plan(output_stride, blocks):
        p = 'backbone.' + prefix
        out += [(p + '.conv1.weight', (pl, inpl, 1, 1), 'conv'),
                (p + '.bn1.weight', (pl,), 'bn_w'), (p + '.bn1.bias', (pl,), 'bn_b'),
                (p + '.conv2.weight', (pl, pl, 3, 3), 'conv'),
                (p + '.bn2.weight', (pl,), 'bn_w'), (p + '.bn2.bias', (pl,), 'bn_b'),
                (p + '.conv3.weight', (pl * 4, pl, 1, 1), 'conv'),
                (p + '.bn3.weight', (pl * 4,), 'bn_w'), (p + '.bn3.bias', (pl * 4,), 'bn_b')]
        if down:
            out += [(p + '.downsample.0.weight', (pl * 4, inpl, 1, 1), 'conv'),
                    (p + '.downsample.1.weight', (pl * 4,), 'bn_w'),
                    (p + '.downsample.1.bias', (pl * 4,), 'bn_b')]
    return out


def deeplabv2_param_shapes(num_classes=21, output_stride=16, blocks=O.R101_BLOCKS):
    """``sseg_oracle.deeplabv2_param_shapes`` with the deep-stem backbone."""
    head = [t for t in _PLAIN_DEEPLABV2_PARAM_SHAPES(num_classes, output_stride, blocks) if not t[0].startswith('backbone.')]
    return backbone_param_shapes(output_stride, blocks) + head


def deeplabv2_buffer_shapes(output_stride=16, blocks=O.R101_BLOCKS):
    """(BN prefix, channels) per BatchNorm layer of the DeepLab-v2 model, in module order."""
    return [(n[:-len('.weight')], s[0]) for n, s, k in deeplabv2_param_shapes(21, output_stride, blocks) if k == 'bn_w']


def stem_forward(x, state, training, prefix='backbone.'):
    """conv 3x3/2 pad 1 -> BN -> ReLU -> conv 3x3 pad 1 -> BN -> ReLU -> conv 3x3 pad 1 -> bn1 -> ReLU -> max-pool
    3x3/2 pad 1; every convolution bias-free."""
    x = F.relu(O.batch_norm(F.conv2d(x, state[prefix + 'conv1.0.weight'], stride=2, padding=1), state, prefix + 'conv1.1',
                            training))
    x = F.relu(O.batch_norm(F.conv2d(x, state[prefix + 'conv1.3.weight'], padding=1), state, prefix + 'conv1.4', training))
    x = F.relu(O.batch_norm(F.conv2d(x, state[prefix + 'conv1.6.weight'], padding=1), state, prefix + 'bn1', training))
    return F.max_pool2d(x, kernel_size=3, stride=2, padding=1)


def layers_forward(x, state, training, output_stride=16, blocks=O.R101_BLOCKS, prefix='backbone.'):
    """layer1..4 on the stem output -> (layer1 output, layer4 output)."""
    low = None
    for bp, inpl, pl, stride, dil, down in resnet_plan(output_stride, blocks):
        x = O.bottleneck(x, state, prefix + bp, stride, dil, down, training)
        if bp.startswith('layer1.'):
            low = x
    return low, x


def resnet_forward(x, state, training, output_stride=16, blocks=O.R101_BLOCKS, prefix='backbone.'):
    return layers_forward(stem_forward(x, state, training, prefix), state, training, output_stride, blocks, prefix)[1]


def backbone_forward(img, state, training, output_stride=16, blocks=O.R101_BLOCKS):
    """``deeplabv3plus_oracle.backbone_forward``: -> (layer1 output, layer4 output)."""
    return layers_forward(stem_forward(img, state, training), state, training, output_stride, blocks)


@contextlib.contextmanager
def deep_stem():
    """Inside the block, ``sseg_oracle`` (DeepLab-v2, PSPNet, MTOracle, init_*) and ``deeplabv3plus_oracle`` (param_shapes,
    init, forward, MTOracle) describe and run the deep-stem backbone.  ``blocks`` keeps selecting R50 / R101."""
    saved = (O.resnet_plan, O.deeplabv2_param_shapes, O.deeplabv2_buffer_shapes, O.resnet_forward,
             D.backbone_forward, D._DEEPLABV2_PARAM_SHAPES)
    O.resnet_plan, O.deeplabv2_param_shapes, O.deeplabv2_buffer_shapes = resnet_plan, deeplabv2_param_shapes, deeplabv2_buffer_shapes
    O.resnet_forward, D.backbone_forward, D._DEEPLABV2_PARAM_SHAPES = resnet_forward, backbone_forward, deeplabv2_param_shapes
    try:
        yield
    finally:
        (O.resnet_plan, O.deeplabv2_param_shapes, O.deeplabv2_buffer_shapes, O.resnet_forward,
         D.backbone_forward, D._DEEPLABV2_PARAM_SHAPES) = saved
