"""Dilated ResNet backbone on the H100 kernels: parameter tree and forward order of
task/sseg/module/backbone/resnet.py:13-131 (Bottleneck, strides/dilations per output stride,
multi-grid layer4), with BN+ReLU(+residual) fused and NHWC activations throughout; plus the deep-stem variant
CPS and UniMatch train (``*-deepstem``)."""
import math
import os

import torch
import torch.nn as nn

from .... import ops
from ....nn.modules import Conv2d, BatchNorm2d
from ....utils import logger


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None):
        super().__init__()
        self.conv1 = Conv2d(inplanes, planes, 1, bias=False)
        self.bn1 = BatchNorm2d(planes)
        self.conv2 = Conv2d(planes, planes, 3, stride=stride, dilation=dilation, padding=dilation, bias=False)
        self.bn2 = BatchNorm2d(planes)
        self.conv3 = Conv2d(planes, planes * 4, 1, bias=False)
        self.bn3 = BatchNorm2d(planes * 4)
        self.downsample = downsample
        self.stride, self.dilation = stride, dilation
        for conv in (self.conv1, self.conv2, self.conv3) + ((downsample[0],) if downsample is not None else ()):
            conv.feeds_bn = True          # the tensor-core epilogue then produces the BN statistics

    def forward(self, x):
        if all(ops.conv_bn_unit_ok(c, b) for c, b in ((self.conv1, self.bn1), (self.conv2, self.bn2), (self.conv3, self.bn3))) \
                and (self.downsample is None or ops.conv_bn_unit_ok(self.downsample[0], self.downsample[1])):
            # fp16-pair tensor-core path: four fused conv+BN(+ReLU/residual) nodes; the inner activations only exist
            # as the fp16 pairs the next convolution reads
            # identity blocks: the residual gradient is added into the block-input gradient by conv1's dgrad epilogue
            # blocks with a downsample branch: the downsample unit's dX is the buffer conv1's dgrad adds into
            key = object() if (torch.is_grad_enabled() and x.requires_grad) else None
            ident = self.downsample is None
            out = ops.conv_bn_act(x, self.conv1, self.bn1, relu=True, out_mode='pair', stash_key=key,
                                  stash_role='take' if key is not None else None)
            out = ops.conv_bn_act(out, self.conv2, self.bn2, relu=True, out_mode='pair')
            residual = x if ident else \
                ops.conv_bn_act(x, self.downsample[0], self.downsample[1], relu=False, out_mode='fp32', stash_key=key,
                                stash_role='give_dx' if key is not None else None)
            return ops.conv_bn_act(out, self.conv3, self.bn3, relu=True, residual=residual, out_mode='both',
                                   stash_key=key if ident else None,
                                   stash_role='give' if (key is not None and ident) else None)
        out = self.bn1(self.conv1(x), relu=True)
        out = self.bn2(self.conv2(out), relu=True)
        out = self.conv3(out)
        residual = x if self.downsample is None else self.downsample[1](self.downsample[0](x))
        return self.bn3(out, relu=True, residual=residual)      # relu(bn3(out) + residual)


class ResNet(nn.Module):
    """deep_stem=False: the reference's network (7x7/2 stem, multi-grid layer4).  deep_stem=True: the deep-stem ResNet
    of CPS / UniMatch (and PSPNet's "deep base"): three 3x3 convolutions 3->64 (stride 2), 64->64, 64->128 with BN and
    ReLU (the last one's BN is bn1), layer1 from 128 channels, and the layers dilated the torchvision way
    (replace_stride_with_dilation: a dilated layer's first block keeps the previous dilation)."""

    def __init__(self, layers, output_stride, pretrained_url=None, deep_stem=False):
        super().__init__()
        if output_stride not in (8, 16):
            raise NotImplementedError
        self.deep_stem = deep_stem
        if deep_stem:
            self.conv1 = nn.Sequential(Conv2d(3, 64, 3, stride=2, padding=1, bias=False), BatchNorm2d(64), nn.ReLU(inplace=True),
                                       Conv2d(64, 64, 3, padding=1, bias=False), BatchNorm2d(64), nn.ReLU(inplace=True),
                                       Conv2d(64, 128, 3, padding=1, bias=False))
            for i in (3, 6):
                self.conv1[i].feeds_bn = True
            self.bn1 = BatchNorm2d(128)
            self.inplanes = 128
            plan = torchvision_dilation_plan(layers, output_stride)
        else:
            self.conv1 = Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
            self.bn1 = BatchNorm2d(64)
            self.inplanes = 64
            plan = multigrid_dilation_plan(layers, output_stride)
        self.layer1 = self._make_layer(64, plan[0][1], plan[0][0])
        self.layer2 = self._make_layer(128, plan[1][1], plan[1][0])
        self.layer3 = self._make_layer(256, plan[2][1], plan[2][0])
        self.layer4 = self._make_layer(512, plan[3][1], plan[3][0])
        self._init_weight()
        if pretrained_url is not None:
            self._load_pretrained_model(pretrained_url)

    def _make_layer(self, planes, block_dilations, stride):
        blocks = []
        for i, d in enumerate(block_dilations):
            s = stride if i == 0 else 1
            down = None
            if i == 0 and (s != 1 or self.inplanes != planes * 4):
                down = nn.Sequential(Conv2d(self.inplanes, planes * 4, 1, stride=s, bias=False),
                                     BatchNorm2d(planes * 4))
            blocks.append(Bottleneck(self.inplanes, planes, s, d, down))
            self.inplanes = planes * 4
        return nn.Sequential(*blocks)

    def stem(self, img):
        """planar image -> stem convolution(s) -> bn1 -> ReLU -> max-pool 3x3/2 (NHWC); the one entry of forward,
        forward_low_level and eval mode."""
        if not self.deep_stem:
            x = ops.stem_conv(img, self.conv1.weight, want_bn_stats=self.training)
            return ops.maxpool3x3s2(self.bn1(x, relu=True))
        c1, b1, c2, b2, c3 = self.conv1[0], self.conv1[1], self.conv1[3], self.conv1[4], self.conv1[6]
        x = b1(ops.stem_conv(img, c1.weight, want_bn_stats=self.training), relu=True)
        if ops.conv_bn_unit_ok(c2, b2) and ops.conv_bn_unit_ok(c3, self.bn1):
            # fp16-pair path, as in Bottleneck: the 64-channel activation between the two units only exists as the
            # fp16 pair the second convolution reads
            x = ops.conv_bn_act(x, c2, b2, relu=True, out_mode='pair')
            x = ops.conv_bn_act(x, c3, self.bn1, relu=True, out_mode='fp32')
        else:
            x = self.bn1(c3(b2(c2(x), relu=True)), relu=True)
        return ops.maxpool3x3s2(x)

    def forward(self, img):
        x = self.layer1(self.stem(img))
        x = self.layer2(x)
        x = self.layer3(x)
        return self.layer4(x)

    def forward_low_level(self, img):
        """-> (layer1 output [N,256,H/4,W/4], layer4 output): the low-level features a DeepLabV3+ decoder reads."""
        low = self.layer1(self.stem(img))
        return low, self.layer4(self.layer3(self.layer2(low)))

    def _init_weight(self):
        for m in self.modules():
            if isinstance(m, Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

    def _load_pretrained_model(self, url):
        """resnet.py:145-156: a local file is loaded as a complete state dict; a URL goes through the model zoo and is
        key-filtered (torchvision / COCO checkpoints carry an ``fc`` head the dilated backbone does not have).  The zoo
        file is looked up in $PXL_PRETRAINED_DIR and the torch-hub cache before any download is attempted; weights that
        were requested but cannot be obtained are an error, never a silent random init.
        Deep stem: the checkpoint (CPS's resnet101_v1c.pth / UniMatch's resnet101.pth layout) may carry a ``module.``
        prefix and keys the backbone does not have (``fc.*``), which are dropped; every parameter and BN running
        statistic of the backbone must be present with its exact shape, so a 7x7-stem file fails instead of loading
        partially."""
        if self.deep_stem:
            load_complete_state_dict(self, url, 'deep-stem')
            return
        if os.path.isfile(url):
            self.load_state_dict(torch.load(url, map_location='cpu'))
            return
        pre = load_zoo_state_dict(url)
        own = self.state_dict()
        own.update({k: v for k, v in pre.items() if k in own})
        self.load_state_dict(own)


def multigrid_dilation_plan(layers, output_stride):
    """-> (stride, block dilations) per layer: resnet.py:58-66 and the multi-grid layer4, (1, 2, 4) x its dilation."""
    strides, dilations = {16: ((1, 2, 2, 1), (1, 1, 1, 2)), 8: ((1, 2, 1, 1), (1, 1, 2, 4))}[output_stride]
    return [(strides[i], [dilations[i]] * layers[i]) for i in range(3)] + \
        [(strides[3], [m * dilations[3] for m in (1, 2, 4)])]


def torchvision_dilation_plan(layers, output_stride):
    """-> (stride, block dilations) per layer: torchvision's ResNet._make_layer with replace_stride_with_dilation
    [F, F, T] (OS16) or [F, T, T] (OS8), the plan of CPS's _nostride_dilate.  A dilated layer has stride 1 and its
    first block keeps the previous layer's dilation."""
    dilate = (False, False, True) if output_stride == 16 else (False, True, True)
    plan, dilation = [(1, [1] * layers[0])], 1
    for n, d in zip(layers[1:], dilate):
        if d:
            prev, dilation = dilation, dilation * 2
            plan.append((1, [prev] + [dilation] * (n - 1)))
        else:
            plan.append((2, [dilation] * n))
    return plan


def load_complete_state_dict(module, url, kind):
    """Load a local file (or zoo URL) that must hold every parameter and BN running statistic of ``module`` with its
    exact shape: an optional ``module.`` prefix is stripped and keys the module does not have (``fc.*``) are dropped;
    a missing or misshapen key stops the load and is named."""
    pre = torch.load(url, map_location='cpu') if os.path.isfile(url) else load_zoo_state_dict(url)
    pre = {(k[len('module.'):] if k.startswith('module.') else k): v for k, v in pre.items()}
    own = module.state_dict()
    for k, v in own.items():
        if k.endswith('.num_batches_tracked') and k not in pre:
            continue
        if k not in pre:
            logger.log_err('pretrained backbone {0} has no key {1} (a {2} backbone needs every parameter and '
                           'BN running statistic of the network)\n'.format(url, k, kind))
        if tuple(pre[k].shape) != tuple(v.shape):
            logger.log_err('pretrained backbone {0}: key {1} has shape {2}, the {3} backbone needs {4}\n'
                           .format(url, k, tuple(pre[k].shape), kind, tuple(v.shape)))
    module.load_state_dict({k: pre.get(k, v) for k, v in own.items()})


def load_zoo_state_dict(url):
    name = os.path.basename(url)
    cands = []
    if os.environ.get('PXL_PRETRAINED_DIR'):
        cands.append(os.path.join(os.environ['PXL_PRETRAINED_DIR'], name))
    try:
        cands.append(os.path.join(torch.hub.get_dir(), 'checkpoints', name))
    except Exception:
        pass
    for path in cands:
        if os.path.isfile(path):
            return torch.load(path, map_location='cpu')
    try:
        return torch.hub.load_state_dict_from_url(url, map_location='cpu')      # model_zoo.load_url
    except Exception as e:
        logger.log_err('pretrained backbone {0} was requested but is neither cached ({1}) nor downloadable ({2}).\n'
                       'Pass --pretrained-backbone none to train from the reference initialisers.\n'
                       .format(url, ', '.join(cands), e))


# name -> (blocks per layer, deep stem)
BACKBONES = {
    'resnet50': ((3, 4, 6, 3), False),
    'resnet101': ((3, 4, 23, 3), False),
    'resnet101-coco': ((3, 4, 23, 3), False),
    'resnet50-deepstem': ((3, 4, 6, 3), True),
    'resnet101-deepstem': ((3, 4, 23, 3), True),
}


def build_backbone(backbone, output_stride, pretrained_url=None):
    if backbone not in BACKBONES:
        raise NotImplementedError(backbone)
    layers, deep_stem = BACKBONES[backbone]
    return ResNet(list(layers), output_stride, pretrained_url, deep_stem=deep_stem)
