"""Dilated ResNet backbone on the H100 kernels: parameter tree and forward order of
task/sseg/module/backbone/resnet.py:13-131 (Bottleneck, strides/dilations per output stride,
multi-grid layer4), with BN+ReLU(+residual) fused and NHWC activations throughout."""
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
    def __init__(self, layers, output_stride, pretrained_url=None):
        super().__init__()
        self.inplanes = 64
        if output_stride == 16:
            strides, dilations = [1, 2, 2, 1], [1, 1, 1, 2]
        elif output_stride == 8:
            strides, dilations = [1, 2, 1, 1], [1, 1, 2, 4]
        else:
            raise NotImplementedError
        self.conv1 = Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = BatchNorm2d(64)
        self.layer1 = self._make_layer(64, [dilations[0]] * layers[0], strides[0])
        self.layer2 = self._make_layer(128, [dilations[1]] * layers[1], strides[1])
        self.layer3 = self._make_layer(256, [dilations[2]] * layers[2], strides[2])
        self.layer4 = self._make_layer(512, [m * dilations[3] for m in (1, 2, 4)], strides[3])   # MG unit
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

    def forward(self, img):
        x = ops.stem_conv(img, self.conv1.weight, want_bn_stats=self.training)          # planar image -> NHWC
        x = self.bn1(x, relu=True)
        x = ops.maxpool3x3s2(x)
        x = self.layer1(x)
        x = self.layer2(x)
        x = self.layer3(x)
        return self.layer4(x)

    def forward_low_level(self, img):
        """-> (layer1 output [N,256,H/4,W/4], layer4 output): the low-level features a DeepLabV3+ decoder reads."""
        x = ops.stem_conv(img, self.conv1.weight, want_bn_stats=self.training)
        x = self.bn1(x, relu=True)
        low = self.layer1(ops.maxpool3x3s2(x))
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
        were requested but cannot be obtained are an error, never a silent random init."""
        if os.path.isfile(url):
            self.load_state_dict(torch.load(url, map_location='cpu'))
            return
        pre = load_zoo_state_dict(url)
        own = self.state_dict()
        own.update({k: v for k, v in pre.items() if k in own})
        self.load_state_dict(own)


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


def build_backbone(backbone, output_stride, pretrained_url=None):
    if backbone in ('resnet101', 'resnet101-coco'):
        return ResNet([3, 4, 23, 3], output_stride, pretrained_url)
    if backbone == 'resnet50':
        return ResNet([3, 4, 6, 3], output_stride, pretrained_url)
    raise NotImplementedError(backbone)
