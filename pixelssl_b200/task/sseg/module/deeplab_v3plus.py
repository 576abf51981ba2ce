"""DeepLabV3+ (Chen et al., ECCV 2018) on the H100 kernels: the dilated ResNet or aligned Xception-65 backbone -> ASPP with image pooling
(parameter layout of torchvision.models.segmentation.deeplabv3.ASPP, without its dropout) -> decoder on the
stride-4 low-level features -> 1x1 classifier -> bilinear (align_corners=True) to the input size.

Every convolution runs on the library's convolution kernels.  The two concatenations are single launches of
``ops.lane_concat`` whose backward gathers in a fixed order.  Two shapes are padded so that the wgmma kernels
(Cin % 64 == 0 on the fp16-pair path) take every head convolution in the tensor-core modes:
  * ``decoder.reduce`` (256 -> 48, or 128 -> 48 on Xception-65) runs as 256 -> 64 with 16 zero output channels (zero weight rows, zero BN affine);
  * the decoder concat holds 256 + 48 channels in 320 lanes, and ``decoder.fuse.0``'s [256, 304, 3, 3] weight is
    zero-padded to 320 input channels at use.
The checkpoint shapes stay the unpadded ones."""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .... import ops
from ....nn.modules import Conv2d, BatchNorm2d
from .resnet import build_backbone
from .xception import AlignedXception

ASPP_RATES = {16: (6, 12, 18), 8: (12, 24, 36)}
DECODER_LANES = 320          # 256 upsampled ASPP channels + 48 reduced low-level channels, rounded up to 64
REDUCE_LANES = 64            # decoder.reduce's 48 output channels, rounded up to 64


def _conv_bn_relu(x, conv, bn):
    if ops.conv_bn_unit_ok(conv, bn):
        return ops.conv_bn_act(x, conv, bn, relu=True, out_mode='fp32')
    return bn(conv(x), relu=True)


class _ConvBnReLU(nn.Sequential):
    """Sequential(Conv2d, BatchNorm2d, ReLU), bias-free: torchvision's ASPPConv / 1x1 branch / projection layout."""

    def __init__(self, in_channels, out_channels, kernel_size=1, dilation=1):
        pad = dilation * (kernel_size // 2)
        super().__init__(Conv2d(in_channels, out_channels, kernel_size, padding=pad, dilation=dilation, bias=False),
                         BatchNorm2d(out_channels), nn.Identity())
        self[0].feeds_bn = True

    def forward(self, x):
        return _conv_bn_relu(x, self[0], self[1])


class _ImagePooling(nn.Sequential):
    """torchvision's ASPPPooling: Sequential(AdaptiveAvgPool2d(1), Conv2d 1x1, BN, ReLU); the broadcast back to h x w
    is done by the ASPP concatenation."""

    def __init__(self, in_channels, out_channels):
        super().__init__(nn.Identity(), Conv2d(in_channels, out_channels, 1, bias=False), BatchNorm2d(out_channels),
                         nn.Identity())
        self[1].feeds_bn = True

    def check_batch(self, x):
        """In training the BN of this branch sees one value per channel and sample; like torch, refuse a global batch
        of one instead of normalising by a zero variance."""
        bn = self[2]
        if not bn.training:
            return
        n = x.shape[0]
        if bn.sync_group is not None:
            import torch.distributed as dist
            n *= dist.get_world_size(bn.sync_group)
        if n <= 1:
            raise ValueError('Expected more than 1 value per channel when training, got input size {0}'.format(
                torch.Size([n, bn.num_features, 1, 1])))

    def forward(self, x):
        return _conv_bn_relu(ops.spatial_mean(x), self[1], self[2])


class ASPP(nn.Module):
    def __init__(self, in_channels, rates, out_channels=256):
        super().__init__()
        self.convs = nn.ModuleList([_ConvBnReLU(in_channels, out_channels, 1)] +
                                   [_ConvBnReLU(in_channels, out_channels, 3, r) for r in rates] +
                                   [_ImagePooling(in_channels, out_channels)])
        self.project = _ConvBnReLU(len(self.convs) * out_channels, out_channels, 1)

    def forward(self, x):
        self.convs[-1].check_batch(x)
        branches = [m(x) for m in self.convs]
        return self.project(ops.lane_concat([(b, b.shape[1]) for b in branches], x.shape[2:]))


class _Reduce(_ConvBnReLU):
    """1x1 256 -> 48 + BN + ReLU, computed on REDUCE_LANES output channels: the extra weight rows and BN affine
    parameters are zero, so the extra lanes hold exact zeros and take no part in any gradient."""

    def forward(self, x):
        conv, bn = self[0], self[1]
        pad = REDUCE_LANES - conv.out_channels
        w = F.pad(conv.weight, (0, 0, 0, 0, 0, 0, 0, pad)).contiguous(memory_format=torch.channels_last)
        y = ops.conv2d(ops.as_cl(x), w, None, want_bn_stats=bn.training)
        gamma, beta = F.pad(bn.weight, (0, pad)), F.pad(bn.bias, (0, pad))
        rm = torch.cat([bn.running_mean, bn.running_mean.new_zeros(pad)])
        rv = torch.cat([bn.running_var, bn.running_var.new_ones(pad)])
        out = ops.bn_act(y, gamma, beta, rm, rv, training=bn.training, momentum=bn.momentum, eps=bn.eps, relu=True,
                         group=bn.sync_group if bn.training else None, clamp_var=bn.multi_replica_formula)
        if bn.training:
            with torch.no_grad():
                bn.running_mean.copy_(rm[:conv.out_channels])
                bn.running_var.copy_(rv[:conv.out_channels])
        return out


class Decoder(nn.Module):
    def __init__(self, low_channels=256, aspp_channels=256, reduced=48, out_channels=256):
        super().__init__()
        self.reduce = _Reduce(low_channels, reduced, 1)
        self.fuse = nn.Sequential(
            Conv2d(aspp_channels + reduced, out_channels, 3, padding=1, bias=False), BatchNorm2d(out_channels), nn.Identity(),
            Conv2d(out_channels, out_channels, 3, padding=1, bias=False), BatchNorm2d(out_channels), nn.Identity())
        self.fuse[0].feeds_bn = self.fuse[3].feeds_bn = True

    def forward(self, aspp_out, low):
        red = self.reduce(low)
        x = ops.lane_concat([(aspp_out, aspp_out.shape[1]), (red, self.reduce[0].out_channels)], low.shape[2:],
                            DECODER_LANES)
        x = _conv_bn_relu(x, self.fuse[0], self.fuse[1])
        return _conv_bn_relu(x, self.fuse[3], self.fuse[4])


class DeepLabV3Plus(nn.Module):
    def __init__(self, backbone='resnet101', output_stride=16, num_classes=21, sync_bn=True, freeze_bn=False,
                 pretrained_backbone_url=None):
        super().__init__()
        self.num_classes = num_classes
        if backbone == 'xception65':
            self.backbone = AlignedXception(output_stride, pretrained_backbone_url)
            self.FP_CHANNELS = (128, 2048)         # block1's (ReLU'd) output is the low-level feature
        else:
            self.backbone = build_backbone(backbone, output_stride, pretrained_backbone_url)
        self.aspp = ASPP(2048, ASPP_RATES[output_stride], 256)
        self.decoder = Decoder(self.FP_CHANNELS[0], 256, 48, 256)
        self.classifier = Conv2d(256, num_classes, 1, bias=True, out_lanes=(num_classes + 31) // 32 * 32)
        for m in list(self.aspp.modules()) + list(self.decoder.modules()):
            if isinstance(m, Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
        self.classifier.weight.data.normal_(0, 0.01)
        self.classifier.bias.data.zero_()
        self._freeze = freeze_bn
        if freeze_bn:
            self.freeze_bn()

    def forward(self, img):
        low, bx = self.backbone.forward_low_level(img)
        x = self.decoder(self.aspp(bx), low)
        x = self.classifier(x)
        x = ops.bilinear(x, img.shape[2:], align_corners=True, channels=self.num_classes, nhwc=True)
        return x, bx

    # the feature maps forward_fp perturbs, in the order of its ``scales``: layer1 (the decoder's low-level input) and
    # layer4 (the ASPP input), as UniMatch drops both; (128, 2048) on Xception-65
    FP_CHANNELS = (256, 2048)

    def forward_fp(self, img, scales):
        """UniMatch's feature-perturbation forward: the head runs once on the clean features followed by their
        Dropout2d copies (``scales``: factors [n, 256] for layer1 and [n, 2048] for layer4) -> (pred, pred_fp,
        latent).  Each half is upsampled on its own, so the backward never splits a full-resolution map."""
        n = img.shape[0]
        low, bx = self.backbone.forward_low_level(img)
        x = self.decoder(self.aspp(ops.fp_dup(bx, scales[1])), ops.fp_dup(low, scales[0]))
        x = self.classifier(x)
        up = [ops.bilinear(x[k * n:(k + 1) * n], img.shape[2:], align_corners=True, channels=self.num_classes,
                           nhwc=True) for k in (0, 1)]
        return up[0], up[1], bx

    # No train() override, as in DeepLabV2: freeze_bn() applies once at construction.

    def freeze_bn(self):
        for m in self.modules():
            if isinstance(m, BatchNorm2d):
                m.eval()

    def _params_of(self, *roots):
        for root in roots:
            for p in root.parameters():
                if p.requires_grad:
                    yield p

    def get_1x_lr_params(self):
        return self._params_of(self.backbone)

    def get_10x_lr_params(self):
        return self._params_of(self.aspp, self.decoder, self.classifier)
