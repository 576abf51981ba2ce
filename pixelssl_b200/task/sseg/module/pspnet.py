"""PSPNet on the H100 kernels: module tree and forward order of task/sseg/module/_pspnet.py:57-128
(pyramid pooling bins 1/2/3/6 -> 1x1 conv + BN + ReLU -> bilinear (align_corners=False) -> concat with
the backbone features -> 3x3 conv 4096->512 + BN + ReLU -> conv1x1 + 3 x PixelShuffle decoder ->
bilinear (align_corners=True) to the input size)."""
import torch.nn as nn

from .... import ops
from ....nn.modules import Conv2d, BatchNorm2d, upsample
from .resnet import build_backbone


class _Stage(nn.Sequential):
    """Sequential(AdaptiveAvgPool2d, Conv2d, BN, ReLU) - indices as in the reference (_pspnet.py:89-94)."""

    def __init__(self, in_channels, out_channels, bin_sz):
        super().__init__(nn.Identity(), Conv2d(in_channels, out_channels, 1, bias=False), BatchNorm2d(out_channels), nn.Identity())
        self.bin_sz = bin_sz
        self[1].feeds_bn = True

    def forward(self, x):
        return self[2](self[1](ops.adaptive_avg_pool(x, self.bin_sz)), relu=True)


class _Bottleneck(nn.Sequential):
    def __init__(self, in_channels, out_channels):
        super().__init__(Conv2d(in_channels, out_channels, 3, padding=1, bias=False), BatchNorm2d(out_channels), nn.Identity())
        self[0].feeds_bn = True

    def forward(self, x):
        return self[1](self[0](x), relu=True)


class _PSPModule(nn.Module):
    def __init__(self, in_channels, bin_sizes):
        super().__init__()
        out_channels = in_channels // len(bin_sizes)
        self.stages = nn.ModuleList([_Stage(in_channels, out_channels, b) for b in bin_sizes])
        self.bottleneck = _Bottleneck(in_channels + out_channels * len(bin_sizes), out_channels)
        for m in self.modules():
            if isinstance(m, Conv2d):
                nn.init.kaiming_uniform_(m.weight, a=0, mode='fan_in', nonlinearity='relu')
            elif isinstance(m, BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def forward(self, features):
        return self.bottleneck(ops.pyramid_concat(features, [stage(features) for stage in self.stages]))


class PSPNet(nn.Module):
    def __init__(self, backbone='resnet50', output_stride=8, num_classes=21, sync_bn=True, freeze_bn=False,
                 pretrained_backbone_url=None):
        super().__init__()
        self.num_classes = num_classes
        self.backbone = build_backbone(backbone, output_stride, pretrained_backbone_url)
        self.psp = _PSPModule(2048, bin_sizes=[1, 2, 3, 6])
        self.decoder = upsample(512, num_classes, upscale=8)
        self._freeze = freeze_bn
        if freeze_bn:
            self.freeze_bn()

    def forward(self, img):
        bx = self.backbone(img)
        px = self.psp(bx)
        x = self.decoder(px)
        x = ops.bilinear(x, img.shape[2:], align_corners=True, channels=self.num_classes, nhwc=True)
        return x, px

    def train(self, mode=True):
        super().train(mode)
        if self._freeze:
            self.freeze_bn()
        return self

    def freeze_bn(self):
        for m in self.modules():
            if isinstance(m, BatchNorm2d):
                m.eval()

    def get_backbone_params(self):
        return self.backbone.parameters()

    def get_psp_params(self):
        return self.psp.parameters()

    def get_decoder_params(self):
        return self.decoder.parameters()
