"""DeepLab-v2 head on the H100 kernels (task/sseg/module/deeplab_v2.py:13-85): backbone ->
ASPP (4 dilated 3x3 convs 2048->C summed, ONE 36-tap kernel here) -> bilinear upsample
(align_corners=True) to the input size."""
import torch.nn as nn

from .... import ops
from ....nn.modules import Conv2d, BatchNorm2d
from .resnet import build_backbone


class Classifier_Module(nn.Module):
    def __init__(self, dilation_series, padding_series, num_classes, in_channels=2048):
        super().__init__()
        assert list(dilation_series) == list(padding_series)
        self.dilations = tuple(dilation_series)
        self.conv2d_list = nn.ModuleList(
            [Conv2d(in_channels, num_classes, 3, stride=1, padding=d, dilation=d, bias=True) for d in dilation_series])
        for m in self.conv2d_list:
            m.weight.data.normal_(0, 0.01)

    def forward(self, x):
        """-> channels_last [N, 32, h, w]; the first num_classes lanes are the logits."""
        return ops.aspp(ops.as_cl(x), [m.weight for m in self.conv2d_list], [m.bias for m in self.conv2d_list],
                        self.dilations)


class DeepLabV2(nn.Module):
    def __init__(self, backbone='resnet101', output_stride=16, num_classes=21, sync_bn=True, freeze_bn=False,
                 pretrained_backbone_url=None):
        super().__init__()
        self.num_classes = num_classes
        self.backbone = build_backbone(backbone, output_stride, pretrained_backbone_url)
        self.classifier = Classifier_Module([6, 12, 18, 24], [6, 12, 18, 24], num_classes)
        self._freeze = freeze_bn
        if freeze_bn:
            self.freeze_bn()

    def forward(self, img):
        bx = self.backbone(img)
        low = self.classifier(bx)
        x = ops.bilinear(low, img.shape[2:], align_corners=True, channels=self.num_classes, nhwc=True)
        return x, bx

    # the feature maps forward_fp perturbs, in the order of its ``scales``: the layer4 output the classifier reads
    FP_CHANNELS = (2048,)

    def forward_fp(self, img, scales):
        """UniMatch's feature-perturbation forward: the classifier runs once on ``[bx; bx * scales[0]]`` (Dropout2d
        factors [n, 2048]) -> (pred, pred_fp, latent).  Each half is upsampled on its own, so the backward
        never splits a full-resolution map."""
        n = img.shape[0]
        bx = self.backbone(img)
        low = self.classifier(ops.fp_dup(bx, scales[0]))
        up = [ops.bilinear(low[k * n:(k + 1) * n], img.shape[2:], align_corners=True, channels=self.num_classes,
                           nhwc=True) for k in (0, 1)]
        return up[0], up[1], bx

    # No train() override: like the reference (deeplab_v2.py:46-52, model.py:69-80) freeze_bn() is applied once at
    # construction and is undone by the .train() call that starts every epoch; BN layers that ARE in eval mode inside
    # a training graph are supported by ops.bn_act (running statistics as constants in the backward).

    def freeze_bn(self):
        for m in self.modules():
            if isinstance(m, BatchNorm2d):
                m.eval()

    def _params_of(self, root):
        for m in root.modules():
            if isinstance(m, (Conv2d, BatchNorm2d)):
                for p in m.parameters(recurse=False):
                    if p.requires_grad:
                        yield p

    def get_1x_lr_params(self):
        return self._params_of(self.backbone)

    def get_10x_lr_params(self):
        return self._params_of(self.classifier)
