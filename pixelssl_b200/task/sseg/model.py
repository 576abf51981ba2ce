"""Task-model plugin for semantic segmentation: the contract of task/sseg/model.py:11-125
(export fns ``deeplabv2()`` / ``pspnet()``, plus ``deeplabv3plus()``, ``cls(args)``, ``.param_groups``,
``forward(inp: tuple) -> (resulter, debugger)`` with 'pred', 'activated_pred', 'ssls4l_rc_inp',
'sslcct_ad_inp').  Inside validation with a multi-view protocol, ``forward`` of an eval-mode model returns the
ensemble of task/sseg/evaluation.py instead (no 'sslcct_ad_inp')."""
import torch.nn as nn

from ... import ops
from ...utils import logger, cmd
from . import evaluation
from .module import deeplab_v2, deeplab_v3plus, pspnet as pspnet_module
from .module.resnet import BACKBONES


def add_parser_arguments(parser):
    parser.add_argument('--output-stride', type=int, default=16)
    parser.add_argument('--backbone', type=str, default='resnet101')
    parser.add_argument('--freeze-bn', type=cmd.str2bool, default=False)
    # 'auto' = the URL the reference hard-codes for args.backbone (task/sseg/model.py:69-80), served from the local
    # torch-hub cache / $PXL_PRETRAINED_DIR when present, downloaded otherwise (the *-deepstem backbones and xception65
    # have none);
    # 'none' = keep the reference initialisers; anything else = a local file or URL.  A requested-but-unloadable
    # backbone is an error.
    parser.add_argument('--pretrained-backbone', type=str, default='auto')


def deeplabv2():
    return DeepLabV2


def pspnet():
    return PSPNet


def deeplabv3plus():
    return DeepLabV3Plus


class LazyActivation:
    """Tuple-like holder of the activated prediction.  The reference computes softmax on every
    forward (model.py:62) although MT/SupOnly training never reads it; here the 8*C B/pixel pass
    only runs if something actually indexes / iterates the tuple."""

    def __init__(self, pred):
        self._pred, self._val = pred, None

    def _get(self):
        if self._val is None:
            self._val = (ops.softmax_planar(self._pred),)
        return self._val

    def __len__(self):
        return 1

    def __iter__(self):
        return iter(self._get())

    def __getitem__(self, i):
        return self._get()[i]


class TaskModel(nn.Module):
    """pixelssl/task_template/model.py:29-85."""

    def __init__(self, args=None):
        super().__init__()
        self.args = args
        self.model = None
        self.param_groups = []


# task/sseg/model.py:69-80 / :89-98
PRETRAINED_BACKBONE_URLS = {
    'resnet50': 'https://download.pytorch.org/models/resnet50-19c8e357.pth',
    'resnet101': 'https://download.pytorch.org/models/resnet101-5d3b4d8f.pth',
    'resnet101-coco': 'http://vllab1.ucmerced.edu/~whung/adv-semi-seg/resnet101COCO-41f33a49.pth',
}


def pretrained_backbone_url(args):
    """-> URL / path handed to the backbone, or None for the reference initialisers."""
    want = getattr(args, 'pretrained_backbone', 'auto')
    if want in (None, '', 'none', 'None', False):
        return None
    if want == 'auto':
        if args.backbone == 'xception65':
            logger.log_err('--pretrained-backbone auto has no download for the backbone xception65: pass the local file '
                           'of its ImageNet weights (in the key layout of the aligned Xception-65 module tree) or '
                           'none\n')
        if args.backbone.endswith('-deepstem'):
            logger.log_err('--pretrained-backbone auto has no download for the backbone {0}: pass the local file of its '
                           'ImageNet weights (CPS resnet101_v1c.pth / UniMatch pretrained/resnet101.pth layout) or '
                           'none\n'.format(args.backbone))
        return PRETRAINED_BACKBONE_URLS.get(args.backbone)
    return want


class DeepLabV2(TaskModel):
    MODULE = deeplab_v2.DeepLabV2
    BACKBONES = tuple(BACKBONES)

    def __init__(self, args):
        super().__init__(args)
        if args.backbone not in self.BACKBONES:
            logger.log_err('{0} does not support the backbone: {1}\n'.format(type(self).__name__, args.backbone))
        self.model = self.MODULE(backbone=args.backbone, output_stride=args.output_stride, num_classes=args.num_classes,
                                 sync_bn=True, freeze_bn=args.freeze_bn,
                                 pretrained_backbone_url=pretrained_backbone_url(args))
        self.param_groups = [
            {'params': list(self.model.get_1x_lr_params()), 'lr': args.lr},
            {'params': list(self.model.get_10x_lr_params()), 'lr': args.lr * 10},
        ]

    def forward(self, inp):
        resulter, debugger = {}, {}
        if not len(inp) == 1:
            logger.log_err('Semantic segmentation model DeepLab requires only one input\n'
                           'However, {0} inputs are given\n'.format(len(inp)))
        if evaluation.multi_view(self):
            return evaluation.forward_views(self, inp)
        pred, latent = self.model(inp[0])
        resulter['pred'] = (pred,)
        resulter['activated_pred'] = LazyActivation(pred)
        resulter['ssls4l_rc_inp'] = pred
        resulter['sslcct_ad_inp'] = latent
        return resulter, debugger

    @property
    def fp_channels(self):
        """Channel counts of the feature maps ``forward_fp`` perturbs, in the order of its ``scales``."""
        return self.model.FP_CHANNELS

    def forward_fp(self, inp, scales):
        """UniMatch's forward with feature perturbation: ``scales`` holds one [n, C] tensor of Dropout2d factors per
        entry of ``fp_channels``.  -> (resulter of the clean features, resulter of the perturbed ones); the head
        runs once on both, so its BatchNorm statistics cover both."""
        if not len(inp) == 1:
            logger.log_err('Semantic segmentation model DeepLab requires only one input\n'
                           'However, {0} inputs are given\n'.format(len(inp)))
        pred, pred_fp, latent = self.model.forward_fp(inp[0], scales)
        resulter = {'pred': (pred,), 'activated_pred': LazyActivation(pred), 'ssls4l_rc_inp': pred,
                    'sslcct_ad_inp': latent}
        resulter_fp = {'pred': (pred_fp,), 'activated_pred': LazyActivation(pred_fp)}
        return resulter, resulter_fp


class DeepLabV3Plus(DeepLabV2):
    """DeepLabV3+ with the DeepLabV2 plugin surface: same backbones, resulter keys and latent (the layer4 output);
    backbone at 1x lr, ASPP, decoder and classifier at 10x.  It also takes the aligned Xception-65 backbone."""
    MODULE = deeplab_v3plus.DeepLabV3Plus
    BACKBONES = tuple(BACKBONES) + ('xception65',)


class PSPNet(TaskModel):
    """task/sseg/model.py:84-125."""

    def __init__(self, args):
        super().__init__(args)
        if args.backbone not in BACKBONES:
            logger.log_err('PSPNet does not support the backbone: {0}\n'.format(args.backbone))
        self.model = pspnet_module.PSPNet(backbone=args.backbone, output_stride=args.output_stride,
                                          num_classes=args.num_classes, sync_bn=True, freeze_bn=args.freeze_bn,
                                          pretrained_backbone_url=pretrained_backbone_url(args))
        self.param_groups = [
            {'params': [p for p in self.model.get_backbone_params() if p.requires_grad], 'lr': args.lr},
            {'params': [p for p in self.model.get_psp_params() if p.requires_grad], 'lr': args.lr * 10},
            {'params': [p for p in self.model.get_decoder_params() if p.requires_grad], 'lr': args.lr * 10},
        ]

    def forward(self, inp):
        resulter, debugger = {}, {}
        if not len(inp) == 1:
            logger.log_err('Semantic segmentation model PSPNet requires only one input\n'
                           'However, {0} inputs are given\n'.format(len(inp)))
        if evaluation.multi_view(self):
            return evaluation.forward_views(self, inp)
        pred, latent = self.model(inp[0])
        resulter['pred'] = (pred,)
        resulter['activated_pred'] = LazyActivation(pred)
        resulter['ssls4l_rc_inp'] = pred
        resulter['sslcct_ad_inp'] = latent
        return resulter, debugger
