"""Aligned Xception-65 backbone of DeepLabV3+ (Chen et al., ECCV 2018) on the H100 kernels, in the module layout of the
PyTorch port whose ``AlignedXception`` UniMatch's backbone file follows (so its checkpoints load key for key).

Layout quirks of that port that are reproduced: ReLU placeholders inside each block's ``rep`` shift its keys; a block
that starts with a ReLU applies it in place, so its skip branch reads the rectified input; the extra separable
convolution of a stride-1 ``is_last`` block has dilation 1.

Every block output in this network is read only through a ReLU (blocks 1 and 20 by the explicit ReLU, every other one
by the next block's leading in-place ReLU, which its skip also reads), so each block's last BatchNorm applies residual
+ ReLU in one launch and writes the rectified tensor the next block's depthwise convolution and skip both read.

Lane padding, invisible in the checkpoints (as ``decoder.reduce`` in deeplab_v3plus.py): maps are carried in lanes
rounded up to 64 channels - the 728-channel maps in 768 lanes and ``conv1``'s 32 outputs in 64 - with zero weight
rows / columns and zero BN affine parameters in the pad lanes, so the pad lanes hold exact zeros and every 1x1 and skip
convolution stays on the fp16-pair tensor-core kernels (Cin, Cout % 64 == 0).  The padded weights and BN vectors are
made at use; a padded BN's running statistics are copied back into the module's unpadded buffers."""
import math
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

from .... import ops
from ....nn.modules import Conv2d, BatchNorm2d, DepthwiseConv2d, LanePaddedBatchNorm
from .resnet import load_complete_state_dict

CL = torch.channels_last


def lanes(c):
    """Channel lanes a map of c channels is carried in."""
    return (c + 63) // 64 * 64


def _conv_view(conv, cin, cout):
    """conv (bias-free Conv2d) with its weight zero-padded to [cout, cin, k, k]; the attributes conv_bn_act reads."""
    w = conv.weight
    if (cin, cout) != (conv.in_channels, conv.out_channels):
        w = F.pad(w, (0, 0, 0, 0, 0, cin - conv.in_channels, 0, cout - conv.out_channels)).contiguous(memory_format=CL)
    return types.SimpleNamespace(weight=w, bias=None, out_lanes=0, in_channels=cin, out_channels=cout,
                                 stride=conv.stride, padding=conv.padding, dilation=conv.dilation)


def _conv_bn(x, conv, bn, cin, cout, relu, residual=None):
    """relu?(bn(conv(x)) + residual) on lane-padded maps: one fused unit on the fp16-pair path, else conv2d + bn_act."""
    cv, bv = _conv_view(conv, cin, cout), LanePaddedBatchNorm(bn, cout)
    if ops.conv_bn_unit_ok(cv, bv):
        y = ops.conv_bn_act(x, cv, bv, relu=relu, residual=residual, out_mode='fp32')
    else:
        y = bv(ops.conv2d(ops.as_cl(x), cv.weight, None, cv.stride, cv.padding, cv.dilation, want_bn_stats=bv.training),
               relu=relu, residual=residual)
    bv.done()
    return y


class SeparableConv2d(nn.Module):
    """Depthwise 3x3 (padding = dilation on every side: the port's fixed_padding) -> BN -> pointwise 1x1, bias-free."""

    def __init__(self, cin, cout, stride=1, dilation=1):
        super().__init__()
        self.conv1 = DepthwiseConv2d(cin, stride, dilation)
        self.bn = BatchNorm2d(cin)
        self.pointwise = Conv2d(cin, cout, 1, bias=False)
        self.pointwise.feeds_bn = True

    def unit(self, x, bn, relu, residual=None):
        """relu?(bn(self(x)) + residual): ``bn`` is the BatchNorm that follows this convolution in the tree.  On the
        fp16-pair path the depthwise BN's apply writes the pair the pointwise unit reads."""
        cin, cout = lanes(self.conv1.in_channels), lanes(self.pointwise.out_channels)
        pw = _conv_view(self.pointwise, cin, cout)
        bin_, bout = LanePaddedBatchNorm(self.bn, cin), LanePaddedBatchNorm(bn, cout)
        if ops.conv_bn_unit_ok(pw, bout):
            h = ops.depthwise_bn_pair(x, self.conv1.weight, bin_, self.conv1.stride, self.conv1.dilation)
            y = ops.conv_bn_act(h, pw, bout, relu=relu, residual=residual, out_mode='fp32')
        else:
            h = bin_(ops.depthwise_conv(x, self.conv1.weight, self.conv1.stride, self.conv1.dilation))
            y = bout(ops.conv2d(h, pw.weight, None, want_bn_stats=bout.training), relu=relu, residual=residual)
        bin_.done()
        bout.done()
        return y


def block_rep(cin, cout, reps, stride, dilation, start_with_relu, grow_first, is_last):
    """The port's Block.rep as (kind, cin, cout, stride, dilation) entries: 'relu', 'sep' or 'bn'."""
    rep, f = [], cin
    if grow_first:
        rep += [('relu',), ('sep', cin, cout, 1, dilation), ('bn', cout)]
        f = cout
    for _ in range(reps - 1):
        rep += [('relu',), ('sep', f, f, 1, dilation), ('bn', f)]
    if not grow_first:
        rep += [('relu',), ('sep', cin, cout, 1, dilation), ('bn', cout)]
    if stride != 1:
        rep += [('relu',), ('sep', cout, cout, 2, 1), ('bn', cout)]
    elif is_last:
        rep += [('relu',), ('sep', cout, cout, 1, 1), ('bn', cout)]
    return rep if start_with_relu else rep[1:]


def block_plan(output_stride):
    """(name, cin, cout, reps, stride, dilation, start_with_relu, grow_first, is_last) per block, and the dilation of
    conv3..5."""
    if output_stride == 16:
        entry3_stride, middle, exit_ = 2, 1, (1, 2)
    elif output_stride == 8:
        entry3_stride, middle, exit_ = 1, 2, (2, 4)
    else:
        raise NotImplementedError
    plan = [('block1', 64, 128, 2, 2, 1, False, True, False),
            ('block2', 128, 256, 2, 2, 1, False, True, False),
            ('block3', 256, 728, 2, entry3_stride, 1, True, True, True)]
    plan += [('block%d' % i, 728, 728, 3, 1, middle, True, True, False) for i in range(4, 20)]
    plan += [('block20', 728, 1024, 2, 1, exit_[0], True, False, True)]
    return plan, exit_[1]


class Block(nn.Module):
    def __init__(self, cin, cout, reps, stride=1, dilation=1, start_with_relu=True, grow_first=True, is_last=False):
        super().__init__()
        if cout != cin or stride != 1:
            self.skip = Conv2d(cin, cout, 1, stride=stride, bias=False)
            self.skip.feeds_bn = True
            self.skipbn = BatchNorm2d(cout)
        else:
            self.skip = None
        self.rep = nn.Sequential(*[nn.ReLU(inplace=True) if e[0] == 'relu' else
                                   SeparableConv2d(*e[1:]) if e[0] == 'sep' else BatchNorm2d(e[1])
                                   for e in block_rep(cin, cout, reps, stride, dilation, start_with_relu, grow_first,
                                                      is_last)])
        self.cin, self.cout = cin, cout

    def forward(self, x):
        """x: the block input, already rectified (see the module docstring) -> relu(rep(x) + skip(x))."""
        skip = x if self.skip is None else _conv_bn(x, self.skip, self.skipbn, lanes(self.cin), lanes(self.cout), False)
        seps = [(m, self.rep[i + 1]) for i, m in enumerate(self.rep) if isinstance(m, SeparableConv2d)]
        for k, (sep, bn) in enumerate(seps):
            last = k == len(seps) - 1
            x = sep.unit(x, bn, relu=True, residual=skip if last else None)
        return x


class AlignedXception(nn.Module):
    def __init__(self, output_stride=16, pretrained_url=None):
        super().__init__()
        plan, exit_dilation = block_plan(output_stride)
        self.conv1 = Conv2d(3, 32, 3, stride=2, padding=1, bias=False)
        self.bn1 = BatchNorm2d(32)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = Conv2d(32, 64, 3, padding=1, bias=False)
        self.conv2.feeds_bn = True
        self.bn2 = BatchNorm2d(64)
        for name, *spec in plan:
            setattr(self, name, Block(*spec))
        self.conv3 = SeparableConv2d(1024, 1536, 1, exit_dilation)
        self.bn3 = BatchNorm2d(1536)
        self.conv4 = SeparableConv2d(1536, 1536, 1, exit_dilation)
        self.bn4 = BatchNorm2d(1536)
        self.conv5 = SeparableConv2d(1536, 2048, 1, exit_dilation)
        self.bn5 = BatchNorm2d(2048)
        self.block_names = [p[0] for p in plan]
        self._init_weight()
        if pretrained_url is not None:
            load_complete_state_dict(self, pretrained_url, 'xception65')

    def forward_low_level(self, img):
        """-> (low-level features [N,128,H/4,W/4] after block1's ReLU, the 2048-channel output at stride OS)."""
        w1 = F.pad(self.conv1.weight, (0, 0, 0, 0, 0, 0, 0, 64 - 32)).contiguous(memory_format=CL)
        b1 = LanePaddedBatchNorm(self.bn1, 64)
        x = b1(ops.stem_conv(img, w1, want_bn_stats=self.training), relu=True)        # 32 channels in 64 lanes
        b1.done()
        x = _conv_bn(x, self.conv2, self.bn2, 64, 64, True)
        low = None
        for name in self.block_names:
            x = getattr(self, name)(x)
            if low is None:
                low = x
        x = self.conv3.unit(x, self.bn3, relu=True)
        x = self.conv4.unit(x, self.bn4, relu=True)
        return low, self.conv5.unit(x, self.bn5, relu=True)

    def forward(self, img):
        return self.forward_low_level(img)[1]

    def _init_weight(self):
        for m in self.modules():
            if isinstance(m, (Conv2d, DepthwiseConv2d)):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
