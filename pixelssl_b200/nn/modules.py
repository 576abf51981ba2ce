"""nn.Module shells around the CUDA ops.  They only hold parameters (in the physical layouts the
kernels want) under the same attribute names as torch's modules, so ``state_dict`` keys and
shapes equal the reference's checkpoints."""
import math

import torch
import torch.nn as nn

from .. import ops

CL = torch.channels_last


class Conv2d(nn.Module):
    """nn.Conv2d replacement: weight is logical [Cout,Cin,kh,kw], stored channels_last
    (= [Cout][kh*kw][Cin], the K-major operand of the implicit GEMM)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, bias=True, out_lanes=0):
        super().__init__()
        self.out_lanes = out_lanes        # > out_channels: zero-padded output lanes (e.g. 21 -> 32)
        self.feeds_bn = False             # set by the owner when a BatchNorm2d consumes the output directly
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size = (kernel_size, kernel_size)
        self.stride, self.padding, self.dilation = stride, padding, dilation
        w = torch.empty(out_channels, in_channels, kernel_size, kernel_size).contiguous(memory_format=CL)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))        # nn.Conv2d default
        self.weight = nn.Parameter(w)
        if bias:
            bound = 1 / math.sqrt(in_channels * kernel_size * kernel_size)
            self.bias = nn.Parameter(torch.empty(out_channels).uniform_(-bound, bound))
        else:
            self.register_parameter('bias', None)

    def forward(self, x):
        w = self.weight
        if x.shape[1] > self.in_channels:
            # input lanes were zero-padded (e.g. 21 -> 32 so the wgmma kernel applies): pad the weight
            # with matching zero channels; tiny tensor, plain autograd ops
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, x.shape[1] - self.in_channels)).contiguous(memory_format=CL)
        return ops.conv2d(ops.as_cl(x), w, self.bias, self.stride, self.padding, self.dilation, self.out_lanes,
                          want_bn_stats=self.feeds_bn and self.training)

    def extra_repr(self):
        return '{in_channels}, {out_channels}, kernel_size={kernel_size}, stride={stride}, padding={padding}, ' \
               'dilation={dilation}'.format(**self.__dict__)


class DepthwiseConv2d(nn.Module):
    """nn.Conv2d(channels, channels, 3, stride, padding=dilation, dilation=dilation, groups=channels, bias=False)
    replacement: weight [C,1,3,3] (contiguous = [C][9], the layout the depthwise kernels read)."""

    def __init__(self, channels, stride=1, dilation=1):
        super().__init__()
        self.in_channels = self.out_channels = channels
        self.kernel_size = (3, 3)
        self.stride, self.dilation, self.padding = stride, dilation, dilation
        w = torch.empty(channels, 1, 3, 3)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))        # nn.Conv2d default
        self.weight = nn.Parameter(w)

    def forward(self, x):
        return ops.depthwise_conv(ops.as_cl(x), self.weight, self.stride, self.dilation)

    def extra_repr(self):
        return '{in_channels}, stride={stride}, dilation={dilation}'.format(**self.__dict__)


class BatchNorm2d(nn.Module):
    """SynchronizedBatchNorm2d of the reference (sync_batchnorm/batchnorm.py:180): momentum 0.1,
    eps 1e-5, affine.  ``forward(x, relu=False, residual=None)`` fuses what follows the BN in
    Bottleneck.forward.  Across processes the batch statistics are all-reduced over
    ``sync_group`` (set by EngineParallel when torch.distributed has world_size > 1), which is the
    reference's cross-replica reduction (batchnorm.py:55-78) over NCCL instead of Python threads."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super().__init__()
        self.num_features, self.eps, self.momentum = num_features, eps, momentum
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.ones(num_features))
        self.register_buffer('num_batches_tracked', torch.tensor(0, dtype=torch.long))
        self.sync_group = None
        self.multi_replica_formula = False     # clamp(var, eps) instead of var + eps (batchnorm.py:125)

    def forward(self, x, relu=False, residual=None):
        # num_batches_tracked stays 0 like the reference's: _SynchronizedBatchNorm.forward calls F.batch_norm
        # directly (batchnorm.py:50-53) and never touches the counter, so its checkpoints always hold 0
        return ops.bn_act(ops.as_cl(x), self.weight, self.bias, self.running_mean, self.running_var,
                          training=self.training, momentum=self.momentum, eps=self.eps, relu=relu,
                          residual=residual, group=self.sync_group if self.training else None,
                          clamp_var=self.multi_replica_formula)

    def extra_repr(self):
        return '{num_features}, eps={eps}, momentum={momentum}'.format(**self.__dict__)


SynchronizedBatchNorm2d = BatchNorm2d


# decoder building blocks shared by the PSPNet head (_pspnet.py:15-54) and the CCT decoders (ssl_cct.py:501-539)
class PixelShuffle(nn.Module):
    """conv1x1 C -> 4C (bias, ICNR init) + ReLU + nn.PixelShuffle(2)."""

    def __init__(self, n_channels, scale=2):
        super().__init__()
        assert scale == 2
        self.n_channels = n_channels
        self.conv = Conv2d(n_channels, n_channels * 4, 1, bias=True)
        k = nn.init.kaiming_normal_(torch.zeros(n_channels, n_channels, 1, 1)).transpose(0, 1)
        k = k.contiguous().view(n_channels, n_channels, -1).repeat(1, 1, 4)
        self.conv.weight.data.copy_(k.contiguous().view(n_channels, n_channels * 4, 1, 1).transpose(0, 1))

    def forward(self, x):
        y = ops.leaky_relu(self.conv(x), 0.0)
        return ops.pixel_shuffle2(y, self.n_channels)


def upsample(in_channels, out_channels, upscale):
    layers = [Conv2d(in_channels, out_channels, 1, bias=False, out_lanes=(out_channels + 31) // 32 * 32)]
    nn.init.kaiming_normal_(layers[0].weight.data, nonlinearity='relu')
    for _ in range(int(math.log(upscale, 2))):
        layers.append(PixelShuffle(out_channels, scale=2))
    return nn.Sequential(*layers)



