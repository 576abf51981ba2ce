"""CPU oracle for DeepLabV3+ on the aligned Xception-65 backbone (``--backbone xception65``).  TEST INFRASTRUCTURE ONLY.

A functional torch-CPU restatement (``F.conv2d(groups=C)`` for the depthwise convolutions) of the module tree of the
PyTorch port whose ``AlignedXception`` UniMatch's backbone file follows, in fp32 or fp64: entry flow (conv1 3x3/2 3->32,
conv2 3x3 32->64, blocks 1-3), middle flow (blocks 4-19, 728 channels), exit flow (block 20, conv3-5).  The low-level
feature is block1's output after the ReLU (128 channels, stride 4); the output has 2048 channels at stride OS.
PixelSSL has no Xception, so there is no reference run to pin this file to; ``tests/test_host_xception.py`` pins it
to an nn.Module restatement built with nn.Conv2d(groups=C) and nn.ReLU(inplace=True).

The DeepLabV3+ head is ``deeplabv3plus_oracle``'s with ``decoder.reduce`` reading the 128-channel low-level feature;
``xception()`` points the names that oracle (and its step oracle) looks up at this backbone for a ``with`` block."""
import contextlib

import torch.nn.functional as F

from . import deeplabv3plus_oracle as D
from . import sseg_oracle as O


def block_rep(cin, cout, reps, stride, dilation, start_with_relu, grow_first, is_last):
    """The port's Block.rep as entries ('relu',), ('sep', cin, cout, stride, dilation), ('bn', channels)."""
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
        rep += [('relu',), ('sep', cout, cout, 1, 1), ('bn', cout)]    # dilation 1: the port's
    return rep if start_with_relu else rep[1:]


def block_plan(output_stride=16):
    """-> ([(name, cin, cout, reps, stride, dilation, start_with_relu, grow_first, is_last)], dilation of conv3-5)."""
    entry3_stride, middle, exit_ = {16: (2, 1, (1, 2)), 8: (1, 2, (2, 4))}[output_stride]
    plan = [('block1', 64, 128, 2, 2, 1, False, True, False),
            ('block2', 128, 256, 2, 2, 1, False, True, False),
            ('block3', 256, 728, 2, entry3_stride, 1, True, True, True)]
    plan += [('block%d' % i, 728, 728, 3, 1, middle, True, True, False) for i in range(4, 20)]
    plan += [('block20', 728, 1024, 2, 1, exit_[0], True, False, True)]
    return plan, exit_[1]


def _sep_shapes(p, cin, cout):
    return [(p + '.conv1.weight', (cin, 1, 3, 3), 'conv'), (p + '.bn.weight', (cin,), 'bn_w'),
            (p + '.bn.bias', (cin,), 'bn_b'), (p + '.pointwise.weight', (cout, cin, 1, 1), 'conv')]


def _bn_shapes(p, c):
    return [(p + '.weight', (c,), 'bn_w'), (p + '.bias', (c,), 'bn_b')]


def backbone_param_shapes(output_stride=16, blocks=None):
    """(name, shape, kind) of the backbone in ``parameters()`` order (``blocks`` is ignored)."""
    out = [('backbone.conv1.weight', (32, 3, 3, 3), 'conv')] + _bn_shapes('backbone.bn1', 32) + \
        [('backbone.conv2.weight', (64, 32, 3, 3), 'conv')] + _bn_shapes('backbone.bn2', 64)
    plan, _ = block_plan(output_stride)
    for name, cin, cout, reps, stride, dil, swr, gf, last in plan:
        p = 'backbone.' + name
        if cout != cin or stride != 1:
            out += [(p + '.skip.weight', (cout, cin, 1, 1), 'conv')] + _bn_shapes(p + '.skipbn', cout)
        for i, e in enumerate(block_rep(cin, cout, reps, stride, dil, swr, gf, last)):
            if e[0] == 'sep':
                out += _sep_shapes('%s.rep.%d' % (p, i), e[1], e[2])
            elif e[0] == 'bn':
                out += _bn_shapes('%s.rep.%d' % (p, i), e[1])
    for i, (cin, cout) in zip((3, 4, 5), ((1024, 1536), (1536, 1536), (1536, 2048))):
        out += _sep_shapes('backbone.conv%d' % i, cin, cout) + _bn_shapes('backbone.bn%d' % i, cout)
    return out


def param_shapes(num_classes=21, output_stride=16, blocks=None):
    """DeepLabV3+ on Xception-65 in ``parameters()`` order: the backbone, then deeplabv3plus_oracle's head with
    decoder.reduce reading 128 channels."""
    head = [(n, (48, 128, 1, 1) if n == 'decoder.reduce.0.weight' else s, k) for n, s, k in D._head_shapes(num_classes)]
    return backbone_param_shapes(output_stride) + head


def separable(x, state, p, stride, dilation, training):
    """fixed_padding (dilation on every side) -> depthwise 3x3 -> BN -> pointwise 1x1."""
    x = F.pad(x, (dilation,) * 4)
    x = F.conv2d(x, state[p + '.conv1.weight'], stride=stride, dilation=dilation, groups=x.shape[1])
    x = O.batch_norm(x, state, p + '.bn', training)
    return F.conv2d(x, state[p + '.pointwise.weight'])


def block(x, state, p, spec, training):
    """The port's Block.forward: rep(inp) + skip(inp), where a block starting with a ReLU rectifies inp in place first,
    so its skip reads relu(x)."""
    cin, cout, reps, stride, dil, swr, gf, last = spec
    rep = block_rep(cin, cout, reps, stride, dil, swr, gf, last)
    if swr:
        x = F.relu(x)
    h = x
    for i, e in enumerate(rep):
        if e[0] == 'relu' and i > 0:
            h = F.relu(h)
        elif e[0] == 'sep':
            h = separable(h, state, '%s.rep.%d' % (p, i), e[3], e[4], training)
        elif e[0] == 'bn':
            h = O.batch_norm(h, state, '%s.rep.%d' % (p, i), training)
    if cout != cin or stride != 1:
        x = O.batch_norm(F.conv2d(x, state[p + '.skip.weight'], stride=stride), state, p + '.skipbn', training)
    return h + x


def backbone_forward(img, state, training, output_stride=16, blocks=None):
    """-> (low-level feature: block1's output after the ReLU, the 2048-channel output)."""
    x = F.relu(O.batch_norm(F.conv2d(img, state['backbone.conv1.weight'], stride=2, padding=1), state, 'backbone.bn1',
                            training))
    x = F.relu(O.batch_norm(F.conv2d(x, state['backbone.conv2.weight'], padding=1), state, 'backbone.bn2', training))
    plan, exit_dil = block_plan(output_stride)
    low = None
    for name, *spec in plan:
        x = block(x, state, 'backbone.' + name, spec, training)
        if name == 'block1':
            x = low = F.relu(x)
    x = F.relu(x)
    for i in (3, 4, 5):
        x = F.relu(O.batch_norm(separable(x, state, 'backbone.conv%d' % i, 1, exit_dil, training), state,
                                'backbone.bn%d' % i, training))
    return low, x


@contextlib.contextmanager
def xception():
    """Inside the block, ``deeplabv3plus_oracle`` (param_shapes, init, forward, MTOracle) describes and runs DeepLabV3+
    on Xception-65."""
    saved = D.param_shapes, D.backbone_forward
    D.param_shapes, D.backbone_forward = param_shapes, backbone_forward
    try:
        yield
    finally:
        D.param_shapes, D.backbone_forward = saved


def init(seed, num_classes=21, output_stride=16, cls_bias_std=0.0):
    """deeplabv3plus_oracle.init on this tree: every convolution ~ N(0, sqrt(2/(k*k*out_channels))), a depthwise one's
    out_channels being its input channels; BN gamma 1, beta 0."""
    with xception():
        return D.init(seed, num_classes, output_stride, None, cls_bias_std)


def forward(img, state, training=True, output_stride=16, blocks=None):
    """-> (logits at the input size, the 2048-channel latent)."""
    with xception():
        return D.forward(img, state, training, output_stride)


class MTOracle(D.MTOracle):
    """Mean Teacher (SupOnly with t_state=None) with DeepLabV3+ on Xception-65 as the task model."""

    def __init__(self, *a, **k):
        with xception():
            super().__init__(*a, **k)

    def step(self, *a, **k):
        with xception():
            return super().step(*a, **k)
