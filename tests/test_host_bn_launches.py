"""Every library call of the BatchNorm nodes, forward and backward, in the order they are issued (CPU only: the calls
are recorded, not made): bn_act in train and eval mode, the fused conv -> BN units of the fp16-pair path with their
output forms and residual-gradient stash roles, the depthwise -> BN pair unit, and the cross-process reduction
through a peer exchange or torch.distributed.  Arguments print as tools/launch_trace.py prints them (pointers as
null / ptr, scalars by value).  Also checks which outputs carry an fp16 pair and which are pair-only carriers."""
import types

import pytest
import torch
import torch.distributed as dist

from pixelssl_b200 import ops
from pixelssl_b200.nn.modules import BatchNorm2d, Conv2d
from tools.launch_trace import fmt

N, H, W, C = 1, 4, 4, 64


def _py(v):
    if isinstance(v, tuple):
        return '(%s)' % ', '.join(_py(a) for a in v)
    if v is None or isinstance(v, torch.Tensor):
        return 'ptr' if v is not None else 'null'
    return repr(v)


class _FakePeer:
    def __init__(self, lines):
        self.lines = lines

    def allreduce_bn(self, sums, finalize=None, param_grads=None):
        self.lines.append('peer.allreduce_bn(%s, %d, finalize=%s, param_grads=%s)'
                          % (_py(sums), sums.numel(), _py(finalize), _py(param_grads)))
        return sums


@pytest.fixture
def lines(monkeypatch):
    """The formatted library calls of the test; nothing reaches the library or a process group."""
    rec = []

    def fake_call(name, *args):
        rec.append(fmt(name, args))
        return 0

    monkeypatch.setattr(ops, 'call', fake_call)
    monkeypatch.setattr(ops, '_stream', lambda: 0)
    monkeypatch.setattr(ops, '_chk', lambda *a, **k: None)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    monkeypatch.setattr(dist, 'all_reduce', lambda t, group=None: rec.append('dist.all_reduce(%d)' % t.numel()))
    ops.new_step()
    return rec


def _act():
    return torch.zeros((N, C, H, W), requires_grad=True).contiguous(memory_format=ops.CL)


def _bn(arena=False):
    """arena: the parameter gradients exist before the backward, as in a training step's gradient arena."""
    bn = BatchNorm2d(C)
    if arena:
        bn.weight.grad, bn.bias.grad = torch.zeros(C), torch.zeros(C)
    return bn


def _backward(out):
    out.backward(torch.ones_like(out))


# ---- bn_act -------------------------------------------------------------------------------------------------------

BN_TRAIN = [(relu, res, sums, arena) for relu in (False, True) for res in (False, True) for sums in (False, True)
            for arena in (False, True)]


def _bn_train_id(relu, res, sums, arena):
    return 'relu%d-res%d-convsums%d-arena%d' % (relu, res, sums, arena)


@pytest.mark.parametrize('relu,res,sums,arena', BN_TRAIN, ids=[_bn_train_id(*c) for c in BN_TRAIN])
def test_bn_act_train(lines, relu, res, sums, arena):
    bn, x = _bn(arena=arena), _act()
    if sums:
        x._pxl_bn_sums = torch.zeros(2 * C, dtype=torch.float64)
    out = bn(x, relu=relu, residual=_act() if res else None)
    _backward(out)
    assert lines == EXPECTED['bn_train-' + _bn_train_id(relu, res, sums, arena)]


@pytest.mark.parametrize('relu,res', [(False, False), (True, True)])
def test_bn_act_eval_in_grad_graph(lines, relu, res):
    bn = _bn().eval()
    out = bn(_act(), relu=relu, residual=_act() if res else None)
    _backward(out)
    assert lines == EXPECTED['bn_eval-relu%d-res%d' % (relu, res)]


@pytest.mark.parametrize('exchange', ['peer', 'nccl'])
@pytest.mark.parametrize('arena', [False, True])
def test_bn_act_group(lines, monkeypatch, exchange, arena):
    bn, group = _bn(arena=arena), object()
    bn.sync_group = group
    if exchange == 'peer':
        monkeypatch.setitem(ops._peer_exchanges, id(group), _FakePeer(lines))
    out = bn(_act(), relu=True, residual=_act())
    _backward(out)
    assert lines == EXPECTED['bn_group-%s-arena%d' % (exchange, arena)]


# ---- conv_bn_act ----------------------------------------------------------------------------------------------------

def _unit(arena=False):
    return Conv2d(C, C, 1, bias=False), _bn(arena=arena)


def _pair_state(t):
    """(has lo plane or None without a pair, carrier flag)."""
    h = ops._step_get(t, '_pxl_h16')
    if h is not None:
        assert isinstance(h, ops.H16) and h.scale == ops.H16_ACT_SCALE and h.slot is None and h.numel == t.numel()
    return (None if h is None else h.has_lo), ops.is_carrier(t)


@pytest.mark.parametrize('precision', ['f16x3', 'f16'])
@pytest.mark.parametrize('out_mode', ['pair', 'both', 'fp32'])
def test_conv_bn_act(lines, monkeypatch, precision, out_mode):
    """relu(bn(conv(x)) + residual) in each output form."""
    monkeypatch.setattr(ops, '_conv_precision', ops.PRECISION[precision])
    conv, bn = _unit()
    out = ops.conv_bn_act(_act(), conv, bn, relu=True, residual=_act(), out_mode=out_mode)
    lo = precision == 'f16x3'
    assert _pair_state(out) == {'pair': (lo, True), 'both': (lo, False), 'fp32': (None, False)}[out_mode]
    _backward(out)
    assert lines == EXPECTED['conv_bn_act-%s-%s' % (precision, out_mode)]


@pytest.mark.parametrize('precision', ['f16x3', 'f16'])
@pytest.mark.parametrize('block', ['identity', 'downsample'])
def test_conv_bn_act_stash(lines, monkeypatch, precision, block):
    """A bottleneck's units as resnet.Bottleneck chains them: 'take' on the first unit, 'give' on the last of an
    identity block, 'give_dx' on the downsample unit; the BN parameter gradients go into a gradient arena."""
    monkeypatch.setattr(ops, '_conv_precision', ops.PRECISION[precision])
    x, key = _act(), object()
    (c1, b1), (c3, b3), (cd, bd) = _unit(True), _unit(True), _unit(True)
    out = ops.conv_bn_act(x, c1, b1, relu=True, out_mode='pair', stash_key=key, stash_role='take')
    if block == 'identity':
        out = ops.conv_bn_act(out, c3, b3, relu=True, residual=x, out_mode='both', stash_key=key, stash_role='give')
    else:
        residual = ops.conv_bn_act(x, cd, bd, relu=False, out_mode='fp32', stash_key=key, stash_role='give_dx')
        out = ops.conv_bn_act(out, c3, b3, relu=True, residual=residual, out_mode='both')
    _backward(out)
    assert not ops._residual_stash
    assert lines == EXPECTED['stash-%s-%s' % (precision, block)]


# ---- depthwise_bn_pair ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('precision', ['f16x3', 'f16'])
def test_depthwise_bn_pair(lines, monkeypatch, precision):
    monkeypatch.setattr(ops, '_conv_precision', ops.PRECISION[precision])
    weight = torch.zeros((48, 1, 3, 3), requires_grad=True)
    bn = types.SimpleNamespace(weight=torch.ones(C, requires_grad=True), bias=torch.zeros(C, requires_grad=True),
                               running_mean=torch.zeros(C), running_var=torch.ones(C), momentum=0.1, eps=1e-5,
                               sync_group=None, multi_replica_formula=False)
    out = ops.depthwise_bn_pair(_act(), weight, bn, stride=1, dilation=2)
    assert _pair_state(out) == (precision == 'f16x3', True)
    _backward(out)
    assert lines == EXPECTED['depthwise_bn_pair-%s' % precision]


EXPECTED = {
    'bn_train-relu0-res0-convsums0-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res0-convsums0-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, ptr, ptr, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res0-convsums1-arena0': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res0-convsums1-arena1': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, ptr, ptr, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res1-convsums0-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res1-convsums0-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, ptr, 16, 64, ptr, ptr, ptr, ptr, null, null, '
        'null, 0, null, null)',
    ],
    'bn_train-relu0-res1-convsums1-arena0': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu0-res1-convsums1-arena1': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 0, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, ptr, 16, 64, ptr, ptr, ptr, ptr, null, null, '
        'null, 0, null, null)',
    ],
    'bn_train-relu1-res0-convsums0-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res0-convsums0-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, null, 16, 64, ptr, ptr, ptr, ptr, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res0-convsums1-arena0': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res0-convsums1-arena1': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, null, 16, 64, ptr, ptr, ptr, ptr, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res1-convsums0-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res1-convsums0-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, ptr, 16, 64, ptr, ptr, ptr, ptr, null, null, '
        'null, 0, null, null)',
    ],
    'bn_train-relu1-res1-convsums1-arena0': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_train-relu1-res1-convsums1-arena1': [
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, ptr, 16, 64, ptr, ptr, ptr, ptr, null, null, '
        'null, 0, null, null)',
    ],
    'bn_eval-relu0-res0': [
        'pxl_bn_eval_coeffs(64, ptr, ptr, ptr, ptr, 1e-05, ptr, ptr, null)',
        'pxl_bn_apply(ptr, ptr, ptr, null, 0, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_eval-relu1-res1': [
        'pxl_bn_eval_coeffs(64, ptr, ptr, ptr, ptr, 1e-05, ptr, ptr, null)',
        'pxl_bn_apply(ptr, ptr, ptr, ptr, 1, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 16.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_group-peer-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'peer.allreduce_bn(ptr, 128, finalize=(32.0, 64, ptr, ptr, ptr, ptr, 0.1, 1e-05, 1, ptr, ptr, ptr, ptr), '
        'param_grads=null)',
        'pxl_bn_apply(ptr, ptr, ptr, ptr, 1, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'peer.allreduce_bn(ptr, 128, finalize=null, param_grads=null)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 32.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_group-nccl-arena0': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'dist.all_reduce(128)',
        'pxl_bn_finalize(ptr, 32.0, 64, ptr, ptr, ptr, ptr, 0.1, 1e-05, 1, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_apply(ptr, ptr, ptr, ptr, 1, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'dist.all_reduce(128)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 32.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_group-peer-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'peer.allreduce_bn(ptr, 128, finalize=(32.0, 64, ptr, ptr, ptr, ptr, 0.1, 1e-05, 1, ptr, ptr, ptr, ptr), '
        'param_grads=null)',
        'pxl_bn_apply(ptr, ptr, ptr, ptr, 1, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'peer.allreduce_bn(ptr, 128, finalize=null, param_grads=(ptr, ptr))',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 32.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'bn_group-nccl-arena1': [
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'dist.all_reduce(128)',
        'pxl_bn_finalize(ptr, 32.0, 64, ptr, ptr, ptr, ptr, 0.1, 1e-05, 1, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_apply(ptr, ptr, ptr, ptr, 1, ptr, 16, 64, null, null, 1.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, ptr, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'dist.all_reduce(128)',
        'pxl_bn_bwd_dx(ptr, ptr, ptr, ptr, ptr, ptr, ptr, 32.0, 1, ptr, ptr, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
    ],
    'conv_bn_act-f16x3-pair': [
        'pxl_h16_split(ptr, ptr, ptr, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, null, '
        '16, 64, ptr, ptr, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'ptr, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
    ],
    'conv_bn_act-f16-pair': [
        'pxl_h16_split(ptr, ptr, null, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, null, '
        '16, 64, ptr, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'null, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
    ],
    'conv_bn_act-f16x3-both': [
        'pxl_h16_split(ptr, ptr, ptr, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, ptr, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'ptr, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
    ],
    'conv_bn_act-f16-both': [
        'pxl_h16_split(ptr, ptr, null, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'null, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
    ],
    'conv_bn_act-f16x3-fp32': [
        'pxl_h16_split(ptr, ptr, ptr, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'ptr, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
    ],
    'conv_bn_act-f16-fp32': [
        'pxl_h16_split(ptr, ptr, null, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, null, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, null, null, ptr, '
        'null, ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
    ],
    'stash-f16x3-identity': [
        'pxl_h16_split(ptr, ptr, ptr, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, null, '
        '16, 64, ptr, ptr, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, ptr, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, ptr, ptr, ptr, ptr, '
        'ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, ptr, '
        'ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=1}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
    ],
    'stash-f16-identity': [
        'pxl_h16_split(ptr, ptr, null, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, null, '
        '16, 64, ptr, null, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, ptr, ptr, ptr, null, '
        'ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, '
        'null, ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=1}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
    ],
    'stash-f16x3-downsample': [
        'pxl_h16_split(ptr, ptr, ptr, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, null, '
        '16, 64, ptr, ptr, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, ptr, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, ptr, ptr, ptr, ptr, '
        'ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, ptr, '
        'ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, ptr, '
        'ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, ptr, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=1}, ptr, ptr, ptr, ptr, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=3}, [0, '
        '0], ptr, ptr, ptr, ptr, ptr, 0.0625, ptr, null)',
    ],
    'stash-f16-downsample': [
        'pxl_h16_split(ptr, ptr, null, 1024, 16.0, null, 14, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 1, null, '
        '16, 64, ptr, null, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, ptr, '
        '16, 64, null, null, 16.0, null, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=ptr '
        'out_scale=0.000244140625 out_scale_dev=null out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, ptr, 1, ptr, '
        '16, 64, ptr, null, 16.0, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, ptr, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, ptr, 16, 64, ptr, ptr, ptr, ptr, ptr, null, '
        'ptr, 12, ptr, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, '
        'null, ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=0}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 1, 16, 64, ptr, ptr, ptr, ptr, null, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 1, null, null, 16, 64, ptr, ptr, ptr, ptr, ptr, '
        'null, ptr, 12, null, null)',
        'pxl_conv_transpose_weights(ptr, ptr, 64, 1, 64, null)',
        'pxl_h16_split(ptr, ptr, null, 4096, 256.0, null, 14, null)',
        'pxl_conv_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, 0], '
        '{w_ntaps=0 widx_host=null out_mul=0 out_offy=0 out_offx=0 out_H=0 out_W=0 bn_stats=null out_scale=0.00390625 '
        'out_scale_dev=ptr out_accumulate=1}, ptr, null, ptr, null, null, ptr, null)',
        'pxl_conv_wgrad_h16_launch({N=1 H=4 W=4 Cin=64 OH=4 OW=4 Cout=64 ldo=64 mul=1 div=1 ntaps=1 precision=4}, [0, '
        '0], ptr, null, ptr, null, ptr, 0.0625, ptr, null)',
    ],
    'depthwise_bn_pair-f16x3': [
        'pxl_dw_conv_fwd(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, null)',
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, null, '
        '16, 64, ptr, ptr, 16.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
        'pxl_dw_conv_dgrad(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, null)',
        'pxl_dw_conv_wgrad(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, 0, null)',
    ],
    'depthwise_bn_pair-f16': [
        'pxl_dw_conv_fwd(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, null)',
        'pxl_bn_stats(ptr, 16, 64, ptr, null)',
        'pxl_bn_finalize_apply(ptr, ptr, 16.0, ptr, ptr, ptr, ptr, 0.1, 1e-05, 0, ptr, ptr, ptr, ptr, null, 0, null, '
        '16, 64, ptr, null, 16.0, null, null)',
        'pxl_bn_bwd_reduce(ptr, null, ptr, ptr, ptr, 0, 16, 64, ptr, ptr, ptr, null, null, null)',
        'pxl_bn_bwd_params(ptr, 64, ptr, ptr, 0, null)',
        'pxl_bn_bwd_dx(ptr, null, ptr, ptr, ptr, ptr, ptr, 16.0, 0, ptr, null, 16, 64, ptr, ptr, null, null, null, '
        'null, null, 0, null, null)',
        'pxl_dw_conv_dgrad(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, null)',
        'pxl_dw_conv_wgrad(ptr, ptr, ptr, 1, 4, 4, 48, 64, 4, 4, 1, 2, 0, null)',
    ],
}
