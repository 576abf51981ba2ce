"""SSL_S4L on the H100 kernels: plugin mirror of pixelssl/ssl_algorithm/ssl_s4l.py (rotation-based
self-supervised semi-supervised learning): same parser arguments, export function, ``_SSLBase`` methods, meter
names and checkpoint layout.

Per step (ssl_s4l.py:113-200): the batch is doubled with one rotated copy per sample (``pxl_s4l_rotate_batch``, one
launch per tensor instead of 2*bs slice assignments), the task model and the rotation classifier
(ssl_s4l.py:381-400: two 4x4/2 convolutions + BatchNorm + LeakyReLU(0.2), global average pool, Linear -> 4) run
forward, and three losses are summed: the task loss on the un-rotated labeled samples, ``rotated_sup_scale`` x the
task loss on their rotated copies and ``rotation_scale`` x the cross entropy of the predicted quarter turn."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..nn import func
from ..nn.arena import EngineParallel
from ..nn.modules import Conv2d, BatchNorm2d
from ..utils import logger, tool
from ..utils import REGRESSION, CLASSIFICATION
from . import ssl_base


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--rotated-sup-scale', type=float, default=-1, help='ssls4l - task-supervised coefficient for rotated labeled data')
    parser.add_argument('--rotation-scale', type=float, default=-1, help='ssls4l - rotation-based self-supervised coefficient')


def ssl_s4l(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    if not len(model_dict) == len(optimizer_dict) == len(lrer_dict) == len(criterion_dict) == 1:
        logger.log_err('The len(element_dict) of SSL_S4L should be 1\n')
    elif list(model_dict.keys())[0] != 'model':
        logger.log_err('In SSL_S4L, the key of element_dict should be \'model\',\n'
                       'but \'{0}\' is given\n'.format(model_dict.keys()))
    algorithm = SSLS4L(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']], [criterion_dict['model']], task_func)
    return algorithm


def _lanes(c):
    return (c + 31) // 32 * 32


class _LaneBatchNorm(nn.Module):
    """``nn.BatchNorm2d(C)`` (ssl_s4l.py:385,387 - the plain torch layer, not SyncBN: per-replica statistics,
    ``num_batches_tracked`` counts) on an NHWC tensor that carries C real channels in ``lanes`` >= C lanes (extra
    lanes hold zeros and stay zero).  Parameters / buffers keep the reference shapes [C]; the padded vectors the
    kernels read are tiny torch ops."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1):
        super().__init__()
        self.num_features, self.eps, self.momentum = num_features, eps, momentum
        self.weight = nn.Parameter(torch.ones(num_features))
        self.bias = nn.Parameter(torch.zeros(num_features))
        self.register_buffer('running_mean', torch.zeros(num_features))
        self.register_buffer('running_var', torch.ones(num_features))
        self.register_buffer('num_batches_tracked', torch.tensor(0, dtype=torch.long))

    def forward(self, x):
        c, lanes = self.num_features, x.shape[1]
        pad = lanes - c
        gamma = F.pad(self.weight, (0, pad), value=1.0)
        beta = F.pad(self.bias, (0, pad))
        rm = F.pad(self.running_mean, (0, pad))
        rv = F.pad(self.running_var, (0, pad), value=1.0)
        y = ops.bn_act(ops.as_cl(x), gamma, beta, rm, rv, training=self.training, momentum=self.momentum, eps=self.eps)
        if self.training:
            with torch.no_grad():
                self.running_mean.copy_(rm[:c])
                self.running_var.copy_(rv[:c])
                self.num_batches_tracked += 1
        return y


class RotationClassifer(nn.Module):
    """ssl_s4l.py:381-400 (spelling of the class name kept): same parameter tree, so ``state_dict`` keys and shapes
    equal the reference's.  Input: the task prediction, planar [n, C, H, W]."""

    def __init__(self, in_channels):
        super().__init__()
        c = in_channels
        self.in_channels = c
        self.conv1 = Conv2d(c, c, 4, stride=2, padding=1, out_lanes=_lanes(c))
        self.bn1 = _LaneBatchNorm(c)
        self.conv2 = Conv2d(c, c * 2, 4, stride=2, padding=1, out_lanes=_lanes(2 * c))
        self.bn2 = _LaneBatchNorm(c * 2)
        self.classifier = nn.Linear(c * 2, 4)

    def forward(self, task_pred):
        n, c = task_pred.shape[0], self.in_channels
        x = ops.planar_to_nhwc(task_pred, ldc=_lanes(c))                       # [n, lanes, H, W] channels_last
        x = ops.leaky_relu(self.bn1(self.conv1(x)), 0.2)
        x = ops.leaky_relu(self.bn2(self.conv2(x)), 0.2)
        x = ops.adaptive_avg_pool(x, 1)                                        # nn.AdaptiveAvgPool2d((1, 1))
        # nn.Linear(2c, 4) as a 1x1 convolution on the pooled [n, lanes, 1, 1] tensor (weight padded with zero lanes)
        w = F.pad(self.classifier.weight, (0, x.shape[1] - 2 * c)).view(4, x.shape[1], 1, 1).contiguous(memory_format=ops.CL)
        return ops.conv2d(x, w, self.classifier.bias).reshape(n, 4)


class WrappedS4LModel(nn.Module):
    """ssl_s4l.py:403-438."""

    def __init__(self, args, task_model, rotation_classifier):
        super().__init__()
        self.args = args
        self.task_model = task_model
        self.rotation_classifier = rotation_classifier
        self.param_groups = self.task_model.param_groups + \
            [{'params': list(self.rotation_classifier.parameters()), 'lr': self.args.lr}]

    def forward(self, inp):
        resulter, debugger = {}, {}
        t_resulter, _ = self.task_model.forward(inp)
        if 'pred' not in t_resulter or 'activated_pred' not in t_resulter:
            logger.log_err('In SSL_S4L, the \'resulter\' dict returned by the task model should contain the following keys:\n'
                           '   (1) \'pred\'\t=>\tunactivated task predictions\n'
                           '   (2) \'activated_pred\'\t=>\tactivated task predictions\n')
        if 'ssls4l_rc_inp' not in t_resulter:
            logger.log_err('In SSL_S4L, the \'resulter\' dict returned by the task model should contain the key:\n'
                           '    \'ssls4l_rc_inp\'\t=>\tinputs of the rotation classifier (a 4-dim tensor)\n')
        rc_inp = tool.dict_value(t_resulter, 'ssls4l_rc_inp')
        resulter['pred'] = tool.dict_value(t_resulter, 'pred')
        resulter['activated_pred'] = tool.dict_value(t_resulter, 'activated_pred')
        resulter['rotation'] = self.rotation_classifier.forward(rc_inp)
        return resulter, debugger


class SSLS4L(ssl_base._SSLBase):
    NAME = 'ssl_s4l'
    SUPPORTED_TASK_TYPES = [REGRESSION, CLASSIFICATION]
    LOG_LINES = ('  task-{3}\t=>\t'
                 'unrotated-task-loss: {meters[unrotated_task_loss]:.6f}\t'
                 'rotated-task-loss: {meters[rotated_task_loss]:.6f}\n'
                 '  rotation-{3}\t=>\t'
                 'rotation-loss: {meters[rotation_loss]:.6f}\t'
                 'rotation-acc: {meters[rotation_acc]:.6f}\n')

    def __init__(self, args):
        super().__init__(args)
        self.task_model = self.rotation_classifier = None
        self.model = self.optimizer = self.lrer = self.criterion = None
        self._first_batch = True             # _inp_warn looks at the first batch of every epoch
        if self.args.rotation_scale < 0:
            logger.log_err('The argument - rotation_scale - is not set (or invalid)\n'
                           'Please set - rotation_scale >= 0 - for training\n')
        if self.args.rotated_sup_scale < 0:
            logger.log_err('The argument - rotated_sup_scale - is not set (or invalid)\n'
                           'Please set - rotated_sup_scale >= 0 - for training\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.task_model = model_funcs[0](args=self.args)
        self.rotation_classifier = RotationClassifer(self.task_func.ssls4l_rc_in_channels())
        wrapped = WrappedS4LModel(self.args, self.task_model, self.rotation_classifier)
        self.model = EngineParallel(wrapped).cuda()          # where the reference has nn.DataParallel (ssl_s4l.py:82)
        self.models = {'model': self.model}
        self.optimizer = optimizer_funcs[0](wrapped.param_groups)
        self.optimizers = {'optimizer': self.optimizer}
        self.lrer = lrer_funcs[0](self.optimizer)
        self.lrers = {'lrer': self.lrer}
        self.criterion = criterion_funcs[0](self.args)
        self.rotation_criterion = _rotation_cross_entropy
        self.criterions = {'criterion': self.criterion, 'rotation_criterion': self.rotation_criterion}
        # the batch size is doubled in S4L since it creates an extra rotated sample for each sample (ssl_s4l.py:101-104)
        self.args.batch_size *= 2
        self.args.labeled_batch_size *= 2
        self.args.unlabeled_batch_size *= 2
        logger.log_info('In SSL_S4L algorithm, batch size are doubled: \n'
                        '  Total labeled batch size: {1}\n'
                        '  Total unlabeled batch size: {2}\n'
                        .format(self.args.lr, self.args.labeled_batch_size, self.args.unlabeled_batch_size))
        self._algorithm_warn()

    # ------------------------------------------------------------------------------------------
    def train_step(self, inp, gt, cur_step, total_steps):
        """Loop body of ssl_s4l.py:120-175 on (host or device) tuples ``inp`` / ``gt``."""
        if self._first_batch:
            self._first_batch = False
            if len(gt) > 1:
                self._inp_warn()
        original_lbs = int(self.args.labeled_batch_size / 2)
        original_bs = int(self.args.batch_size / 2)
        inp, gt = self._batch_prehandle(inp, gt, True)
        arena = self.model.arena
        arena.zero_grad()
        resulter, _ = self.model.forward(inp)
        pred = tool.dict_value(resulter, 'pred')
        pred_rotation = tool.dict_value(resulter, 'rotation')
        l_pred = func.split_tensor_tuple(pred, 0, original_lbs)
        l_gt = func.split_tensor_tuple(gt, 0, original_lbs)
        l_inp = func.split_tensor_tuple(inp, 0, original_lbs)
        unrotated_task_loss = torch.mean(self.criterion.forward(l_pred, l_gt[:-1], l_inp))
        self.meters.update('unrotated_task_loss', unrotated_task_loss.data)
        l_rotated_pred = func.split_tensor_tuple(pred, original_bs, original_bs + original_lbs)
        l_rotated_gt = func.split_tensor_tuple(gt, original_bs, original_bs + original_lbs)
        l_rotated_inp = func.split_tensor_tuple(inp, original_bs, original_bs + original_lbs)
        rotated_task_loss = self.args.rotated_sup_scale * torch.mean(
            self.criterion.forward(l_rotated_pred, l_rotated_gt[:-1], l_rotated_inp))
        self.meters.update('rotated_task_loss', rotated_task_loss.data)
        task_loss = unrotated_task_loss + rotated_task_loss
        rotation_loss = self.args.rotation_scale * torch.mean(self.rotation_criterion(pred_rotation, gt[-1]))
        self.meters.update('rotation_loss', rotation_loss.data)
        loss = task_loss + rotation_loss
        loss.backward()
        arena.all_reduce_grads()
        arena.sgd_step(self.optimizer)
        # accuracy of the rotation classifier (ssl_s4l.py:169-173); tiny device-side ops, read lazily by the logger
        angle_idx = pred_rotation.detach().argmax(dim=1)
        rotation_acc = (angle_idx == gt[-1]).float().sum(0, keepdim=True).mul_(100.0 / self.args.batch_size)
        self.meters.update('rotation_acc', rotation_acc[0])

    def _train(self, data_loader, epoch):
        self._first_batch = True
        super()._train(data_loader, epoch)

    def validate_step(self, inp, gt):
        inp, gt = self._batch_prehandle(inp, gt, False)
        resulter, _ = self.model.forward(inp)
        pred = tool.dict_value(resulter, 'pred')
        pred_rotation = tool.dict_value(resulter, 'rotation')
        self.meters.update('task_loss', torch.mean(self.criterion.forward(pred, gt[:-1], inp)).data)
        rotation_loss = self.args.rotation_scale * torch.mean(self.rotation_criterion(pred_rotation, gt[-1]))
        self.meters.update('rotation_loss', rotation_loss.data)
        self._metrics(resulter, gt[:-1], inp, 'task')

    # ------------------------------------------------------------------------------------------
    def _batch_prehandle(self, inp, gt, is_train):
        """ssl_s4l.py:296-350.  The quarter turns come from ``np.random.randint(1, 4, bs)`` exactly like the
        reference (drawn in validation too, so the host RNG stream stays aligned)."""
        bs = inp[0].shape[0]
        rotation_angles = np.random.randint(low=1, high=4, size=bs)
        inp = ssl_base.to_device(inp)
        gt = ssl_base.to_device(gt)
        dev = inp[0].device
        if is_train:
            angles = torch.from_numpy(rotation_angles.astype(np.int32)).to(dev, non_blocking=True)
            inp = tuple(_rotate_batch(i, angles) for i in inp)
            gt = tuple(_rotate_batch(g, angles) for g in gt)
            rotation_gt = torch.cat((torch.zeros(bs, dtype=torch.long, device=dev), angles.long()))
        else:
            rotation_gt = torch.zeros(bs, dtype=torch.long, device=dev)
        return inp, tuple(gt) + (rotation_gt,)

    def _inp_warn(self):
        logger.log_warn('More than one ground truth of the task model is given in SSL_S4L\n'
                        'You try to train the task model with more than one (pred & gt) pairs\n'
                        'Please make sure that:\n'
                        '  (1) The prediction tuple has the same size as the ground truth tuple\n'
                        '  (2) The elements with the same index in the two tuples are corresponding\n'
                        '  (3) All elements in the ground truth tuple should be 4-dim tensors since S4L\n'
                        '      will rotate them to match the rotated inputs\n')

    def _algorithm_warn(self):
        logger.log_warn('This SSL_S4L algorithm reproduces the SSL algorithm from the paper:\n'
                        '  \'S4L: Self-Supervised Semi-Supervised Learning\'\n'
                        'The main differences between this implementation and the original paper are:\n'
                        '  (1) This is an implementation for pixel-wise vision tasks\n'
                        '  (2) This implementation only supports the 4-angle (0, 90, 180, 270) rotation-based self-supervised pretext task\n')


def _rotate_batch(t, angles):
    """[bs,C,H,W] -> [2*bs,C,H,W]: the batch followed by its rotated copies (one launch)."""
    t = t.contiguous()
    bs, c, h, w = t.shape
    out = torch.empty((2 * bs, c, h, w), dtype=torch.float32, device=t.device)
    ops.call('pxl_s4l_rotate_batch', ops._p(t), ops._p(out), ops._p(angles), bs, c, h, w, 1, ops._stream())
    return out


def _rotation_cross_entropy(pred_rotation, rotation_gt):
    """``nn.CrossEntropyLoss()`` (ssl_s4l.py:97) on [n, 4] logits: the 2-D criterion kernel with a 1x1 map per sample
    -> [n] per-sample losses (their mean is the reference's scalar)."""
    n = pred_rotation.shape[0]
    return ops.cross_entropy2d(pred_rotation.reshape(n, 4, 1, 1), rotation_gt.float().reshape(n, 1, 1, 1), ignore_index=255)
