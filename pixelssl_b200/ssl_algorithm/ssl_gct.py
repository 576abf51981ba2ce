"""Guided Collaborative Training (pixelssl/ssl_algorithm/ssl_gct.py:176-298, 401-480) on the H100 kernels.

Per step: (0) no-grad forwards of the two task models; flaw detector (FD) on both (graph kept for
step 2); handled flaw maps (clamp -> separable Gaussian blur -> clip -> min-max) and the dynamic-
consistency pseudo ground truth; (1) per task model: forward, FD (frozen), CE on the labeled rows,
flaw-correction loss both_bad * flawmap^2, dynamic-consistency MSE(softmax, dc_gt), backward, SGD;
(2) FD ground truth on the labeled rows (|onehot - softmax| -> blur -> nu x (dilate -> blur) ->
min-max, the 179x179 depthwise convolutions of the reference run as separable 1-D passes),
MSE, backward through the step-0 FD graphs, Adam(0.9, 0.99), PolynomialLR."""
import torch
import torch.nn as nn
import torch.optim as optim

from .. import ops
from ..utils import REGRESSION, CLASSIFICATION, logger, tool
from ..nn import func
from ..nn.lrer import PolynomialLR
from ..nn.modules import Conv2d
from . import ssl_base

MODE_GCT, MODE_FC, MODE_DC = 'gct', 'fc', 'dc'


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--ssl-mode', type=str, default=MODE_GCT, choices=[MODE_GCT, MODE_DC, MODE_FC])
    parser.add_argument('--fc-ssl-scale', type=float, default=-1.0)
    parser.add_argument('--dc-ssl-scale', type=float, default=-1.0)
    parser.add_argument('--dc-threshold', type=float, default=-1.0)
    parser.add_argument('--dc-rampup-epochs', type=int, default=-1)
    parser.add_argument('--fd-lr', type=float, default=1e-4)
    parser.add_argument('--fd-scale', type=float, default=1.0)
    parser.add_argument('--mu', type=float, default=-1.0)
    parser.add_argument('--nu', type=int, default=-1)


def ssl_gct(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    pick = ssl_base.pair_picker(SSLGCT.NAME, model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLGCT(args)
    algorithm.build(pick(model_dict), pick(optimizer_dict), pick(lrer_dict), pick(criterion_dict), task_func)
    return algorithm


class IBNorm(nn.Module):
    """ssl_gct.py:588-607; parameter names follow the reference (``bnorm.weight`` ...)."""

    def __init__(self, num_features, split=0.5):
        super().__init__()
        self.num_features = num_features
        self.num_BN = int(num_features * split + 0.5)
        self.bnorm = nn.Module()
        self.bnorm.weight = nn.Parameter(torch.ones(self.num_BN))
        self.bnorm.bias = nn.Parameter(torch.zeros(self.num_BN))
        self.bnorm.register_buffer('running_mean', torch.zeros(self.num_BN))
        self.bnorm.register_buffer('running_var', torch.ones(self.num_BN))
        self.bnorm.register_buffer('num_batches_tracked', torch.tensor(0, dtype=torch.long))
        self.sync_group = None

    def forward(self, x):
        if self.training:
            self.bnorm.num_batches_tracked += 1
        return ops.ibnorm(x, self.bnorm.weight, self.bnorm.bias, self.bnorm.running_mean, self.bnorm.running_var,
                          training=self.training, group=self.sync_group)


class FlawDetector(nn.Module):
    """ssl_gct.py:539-585: cat(image, softmax) -> 7 x [conv 4x4 (stride 2/2/1/2/1/2/1) + IBNorm +
    LeakyReLU(0.2)] -> conv 4x4/2 -> bilinear (align_corners) to the input size; un-activated."""
    ndf = 64

    def __init__(self, in_channels):
        super().__init__()
        n = self.ndf
        spec = [('conv1', 'ibn1', in_channels, n, 2), ('conv2', 'ibn2', n, n * 2, 2), ('conv2_1', 'ibn2_1', n * 2, n * 2, 1),
                ('conv3', 'ibn3', n * 2, n * 4, 2), ('conv3_1', 'ibn3_1', n * 4, n * 4, 1), ('conv4', 'ibn4', n * 4, n * 8, 2),
                ('conv4_1', 'ibn4_1', n * 8, n * 8, 1)]
        self._order = []
        for cname, iname, cin, cout, stride in spec:
            setattr(self, cname, Conv2d(cin, cout, 4, stride=stride, padding=1))
            setattr(self, iname, IBNorm(cout))
            self._order.append((cname, iname))
        self.classifier = Conv2d(n * 8, 1, 4, stride=2, padding=1)

    def forward(self, task_inp, task_pred):
        resulter, debugger = {}, {}
        x = ops.cat_planar_to_nhwc(list(task_inp) + [task_pred])
        for cname, iname in self._order:
            x = ops.leaky_relu(getattr(self, iname)(getattr(self, cname)(x)), 0.2)
        x = self.classifier(x)
        resulter['flawmap'] = ops.bilinear(x, task_pred.shape[2:], align_corners=True, channels=1, nhwc=True)
        return resulter, debugger


class SSLGCT(ssl_base._SSLBase):
    NAME = 'ssl_gct'
    SUPPORTED_TASK_TYPES = [REGRESSION, CLASSIFICATION]
    RAMPUP_EPOCHS = 'dc_rampup_epochs'
    LOG_LINES = ('  l-{3}\t=>\tl-task-loss: {meters[l_task_loss]:.6f}\tl-dc-loss: {meters[l_dc_loss]:.6f}\t'
                 'l-fc-loss: {meters[l_fc_loss]:.6f}\n'
                 '  r-{3}\t=>\tr-task-loss: {meters[r_task_loss]:.6f}\tr-dc-loss: {meters[r_dc_loss]:.6f}\t'
                 'r-fc-loss: {meters[r_fc_loss]:.6f}\n'
                 '  fd\t=>\tl-fd-loss: {meters[l_fd_loss]:.6f}\tr-fd-loss: {meters[r_fd_loss]:.6f}\n')
    ITER_LRERS = ('fd_lrer',)
    VALIDATION_IDS = ('l', 'r')

    def __init__(self, args):
        super().__init__(args)
        self.l_model = self.r_model = self.fd_model = None
        self.args.fd_lr *= self.args.gpus                 # ssl_gct.py:107
        a = self.args
        if a.unlabeled_batch_size > 0:
            if a.ssl_mode in (MODE_GCT, MODE_FC) and a.fc_ssl_scale < 0:
                logger.log_err('The argument - fc_ssl_scale - is not set (or invalid)\n')
            if a.ssl_mode in (MODE_GCT, MODE_DC):
                if a.dc_rampup_epochs < 0 or a.dc_ssl_scale < 0 or a.dc_threshold < 0 or a.mu < 0 or a.nu < 0:
                    logger.log_err('The dynamic consistency constraint needs dc_rampup_epochs, dc_ssl_scale, '
                                   'dc_threshold, mu and nu to be set\n')
        if a.im_size is None:
            logger.log_err('SSL_GCT needs - im_size - (blur kernel sizes derive from it)\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.l_model = func.create_model(model_funcs[0], 'l_model', args=self.args)
        self.r_model = func.create_model(model_funcs[1], 'r_model', args=self.args)
        self.fd_model = func.create_model(FlawDetector, 'fd_model', in_channels=self.args.num_classes + 3)
        self.models = {'l_model': self.l_model, 'r_model': self.r_model, 'fd_model': self.fd_model}
        self.l_optimizer = optimizer_funcs[0](self.l_model.module.param_groups)
        self.r_optimizer = optimizer_funcs[1](self.r_model.module.param_groups)
        self.fd_optimizer = optim.Adam([p for p in self.fd_model.parameters() if p.requires_grad],
                                       lr=self.args.fd_lr, betas=(0.9, 0.99))
        self.optimizers = {'l_optimizer': self.l_optimizer, 'r_optimizer': self.r_optimizer,
                           'fd_optimizer': self.fd_optimizer}
        self.l_lrer = lrer_funcs[0](self.l_optimizer)
        self.r_lrer = lrer_funcs[1](self.r_optimizer)
        self.fd_lrer = PolynomialLR(self.fd_optimizer, self.args.epochs, self.args.iters_per_epoch, power=0.9, last_epoch=-1)
        self.lrers = {'l_lrer': self.l_lrer, 'r_lrer': self.r_lrer, 'fd_lrer': self.fd_lrer}
        self.l_criterion = criterion_funcs[0](self.args)
        self.r_criterion = criterion_funcs[1](self.args)
        self.criterions = {'l_criterion': self.l_criterion, 'r_criterion': self.r_criterion,
                           'fd_criterion': ops.mse_consistency, 'dc_criterion': ops.mse_consistency}

    # ------------------------------------------------------------------------------------------
    def _task_model_iter(self, mid, lbs, inp, gt, dc_gt, fc_mask, dc_rampup_scale):
        a = self.args
        model, criterion = (self.l_model, self.l_criterion) if mid == 'l' else (self.r_model, self.r_criterion)
        resulter, _ = model.forward(inp)
        if 'pred' not in resulter or 'activated_pred' not in resulter:
            logger.log_err('In SSL_GCT, the \'resulter\' dict returned by the task model should contain \'pred\' '
                           'and \'activated_pred\'\n')
        pred = tool.dict_value(resulter, 'pred')
        activated = tool.dict_value(resulter, 'activated_pred')[0]
        flawmap = self.fd_model.forward(inp, activated)[0]['flawmap']
        task_loss = torch.mean(criterion.forward(func.split_tensor_tuple(pred, 0, lbs), func.split_tensor_tuple(gt, 0, lbs),
                                                 func.split_tensor_tuple(inp, 0, lbs)))
        self.meters.update('{0}_task_loss'.format(mid), task_loss.data)
        if a.ssl_mode in (MODE_GCT, MODE_FC):
            fc = flawmap * flawmap                        # F.mse_loss(flawmap, 0, 'none'): one-channel maps
            if a.ssl_mode == MODE_GCT:
                fc = fc_mask * fc
            fc_ssl_loss = a.fc_ssl_scale * torch.mean(fc)
            self.meters.update('{0}_fc_loss'.format(mid), fc_ssl_loss.data)
        else:
            fc_ssl_loss = 0
            self.meters.update('{0}_fc_loss'.format(mid), fc_ssl_loss)
        if a.ssl_mode in (MODE_GCT, MODE_DC):
            if dc_gt is None:
                logger.log_err('The dynamic consistency constraint is enabled, but no pseudo ground truth is given.')
            dc_ssl_loss = ops.mse_consistency(activated, dc_gt, dc_rampup_scale * a.dc_ssl_scale, unit_upstream=True)
            self.meters.update('{0}_dc_loss'.format(mid), dc_ssl_loss.data)
        else:
            dc_ssl_loss = 0
            self.meters.update('{0}_dc_loss'.format(mid), dc_ssl_loss)
        return task_loss + fc_ssl_loss + dc_ssl_loss

    def train_step(self, inp, gt, cur_steps, total_steps):
        a = self.args
        lbs = a.labeled_batch_size
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        l_inp = r_inp = inp
        l_gt = r_gt = gt
        dc_rampup_scale = func.sigmoid_rampup(cur_steps, total_steps)

        # ---- step 0: pre-forward
        with torch.no_grad():
            l_act = tool.dict_value(self.l_model.forward(l_inp)[0], 'activated_pred')[0]
            r_act = tool.dict_value(self.r_model.forward(r_inp)[0], 'activated_pred')[0]
        for p in self.fd_model.parameters():
            p.requires_grad_(True)
        l_flawmap = self.fd_model.forward(l_inp, l_act)[0]['flawmap']
        r_flawmap = self.fd_model.forward(r_inp, r_act)[0]['flawmap']
        l_dc_gt = r_dc_gt = l_fc_mask = r_fc_mask = None
        if a.ssl_mode in (MODE_GCT, MODE_DC):
            with torch.no_grad():
                l_handled = ops.flawmap_handle(l_flawmap, a.im_size)
                r_handled = ops.flawmap_handle(r_flawmap, a.im_size)
                l_dc_gt, r_dc_gt, both_bad = ops.gct_dcgt(l_act, r_act, l_handled, r_handled, a.dc_threshold)
                l_fc_mask = r_fc_mask = both_bad

        # ---- step 1: task models (flaw detector frozen)
        for p in self.fd_model.parameters():
            p.requires_grad_(False)
        for mid, model, opt, m_inp, m_gt, dc_gt, fc_mask in (('l', self.l_model, self.l_optimizer, l_inp, l_gt, l_dc_gt, l_fc_mask),
                                                            ('r', self.r_model, self.r_optimizer, r_inp, r_gt, r_dc_gt, r_fc_mask)):
            model.arena.zero_grad()
            loss = self._task_model_iter(mid, lbs, m_inp, m_gt, dc_gt, fc_mask, dc_rampup_scale)
            loss.backward()
            model.arena.all_reduce_grads()
            model.arena.sgd_step(opt)

        # ---- step 2: flaw detector
        for p in self.fd_model.parameters():
            p.requires_grad_(True)
        with torch.no_grad():
            l_fm_gt = ops.fdgt_generate(l_act[:lbs].contiguous(), l_gt[0][:lbs].contiguous(), a.im_size, a.mu, a.nu)
            r_fm_gt = ops.fdgt_generate(r_act[:lbs].contiguous(), r_gt[0][:lbs].contiguous(), a.im_size, a.mu, a.nu)
        l_fd_loss = ops.mse_consistency(l_flawmap[:lbs], l_fm_gt, a.fd_scale)
        r_fd_loss = ops.mse_consistency(r_flawmap[:lbs], r_fm_gt, a.fd_scale)
        self.meters.update('l_fd_loss', l_fd_loss.data)
        self.meters.update('r_fd_loss', r_fd_loss.data)
        fd_loss = (l_fd_loss + r_fd_loss) / 2
        self.fd_model.arena.zero_grad()
        fd_loss.backward()
        self.fd_model.arena.all_reduce_grads()
        self.fd_model.arena.adam_step(self.fd_optimizer)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        for mid, model, crit in (('l', self.l_model, self.l_criterion), ('r', self.r_model, self.r_criterion)):
            self._validate_model(model, crit, inp, gt, mid + '_task_loss', mid)
