"""Adversarial SSL (pixelssl/ssl_algorithm/ssl_adv.py:118-283) on the H100 kernels.

step 1 (task model): forward -> softmax -> FC discriminator (frozen for this step) -> CE on the
labeled rows + BCE(confidence, real) adversarial terms -> backward -> SGD.
step 2 (discriminator): forward on the detached softmax (fake, target 0) and on the one-hot ground
truth (real, target 1) -> (fake + real)/2 -> backward -> Adam(0.9, 0.99) -> PolynomialLR.

Device-side replacements of the reference's host round trips: ``ssladv_preprocess_fcd_criterion`` +
``FCDiscriminatorCriterion`` (numpy masks every step, task/sseg/func.py:137-155) are one masked-BCE
kernel; ``ssladv_convert_task_gt_to_fcd_input`` (numpy one-hot, func.py:157-168) is one kernel that
writes the NHWC one-hot the first discriminator convolution reads."""
import torch
import torch.nn as nn
import torch.optim as optim

from .. import ops
from ..utils import REGRESSION, CLASSIFICATION, logger, cmd, tool
from ..nn import func
from ..nn.lrer import PolynomialLR
from ..nn.modules import Conv2d
from . import ssl_base


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--adv-for-labeled', type=cmd.str2bool, default=False)
    parser.add_argument('--labeled-adv-scale', type=float, default=-1)
    parser.add_argument('--unlabeled-adv-scale', type=float, default=-1)
    parser.add_argument('--discriminator-lr', type=float, default=1e-4)
    parser.add_argument('--discriminator-power', type=float, default=0.9)
    parser.add_argument('--unlabeled-for-discriminator', type=cmd.str2bool, default=False)
    parser.add_argument('--discriminator-scale', type=float, default=1.0)


def ssl_adv(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_adv', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLADV(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


class FCDiscriminator(nn.Module):
    """ssl_adv.py:466-493: 5 convs 4x4 / stride 2 / pad 1 (C -> 64 -> 128 -> 256 -> 512 -> 1), LeakyReLU(0.2),
    bilinear (align_corners) back to the input size; un-activated confidence map."""
    ndf = 64

    def __init__(self, in_channels):
        super().__init__()
        n = self.ndf
        self.in_channels = in_channels
        self.conv1 = Conv2d(in_channels, n, 4, stride=2, padding=1)
        self.conv2 = Conv2d(n, n * 2, 4, stride=2, padding=1)
        self.conv3 = Conv2d(n * 2, n * 4, 4, stride=2, padding=1)
        self.conv4 = Conv2d(n * 4, n * 8, 4, stride=2, padding=1)
        self.classifier = Conv2d(n * 8, 1, 4, stride=2, padding=1)

    def forward(self, task_pred, nhwc_padded=False):
        """task_pred: planar [B,C,H,W] class map, or (nhwc_padded=True) an already NHWC zero-padded one."""
        resulter, debugger = {}, {}
        size = task_pred.shape[2:]
        x = task_pred if nhwc_padded else ops.planar_to_nhwc(task_pred)
        x = ops.leaky_relu(self.conv1(x), 0.2)
        x = ops.leaky_relu(self.conv2(x), 0.2)
        x = ops.leaky_relu(self.conv3(x), 0.2)
        x = ops.leaky_relu(self.conv4(x), 0.2)
        x = self.classifier(x)
        resulter['confidence'] = ops.bilinear(x, size, align_corners=True, channels=1, nhwc=True)
        return resulter, debugger


class SSLADV(ssl_base._SSLBase):
    NAME = 'ssl_adv'
    SUPPORTED_TASK_TYPES = [REGRESSION, CLASSIFICATION]
    LOG_LINES = ('  task-{3}\t=>\t'
                 'task-loss: {meters[task_loss]:.6f}\t'
                 'labeled-adv-loss: {meters[labeled_adv_loss]:.6f}\t'
                 'unlabeled-adv-loss: {meters[unlabeled_adv_loss]:.6f}\n'
                 '  fc-discriminator\t=>\t'
                 'fake-d-loss: {meters[fake_d_loss]:.6f}\t'
                 'real-d-loss: {meters[real_d_loss]:.6f}\n')
    ITER_LRERS = ('d_lrer',)

    def __init__(self, args):
        super().__init__(args)
        self.model = self.d_model = None
        self.args.discriminator_lr *= self.args.gpus          # ssl_adv.py:72
        if self.args.adv_for_labeled and self.args.labeled_adv_scale < 0:
            logger.log_err('The argument - labeled_adv_scale - is not set (or invalid)\n')
        if self.args.unlabeled_batch_size > 0 and self.args.unlabeled_adv_scale < 0:
            logger.log_err('The argument - unlabeled_adv_scale - is not set (or invalid)\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.model = func.create_model(model_funcs[0], 'model', args=self.args)
        self.d_model = func.create_model(FCDiscriminator, 'd_model', in_channels=self.args.num_classes)
        self.models = {'model': self.model, 'd_model': self.d_model}
        self.optimizer = optimizer_funcs[0](self.model.module.param_groups)
        self.d_optimizer = optim.Adam([p for p in self.d_model.parameters() if p.requires_grad],
                                      lr=self.args.discriminator_lr, betas=(0.9, 0.99))
        self.optimizers = {'optimizer': self.optimizer, 'd_optimizer': self.d_optimizer}
        self.lrer = lrer_funcs[0](self.optimizer)
        self.d_lrer = PolynomialLR(self.d_optimizer, self.args.epochs, self.args.iters_per_epoch,
                                   power=self.args.discriminator_power, last_epoch=-1)
        self.lrers = {'lrer': self.lrer, 'd_lrer': self.d_lrer}
        self.criterion = criterion_funcs[0](self.args)
        self.criterions = {'criterion': self.criterion, 'd_criterion': ops.bce_logits_masked}

    def train_step(self, inp, gt, cur_step, total_steps):
        lbs, bs = self.args.labeled_batch_size, self.args.batch_size
        ignore = self.args.ignore_index
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        arena, d_arena = self.model.arena, self.d_model.arena

        # ---------------- step 1: task model ----------------
        arena.zero_grad()
        for p in self.d_model.parameters():
            p.requires_grad_(False)              # its gradients of this pass would be discarded (ssl_adv.py:204)
        resulter, _ = self.model.forward(inp)
        pred = tool.dict_value(resulter, 'pred')
        activated = tool.dict_value(resulter, 'activated_pred')[0]
        confidence_map = self.d_model.forward(activated)[0]['confidence']
        l_pred = func.split_tensor_tuple(pred, 0, lbs)
        l_gt = func.split_tensor_tuple(gt, 0, lbs)
        task_loss = torch.mean(self.criterion.forward(l_pred, l_gt, func.split_tensor_tuple(inp, 0, lbs)))
        self.meters.update('task_loss', task_loss.data)
        if self.args.adv_for_labeled:
            labeled_adv_loss = self.args.labeled_adv_scale * torch.mean(
                ops.bce_logits_masked(confidence_map[:lbs], l_gt[0], 1.0, ignore))
            self.meters.update('labeled_adv_loss', labeled_adv_loss.data)
        else:
            labeled_adv_loss = 0
            self.meters.update('labeled_adv_loss', labeled_adv_loss)
        if self.args.unlabeled_batch_size > 0:
            unlabeled_adv_loss = self.args.unlabeled_adv_scale * torch.mean(
                ops.bce_logits_masked(confidence_map[lbs:bs], None, 1.0, ignore))
            self.meters.update('unlabeled_adv_loss', unlabeled_adv_loss.data)
        else:
            unlabeled_adv_loss = 0
            self.meters.update('unlabeled_adv_loss', unlabeled_adv_loss)
        loss = task_loss + labeled_adv_loss + unlabeled_adv_loss
        loss.backward()
        arena.all_reduce_grads()
        arena.sgd_step(self.optimizer)

        # ---------------- step 2: FC discriminator ----------------
        for p in self.d_model.parameters():
            p.requires_grad_(True)
        d_arena.zero_grad()
        use_unl = self.args.unlabeled_for_discriminator and self.args.unlabeled_batch_size != 0
        fake_pred = activated.detach() if self.args.unlabeled_for_discriminator else activated[:lbs].detach()
        fake_conf = self.d_model.forward(fake_pred)[0]['confidence']
        fake_losses = ops.bce_logits_masked(fake_conf[:lbs], l_gt[0], 0.0, ignore)
        if use_unl:
            fake_losses = torch.cat((fake_losses, ops.bce_logits_masked(fake_conf[lbs:bs], None, 0.0, ignore)), dim=0)
        fake_d_loss = self.args.discriminator_scale * torch.mean(fake_losses)
        self.meters.update('fake_d_loss', fake_d_loss.data)
        real_gt = ops.onehot_nhwc(l_gt[0], self.args.num_classes)
        real_conf = self.d_model.forward(real_gt, nhwc_padded=True)[0]['confidence']
        real_d_loss = self.args.discriminator_scale * torch.mean(ops.bce_logits_masked(real_conf, l_gt[0], 1.0, ignore))
        self.meters.update('real_d_loss', real_d_loss.data)
        d_loss = (fake_d_loss + real_d_loss) / 2
        d_loss.backward()
        d_arena.all_reduce_grads()
        d_arena.adam_step(self.d_optimizer)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        self._validate_model(self.model, self.criterion, inp, gt, 'task_loss', 'task')
