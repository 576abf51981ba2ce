"""Cross Pseudo Supervision (Chen, Yuan, Zeng, Wang, "Semi-Supervised Semantic Segmentation with Cross Pseudo
Supervision", CVPR 2021) on the H100 kernels.

Two task models with independent initialisations; each is supervised by the other's per-pixel argmax (one fused
kernel, ``ops.cps_cross_entropy``, computes both cross-entropies and both gradients).

Plain step: one forward per model over the whole ``[labeled..., unlabeled...]`` batch (PixelSSL's convention, as the
Mean-Teacher student), task criterion on the labeled rows, CPS term on ALL rows (as in the paper), one backward of
the sum, SGD on each model.
CutMix step (``--cps-cutmix``, the paper's VOC configuration): per model a forward of the labeled rows + task
criterion, a no-grad forward of the unlabeled rows whose two halves are mixed with the box mask (the pseudo-label
source), and a forward of the mixed images, which the CPS term supervises."""
import torch

from .. import ops
from ..utils import CLASSIFICATION, logger, cmd, tool
from ..nn import func
from . import ssl_base
from .ssl_cutmix import BoxMaskGenerator


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--cps-scale', type=float, default=-1)
    parser.add_argument('--cps-rampup-epochs', type=int, default=-1)
    parser.add_argument('--cps-cutmix', type=cmd.str2bool, default=False)
    parser.add_argument('--mask-prop-range', type=cmd.str2floatlist, default='(0.5, 0.5)')


def ssl_cps(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    pick = ssl_base.pair_picker(SSLCPS.NAME, model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLCPS(args)
    algorithm.build(pick(model_dict), pick(optimizer_dict), pick(lrer_dict), pick(criterion_dict), task_func)
    return algorithm


class SSLCPS(ssl_base._SSLBase):
    NAME = 'ssl_cps'
    SUPPORTED_TASK_TYPES = [CLASSIFICATION]
    RAMPUP_EPOCHS = 'cps_rampup_epochs'
    LOG_LINES = ('  l-{3}\t=>\tl-task-loss: {meters[l_task_loss]:.6f}\tl-cps-loss: {meters[l_cps_loss]:.6f}\n'
                 '  r-{3}\t=>\tr-task-loss: {meters[r_task_loss]:.6f}\tr-cps-loss: {meters[r_cps_loss]:.6f}\n')
    VALIDATION_IDS = ('l', 'r')

    def __init__(self, args):
        super().__init__(args)
        self.l_model = self.r_model = None
        self.mask_generator = None
        a = self.args
        if a.unlabeled_batch_size > 0:
            if a.cps_scale < 0:
                logger.log_err('The argument - cps_scale - is not set (or invalid)\n')
            if a.cps_rampup_epochs < 0:
                logger.log_err('The argument - cps_rampup_epochs - is not set (or invalid)\n')
            if a.cps_cutmix and (a.unlabeled_batch_size <= 2 or a.unlabeled_batch_size % 2 != 0):
                logger.log_err('SSL_CPS with cps_cutmix requires an unlabeled batch size that is larger than 2 and '
                               'divisible by 2 (pairs of unlabeled samples are mixed)\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        # two create_model calls: independent initialisations even when one model class serves both sides
        self.l_model = func.create_model(model_funcs[0], 'l_model', args=self.args)
        self.r_model = func.create_model(model_funcs[1], 'r_model', args=self.args)
        self.models = {'l_model': self.l_model, 'r_model': self.r_model}
        self.l_optimizer = optimizer_funcs[0](self.l_model.module.param_groups)
        self.r_optimizer = optimizer_funcs[1](self.r_model.module.param_groups)
        self.optimizers = {'l_optimizer': self.l_optimizer, 'r_optimizer': self.r_optimizer}
        self.l_lrer = lrer_funcs[0](self.l_optimizer)
        self.r_lrer = lrer_funcs[1](self.r_optimizer)
        self.lrers = {'l_lrer': self.l_lrer, 'r_lrer': self.r_lrer}
        self.l_criterion = criterion_funcs[0](self.args)
        self.r_criterion = criterion_funcs[1](self.args)
        self.criterions = {'l_criterion': self.l_criterion, 'r_criterion': self.r_criterion,
                           'cps_criterion': ops.cps_cross_entropy}
        if self.args.cps_cutmix:
            prop = self.args.mask_prop_range
            if isinstance(prop, str):
                prop = cmd.str2floatlist(prop)
            self.mask_generator = BoxMaskGenerator(prop_range=prop, boxes_num=1, invert=True)

    # ------------------------------------------------------------------------------------------
    def _pred(self, model, inp):
        resulter, _ = model.forward(inp)
        if 'pred' not in resulter or 'activated_pred' not in resulter:
            self._pred_err()
        return tool.dict_value(resulter, 'pred')

    def _task_loss(self, mid, criterion, pred, gt, inp, lbs):
        # torch.mean(per-sample) goes straight into the loss -> d loss / d per_sample = 1/lbs
        loss = torch.mean(criterion.forward(func.split_tensor_tuple(pred, 0, lbs), func.split_tensor_tuple(gt, 0, lbs),
                                            func.split_tensor_tuple(inp, 0, lbs), mean_upstream=1.0 / lbs))
        self.meters.update('{0}_task_loss'.format(mid), loss.data)
        return loss

    def _plain_losses(self, inp, gt, lbs, ubs, scale):
        l_pred = self._pred(self.l_model, inp)
        r_pred = self._pred(self.r_model, inp)
        task = (self._task_loss('l', self.l_criterion, l_pred, gt, inp, lbs) +
                self._task_loss('r', self.r_criterion, r_pred, gt, inp, lbs))
        if ubs == 0:
            return task, None
        return task, ops.cps_cross_entropy(l_pred[0], r_pred[0], loss_scale=scale, unit_upstream=True)

    def _cutmix_losses(self, inp, gt, lbs, ubs, scale):
        l_inp = func.split_tensor_tuple(inp, 0, lbs)
        l_gt = func.split_tensor_tuple(gt, 0, lbs)
        task = (self._task_loss('l', self.l_criterion, self._pred(self.l_model, l_inp), l_gt, l_inp, lbs) +
                self._task_loss('r', self.r_criterion, self._pred(self.r_model, l_inp), l_gt, l_inp, lbs))
        if ubs == 0:
            return task, None
        half = ubs // 2
        mask = torch.from_numpy(self.mask_generator.produce(half, tuple(inp[0].shape[2:]))).cuda(non_blocking=True)
        u1 = func.split_tensor_tuple(inp, lbs, lbs + half)
        u2 = func.split_tensor_tuple(inp, lbs + half, lbs + ubs)
        mix_u_inp = tuple(ops.cutmix_mix(mask, a.contiguous(), b.contiguous()) for a, b in zip(u1, u2))
        u_inp = func.split_tensor_tuple(inp, lbs, lbs + ubs)
        with torch.no_grad():
            # pseudo-label sources: each model's logits on the unlabeled rows, halves mixed like the images
            mixed_t = []
            for model in (self.l_model, self.r_model):
                up = self._pred(model, u_inp)[0]
                mixed_t.append(ops.cutmix_mix(mask, up[:half].contiguous(), up[half:ubs].contiguous()))
        l_mixed = self._pred(self.l_model, mix_u_inp)[0]
        r_mixed = self._pred(self.r_model, mix_u_inp)[0]
        return task, ops.cps_cross_entropy(l_mixed, r_mixed, t_l=mixed_t[0], t_r=mixed_t[1], loss_scale=scale,
                                           unit_upstream=True)

    def train_step(self, inp, gt, cur_step, total_rampup_steps):
        a = self.args
        lbs, ubs = a.labeled_batch_size, a.unlabeled_batch_size
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        scale = func.sigmoid_rampup(cur_step, total_rampup_steps) * a.cps_scale
        self.l_model.arena.zero_grad()
        self.r_model.arena.zero_grad()
        task, cps = (self._cutmix_losses if a.cps_cutmix else self._plain_losses)(inp, gt, lbs, ubs, scale)
        if cps is None:
            self.meters.update('l_cps_loss', 0)
            self.meters.update('r_cps_loss', 0)
            loss = task
        else:
            self.meters.update('l_cps_loss', cps[0].data)
            self.meters.update('r_cps_loss', cps[1].data)
            loss = task + cps[0] + cps[1]
        loss.backward()
        for model, opt in ((self.l_model, self.l_optimizer), (self.r_model, self.r_optimizer)):
            model.arena.all_reduce_grads()
            model.arena.sgd_step(opt)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        for mid, model, crit in (('l', self.l_model, self.l_criterion), ('r', self.r_model, self.r_criterion)):
            self._validate_model(model, crit, inp, gt, mid + '_task_loss', mid)
