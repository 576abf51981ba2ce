"""Pixel-wise Mean Teacher on the H100 kernels: the per-step loop of
pixelssl/ssl_algorithm/ssl_mt.py:124-224 with the same order of operations

    zero_grad -> student fwd -> CE(labeled) -> teacher fwd (no grad) + teacher CE (meter only)
    -> MSE(student logits, teacher logits) * rampup * cons_scale -> backward -> SGD -> EMA
    -> per-iteration LR step

but: the consistency loss and its gradient come from ONE fused kernel launch (12 B/element),
the CE gradient is written by the CE forward launch, SGD+EMA is one kernel per LR group over the
flat parameter arena, softmax ('activated_pred') is only materialised if something reads it, and
multi-GPU is one process per GPU with a single NCCL gradient all-reduce."""
import torch

from .. import ops
from ..utils import REGRESSION, CLASSIFICATION, logger, cmd, tool
from ..nn import func
from . import ssl_base


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--cons-for-labeled', type=cmd.str2bool, default=True)
    parser.add_argument('--cons-scale', type=float, default=-1)
    parser.add_argument('--cons-rampup-epochs', type=int, default=-1)
    parser.add_argument('--ema-decay', type=float, default=0.999)
    parser.add_argument('--gaussian-noise-std', type=float, default=None)


def ssl_mt(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_mt', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLMT(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


class SSLMT(ssl_base._SSLBase):
    NAME = 'ssl_mt'
    SUPPORTED_TASK_TYPES = [REGRESSION, CLASSIFICATION]
    RAMPUP_EPOCHS = 'cons_rampup_epochs'
    LOG_LINES = ('  student-{3}\t=>\t'
                 's-task-loss: {meters[s_task_loss]:.6f}\t'
                 's-cons-loss: {meters[cons_loss]:.6f}\n'
                 '  teacher-{3}\t=>\t'
                 't-task-loss: {meters[t_task_loss]:.6f}\n')
    VALIDATION_IDS = ('student', 'teacher')

    def __init__(self, args):
        super().__init__(args)
        self.s_model = self.t_model = None
        self.s_optimizer = self.s_lrer = self.s_criterion = None
        # argument checks of ssl_mt.py:76-89
        if self.args.cons_for_labeled or self.args.unlabeled_batch_size > 0:
            if self.args.cons_scale < 0:
                logger.log_err('The argument - cons_scale - is not set (or invalid)\n'
                               'Please set - cons_scale >= 0 - for training\n')
            if self.args.cons_rampup_epochs < 0:
                logger.log_err('The argument - cons_rampup_epochs - is not set (or invalid)\n'
                               'Please set - cons_rampup_epochs >= 0 - for training\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.s_model = func.create_model(model_funcs[0], 's_model', args=self.args)
        self.t_model = func.create_model(model_funcs[0], 't_model', args=self.args)
        for p in self.t_model.parameters():
            p.requires_grad_(False)              # the reference detaches the teacher (ssl_mt.py:101-102)
        self.models = {'s_model': self.s_model, 't_model': self.t_model}
        self.s_optimizer = optimizer_funcs[0](self.s_model.module.param_groups)
        self.optimizers = {'s_optimizer': self.s_optimizer}
        self.s_lrer = lrer_funcs[0](self.s_optimizer)
        self.lrers = {'s_lrer': self.s_lrer}
        self.s_criterion = criterion_funcs[0](self.args)
        self.criterions = {'s_criterion': self.s_criterion, 'cons_criterion': ops.mse_consistency}

    # ------------------------------------------------------------------------------------------
    def train_step(self, inp, gt, cur_step, total_rampup_steps):
        """One iteration of the loop body of ssl_mt.py:131-220 on host tensors ``inp``/``gt``
        (tuples).  Returns nothing; results land in ``self.meters`` as device tensors."""
        lbs = self.args.labeled_batch_size
        s_inp, t_inp, gt = self._batch_prehandle(inp, gt, True)
        cons_rampup_scale = func.sigmoid_rampup(cur_step, total_rampup_steps)
        s_arena, t_arena = self.s_model.arena, self.t_model.arena
        s_arena.zero_grad()

        s_resulter, _ = self.s_model.forward(s_inp)
        if 'pred' not in s_resulter or 'activated_pred' not in s_resulter:
            self._pred_err()
        s_pred = tool.dict_value(s_resulter, 'pred')
        l_s_pred = func.split_tensor_tuple(s_pred, 0, lbs)
        l_gt = func.split_tensor_tuple(gt, 0, lbs)
        l_s_inp = func.split_tensor_tuple(s_inp, 0, lbs)
        # torch.mean(per-sample) goes straight into the loss -> d loss / d per_sample = 1/lbs
        s_task_loss = torch.mean(self.s_criterion.forward(l_s_pred, l_gt, l_s_inp, mean_upstream=1.0 / lbs))
        self.meters.update('s_task_loss', s_task_loss.data)

        with torch.no_grad():
            t_resulter, _ = self.t_model.forward(t_inp)
            if 'pred' not in t_resulter:
                self._pred_err()
            t_pred = tool.dict_value(t_resulter, 'pred')
            l_t_pred = func.split_tensor_tuple(t_pred, 0, lbs)
            t_task_loss = torch.mean(self.s_criterion.forward(l_t_pred, l_gt, func.split_tensor_tuple(t_inp, 0, lbs)))
            self.meters.update('t_task_loss', t_task_loss.data)

        t_pseudo_gt = t_pred[0].detach()
        scale = cons_rampup_scale * self.args.cons_scale
        if self.args.cons_for_labeled:
            cons_loss = ops.mse_consistency(s_pred[0], t_pseudo_gt, scale, unit_upstream=True)
        elif self.args.unlabeled_batch_size > 0:
            cons_loss = ops.mse_consistency(s_pred[0][lbs:, ...], t_pseudo_gt[lbs:, ...], scale, unit_upstream=True)
        else:
            cons_loss = torch.zeros((), device=s_pred[0].device)
        self.meters.update('cons_loss', cons_loss.data)

        loss = s_task_loss + cons_loss
        loss.backward()
        s_arena.all_reduce_grads()
        # SGD step fused with the teacher EMA (order optimizer.step -> EMA as ssl_mt.py:193-196)
        ema_decay = min(1 - 1 / (cur_step + 1), self.args.ema_decay)
        s_arena.sgd_step(self.s_optimizer, teacher=t_arena, ema_d=ema_decay)

    def _batch_prehandle(self, inp, gt, is_train):
        """ssl_mt.py:337-357: host -> HBM; while training the first input element gets independent
        Gaussian noise for the student and the teacher (``pxl_gaussian_noise`` in place on each device
        copy).  With the noise disabled both models read the same device tensor."""
        std = getattr(self.args, 'gaussian_noise_std', None)
        s_inp = ssl_base.to_device(inp)
        if is_train and std is not None:
            t_first = s_inp[0].clone()
            s_inp = (ops.gaussian_noise_(s_inp[0], std),) + tuple(s_inp[1:])
            t_inp = (ops.gaussian_noise_(t_first, std),) + tuple(s_inp[1:])
        else:
            t_inp = s_inp
        return s_inp, t_inp, ssl_base.to_device(gt)

    def validate_step(self, inp, gt):
        s_inp, t_inp, gt = self._batch_prehandle(inp, gt, False)
        s_resulter, _ = self.s_model.forward(s_inp)
        s_pred = tool.dict_value(s_resulter, 'pred')
        self.meters.update('s_task_loss', torch.mean(self.s_criterion.forward(s_pred, gt, s_inp)).data)
        t_resulter, _ = self.t_model.forward(t_inp)
        t_pred = tool.dict_value(t_resulter, 'pred')
        self.meters.update('t_task_loss', torch.mean(self.s_criterion.forward(t_pred, gt, t_inp)).data)
        cons_loss = ops.mse_consistency(s_pred[0], t_pred[0].detach(), self.args.cons_scale)
        self.meters.update('cons_loss', cons_loss.data)
        self._metrics(s_resulter, gt, s_inp, 'student')
        self._metrics(t_resulter, gt, t_inp, 'teacher')
