"""CutMix consistency (pixelssl/ssl_algorithm/ssl_cutmix.py:132-255) on the H100 kernels.

Per step: host box masks (numpy RNG, identical draws to the reference) -> bit-exact device mix
of the two unlabeled halves -> student fwd on the labeled rows + CE -> teacher fwd (no grad) on
the unlabeled rows -> softmax -> mix of the two halves with the same mask (pseudo label) ->
batch-global confidence scalar -> student fwd on the mixed images -> fused softmax+MSE
(confidence * rampup * cons_scale) -> backward -> SGD fused with the teacher EMA.
Three separate forwards are kept (BN batch statistics depend on the grouping, SURVEY.md 7)."""
import numpy as np
import torch

from .. import ops
from ..utils import CLASSIFICATION, logger, cmd, tool
from ..nn import func
from . import ssl_base


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--cons-scale', type=float, default=-1)
    parser.add_argument('--cons-rampup-epochs', type=int, default=-1)
    parser.add_argument('--cons-type', type=str, default='mse', choices=['mse'])
    parser.add_argument('--cons-threshold', type=float, default=-1)
    parser.add_argument('--ema-decay', type=float, default=0.99)
    parser.add_argument('--mask-prop-range', type=cmd.str2floatlist, default='(0.5, 0.5)')


def ssl_cutmix(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_cutmix', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLCUTMIX(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


class BoxMaskGenerator:
    """Host-side box masks, one box per mask with area = prop * H * W, log-uniform aspect ratio,
    placed within bounds; invert=True -> 1 inside the box (ssl_cutmix.py:470-547 as configured at
    :126-128).  Uses the global ``np.random`` stream in the reference's draw order (proportions,
    aspect exponents, positions), so a seeded run reproduces the reference masks bit for bit."""

    def __init__(self, prop_range, boxes_num=1, invert=True, rng=None):
        self.prop_range, self.boxes_num, self.invert = tuple(prop_range), boxes_num, invert
        self.rng = rng

    def produce(self, mask_num, mask_shape):
        rng = self.rng if self.rng is not None else np.random
        shape2 = (mask_num, self.boxes_num)
        props = rng.uniform(self.prop_range[0], self.prop_range[1], size=shape2)
        degenerate = props == 0.0
        y_frac = np.exp(rng.uniform(low=0.0, high=1.0, size=shape2) * np.log(props))
        x_frac = props / y_frac
        shrink = np.sqrt(1.0 / self.boxes_num)
        y_frac, x_frac = y_frac * shrink, x_frac * shrink
        y_frac[degenerate] = 0
        x_frac[degenerate] = 0
        extent = np.array(mask_shape)
        sizes = np.round(np.stack([y_frac, x_frac], axis=2) * extent[None, None, :])
        corner = np.round((extent - sizes) * rng.uniform(low=0.0, high=1.0, size=sizes.shape))
        boxes = np.append(corner, corner + sizes, axis=2)
        fill = 0.0 if self.invert else 1.0
        masks = np.full((mask_num, 1) + tuple(mask_shape), fill, dtype=np.float64)
        for i in range(mask_num):
            for y0, x0, y1, x1 in boxes[i]:
                region = masks[i, 0, int(y0):int(y1), int(x0):int(x1)]
                masks[i, 0, int(y0):int(y1), int(x0):int(x1)] = 1 - region
        return masks.astype(np.float32)


class SSLCUTMIX(ssl_base._SSLBase):
    NAME = 'ssl_cutmix'
    SUPPORTED_TASK_TYPES = [CLASSIFICATION]
    RAMPUP_EPOCHS = 'cons_rampup_epochs'
    LOG_LINES = ('  student-{3}\t=>\t'
                 's-task-loss: {meters[task_loss]:.6f}\t'
                 's-cons-loss: {meters[cons_loss]:.6f}\n')
    VALIDATION_IDS = ('student', 'teacher')

    def __init__(self, args):
        super().__init__(args)
        self.s_model = self.t_model = None
        self.s_optimizer = self.s_lrer = self.s_criterion = None
        self.mask_generator = None
        if self.args.unlabeled_batch_size > 0:
            if self.args.cons_scale < 0:
                logger.log_err('The argument - cons_scale - is not set (or invalid)\n')
            if self.args.cons_rampup_epochs < 0:
                logger.log_err('The argument - cons_rampup_epochs - is not set (or invalid)\n')
            if self.args.unlabeled_batch_size <= 2 or self.args.unlabeled_batch_size % 2 != 0:
                logger.log_err('SSL_CUTMIX requires an unlabeled batch size that is larger than 2 and divisible by 2 '
                               '(pairs of unlabeled samples are mixed)\n')
            if self.args.cons_threshold < 0 or self.args.cons_threshold > 1:
                logger.log_err('The argument - cons_threshold - is not set (or invalid)\n'
                               'Please set - 0 <= cons_threshold < 1 - for training\n')
        if self.args.cons_type != 'mse':
            logger.log_err('SSL_CUTMIX only supports cons_type == mse\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        self.task_func = task_func
        self.s_model = func.create_model(model_funcs[0], 's_model', args=self.args)
        self.t_model = func.create_model(model_funcs[0], 't_model', args=self.args)
        for p in self.t_model.parameters():
            p.requires_grad_(False)
        self.models = {'s_model': self.s_model, 't_model': self.t_model}
        self.s_optimizer = optimizer_funcs[0](self.s_model.module.param_groups)
        self.optimizers = {'s_optimizer': self.s_optimizer}
        self.s_lrer = lrer_funcs[0](self.s_optimizer)
        self.lrers = {'s_lrer': self.s_lrer}
        self.s_criterion = criterion_funcs[0](self.args)
        self.criterions = {'s_criterion': self.s_criterion, 'cons_criterion': ops.softmax_mse}
        prop = self.args.mask_prop_range
        if isinstance(prop, str):
            prop = cmd.str2floatlist(prop)
        self.mask_generator = BoxMaskGenerator(prop_range=prop, boxes_num=1, invert=True)

    def train_step(self, inp, gt, cur_step, total_rampup_steps):
        lbs, ubs = self.args.labeled_batch_size, self.args.unlabeled_batch_size
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        cons_rampup_scale = func.sigmoid_rampup(cur_step, total_rampup_steps)
        s_arena, t_arena = self.s_model.arena, self.t_model.arena
        s_arena.zero_grad()

        l_inp = func.split_tensor_tuple(inp, 0, lbs)
        l_gt = func.split_tensor_tuple(gt, 0, lbs)
        l_s_resulter, _ = self.s_model.forward(l_inp)
        l_s_pred = tool.dict_value(l_s_resulter, 'pred')
        task_loss = torch.mean(self.s_criterion.forward(l_s_pred, l_gt, l_inp, mean_upstream=1.0 / lbs))
        self.meters.update('task_loss', task_loss.data)

        if ubs > 0:
            half = ubs // 2
            hw = tuple(inp[0].shape[2:])
            mask = torch.from_numpy(self.mask_generator.produce(half, hw)).cuda(non_blocking=True)
            u1 = func.split_tensor_tuple(inp, lbs, lbs + half)
            u2 = func.split_tensor_tuple(inp, lbs + half, lbs + ubs)
            mix_u_inp = tuple(ops.cutmix_mix(mask, a.contiguous(), b.contiguous()) for a, b in zip(u1, u2))
            u_inp = func.split_tensor_tuple(inp, lbs, lbs + ubs)
            with torch.no_grad():
                u_t_resulter, _ = self.t_model.forward(u_inp)
                u_t_act = tool.dict_value(u_t_resulter, 'activated_pred')
                mixed_t, confidences = [], []
                for up in u_t_act:
                    mp = ops.cutmix_mix(mask, up[:half].contiguous(), up[half:ubs].contiguous())
                    mixed_t.append(mp)
                    confidences.append(ops.cutmix_confidence(mp, self.args.cons_threshold))
            u_s_resulter, _ = self.s_model.forward(mix_u_inp)
            u_s_pred = tool.dict_value(u_s_resulter, 'pred')
            cons_loss = 0
            for s_logits, mp, conf in zip(u_s_pred, mixed_t, confidences):
                cons_loss = cons_loss + ops.softmax_mse(s_logits, mp, cons_rampup_scale * self.args.cons_scale) * conf
            self.meters.update('cons_loss', cons_loss.data)
        else:
            cons_loss = 0
            self.meters.update('cons_loss', cons_loss)

        loss = task_loss + cons_loss
        loss.backward()
        s_arena.all_reduce_grads()
        ema_decay = min(1 - 1 / (cur_step + 1), self.args.ema_decay)
        s_arena.sgd_step(self.s_optimizer, teacher=t_arena, ema_d=ema_decay)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        self._validate_model(self.s_model, self.s_criterion, inp, gt, 's_task_loss', 'student')
        self._validate_model(self.t_model, self.s_criterion, inp, gt, 't_task_loss', 'teacher')
