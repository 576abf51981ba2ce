"""UniMatch (Yang, Qi, Feng, Zhang, Shi, "Revisiting Weak-to-Strong Consistency in Semi-Supervised Semantic
Segmentation", CVPR 2023) on the H100 kernels.

One task model, one SGD optimizer, one lrer; no teacher.  The batch is ``[labeled..., unlabeled...]``; the unlabeled
rows are the weak view ``u_w``.  Image i's CutMix partner is image ``(i + ubs/2) mod ubs`` of the same batch (UniMatch
draws partners from a second unlabeled loader).  Per step:
  1. eval-mode no-grad forward of u_w, rolled by ubs/2 (inside the loss kernel): the pseudo-label source in the boxes;
  2. two strongly augmented views of u_w on the device (``ops.strong_aug``), each with a box of its partner's view;
  3. one training forward of the whole batch whose head also runs on Dropout2d copies of the features (``forward_fp``);
  4. one training forward of the two strong views;
  5. one fused kernel (``ops.unimatch_cross_entropy``): confidence-thresholded cross-entropies of both strong views
     and the FP prediction against the weak view's pseudo-labels, and their gradients;
  6. loss = (task + r * s * (L_s1 / 4 + L_s2 / 4 + L_fp / 2)) / 2, one backward, SGD.

Host draws, once per step and in this order:
  * ``draw_strong_params`` from the global ``np.random`` stream: for each unlabeled image i and for its view 1 then
    view 2 - the ColorJitter coin (applied if < 0.8) and, if applied, the op order (``np.random.permutation(4)``:
    0 brightness, 1 contrast, 2 saturation, 3 hue) and the factors b, c, s ~ U[0.5, 1.5], h ~ U[-0.25, 0.25]; the
    grayscale coin (< 0.2); the blur coin (< 0.5) and, if applied, sigma ~ U[0.1, 2.0]; the box coin (no box if
    > cutmix_prob) and, if a box, UniMatch's ``obtain_cutmix_box`` draws (area ~ U[0.02, 0.4] * H * W, then aspect
    ratio ~ U[0.3, 1/0.3], x, y until the box fits).
  * the Dropout2d factors from torch's CPU generator, as CCT's DropOutDecoder draws them: one [n, C] tensor per
    feature map the task model perturbs (``fp_channels``), n = lbs + ubs."""
import math

import numpy as np
import torch

from .. import ops
from ..utils import CLASSIFICATION, logger, tool
from ..nn import func
from . import ssl_base

AUG_COLS = 32            # per-view parameter row of ops.strong_aug (layout in csrc/strong_aug.cu)
AUG_MAXK = 6             # blur half width at sigma = 2.0: ceil(3 * sigma)


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--uni-threshold', type=float, default=-1)
    parser.add_argument('--uni-scale', type=float, default=-1)
    parser.add_argument('--uni-rampup-epochs', type=int, default=-1)
    parser.add_argument('--uni-fp-drop', type=float, default=0.5)
    parser.add_argument('--uni-cutmix-prob', type=float, default=0.5)


def ssl_unimatch(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_unimatch', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLUNIMATCH(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


def gaussian_weights(sigma):
    """1-D weights of torchvision's ``gaussian_blur`` with kernel size 2 * ceil(3 sigma) + 1 (fp64)."""
    half = int(math.ceil(3.0 * sigma))
    ks = 2 * half + 1
    lim = (ks - 1) / (2.0 * math.sqrt(2.0) * sigma)
    x = np.linspace(-lim, lim, ks)
    e = np.exp(-x * x - np.max(-x * x))
    return e / e.sum()


def cutmix_box(h, w, cutmix_prob, rng):
    """UniMatch's ``obtain_cutmix_box`` on an h x w image -> (y0, x0, y1, x1), or None (no box)."""
    if rng.random_sample() > cutmix_prob:
        return None
    size = rng.uniform(0.02, 0.4) * h * w
    while True:
        ratio = rng.uniform(0.3, 1 / 0.3)
        cw, ch = int(np.sqrt(size / ratio)), int(np.sqrt(size * ratio))
        x, y = rng.randint(0, w), rng.randint(0, h)
        if x + cw <= w and y + ch <= h:
            return y, x, y + ch, x + cw


def draw_strong_params(ubs, h, w, cutmix_prob=0.5, rng=None):
    """The strong-view parameters of one step (draw order in the module docstring) -> (table float32
    [2*ubs, AUG_COLS] for ``ops.strong_aug``, boxes int32 [2*ubs, 4] for ``ops.unimatch_cross_entropy``).  Row
    k * ubs + i is view k of image i."""
    rng = np.random if rng is None else rng
    table = np.zeros((2 * ubs, AUG_COLS), dtype=np.float64)
    boxes = np.zeros((2 * ubs, 4), dtype=np.int32)
    for i in range(ubs):
        for k in range(2):
            row = table[k * ubs + i]
            if rng.random_sample() < 0.8:
                row[0] = 1.0
                row[5:9] = rng.permutation(4)
                row[1] = rng.uniform(0.5, 1.5)
                row[2] = rng.uniform(0.5, 1.5)
                row[3] = rng.uniform(0.5, 1.5)
                row[4] = rng.uniform(-0.25, 0.25)
            else:
                row[5:9] = (0, 1, 2, 3)
            row[9] = 1.0 if rng.random_sample() < 0.2 else 0.0
            if rng.random_sample() < 0.5:
                sigma = rng.uniform(0.1, 2.0)
                wts = gaussian_weights(sigma)
                row[10], row[11] = (len(wts) - 1) // 2, sigma
                row[16:16 + len(wts)] = wts
            box = cutmix_box(h, w, cutmix_prob, rng)
            if box is not None:
                row[12:16] = box
                boxes[k * ubs + i] = box
    return table.astype(np.float32), boxes


def draw_fp_scales(n, channels, p):
    """Dropout2d factors for ``forward_fp``: per feature map one [n, C] tensor of Bernoulli(1 - p) / (1 - p) draws
    from torch's CPU generator (CCT's DropOutDecoder, ssl_cct.py)."""
    return [(torch.empty(n, c, 1, 1).bernoulli_(1 - p) / (1 - p)).view(n, c) for c in channels]


class SSLUNIMATCH(ssl_base._SSLBase):
    NAME = 'ssl_unimatch'
    SUPPORTED_TASK_TYPES = [CLASSIFICATION]
    RAMPUP_EPOCHS = 'uni_rampup_epochs'
    LOG_LINES = ('  task-{3}\t=>\ttask-loss: {meters[task_loss]:.6f}\ts1-loss: {meters[s1_loss]:.6f}\t'
                 's2-loss: {meters[s2_loss]:.6f}\tfp-loss: {meters[fp_loss]:.6f}\t'
                 'mask-ratio: {meters[mask_ratio]:.4f}\n')

    def __init__(self, args):
        super().__init__(args)
        self.model = self.optimizer = self.lrer = self.criterion = None
        a = self.args
        if not 0.0 <= a.uni_threshold <= 1.0:
            logger.log_err('The argument - uni_threshold - is not set (or invalid): it must lie in [0, 1]\n')
        if a.uni_scale < 0:
            logger.log_err('The argument - uni_scale - is not set (or invalid)\n')
        if a.uni_rampup_epochs < 0:
            logger.log_err('The argument - uni_rampup_epochs - is not set (or invalid)\n')
        if not 0.0 <= a.uni_fp_drop < 1.0:
            logger.log_err('The argument - uni_fp_drop - must lie in [0, 1)\n')
        if not 0.0 <= a.uni_cutmix_prob <= 1.0:
            logger.log_err('The argument - uni_cutmix_prob - must lie in [0, 1]\n')
        if a.unlabeled_batch_size < 2 or a.unlabeled_batch_size % 2 != 0:
            logger.log_err('SSL_UNIMATCH requires an unlabeled batch size that is at least 2 and divisible by 2 '
                           '(image i is mixed with image i + unlabeled_batch_size / 2)\n')

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        if getattr(model_funcs[0], 'forward_fp', None) is None:
            logger.log_err('SSL_UNIMATCH needs a task model with a feature-perturbation forward (forward_fp): '
                           'deeplabv2 or deeplabv3plus; {0} does not have one\n'.format(
                               getattr(model_funcs[0], '__name__', model_funcs[0])))
        self.task_func = task_func
        self.model = func.create_model(model_funcs[0], 'model', args=self.args)
        self.models = {'model': self.model}
        self.optimizer = optimizer_funcs[0](self.model.module.param_groups)
        self.optimizers = {'optimizer': self.optimizer}
        self.lrer = lrer_funcs[0](self.optimizer)
        self.lrers = {'lrer': self.lrer}
        self.criterion = criterion_funcs[0](self.args)
        self.criterions = {'criterion': self.criterion, 'unimatch_criterion': ops.unimatch_cross_entropy}

    def _pred(self, inp):
        resulter, _ = self.model.forward(inp)
        if 'pred' not in resulter or 'activated_pred' not in resulter:
            self._pred_err()
        return tool.dict_value(resulter, 'pred')[0]

    def train_step(self, inp, gt, cur_step, total_rampup_steps):
        a = self.args
        lbs, ubs = a.labeled_batch_size, a.unlabeled_batch_size
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        img = inp[0]
        h, w = img.shape[2:]
        scale = func.sigmoid_rampup(cur_step, total_rampup_steps) * a.uni_scale
        table, boxes = draw_strong_params(ubs, h, w, a.uni_cutmix_prob)
        fp_scales = [s.cuda(non_blocking=True)
                     for s in draw_fp_scales(lbs + ubs, self.model.module.fp_channels, a.uni_fp_drop)]
        table = torch.from_numpy(table).cuda(non_blocking=True)
        boxes = torch.from_numpy(boxes)
        u_w = img[lbs:].contiguous()
        self.model.arena.zero_grad()

        # 1. the pseudo-label source inside the boxes: eval mode, as UniMatch
        self.model.eval()
        with torch.no_grad():
            mix = self._pred((u_w,))
        self.model.train()
        # 2-4. strong views, the forward with feature perturbation, the forward of the strong views
        strong, _ = ops.strong_aug(u_w, table)
        resulter, resulter_fp = self.model.module.forward_fp(inp, fp_scales)
        pred, pred_fp = tool.dict_value(resulter, 'pred')[0], tool.dict_value(resulter_fp, 'pred')[0]
        pred_s = self._pred((strong,))
        # 5-6. losses; the task term enters the total with weight 1/2, so d total / d per_sample = 1 / (2 lbs)
        task = torch.mean(self.criterion.forward((pred[:lbs],), func.split_tensor_tuple(gt, 0, lbs), (img[:lbs],),
                                                 mean_upstream=0.5 / lbs))
        weights = (scale / 8.0, scale / 8.0, scale / 4.0)
        l_s1, l_s2, l_fp, count = ops.unimatch_cross_entropy(pred_s, pred_fp, pred[lbs:], mix, boxes, a.uni_threshold,
                                                             weights=weights, fp_offset=lbs, unit_upstream=True)
        loss = 0.5 * task + weights[0] * l_s1 + weights[1] * l_s2 + weights[2] * l_fp
        self.meters.update('task_loss', task.data)
        self.meters.update('s1_loss', l_s1.data)
        self.meters.update('s2_loss', l_s2.data)
        self.meters.update('fp_loss', l_fp.data)
        self.meters.update('mask_ratio', count.data / float(ubs * h * w))
        # 7. update
        loss.backward()
        self.model.arena.all_reduce_grads()
        self.model.arena.sgd_step(self.optimizer)

    def validate_step(self, inp, gt):
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        self._validate_model(self.model, self.criterion, inp, gt, 'task_loss', 'task')
