"""Cross-Consistency Training (pixelssl/ssl_algorithm/ssl_cct.py:226-301, 438-745) on the H100 kernels.

One shared encoder (the task model) and K perturbation decoders (VAT, Dropout, G-Cutout, context /
object masking, feature drop, feature noise).  Per step: labeled rows -> task model -> CE; unlabeled
rows -> task model -> every auxiliary decoder consumes the SAME latent (autograd fans the K
gradients back into it) -> conv1x1 + 3 x (conv1x1 + ReLU + PixelShuffle) -> bilinear to the logit
size -> fused softmax + MSE against the detached main softmax; one backward, one fused SGD step
over backbone / head / decoder learning-rate groups.

Random draws use the same host generators in the same order as the reference (python ``random``,
``np.random``, torch's CPU generator; the reference itself draws them on the CPU and uploads), so a
seeded run reproduces the reference's perturbations; Dropout2d's per-(sample, channel) mask is
drawn with the CPU generator as well."""
import math
import os
import random
import time

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..utils import CLASSIFICATION, logger, cmd, tool
from ..nn import func
from ..nn.arena import EngineParallel
from ..nn.modules import Conv2d, PixelShuffle, upsample
from . import ssl_base
from ..task.sseg import func as sseg_func


def add_parser_arguments(parser):
    ssl_base.add_parser_arguments(parser)
    parser.add_argument('--cons-scale', type=float, default=-1)
    parser.add_argument('--cons-rampup-epochs', type=int, default=-1)
    parser.add_argument('--ad-lr-scale', type=float, default=-1)
    parser.add_argument('--vat-dec-num', type=int, default=0)
    parser.add_argument('--vat-dec-xi', type=float, default=1e-6)
    parser.add_argument('--vat-dec-eps', type=float, default=2.0)
    parser.add_argument('--drop-dec-num', type=int, default=0)
    parser.add_argument('--drop-dec-rate', type=float, default=0.5)
    parser.add_argument('--drop-dec-spatial', type=cmd.str2bool, default=True)
    parser.add_argument('--cut-dec-num', type=int, default=0)
    parser.add_argument('--cut-dec-erase', type=float, default=0.4)
    parser.add_argument('--context-dec-num', type=int, default=0)
    parser.add_argument('--object-dec-num', type=int, default=0)
    parser.add_argument('--fn-dec-num', type=int, default=0)
    parser.add_argument('--fn-dec-uniform', type=float, default=0.3)
    parser.add_argument('--fd-dec-num', type=int, default=0)


def ssl_cct(args, model_dict, optimizer_dict, lrer_dict, criterion_dict, task_func):
    ssl_base.check_single_model_dicts('ssl_cct', model_dict, optimizer_dict, lrer_dict, criterion_dict)
    algorithm = SSLCCT(args)
    algorithm.build([model_dict['model']], [optimizer_dict['model']], [lrer_dict['model']],
                    [criterion_dict['model']], task_func)
    return algorithm


# ------------------------------------------------------------------------------------------------
# decoder building blocks (ssl_cct.py:501-539; shared with the PSPNet head, _pspnet.py:15-54)
# ------------------------------------------------------------------------------------------------

def _nearest_mask(mask_full, size):
    """F.interpolate(mask, size, mode='nearest') of a [n,1,H,W] {0,1} mask (small, torch op)."""
    return F.interpolate(mask_full, size=size, mode='nearest')


class _Decoder(nn.Module):
    def __init__(self, upscale, in_channels, num_classes):
        super().__init__()
        self.upscale = upscale
        self.upsample = upsample(in_channels, num_classes, upscale=upscale)


class VATDecoder(_Decoder):
    """ssl_cct.py:542-582.  d(KL(p || softmax(f(x + xi d)))) / d d is back-propagated through the
    decoder with the analytic logit gradient (softmax(f) - p) / B, one power iteration."""

    def __init__(self, upscale, in_channels, num_classes, xi=1e-1, eps=10.0, iterations=1):
        super().__init__(upscale, in_channels, num_classes)
        self.xi, self.eps, self.it = xi, eps, iterations

    @staticmethod
    def _l2_normalize(d):
        norm = torch.norm(d.reshape(d.shape[0], -1), dim=1).view(-1, 1, 1, 1)
        return d / (norm + 1e-8)

    def get_r_adv(self, x):
        x_detached = x.detach()
        with torch.no_grad():
            pred = ops.softmax_planar(ops.nhwc_to_planar(self.upsample(x_detached), self._nc()))
        d = torch.rand(x.shape).sub(0.5).to(x.device).contiguous(memory_format=ops.CL)       # CPU draw, like the reference
        d = self._l2_normalize(d)
        for _ in range(self.it):
            d = d.detach().requires_grad_(True)
            with torch.enable_grad():
                pred_hat = ops.nhwc_to_planar(self.upsample(x_detached + self.xi * d), self._nc())
                g_logits = (ops.softmax_planar(pred_hat.detach()) - pred) / pred.shape[0]     # d KL(batchmean) / d logits
                (grad_d,) = torch.autograd.grad(pred_hat, d, grad_outputs=g_logits)
            d = self._l2_normalize(grad_d)
        return d * self.eps

    def _nc(self):
        return self.upsample[0].out_channels

    def forward(self, x, pred_of_main_decoder=None):
        params = list(self.upsample.parameters())
        flags = [p.requires_grad for p in params]
        for p in params:
            p.requires_grad_(False)          # the reference discards these gradients (decoder.zero_grad())
        try:
            r_adv = self.get_r_adv(x)
        finally:
            for p, f in zip(params, flags):
                p.requires_grad_(f)
        return self.upsample(x + r_adv)


class DropOutDecoder(_Decoder):
    def __init__(self, upscale, in_channels, num_classes, drop_rate=0.3, spatial_dropout=True):
        super().__init__(upscale, in_channels, num_classes)
        self.p, self.spatial = drop_rate, spatial_dropout

    def forward(self, x, pred_of_main_decoder=None):
        if not self.training:
            return self.upsample(x)
        n, c, h, w = x.shape
        if self.spatial:         # nn.Dropout2d: one Bernoulli(1-p) per (sample, channel), scaled by 1/(1-p)
            scale = (torch.empty(n, c, 1, 1).bernoulli_(1 - self.p) / (1 - self.p)).view(n, c).to(x.device)
            return self.upsample(ops.perturb(x, chan_scale=scale))
        mask = (torch.empty(n, c, h, w).bernoulli_(1 - self.p) / (1 - self.p)).to(x.device)
        return self.upsample(x * mask.contiguous(memory_format=ops.CL))


class CutOutDecoder(_Decoder):
    def __init__(self, upscale, in_channels, num_classes, erase=0.4):
        super().__init__(upscale, in_channels, num_classes)
        self.erase = erase

    def guided_cutout(self, output, resize):
        """ssl_cct.py:604-651: host contours (cv2) of argmax>0, one random box per long contour."""
        import cv2
        masks = ops.argmax_nonzero_mask(output)[:, 0]
        masks_np = []
        for mask in masks:
            mask_np = np.uint8(mask.cpu().numpy())
            mask_ones = np.ones_like(mask_np)
            found = cv2.findContours(mask_np, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)
            contours = found[0] if len(found) == 2 else found[1]
            polys = [c.reshape(c.shape[0], c.shape[-1]) for c in contours if c.shape[0] > 50]
            for poly in polys:
                min_w, max_w = poly[:, 0].min(), poly[:, 0].max()
                min_h, max_h = poly[:, 1].min(), poly[:, 1].max()
                bb_w, bb_h = max_w - min_w, max_h - min_h
                rnd_start_w = random.randint(0, int(bb_w * (1 - self.erase)))
                rnd_start_h = random.randint(0, int(bb_h * (1 - self.erase)))
                h_start, h_end = min_h + rnd_start_h, min_h + rnd_start_h + int(bb_h * self.erase)
                w_start, w_end = min_w + rnd_start_w, min_w + rnd_start_w + int(bb_w * self.erase)
                mask_ones[h_start:h_end, w_start:w_end] = 0
            masks_np.append(mask_ones)
        maskcut = torch.from_numpy(np.stack(masks_np)).float().unsqueeze_(1)
        return _nearest_mask(maskcut, resize).to(output.device)

    def forward(self, x, pred_of_main_decoder=None):
        maskcut = self.guided_cutout(pred_of_main_decoder, (x.size(2), x.size(3)))
        return self.upsample(ops.perturb(x, pixel_mask=maskcut))


class ContextMaskingDecoder(_Decoder):
    def forward(self, x, pred_of_main_decoder=None):
        m = _nearest_mask(ops.argmax_nonzero_mask(pred_of_main_decoder), (x.size(2), x.size(3)))
        return self.upsample(ops.perturb(x, pixel_mask=m))


class ObjectMaskingDecoder(_Decoder):
    def forward(self, x, pred_of_main_decoder=None):
        m = _nearest_mask(ops.argmax_nonzero_mask(pred_of_main_decoder), (x.size(2), x.size(3)))
        return self.upsample(ops.perturb(x, pixel_mask=1 - m))


class FeatureDropDecoder(_Decoder):
    def forward(self, x, pred_of_main_decoder=None):
        attention = ops.channel_mean(ops.as_cl(x.detach()))
        max_val = attention.view(x.size(0), -1).max(dim=1, keepdim=True)[0]
        threshold = (max_val * np.random.uniform(0.7, 0.9)).view(x.size(0), 1, 1, 1)
        drop_mask = (attention < threshold).float()
        return self.upsample(ops.perturb(x, pixel_mask=drop_mask))


class FeatureNoiseDecoder(_Decoder):
    def __init__(self, upscale, in_channels, num_classes, uniform_range=0.3):
        super().__init__(upscale, in_channels, num_classes)
        self.uni_dist = torch.distributions.uniform.Uniform(-uniform_range, uniform_range)

    def forward(self, x, pred_of_main_decoder=None):
        noise = self.uni_dist.sample(x.shape[1:]).to(x.device)         # [C,H,W], CPU draw, shared over the batch
        return self.upsample(ops.perturb(x, elem_noise=noise))


class WrappedCCTModel(nn.Module):
    """ssl_cct.py:422-491."""

    def __init__(self, args, main_model, auxiliary_decoders, task_criterion):
        super().__init__()
        self.args = args
        self.main_model = main_model
        self.auxiliary_decoders = auxiliary_decoders
        self.task_criterion = task_criterion
        self.param_groups = self.main_model.param_groups + \
            [{'params': list(self.auxiliary_decoders.parameters()), 'lr': self.args.lr * self.args.ad_lr_scale}]

    def forward(self, inp, gt, is_unlabeled):
        resulter, debugger = {}, {}
        m_resulter, _ = self.main_model.forward(inp)
        if 'pred' not in m_resulter or 'activated_pred' not in m_resulter:
            logger.log_err('In SSL_CCT, the \'resulter\' dict returned by the task model should contain \'pred\' and '
                           '\'activated_pred\'\n')
        resulter['pred'] = tool.dict_value(m_resulter, 'pred')
        resulter['activated_pred'] = tool.dict_value(m_resulter, 'activated_pred')
        if not len(resulter['pred']) == len(resulter['activated_pred']) == 1:
            logger.log_err('This implementation of SSL_CCT only support the task model with only one prediction\n')
        resulter['task_loss'] = None if is_unlabeled else torch.mean(self.task_criterion.forward(resulter['pred'], gt, inp))
        if is_unlabeled and self.args.unlabeled_batch_size > 0:
            if 'sslcct_ad_inp' not in m_resulter:
                logger.log_err('In SSL_CCT, the \'resulter\' dict returned by the task model should contain the key '
                               '\'sslcct_ad_inp\'\n')
            ul_ad_inp = tool.dict_value(m_resulter, 'sslcct_ad_inp')
            ul_main_pred = resulter['pred'][0].detach()
            ul_ad_gt = resulter['activated_pred'][0].detach()
            size = ul_ad_gt.shape[2:]
            nc = ul_ad_gt.shape[1]
            ul_ad_preds, cons = [], 0
            for ad in self.auxiliary_decoders:
                low = ad.forward(ul_ad_inp, pred_of_main_decoder=ul_main_pred)        # NHWC, nc real lanes
                ul_ad_preds.append(low)
                logits = ops.bilinear(low, size, align_corners=False, channels=nc, nhwc=True)
                cons = cons + ops.softmax_mse(logits, ul_ad_gt, 1.0)                  # MSELoss(softmax(pred), target)
            resulter['ul_ad_preds'] = ul_ad_preds
            resulter['cons_loss'] = torch.mean(cons) / len(ul_ad_preds)
        else:
            resulter['ul_ad_preds'] = None
            resulter['cons_loss'] = None
        return resulter, debugger


class SSLCCT(ssl_base._SSLBase):
    NAME = 'ssl_cct'
    SUPPORTED_TASK_TYPES = [CLASSIFICATION]

    def __init__(self, args):
        super().__init__(args)
        a = self.args
        if a.unlabeled_batch_size > 0:
            if a.cons_scale < 0:
                logger.log_err('The argument - cons_scale - is not set (or invalid)\n')
            elif a.cons_rampup_epochs < 0:
                logger.log_err('The argument - cons_rampup_epochs - is not set (or invalid)\n')
            if a.ad_lr_scale < 0:
                logger.log_err('The argument - ad_lr_scale - is not set (or invalid)\n')
        else:
            a.ad_lr_scale = 0

    def _build(self, model_funcs, optimizer_funcs, lrer_funcs, criterion_funcs, task_func):
        a = self.args
        self.task_func = task_func
        self.criterion = criterion_funcs[0](a)
        self.criterions = {'criterion': self.criterion, 'cons_criterion': ops.softmax_mse}
        self.main_model = model_funcs[0](args=a)
        arch = (a.models or {'model': 'deeplabv2'})['model']
        ad_in = sseg_func.CCT_AD_IN_CHANNELS[arch]                    # task/sseg/func.py:222-253
        up, nc = 8, a.num_classes
        decoders = [VATDecoder(up, ad_in, nc, xi=a.vat_dec_xi, eps=a.vat_dec_eps) for _ in range(a.vat_dec_num)]
        decoders += [DropOutDecoder(up, ad_in, nc, drop_rate=a.drop_dec_rate, spatial_dropout=a.drop_dec_spatial)
                     for _ in range(a.drop_dec_num)]
        decoders += [CutOutDecoder(up, ad_in, nc, erase=a.cut_dec_erase) for _ in range(a.cut_dec_num)]
        decoders += [ContextMaskingDecoder(up, ad_in, nc) for _ in range(a.context_dec_num)]
        decoders += [ObjectMaskingDecoder(up, ad_in, nc) for _ in range(a.object_dec_num)]
        decoders += [FeatureDropDecoder(up, ad_in, nc) for _ in range(a.fd_dec_num)]
        decoders += [FeatureNoiseDecoder(up, ad_in, nc, uniform_range=a.fn_dec_uniform) for _ in range(a.fn_dec_num)]
        self.auxiliary_decoders = nn.ModuleList(decoders)
        wrapped = WrappedCCTModel(a, self.main_model, self.auxiliary_decoders, self.criterion)
        self.model = EngineParallel(wrapped).cuda()        # where the reference has nn.DataParallel (ssl_cct.py:205)
        self.models = {'model': self.model}
        self.optimizer = optimizer_funcs[0](wrapped.param_groups)
        self.optimizers = {'optimizer': self.optimizer}
        self.lrer = lrer_funcs[0](self.optimizer)
        self.lrers = {'lrer': self.lrer}

    def train_step(self, inp, gt, cur_step, total_steps):
        a = self.args
        lbs = a.labeled_batch_size
        inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
        cons_rampup_scale = func.sigmoid_rampup(cur_step, total_steps)
        arena = self.model.arena
        arena.zero_grad()
        resulter, _ = self.model.forward(func.split_tensor_tuple(inp, 0, lbs), func.split_tensor_tuple(gt, 0, lbs), False)
        task_loss = tool.dict_value(resulter, 'task_loss', err=True).mean()
        self.meters.update('task_loss', task_loss.data)
        if a.unlabeled_batch_size > 0:
            resulter, _ = self.model.forward(func.split_tensor_tuple(inp, lbs, a.batch_size),
                                             func.split_tensor_tuple(gt, lbs, a.batch_size), True)
            cons_loss = cons_rampup_scale * a.cons_scale * tool.dict_value(resulter, 'cons_loss', err=True).mean()
            self.meters.update('cons_loss', cons_loss.data)
        else:
            cons_loss = 0
            self.meters.update('cons_loss', cons_loss)
        (task_loss + cons_loss).backward()
        arena.all_reduce_grads()
        arena.sgd_step(self.optimizer)

    def _train(self, data_loader, epoch):
        self.meters.reset()
        self.model.train()
        for idx, (inp, gt) in enumerate(ssl_base.device_prefetch(data_loader)):
            timer = time.time()
            cur_step = len(data_loader) * epoch + idx
            total_steps = len(data_loader) * self.args.cons_rampup_epochs
            self.train_step(inp, gt, cur_step, total_steps)
            self.meters.update('batch_time', time.time() - timer)
            if idx % self.args.log_freq == 0:
                self._log_step(lambda m, a=(epoch + 1, idx, len(data_loader), self.args.task): ('step: [{0}][{1}/{2}]\tbatch-time: {meters[batch_time]:.3f}\n'
                                '  task-{3}\t=>\ttask-loss: {meters[task_loss]:.6f}\tcons-loss: {meters[cons_loss]:.6f}\n'
                                ).format(*a, meters=m))
            if not self.args.is_epoch_lrer:
                self.lrer.step()
        if self.args.is_epoch_lrer:
            self.lrer.step()

    def _validate(self, data_loader, epoch):
        self.meters.reset()
        self.model.eval()
        for idx, (inp, gt) in enumerate(data_loader):
            inp, gt = ssl_base.to_device(inp), ssl_base.to_device(gt)
            resulter, _ = self.model.forward(inp, gt, False)
            self.meters.update('task_loss', tool.dict_value(resulter, 'task_loss', err=True).mean().data)
            self._metrics(resulter, gt, inp, 'task')
        self._log_validation_metrics(('task',))

    def _save_checkpoint(self, epoch):
        state = {'algorithm': self.NAME, 'epoch': epoch, 'model': self.model.state_dict(),
                 'optimizer': self.optimizer.state_dict(), 'lrer': self.lrer.state_dict()}
        torch.save(state, os.path.join(self.args.checkpoint_path, 'checkpoint_{0}.ckpt'.format(epoch)))

    def _load_checkpoint(self):
        checkpoint = torch.load(self.args.resume, weights_only=False)
        name = tool.dict_value(checkpoint, 'algorithm', default='unknown')
        if name != self.NAME:
            logger.log_err('Unmatched SSL algorithm format in checkpoint => required: {0} - given: {1}\n'
                           .format(self.NAME, name))
        self.model.load_state_dict(checkpoint['model'])
        self.optimizer.load_state_dict(checkpoint['optimizer'])
        self.model.arena.adopt_optimizer_state(self.optimizer)
        self.lrer.load_state_dict(checkpoint['lrer'])
        return checkpoint['epoch']
