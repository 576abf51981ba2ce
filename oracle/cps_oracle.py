"""Functional torch restatement of the Cross Pseudo Supervision step (pixelssl_b200/ssl_algorithm/ssl_cps.py) for
DeepLab-v2 or DeepLabV3+, on the CPU or any device, in fp32 or fp64.  TEST INFRASTRUCTURE ONLY.

CPS (Chen et al., CVPR 2021) post-dates PixelSSL, so there is no reference run to generate goldens from; the tests
evaluate this oracle on the fly.  Every piece but the CPS term is ``sseg_oracle``'s (forwards, criterion, box masks,
mix, poly LR, SGD); the CPS term is ``F.cross_entropy(s_l, t_r.argmax(1))`` and the symmetric one."""
import torch
import torch.nn.functional as F

from . import deeplabv3plus_oracle as D
from . import sseg_oracle as O

MODELS = {'deeplabv2': (O.deeplabv2_forward, O.deeplabv2_param_shapes, O.lr_multipliers),
          'deeplabv3plus': (D.forward, D.param_shapes, D.lr_multipliers)}


def cps_term(s, t):
    """Cross-entropy of logits ``s`` against the per-pixel argmax of ``t`` (detached), mean over every pixel of every
    sample.  torch's argmax takes the first maximal index."""
    return F.cross_entropy(s, t.detach().argmax(1))


class CPSOracle:
    """Two task-model states (dict name -> tensor) with their own SGD momentum buffers and a shared PolynomialLR
    iteration counter (both lrers step together)."""

    def __init__(self, l_state, r_state, model='deeplabv2', lr=2.5e-4, momentum=0.9, weight_decay=5e-4,
                 max_iters=1000, power=0.9, cps_scale=1.5, rampup_steps=0, cutmix=False, mask_prop_range=(0.5, 0.5),
                 num_classes=21, output_stride=16, blocks=O.R101_BLOCKS, ignore_index=255):
        self.forward, shapes, mult = MODELS[model]
        self.states = [l_state, r_state]
        self.names = [n for n, _, _ in shapes(num_classes, output_stride, blocks)]
        self.mult = mult(self.names)
        self.base_lr, self.momentum, self.wd = lr, momentum, weight_decay
        self.max_iters, self.power = max_iters, power
        self.cur_iter = 1            # _LRScheduler.__init__ already stepped once (lrer.py:152)
        self.cps_scale, self.rampup_steps = cps_scale, rampup_steps
        self.cutmix, self.prop = cutmix, mask_prop_range
        self.os, self.blocks, self.ignore = output_stride, blocks, ignore_index
        self.bufs = [[torch.zeros_like(st[n]) for n in self.names] for st in self.states]
        self.step_idx = 0

    def _fwd(self, img, st):
        return self.forward(img, st, True, self.os, self.blocks)[0]

    def _task(self, logits, gt):
        return O.sseg_criterion(logits, gt, self.ignore).mean()

    def step(self, img, gt, lbs, rng=None):
        """One step; ``rng`` (a numpy RandomState) draws the CutMix box masks.  Returns the four losses and both
        models' gradients (``l_grads`` / ``r_grads``: name -> tensor)."""
        ubs = img.shape[0] - lbs
        for st in self.states:
            for n in self.names:
                st[n].requires_grad_(True)
                st[n].grad = None
        ramp = O.sigmoid_rampup(self.step_idx, self.rampup_steps)
        if not self.cutmix:
            logits = [self._fwd(img, st) for st in self.states]
            task = [self._task(lg[:lbs], gt[:lbs]) for lg in logits]
            students = targets = logits
        else:
            task = [self._task(self._fwd(img[:lbs], st), gt[:lbs]) for st in self.states]
            if ubs > 0:
                half = ubs // 2
                masks, _ = O.box_masks(rng, half, tuple(img.shape[2:]), prop_range=self.prop)
                mask = torch.from_numpy(masks).to(device=img.device, dtype=img.dtype)
                mix_inp = O.cutmix_mix(mask, img[lbs:lbs + half], img[lbs + half:lbs + ubs])
                with torch.no_grad():
                    u = [self._fwd(img[lbs:lbs + ubs], st) for st in self.states]
                    targets = [O.cutmix_mix(mask, x[:half], x[half:ubs]) for x in u]
                students = [self._fwd(mix_inp, st) for st in self.states]
        out = {'l_task_loss': task[0].detach(), 'r_task_loss': task[1].detach()}
        loss = task[0] + task[1]
        if ubs > 0:
            l_cps = ramp * self.cps_scale * cps_term(students[0], targets[1])
            r_cps = ramp * self.cps_scale * cps_term(students[1], targets[0])
            out['l_cps_loss'], out['r_cps_loss'] = l_cps.detach(), r_cps.detach()
            loss = loss + l_cps + r_cps
        else:
            out['l_cps_loss'] = out['r_cps_loss'] = torch.zeros((), dtype=img.dtype)
        loss.backward()
        lrs = [O.poly_lr(self.base_lr * m, self.cur_iter, self.max_iters, self.power) for m in self.mult]
        for side, st, bufs in (('l', self.states[0], self.bufs[0]), ('r', self.states[1], self.bufs[1])):
            grads = [st[n].grad for n in self.names]
            out[side + '_grads'] = {n: g.detach().clone() for n, g in zip(self.names, grads)}
            with torch.no_grad():
                for n in self.names:
                    st[n].requires_grad_(False)
                O.sgd_momentum_step([st[n] for n in self.names], grads, bufs, lrs, self.momentum, self.wd,
                                    first_step=(self.step_idx == 0))
        self.cur_iter += 1
        self.step_idx += 1
        return out
