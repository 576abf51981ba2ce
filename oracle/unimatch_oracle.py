"""Functional torch restatement of the UniMatch step (pixelssl_b200/ssl_algorithm/ssl_unimatch.py) for DeepLab-v2 or
DeepLabV3+, on the CPU or any device, in fp32 or fp64.  TEST INFRASTRUCTURE ONLY.

UniMatch (Yang et al., CVPR 2023) post-dates PixelSSL, so there is no reference run to generate goldens from; the
tests evaluate this oracle on the fly.  The forwards, criterion, poly LR and SGD are ``sseg_oracle``'s and
``deeplabv3plus_oracle``'s; the strong augmentation is torchvision's float-tensor functional ops
(``torchvision.transforms.v2.functional``) driven by the parameter table the engine draws
(``ssl_unimatch.draw_strong_params``); the Dropout2d factors are inputs too."""
import torch
import torch.nn.functional as F

from . import deeplabv3plus_oracle as D
from . import sseg_oracle as O

MEAN = (0.485, 0.456, 0.406)          # the input pipeline's normalisation (task/sseg/gpu_input.py)
STD = (0.229, 0.224, 0.225)


# ---- strong augmentation ---------------------------------------------------------------------------------------------

def colour_view(x01, row):
    """One view before the paste, in [0, 1] space: ColorJitter in the row's order, grayscale, Gaussian blur."""
    import torchvision.transforms.v2.functional as TF
    x = x01
    if row[0] != 0:
        for op in (int(v) for v in row[5:9]):
            if op == 0:
                x = TF.adjust_brightness(x, float(row[1]))
            elif op == 1:
                x = TF.adjust_contrast(x, float(row[2]))
            elif op == 2:
                x = TF.adjust_saturation(x, float(row[3]))
            else:
                x = TF.adjust_hue(x, float(row[4]))
    if row[9] != 0:
        x = TF.rgb_to_grayscale(x, num_output_channels=3)
    k = int(row[10])
    if k > 0:
        x = TF.gaussian_blur(x, kernel_size=[2 * k + 1, 2 * k + 1], sigma=[float(row[11])] * 2)
    return x


def strong_views(weak, table):
    """weak [ubs,3,H,W] normalised images, table [2*ubs,32] (numpy or tensor) -> [2*ubs,3,H,W] normalised views: view
    k of image i at row k*ubs + i, the box of row v filled from view k of image (i + ubs/2) mod ubs before its own
    paste."""
    table = torch.as_tensor(table, dtype=torch.float64)
    ubs = weak.shape[0]
    mean = torch.tensor(MEAN, dtype=weak.dtype, device=weak.device).view(3, 1, 1)
    std = torch.tensor(STD, dtype=weak.dtype, device=weak.device).view(3, 1, 1)
    x01 = (weak * std + mean).clamp(0, 1)
    pre = [colour_view(x01[v % ubs], table[v]) for v in range(2 * ubs)]
    out = []
    for v in range(2 * ubs):
        x = pre[v].clone()
        y0, x0, y1, x1 = (int(t) for t in table[v, 12:16])
        k, i = divmod(v, ubs)
        x[:, y0:y1, x0:x1] = pre[k * ubs + (i + ubs // 2) % ubs][:, y0:y1, x0:x1]
        out.append((x - mean) / std)
    return torch.stack(out)


# ---- the loss --------------------------------------------------------------------------------------------------------

def pseudo_labels(logits):
    """-> (label, confidence): the first maximal index of the logits and the largest softmax probability."""
    return logits.argmax(1), F.softmax(logits, dim=1).amax(1)


def box_masks(boxes, ubs, h, w):
    m = torch.zeros(2 * ubs, h, w, dtype=torch.bool)
    for v, (y0, x0, y1, x1) in enumerate(torch.as_tensor(boxes).tolist()):
        m[v, y0:y1, x0:x1] = True
    return m


def unimatch_terms(w, mix, s, pred_fp, boxes, tau):
    """-> (L_s1, L_s2, L_fp, confident count) of ops.unimatch_cross_entropy: w [ubs] weak logits, mix [ubs] the box
    source before the roll by ubs/2, s [2*ubs] strong logits, pred_fp [ubs] FP logits of the unlabeled rows."""
    ubs, _, h, wd = w.shape
    lab, conf = pseudo_labels(w.detach())
    lab_m, conf_m = pseudo_labels(torch.roll(mix.detach(), ubs // 2, 0))
    inside = box_masks(boxes, ubs, h, wd).to(w.device)
    n = ubs * h * wd
    out = []
    for k in range(2):
        b = inside[k * ubs:(k + 1) * ubs]
        y, c = torch.where(b, lab_m, lab), torch.where(b, conf_m, conf)
        ce = F.cross_entropy(s[k * ubs:(k + 1) * ubs], y, reduction='none')
        out.append((ce * (c >= tau).to(ce.dtype)).sum() / n)
    ce = F.cross_entropy(pred_fp, lab, reduction='none')
    out.append((ce * (conf >= tau).to(ce.dtype)).sum() / n)
    out.append((conf >= tau).sum())
    return tuple(out)


# ---- forwards --------------------------------------------------------------------------------------------------------

def _drop(x, scale):
    return torch.cat([x, x * scale.to(device=x.device, dtype=x.dtype)[:, :, None, None]])


def deeplabv2_forward_fp(img, st, scales, output_stride=16, blocks=O.R101_BLOCKS):
    n = img.shape[0]
    latent = O.resnet_forward(img, st, True, output_stride, blocks)
    up = O.bilinear_align_corners(O.aspp_classifier(_drop(latent, scales[0]), st), img.shape[2:])
    return up[:n], up[n:]


def deeplabv3plus_forward_fp(img, st, scales, output_stride=16, blocks=O.R101_BLOCKS):
    n = img.shape[0]
    low, latent = D.backbone_forward(img, st, True, output_stride, blocks)
    a = D.aspp(_drop(latent, scales[1]), st, True, D.ASPP_RATES[output_stride])
    low = _drop(low, scales[0])
    r = D._cbr(low, st, 'decoder.reduce.0', 'decoder.reduce.1', True)
    x = torch.cat([F.interpolate(a, size=low.shape[2:], mode='bilinear', align_corners=True), r], dim=1)
    x = D._cbr(x, st, 'decoder.fuse.0', 'decoder.fuse.1', True, padding=1)
    x = D._cbr(x, st, 'decoder.fuse.3', 'decoder.fuse.4', True, padding=1)
    x = F.conv2d(x, st['classifier.weight'], st['classifier.bias'])
    up = F.interpolate(x, size=img.shape[2:], mode='bilinear', align_corners=True)
    return up[:n], up[n:]


MODELS = {'deeplabv2': (O.deeplabv2_forward, deeplabv2_forward_fp, O.deeplabv2_param_shapes, O.lr_multipliers),
          'deeplabv3plus': (D.forward, deeplabv3plus_forward_fp, D.param_shapes, D.lr_multipliers)}


class UniMatchOracle:
    """One task-model state (dict name -> tensor) with its SGD momentum buffers and PolynomialLR counter."""

    def __init__(self, state, model='deeplabv2', lr=2.5e-4, momentum=0.9, weight_decay=5e-4, max_iters=1000,
                 power=0.9, threshold=0.95, scale=1.0, rampup_steps=0, num_classes=21, output_stride=16,
                 blocks=O.R101_BLOCKS, ignore_index=255):
        self.forward, self.forward_fp, shapes, mult = MODELS[model]
        self.state = state
        self.names = [n for n, _, _ in shapes(num_classes, output_stride, blocks)]
        self.mult = mult(self.names)
        self.base_lr, self.momentum, self.wd = lr, momentum, weight_decay
        self.max_iters, self.power = max_iters, power
        self.cur_iter = 1            # _LRScheduler.__init__ already stepped once (lrer.py:152)
        self.tau, self.scale, self.rampup_steps = threshold, scale, rampup_steps
        self.os, self.blocks, self.ignore = output_stride, blocks, ignore_index
        self.bufs = [torch.zeros_like(state[n]) for n in self.names]
        self.step_idx = 0

    def mix_source(self, u_w):
        """The eval-mode logits of the weak view (before the roll)."""
        with torch.no_grad():
            return self.forward(u_w, self.state, False, self.os, self.blocks)[0]

    def step(self, img, gt, lbs, table, boxes, fp_scales, strong=None):
        """One step.  table / boxes: ``ssl_unimatch.draw_strong_params``; fp_scales: the Dropout2d factors, one
        [lbs+ubs, C] tensor per perturbed feature map; strong: the strong views [2*ubs,3,H,W] to use instead of
        computing them from the table.  Returns the losses, the mask ratio and the gradients (``grads``)."""
        st = self.state
        ubs = img.shape[0] - lbs
        for n in self.names:
            st[n].requires_grad_(True)
            st[n].grad = None
        ramp = O.sigmoid_rampup(self.step_idx, self.rampup_steps)
        u_w = img[lbs:]
        mix = self.mix_source(u_w)
        if strong is None:
            strong = strong_views(u_w, table)
        strong = strong.to(img.dtype)
        pred, pred_fp = self.forward_fp(img, st, fp_scales, self.os, self.blocks)
        pred_s = self.forward(strong, st, True, self.os, self.blocks)[0]
        task = O.sseg_criterion(pred[:lbs], gt[:lbs], self.ignore).mean()
        l_s1, l_s2, l_fp, count = unimatch_terms(pred[lbs:], mix, pred_s, pred_fp[lbs:], boxes, self.tau)
        s = ramp * self.scale
        loss = 0.5 * (task + s * (0.25 * l_s1 + 0.25 * l_s2 + 0.5 * l_fp))
        loss.backward()
        out = {'task_loss': task.detach(), 's1_loss': l_s1.detach(), 's2_loss': l_s2.detach(),
               'fp_loss': l_fp.detach(), 'mask_ratio': float(count) / (ubs * img.shape[2] * img.shape[3]),
               'pred_u': pred[lbs:].detach()}
        lrs = [O.poly_lr(self.base_lr * m, self.cur_iter, self.max_iters, self.power) for m in self.mult]
        grads = [st[n].grad for n in self.names]
        out['grads'] = {n: g.detach().clone() for n, g in zip(self.names, grads)}
        with torch.no_grad():
            for n in self.names:
                st[n].requires_grad_(False)
            O.sgd_momentum_step([st[n] for n in self.names], grads, self.bufs, lrs, self.momentum, self.wd,
                                first_step=(self.step_idx == 0))
        self.cur_iter += 1
        self.step_idx += 1
        return out
