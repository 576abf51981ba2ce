"""Torch restatement of the OHEM cross-entropy (``ohem_sseg_criterion``, the probability OHEM of
ProbOhemCrossEntropy2d), on the CPU or any device, in fp32 or fp64.  TEST INFRASTRUCTURE ONLY.

PixelSSL has no OHEM criterion, so there is no reference run to generate goldens from; the tests evaluate this
oracle on the fly.  Over the whole batch of one call:
  * a pixel is valid when y = trunc(label) != ignore_index and 0 <= y < C; V = number of valid pixels;
  * q = softmax(logits)[y] on valid pixels, 1 on the others;
  * k == 0 or k > V (or V == 0): every valid pixel is kept; else t_k = torch.sort(q)[k-1] over all pixels (NaN last),
    T = t_k if t_k > thresh else thresh, and the valid pixels with q <= T are kept;
  * K = number of kept pixels; per_sample[i] = n * sum over image i's kept pixels of CE / K (NaN when K == 0)."""
import contextlib
import math

import torch
import torch.nn.functional as F

from . import sseg_oracle as O


def q_map(logits, gt, ignore_index=255):
    """-> (q [n,H,W], valid [n,H,W] bool, y [n,H,W] long with invalid labels replaced by 0)."""
    n, c, h, w = logits.shape
    y = gt.reshape(n, h, w).long()                  # truncation toward zero, as .long()
    valid = (y != ignore_index) & (y >= 0) & (y < c)
    y = torch.where(valid, y, torch.zeros_like(y))
    p = F.softmax(logits, dim=1).gather(1, y[:, None])[:, 0]
    q = torch.where(valid, p, torch.ones_like(p))
    return q, valid, y


def select(q, valid, thresh, min_kept):
    """-> dict V, K (ints), T, t_k (floats; T = inf when every valid pixel is kept, t_k NaN when not selected) and the
    kept mask."""
    V = int(valid.sum())
    k = int(min_kept)
    if V == 0 or k == 0 or k > V:
        return {'V': V, 'K': V, 'T': math.inf, 't_k': math.nan, 'kept': valid.clone()}
    t_k = torch.sort(q.flatten())[0][k - 1]
    T = t_k if bool(t_k > thresh) else torch.tensor(thresh, dtype=q.dtype)
    kept = valid & (q <= T)
    return {'V': V, 'K': int(kept.sum()), 'T': float(T), 't_k': float(t_k), 'kept': kept}


def ohem_criterion(logits, gt, ignore_index=255, thresh=0.7, min_kept=200000, return_selection=False):
    """Per-sample OHEM loss [n] (``torch.mean`` of it is the OHEM loss); differentiable in ``logits``; the selection
    is a constant."""
    n = logits.shape[0]
    q, valid, y = q_map(logits.detach(), gt, ignore_index)
    sel = select(q, valid, thresh, min_kept)
    nll = F.cross_entropy(logits, y, reduction='none')
    per = n * torch.where(sel['kept'], nll, torch.zeros_like(nll)).sum(dim=(1, 2)) / sel['K']
    return (per, q, sel) if return_selection else per


def criterion(thresh, min_kept):
    """``ohem_criterion`` with fixed hyper-parameters, in ``sseg_oracle.sseg_criterion``'s signature."""
    def crit(logits, gt, ignore_index=255):
        return ohem_criterion(logits, gt, ignore_index, thresh, min_kept)
    return crit


@contextlib.contextmanager
def supervised_criterion(crit):
    """Run the step oracles (``sseg_oracle.MTOracle``, ``cps_oracle.CPSOracle``, ``unimatch_oracle.UniMatchOracle``),
    which look ``sseg_oracle.sseg_criterion`` up at each call, with ``crit`` as their supervised criterion."""
    saved = O.sseg_criterion
    O.sseg_criterion = crit
    try:
        yield
    finally:
        O.sseg_criterion = saved
