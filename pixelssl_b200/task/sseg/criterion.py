"""Criterion plugin: CommonSSEGCriterion (task/sseg/criterion.py:18-38) on the fused CE kernel, and the OHEM
cross-entropy (``ohem_sseg_criterion``) on the OHEM kernels."""
import math

import torch.nn as nn

from ... import ops
from ...utils import logger

OHEM_CRITERIONS = ['ohem_sseg_criterion']


def add_parser_arguments(parser):
    pass


def add_ohem_parser_arguments(parser):
    """The flags of ``ohem_sseg_criterion``; added only where a configuration uses it, so the default parser stays
    PixelSSL's."""
    parser.add_argument('--ohem-thresh', type=float, default=0.7,
                        help='OHEM probability threshold: pixels whose target probability is at most this are kept')
    parser.add_argument('--ohem-min-kept', type=int, default=200000,
                        help='OHEM: at least this many pixels of the batch are kept (0 keeps every valid pixel)')


def sseg_criterion():
    return CommonSSEGCriterion


def ohem_sseg_criterion():
    return OHEMSSEGCriterion


def _check_single(pred, gt, inp):
    if len(pred) != 1 or len(gt) != 1 or len(inp) != 1:
        logger.log_err('DeepLab criterion for semantic segmentation requires\t=>\t'
                       'len(pred) == 1 \t len(gt) == 1 \t len(inp) == 1\n')


class CommonSSEGCriterion(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.ignore_index = args.ignore_index

    def forward(self, pred, gt, inp, mean_upstream=None):
        """-> per-sample loss Tensor[n].  ``mean_upstream`` (engine-only, optional): 1/n when the
        caller's next op is ``torch.mean`` feeding the final loss directly, which lets the
        gradient be written by the forward kernel."""
        _check_single(pred, gt, inp)
        return ops.cross_entropy2d(pred[0], gt[0], self.ignore_index, upstream_const=mean_upstream)


class OHEMSSEGCriterion(nn.Module):
    """Online hard example mining cross-entropy (the probability OHEM of ProbOhemCrossEntropy2d): the mean CE over the
    pixels of the batch whose target probability is at most max(ohem_thresh, the ohem_min_kept-th smallest target
    probability).  ``forward`` returns per-sample values whose ``torch.mean`` is that loss, so every algorithm uses it
    as it uses ``sseg_criterion``.  Selection is per call, over the batch the call sees (each rank's under DDP)."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        self.ignore_index = args.ignore_index
        self.thresh = getattr(args, 'ohem_thresh', None)
        self.min_kept = getattr(args, 'ohem_min_kept', None)
        if self.thresh is None or self.min_kept is None:
            logger.log_err('ohem_sseg_criterion needs --ohem-thresh and --ohem-min-kept (register them with '
                           'add_ohem_parser_arguments)\n')
        if not math.isfinite(float(self.thresh)):
            logger.log_err('ohem_sseg_criterion: --ohem-thresh must be finite (got {0})\n'.format(self.thresh))
        if int(self.min_kept) < 0:
            logger.log_err('ohem_sseg_criterion: --ohem-min-kept must be >= 0 (got {0})\n'.format(self.min_kept))

    def forward(self, pred, gt, inp, mean_upstream=None):
        """-> per-sample loss Tensor[n] (see CommonSSEGCriterion.forward for ``mean_upstream``)."""
        _check_single(pred, gt, inp)
        return ops.ohem_cross_entropy2d(pred[0], gt[0], self.ignore_index, self.thresh, self.min_kept,
                                        upstream_const=mean_upstream)
