"""TaskFunc hooks used inside the training step (task/sseg/func.py:134-253) and the validation
``metrics`` (task/sseg/func.py:36-80).  ``visualize`` (PIL colourisation to disk) stays with the
reference."""
import numpy as np
import torch

from ... import ops


# channels of each task model's ``resulter['sslcct_ad_inp']``
CCT_AD_IN_CHANNELS = {'pspnet': 512, 'deeplabv2': 2048, 'deeplabv3plus': 2048}


def task_func():
    return SemanticSegmentationFunc


class SemanticSegmentationFunc:
    METRIC_STR = 'metric'

    def __init__(self, args):
        self.args = args

    def metrics(self, pred, gt, inp, meters, id_str=''):
        """Confusion matrix of this batch on the device (``pxl_confusion_matrix``; the reference moves
        the whole probability map to the host and uses np.argmax/np.bincount, func.py:39-47); only the
        C x C int64 matrix crosses PCIe.  acc / acc-class / mIoU / fwIoU are the reference's formulas
        on the meter's running sum (func.py:64-80)."""
        assert len(pred) == len(gt) == 1
        nc = self.args.num_classes
        cmat = torch.zeros((nc, nc), dtype=torch.int64, device=pred[0].device)
        ops.confusion_matrix_(cmat, pred[0].detach().contiguous(), gt[0].detach().contiguous(), nc)
        confusion_matrix = cmat.cpu().numpy()
        meters.update('{0}_confusion_matrix'.format(id_str), confusion_matrix)

        names = {k: '{0}_{1}_{2}'.format(id_str, self.METRIC_STR, k) for k in ('acc', 'acc-class', 'mIoU', 'fwIoU')}
        for name in names.values():
            if meters.has_key(name):
                meters.reset(name)
        values = summarize_confusion_matrix(meters['{0}_confusion_matrix'.format(id_str)].sum)
        for k, name in names.items():
            meters.update(name, values[k])

    def _arch(self, hook):
        arch = (self.args.models or {'model': 'deeplabv2'})['model']
        if arch not in CCT_AD_IN_CHANNELS:
            from ...utils import logger
            logger.log_err('In the SSL_CCT algorithm, the task model \'{0}\' is not supported by the hook \'{1}\'\n'
                           .format(arch, hook))
        return arch

    def sslcct_ad_in_channels(self):
        """Channels of ``resulter['sslcct_ad_inp']`` (task/sseg/func.py:222-236): the PSP feature for pspnet, the
        backbone latent for deeplabv2 and deeplabv3plus."""
        return CCT_AD_IN_CHANNELS[self._arch('sslcct_ad_in_channels')]

    def sslcct_ad_out_channels(self):
        return self.args.num_classes

    def sslcct_ad_upsample_scale(self):
        self._arch('sslcct_ad_upsample_scale')
        return 8

    def ssls4l_rc_in_channels(self):
        return self.args.num_classes

    def sslgct_fd_in_channels(self):
        return self.args.num_classes + 3

    def ssladv_fcd_in_channels(self):
        return self.args.num_classes


def summarize_confusion_matrix(cmat_sum):
    """acc, acc-class, mIoU, fwIoU of an accumulated confusion matrix (rows = gt), func.py:64-80;
    0/0 classes are skipped through nanmean exactly like the reference."""
    cmat_sum = np.asarray(cmat_sum)
    diag = np.diag(cmat_sum)
    with np.errstate(divide='ignore', invalid='ignore'):
        acc = diag.sum() / cmat_sum.sum()
        acc_class = np.nanmean(diag / cmat_sum.sum(axis=1))
        iou = diag / (np.sum(cmat_sum, axis=1) + np.sum(cmat_sum, axis=0) - diag)
        miou = np.nanmean(iou)
        freq = np.sum(cmat_sum, axis=1) / np.sum(cmat_sum)
        fwiou = (freq[freq > 0] * iou[freq > 0]).sum()
    return {'acc': acc, 'acc-class': acc_class, 'mIoU': miou, 'fwIoU': fwiou}
