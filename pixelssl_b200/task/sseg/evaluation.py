"""Multi-view evaluation of a segmentation model: UniMatch's sliding window, multi-scale and flipped inference.

Validation normally makes one whole-image forward per model.  With ``--val-protocol``, ``--val-crop-size``,
``--val-scales`` and ``--val-flip`` the prediction becomes the ensemble over views (s, f): for s in the given scales,
f = False, then f = True if flipping.  Each view image is the batch resized by s (bilinear, align_corners=True, the
engine's convention) and flipped along W if f.  Its probability map is

  * ``whole``:   softmax(model(view));
  * ``sliding``: UniMatch's ``evaluate(mode='sliding_window')``: tiles of ``crop`` x ``crop`` clipped to the view,
    origins every int(2 crop / 3) pixels (rows r = 0, stride, ... while r < h, likewise the columns, tail tiles kept
    even where an earlier tile covers them), softmax(model(tile)) summed over the overlaps in row-major tile order.

The map is un-flipped, resized back to (H, W) (bilinear, align_corners=True) and summed over the views, S.  The
resulter then holds ``activated_pred`` = (S / V,) and ``pred`` = (log(max(S / V, FLT_MIN)),), so every algorithm's
validation loss is the NLL of the ensemble.

The multi-view path runs only inside ``_SSLBase.validate`` (the ``validating()`` scope), for a task model in eval mode,
when the protocol differs from the default (whole, scales [1.0], no flip); anywhere else the plain forward runs.

On the device each view takes one ``pxl_eval_tiles`` launch per tile shape (its tiles batched into one forward), one
``pxl_eval_merge``, one ``pxl_eval_view_add`` if s changes the size, and the batch one ``pxl_eval_finish``
(csrc/eval_views.cu).  All tile logits of a view are held at once."""
import contextlib
import itertools

import torch

from ... import ops
from ...utils import cmd, logger

PROTOCOLS = ('whole', 'sliding')
FLAGS = ('val_protocol', 'val_crop_size', 'val_scales', 'val_flip')
DEFAULTS = {'val_protocol': 'whole', 'val_crop_size': None, 'val_scales': [1.0], 'val_flip': False}


def add_val_protocol_parser_arguments(parser):
    """The flags of the multi-view evaluation; added only where a configuration uses them, so the default parser stays
    PixelSSL's."""
    parser.add_argument('--val-protocol', type=str, default='whole', choices=PROTOCOLS,
                        help='validation forward per view: the whole view, or the sliding window of --val-crop-size')
    parser.add_argument('--val-crop-size', type=int, default=None,
                        help='window size of the sliding-window validation (required for it, >= 2)')
    parser.add_argument('--val-scales', type=cmd.str2floatlist, default=[1.0],
                        help='validation scales, e.g. [0.75,1.0,1.25]')
    parser.add_argument('--val-flip', type=cmd.str2bool, default=False,
                        help='also validate on the horizontally flipped copy of every scale')


def settings(args):
    """-> (protocol, crop, scales, flip) of ``args``; an args namespace without the flags gives the defaults."""
    return (getattr(args, 'val_protocol', 'whole'), getattr(args, 'val_crop_size', None),
            [float(s) for s in getattr(args, 'val_scales', [1.0])], bool(getattr(args, 'val_flip', False)))


def is_default(args):
    protocol, _, scales, flip = settings(args)
    return protocol == 'whole' and scales == [1.0] and not flip


def check_args(args):
    """Fail through logger.log_err on an invalid protocol configuration."""
    protocol, crop, scales, flip = settings(args)
    if protocol not in PROTOCOLS:
        logger.log_err('--val-protocol must be one of {0} (got {1})\n'.format(PROTOCOLS, protocol))
    if protocol == 'sliding' and (crop is None or int(crop) < 2):
        logger.log_err('--val-protocol sliding needs --val-crop-size >= 2 (got {0})\n'.format(crop))
    if crop is not None and int(crop) < 2:
        logger.log_err('--val-crop-size must be >= 2 (got {0})\n'.format(crop))
    if not scales or not all(s > 0 for s in scales):      # also false for NaN
        logger.log_err('--val-scales must be a non-empty list of positive scales (got {0})\n'.format(scales))


_scope = {'depth': 0}


@contextlib.contextmanager
def validating():
    """The scope in which an eval-mode task model runs the multi-view protocol (``_SSLBase.validate`` sets it)."""
    _scope['depth'] += 1
    try:
        yield
    finally:
        _scope['depth'] -= 1


def multi_view(task_model):
    """Whether ``task_model.forward`` takes the multi-view path."""
    return _scope['depth'] > 0 and not task_model.training and not is_default(task_model.args)


# ---- views and tiles -----------------------------------------------------------------------------------------------

def views(scales, flip):
    """-> [(s, f)] in ensemble order."""
    return [(float(s), f) for s in scales for f in ((False, True) if flip else (False,))]


def view_size(H, W, s):
    """Size of the view at scale s: (int(H s + 0.5), int(W s + 0.5)), (H, W) itself at s = 1."""
    if s == 1.0:
        return H, W
    hv, wv = int(H * s + 0.5), int(W * s + 0.5)
    if hv < 1 or wv < 1:
        raise ValueError('scale {0} shrinks a {1}x{2} image to {3}x{4}'.format(s, H, W, hv, wv))
    return hv, wv


def window(length, protocol, crop):
    """-> (tile length, stride) along an axis of ``length`` view pixels."""
    if protocol == 'whole':
        return length, length
    return int(crop), int(int(crop) * 2 / 3)


def axis_classes(length, g, stride):
    """The tile classes along one axis: [(first origin, number of origins, tile length)]: the full-length tiles (if
    any), then each clipped tail tile.  Their order is the order of csrc/eval_views.cu."""
    origins = list(range(0, length, stride))
    full = [r for r in origins if r + g <= length]
    out = [(0, len(full), g)] if full else []
    out += [(r, 1, length - r) for r in origins[len(full):]]
    return out


def tile_groups(hv, wv, protocol, crop):
    """-> (gh, gw, sh, sw, groups) of a view: groups = [(r0, nr, c0, nc, th, tw)], one per tile shape, (row class,
    column class) row-class major."""
    gh, sh = window(hv, protocol, crop)
    gw, sw = window(wv, protocol, crop)
    groups = [(r0, nr, c0, nc, th, tw) for (r0, nr, th), (c0, nc, tw) in
              itertools.product(axis_classes(hv, gh, sh), axis_classes(wv, gw, sw))]
    return gh, gw, sh, sw, groups


def tiles(hv, wv, protocol, crop):
    """-> [(r, c, th, tw)] of a view in row-major tile order (UniMatch's loop order)."""
    gh, sh = window(hv, protocol, crop)
    gw, sw = window(wv, protocol, crop)
    return [(r, c, min(gh, hv - r), min(gw, wv - c)) for r in range(0, hv, sh) for c in range(0, wv, sw)]


def plan(H, W, protocol, crop, scales, flip):
    """-> [(s, f, hv, wv, tile_groups(...))] for a batch of H x W images."""
    out = []
    for s, f in views(scales, flip):
        hv, wv = view_size(H, W, s)
        out.append((s, f, hv, wv, tile_groups(hv, wv, protocol, crop)))
    return out


# ---- the driver ----------------------------------------------------------------------------------------------------

def evaluate_views(forward_fn, x, protocol='whole', crop=None, scales=(1.0,), flip=False):
    """The ensemble of ``forward_fn`` (planar images [m,3,h,w] -> planar logits [m,C,h,w]) over the views of the batch
    x [n,3,H,W] -> (S / V, log(max(S / V, FLT_MIN))), both [n,C,H,W].  No host synchronisation of its own."""
    ops._chk(x, 'x')
    n, _, H, W = x.shape
    steps = plan(H, W, protocol, crop, scales, flip)
    S = None
    for vi, (s, f, hv, wv, (gh, gw, sh, sw, groups)) in enumerate(steps):
        logits = []
        for r0, nr, c0, nc, th, tw in groups:
            lg = forward_fn(ops.eval_tiles(x, hv, wv, f, r0, nr, c0, nc, sh, sw, th, tw))
            if tuple(lg.shape[2:]) != (th, tw) or lg.shape[0] != nr * nc * n:
                raise ValueError('forward_fn returned {0} for {1} tiles of {2}x{3}'.format(
                    tuple(lg.shape), nr * nc * n, th, tw))
            logits.append(lg.contiguous())
        if S is None:
            S = torch.empty((n, logits[0].shape[1], H, W), dtype=torch.float32, device=x.device)
        if (hv, wv) == (H, W):
            ops.eval_merge(logits, n, hv, wv, gh, gw, sh, sw, f, out=S, accumulate=vi > 0)
        else:
            P = ops.eval_merge(logits, n, hv, wv, gh, gw, sh, sw, f)
            ops.eval_view_add(P, S, accumulate=vi > 0)
    return ops.eval_finish(S, len(steps))


def forward_views(task_model, inp):
    """The multi-view forward of a segmentation task model (``TaskModel.forward`` inside ``validating()``): the
    protocol of ``task_model.args`` around the plain forward of ``task_model.model`` -> (resulter, debugger)."""
    protocol, crop, scales, flip = settings(task_model.args)
    with torch.no_grad():
        mean, logmean = evaluate_views(lambda t: task_model.model(t)[0], inp[0].contiguous(), protocol, crop, scales,
                                       flip)
    resulter = {'pred': (logmean,), 'activated_pred': (mean,), 'ssls4l_rc_inp': logmean}
    return resulter, {}
