"""Multi-view evaluation restated as a plain torch loop (task/sseg/evaluation.py has the semantics): views (s, f) in
scale order, each view image resized (bilinear, align_corners=True) and flipped, its probability map from one whole
forward or UniMatch's sliding window (tiles every int(2 crop / 3) pixels, clipped to the view, softmax added in
row-major tile order), un-flipped, resized back and summed; -> (S / V, log(max(S / V, FLT_MIN))).

``forward_fn(x) -> logits`` is any network at the dtype of x: an oracle model, the engine's model, a stub."""
import torch
import torch.nn.functional as F

FLT_MIN = torch.finfo(torch.float32).tiny


def views(scales, flip):
    out = []
    for s in scales:
        out.append((float(s), False))
        if flip:
            out.append((float(s), True))
    return out


def view_image(x, s, f):
    H, W = x.shape[2:]
    if s != 1.0:
        x = F.interpolate(x, (int(H * s + 0.5), int(W * s + 0.5)), mode='bilinear', align_corners=True)
    if f:
        x = torch.flip(x, dims=(3,))
    return x


def sliding_tiles(h, w, crop):
    """[(row, col, tile height, tile width)] in UniMatch's loop order."""
    stride = int(crop * 2 / 3)
    out = []
    row = 0
    while row < h:
        col = 0
        while col < w:
            out.append((row, col, min(h, row + crop) - row, min(w, col + crop) - col))
            col += stride
        row += stride
    return out


def view_prob(forward_fn, xv, protocol, crop):
    if protocol == 'whole':
        return torch.softmax(forward_fn(xv), dim=1)
    n, _, h, w = xv.shape
    P = None
    for r, c, th, tw in sliding_tiles(h, w, crop):
        p = torch.softmax(forward_fn(xv[:, :, r:r + th, c:c + tw].contiguous()), dim=1)
        if P is None:
            P = torch.zeros((n, p.shape[1], h, w), dtype=p.dtype, device=p.device)
        P[:, :, r:r + th, c:c + tw] += p
    return P


def evaluate(forward_fn, x, protocol='whole', crop=None, scales=(1.0,), flip=False):
    """-> (mean, log(max(mean, FLT_MIN))) of the ensemble, at the dtype of x."""
    H, W = x.shape[2:]
    vs = views(scales, flip)
    S = None
    for s, f in vs:
        P = view_prob(forward_fn, view_image(x, s, f), protocol, crop)
        if f:
            P = torch.flip(P, dims=(3,))
        if s != 1.0:
            P = F.interpolate(P, (H, W), mode='bilinear', align_corners=True)
        S = P if S is None else S + P
    mean = S / len(vs)
    return mean, torch.log(torch.clamp(mean, min=FLT_MIN))
