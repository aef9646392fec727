"""Float64 reference of the depth supervision (get_downsampled_gt_depth +
get_depth_loss, mmdet3d/models/fbbev/modules/depth_net.py:396-450 and
mmdet3d/models/necks/view_transformer.py:1036-1081), restated in numpy.

The labels are the fp32 arithmetic the reference performs on the GPU (they
decide which bin is hot, so they must be exact): the patch minimum with exact
zeros replaced by 1e5 and NaN propagating, t = (m - c0) * fl(1 / c1) and the
range test.  The loss and its gradient are then evaluated in float64.
"""
import numpy as np


def labels_ref(gt, ds, depth_cfg, D):
    """gt (..., H, W) -> class per output pixel, (BN*h*w,) int32 in [0, D]."""
    gt = np.asarray(gt, np.float32)
    H, W = gt.shape[-2:]
    h, w = H // ds, W // ds
    x = gt.reshape(-1, h, ds, w, ds).transpose(0, 1, 3, 2, 4)
    x = x.reshape(-1, h, w, ds * ds)
    x = np.where(x == 0, np.float32(1e5), x)
    m = x.min(-1)                              # NaN propagates, as torch.min
    lo, _, step = depth_cfg
    c0, c1 = np.float32(lo - step), np.float32(step)
    t = (m - c0) * (np.float32(1.0) / c1)
    with np.errstate(invalid='ignore'):
        ok = (t >= 0) & (t < D + 1)
    return np.where(ok, np.trunc(np.where(ok, t, 0)), 0).astype(
        np.int32).reshape(-1)


def onehot_ref(labels, D):
    return (labels.reshape(-1, 1) == np.arange(1, D + 1)).astype(np.float32)


def _preds_rows(preds, D):
    """(BN, D, h, w) or (B, N, D, h, w) -> (BN*h*w, D) float64."""
    p = np.asarray(preds, np.float64)
    h, w = p.shape[-2:]
    return np.moveaxis(p.reshape(-1, D, h, w), 1, 3).reshape(-1, D)


def loss_ref64(labels, preds, D, weight):
    p = _preds_rows(preds, D)
    fg = labels > 0
    y = onehot_ref(labels, D).astype(np.float64)[fg]
    p = p[fg]
    with np.errstate(divide='ignore'):
        lp = np.maximum(np.log(p), -100.0)
        l1p = np.maximum(np.log1p(-p), -100.0)
    s = float((-(y * lp + (1 - y) * l1p)).sum())
    return weight * s / max(1, int(fg.sum()))


def grad_ref64(labels, preds, D, weight, grad_loss=1.0):
    """d loss / d preds in the layout of ``preds``."""
    shape = np.shape(preds)
    h, w = shape[-2:]
    p = _preds_rows(preds, D)
    fg = labels > 0
    y = onehot_ref(labels, D).astype(np.float64)
    k = grad_loss * weight / max(1, int(fg.sum()))
    g = k * (p - y) / np.maximum((1 - p) * p, 1e-12)
    g[~fg] = 0.0
    g = np.moveaxis(g.reshape(-1, h, w, D), 3, 1)
    return g.reshape(shape)
