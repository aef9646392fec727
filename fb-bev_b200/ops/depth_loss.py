"""Depth supervision of the lift step (``fbbev_depth_loss_fwd`` / ``_bwd``,
csrc/depth_loss.cu).

Replaces ``get_downsampled_gt_depth`` + ``get_depth_loss`` of

* ``CM_DepthNet``  (mmdet3d/models/fbbev/modules/depth_net.py:396-450) and
* ``LSSViewTransformerBEVDepth``  (mmdet3d/models/necks/view_transformer.py:
  1036-1081),

with ``sid=False``.  The reference permutes the gt map and the predictions,
builds an int64 one-hot, gathers the foreground rows with boolean masks and
normalises by ``max(1.0, fg_mask.sum())`` -- three host syncs.  Here the
labels, the loss, the foreground count and the gradient stay on the device, so
a training step that includes the loss can be captured as a CUDA graph.
"""
import torch

from .. import _lib

__all__ = ['depth_loss', 'downsampled_gt_depth', 'depth_labels', 'DepthLoss']


def _label_constants(depth_cfg):
    """(c0, c1) of ``(gt - (lo - step)) / step``: the difference is taken in
    Python double, as the reference does, and each constant reaches the kernel
    rounded to fp32, as torch rounds a Python scalar for a float32 tensor."""
    lo, _, step = depth_cfg
    return float(lo - step), float(step)


def _gt_view(gt_depths, downsample):
    H, W = gt_depths.shape[-2:]
    if H % downsample or W % downsample:
        raise _lib.FbbevError(
            f'gt depth {H}x{W} is not a multiple of downsample {downsample}')
    gt = gt_depths.float().contiguous().view(-1, H, W)
    return gt, H // downsample, W // downsample


def _fwd(gt_depths, depth_preds, downsample, depth_cfg, loss_weight):
    """-> (loss 0-d fp32, labels (BN*h*w,) int32, n_fg 0-d int32, preds
    (BN, D, h, w) fp32 dense); depth_preds (.., D, h, w) of BN images."""
    dev = _lib.require_cuda(gt_depths, depth_preds)
    gt, h, w = _gt_view(gt_depths, downsample)
    BN, H, W = gt.shape
    D = depth_preds.shape[-3]
    if tuple(depth_preds.shape[-2:]) != (h, w) or \
            depth_preds.numel() != BN * D * h * w:
        raise ValueError(
            f'depth_preds {tuple(depth_preds.shape)} does not match gt '
            f'{tuple(gt_depths.shape)} at downsample {downsample}')
    preds = depth_preds.float().contiguous().view(BN, D, h, w)
    c0, c1 = _label_constants(depth_cfg)
    labels = torch.empty(BN * h * w, dtype=torch.int32, device=dev)
    alloc = torch.empty if BN else torch.zeros     # bn == 0 is a no-op
    loss = alloc((), dtype=torch.float32, device=dev)
    n_fg = alloc((), dtype=torch.int32, device=dev)
    L = _lib.lib()
    ws_bytes = L.fbbev_depth_loss_workspace_bytes(BN, H, downsample)
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = L.fbbev_depth_loss_fwd(
            _lib.ptr(gt), _lib.ptr(preds), BN, H, W, downsample, D, c0, c1,
            float(loss_weight), _lib.ptr(labels), _lib.ptr(loss),
            _lib.ptr(n_fg), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_depth_loss_fwd')
    return loss, labels, n_fg, preds


def _bwd(grad_loss, labels, preds, n_fg, loss_weight):
    dev = preds.device
    BN, D, h, w = preds.shape
    g = grad_loss.to(device=dev, dtype=torch.float32).reshape(())
    grad = torch.empty_like(preds)
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_depth_loss_bwd(
            _lib.ptr(labels), _lib.ptr(preds), _lib.ptr(n_fg), _lib.ptr(g), BN,
            h, w, D, float(loss_weight), _lib.ptr(grad), _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_depth_loss_bwd')
    return grad


class DepthLoss(torch.autograd.Function):
    """Loss of ``depth_preds`` against the gt depth map; the backward writes
    the dense d preds (zero at background pixels) from the saved labels."""

    @staticmethod
    def forward(ctx, depth_preds, gt_depths, downsample, depth_cfg,
                loss_weight):
        loss, labels, n_fg, preds = _fwd(gt_depths.detach(),
                                         depth_preds.detach(), downsample,
                                         depth_cfg, loss_weight)
        ctx.save_for_backward(labels, preds, n_fg)
        ctx.loss_weight = loss_weight
        ctx.preds_shape = depth_preds.shape
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        labels, preds, n_fg = ctx.saved_tensors
        grad = _bwd(grad_loss, labels, preds, n_fg, ctx.loss_weight)
        return grad.view(ctx.preds_shape), None, None, None, None


def depth_loss(gt_depths, depth_preds, downsample, depth_cfg, loss_weight):
    """``loss_weight * BCE(depth_preds, one-hot gt) / max(1, n_fg)`` as a 0-d
    CUDA tensor, without a host sync.

    gt_depths (B, N, H, W) (any leading shape of B*N images); depth_preds
    (B, N, D, h, w) or (B*N, D, h, w) probabilities, h = H / downsample;
    depth_cfg = grid_config['depth'] = [lo, hi, step]."""
    if torch.is_grad_enabled() and depth_preds.requires_grad:
        return DepthLoss.apply(depth_preds, gt_depths, downsample, depth_cfg,
                               loss_weight)
    return _fwd(gt_depths, depth_preds, downsample, depth_cfg,
                loss_weight)[0]


def depth_labels(gt_depths, downsample, depth_cfg, D):
    """Class of every output pixel, (B*N*h*w,) int32 in [0, D]: 0 is
    background, c >= 1 is depth bin c - 1."""
    dev = _lib.require_cuda(gt_depths)
    gt, h, w = _gt_view(gt_depths, downsample)
    BN, H, W = gt.shape
    c0, c1 = _label_constants(depth_cfg)
    labels = torch.empty(BN * h * w, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_depth_loss_fwd(
            _lib.ptr(gt), None, BN, H, W, downsample, D, c0, c1, 0.0,
            _lib.ptr(labels), None, None, None, 0, _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_depth_loss_fwd')
    return labels


def downsampled_gt_depth(gt_depths, downsample, depth_cfg, D):
    """The reference's ``get_downsampled_gt_depth``: float one-hot
    (B*N*h*w, D), all zeros at background pixels."""
    labels = depth_labels(gt_depths, downsample, depth_cfg, D)
    bins = torch.arange(1, D + 1, dtype=torch.int32, device=labels.device)
    return (labels.view(-1, 1) == bins).float()
