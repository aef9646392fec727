"""The tail of ``CM_DepthNet`` as the producer of the pooling op's inputs
(SURVEY.md section 8 f4).

Reference: ``mmdet3d/models/fbbev/modules/depth_net.py:346-363`` --

    context = self.context_conv(context)          # 1x1, mid -> C  (:349)
    depth   = self.depth_conv(depth)              # ... -> D logits (:358)
    depth   = depth.softmax(dim=1)                # (:359)
    context = context.view(B, N, C, H, W)         # (:360)
    depth   = depth.view(B, N, D, H, W)           # (:361)

after which the view transformer's pooling op permutes ``context`` to
(B, N, H, W, C) and copies it (view_transformer.py:530, bev_pool.py:19).

Here the tail produces both tensors directly in the layouts the pooling
kernels read:

* ``context_conv`` is a row-wise Linear over the pixels.  When the gated
  feature map arrives channels-last (``torch.channels_last`` -- the layout
  cuDNN's NHWC convolutions of the body produce), its pixels ARE the rows, so
  the wgmma Linear (``fbbev_linear_fwd``) writes ``feat`` as (B, N, H, W, C)
  with no transposition anywhere; otherwise the convolution stays a cuDNN call
  and ``fbbev_lift_tail_fwd`` transposes its output;
* the softmax over the depth bins is the other half of the same
  ``fbbev_lift_tail_fwd`` launch.

``LSSViewTransformerFunction3D.forward(..., context_layout='nhwc')`` takes the
result as it is.  ``get_depth_loss`` / ``get_downsampled_gt_depth``
(depth_net.py:396-450), the depth supervision FB-OCC trains with, run on the
``fbbev_depth_loss_*`` kernels (ops/depth_loss.py) without a host sync.  The
body of the depth net (ResNet blocks, ASPP, DCN, the SE gates) is the step
before and stays what it is (SURVEY.md section 2).
"""
import torch
import torch.nn as nn

from ..ops import depth_loss as _depth_loss
from ..ops import linear as _linear_ops
from ..ops.lift_tail import lift_tail
from ..registry import BaseModule

__all__ = ['CM_DepthNetTail']


class CM_DepthNetTail(BaseModule):
    """``context_conv`` + depth softmax + layouts of CM_DepthNet.forward.

    The parameter name (``context_conv.{weight,bias}``) is the reference's, so
    ``tail.load_state_dict(depth_net.state_dict(), strict=False)`` adopts a
    trained CM_DepthNet's weights.

    ``downsample``, ``grid_config``, ``depth_channels``, ``loss_depth_weight``
    and ``sid`` are the reference's depth-supervision keywords (plain
    attributes, no state).  ``depth_channels=None`` takes D from the logits
    (``get_depth_loss``) or from ``grid_config['depth']``
    (``get_downsampled_gt_depth``); ``sid=True`` is not supported."""

    def __init__(self, mid_channels=512, context_channels=64, downsample=16,
                 grid_config=None, depth_channels=None, loss_depth_weight=3.0,
                 sid=False):
        super().__init__()
        if sid:
            raise NotImplementedError(
                'CM_DepthNetTail: sid=True (spacing-increasing depth bins) is '
                'not supported')
        self.context_channels = context_channels
        self.downsample = downsample
        self.grid_config = grid_config
        self.depth_channels = depth_channels
        self.loss_depth_weight = loss_depth_weight
        self.sid = sid
        self.context_conv = nn.Conv2d(mid_channels, context_channels,
                                      kernel_size=1, stride=1, padding=0)

    def forward(self, context_feat, depth_logits, B, N):
        """context_feat (B*N, mid, H, W): output of ``context_se`` (:346-348);
        depth_logits (B*N, D, H, W): output of ``depth_conv`` (:358).
        Returns ``(feat (B, N, H, W, C), depth (B, N, D, H, W))``."""
        BN, mid, H, W = context_feat.shape
        D = depth_logits.shape[1]
        C = self.context_channels
        w = self.context_conv.weight.view(C, mid)
        tokens_ready = (
            context_feat.is_cuda and
            context_feat.is_contiguous(memory_format=torch.channels_last) and
            _linear_ops.supported(context_feat, w))
        if tokens_ready:
            rows = context_feat.permute(0, 2, 3, 1).reshape(BN * H * W, mid)
            feat = _linear_ops.linear_fused(rows, w, self.context_conv.bias)
            depth, _ = _softmax_only(depth_logits)
            feat = feat.view(B, N, H, W, C)
        else:
            depth, feat = lift_tail(depth_logits,
                                    self.context_conv(context_feat))
            feat = feat.view(B, N, H, W, C)
        return feat, depth.view(B, N, D, H, W)

    def _depth_cfg(self):
        if self.grid_config is None:
            raise ValueError('CM_DepthNetTail: the depth loss needs grid_config')
        return self.grid_config['depth']

    # -- depth_net.py:396-434 ----------------------------------------------
    def get_downsampled_gt_depth(self, gt_depths):
        """gt_depths (B, N, H, W) -> float one-hot (B*N*h*w, D)."""
        cfg = self._depth_cfg()
        D = self.depth_channels
        if D is None:
            D = torch.arange(*cfg, dtype=torch.float).shape[0]
        return _depth_loss.downsampled_gt_depth(gt_depths, self.downsample,
                                                cfg, D)

    # -- depth_net.py:436-450 ----------------------------------------------
    def get_depth_loss(self, depth_labels, depth_preds):
        """depth_labels: gt depth (B, N, H, W); depth_preds (B, N, D, h, w).
        Returns ``dict(loss_depth=0-d tensor)``."""
        D = depth_preds.shape[2]
        if self.depth_channels is not None and D != self.depth_channels:
            raise ValueError(f'depth_preds has {D} bins, depth_channels is '
                             f'{self.depth_channels}')
        return dict(loss_depth=_depth_loss.depth_loss(
            depth_labels, depth_preds, self.downsample, self._depth_cfg(),
            self.loss_depth_weight))


def _softmax_only(depth_logits):
    """The softmax half of the launch alone (context == NULL)."""
    from .. import _lib
    dev = _lib.require_cuda(depth_logits)
    BN, D, H, W = depth_logits.shape
    lg = depth_logits.float().contiguous()
    depth = torch.empty_like(lg)
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_lift_tail_fwd(
            _lib.ptr(lg), D * H * W, None, 0, BN, D, 0, H * W, _lib.ptr(depth),
            None, _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_lift_tail_fwd')
    return depth, None
