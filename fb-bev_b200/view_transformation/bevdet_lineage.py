"""BEVDet-lineage callers of the pooling op (SURVEY.md section 8 f3).

Mirror of ``mmdet3d/models/necks/view_transformer.py``:

* ``LSSViewTransformer``          (:15-326)  1x1 ``depth_net`` conv -> depth
  softmax + context -> voxel pooling, Z collapsed into channels (:191);
* ``LSSViewTransformer2``         (:331-724) the same with the depth-threshold
  sparsification: points with depth probability <= 0.01 are dropped from the
  index (:556-557; cached-index form :657-678);
* ``LSSViewTransformerBEVDepth``  (:1000-1105) ``LSSViewTransformer2`` with the
  camera-aware depth net and ``get_mlp_input`` (:1010-1034).

Same registry names, constructor keywords, ``forward(input)`` contract
(``input = [img_feat, rots, trans, intrins, post_rots, post_trans, bda(,
mlp_input)]``), return value ``(bev_feat, depth)`` and state-dict keys
(``depth_net.*`` only -- these classes carry no ``dx/bx/nx``).

What runs underneath: the tail of ``forward`` -- channel split, softmax over
the depth bins, and the NCHW -> NHWC copy the pooling op would start with --
is one launch (``ops.lift_tail``); index building with the threshold is the
device counting sort (``fbbev_voxel_prepare(_cams)``); pooling is the
dense op.  The ``depth_net`` convolution stays a library call (cuDNN): it is
the step before the path.
"""
import torch
import torch.nn as nn

from ..ops import depth_loss as _depth_loss
from ..ops.bev_pool_v2 import voxel_pooling_prepare_v2
from ..ops.lift_tail import lift_tail
from ..registry import register
from .forward_projection import _LSSBase

__all__ = ['LSSViewTransformer', 'LSSViewTransformer2',
           'LSSViewTransformerBEVDepth', 'DEPTH_THRESHOLD']

DEPTH_THRESHOLD = 0.01   # necks/view_transformer.py:556, :657


@register('NECKS')
class LSSViewTransformer(_LSSBase):
    r"""``NECKS.LSSViewTransformer`` (necks/view_transformer.py:15-326).

    Args:
        grid_config, input_size, downsample: as the reference.
        in_channels (int): channels of the image feature.
        out_channels (int): channels of the lifted context feature.
        accelerate (bool): cache the index of the first camera rig (:260-283).
        uniform (bool): uniform depth distribution (``depth_digit * 0``, :316).
    """

    def __init__(self, grid_config, input_size, downsample=16, in_channels=512,
                 out_channels=64, accelerate=False, uniform=False,
                 with_cp=False):
        super().__init__(grid_config, input_size, downsample, accelerate,
                         uniform, with_cp)
        # the reference's necks classes have no dx / bx / nx (state-dict keys)
        del self.dx, self.bx, self.nx
        self.out_channels = out_channels
        self.in_channels = in_channels
        self.depth_net = nn.Conv2d(in_channels, self.D + self.out_channels,
                                   kernel_size=1, padding=0)

    @staticmethod
    def _collapse(bev_feat):
        # (B,C,Z,Y,X) -> (B, Z*C, Y, X)   torch.cat(x.unbind(dim=2), 1)  (:191)
        return torch.cat(bev_feat.unbind(dim=2), 1)

    # -- necks/view_transformer.py:165-192 ---------------------------------
    def voxel_pooling_v2(self, coor, depth, feat):
        idx = voxel_pooling_prepare_v2(coor, self.grid_lower_bound,
                                       self.grid_interval, self.grid_size)
        return self._collapse(self._pool(idx, depth, feat))

    def pre_compute(self, input):
        if self.initial_flag:
            # static rig: remember the cameras the index belongs to; the
            # reference-visible attributes are filled from the geometric index
            # (no depth: no threshold)
            self._cached_cams = [t.detach().clone() for t in input[1:7]]
            self.init_acceleration_v2(self._build_index(self._cached_cams))
            self.initial_flag = False

    # -- necks/view_transformer.py:266-289 ---------------------------------
    def view_transform_core(self, input, depth, feat_nhwc):
        """depth (B*N, D, H, W) softmax; feat_nhwc (B*N, H, W, C)."""
        B, N, _, H, W = input[0].shape
        depth5 = depth.view(B, N, self.D, H, W)
        feat5 = feat_nhwc.view(B, N, H, W, self.out_channels)
        if self.accelerate:
            if self.depth_threshold is None:
                idx = self._index
            else:   # the cached geometry filtered by today's depth (:657-678)
                idx = self._build_index(self._cached_cams, depth5,
                                        pool_channels=self.out_channels)
            bev = self._pool(idx, depth5, feat5, nhwc=True).squeeze(2)  # :283
        else:
            idx = self._build_index(input[1:7], depth5,
                                    pool_channels=self.out_channels)
            bev = self._collapse(self._pool(idx, depth5, feat5, nhwc=True))
        return bev, depth

    def view_transform(self, input, depth, feat_nhwc):
        if self.accelerate:
            self.pre_compute(input)
        return self.view_transform_core(input, depth, feat_nhwc)

    def _depth_net_out(self, input):
        x = input[0]
        B, N, C, H, W = x.shape
        return self.depth_net(x.view(B * N, C, H, W))

    # -- necks/view_transformer.py:296-324 ---------------------------------
    def forward(self, input, return_depth_digit=False):
        """input = [img_feat (B,N,C,H,W), rots, trans, intrins, post_rots,
        post_trans, bda, ...] -> (bev_feat (B, Z*C, Y, X), depth (B*N,D,H,W))."""
        x = self._depth_net_out(input)
        depth_digit = x[:, :self.D]
        tran_feat = x[:, self.D:self.D + self.out_channels]
        logits = depth_digit * 0 if self.uniform else depth_digit
        depth, feat_nhwc = lift_tail(logits, tran_feat)
        out = self.view_transform(input, depth, feat_nhwc)
        if return_depth_digit:
            return out + (depth_digit,)
        return out


@register('NECKS')
class LSSViewTransformer2(LSSViewTransformer):
    r"""``NECKS.LSSViewTransformer2`` (necks/view_transformer.py:331-724): points
    whose depth probability is <= 0.01 never enter the index (:556-557)."""

    depth_threshold = DEPTH_THRESHOLD

    # -- :520-578: (ranks_bev, ranks_depth, ranks_feat) of the thresholded list
    def voxel_pooling_prepare_v2(self, depth, coor):
        idx = voxel_pooling_prepare_v2(
            coor, self.grid_lower_bound, self.grid_interval, self.grid_size,
            depth=depth, depth_thresh=self.depth_threshold)
        rb, rd, rf, _, _ = idx.trimmed()
        return rb, rd, rf

    # -- :580-637: the geometric list and the mask it was compacted with
    def voxel_pooling_prepare_v2_inf(self, coor):
        idx = voxel_pooling_prepare_v2(coor, self.grid_lower_bound,
                                       self.grid_interval, self.grid_size)
        rb, rd, rf, _, _ = idx.trimmed()
        kept = torch.zeros(coor.shape[:-1].numel(), dtype=torch.bool,
                           device=coor.device)
        if rd is not None:
            kept[rd.long()] = True
        return kept, rb, rd, rf

    def voxel_pooling_v2(self, coor, depth, feat):
        idx = voxel_pooling_prepare_v2(
            coor, self.grid_lower_bound, self.grid_interval, self.grid_size,
            depth=depth, depth_thresh=self.depth_threshold)
        return self._collapse(self._pool(idx, depth, feat))

    def init_acceleration_v2(self, coor):
        super().init_acceleration_v2(coor)
        # `kept` (:472): the geometric in-grid mask over all points
        kept = torch.zeros(self._index.ranks_depth.numel(), dtype=torch.bool,
                           device=self._index.ranks_depth.device)
        if self.ranks_depth is not None:
            kept[self.ranks_depth.long()] = True
        self.kept = kept


@register('NECKS')
class LSSViewTransformerBEVDepth(LSSViewTransformer2):
    r"""``NECKS.LSSViewTransformerBEVDepth`` (necks/view_transformer.py:
    1000-1105).  ``depth_net`` is the camera-aware ``DepthNet`` (:876-937:
    ResNet blocks, ASPP, DCN -- the step before the path, out of scope here):
    pass the module as ``depthnet_cfg=dict(module=net)``; it is called as
    ``net(x (B*N, C, H, W), mlp_input)`` and returns (B*N, D + C_out, H, W)
    exactly like the reference's."""

    def __init__(self, loss_depth_weight=3.0, depthnet_cfg=dict(),
                 with_cp=False, **kwargs):
        super().__init__(**kwargs)
        self.with_cp = with_cp
        self.loss_depth_weight = loss_depth_weight
        net = dict(depthnet_cfg).get('module')
        if net is None:
            raise ValueError(
                'LSSViewTransformerBEVDepth: the camera-aware DepthNet is '
                'outside this package (SURVEY.md section 2); pass it as '
                'depthnet_cfg=dict(module=<nn.Module>)')
        self.depth_net = net

    # -- :1010-1034 --------------------------------------------------------
    def get_mlp_input(self, rot, tran, intrin, post_rot, post_tran, bda):
        B, N, _, _ = rot.shape
        bda = bda.view(B, 1, 3, 3).repeat(1, N, 1, 1)
        mlp_input = torch.stack([
            intrin[:, :, 0, 0], intrin[:, :, 1, 1], intrin[:, :, 0, 2],
            intrin[:, :, 1, 2], post_rot[:, :, 0, 0], post_rot[:, :, 0, 1],
            post_tran[:, :, 0], post_rot[:, :, 1, 0], post_rot[:, :, 1, 1],
            post_tran[:, :, 1], bda[:, :, 0, 0], bda[:, :, 0, 1],
            bda[:, :, 1, 0], bda[:, :, 1, 1], bda[:, :, 2, 2]], dim=-1)
        sensor2ego = torch.cat([rot, tran.reshape(B, N, 3, 1)],
                               dim=-1).reshape(B, N, -1)
        return torch.cat([mlp_input, sensor2ego], dim=-1)

    # -- :1036-1065 --------------------------------------------------------
    def get_downsampled_gt_depth(self, gt_depths):
        """gt_depths (B, N, H, W) -> float one-hot (B*N*h*w, D)."""
        return _depth_loss.downsampled_gt_depth(
            gt_depths, self.downsample, self.grid_config['depth'], self.D)

    # -- :1067-1081 --------------------------------------------------------
    def get_depth_loss(self, depth_labels, depth_preds):
        """depth_labels: gt depth (B, N, H, W); depth_preds (B*N, D, h, w).
        Returns the weighted 0-d loss, computed without a host sync."""
        if depth_preds.shape[1] != self.D:
            raise ValueError(f'depth_preds has {depth_preds.shape[1]} bins, '
                             f'the grid has {self.D}')
        return _depth_loss.depth_loss(depth_labels, depth_preds,
                                      self.downsample,
                                      self.grid_config['depth'],
                                      self.loss_depth_weight)

    def _depth_net_out(self, input):
        x, mlp_input = input[0], input[7]
        B, N, C, H, W = x.shape
        return self.depth_net(x.view(B * N, C, H, W), mlp_input)
