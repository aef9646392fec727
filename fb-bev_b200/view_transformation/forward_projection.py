"""Forward projection (lift-splat) plugin classes.

Mirror of ``mmdet3d/models/fbbev/view_transformation/forward_projection/
view_transformer.py`` -- same registry names, constructor arguments, attributes
read by callers (``dx/bx/nx``, ``grid_size``, ``D``, ``frustum``) and method
signatures -- so FB-OCC's detector (``fbocc.py:339``) and its config
(``fbocc-r50 ... :150-154``) use it unchanged.

What changed underneath:

* ``voxel_pooling_prepare_v2`` (view_transformer.py:547-605) runs as six small
  CUDA kernels with no host synchronisation (``fbbev_voxel_prepare``);
* ``bev_pool_v2`` (bev_pool.py:84-90) is one fused kernel that writes the
  ``(B,C,Z,Y,X)`` volume once (``fbbev_bev_pool_v2_fwd_dense_planned``);
* ``accelerate=True`` caches the device index (the reference's 3-D class
  asserts out at view_transformer.py:628; the 2-D class supports it, :271-283).

Geometry: ``get_lidar_coor`` keeps the reference's operation sequence in
PyTorch.  ``forward`` evaluates the same chain inside the voxelisation kernel
(``fused_geometry``), rounding every 3x3 product exactly as torch's broadcast
matmul does, so the integer index is bit-identical to
``voxel_pooling_prepare_v2(get_lidar_coor(...))`` -- the integer voxel path is
only bit-exact if the fp32 coordinates it starts from are rounded identically
(SURVEY.md section 7.3; tests/test_forward_gpu.py::test_fused_geometry_bit_exact).
"""
import torch
import torch.nn as nn

from ..ops.bev_pool_v2 import (DeferredVolumeTrain, VoxelIndex, bev_pool_v2,
                               bev_pool_v2_deferred,
                               bev_pool_v2_dense, deferred_supported,
                               voxel_pooling_prepare_from_cams,
                               voxel_pooling_prepare_v2)
from ..registry import BaseModule, register

__all__ = ['gen_dx_bx', 'LSSViewTransformerFunction3D',
           'LSSViewTransformerFunction', 'forward_backward_readd']


def inv3x3_many(*mats):
    """Inverses of several stacks of small square matrices with ONE batched
    ``torch.linalg.inv_ex`` call (== torch.inverse per matrix, without the
    host-side error check and its device synchronisation).  Each inverse call
    costs ~7 kernel launches (LU, pivots, two triangular solves), so sharing it
    matters in a 0.7 ms step."""
    n = mats[0].shape[-1]
    flat = [m.reshape(-1, n, n) for m in mats]
    inv = torch.linalg.inv_ex(torch.cat(flat, 0) if len(flat) > 1 else flat[0])[0]
    out, o = [], 0
    for m, f in zip(mats, flat):
        out.append(inv[o:o + f.shape[0]].reshape(m.shape))
        o += f.shape[0]
    return out


def gen_dx_bx(xbound, ybound, zbound):
    """Voxel size, first-voxel centre and voxel count per axis
    (view_transformer.py:17-21); consumed by FBOCC (fbocc.py:110, 183-188)."""
    bounds = (xbound, ybound, zbound)
    dx = torch.Tensor([b[2] for b in bounds])
    bx = torch.Tensor([b[0] + b[2] / 2.0 for b in bounds])
    nx = torch.Tensor([(b[1] - b[0]) / b[2] for b in bounds])
    return dx, bx, nx


class _LSSBase(BaseModule):
    """Shared geometry / index machinery of the 2-D and 3-D transformers.

    ``fused_geometry`` (class attribute, default True; setting the attribute
    to False turns it off): ``forward`` evaluates the frustum -> ego chain
    inside the voxelisation kernel instead of materialising
    ``get_lidar_coor``'s (B,N,D,H,W,3) tensor
    through eager PyTorch (cuBLAS batched 3x3 products for 338k points, many
    times the pooling kernel).  Both routes implement the same fp32
    chain with the same rounding order (``mat3_apply_ref`` in csrc/common.cuh
    reproduces the order of torch's broadcast matmul on this device, found with
    tools/micro/matmul_order2.py), so the resulting index is identical, point
    for point.  ``get_lidar_coor`` and ``voxel_pooling_prepare_v2(coor)`` keep
    the reference's exact contract.
    """

    fused_geometry = True
    # LSSViewTransformer2 keeps the points whose depth probability exceeds it
    depth_threshold = None

    def __init__(self, grid_config, input_size, downsample, accelerate,
                 uniform, with_cp):
        super().__init__()
        self.uniform = uniform
        self.with_cp = with_cp
        self.grid_config = grid_config
        self.downsample = downsample
        self.create_grid_infos(**grid_config)
        dx, bx, nx = gen_dx_bx(grid_config['x'], grid_config['y'],
                               grid_config['z'])
        self.dx = nn.Parameter(dx, requires_grad=False)
        self.bx = nn.Parameter(bx, requires_grad=False)
        self.nx = nn.Parameter(nx, requires_grad=False)
        self.input_size = input_size
        self.create_frustum(grid_config['depth'], input_size, downsample)
        self.accelerate = accelerate
        self.initial_flag = True
        self._index = None  # cached VoxelIndex when accelerate=True

    # -- view_transformer.py:371-387 ------------------------------------
    def create_grid_infos(self, x, y, z, **kwargs):
        """Grid lower bound / interval / size as float32 tensors.  The size is
        evaluated in Python double precision and rounded to float32 exactly as
        the reference does (e.g. (5.4 - -1)/0.8 = 8.000000000000002 -> 8.0f)."""
        axes = (x, y, z)
        self.grid_lower_bound = torch.Tensor([a[0] for a in axes])
        self.grid_interval = torch.Tensor([a[2] for a in axes])
        self.grid_size = torch.Tensor([(a[1] - a[0]) / a[2] for a in axes])

    # -- view_transformer.py:389-411 ------------------------------------
    def create_frustum(self, depth_cfg, input_size, downsample):
        """Frustum template (D, H_feat, W_feat, 3) = (u, v, depth)."""
        H_in, W_in = input_size
        H_feat, W_feat = H_in // downsample, W_in // downsample
        d = torch.arange(*depth_cfg, dtype=torch.float).view(-1, 1, 1)
        self.D = d.shape[0]
        d = d.expand(self.D, H_feat, W_feat)
        u = torch.linspace(0, W_in - 1, W_feat, dtype=torch.float).view(
            1, 1, W_feat).expand(self.D, H_feat, W_feat)
        v = torch.linspace(0, H_in - 1, H_feat, dtype=torch.float).view(
            1, H_feat, 1).expand(self.D, H_feat, W_feat)
        self.frustum = torch.stack((u, v, d), -1)

    # -- view_transformer.py:458-498 ------------------------------------
    def get_lidar_coor(self, rots, trans, cam2imgs, post_rots, post_trans,
                       bda):
        """Frustum points in the ego/lidar frame, (B, N, D, H, W, 3).

        Same operation sequence as the reference so the fp32 results -- and
        therefore the voxel each point truncates into -- are identical."""
        B, N, _ = trans.shape
        # undo the image-view augmentation
        pts = self.frustum.to(rots) - post_trans.view(B, N, 1, 1, 1, 3)
        pts = torch.inverse(post_rots).view(B, N, 1, 1, 1, 3, 3).matmul(
            pts.unsqueeze(-1))
        # pixel * depth -> camera frame -> ego frame
        pts = torch.cat((pts[..., :2, :] * pts[..., 2:3, :], pts[..., 2:3, :]),
                        5)
        cam2ego = rots.matmul(torch.inverse(cam2imgs))
        pts = cam2ego.view(B, N, 1, 1, 1, 3, 3).matmul(pts).squeeze(-1)
        pts += trans.view(B, N, 1, 1, 1, 3)
        pts = bda.view(B, 1, 1, 1, 1, 3, 3).matmul(pts.unsqueeze(-1)).squeeze(-1)
        return pts

    def _frustum_axes(self, device):
        key = str(device)
        cache = self.__dict__.setdefault('_axes_cache', {})
        if key not in cache:
            f = self.frustum
            cache[key] = (f[0, 0, :, 0].contiguous().to(device),
                          f[0, :, 0, 1].contiguous().to(device),
                          f[:, 0, 0, 2].contiguous().to(device))
        return cache[key]

    def prepare_index_from_cams(self, rots, trans, cam2imgs, post_rots,
                                post_trans, bda, pool_channels=None, **thresh):
        """Index straight from the camera parameters (fused geometry).  The
        two 3x3 products the reference forms before touching the points
        (view_transformer.py:483-491) are formed here by the same torch ops
        (inv_ex == torch.inverse without the host-side error check; the two
        inverses share one batched call).  ``thresh``: ``depth`` and
        ``depth_thresh`` of :func:`voxel_pooling_prepare_from_cams`."""
        inv_pr, inv_k = inv3x3_many(post_rots, cam2imgs)
        cam2ego = rots.matmul(inv_k)
        return voxel_pooling_prepare_from_cams(
            self._frustum_axes(rots.device), inv_pr, post_trans, cam2ego,
            trans, bda, self.D, self.grid_lower_bound, self.grid_interval,
            self.grid_size, pool_channels=pool_channels, **thresh)

    # -- view_transformer.py:547-605 ------------------------------------
    def prepare_index(self, coor, pool_channels=None, **thresh):
        """Device-resident index of ``coor`` (no host sync).  ``pool_channels``:
        the channel count of the pooling call that follows, so that the index
        builder can fill that call's plan while it scans.  ``thresh``:
        ``depth`` and ``depth_thresh`` of :func:`voxel_pooling_prepare_v2`."""
        return voxel_pooling_prepare_v2(coor, self.grid_lower_bound,
                                        self.grid_interval, self.grid_size,
                                        pool_channels=pool_channels, **thresh)

    def _build_index(self, cam_params, depth=None, pool_channels=None):
        """VoxelIndex of this call's cameras: geometry fused into the index
        builder or through ``get_lidar_coor`` (``fused_geometry``), bounds
        test and -- with a ``depth_threshold`` and ``depth`` (B,N,D,H,W) --
        the depth threshold."""
        kw = dict(pool_channels=pool_channels)
        if self.depth_threshold is not None and depth is not None:
            kw.update(depth=depth, depth_thresh=self.depth_threshold)
        if self.fused_geometry:
            return self.prepare_index_from_cams(*cam_params, **kw)
        return self.prepare_index(self.get_lidar_coor(*cam_params), **kw)

    def voxel_pooling_prepare_v2(self, coor):
        """Same return contract as the reference: five exact-length int32
        tensors ``(ranks_bev, ranks_depth, ranks_feat, interval_starts,
        interval_lengths)`` or five ``None`` when no point falls in the grid.
        (Reading the two counts is the only host sync; the internal fast path
        ``voxel_pooling_v2`` does not need it.)"""
        return self.prepare_index(coor).trimmed()

    # -- view_transformer.py:500-519 ------------------------------------
    def init_acceleration_v2(self, coor):
        idx = coor if isinstance(coor, VoxelIndex) else self.prepare_index(coor)
        self._index = idx
        rb, rd, rf, st, ln = idx.trimmed()
        self.ranks_bev, self.ranks_depth, self.ranks_feat = rb, rd, rf
        self.interval_starts, self.interval_lengths = st, ln

    def pre_compute(self, cam_params):
        if self.initial_flag:
            self.init_acceleration_v2(self._build_index(cam_params))
            self.initial_flag = False

    def _bev_feat_shape(self, depth, feat_nhwc):
        return (depth.shape[0], int(self.grid_size[2]), int(self.grid_size[1]),
                int(self.grid_size[0]), feat_nhwc.shape[-1])  # (B, Z, Y, X, C)

    def _pool(self, idx, depth, feat, nhwc=False):
        """depth (B,N,D,H,W), feat (B,N,C,H,W) -- or, ``nhwc``, already the
        (B,N,H,W,C) tensor ``bev_pool_v2`` reads (ops.lift_tail produces it, so
        the permute + ``contiguous()`` copy of view_transformer.py:530 /
        bev_pool.py:19 never runs) -> (B,C,Z,Y,X) contiguous."""
        if not nhwc:
            feat = feat.permute(0, 1, 3, 4, 2)
        shape = self._bev_feat_shape(depth, feat)
        if isinstance(idx, VoxelIndex):
            return bev_pool_v2_dense(
                depth, feat, idx.ranks_depth, idx.ranks_feat, idx.ranks_bev,
                shape, idx.interval_starts, idx.interval_lengths,
                n_intervals_dev=idx.n_intervals_dev, n_kept_dev=idx.n_kept_dev,
                plan=idx.plan, index=idx)
        rb, rd, rf, st, ln = idx
        return bev_pool_v2(depth, feat, rd, rf, rb, shape, st, ln)

    def get_mlp_input(self, rot, tran, intrin, post_rot, post_tran, bda):
        return None


@register('NECKS')
class LSSViewTransformerFunction3D(_LSSBase):
    r"""Lift-Splat-Shoot view transformer producing a voxel volume.

    Drop-in for ``NECKS.LSSViewTransformerFunction3D``
    (view_transformer.py:315-663).

    Args:
        grid_config (dict): (lower_bound, upper_bound, interval) per axis in
            {x, y, z, depth}.
        input_size (tuple[int]): input image (height, width).
        downsample (int): image -> feature map down-sampling factor.
        accelerate (bool): cache the voxel index computed from the first
            ``cam_params`` (valid only for a static camera rig).
        uniform, with_cp: accepted for config compatibility (unused by the
            reference's forward as well).
        extra_relu (bool): apply ReLU to the output (view_transformer.py:657).
    """

    def __init__(self, grid_config, input_size, downsample=16,
                 accelerate=False, uniform=False, with_cp=False,
                 extra_relu=False):
        super().__init__(grid_config, input_size, downsample, accelerate,
                         uniform, with_cp)
        self.extra_relu = extra_relu

    # -- view_transformer.py:521-545 ------------------------------------
    def voxel_pooling_v2(self, coor, depth, feat):
        """Returns (B, C, Y, X, Z): a view of the contiguous (B,C,Z,Y,X)
        volume, exactly like the reference (view_transformer.py:543).  An empty
        index yields the all-zero volume (the reference prints a warning and
        returns zeros, :525-535) without a host round-trip."""
        bev_feat = self._pool(self.prepare_index(coor), depth, feat)
        return bev_feat.permute(0, 1, 3, 4, 2)

    # -- view_transformer.py:613-643 ------------------------------------
    def view_transform_core(self, cam_params, depth, tran_feat, nhwc=False):
        if self.accelerate:
            bev_feat = self._pool(self._index, depth, tran_feat, nhwc)
            return bev_feat.permute(0, 1, 3, 4, 2)
        C = tran_feat.shape[-1 if nhwc else 2]
        idx = self._build_index(cam_params, pool_channels=C)
        return self._pool(idx, depth, tran_feat, nhwc).permute(0, 1, 3, 4, 2)

    def view_transform(self, cam_params, depth, tran_feat, nhwc=False):
        if self.accelerate:
            self.pre_compute(cam_params)
        return self.view_transform_core(cam_params, depth, tran_feat, nhwc)

    def forward_deferred(self, cam_params, context, depth):
        """Index + interval sums only: a :class:`~..ops.bev_pool_v2.
        DeferredVolume` whose ``mean_z()`` is ``forward(...).mean(-1)`` and
        whose ``materialize(add)`` is ``forward(...)`` (+ ``add[..., None]``)
        in the contiguous (B, C, Z, Y, X) layout -- see
        :func:`forward_backward_readd`.  When autograd records, a
        :class:`~..ops.bev_pool_v2.DeferredVolumeTrain` with the same outputs
        and a backward that reads the volume's gradient once (call
        ``mean_z()`` before ``materialize``).  Returns None when the shape is
        not covered (caller falls back to ``forward``)."""
        feat = context.permute(0, 1, 3, 4, 2)
        shape = self._bev_feat_shape(depth, feat)
        if not deferred_supported(shape) or not depth.is_cuda:
            return None
        if self.accelerate:
            self.pre_compute(cam_params)
            idx = self._index
        else:
            idx = self._build_index(cam_params, pool_channels=shape[-1])
        if torch.is_grad_enabled() and (context.requires_grad or
                                        depth.requires_grad):
            return DeferredVolumeTrain(depth, feat, idx, shape)
        return bev_pool_v2_deferred(
            depth, feat, idx.ranks_depth, idx.ranks_feat, idx.ranks_bev, shape,
            idx.interval_starts, idx.interval_lengths,
            n_intervals_dev=idx.n_intervals_dev, plan=idx.plan)

    # -- view_transformer.py:646-660 ------------------------------------
    def forward(self, cam_params, context, depth, context_layout='nchw',
                **kwargs):
        """cam_params = (rots, trans, intrins, post_rots, post_trans, bda);
        context (B,N,C,H,W); depth (B,N,D,H,W) -> (B, C, Y, X, Z).
        ``context_layout='nhwc'``: context is already (B,N,H,W,C), the layout
        the pooling op reads (``CM_DepthNetTail`` / ``ops.lift_tail`` produce
        it), and the op's own permute + copy is skipped."""
        assert context_layout in ('nchw', 'nhwc')
        bev = self.view_transform(cam_params, depth, context,
                                  context_layout == 'nhwc')
        if self.extra_relu:
            return bev.relu()
        return bev


@register('NECKS')
class LSSViewTransformerFunction(_LSSBase):
    r"""2-D (height-collapsed) variant: ``NECKS.LSSViewTransformerFunction``
    (view_transformer.py:24-311).  Same pooling op; the Z slices of the
    volume are concatenated along channels (:192, :283)."""

    def __init__(self, grid_config, input_size, downsample=16,
                 accelerate=False, uniform=False, with_cp=False):
        super().__init__(grid_config, input_size, downsample, accelerate,
                         uniform, with_cp)

    @staticmethod
    def _collapse(bev_feat):
        # (B,C,Z,Y,X) -> (B, Z*C, Y, X)   torch.cat(x.unbind(dim=2), 1)
        return torch.cat(bev_feat.unbind(dim=2), 1)

    def voxel_pooling_v2(self, coor, depth, feat):
        return self._collapse(self._pool(self.prepare_index(coor), depth,
                                         feat))

    def view_transform_core(self, cam_params, depth, tran_feat):
        if self.accelerate:
            # the reference squeezes Z here (:283): 4-D only when Z == 1
            return self._pool(self._index, depth, tran_feat).squeeze(2)
        return self._collapse(self._pool(self._build_index(cam_params), depth,
                                         tran_feat))

    def view_transform(self, cam_params, depth, tran_feat):
        if self.accelerate:
            self.pre_compute(cam_params)
        return self.view_transform_core(cam_params, depth, tran_feat)

    def forward(self, cam_params, context, depth, **kwargs):
        return self.view_transform(cam_params, depth, context)


def forward_backward_readd(forward_projection, backward_projection, cam_params,
                           context, depth, img_metas=None, readd=True,
                           bev_mask=None):
    """The three lines of ``FBOCC.extract_img_bev_feat`` around the two
    projections (fbocc.py:339, 357-366)::

        bev_feat = forward_projection(cam_params, context, depth)
        refined  = backward_projection([context], img_metas,
                                       lss_bev=bev_feat.mean(-1), ...)
        bev_feat = refined[..., None] + bev_feat     # if self.readd

    with the dense volume written once instead of written, read twice and
    written again: ``mean(-1)`` comes from the interval sums
    (``fbbev_bev_pool_v2_zmean_planned``) and the re-add rides on the dense
    write (``fbbev_bev_pool_v2_write_planned``).  Under autograd the
    backward reads the volume's gradient once (``DeferredVolumeTrain``).
    Returns ``(bev_feat (B, C, Y, X, Z), refined (B, C, Y, X))``; falls back
    to the literal sequence when the deferred path does not cover the call
    (odd shapes, ``extra_relu``, other forward projections)."""
    dv = None
    if isinstance(forward_projection, LSSViewTransformerFunction3D) and \
            not forward_projection.extra_relu:
        dv = forward_projection.forward_deferred(cam_params, context, depth)
    if dv is None:
        bev_feat = forward_projection(cam_params, context, depth)
        refined = backward_projection(
            [context], img_metas, lss_bev=bev_feat.mean(-1),
            cam_params=cam_params, bev_mask=bev_mask, gt_bboxes_3d=None,
            pred_img_depth=depth)
        return (refined[..., None] + bev_feat if readd else refined), refined
    refined = backward_projection(
        [context], img_metas, lss_bev=dv.mean_z(), cam_params=cam_params,
        bev_mask=bev_mask, gt_bboxes_3d=None, pred_img_depth=depth)
    if not readd:
        return refined, refined
    return dv.materialize(add=refined).permute(0, 1, 3, 4, 2), refined
