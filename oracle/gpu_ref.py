"""Eager-PyTorch restatement of the reference's GPU execution of the path: the
"reference on the same GPU" comparator of BASELINE.md sections 2.1-2.2.

TEST INFRASTRUCTURE ONLY -- see ``oracle/__init__.py``.  Used by ``bench.py``
(the ``reference_cuda`` block) and by tests as a second, device-side checker.
Nothing here calls a kernel of ``libfbbev_b200.so``: every op is a stock
PyTorch op (plus, for the pooling kernel itself, the reference's own
``bev_pool_cuda.cu`` through ``oracle.ref_cuda`` when it is built).

What is restated, launch for launch:

* ``voxel_pooling_prepare_v2``  view_transformer.py:547-605 (the ~25 eager ops
  incl. ``argsort`` and the three host synchronisations);
* ``DA_SpatialCrossAttention.forward`` spatial_cross_attention_depth.py:86-223
  (per-camera ``nonzero()`` loops, zero-padded re-batching, int64 one-hot,
  scatter loops) and ``DA_MSDeformableAttention.forward`` :465-601 (two MSDA
  launches);
* mmcv ``MultiScaleDeformableAttention.forward`` (self-attention) and ``FFN`` /
  ``LayerNorm`` through cuBLAS / eager kernels.

The MSDA CUDA kernel belongs to mmcv-full 1.5.2, which is not installable here;
its stand-in is mmcv's own documented PyTorch equivalent
(``multi_scale_deformable_attn_pytorch``, the ``F.grid_sample`` formulation the
reference itself falls back to at spatial_cross_attention_depth.py:597-598).
Results tables must label this "reference (PyTorch restatement; mmcv kernel
unavailable)".
"""
import contextlib

import torch
import torch.nn.functional as F

from .torch_ref import multi_scale_deformable_attn_pytorch


# --------------------------------------------------------------------- F ---
def voxel_pooling_prepare_v2(coor, grid_lower_bound, grid_interval, grid_size):
    """view_transformer.py:547-605, op for op (float32 ranks, unstable argsort,
    boolean-mask compactions, ``len()`` host syncs)."""
    B, N, D, H, W, _ = coor.shape
    num_points = B * N * D * H * W
    dev = coor.device
    ranks_depth = torch.arange(0, num_points, dtype=torch.int, device=dev)
    ranks_feat = torch.arange(0, num_points // D, dtype=torch.int, device=dev)
    ranks_feat = ranks_feat.reshape(B, N, 1, H, W)
    ranks_feat = ranks_feat.expand(B, N, D, H, W).flatten()
    coor = ((coor - grid_lower_bound.to(coor)) / grid_interval.to(coor))
    coor = coor.long().view(num_points, 3)
    batch_idx = torch.arange(0, B, dtype=torch.float).reshape(B, 1).expand(
        B, num_points // B).reshape(num_points, 1).to(coor)
    coor = torch.cat((coor, batch_idx), 1)
    gs = grid_size.to(dev)
    kept = (coor[:, 0] >= 0) & (coor[:, 0] < gs[0]) & \
           (coor[:, 1] >= 0) & (coor[:, 1] < gs[1]) & \
           (coor[:, 2] >= 0) & (coor[:, 2] < gs[2])
    if len(kept) == 0:
        return None, None, None, None, None
    coor, ranks_depth, ranks_feat = \
        coor[kept], ranks_depth[kept], ranks_feat[kept]
    ranks_bev = coor[:, 3] * (gs[2] * gs[1] * gs[0])
    ranks_bev += coor[:, 2] * (gs[1] * gs[0])
    ranks_bev += coor[:, 1] * gs[0] + coor[:, 0]
    order = ranks_bev.argsort()
    ranks_bev, ranks_depth, ranks_feat = \
        ranks_bev[order], ranks_depth[order], ranks_feat[order]
    kept = torch.ones(ranks_bev.shape[0], device=dev, dtype=torch.bool)
    kept[1:] = ranks_bev[1:] != ranks_bev[:-1]
    interval_starts = torch.where(kept)[0].int()
    if len(interval_starts) == 0:
        return None, None, None, None, None
    interval_lengths = torch.zeros_like(interval_starts)
    interval_lengths[:-1] = interval_starts[1:] - interval_starts[:-1]
    interval_lengths[-1] = ranks_bev.shape[0] - interval_starts[-1]
    return (ranks_bev.int().contiguous(), ranks_depth.int().contiguous(),
            ranks_feat.int().contiguous(), interval_starts.int().contiguous(),
            interval_lengths.int().contiguous())


def bev_pool_v2_index_add(depth, feat_nhwc, ranks_depth, ranks_feat, ranks_bev,
                          bev_feat_shape):
    """The op's arithmetic with stock torch ops (no reference kernel needed):
    zeros + scatter-add of feat*depth + permute (bev_pool.py:25-36, 89)."""
    B, Z, Y, X, C = bev_feat_shape
    out = feat_nhwc.new_zeros((B * Z * Y * X, C))
    contrib = feat_nhwc.reshape(-1, C)[ranks_feat.long()] * \
        depth.reshape(-1)[ranks_depth.long()][:, None]
    out.index_add_(0, ranks_bev.long(), contrib)
    return out.view(B, Z, Y, X, C).permute(0, 4, 1, 2, 3).contiguous()


# --------------------------------------------------------------------- B ---
def msda_fused_eager(value, spatial_shapes, level_start_index,
                     reference_points, sampling_offsets, attention_logits,
                     map_width=0):
    """mmcv MultiScaleDeformableAttention.forward core with eager ops."""
    w = attention_logits.flatten(3).softmax(-1).view_as(attention_logits)
    wh = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
    loc = reference_points[:, :, None, :, None, :] + \
        sampling_offsets / wh[None, None, None, :, None, :]
    return multi_scale_deformable_attn_pytorch(
        value.float(), spatial_shapes.tolist(), loc, w)


def da_sca_core_eager(value, depth_prob, reference_points_cam, bev_query_depth,
                      per_cam_mask, sampling_offsets, attention_logits,
                      spatial_shapes, level_start_index, dbound, num_Z_anchors,
                    prepared=None):
    """spatial_cross_attention_depth.py:156-216 + 540-595 with eager ops on the
    tensors' device (same contract as ops.da_spatial_cross_attention_core)."""
    shapes = spatial_shapes.tolist()
    N, bs, nq, Z, _ = reference_points_cam.shape
    _, n_value, heads, ch = value.shape
    L, P = sampling_offsets.shape[3], sampling_offsets.shape[4]
    DC = depth_prob.shape[-1]
    E = heads * ch
    if bev_query_depth.dim() == 4:
        bev_query_depth = bev_query_depth[..., None]
    idxs = []
    for j in range(bs):                                             # :163-169
        row = []
        for i in range(N):
            row.append(per_cam_mask[i, j].sum(-1).nonzero().squeeze(-1))
        idxs.append(row)
    max_len = max(1, max(len(i) for r in idxs for i in r))          # :170
    off_re = sampling_offsets.new_zeros(bs, N, max_len, heads, L, P, 2)
    log_re = attention_logits.new_zeros(bs, N, max_len, heads, L, P)
    ref_re = reference_points_cam.new_zeros(bs, N, max_len, Z, 2)
    dep_re = reference_points_cam.new_zeros(bs, N, max_len, Z, 1)
    for j in range(bs):                                             # :173-186
        for i in range(N):
            k = idxs[j][i]
            off_re[j, i, :len(k)] = sampling_offsets[j, k]
            log_re[j, i, :len(k)] = attention_logits[j, k]
            ref_re[j, i, :len(k)] = reference_points_cam[i, j, k]
            dep_re[j, i, :len(k)] = bev_query_depth[i, j, k]
    bins = torch.floor((dep_re - dbound[0]) / dbound[2])           # :196-199
    bins = torch.clip(bins, 0, DC - 1).to(torch.long)
    onehot = F.one_hot(bins.squeeze(-1), num_classes=DC)
    B2 = bs * N
    off = off_re.view(B2, max_len, heads, L, P, 2)
    w = log_re.view(B2, max_len, heads, L * P).softmax(-1).view(
        B2, max_len, heads, L, P)                                   # :540
    ref = ref_re.view(B2, max_len, Z, 2)
    wh = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]],
                     -1).float()
    off = off / wh[None, None, None, :, None, :]
    loc = ref[:, :, None, None, None, :, :] + off.view(
        B2, max_len, heads, L, P // Z, Z, 2)
    loc = loc.view(B2, max_len, heads, L, P, 2)
    dref = ref.reshape(B2, max_len * Z, 1, 1, 1, 2)                # :584-591
    dw = multi_scale_deformable_attn_pytorch(
        depth_prob.unsqueeze(2).float(), shapes[0:1], dref,
        torch.ones_like(dref[..., 0]))
    dw = (dw.reshape(B2, max_len, Z, -1) *
          onehot.view(B2, max_len, Z, DC)).sum(-1)
    dw = dw.unsqueeze(2).repeat(1, 1, P // Z, 1).reshape(B2, max_len, P)
    w = w * dw[:, :, None, None, :]                                 # :592
    out = multi_scale_deformable_attn_pytorch(
        value.float(), shapes, loc, w).view(bs, N, max_len, E)
    slots = out.new_zeros(bs, nq, E)                                # :208-216
    for j in range(bs):
        for i in range(N):
            k = idxs[j][i]
            slots[j, k] += out[j, i, :len(k)]
    count = (per_cam_mask.sum(-1) > 0).permute(1, 2, 0).sum(-1)
    count = torch.clamp(count, min=1.0)
    return slots / count[..., None]


@contextlib.contextmanager
def eager_reference_mode(*modules):
    """Run the plugin's host-side Python as the reference executes it on a GPU:
    eager geometry (cuBLAS batched products), cuBLAS Linears + separate
    bias / add / LayerNorm kernels, and the attention cores above instead of
    the fused kernels.  ``modules``: the bevformer_encoder / LSS instances whose
    ``fused_geometry`` is switched off for the duration."""
    from fbbev_b200.view_transformation import backward_projection as bp_mod
    saved = (bp_mod.ms_deform_attn_fused,
             bp_mod.da_spatial_cross_attention_core,
             bp_mod._fused_linear_on)
    saved_geo = [(m, m.__dict__.get('fused_geometry')) for m in modules]
    bp_mod.ms_deform_attn_fused = msda_fused_eager
    bp_mod.da_spatial_cross_attention_core = da_sca_core_eager
    bp_mod._fused_linear_on = lambda x, *dropouts: False
    for m in modules:
        m.fused_geometry = False
    try:
        yield
    finally:
        (bp_mod.ms_deform_attn_fused,
         bp_mod.da_spatial_cross_attention_core,
         bp_mod._fused_linear_on) = saved
        for m, v in saved_geo:
            if v is None:
                m.__dict__.pop('fused_geometry', None)
            else:
                m.fused_geometry = v
