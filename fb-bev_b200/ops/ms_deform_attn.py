"""Multi-scale deformable attention operators -- host-side mirror.

* ``MultiScaleDeformableAttnFunction_fp32`` mirrors the reference's autograd
  wrapper over mmcv's ``_ext`` op
  (``.../bevformer_utils/multi_scale_deformable_attn_function.py:99-172``):
  same ``apply(value, spatial_shapes, level_start_index, sampling_locations,
  attention_weights, im2col_step)`` signature, fp32 forced as at :102.
  ``MultiScaleDeformableAttnFunction_fp16`` maps to the same function, exactly
  like the reference does at spatial_cross_attention_depth.py:580-583.
* ``ms_deform_attn_fused`` / ``da_spatial_cross_attention_core`` expose the two
  fused kernels (see ``include/fbbev_b200.h``); ``MsdaFusedFunction`` /
  ``DaScaFunction`` make them differentiable with the fused backward kernels.

All compute is in ``libfbbev_b200.so``; CUDA tensors only.
"""
import torch
from torch.autograd.function import Function, once_differentiable

from .. import _lib

__all__ = ['MultiScaleDeformableAttnFunction_fp32',
           'MultiScaleDeformableAttnFunction_fp16', 'ms_deform_attn_forward',
           'ms_deform_attn_fused', 'ms_deform_attn_unfused',
           'MsdaFusedFunction', 'ms_deform_attn_fused_autograd',
           'DaScaFunction', 'fused_grad_supported',
           'da_spatial_cross_attention_core',
           'da_spatial_cross_attention_core_autograd', 'da_sca_prepare',
           'point_sampling',
           'bev_query_init', 'tokens_to_map',
           'needs_grad']


def needs_grad(*tensors):
    """True when autograd is recording and one of ``tensors`` takes part in it:
    the plain fused calls must not be used then (their outputs carry no
    grad_fn and would silently cut the graph); the autograd Functions over them
    or the differentiable routes are."""
    return torch.is_grad_enabled() and any(
        t is not None and t.requires_grad for t in tensors)


def _i64(t, dev):
    return t.to(device=dev, dtype=torch.int64).contiguous()


def deterministic():
    """Deterministic mode: on exactly when
    ``torch.are_deterministic_algorithms_enabled()``.  The autograd Functions
    read it in forward and keep it for their backward, which then calls the
    ``*_bwd_det`` entry points (no float atomics, a defined summation order);
    the cross-attention forward then takes its global-memory kernel."""
    return torch.are_deterministic_algorithms_enabled()


def _run_backward(name, det, dev, args, ws_args):
    """Calls backward entry point ``name`` with ``args`` on ``dev``'s current
    stream; in deterministic mode its ``name + '_det'`` twin instead, with a
    workspace sized by ``name + '_det_workspace_bytes'(*ws_args)``."""
    L = _lib.lib()
    with torch.cuda.device(dev):
        if det:
            name += '_det'
            nb = getattr(L, name + '_workspace_bytes')(*ws_args)
            ws = torch.empty(max(nb, 1), dtype=torch.uint8, device=dev)
            rc = getattr(L, name)(*args, _lib.ptr(ws), nb,
                                  _lib.stream_ptr(dev))
        else:
            rc = getattr(L, name)(*args, _lib.stream_ptr(dev))
    _lib.check(rc, name)


def ms_deform_attn_forward(value, spatial_shapes, level_start_index,
                           sampling_locations, attention_weights,
                           im2col_step=64):
    """Same contract as ``ext_module.ms_deform_attn_forward``
    (multi_scale_deformable_attn_function.py:127-133).  ``im2col_step`` is
    accepted and ignored (no batch-chunking restriction here)."""
    dev = _lib.require_cuda(value, sampling_locations, attention_weights)
    value = value.contiguous().float()
    loc = sampling_locations.contiguous().float()
    attw = attention_weights.contiguous().float()
    ss, ls = _i64(spatial_shapes, dev), _i64(level_start_index, dev)
    bs, n_value, heads, ch = value.shape
    _, nq, _, levels, points, _ = loc.shape
    out = value.new_empty((bs, nq, heads * ch))
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_msda_fwd(
            _lib.ptr(value), _lib.ptr(ss), _lib.ptr(ls), _lib.ptr(loc),
            _lib.ptr(attw), bs, n_value, heads, ch, levels, nq, points,
            _lib.ptr(out), _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_msda_fwd')
    return out


class MultiScaleDeformableAttnFunction_fp32(Function):

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index,
                sampling_locations, attention_weights, im2col_step):
        value = value.float()
        sampling_locations = sampling_locations.float()
        attention_weights = attention_weights.float()
        ctx.im2col_step = im2col_step
        ctx.det = deterministic()
        output = ms_deform_attn_forward(
            value, value_spatial_shapes, value_level_start_index,
            sampling_locations, attention_weights, im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes,
                              value_level_start_index, sampling_locations,
                              attention_weights)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, lstart, loc, attw = ctx.saved_tensors
        dev = value.device
        value, loc, attw = value.contiguous(), loc.contiguous(), \
            attw.contiguous()
        ss, ls = _i64(shapes, dev), _i64(lstart, dev)
        # samples outside the map leave their loc / attw gradient untouched
        grad_loc = torch.zeros_like(loc)
        grad_attw = torch.zeros_like(attw)
        # the atomic kernel adds into grad_value; the deterministic one
        # writes it whole
        grad_value = (torch.empty_like if ctx.det else torch.zeros_like)(value)
        go = grad_output.contiguous().float()
        bs, n_value, heads, ch = value.shape
        _, nq, _, levels, points, _ = loc.shape
        _run_backward(
            'fbbev_msda_bwd', ctx.det, dev,
            (_lib.ptr(value), _lib.ptr(ss), _lib.ptr(ls), _lib.ptr(loc),
             _lib.ptr(attw), _lib.ptr(go), bs, n_value, heads, ch, levels, nq,
             points, _lib.ptr(grad_value), _lib.ptr(grad_loc),
             _lib.ptr(grad_attw)),
            (nq, n_value, heads, levels, points))
        return grad_value, None, None, grad_loc, grad_attw, None


# spatial_cross_attention_depth.py:580-583 maps both dtypes to the fp32 op
MultiScaleDeformableAttnFunction_fp16 = MultiScaleDeformableAttnFunction_fp32


def ms_deform_attn_fused(value, spatial_shapes, level_start_index,
                         reference_points, sampling_offsets, attention_logits,
                         map_width=0):
    """softmax + location arithmetic + sampling of mmcv
    ``MultiScaleDeformableAttention.forward`` in one kernel.

    value (bs, n_value, heads, ch); reference_points (bs, nq, levels, 2);
    sampling_offsets (bs, nq, heads, levels, points, 2) raw Linear output;
    attention_logits (bs, nq, heads, levels, points) raw Linear output.
    ``map_width``: for self-attention over the map itself (one level, one
    query per value pixel) the map's width -- a scheduling hint (square query
    patches per block), results do not depend on it.
    Returns (bs, nq, heads*ch).  Forward only (inference path)."""
    dev = _lib.require_cuda(value, reference_points, sampling_offsets,
                            attention_logits)
    value = value.contiguous().float()
    ref = reference_points.contiguous().float()
    off = sampling_offsets.contiguous().float()
    lg = attention_logits.contiguous().float()
    ss, ls = _i64(spatial_shapes, dev), _i64(level_start_index, dev)
    bs, n_value, heads, ch = value.shape
    _, nq, _, levels, points, _ = off.shape
    out = value.new_empty((bs, nq, heads * ch))
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_msda_fused_fwd(
            _lib.ptr(value), _lib.ptr(ss), _lib.ptr(ls), _lib.ptr(ref),
            _lib.ptr(off), _lib.ptr(lg), bs, n_value, heads, ch, levels, nq,
            points, int(map_width), _lib.ptr(out), _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_msda_fused_fwd')
    return out


# head widths / anchor counts the fused kernels are built for (HeadWidths /
# ZAnchors in csrc/msda_common.cuh; tests/test_fused_backward_abi.py checks
# that the two agree)
FUSED_HEAD_WIDTHS = (4, 8, 10, 16, 20, 32, 64)
FUSED_Z_ANCHORS = (1, 2, 4, 8)


def fused_grad_supported(value, *tensors, num_Z_anchors=1):
    """True when :class:`MsdaFusedFunction` / :class:`DaScaFunction` can train
    this call: every tensor CUDA fp32 and a head width (and Z) the kernels are
    built for.  Otherwise the differentiable routes
    (:func:`ms_deform_attn_unfused`,
    :func:`da_spatial_cross_attention_core_autograd`) serve it."""
    return (all(t.is_cuda and t.dtype == torch.float32
                for t in (value,) + tensors) and
            value.shape[-1] in FUSED_HEAD_WIDTHS and
            num_Z_anchors in FUSED_Z_ANCHORS)


class MsdaFusedFunction(Function):
    """Autograd over the fused self-attention core: forward
    ``fbbev_msda_fused_fwd`` (as :func:`ms_deform_attn_fused`), backward
    ``fbbev_msda_fused_bwd``, which recomputes softmax and locations from the
    saved inputs (``fbbev_msda_fused_bwd_det`` in deterministic mode, see
    :func:`deterministic`).  Gradients reach value, sampling_offsets and
    attention_logits; reference_points get none."""

    @staticmethod
    def forward(ctx, value, spatial_shapes, level_start_index,
                reference_points, sampling_offsets, attention_logits,
                map_width=0):
        dev = _lib.require_cuda(value, reference_points, sampling_offsets,
                                attention_logits)
        value = value.contiguous().float()
        ref = reference_points.contiguous().float()
        off = sampling_offsets.contiguous().float()
        lg = attention_logits.contiguous().float()
        ss, ls = _i64(spatial_shapes, dev), _i64(level_start_index, dev)
        out = ms_deform_attn_fused(value, ss, ls, ref, off, lg, map_width)
        ctx.save_for_backward(value, ss, ls, ref, off, lg)
        ctx.det = deterministic()
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        value, ss, ls, ref, off, lg = ctx.saved_tensors
        need = ctx.needs_input_grad
        dev = value.device
        # the atomic kernel adds into grad_value; the deterministic one
        # writes it whole
        gv = (torch.empty_like if ctx.det else torch.zeros_like)(value) \
            if need[0] else None
        goff = torch.empty_like(off) if need[4] else None
        glg = torch.empty_like(lg) if need[5] else None
        go = grad_out.contiguous().float()
        bs, n_value, heads, ch = value.shape
        _, nq, _, levels, points, _ = off.shape
        _run_backward(
            'fbbev_msda_fused_bwd', ctx.det, dev,
            (_lib.ptr(value), _lib.ptr(ss), _lib.ptr(ls), _lib.ptr(ref),
             _lib.ptr(off), _lib.ptr(lg), _lib.ptr(go), bs, n_value, heads,
             ch, levels, nq, points, _lib.ptr(gv), _lib.ptr(goff),
             _lib.ptr(glg)),
            (nq, n_value, heads, levels, points))
        return gv, None, None, None, goff, glg, None


def ms_deform_attn_fused_autograd(value, spatial_shapes, level_start_index,
                                  reference_points, sampling_offsets,
                                  attention_logits, map_width=0):
    """:func:`ms_deform_attn_fused` with gradients (:class:`MsdaFusedFunction`);
    same arguments and result."""
    return MsdaFusedFunction.apply(value, spatial_shapes, level_start_index,
                                   reference_points, sampling_offsets,
                                   attention_logits, map_width)


def ms_deform_attn_unfused(value, spatial_shapes, level_start_index,
                           reference_points, sampling_offsets,
                           attention_logits, map_width=0, im2col_step=64):
    """Differentiable twin of :func:`ms_deform_attn_fused`: softmax and the
    sampling locations in PyTorch (as mmcv's module does), the sampling through
    ``MultiScaleDeformableAttnFunction_fp32`` (forward ``fbbev_msda_fwd``,
    backward ``fbbev_msda_bwd``).  Same arguments and result."""
    lg = attention_logits
    w = lg.flatten(3).softmax(-1).view_as(lg)
    wh = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]], -1)
    loc = reference_points[:, :, None, :, None, :] + \
        sampling_offsets / wh[None, None, None, :, None, :]
    return MultiScaleDeformableAttnFunction_fp32.apply(
        value, spatial_shapes, level_start_index, loc, w, im2col_step)


def da_spatial_cross_attention_core_autograd(
        value, depth_prob, reference_points_cam, bev_query_depth, per_cam_mask,
        sampling_offsets, attention_logits, spatial_shapes, level_start_index,
        dbound, num_Z_anchors, im2col_step=64):
    """Differentiable twin of :func:`da_spatial_cross_attention_core` (same
    arguments and result) for training: every (camera, query) pair is evaluated
    densely and the pairs a camera does not see are masked out of the mean, so
    there is no ``nonzero()`` host synchronisation and gradients reach
    ``value`` (-> value_proj, image features), the offsets / logits (-> their
    Linears, the BEV queries) and ``depth_prob`` (-> the depth net), as through
    the reference's ``MultiScaleDeformableAttnFunction`` calls
    (spatial_cross_attention_depth.py:584-595)."""
    apply = MultiScaleDeformableAttnFunction_fp32.apply
    N, bs, nq, Z, _ = reference_points_cam.shape
    _, _, heads, L, P, _ = sampling_offsets.shape
    DC = depth_prob.shape[-1]
    E = value.shape[2] * value.shape[3]
    assert Z == num_Z_anchors and P % Z == 0
    w = attention_logits.flatten(3).softmax(-1).view_as(attention_logits)
    wh = torch.stack([spatial_shapes[..., 1], spatial_shapes[..., 0]],
                     -1).to(sampling_offsets.dtype)
    off = sampling_offsets / wh[None, None, None, :, None, :]
    ref = reference_points_cam.permute(1, 0, 2, 3, 4)       # (bs, N, nq, Z, 2)
    # point index = p * Z + z   (:563-570)
    loc = ref[:, :, :, None, None, None, :, :] + off.view(
        bs, 1, nq, heads, L, P // Z, Z, 2)
    loc = loc.reshape(bs * N, nq, heads, L, P, 2)
    d = bev_query_depth
    if d.dim() == 5:
        d = d[..., 0]
    bins = torch.floor((d.permute(1, 0, 2, 3) - dbound[0]) / dbound[2])
    bins = bins.clamp(0, DC - 1).long().reshape(bs * N, nq, Z, 1)
    depth_ref = ref.reshape(bs * N, nq * Z, 1, 1, 1, 2).contiguous()
    dsamp = apply(depth_prob.unsqueeze(2).contiguous(), spatial_shapes[0:1],
                  level_start_index[0:1], depth_ref,
                  torch.ones_like(depth_ref[..., 0]), im2col_step)
    dw = dsamp.view(bs * N, nq, Z, DC).gather(-1, bins).squeeze(-1)
    dw = dw.unsqueeze(2).repeat(1, 1, P // Z, 1).reshape(bs * N, nq, P)
    wts = w.unsqueeze(1).expand(bs, N, nq, heads, L, P).reshape(
        bs * N, nq, heads, L, P) * dw[:, :, None, None, :]      # :592
    out = apply(value, spatial_shapes, level_start_index, loc, wts,
                im2col_step).view(bs, N, nq, E)
    # mask bytes: != 0 visible, bit 0 counted (see bev_mask_fold)
    m8 = per_cam_mask if per_cam_mask.dtype == torch.uint8 else \
        per_cam_mask.to(torch.uint8)
    seen = (m8 != 0).any(-1).permute(1, 0, 2)                # (bs, N, nq)
    counted = ((m8 & 1) != 0).any(-1).permute(1, 0, 2)
    slots = (out * seen[..., None].to(out.dtype)).sum(1)
    count = counted.sum(1).clamp(min=1).to(out.dtype)
    return slots / count[..., None]


def _mask_u8(per_cam_mask):
    mask = per_cam_mask.contiguous()
    return mask if mask.dtype == torch.uint8 else mask.view(torch.uint8) \
        if mask.dtype == torch.bool else mask.to(torch.uint8)


def bev_mask_fold(per_cam_mask, bev_mask):
    """``per_cam_mask_list & bev_mask[None, :, :, None]`` with the reference's
    empty-camera rule (spatial_cross_attention_depth.py:156-169, 213-214) as a
    device-side pass (``fbbev_bev_mask_fold``): the result goes to the fused
    cross-attention as its mask (1 = visible and counted, 2 = visible, not
    counted), so a ``bev_mask`` needs no nonzero() / re-batching loops.
    per_cam_mask (n_cams, bs, nq, Z) bool / uint8; bev_mask (bs, nq)."""
    dev = _lib.require_cuda(per_cam_mask, bev_mask)
    mask = _mask_u8(per_cam_mask)
    bev = _mask_u8(bev_mask != 0 if bev_mask.dtype not in
                   (torch.bool, torch.uint8) else bev_mask)
    n_cams, bs, nq, Z = mask.shape
    assert tuple(bev.shape) == (bs, nq)
    L = _lib.lib()
    out = torch.empty_like(mask)
    ws_bytes = L.fbbev_bev_mask_fold_workspace_bytes(bs, n_cams)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = L.fbbev_bev_mask_fold(_lib.ptr(mask), _lib.ptr(bev), bs, n_cams,
                                   nq, Z, _lib.ptr(out), _lib.ptr(ws),
                                   ws_bytes, _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_bev_mask_fold')
    return out


def da_sca_prepare(per_cam_mask, bs, nq, n_value, heads, ch, levels, points, Z):
    """The mask-only part of the camera-resident cross-attention (per-camera
    visible-query counts, zero-filled output): ``fbbev_da_sca_prologue``.  The
    encoder runs it on its side stream right after ``point_sampling``; the
    result goes to :func:`da_spatial_cross_attention_core` as ``prepared``.
    Returns None when the shape takes the global-memory kernel."""
    dev = _lib.require_cuda(per_cam_mask)
    mask = _mask_u8(per_cam_mask)
    n_cams = mask.shape[0]
    L = _lib.lib()
    ws_bytes = L.fbbev_da_sca_workspace_bytes(bs, n_cams)
    ws = torch.empty(max(ws_bytes, 4), dtype=torch.uint8, device=dev)
    out = torch.empty((bs, nq, heads * ch), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = L.fbbev_da_sca_prologue(
            _lib.ptr(mask), bs, n_cams, nq, n_value, heads, ch, levels, points,
            Z, _lib.ptr(out), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev))
    if rc == -3:        # FBBEV_ERR_UNSUPPORTED: global-memory kernel, no prologue
        return None
    _lib.check(rc, 'fbbev_da_sca_prologue')
    return out, ws, ws_bytes, mask


def da_spatial_cross_attention_core(value, depth_prob, reference_points_cam,
                                    bev_query_depth, per_cam_mask,
                                    sampling_offsets, attention_logits,
                                    spatial_shapes, level_start_index, dbound,
                                    num_Z_anchors, prepared=None):
    """Fused depth-aware spatial cross-attention between the input Linears and
    ``output_proj`` (spatial_cross_attention_depth.py:156-216, 540-595).

    value (bs*n_cams, n_value, heads, ch)        value_proj(feat)
    depth_prob (bs*n_cams, H0*W0, DC)            pred_img_depth, pixel-major
    reference_points_cam (n_cams, bs, nq, Z, 2)
    bev_query_depth (n_cams, bs, nq, Z[, 1])
    per_cam_mask (n_cams, bs, nq, Z) bool
    sampling_offsets (bs, nq, heads, levels, points, 2), attention_logits
    (bs, nq, heads, levels, points): raw Linear outputs on the BEV queries.
    Returns slots / clamp(count, 1): (bs, nq, heads*ch).
    In deterministic mode (:func:`deterministic`) no workspace is passed and
    ``prepared`` is not used: the global-memory kernel, which loops over the
    cameras inside a thread, runs instead of the camera-resident one, whose
    per-camera additions have no fixed order."""
    det = deterministic()
    if det:
        prepared = None
    dev = _lib.require_cuda(value, depth_prob, reference_points_cam,
                            bev_query_depth, per_cam_mask, sampling_offsets,
                            attention_logits)
    value = value.contiguous().float()
    depth_prob = depth_prob.contiguous().float()
    ref = reference_points_cam.contiguous().float()
    rdep = bev_query_depth.contiguous().float()
    mask = _mask_u8(per_cam_mask) if prepared is None else prepared[3]
    off = sampling_offsets.contiguous().float()
    lg = attention_logits.contiguous().float()
    ss, ls = _i64(spatial_shapes, dev), _i64(level_start_index, dev)
    bn, n_value, heads, ch = value.shape
    n_cams, bs, nq, Z, _ = ref.shape
    assert bn == bs * n_cams and Z == num_Z_anchors
    _, _, _, levels, points, _ = off.shape
    DC = depth_prob.shape[-1]
    L = _lib.lib()
    if prepared is not None:
        out, ws, ws_bytes, _ = prepared
        assert tuple(out.shape) == (bs, nq, heads * ch)
    elif det:
        out = value.new_empty((bs, nq, heads * ch))
        ws, ws_bytes = None, 0
    else:
        out = value.new_empty((bs, nq, heads * ch))
        ws_bytes = L.fbbev_da_sca_workspace_bytes(bs, n_cams)
        ws = torch.empty(max(ws_bytes, 4), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = L.fbbev_da_sca_fwd(
            _lib.ptr(value), _lib.ptr(depth_prob), _lib.ptr(ref),
            _lib.ptr(rdep), _lib.ptr(mask), _lib.ptr(off), _lib.ptr(lg),
            _lib.ptr(ss), _lib.ptr(ls), _lib.c_floats(dbound), bs, n_cams, nq,
            n_value, heads, ch, levels, points, Z, DC, _lib.ptr(out),
            _lib.ptr(ws), ws_bytes, 1 if prepared is not None else 0,
            _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_da_sca_fwd')
    return out


class DaScaFunction(Function):
    """Autograd over the fused depth-aware cross-attention:
    ``DaScaFunction.apply`` takes the positional arguments of
    :func:`da_spatial_cross_attention_core` (without ``prepared``).  The
    forward is that function (the camera-resident kernel runs as in
    inference); the backward, ``fbbev_da_sca_bwd``, recomputes everything from
    the saved inputs and visits only the (camera, query) pairs the mask marks
    seen.  In deterministic mode (:func:`deterministic`, read in forward) the
    forward takes the global-memory kernel and the backward is
    ``fbbev_da_sca_bwd_det``.  Gradients reach value, depth_prob, sampling_offsets and
    attention_logits; reference_points_cam / bev_query_depth / the mask get
    none.  ``depth_prob`` may be the permuted (B*N, HW, DC) view of the depth
    net's output: its gradient flows back through the view."""

    @staticmethod
    def forward(ctx, value, depth_prob, reference_points_cam, bev_query_depth,
                per_cam_mask, sampling_offsets, attention_logits,
                spatial_shapes, level_start_index, dbound, num_Z_anchors):
        dev = _lib.require_cuda(value, depth_prob, reference_points_cam,
                                bev_query_depth, per_cam_mask,
                                sampling_offsets, attention_logits)
        args = [t.contiguous().float() for t in
                (value, depth_prob, reference_points_cam, bev_query_depth)]
        mask = _mask_u8(per_cam_mask)
        off = sampling_offsets.contiguous().float()
        lg = attention_logits.contiguous().float()
        ss, ls = _i64(spatial_shapes, dev), _i64(level_start_index, dev)
        ctx.det = deterministic()
        out = da_spatial_cross_attention_core(*args, mask, off, lg, ss, ls,
                                              dbound, num_Z_anchors)
        ctx.save_for_backward(*args, mask, off, lg, ss, ls)
        ctx.dbound = [float(v) for v in dbound]
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        value, depth_prob, ref, rdep, mask, off, lg, ss, ls = ctx.saved_tensors
        need = ctx.needs_input_grad
        dev = value.device
        # the two atomic targets are zero-filled (the deterministic kernels
        # write them whole); the others are written whole
        acc = torch.empty_like if ctx.det else torch.zeros_like
        gv = acc(value) if need[0] else None
        gdp = acc(depth_prob) if need[1] else None
        goff = torch.empty_like(off) if need[5] else None
        glg = torch.empty_like(lg) if need[6] else None
        go = grad_out.contiguous().float()
        bn, n_value, heads, ch = value.shape
        n_cams, bs, nq, Z, _ = ref.shape
        _, _, _, levels, points, _ = off.shape
        DC = depth_prob.shape[-1]
        _run_backward(
            'fbbev_da_sca_bwd', ctx.det, dev,
            (_lib.ptr(value), _lib.ptr(depth_prob), _lib.ptr(ref),
             _lib.ptr(rdep), _lib.ptr(mask), _lib.ptr(off), _lib.ptr(lg),
             _lib.ptr(ss), _lib.ptr(ls), _lib.c_floats(ctx.dbound),
             _lib.ptr(go), bs, n_cams, nq, n_value, heads, ch, levels, points,
             Z, DC, _lib.ptr(gv), _lib.ptr(gdp), _lib.ptr(goff),
             _lib.ptr(glg)),
            (n_cams, nq, n_value, heads, ch, levels, points, Z, DC))
        return (gv, gdp, None, None, None, goff, glg, None, None, None, None)


def bev_query_init(embedding, lss_bev):
    """``embedding[:, None] + lss_bev.flatten(2).permute(2, 0, 1)`` of
    BackwardProjection.forward (backward_projection.py:93-97) in one pass
    (``fbbev_bev_query_init``).  embedding (nq, E); lss_bev (bs, E, h, w).
    Returns the (nq, bs, E) tensor of the reference as a view of a
    (bs, nq, E)-contiguous buffer."""
    dev = _lib.require_cuda(embedding, lss_bev)
    emb = embedding.detach().contiguous().float()
    bs, E = lss_bev.shape[:2]
    nq = emb.shape[0]
    assert emb.shape[1] == E and lss_bev[0, 0].numel() == nq
    if lss_bev.dim() == 4 and lss_bev.stride(1) == 1 and \
            lss_bev.permute(0, 2, 3, 1).is_contiguous():
        # token-major already (e.g. DeferredVolume.mean_z()): a plain add
        tok = lss_bev.permute(0, 2, 3, 1).reshape(bs, nq, E).float()
        return (emb.unsqueeze(0) + tok).permute(1, 0, 2)
    lss = lss_bev.contiguous().float()
    out = torch.empty((bs, nq, E), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_bev_query_init(
            _lib.ptr(emb), _lib.ptr(lss), bs, nq, E, _lib.ptr(out),
            _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_bev_query_init')
    return out.permute(1, 0, 2)


def tokens_to_map(tokens, bev_h, bev_w, out=None):
    """``tokens.permute(0, 2, 1).view(bs, E, bev_h, bev_w).contiguous()``
    (backward_projection.py:131-133) as one transposing kernel
    (``fbbev_tokens_to_map``); ``out``: optional destination (e.g. a gather
    slot).  Returns None when the shape is not covered (caller falls back)."""
    bs, nq, E = tokens.shape
    if not tokens.is_cuda or tokens.dtype != torch.float32 or nq % 4 or E % 4 \
            or not tokens.is_contiguous():
        return None
    if out is None:
        out = torch.empty((bs, E, bev_h, bev_w), dtype=torch.float32,
                          device=tokens.device)
    elif not out.is_contiguous() or tuple(out.shape) != (bs, E, bev_h, bev_w):
        return None
    with torch.cuda.device(tokens.device):
        rc = _lib.lib().fbbev_tokens_to_map(
            _lib.ptr(tokens), bs, nq, E, _lib.ptr(out),
            _lib.stream_ptr(tokens.device))
    _lib.check(rc, 'fbbev_tokens_to_map')
    return out


def point_sampling(axes, inv_bda, trans, ego2cam, post_rots, post_trans,
                   input_size, eps=1e-5):
    """One-kernel ``bevformer_encoder.point_sampling``
    (bevformer_encoder.py:92-120), ``fbbev_point_sampling``.

    axes = (X [nX], Y [nY], Z [nZ]) voxel-centre coordinates; inv_bda (B,3,3);
    ego2cam / post_rots (B,N,3,3); trans / post_trans (B,N,3);
    input_size = (H_in, W_in).  Returns ``(reference_points_cam (N,B,nq,Z,2),
    mask (N,B,nq,Z) bool, depth (N,B,nq,Z,1))`` with nq = nY*nX, bit-identical
    to the eager chain on this device."""
    X, Y, Z = (t.contiguous().float() for t in axes)
    dev = _lib.require_cuda(X, Y, Z, inv_bda, trans, ego2cam, post_rots,
                            post_trans)
    B, N = trans.shape[:2]
    nX, nY, nZ = X.shape[0], Y.shape[0], Z.shape[0]
    # the eager chain's three broadcast matmuls, viewed as it views them
    order = _lib.matmul_order_codes(
        [inv_bda.float().view(B, 1, 1, 1, 1, 3, 3),
         ego2cam.float().view(B, N, 1, 1, 1, 3, 3),
         post_rots.float().view(B, N, 1, 1, 1, 3, 3)], (B, N, nY, nX, nZ, 3))
    mats = [t.contiguous().float() for t in
            (inv_bda, trans, ego2cam, post_rots, post_trans)]
    nq = nX * nY
    ref = torch.empty((N, B, nq, nZ, 2), dtype=torch.float32, device=dev)
    dep = torch.empty((N, B, nq, nZ, 1), dtype=torch.float32, device=dev)
    msk = torch.empty((N, B, nq, nZ), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.lib().fbbev_point_sampling(
            _lib.ptr(X), _lib.ptr(Y), _lib.ptr(Z), nX, nY, nZ,
            _lib.ptr(mats[0]), _lib.ptr(mats[1]), _lib.ptr(mats[2]),
            _lib.ptr(mats[3]), _lib.ptr(mats[4]), order, B, N,
            float(input_size[1]), float(input_size[0]), float(eps),
            float(1.0 - eps), _lib.ptr(ref), _lib.ptr(dep), _lib.ptr(msk),
            _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_point_sampling')
    return ref, msk.view(torch.bool), dep
