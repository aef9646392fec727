"""``bev_pool_v2`` -- host-side mirror of the reference operator.

Mirrors ``mmdet3d/ops/bev_pool_v2/bev_pool.py`` (names, argument order and
meaning, output layout):

* ``QuickCumsumCuda``   -- bev_pool.py:12-81: autograd function over the
  reference-layout kernels; ``forward`` returns ``(B, Z, Y, X, C)``.
* ``bev_pool_v2()``     -- bev_pool.py:84-90: returns the contiguous
  ``(B, C, Z, Y, X)`` tensor.  Here it is the library's dense op
  (``fbbev_bev_pool_v2_plan`` + ``_fwd_dense_planned``), which writes the
  volume in that layout directly instead of memset + kernel + transpose copy:
  two kernels that write every element once on the shapes the model runs, and
  zero fill + the interval kernel with the transpose folded into its stores on
  any other shape.
* ``voxel_pooling_prepare_v2`` -- device implementation of
  view_transformer.py:547-605 (``fbbev_voxel_prepare``).

All compute is in ``libfbbev_b200.so``; tensors must be CUDA tensors.
"""
import torch

from .. import _lib

__all__ = ['DeferredVolume', 'DeferredVolumeTrain', 'bev_pool_v2_deferred',
           'bev_pool_v2', 'bev_pool_v2_dense', 'QuickCumsumCuda',
           'voxel_pooling_prepare_v2', 'voxel_pooling_prepare_from_cams',
           'VoxelIndex']


def _feat_intervals(ranks_feat, ranks_depth, ranks_bev):
    """Re-sort the point list by feature pixel and rebuild intervals --
    QuickCumsumCuda.backward, bev_pool.py:45-55 (torch ops; plumbing)."""
    order = torch.sort(ranks_feat, stable=True)[1]
    ranks_feat, ranks_depth, ranks_bev = \
        ranks_feat[order], ranks_depth[order], ranks_bev[order]
    kept = torch.ones(ranks_bev.shape[0], device=ranks_bev.device,
                      dtype=torch.bool)
    kept[1:] = ranks_feat[1:] != ranks_feat[:-1]
    interval_starts_bp = torch.where(kept)[0].int()
    interval_lengths_bp = torch.zeros_like(interval_starts_bp)
    interval_lengths_bp[:-1] = interval_starts_bp[1:] - interval_starts_bp[:-1]
    interval_lengths_bp[-1] = ranks_bev.shape[0] - interval_starts_bp[-1]
    return (ranks_feat.contiguous(), ranks_depth.contiguous(),
            ranks_bev.contiguous(), interval_starts_bp.contiguous(),
            interval_lengths_bp.contiguous())


class QuickCumsumCuda(torch.autograd.Function):
    """Same contract as the reference class (bev_pool.py:12-81)."""

    @staticmethod
    def forward(ctx, depth, feat, ranks_depth, ranks_feat, ranks_bev,
                bev_feat_shape, interval_starts, interval_lengths):
        dev = _lib.require_cuda(depth, feat, ranks_depth, ranks_feat,
                                ranks_bev, interval_starts, interval_lengths)
        ranks_bev = ranks_bev.int()
        depth = depth.contiguous().float()
        feat = feat.contiguous().float()
        ranks_depth = ranks_depth.contiguous().int()
        ranks_feat = ranks_feat.contiguous().int()
        interval_lengths = interval_lengths.contiguous().int()
        interval_starts = interval_starts.contiguous().int()

        out = feat.new_zeros(bev_feat_shape)
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_fwd(
                _lib.ptr(depth), _lib.ptr(feat), _lib.ptr(ranks_depth),
                _lib.ptr(ranks_feat), _lib.ptr(ranks_bev),
                _lib.ptr(interval_starts), _lib.ptr(interval_lengths),
                interval_lengths.shape[0], feat.shape[-1], _lib.ptr(out),
                _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_fwd')
        ctx.save_for_backward(ranks_bev, depth, feat, ranks_feat, ranks_depth)
        return out

    @staticmethod
    def backward(ctx, out_grad):
        ranks_bev, depth, feat, ranks_feat, ranks_depth = ctx.saved_tensors
        dev = depth.device
        ranks_feat, ranks_depth, ranks_bev, starts_bp, lengths_bp = \
            _feat_intervals(ranks_feat, ranks_depth, ranks_bev)
        depth_grad = depth.new_zeros(depth.shape)
        feat_grad = feat.new_zeros(feat.shape)
        out_grad = out_grad.contiguous().float()
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_bwd(
                _lib.ptr(out_grad), _lib.ptr(depth), _lib.ptr(feat),
                _lib.ptr(ranks_depth), _lib.ptr(ranks_feat),
                _lib.ptr(ranks_bev), _lib.ptr(starts_bp), _lib.ptr(lengths_bp),
                lengths_bp.shape[0], feat.shape[-1], _lib.ptr(depth_grad),
                _lib.ptr(feat_grad), _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_bwd')
        return depth_grad, feat_grad, None, None, None, None, None, None


# Optional instrumentation: when set to an object with ``before(stream)`` /
# ``after(stream)`` methods, they are called around the launch of the dense
# pooling kernel (bench.py uses it to bracket that one kernel with CUDA events).
KERNEL_HOOK = None


def _dense_workspace(L, B, zyx, n_int, n_points, C):
    """``(cap, nbytes)``: the interval capacity of a dense-pooling workspace
    for an index of ``n_int`` interval slots, and its size in bytes.  An index
    can never hold more intervals than there are voxels: the cap bounds the
    V[n_intervals][C] workspace of the sync-free path (whose index buffers are
    n_points long) -- 1.7 GB -> 0.8 GB for 16 frames of 200x200x16."""
    cap = min(n_int, B * zyx)
    return cap, L.fbbev_bev_pool_v2_dense_workspace_bytes(B, zyx, cap,
                                                          n_points, C)


def _planned_workspace(L, dev, shape, ranks_bev, interval_starts,
                       interval_lengths, n_intervals_dev, plan):
    """``(ws, ws_bytes, n_int_cap)``: a dense-pooling workspace holding the
    plan of this index -- the one the index builder filled when it was laid
    out for the same volume, channel count and capacity (the workspace layout
    depends on them), else a new one planned here (``fbbev_bev_pool_v2_plan``,
    enqueued on the current stream of ``dev``)."""
    B, Z, Y, X, C = shape
    n_points = ranks_bev.shape[0]
    cap, ws_bytes = _dense_workspace(L, B, Z * Y * X, interval_lengths.shape[0],
                                     n_points, C)
    if plan is not None:
        pws, pbytes, pshape, pcap = plan
        if tuple(pshape) == shape and pcap == cap:
            return pws, pbytes, cap
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        rc = L.fbbev_bev_pool_v2_plan(
            _lib.ptr(ranks_bev), _lib.ptr(interval_starts),
            _lib.ptr(interval_lengths), cap, _lib.ptr(n_intervals_dev),
            n_points, C, B, Z * Y * X, _lib.ptr(ws), ws_bytes,
            _lib.stream_ptr(dev))
    _lib.check(rc, 'fbbev_bev_pool_v2_plan')
    return ws, ws_bytes, cap


def _dense_forward(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                   bev_feat_shape, interval_starts, interval_lengths,
                   n_intervals_dev, plan=None):
    dev = _lib.require_cuda(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                            interval_starts, interval_lengths, n_intervals_dev)
    shape = tuple(int(s) for s in bev_feat_shape)
    B, Z, Y, X, C = shape
    assert feat.shape[-1] == C, (feat.shape, bev_feat_shape)
    L = _lib.lib()
    out = torch.empty((B, C, Z, Y, X), dtype=torch.float32, device=dev)
    ws, ws_bytes, cap = _planned_workspace(L, dev, shape, ranks_bev,
                                           interval_starts, interval_lengths,
                                           n_intervals_dev, plan)
    hook = KERNEL_HOOK
    with torch.cuda.device(dev):
        if hook is not None:
            hook.before()
        rc = L.fbbev_bev_pool_v2_fwd_dense_planned(
            _lib.ptr(depth), _lib.ptr(feat), _lib.ptr(ranks_depth),
            _lib.ptr(ranks_feat), _lib.ptr(ranks_bev),
            _lib.ptr(interval_starts), _lib.ptr(interval_lengths),
            cap, ranks_bev.shape[0], C, B, Z * Y * X,
            _lib.ptr(out), _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev))
        if hook is not None:
            hook.after()
    _lib.check(rc, 'fbbev_bev_pool_v2_fwd_dense_planned')
    return out


class BackwardOrder:
    """The pooling backward's feature-major order of one index
    (``fbbev_bev_pool_v2_bwd_order``): the kept points sorted stably by
    ``ranks_feat`` on the device, plus every point's and voxel's interval.
    :meth:`grad_rows` and :meth:`grad_inputs` run the backward from it without
    a host sync."""

    def __init__(self, ws, n_points, n_pix, n_int_cap, C, B, zyx):
        self.ws, self.n_points, self.n_pix = ws, n_points, n_pix
        self.n_int_cap, self.C, self.B, self.zyx = n_int_cap, C, B, zyx

    def grad_rows(self, out_grad, yx, sum_z=False):
        """``(rows, sum_z)``: the gradient row of every live interval,
        (n_int_cap, C), read from the (B, C, Z, Y, X) ``out_grad``; with
        ``sum_z`` also its sum over Z, (B, C, yx) (else None)."""
        C, B = self.C, self.B
        dev = self.ws.device
        g = out_grad.contiguous().float()
        if g.data_ptr() % 16:
            g = g.clone()
        rows = torch.empty((max(self.n_int_cap, 1), C), dtype=torch.float32,
                           device=dev)
        sz = (torch.empty((B, C, yx), dtype=torch.float32, device=dev)
              if sum_z else None)
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_bwd_rows(
                _lib.ptr(g), C, B, self.zyx, yx, _lib.ptr(self.ws),
                self.ws.numel(), self.n_points, self.n_pix, _lib.ptr(rows),
                _lib.ptr(sz), _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_bwd_rows')
        return rows, sz

    def grad_inputs(self, rows, g_lss_tokens, depth, feat, yx):
        """``(depth_grad, feat_grad)`` from the rows; ``g_lss_tokens`` (B, yx,
        C) or None: the Z-mean's gradient, folded into every row.  ``rows``
        None (with ``g_lss_tokens``): the volume itself has no gradient."""
        dev = self.ws.device
        depth_grad = torch.zeros_like(depth)
        feat_grad = torch.empty_like(feat)
        if g_lss_tokens is not None:
            g_lss_tokens = g_lss_tokens.contiguous().float()
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_bwd_ordered(
                _lib.ptr(rows), _lib.ptr(g_lss_tokens), _lib.ptr(depth),
                _lib.ptr(feat), self.C, self.B, self.zyx, yx,
                _lib.ptr(self.ws), self.ws.numel(), self.n_points, self.n_pix,
                _lib.ptr(depth_grad), _lib.ptr(feat_grad),
                _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_bwd_ordered')
        return depth_grad, feat_grad


def backward_order(ranks_depth, ranks_feat, ranks_bev, interval_starts,
                   interval_lengths, n_kept_dev, n_intervals_dev, n_pix, C, B,
                   zyx, index=None):
    """The :class:`BackwardOrder` of an index, or None on a shape the ordered
    backward does not cover (``FBBEV_ERR_UNSUPPORTED``).  With ``index`` (a
    :class:`VoxelIndex`) the order is built once and kept on it."""
    n_points = ranks_bev.shape[0]
    n_int_cap = min(interval_lengths.shape[0], B * zyx)
    key = (n_pix, C, B, zyx)
    cache = getattr(index, '_bwd_orders', None)
    if cache is not None and key in cache:
        return cache[key]
    L = _lib.lib()
    dev = ranks_bev.device
    nbytes = L.fbbev_bev_pool_v2_bwd_order_workspace_bytes(n_points, n_pix, B,
                                                           zyx)

    def build(ws, ws_bytes):
        with torch.cuda.device(dev):
            return L.fbbev_bev_pool_v2_bwd_order(
                _lib.ptr(ranks_depth), _lib.ptr(ranks_feat),
                _lib.ptr(ranks_bev), _lib.ptr(interval_starts),
                _lib.ptr(interval_lengths), n_points, n_int_cap,
                _lib.ptr(n_kept_dev), _lib.ptr(n_intervals_dev), n_pix, C, B,
                zyx, _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev))
    # the shape check comes before the workspace check: a call without a
    # workspace enqueues nothing and tells an unsupported shape apart
    if build(None, 0) == _lib.ERR_UNSUPPORTED:
        return None
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    _lib.check(build(ws, nbytes), 'fbbev_bev_pool_v2_bwd_order')
    order = BackwardOrder(ws, n_points, n_pix, n_int_cap, C, B, zyx)
    # an order recorded into a CUDA graph holds data only once it replays
    if cache is not None and not torch.cuda.is_current_stream_capturing():
        cache[key] = order
    return order


class _BevPoolV2Dense(torch.autograd.Function):
    """Fused op: (B,C,Z,Y,X) out, gradient consumed in that layout."""

    @staticmethod
    def forward(ctx, depth, feat, ranks_depth, ranks_feat, ranks_bev,
                bev_feat_shape, interval_starts, interval_lengths,
                n_intervals_dev, n_kept_dev, plan=None, index=None):
        ranks_bev = ranks_bev.contiguous().int()
        depth = depth.contiguous().float()
        feat = feat.contiguous().float()
        ranks_depth = ranks_depth.contiguous().int()
        ranks_feat = ranks_feat.contiguous().int()
        interval_lengths = interval_lengths.contiguous().int()
        interval_starts = interval_starts.contiguous().int()
        out = _dense_forward(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                             bev_feat_shape, interval_starts, interval_lengths,
                             n_intervals_dev, plan)
        ctx.save_for_backward(ranks_bev, depth, feat, ranks_feat, ranks_depth,
                              n_kept_dev, interval_starts, interval_lengths,
                              n_intervals_dev)
        ctx.index = index
        return out

    @staticmethod
    def backward(ctx, out_grad):
        (ranks_bev, depth, feat, ranks_feat, ranks_depth, n_kept_dev,
         interval_starts, interval_lengths, n_intervals_dev) = ctx.saved_tensors
        B, C, Z, Y, X = out_grad.shape
        order = backward_order(ranks_depth, ranks_feat, ranks_bev,
                               interval_starts, interval_lengths, n_kept_dev,
                               n_intervals_dev, feat.numel() // C, C, B,
                               Z * Y * X, ctx.index)
        if order is not None:
            rows, _ = order.grad_rows(out_grad, Z * Y * X)
            depth_grad, feat_grad = order.grad_inputs(rows, None, depth, feat,
                                                      Z * Y * X)
            return (depth_grad, feat_grad) + (None,) * 10
        dev = depth.device
        if n_kept_dev is not None:
            # padded index buffers from the sync-free path: trim (one sync,
            # backward only)
            n = int(n_kept_dev.item())
            ranks_bev, ranks_feat, ranks_depth = \
                ranks_bev[:n], ranks_feat[:n], ranks_depth[:n]
        depth_grad = depth.new_zeros(depth.shape)
        feat_grad = feat.new_zeros(feat.shape)
        if ranks_bev.shape[0] > 0:
            ranks_feat, ranks_depth, ranks_bev, starts_bp, lengths_bp = \
                _feat_intervals(ranks_feat, ranks_depth, ranks_bev)
            out_grad = out_grad.contiguous().float()  # (B,C,Z,Y,X)
            B, C, Z, Y, X = out_grad.shape
            with torch.cuda.device(dev):
                rc = _lib.lib().fbbev_bev_pool_v2_bwd_bczyx(
                    _lib.ptr(out_grad), _lib.ptr(depth), _lib.ptr(feat),
                    _lib.ptr(ranks_depth), _lib.ptr(ranks_feat),
                    _lib.ptr(ranks_bev), _lib.ptr(starts_bp),
                    _lib.ptr(lengths_bp), lengths_bp.shape[0], C, Z * Y * X,
                    _lib.ptr(depth_grad), _lib.ptr(feat_grad),
                    _lib.stream_ptr(dev))
            _lib.check(rc, 'fbbev_bev_pool_v2_bwd_bczyx')
        return (depth_grad, feat_grad) + (None,) * 10


def bev_pool_v2_dense(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                      bev_feat_shape, interval_starts, interval_lengths,
                      n_intervals_dev=None, n_kept_dev=None, plan=None,
                      index=None):
    """Fused ``bev_pool_v2``: returns contiguous ``(B, C, Z, Y, X)``.

    ``n_intervals_dev`` / ``n_kept_dev`` (0-dim int32 CUDA tensors) mark the
    live prefix of over-allocated index buffers, as produced by
    :func:`voxel_pooling_prepare_v2` with ``sync=False``.  ``index``: the
    :class:`VoxelIndex` the index tensors belong to; the backward keeps its
    feature-major order there, so a reused index sorts once.
    """
    return _BevPoolV2Dense.apply(depth, feat, ranks_depth, ranks_feat,
                                 ranks_bev, bev_feat_shape, interval_starts,
                                 interval_lengths, n_intervals_dev, n_kept_dev,
                                 plan, index)


class DeferredVolume:
    """The pooled volume held as interval sums, materialised on demand.

    FBOCC's glue around the two projections (fbocc.py:339, 357-366)

        bev_feat = forward_projection(...)
        refined  = backward_projection(..., lss_bev=bev_feat.mean(-1), ...)
        bev_feat = refined[..., None] + bev_feat

    reads the dense volume twice and writes it twice (820 MB for 200x200x16 x
    80).  Here the forward projection stops after the interval-sum stage;
    :meth:`mean_z` produces ``bev_feat.mean(-1)`` from the ~n_int interval sums
    and :meth:`materialize` writes the volume ONCE, adding the refined BEV to
    every Z slice on the way out.  No autograd: :class:`DeferredVolumeTrain`
    is the same under autograd."""

    def __init__(self, shape, idx, ws, ws_bytes, n_int_cap, n_points):
        self.shape = shape            # (B, Z, Y, X, C)
        self._idx, self._ws, self._ws_bytes = idx, ws, ws_bytes
        self._cap, self._n_points = n_int_cap, n_points

    def mean_z(self):
        """``volume.mean(-1)`` of the (B, C, Y, X, Z) view: (B, C, Y, X), a
        channels-last-strided view of a token-major (B, Y*X, C) buffer (the
        layout BackwardProjection's BEV queries use)."""
        B, Z, Y, X, C = self.shape
        st, ln = self._idx
        dev = self._ws.device
        lss = torch.empty((B, Y * X, C), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_zmean_planned(
                _lib.ptr(st), _lib.ptr(ln), self._cap, self._n_points, C, B,
                Z * Y * X, Y * X, _lib.ptr(lss), _lib.ptr(self._ws),
                self._ws_bytes, _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_zmean_planned')
        return lss.view(B, Y, X, C).permute(0, 3, 1, 2)

    def materialize(self, add=None):
        """The contiguous (B, C, Z, Y, X) volume, plus ``add[..., None]``
        ((B, C, Y, X), e.g. the refined BEV) broadcast over Z when given."""
        B, Z, Y, X, C = self.shape
        st, ln = self._idx
        dev = self._ws.device
        out = torch.empty((B, C, Z, Y, X), dtype=torch.float32, device=dev)
        if add is not None:
            _lib.require_cuda(add)
            assert tuple(add.shape) == (B, C, Y, X), add.shape
            add = add.contiguous().float()
        with torch.cuda.device(dev):
            rc = _lib.lib().fbbev_bev_pool_v2_write_planned(
                _lib.ptr(st), _lib.ptr(ln), self._cap, self._n_points, C, B,
                Z * Y * X, Y * X, _lib.ptr(add), _lib.ptr(out),
                _lib.ptr(self._ws), self._ws_bytes, _lib.stream_ptr(dev))
        _lib.check(rc, 'fbbev_bev_pool_v2_write_planned')
        return out


class _GlueState:
    """What the two halves of :class:`DeferredVolumeTrain` share: the index,
    the interval sums (``DeferredVolume``), the backward order and the
    gradient rows the write's backward hands to the pool's backward."""

    def __init__(self, index, shape, n_pix):
        self.index, self.shape, self.n_pix = index, shape, n_pix
        self.dv = None
        self.rows = None
        self._order = None

    def order(self):
        if self._order is None:
            B, Z, Y, X, C = self.shape
            i = self.index
            self._order = backward_order(
                i.ranks_depth, i.ranks_feat, i.ranks_bev, i.interval_starts,
                i.interval_lengths, i.n_kept_dev, i.n_intervals_dev,
                self.n_pix, C, B, Z * Y * X, i)
            assert self._order is not None, self.shape  # deferred_supported
        return self._order


class _GluePool(torch.autograd.Function):
    """(depth, feat) -> ``lss_bev`` = volume.mean(-1) from the interval sums
    (``sums_planned`` + ``zmean_planned``), plus an empty ``link`` output that
    the write half takes as input, so that its backward runs first."""

    @staticmethod
    def forward(ctx, depth, feat, state):
        ctx.set_materialize_grads(False)
        B, Z, Y, X, C = state.shape
        depth = depth.contiguous().float()
        feat = feat.contiguous().float()
        i = state.index
        state.dv = bev_pool_v2_deferred(
            depth, feat, i.ranks_depth, i.ranks_feat, i.ranks_bev, state.shape,
            i.interval_starts, i.interval_lengths,
            n_intervals_dev=i.n_intervals_dev, plan=i.plan)
        ctx.save_for_backward(depth, feat)
        ctx.state = state
        return state.dv.mean_z(), depth.new_empty(0)

    @staticmethod
    def backward(ctx, g_lss, g_link):
        state = ctx.state
        rows, state.rows = state.rows, None
        if rows is None and g_lss is None:
            return None, None, None
        depth, feat = ctx.saved_tensors
        B, Z, Y, X, C = state.shape
        tok = None
        if g_lss is not None:       # (B, C, Y, X) -> token-major (B, Y*X, C)
            tok = g_lss.permute(0, 2, 3, 1).reshape(B, Y * X, C)
        dg, fg = state.order().grad_inputs(rows, tok, depth, feat, Y * X)
        return dg, fg, None


class _GlueWrite(torch.autograd.Function):
    """``refined`` -> the (B, C, Z, Y, X) volume + ``refined[..., None]``
    (``write_planned`` with the add).  Backward: one read of the volume's
    gradient G gives Σ_z G (``refined``'s gradient) and the gradient rows of
    the intervals, kept in the shared state for the pool half."""

    @staticmethod
    def forward(ctx, refined, link, state):
        ctx.set_materialize_grads(False)
        ctx.state = state
        ctx.has_add = refined is not None
        return state.dv.materialize(add=refined)

    @staticmethod
    def backward(ctx, G):
        if G is None:
            return None, None, None
        state = ctx.state
        B, Z, Y, X, C = state.shape
        rows, sz = state.order().grad_rows(G, Y * X, sum_z=ctx.has_add)
        state.rows = rows
        return (sz.view(B, C, Y, X) if ctx.has_add else None), None, None


class DeferredVolumeTrain:
    """:class:`DeferredVolume` under autograd: the same kernels and outputs,
    and a backward that reads the volume's gradient once.  FBOCC's glue
    (fbocc.py:357-366) literally differentiates ``mean(-1)`` and the re-add
    over the dense volume: three more passes over it in the backward.  Here
    the write's backward gathers the gradient rows of the intervals and Σ_z G
    in one read, and the pool's backward folds the Z-mean's gradient into the
    rows on load (``fbbev_bev_pool_v2_bwd_rows`` / ``_ordered``).  Call
    :meth:`mean_z` first; :meth:`materialize` is optional."""

    def __init__(self, depth, feat, index, shape):
        self.shape = shape
        self._depth, self._feat = depth, feat
        self._state = _GlueState(index, shape, feat.numel() // shape[-1])
        self._link = None

    def mean_z(self):
        lss, self._link = _GluePool.apply(self._depth, self._feat,
                                          self._state)
        return lss

    def materialize(self, add=None):
        assert self._link is not None, "mean_z() comes first"
        B, Z, Y, X, C = self.shape
        if add is not None:
            _lib.require_cuda(add)
            assert tuple(add.shape) == (B, C, Y, X), add.shape
        return _GlueWrite.apply(add, self._link, self._state)


def deferred_supported(bev_feat_shape):
    B, Z, Y, X, C = (int(s) for s in bev_feat_shape)
    return (C % 4 == 0 and C <= 512 and (Z * Y * X) % 4 == 0 and
            (Y * X) % 4 == 0 and B * Z * Y * X <= 2 ** 31 - 1)


def bev_pool_v2_deferred(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                         bev_feat_shape, interval_starts, interval_lengths,
                         n_intervals_dev=None, plan=None):
    """Plan + interval sums of the dense op; returns a :class:`DeferredVolume`
    (``fbbev_bev_pool_v2_plan`` + ``fbbev_bev_pool_v2_sums_planned``)."""
    dev = _lib.require_cuda(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                            interval_starts, interval_lengths, n_intervals_dev)
    shape = tuple(int(s) for s in bev_feat_shape)
    B, Z, Y, X, C = shape
    assert feat.shape[-1] == C and deferred_supported(bev_feat_shape)
    depth = depth.contiguous().float()
    feat = feat.contiguous().float()
    rb, rd, rf = (t.contiguous().int() for t in
                  (ranks_bev, ranks_depth, ranks_feat))
    st, ln = interval_starts.contiguous().int(), interval_lengths.contiguous().int()
    L = _lib.lib()
    n_points = rb.shape[0]
    ws, ws_bytes, cap = _planned_workspace(L, dev, shape, rb, st, ln,
                                           n_intervals_dev, plan)
    with torch.cuda.device(dev):
        _lib.check(L.fbbev_bev_pool_v2_sums_planned(
            _lib.ptr(depth), _lib.ptr(feat), _lib.ptr(rd), _lib.ptr(rf),
            _lib.ptr(rb), _lib.ptr(st), _lib.ptr(ln), cap, n_points, C, B,
            Z * Y * X, _lib.ptr(ws), ws_bytes, _lib.stream_ptr(dev)),
            'fbbev_bev_pool_v2_sums_planned')
    return DeferredVolume((B, Z, Y, X, C), (st, ln), ws, ws_bytes, cap, n_points)


def bev_pool_v2(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                bev_feat_shape, interval_starts, interval_lengths):
    """Drop-in for the reference ``bev_pool_v2`` (bev_pool.py:84-90).

    depth ``(B,N,D,H,W)``, feat ``(B,N,H,W,C)`` (any strides), int index
    tensors as returned by ``voxel_pooling_prepare_v2``; ``bev_feat_shape`` =
    ``(B, Z, Y, X, C)``.  Returns contiguous ``(B, C, Z, Y, X)``.
    Requires the interval list to be ordered by voxel rank (it always is when
    it comes from ``voxel_pooling_prepare_v2``); use ``QuickCumsumCuda`` for
    arbitrary interval lists.
    """
    return bev_pool_v2_dense(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                             bev_feat_shape, interval_starts, interval_lengths)


class VoxelIndex:
    """Index tensors of one ``voxel_pooling_prepare_v2`` call, device-resident.

    The five index tensors are over-allocated (``n_points`` entries); the live
    prefix lengths are ``counts[0]`` (points kept) and ``counts[1]``
    (intervals), int32 on the device.  Nothing here forces a host sync.
    """

    def __init__(self, ranks_bev, ranks_depth, ranks_feat, interval_starts,
                 interval_lengths, counts, plan=None):
        self.ranks_bev = ranks_bev
        self.ranks_depth = ranks_depth
        self.ranks_feat = ranks_feat
        self.interval_starts = interval_starts
        self.interval_lengths = interval_lengths
        self.counts = counts
        # (workspace, bytes, shape (B, Z, Y, X, C), n_int_cap) of a dense-pooling
        # plan the index builder filled while scanning (no plan launch needed)
        self.plan = plan
        # the pooling backward's BackwardOrder per (n_pix, C, B, Z*Y*X)
        self._bwd_orders = {}

    @property
    def n_kept_dev(self):
        return self.counts[0]

    @property
    def n_intervals_dev(self):
        return self.counts[1]

    def trimmed(self):
        """Exact-length tensors as the reference returns them (host sync);
        five ``None`` when nothing is kept (view_transformer.py:598-599)."""
        n_kept, n_int = (int(v) for v in self.counts.tolist())
        if n_int == 0:
            return None, None, None, None, None
        return (self.ranks_bev[:n_kept], self.ranks_depth[:n_kept],
                self.ranks_feat[:n_kept], self.interval_starts[:n_int],
                self.interval_lengths[:n_int])


def _plan_workspace(L, dev, B, gs, n_pts, pool_channels):
    """Dense-pooling workspace for the index builder to fill the plan into, or
    ``(None, 0, None)`` without ``pool_channels``."""
    if not pool_channels:
        return None, 0, None
    X, Y, Z = int(gs[0]), int(gs[1]), int(gs[2])
    C = int(pool_channels)
    cap, nbytes = _dense_workspace(L, B, Z * Y * X, n_pts, n_pts, C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    return ws, nbytes, (ws, nbytes, (B, Z, Y, X, C), cap)


def _depth_arg(depth, n_pts, dev):
    """Contiguous fp32 depth tensor for the depth-threshold sparsification
    (necks/view_transformer.py:556-557), or None."""
    if depth is None:
        return None
    d = depth.detach().contiguous().float()
    assert d.numel() == n_pts and d.device == dev
    return d


def _prepare(entry, geometry, dev, B, N, D, H, W, grid_lower_bound,
             grid_interval, grid_size, pool_channels, depth, depth_thresh):
    """Build a :class:`VoxelIndex` with the C entry point named ``entry``,
    called with its ``geometry`` arguments followed by the depth threshold,
    sizes, grid, index buffers, workspace and pooling plan laid out here."""
    lo, iv, gs = ([float(v) for v in torch.as_tensor(t).float().cpu()]
                  for t in (grid_lower_bound, grid_interval, grid_size))
    n_pts = B * N * D * H * W
    n_vox = B * int(gs[0]) * int(gs[1]) * int(gs[2])
    L = _lib.lib()
    idx = torch.empty((5, n_pts), dtype=torch.int32, device=dev)
    counts = torch.empty(2, dtype=torch.int32, device=dev)
    ws_bytes = L.fbbev_voxel_prepare_workspace_bytes(n_pts, n_vox)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    pws, pbytes, plan = _plan_workspace(L, dev, B, gs, n_pts, pool_channels)
    dprob = _depth_arg(depth, n_pts, dev)
    with torch.cuda.device(dev):
        rc = getattr(L, entry)(
            *geometry, _lib.ptr(dprob), float(depth_thresh), B, N, D, H, W,
            _lib.c_floats(lo), _lib.c_floats(iv), _lib.c_floats(gs),
            *(_lib.ptr(t) for t in idx), _lib.ptr(counts), _lib.ptr(ws),
            ws_bytes, int(pool_channels or 0), _lib.ptr(pws), pbytes,
            _lib.stream_ptr(dev))
    _lib.check(rc, entry)
    return VoxelIndex(*idx, counts, plan)


def voxel_pooling_prepare_v2(coor, grid_lower_bound, grid_interval, grid_size,
                             pool_channels=None, depth=None,
                             depth_thresh=0.01):
    """Device ``voxel_pooling_prepare_v2`` (view_transformer.py:547-605).

    coor ``(B,N,D,H,W,3)`` fp32 CUDA; the three grid descriptors are the
    3-element float32 tensors of ``create_grid_infos`` (:384-387) -- host
    tensors or python sequences.  Returns a :class:`VoxelIndex`;
    ``pool_channels`` = C of the pooling call that will consume the index lets
    the builder fill that call's plan on the way (``VoxelIndex.plan``).
    ``depth`` (B,N,D,H,W): additionally drop the points whose depth
    probability is <= ``depth_thresh`` -- LSSViewTransformer2's sparsification
    (necks/view_transformer.py:556-557).
    """
    dev = _lib.require_cuda(coor)
    coor = coor.contiguous().float()
    B, N, D, H, W, three = coor.shape
    assert three == 3
    return _prepare('fbbev_voxel_prepare', (_lib.ptr(coor),), dev, B, N, D, H,
                    W, grid_lower_bound, grid_interval, grid_size,
                    pool_channels, depth, depth_thresh)


def voxel_pooling_prepare_from_cams(frustum_axes, inv_post_rots, post_trans,
                                    cam2ego, trans, bda, depth_bins,
                                    grid_lower_bound, grid_interval,
                                    grid_size, pool_channels=None, depth=None,
                                    depth_thresh=0.01):
    """``get_lidar_coor`` + ``voxel_pooling_prepare_v2`` in one pass
    (view_transformer.py:458-498, 547-605): the (B,N,D,H,W,3) coordinate
    tensor is never materialised (``fbbev_voxel_prepare_cams``).

    frustum_axes = (u [W], v [H], d [D]) CUDA float tensors;
    inv_post_rots / cam2ego (B,N,3,3); post_trans / trans (B,N,3); bda (B,3,3).
    Returns a :class:`VoxelIndex`, bit-identical to the two-step route: the
    kernel rounds every 3x3 product as torch's broadcast matmul does on this
    device (see include/fbbev_b200.h, ``_lib.matmul_order_flags``)."""
    fu, fv, fd = (t.contiguous().float() for t in frustum_axes)
    dev = _lib.require_cuda(fu, fv, fd, inv_post_rots, post_trans, cam2ego,
                            trans, bda)
    order = _lib.matmul_order_flags(inv_post_rots, cam2ego, bda)
    mats = [t.contiguous().float() for t in
            (inv_post_rots, post_trans, cam2ego, trans, bda)]
    B, N = mats[0].shape[:2]
    D, H, W = fd.shape[0], fv.shape[0], fu.shape[0]
    assert D == depth_bins
    geometry = [_lib.ptr(t) for t in (fu, fv, fd, *mats)] + [order]
    return _prepare('fbbev_voxel_prepare_cams', geometry, dev, B, N, D, H, W,
                    grid_lower_bound, grid_interval, grid_size, pool_channels,
                    depth, depth_thresh)
