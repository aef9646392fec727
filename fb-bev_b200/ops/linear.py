"""Row-wise Linear (+ bias, ReLU, residual, LayerNorm) on the Hopper tensor cores (wgmma).

Host side of ``fbbev_linear_fwd`` / ``fbbev_ffn_fwd`` (include/fbbev_b200.h): the
nn.Linear / LayerNorm / residual chain of the reference's encoder layer
(bevformer_encoder.py:251-377, spatial_cross_attention_depth.py:219, 420-427)
as one kernel per Linear (one for the whole FFN).  With autograd recording,
:class:`LinearTF32Function` keeps the forward on the same kernel and forms the
three gradient products with plain library GEMMs (cuBLAS through torch).
The LayerNorm-epilogue Linear and the whole FFN train on their fused kernels
too (:class:`LinearLNTrainFunction`, :class:`FFNTrainFunction`): the forward
is the inference arithmetic plus the saved row statistics, the backward runs
the LayerNorm backward and the FFN's data path as kernels of their own.
"""
import torch

from .. import _lib

MAX_N = 192  # widest column block of one launch
# the packed images cached on a weight: of W, of W as FFN W1 blocks, and of W^T
# in both layouts (the backward kernels' operands)
_CACHE_ATTRS = ("_fbbev_packed", "_fbbev_packed_ffn", "_fbbev_packed_t",
                "_fbbev_packed_ffn_t")
# set on a tensor that a training step captured into a CUDA graph reads: the
# graph's replays (its optimizer step) may change it in place without moving
# its version counter, so no cache keyed on that counter holds anything derived
# from it from then on
_GRAPHED_ATTR = "_fbbev_graph_trained"


def mark_graph_trained(*tensors):
    """Mark parameters read by a training step under CUDA-graph capture and
    drop the images cached on them.  From then on no cache keyed on their
    version counters (the packed images here, :func:`linear_pair`'s
    concatenation, ``CustormLearnedPositionalEncoding``'s encoding) holds
    anything derived from them, so eager and inference calls after replays
    see their current values."""
    for t in tensors:
        if t is None:
            continue
        for a in _CACHE_ATTRS:
            if hasattr(t, a):
                delattr(t, a)
        try:
            setattr(t, _GRAPHED_ATTR, True)
        except AttributeError:  # a tensor type without a __dict__
            pass


def graph_trained(*tensors):
    """True when one of ``tensors`` was marked by :func:`mark_graph_trained`."""
    return any(t is not None and getattr(t, _GRAPHED_ATTR, False)
               for t in tensors)


def _cached(weight, attr, key, train):
    """The cached image ``attr`` of ``weight`` under ``key``, or None; decides
    whether the caller may cache the image it builds (returns ``(hit, may)``).

    A training call (``train``) captured into a CUDA graph records its pack
    launch: the graph then re-forms the image from the weight's storage on
    every replay, so in-place weight updates between or inside replays
    (optimizer steps) are honoured.  Such a call neither reads nor writes the
    cache -- a hit would bake the capture-time weights into the graph, and an
    image allocated from the graph's pool would be overwritten by replays --
    and it marks the weight so that no later call caches its image either.
    Inference captures (grad disabled) keep the cache: their graph treats the
    weights as constants (see :func:`invalidate`)."""
    if train and torch.cuda.is_current_stream_capturing():
        mark_graph_trained(weight)
        return None, False
    if graph_trained(weight):
        return None, False
    hit = getattr(weight, attr, None)
    if hit is not None and hit[0] == key:
        return hit[1], True
    return None, True


def _pack(weight, transpose=False, train=False):
    """hi / lo split image of `weight` (n, k), one block per <= MAX_N columns;
    with ``transpose`` the image of ``weight.T``.

    Cached ON the weight tensor (so it dies with it and can never be mistaken
    for another tensor's) and keyed by storage address and version counter, so
    an optimizer step or ``load_state_dict`` triggers a re-pack.  ``train``:
    the call belongs to a training step, which never caches under CUDA-graph
    capture (:func:`_cached`)."""
    attr = "_fbbev_packed_t" if transpose else "_fbbev_packed"
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), weight.device)
    hit, may_cache = _cached(weight, attr, key, train)
    if hit is not None:
        return hit
    L = _lib.lib()
    w = weight.detach()
    w = (w.t() if transpose else w).contiguous().float()
    n, k = w.shape
    blocks = []
    for n0 in range(0, n, MAX_N):
        n1 = min(n, n0 + MAX_N)
        nbytes = L.fbbev_linear_packed_bytes(n1 - n0, k)
        buf = torch.empty(nbytes // 4, dtype=torch.float32, device=w.device)
        _lib.check(L.fbbev_linear_pack(_lib.ptr(w[n0:n1]), n1 - n0, k, _lib.ptr(buf),
                                       _lib.stream_ptr(w.device)), "fbbev_linear_pack")
        blocks.append((n0, n1, buf))
    if may_cache:
        try:
            setattr(weight, attr, (key, blocks))
        except AttributeError:  # a tensor type without a __dict__: no caching
            pass
    return blocks


def invalidate(obj):
    """Drop the packed-weight images cached for ``obj`` (an nn.Module, walked
    recursively, or a single weight tensor).

    The caches key on ``Tensor._version``, which in-place updates through
    ``param.data`` (EMA hooks, some checkpoint loaders) do NOT bump -- call
    this after such an update.  ``optimizer.step()``, ``load_state_dict`` and
    ordinary in-place ops on the parameter are detected automatically.

    A CUDA graph captured with gradients off (inference) reads the images the
    capture found and treats the weights as constants: after
    ``load_state_dict`` or any other weight change, call this and capture
    again.  Training steps captured with autograd recording re-form the
    images inside the graph and need neither (see :func:`_cached`)."""
    if isinstance(obj, torch.Tensor):
        for attr in _CACHE_ATTRS:
            if hasattr(obj, attr):
                delattr(obj, attr)
        return
    for m in obj.modules():
        m.__dict__.pop("_pair_cache", None)
        m.__dict__.pop("_pos_cache", None)   # the learned positional encoding
        m.__dict__.pop("_pos_tokens", None)  # and its token-major copy
        m.__dict__.pop("_fuse_cache", None)  # TemporalFusion's folded weights
        for p in m.parameters(recurse=False):
            for attr in _CACHE_ATTRS:
                if hasattr(p, attr):
                    delattr(p, attr)


def ln_supported(n):
    """The LayerNorm epilogue takes rows of up to 80 columns (linear_tf32.cu,
    kMaxLnN: the encoder's embed_dims)."""
    return 0 < n <= 80


def supported(x, weight):
    n, k = weight.shape
    return (x.is_cuda and x.dtype == torch.float32 and weight.dtype == torch.float32
            and k % 4 == 0 and n % 4 == 0 and not torch.is_grad_enabled())


def linear_fused(x, weight, bias=None, relu=False, residual=None, ln_weight=None,
                 ln_bias=None, eps=1e-5, train=False):
    """``LN(act(x @ weight.T + bias) + residual)`` with every part optional.
    ``train``: the call is the forward of a training step (weight image per
    :func:`_pack`)."""
    _lib.require_cuda(x)
    n, k = weight.shape
    assert x.shape[-1] == k
    lead = x.shape[:-1]
    x2 = x.reshape(-1, k)
    if x2.stride(-1) != 1 or x2.stride(0) % 4 or x2.data_ptr() % 16:
        x2 = x2.contiguous()
    m = x2.shape[0]
    y = torch.empty((m, n), dtype=torch.float32, device=x.device)
    r2 = None
    if residual is not None:
        r2 = residual.reshape(-1, n)
        if r2.stride(-1) != 1 or r2.stride(0) % 4 or r2.data_ptr() % 16:
            r2 = r2.contiguous()
    blocks = _pack(weight, train=train)
    if ln_weight is not None and not ln_supported(n):
        raise _lib.FbbevError("LayerNorm epilogue: n = %d does not fit" % n)
    L = _lib.lib()
    sp = _lib.stream_ptr(x.device)
    b = bias.detach().contiguous() if bias is not None else None
    for n0, n1, buf in blocks:
        _lib.check(L.fbbev_linear_fwd(
            _lib.ptr(x2), x2.stride(0), _lib.ptr(buf),
            _lib.ptr(b[n0:n1]) if b is not None else None,
            _lib.ptr(r2[:, n0:n1]) if r2 is not None else None,
            r2.stride(0) if r2 is not None else 0,
            _lib.ptr(ln_weight) if ln_weight is not None else None,
            _lib.ptr(ln_bias) if ln_bias is not None else None,
            m, k, n1 - n0, int(bool(relu)), float(eps),
            _lib.ptr(y[:, n0:n1]), y.stride(0), sp), "fbbev_linear_fwd")
    return y.view(*lead, n)


def _rows(t, k):
    """(-1, k) view of ``t`` usable by the kernels (dense rows, 16-byte
    aligned), copying only when the layout demands it."""
    t2 = t.reshape(-1, k)
    if t2.stride(-1) != 1 or t2.stride(0) % 4 or t2.data_ptr() % 16:
        t2 = t2.contiguous()
    return t2


def linear_pair(x, weight_a, bias_a, weight_b, bias_b, cache, x_add=None):
    """``(x @ weight_a.T + bias_a, x @ weight_b.T + bias_b)`` as ONE launch when
    both fit a column block (sampling_offsets + attention_weights of an
    attention module: same input, one consumer kernel).  With ``x_add`` the
    input is ``x + x_add`` (``query + query_pos``), added in the kernel's loader.

    ``cache`` is a dict owned by the calling module; it keeps the concatenated
    weight / bias, keyed by the parameters' storage and version counters, and
    is bypassed for parameters a captured training step updates
    (:func:`mark_graph_trained`)."""
    _lib.require_cuda(x)
    na, k = weight_a.shape
    nb = weight_b.shape[0]
    if na + nb > MAX_N or na % 4 or nb % 4 or (bias_a is None) != (bias_b is None):
        if x_add is not None:
            x = x + x_add
        return (linear_fused(x, weight_a, bias_a), linear_fused(x, weight_b, bias_b))
    key = tuple((t.data_ptr(), t._version) for t in
                (weight_a, weight_b, bias_a, bias_b) if t is not None)
    graphed = graph_trained(weight_a, weight_b, bias_a, bias_b)
    if graphed:
        cache.pop("pair", None)
    hit = None if graphed else cache.get("pair")
    if hit is None or hit[0] != key:
        w = torch.cat((weight_a.detach(), weight_b.detach()), 0).float().contiguous()
        b = None if bias_a is None else torch.cat(
            (bias_a.detach(), bias_b.detach()), 0).float().contiguous()
        hit = (key, w, b)
        if not graphed:
            cache["pair"] = hit
    _, w, b = hit
    lead = x.shape[:-1]
    x2 = _rows(x, k)
    m = x2.shape[0]
    xa = None
    if x_add is not None:
        if x_add.shape != x.shape:
            x_add = x_add.expand_as(x)
        xa = _rows(x_add, k)
    ya = torch.empty((m, na), dtype=torch.float32, device=x.device)
    yb = torch.empty((m, nb), dtype=torch.float32, device=x.device)
    (_, _, buf), = _pack(w)
    L = _lib.lib()
    _lib.check(L.fbbev_linear_fwd_split(
        _lib.ptr(x2), x2.stride(0), _lib.ptr(xa),
        xa.stride(0) if xa is not None else 0, _lib.ptr(buf), _lib.ptr(b), m, k,
        na + nb, na, 0, _lib.ptr(ya), na, _lib.ptr(yb), nb,
        _lib.stream_ptr(x.device)), "fbbev_linear_fwd_split")
    return ya.view(*lead, na), yb.view(*lead, nb)


def _pack_ffn_w1(weight, transpose=False, train=False):
    """W1 (hidden, embed) as hidden / 80 separately packed 80-row blocks, one
    buffer (the layout ``fbbev_ffn_fwd`` streams); with ``transpose`` the same
    layout of ``weight.T`` (W2^T for ``fbbev_ffn_bwd``).  Cached like
    :func:`_pack`."""
    attr = "_fbbev_packed_ffn_t" if transpose else "_fbbev_packed_ffn"
    key = (weight.data_ptr(), weight._version, tuple(weight.shape), weight.device)
    hit, may_cache = _cached(weight, attr, key, train)
    if hit is not None:
        return hit
    L = _lib.lib()
    w = weight.detach()
    w = (w.t() if transpose else w).contiguous().float()
    hidden, k = w.shape
    assert hidden % 80 == 0
    per = L.fbbev_linear_packed_bytes(80, k) // 4
    buf = torch.empty(per * (hidden // 80), dtype=torch.float32, device=w.device)
    for c in range(hidden // 80):
        _lib.check(L.fbbev_linear_pack(
            _lib.ptr(w[80 * c:80 * c + 80]), 80, k, _lib.ptr(buf[per * c:]),
            _lib.stream_ptr(w.device)), "fbbev_linear_pack")
    if may_cache:
        try:
            setattr(weight, attr, (key, buf))
        except AttributeError:
            pass
    return buf


def ffn_supported(x, w1, w2):
    hidden, embed = w1.shape
    return (supported(x, w1) and tuple(w2.shape) == (embed, hidden) and
            bool(_lib.lib().fbbev_ffn_supported(embed, hidden)))


def ffn_fused(x, w1, b1, w2, b2, residual=None, ln_weight=None, ln_bias=None,
              eps=1e-5):
    """``LN(residual + relu(x @ w1.T + b1) @ w2.T + b2)`` as ONE kernel
    (``fbbev_ffn_fwd``): the hidden activation never leaves the SM."""
    _lib.require_cuda(x)
    hidden, embed = w1.shape
    assert x.shape[-1] == embed and tuple(w2.shape) == (embed, hidden)
    lead = x.shape[:-1]
    x2 = _rows(x, embed)
    m = x2.shape[0]
    r2 = _rows(residual, embed) if residual is not None else None
    y = torch.empty((m, embed), dtype=torch.float32, device=x.device)
    w1p = _pack_ffn_w1(w1)
    (_, _, w2p), = _pack(w2)
    _lib.check(_lib.lib().fbbev_ffn_fwd(
        _lib.ptr(x2), x2.stride(0), _lib.ptr(w1p),
        _lib.ptr(b1.detach().contiguous()) if b1 is not None else None,
        _lib.ptr(w2p),
        _lib.ptr(b2.detach().contiguous()) if b2 is not None else None,
        _lib.ptr(r2), r2.stride(0) if r2 is not None else 0,
        _lib.ptr(ln_weight) if ln_weight is not None else None,
        _lib.ptr(ln_bias) if ln_bias is not None else None,
        m, embed, hidden, float(eps), _lib.ptr(y), y.stride(0),
        _lib.stream_ptr(x.device)), "fbbev_ffn_fwd")
    return y.view(*lead, embed)


class LinearTF32Function(torch.autograd.Function):
    """``act(x @ weight.T + bias) + residual`` with the forward on the wgmma
    kernel (``fbbev_linear_fwd``: same 3xTF32 arithmetic as inference) and the
    backward as plain library GEMMs::

        g  = grad * (y > 0)           (ReLU only)
        dx = g @ weight    dW = g^T @ x    db = sum_rows(g)    dresidual = grad

    The reference trains these layers through cuBLAS in both directions
    (nn.Linear); here only the backward is a library call.  LayerNorm stays a
    torch op on this route (its backward needs the row statistics)."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu, residual):
        assert not (relu and residual is not None)
        y = linear_fused(
            x.detach(), weight.detach(),
            None if bias is None else bias.detach(), relu=relu,
            residual=None if residual is None else residual.detach(),
            train=True)
        ctx.relu = relu
        ctx.has_bias = bias is not None
        ctx.has_res = residual is not None
        ctx.save_for_backward(x, weight, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, grad):
        x, weight, y = ctx.saved_tensors
        g = grad * (y > 0).to(grad.dtype) if ctx.relu else grad
        n, k = weight.shape
        g2 = g.reshape(-1, n)
        gx = gw = gb = gr = None
        if ctx.needs_input_grad[0]:
            gx = (g2 @ weight).view(x.shape)
        if ctx.needs_input_grad[1]:
            gw = g2.t() @ x.reshape(-1, k)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = g2.sum(0)
        if ctx.has_res and ctx.needs_input_grad[4]:
            gr = grad
        return gx, gw, gb, None, gr


def linear_train(x, weight, bias=None, relu=False, residual=None):
    """Differentiable ``act(x @ weight.T + bias) + residual``; forward on the
    tensor-core kernel.  Shapes the kernel does not take (k or n not a multiple
    of 4) must be handled by the caller."""
    if relu and residual is not None:
        return LinearTF32Function.apply(x, weight, bias, True, None) + residual
    return LinearTF32Function.apply(x, weight, bias, relu, residual)


# ------------------------- training on the fused kernels -------------------------

def _f32_cuda(*ts):
    return all(t.is_cuda and t.dtype == torch.float32 for t in ts if t is not None)


def ln_train_supported(x, weight, norm):
    """``norm(x @ weight.T + bias + residual)`` trains on the LayerNorm
    epilogue (:class:`LinearLNTrainFunction`): CUDA fp32, k % 4 == 0,
    n % 4 == 0, n <= 80, an affine LayerNorm."""
    n, k = weight.shape
    return (_f32_cuda(x, weight, norm.weight, norm.bias) and
            norm.weight is not None and norm.bias is not None and
            k % 4 == 0 and n % 4 == 0 and ln_supported(n) and
            tuple(norm.normalized_shape) == (n,))


def ffn_train_supported(x, w1, w2, norm=None):
    """The FFN (+ LayerNorm) trains on the fused kernels
    (:class:`FFNTrainFunction`) for the shapes ``fbbev_ffn_fwd`` takes."""
    hidden, embed = w1.shape
    return (_f32_cuda(x, w1, w2) and tuple(w2.shape) == (embed, hidden) and
            bool(_lib.lib().fbbev_ffn_supported(embed, hidden)) and
            (norm is None or ln_train_supported(x, w2, norm)))


def _layernorm_bwd(g2, xhat, rstd, gamma):
    """dz, dgamma, dbeta of ``y = xhat * gamma + beta`` (``fbbev_layernorm_bwd``)."""
    m, n = xhat.shape
    L = _lib.lib()
    dz = torch.empty_like(xhat)
    dgb = torch.empty(2, n, dtype=torch.float32, device=xhat.device)
    ws = torch.empty(L.fbbev_layernorm_bwd_workspace_bytes(m, n), dtype=torch.uint8,
                     device=xhat.device)
    _lib.check(L.fbbev_layernorm_bwd(
        _lib.ptr(g2), g2.stride(0), _lib.ptr(xhat), _lib.ptr(rstd),
        _lib.ptr(gamma.detach()), m, n, _lib.ptr(dz), dz.stride(0),
        _lib.ptr(dgb[0]), _lib.ptr(dgb[1]), _lib.ptr(ws), ws.numel(),
        _lib.stream_ptr(xhat.device)), "fbbev_layernorm_bwd")
    return dz, dgb[0], dgb[1]


class LinearLNTrainFunction(torch.autograd.Function):
    """``LN(x @ weight.T + bias + residual)`` with the LayerNorm in the wgmma
    kernel's epilogue, as at inference (``fbbev_linear_fwd_ln_train``: the
    same bits, plus x^ and 1 / sigma).  Backward::

        dz = LayerNorm backward (fbbev_layernorm_bwd; also dgamma, dbeta)
        dx = dz @ weight  (fbbev_linear_fwd on the packed image of weight.T)
        dW = dz^T @ x    db = sum_rows(dz)    dresidual = dz

    The weight and bias gradients are library GEMMs / sums."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, ln_weight, ln_bias, eps):
        n, k = weight.shape
        lead = x.shape[:-1]
        x2 = _rows(x.detach(), k)
        m = x2.shape[0]
        r2 = _rows(residual.detach(), n) if residual is not None else None
        dev = x.device
        y = torch.empty((m, n), dtype=torch.float32, device=dev)
        xhat = torch.empty((m, n), dtype=torch.float32, device=dev)
        rstd = torch.empty((m,), dtype=torch.float32, device=dev)
        (_, _, buf), = _pack(weight, train=True)
        _lib.check(_lib.lib().fbbev_linear_fwd_ln_train(
            _lib.ptr(x2), x2.stride(0), _lib.ptr(buf),
            _lib.ptr(bias.detach().contiguous()) if bias is not None else None,
            _lib.ptr(r2), r2.stride(0) if r2 is not None else 0,
            _lib.ptr(ln_weight.detach()), _lib.ptr(ln_bias.detach()),
            m, k, n, float(eps), _lib.ptr(y), y.stride(0), _lib.ptr(xhat),
            _lib.ptr(rstd), _lib.stream_ptr(dev)), "fbbev_linear_fwd_ln_train")
        ctx.has_bias = bias is not None
        ctx.res_shape = None if residual is None else residual.shape
        ctx.x_shape = x.shape
        ctx.save_for_backward(x2, weight, xhat, rstd, ln_weight)
        return y.view(*lead, n)

    @staticmethod
    def backward(ctx, grad):
        x2, weight, xhat, rstd, ln_weight = ctx.saved_tensors
        n, k = weight.shape
        dz, dgamma, dbeta = _layernorm_bwd(_rows(grad, n), xhat, rstd, ln_weight)
        gx = gw = gb = gr = None
        if ctx.needs_input_grad[0]:
            gx = torch.empty((dz.shape[0], k), dtype=torch.float32, device=dz.device)
            _run_blocks(dz, _pack(weight, transpose=True, train=True), n, gx)
            gx = gx.view(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            gw = dz.t() @ x2
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = dz.sum(0)
        if ctx.res_shape is not None and ctx.needs_input_grad[3]:
            gr = dz.view(ctx.res_shape)
        return (gx, gw, gb, gr, dgamma if ctx.needs_input_grad[4] else None,
                dbeta if ctx.needs_input_grad[5] else None, None)


def _run_blocks(x2, blocks, k, y):
    """``y = x2 @ W.T`` for a packed W (``blocks`` of :func:`_pack`)."""
    L = _lib.lib()
    sp = _lib.stream_ptr(x2.device)
    for n0, n1, buf in blocks:
        _lib.check(L.fbbev_linear_fwd(
            _lib.ptr(x2), x2.stride(0), _lib.ptr(buf), None, None, 0, None, None,
            x2.shape[0], k, n1 - n0, 0, 0.0, _lib.ptr(y[:, n0:n1]), y.stride(0), sp),
            "fbbev_linear_fwd")


def linear_ln_train(x, weight, bias, residual, norm):
    """Differentiable ``norm(x @ weight.T + bias + residual)`` on the fused
    kernels; the caller checks :func:`ln_train_supported`."""
    return LinearLNTrainFunction.apply(x, weight, bias, residual, norm.weight,
                                       norm.bias, norm.eps)


class FFNTrainFunction(torch.autograd.Function):
    """``LN(identity + relu(x @ w1.T + b1) @ w2.T + b2)`` (LayerNorm and
    identity optional) with the forward on the fused FFN kernel, as at
    inference (``fbbev_ffn_fwd_train``: the same bits, plus the hidden
    activation ``act`` and the LayerNorm's x^ and 1 / sigma).  Backward::

        dz  = LayerNorm backward (fbbev_layernorm_bwd), or the output gradient
        dh  = (dz @ w2) * [act > 0]           } one kernel, fbbev_ffn_bwd
        dx  = dh @ w1 (+ dz: identity is x)   }
        dW2 = dz^T @ act   db2 = sum(dz)   dW1 = dh^T @ x   db1 = sum(dh)
        didentity = dz  (identity another tensor)

    ``res``: 0 no identity, 1 the identity is ``x``, 2 it is ``identity``."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, identity, ln_weight, ln_bias, eps, res):
        hidden, embed = w1.shape
        lead = x.shape[:-1]
        x2 = _rows(x.detach(), embed)
        m = x2.shape[0]
        r2 = (x2 if res == 1 else
              _rows(identity.detach(), embed) if res == 2 else None)
        dev = x.device
        y = torch.empty((m, embed), dtype=torch.float32, device=dev)
        act = torch.empty((m, hidden), dtype=torch.float32, device=dev)
        xhat = rstd = None
        if ln_weight is not None:
            xhat = torch.empty((m, embed), dtype=torch.float32, device=dev)
            rstd = torch.empty((m,), dtype=torch.float32, device=dev)
        (_, _, w2p), = _pack(w2, train=True)
        _lib.check(_lib.lib().fbbev_ffn_fwd_train(
            _lib.ptr(x2), x2.stride(0), _lib.ptr(_pack_ffn_w1(w1, train=True)),
            _lib.ptr(b1.detach().contiguous()) if b1 is not None else None,
            _lib.ptr(w2p),
            _lib.ptr(b2.detach().contiguous()) if b2 is not None else None,
            _lib.ptr(r2), r2.stride(0) if r2 is not None else 0,
            _lib.ptr(ln_weight.detach()) if ln_weight is not None else None,
            _lib.ptr(ln_bias.detach()) if ln_bias is not None else None,
            m, embed, hidden, float(eps), _lib.ptr(y), y.stride(0), _lib.ptr(act),
            _lib.ptr(xhat), _lib.ptr(rstd), _lib.stream_ptr(dev)),
            "fbbev_ffn_fwd_train")
        ctx.res = res
        ctx.has_b = (b1 is not None, b2 is not None)
        ctx.x_shape = x.shape
        ctx.id_shape = identity.shape if res == 2 else None
        ctx.save_for_backward(x2, w1, w2, act, xhat, rstd, ln_weight)
        return y.view(*lead, embed)

    @staticmethod
    def backward(ctx, grad):
        x2, w1, w2, act, xhat, rstd, ln_weight = ctx.saved_tensors
        hidden, embed = w1.shape
        g2 = _rows(grad, embed)
        dgamma = dbeta = None
        if ln_weight is not None:
            dz, dgamma, dbeta = _layernorm_bwd(g2, xhat, rstd, ln_weight)
        else:
            dz = g2
        m = dz.shape[0]
        dh = torch.empty_like(act)
        dx = torch.empty((m, embed), dtype=torch.float32, device=dz.device)
        (_, _, w1tp), = _pack(w1, transpose=True, train=True)
        _lib.check(_lib.lib().fbbev_ffn_bwd(
            _lib.ptr(dz), dz.stride(0), _lib.ptr(act),
            _lib.ptr(_pack_ffn_w1(w2, transpose=True, train=True)), _lib.ptr(w1tp),
            int(ctx.res == 1), m, embed, hidden, _lib.ptr(dh), _lib.ptr(dx),
            dx.stride(0), _lib.stream_ptr(dz.device)), "fbbev_ffn_bwd")
        need = ctx.needs_input_grad
        gw1 = dh.t() @ x2 if need[1] else None
        gb1 = dh.sum(0) if ctx.has_b[0] and need[2] else None
        gw2 = dz.t() @ act if need[3] else None
        gb2 = dz.sum(0) if ctx.has_b[1] and need[4] else None
        gid = dz.view(ctx.id_shape) if ctx.res == 2 and need[5] else None
        return (dx.view(ctx.x_shape) if need[0] else None, gw1, gb1, gw2, gb2, gid,
                dgamma if need[6] else None, dbeta if need[7] else None, None, None)


def ffn_train(x, w1, b1, w2, b2, identity=None, add_identity=True, norm=None):
    """Differentiable ``norm(identity + relu(x @ w1.T + b1) @ w2.T + b2)`` on
    the fused kernels (``identity`` defaults to ``x``; none without
    ``add_identity``); the caller checks :func:`ffn_train_supported`."""
    if not add_identity:
        res, identity = 0, None
    elif identity is None or identity is x:
        res, identity = 1, None
    else:
        res = 2
    return FFNTrainFunction.apply(
        x, w1, b1, w2, b2, identity,
        None if norm is None else norm.weight, None if norm is None else norm.bias,
        1e-5 if norm is None else norm.eps, res)
