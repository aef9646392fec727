"""GPU tests of the depth supervision (csrc/depth_loss.cu, ops/depth_loss.py,
CM_DepthNetTail / LSSViewTransformerBEVDepth ``get_depth_loss``).

Labels and d preds are compared bit for bit with the eager torch expression of
get_downsampled_gt_depth / get_depth_loss (depth_net.py:396-450,
view_transformer.py:1036-1081) evaluated on the same GPU, and with the
reference's golden; the loss, whose sum order differs, within 1e-5 relative."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from depth_loss_ref64 import labels_ref, loss_ref64

pytestmark = pytest.mark.gpu
DEV = "cuda"
FBOCC = (2.0, 42.0, 0.5)


def _dl():
    from fbbev_b200.ops import depth_loss
    return depth_loss


# -- the eager expression, as the reference evaluates it ----------------------
def eager_onehot(gt, ds, cfg, D):
    H, W = gt.shape[-2:]
    x = gt.reshape(-1, H // ds, ds, W // ds, ds)
    x = x.permute(0, 1, 3, 2, 4).reshape(-1, ds * ds)
    x = torch.where(x == 0.0, 1e5 * torch.ones_like(x), x)
    m = torch.min(x, dim=-1).values
    t = (m - (cfg[0] - cfg[2])) / cfg[2]        # a CUDA tensor by Python floats
    t = torch.where((t < D + 1) & (t >= 0.0), t, torch.zeros_like(t))
    return F.one_hot(t.long(), num_classes=D + 1)[:, 1:].float()


def eager_loss(gt, preds, ds, cfg, weight):
    D, h, w = preds.shape[-3:]
    onehot = eager_onehot(gt, ds, cfg, D)
    p = preds.reshape(-1, D, h, w).permute(0, 2, 3, 1).reshape(-1, D)
    fg = torch.max(onehot, dim=1).values > 0.0
    s = F.binary_cross_entropy(p[fg], onehot[fg], reduction='none').sum()
    return weight * (s / max(1.0, fg.sum()))


def eager_grad(gt, preds, ds, cfg, weight):
    p = preds.detach().clone().requires_grad_()
    loss = eager_loss(gt, p, ds, cfg, weight)
    loss.backward()
    return loss.detach(), p.grad


def ours(gt, preds, ds, cfg, weight):
    p = preds.detach().clone().requires_grad_()
    loss = _dl().depth_loss(gt, p, ds, cfg, weight)
    loss.backward()
    return loss.detach(), p.grad


def lidar_gt(BN, H, W, lo, hi, seed, density=0.05, spill=True):
    """Sparse depths; with ``spill`` some lie below lo - step or beyond hi."""
    g = torch.Generator().manual_seed(seed)
    hit = torch.rand(BN, H, W, generator=g) < density
    if spill:
        val = torch.rand(BN, H, W, generator=g) * (hi - lo + 10.0) + lo - 3.0
    else:
        val = torch.rand(BN, H, W, generator=g) * (hi - lo) + lo
    return torch.where(hit, val, torch.zeros(())).to(DEV)


def softmax_preds(BN, D, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(BN, D, h, w, generator=g) * 3.0).softmax(1).to(DEV)


def _rel(a, b):
    a, b = float(a), float(b)
    return abs(a - b) / max(abs(b), 1e-30)


def _assert_bitwise(got, want, what):
    if not torch.equal(got, want):
        bad = (got != want).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} elements differ, first "
                             f"at {i}: {got[i].item()!r} vs {want[i].item()!r}")


# -- golden --------------------------------------------------------------------
@pytest.mark.parametrize("case", ["fbocc", "lineage", "ds8"])
def test_golden(case):
    z = load_golden("d_depth_loss")
    c = {k.split("/", 1)[1]: v for k, v in z.items()
         if k.startswith(case + "/")}
    D, ds, wt = int(c["D"]), int(c["downsample"]), float(c["loss_weight"])
    cfg = tuple(float(v) for v in c["depth_cfg"])
    gt = torch.from_numpy(c["gt"]).to(DEV)
    preds = torch.from_numpy(c["preds"]).to(DEV)
    labels = _dl().depth_labels(gt, ds, cfg, D)
    np.testing.assert_array_equal(labels.cpu().numpy(), c["labels"])
    onehot = _dl().downsampled_gt_depth(gt, ds, cfg, D)
    np.testing.assert_array_equal(onehot.cpu().numpy(),
                                  c["onehot"].astype(np.float32))
    loss, grad = ours(gt, preds, ds, cfg, wt)
    assert _rel(loss, c["loss"]) <= 1e-5
    ref64 = loss_ref64(labels_ref(c["gt"], ds, cfg, D), c["preds"], D, wt)
    assert _rel(loss, ref64) <= 1e-5
    _assert_bitwise(grad.cpu(), torch.from_numpy(c["grad"]), "d preds")


# -- labels at the edges, against the eager expression on this GPU ------------
def _edge_values(cfg, D):
    lo, hi, step = cfg
    f32 = np.float32
    vals = []
    for k in range(-2, D + 3):
        base = f32(lo - step + k * step)
        for n in range(-3, 4):
            v = base
            for _ in range(abs(n)):
                v = np.nextafter(v, f32(np.inf if n > 0 else -np.inf))
            vals.append(v)
    for edge in (lo - step, lo, hi - step, hi):
        e = f32(edge)
        vals += [np.nextafter(np.nextafter(e, f32(-np.inf)), f32(-np.inf)),
                 np.nextafter(e, f32(-np.inf)), e, np.nextafter(e, f32(np.inf)),
                 np.nextafter(np.nextafter(e, f32(np.inf)), f32(np.inf))]
    return np.array(vals, np.float32)


@pytest.mark.parametrize("cfg", [FBOCC, (2.0, 42.0, 0.8)])
def test_labels_at_bin_edges_match_eager(cfg):
    """Each candidate depth is the only non-zero value of its 8 x 8 patch:
    t on each integer and a few ulp either side, gt around lo - step, lo,
    hi - step and hi; plus all-zero patches, a patch of -0.0, and NaN in a
    patch that also holds a valid depth."""
    D = len(np.arange(*cfg))
    vals = _edge_values(cfg, D)
    ds, w = 8, 32
    extra = 4
    n = len(vals) + extra
    h = (n + w - 1) // w
    gt = torch.zeros(1, h * ds, w * ds)
    for i, v in enumerate(vals):
        y, x = divmod(i, w)
        gt[0, y * ds + (i % ds), x * ds + (i * 3) % ds] = float(v)
    i = len(vals)                                   # all-zero patch: i
    y, x = divmod(i + 1, w)                         # -0.0 next to a depth
    gt[0, y * ds, x * ds] = -0.0
    gt[0, y * ds + 1, x * ds + 2] = 7.3
    y, x = divmod(i + 2, w)                         # NaN next to a depth
    gt[0, y * ds + 3, x * ds + 3] = float("nan")
    gt[0, y * ds + 5, x * ds] = 7.3
    gt = gt.to(DEV)
    want = eager_onehot(gt, ds, cfg, D)
    got = _dl().downsampled_gt_depth(gt, ds, cfg, D)
    _assert_bitwise(got, want, "one-hot")
    labels = _dl().depth_labels(gt, ds, cfg, D).view(-1)
    assert labels[i].item() == 0 and labels[i + 2].item() == 0
    assert labels[i + 1].item() > 0
    # the grid does reach exact integers of t and both sides of them
    m = torch.from_numpy(vals).to(DEV)
    t = (m - (cfg[0] - cfg[2])) / cfg[2]
    assert bool((t == t.round()).any()) and bool((t != t.round()).any())
    np.testing.assert_array_equal(labels.cpu().numpy(),
                                  labels_ref(gt.cpu().numpy(), ds, cfg, D))


# -- loss and gradient ----------------------------------------------------------
def test_probabilities_exactly_zero_and_one():
    """p = 0 and p = 1 on hot and cold bins of foreground pixels: the -100
    clamp of the logs and the 1e-12 floor of the gradient's denominator."""
    D, ds = 80, 16
    gt = lidar_gt(2, 64, 176, *FBOCC[:2], seed=5, density=0.05, spill=False)
    preds = softmax_preds(2, D, 4, 11, seed=6)
    labels = _dl().depth_labels(gt, ds, FBOCC, D).view(2, 4, 11)
    fg = (labels > 0).nonzero().tolist()
    assert len(fg) >= 8
    for j, (n, y, x) in enumerate(fg[:8]):
        hot = labels[n, y, x].item() - 1
        cold = (hot + 7) % D
        preds[n, :, y, x] = 0.0
        preds[n, hot, y, x] = (0.0, 1.0)[j % 2]
        preds[n, cold, y, x] = (1.0, 0.0)[(j // 2) % 2]
    loss, grad = ours(gt, preds, ds, FBOCC, 3.0)
    want_loss, want_grad = eager_grad(gt, preds, ds, FBOCC, 3.0)
    assert torch.isfinite(loss) and _rel(loss, want_loss) <= 1e-5
    _assert_bitwise(grad, want_grad, "d preds")


def test_no_foreground():
    """Nothing in range: loss 0, all-zero gradient, no host sync."""
    gt = torch.zeros(6, 64, 176, device=DEV)
    gt[:, ::3, ::5] = 99.0                         # beyond hi
    preds = softmax_preds(6, 80, 4, 11, seed=1).requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = _dl().depth_loss(gt, preds, 16, FBOCC, 3.0)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert loss.item() == 0.0
    assert not preds.grad.any()


@pytest.mark.parametrize("D", [59, 80, 118])
@pytest.mark.parametrize("ds", [8, 16])
@pytest.mark.parametrize("BN", [1, 6, 24])
def test_shapes_match_eager(D, ds, BN):
    cfg = (2.0, 2.0 + 0.5 * D, 0.5)
    H, W = ds * 8, ds * 22
    gt = lidar_gt(BN, H, W, cfg[0], cfg[1], seed=D + ds + BN)
    preds = softmax_preds(BN, D, 8, 22, seed=BN)
    loss, grad = ours(gt, preds, ds, cfg, 3.0)
    want_loss, want_grad = eager_grad(gt, preds, ds, cfg, 3.0)
    assert _rel(loss, want_loss) <= 1e-5, (loss.item(), want_loss.item())
    _assert_bitwise(grad, want_grad, "d preds")
    _assert_bitwise(_dl().downsampled_gt_depth(gt, ds, cfg, D),
                    eager_onehot(gt, ds, cfg, D), "one-hot")


def test_fbocc_training_size():
    """B = 4, N = 6, 256 x 704, D = 80, ds 16, CM's (B, N, D, h, w) layout."""
    B, N, D = 4, 6, 80
    gt = lidar_gt(B * N, 256, 704, *FBOCC[:2], seed=9, density=0.03)
    gt = gt.view(B, N, 256, 704)
    preds = softmax_preds(B * N, D, 16, 44, seed=10).view(B, N, D, 16, 44)
    loss, grad = ours(gt, preds, 16, FBOCC, 3.0)
    want_loss, want_grad = eager_grad(gt, preds, 16, FBOCC, 3.0)
    assert grad.shape == preds.shape
    assert _rel(loss, want_loss) <= 1e-5
    _assert_bitwise(grad, want_grad, "d preds")


# -- determinism, no sync, CUDA graphs ------------------------------------------
def test_deterministic_and_independent_of_the_batch():
    D, ds = 80, 16
    gt = lidar_gt(6, 128, 352, *FBOCC[:2], seed=3)
    preds = softmax_preds(6, D, 8, 22, seed=4)
    a = ours(gt, preds, ds, FBOCC, 3.0)
    b = ours(gt, preds, ds, FBOCC, 3.0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # sample 0 alone == sample 0 in a batch whose other images have no
    # foreground (same n_fg); its gradient at any batch position
    alone = ours(gt[:1], preds[:1], ds, FBOCC, 3.0)
    for pos in (0, 3):
        gb = torch.zeros_like(gt)
        gb[pos] = gt[0]
        pb = preds.clone()
        pb[pos] = preds[0]
        loss, grad = ours(gb, pb, ds, FBOCC, 3.0)
        if pos == 0:
            assert torch.equal(loss, alone[0])
        assert torch.equal(grad[pos], alone[1][0])
        assert not grad[torch.arange(6, device=DEV) != pos].any()


def test_no_sync_and_cuda_graph_replay():
    D, ds = 80, 16
    static_gt = lidar_gt(6, 128, 352, *FBOCC[:2], seed=11)
    static_p = softmax_preds(6, D, 8, 22, seed=12).requires_grad_()
    p0 = static_p.detach().clone().requires_grad_()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _dl().depth_loss(static_gt, p0, ds, FBOCC, 3.0).backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert p0.grad.any()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            static_p.grad = None
            _dl().depth_loss(static_gt, static_p, ds, FBOCC, 3.0).backward()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    static_p.grad = None
    with torch.cuda.graph(graph):
        static_loss = _dl().depth_loss(static_gt, static_p, ds, FBOCC, 3.0)
        static_loss.backward()
    new_gt = lidar_gt(6, 128, 352, *FBOCC[:2], seed=13)
    new_p = softmax_preds(6, D, 8, 22, seed=14)
    with torch.no_grad():
        static_gt.copy_(new_gt)
        static_p.copy_(new_p)
    graph.replay()
    torch.cuda.synchronize()
    want_loss, want_grad = ours(new_gt, new_p, ds, FBOCC, 3.0)
    assert torch.equal(static_loss, want_loss)
    assert torch.equal(static_p.grad, want_grad)


# -- module surface -------------------------------------------------------------
def _cm_tail(D=80, grid=None):
    from fbbev_b200.view_transformation.depth_net_tail import CM_DepthNetTail
    return CM_DepthNetTail(16, 8, downsample=16,
                           grid_config=grid or dict(depth=list(FBOCC)),
                           depth_channels=D, loss_depth_weight=3.0).to(DEV)


def test_cm_tail_methods():
    z = load_golden("d_depth_loss")
    gt = torch.from_numpy(z["fbocc/gt"]).to(DEV)
    preds = torch.from_numpy(z["fbocc/preds"]).to(DEV)
    tail = _cm_tail()
    out = tail.get_depth_loss(gt, preds)
    assert list(out) == ["loss_depth"]
    loss = out["loss_depth"]
    assert loss.is_cuda and loss.dim() == 0
    assert _rel(loss, z["fbocc/loss"]) <= 1e-5
    onehot = tail.get_downsampled_gt_depth(gt)
    np.testing.assert_array_equal(onehot.cpu().numpy(),
                                  z["fbocc/onehot"].astype(np.float32))
    # depth_channels=None: D of the logits / of grid_config['depth']
    auto = _cm_tail(D=None)
    assert torch.equal(auto.get_depth_loss(gt, preds)["loss_depth"], loss)
    assert torch.equal(auto.get_downsampled_gt_depth(gt), onehot)
    from fbbev_b200._lib import FbbevError
    with pytest.raises(FbbevError):
        tail.get_depth_loss(gt.cpu(), preds.cpu())


def test_bevdepth_methods():
    import torch.nn as nn
    from fbbev_b200.view_transformation.bevdet_lineage import \
        LSSViewTransformerBEVDepth
    z = load_golden("d_depth_loss")
    cfg = [float(v) for v in z["lineage/depth_cfg"]]
    grid = dict(x=[-40, 40, 4.0], y=[-40, 40, 4.0], z=[-1, 5.4, 3.2],
                depth=cfg)
    H, W = z["lineage/gt"].shape[-2:]
    vt = LSSViewTransformerBEVDepth(
        grid_config=grid, input_size=(H, W), downsample=16, in_channels=16,
        out_channels=8, depthnet_cfg=dict(module=nn.Identity()))
    assert vt.D == int(z["lineage/D"])
    gt = torch.from_numpy(z["lineage/gt"]).to(DEV)
    preds = torch.from_numpy(z["lineage/preds"]).to(DEV).requires_grad_()
    loss = vt.get_depth_loss(gt, preds)
    assert torch.is_tensor(loss) and loss.is_cuda and loss.dim() == 0
    assert _rel(loss.detach(), z["lineage/loss"]) <= 1e-5
    loss.backward()
    _assert_bitwise(preds.grad.cpu(), torch.from_numpy(z["lineage/grad"]),
                    "d preds")
    np.testing.assert_array_equal(
        vt.get_downsampled_gt_depth(gt).cpu().numpy(),
        z["lineage/onehot"].astype(np.float32))


# -- end to end ---------------------------------------------------------------
def test_end_to_end_gradient_of_both_consumers():
    """CM_DepthNetTail -> LSSViewTransformerFunction3D(context_layout='nhwc')
    -> weighted sum of the volume, plus get_depth_loss: autograd adds the
    loss's d depth to the pooling backward's.  Against the same graph with the
    eager loss."""
    from fbbev_b200 import _lib, synthetic
    from fbbev_b200.view_transformation.forward_projection import \
        LSSViewTransformerFunction3D
    B, N, mid, C = 2, 6, 16, 8
    grid = dict(x=[-40, 40, 1.6], y=[-40, 40, 1.6], z=[-1, 5.4, 1.6],
                depth=list(FBOCC))
    vt = LSSViewTransformerFunction3D(grid, (128, 352), 16)
    D = vt.D
    tail = _cm_tail(D, grid)
    cam = synthetic.make_cam_params(B, N, (128, 352), device=DEV, jitter=1.0)
    g = torch.Generator().manual_seed(21)
    ctx_in = torch.randn(B * N, mid, 8, 22, generator=g).to(DEV)
    logits0 = (torch.randn(B * N, D, 8, 22, generator=g) * 3.0).to(DEV)
    gt = lidar_gt(B * N, 128, 352, *FBOCC[:2], seed=22).view(B, N, 128, 352)

    def run(loss_fn):
        logits = logits0.clone().requires_grad_()
        feat, depth = tail(ctx_in, logits, B, N)
        bev = vt(cam, feat, depth, context_layout='nhwc')
        wts = torch.rand(bev.shape, generator=torch.Generator().manual_seed(
            23)).to(DEV)
        total = (bev * wts).sum() + loss_fn(depth)
        total.backward()
        return logits.grad

    with _lib.KernelTimer() as kt:
        got = run(lambda d: tail.get_depth_loss(gt, d)["loss_depth"])
    names = {r[0] for r in kt.records}
    assert {"fbbev_depth_loss_fwd", "fbbev_depth_loss_bwd"} <= names, names
    want = run(lambda d: eager_loss(gt, d, 16, FBOCC, 3.0))
    bar = 1e-5 * max(1.0, want.abs().max().item())
    err = (got - want).abs().max().item()
    assert err <= bar, (err, bar)
