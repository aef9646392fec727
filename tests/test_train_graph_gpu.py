"""A view-transformation training step captured in a CUDA graph.

The step: CM_DepthNetTail (LiftTail) -> LSSViewTransformerFunction3D forward
(``context_layout`` 'nhwc' and 'nchw') and forward_backward_readd (Z-mean, the
BackwardProjection encoder under grad, re-add; DeferredVolumeTrain) ->
get_depth_loss plus a seeded weighted sum of the outputs -> backward() ->
optimizer.step().  The voxel index is rebuilt inside the step from the camera
parameters, which change per replay (a bda flip and new jitter).

- replay == eager, bit for bit, under torch.use_deterministic_algorithms (run
  in a child process: cuBLAS needs CUBLAS_WORKSPACE_CONFIG before it starts),
  for SGD and AdamW(capturable=True), at configs[1] and at a small shape; in
  the default (atomic) mode within 1e-4 * max(1, max |ref|);
- the eager step is unchanged by a capture;
- the eager step runs without a host synchronisation;
- the encoder's packed weight images: a graph captured with a warm cache
  honours in-place weight updates between replays, and an eager call after
  replays that stepped the weights inside the graph sees the new weights;
  so does a no_grad BackwardProjection forward (the sampling pair's
  concatenated weights, the learned positional encoding); a capture with
  gradients off keeps reading the cached images."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
DEV = "cuda"
K = 3  # replays / eager steps compared
SIZES = ("small", "configs1")


# ------------------------------------------------------------------ the step --
def _shape(size):
    import bench
    c = dict(bench.CONFIGS["fbocc200"])
    if size == "small":
        c.update(bev=(50, 50), input_size=(128, 352))
        grid = dict(x=[-40, 40, 1.6], y=[-40, 40, 1.6], z=[-1, 5.4, 1.6],
                    depth=list(c["dbound"]))
    else:
        from fbbev_b200 import synthetic
        grid = synthetic.GRID_CONFIGS[c["grid"]]
    return c, grid


class Step:
    """Modules, static input buffers and the training step over them."""

    def __init__(self, size, optim, lr, B=1, mid=32, seed=0):
        import bench
        from fbbev_b200.registry import build_head
        from fbbev_b200.view_transformation.depth_net_tail import \
            CM_DepthNetTail
        from fbbev_b200.view_transformation.forward_projection import \
            LSSViewTransformerFunction3D
        c, grid = _shape(size)
        self.c, self.B = c, B
        self.N = c["n_cams"]
        self.vt = LSSViewTransformerFunction3D(grid, c["input_size"],
                                               c["downsample"])
        self.D = self.vt.D
        self.H, self.W = (s // c["downsample"] for s in c["input_size"])
        torch.manual_seed(1234 + seed)
        bp = build_head(bench.bp_config(c))
        bp.init_weights()
        g = torch.Generator().manual_seed(4321 + seed)
        with torch.no_grad():
            for p in bp.parameters():
                p.add_(torch.randn(p.shape, generator=g) * 0.02)
        self.bp = bp.to(DEV).eval()
        self.tail = CM_DepthNetTail(mid, c["C"], downsample=c["downsample"],
                                    grid_config=grid, depth_channels=self.D,
                                    loss_depth_weight=3.0).to(DEV)
        self.params = list(self.tail.parameters()) + list(self.bp.parameters())
        for p in self.params:
            p.requires_grad_(True)
        self.state0 = [p.detach().clone() for p in self.params]
        self.opt = self._optimizer(optim, lr)
        # static inputs: every step reads these buffers
        self.inputs = self.make_inputs(0)
        self.logits = self.inputs["logits"].requires_grad_()
        self.loss_w = None

    def _optimizer(self, optim, lr):
        if optim == "sgd":
            return torch.optim.SGD(self.params, lr=lr)
        return torch.optim.AdamW(self.params, lr=lr, capturable=True)

    def make_inputs(self, i):
        """Seeded inputs of step ``i``: context, depth logits, lidar depth and
        camera parameters (odd steps flip the BEV x axis through bda)."""
        from fbbev_b200 import synthetic
        B, N, D, H, W = self.B, self.N, self.D, self.H, self.W
        g = torch.Generator().manual_seed(100 + i)
        ctx = torch.randn(B * N, self.tail.context_conv.in_channels, H, W,
                          generator=g)
        logits = torch.randn(B * N, D, H, W, generator=g) * 3.0
        Hi, Wi = self.c["input_size"]
        gt = torch.rand(B, N, Hi, Wi, generator=g) * 48.0 + 1.0
        gt = gt * (torch.rand(B, N, Hi, Wi, generator=g) < 0.05)
        cam = list(synthetic.make_cam_params(B, N, self.c["input_size"],
                                             jitter=1.0, seed=7 + i))
        if i % 2:
            cam[5] = cam[5] @ torch.diag(torch.tensor([-1.0, 1.0, 1.0]))
        return dict(ctx=ctx.to(DEV), logits=logits.to(DEV), gt=gt.to(DEV),
                    cam=[t.to(DEV) for t in cam])

    def load_inputs(self, i):
        new = self.make_inputs(i)
        with torch.no_grad():
            for k in ("ctx", "logits", "gt"):
                self.inputs[k].copy_(new[k])
            for d, s in zip(self.inputs["cam"], new["cam"]):
                d.copy_(s)

    def reset(self):
        """Parameters back to their initial values (in place), optimizer state
        to a fresh optimizer's, gradients to None."""
        with torch.no_grad():
            for p, p0 in zip(self.params, self.state0):
                p.copy_(p0)
            for st in self.opt.state.values():
                for t in st.values():
                    if torch.is_tensor(t):
                        t.zero_()
        self.zero_grad()

    def zero_grad(self):
        self.opt.zero_grad(set_to_none=True)
        self.logits.grad = None

    def forward_loss(self):
        from fbbev_b200.view_transformation.forward_projection import \
            forward_backward_readd
        B, N = self.B, self.N
        x = self.inputs
        feat, depth = self.tail(x["ctx"], self.logits, B, N)   # (B,N,H,W,C)
        nchw = feat.permute(0, 1, 4, 2, 3)
        outs = (self.vt(x["cam"], feat, depth, context_layout="nhwc"),
                self.vt(x["cam"], nchw, depth)) + forward_backward_readd(
                    self.vt, self.bp, x["cam"], nchw, depth)
        if self.loss_w is None:
            g = torch.Generator(device=DEV).manual_seed(29)
            self.loss_w = [torch.randn(o.shape, generator=g, device=DEV) * 1e-2
                           for o in outs]
        loss = self.tail.get_depth_loss(x["gt"], depth)["loss_depth"]
        for o, w in zip(outs, self.loss_w):
            loss = loss + (o * w).sum()
        return loss

    def step(self):
        loss = self.forward_loss()
        loss.backward()
        self.opt.step()
        return loss

    def snapshot(self, loss):
        return ([loss.detach().clone(), self.logits.grad.clone()] +
                [p.grad.clone() for p in self.params] +
                [p.detach().clone() for p in self.params])

    def capture(self):
        """Warm up on a side stream, reset, capture one step (gradients and the
        loss allocated in the graph's pool)."""
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(2):
                self.zero_grad()
                self.step()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.reset()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self.static_loss = self.step()
        torch.cuda.synchronize()
        return graph


def _compare(got, want, exact, what):
    assert len(got) == len(want)
    worst = 0.0
    for j, (a, b) in enumerate(zip(got, want)):
        if exact:
            assert torch.equal(a, b), (what, j, (a - b).abs().max().item())
            continue
        err = (a.double() - b.double()).abs().max().item() / \
            max(1.0, b.abs().max().item())
        worst = max(worst, err)
        assert err <= 1e-4, (what, j, err)
    return worst


def check_replay(size, optim, deterministic):
    """K eager steps vs K replays from the same initial state; then the eager
    step after the capture vs the eager step before it."""
    torch.use_deterministic_algorithms(deterministic)
    lr = 1e-3 if deterministic else 1e-7
    st = Step(size, optim, lr)
    eager = []
    for i in range(K):
        st.load_inputs(i)
        st.zero_grad()
        eager.append(st.snapshot(st.step()))
    torch.cuda.synchronize()
    st.load_inputs(0)
    graph = st.capture()
    for i in range(K):
        st.load_inputs(i)
        graph.replay()
        got = st.snapshot(st.static_loss)
        _compare(got, eager[i], deterministic, (size, optim, "replay", i))
    # an eager step after the capture and its replays
    del graph
    st.static_loss = None
    st.reset()
    st.load_inputs(0)
    after = st.snapshot(st.step())
    _compare(after, eager[0], deterministic, (size, optim, "eager after"))
    return True


# ------------------------------------------------------------------- tests ----
def _child(*args):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    res = subprocess.run([sys.executable, os.path.abspath(__file__)] +
                         [str(a) for a in args], cwd=ROOT, env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                         text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-4000:] + res.stderr[-8000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("size", SIZES)
def test_replay_equals_eager_deterministic(size):
    """Bitwise, SGD and AdamW(capturable=True), the index rebuilt per replay
    from new camera parameters, the *_bwd_det attention backwards."""
    out = _child("replay", size, 1)
    assert out == {"sgd": True, "adamw": True}, out


@pytest.mark.parametrize("size", SIZES)
def test_replay_matches_eager_atomic(size):
    for optim in ("sgd", "adamw"):
        check_replay(size, optim, deterministic=False)


def test_eager_step_has_no_host_sync():
    st = Step("configs1", "adamw", 1e-7)
    st.step()  # first call: module constants, optimizer state
    torch.cuda.synchronize()
    st.zero_grad()
    st.load_inputs(1)
    torch.cuda.set_sync_debug_mode("error")
    try:
        st.step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# -- packed weight images under capture (ops.linear) --------------------------
def _encoder_layer(seed):
    from fbbev_b200.view_transformation.backward_projection import FFN
    torch.manual_seed(seed)
    ffn, lin = FFN(80, 320).to(DEV), nn.Linear(80, 80).to(DEV)
    norms = [nn.LayerNorm(80).to(DEV), nn.LayerNorm(80).to(DEV)]
    return [ffn, lin] + norms


def _layer_loss(mods, x, gy):
    from fbbev_b200.view_transformation.backward_projection import _linear
    ffn, lin, n0, n1 = mods
    q = _linear(lin, x, residual=x, norm=n0)
    return (ffn(q, post_norm=n1) * gy).sum()


def _params(mods):
    return [p for m in mods for p in m.parameters()]


def _eager_grads(mods, x, gy):
    """Gradients of a step on a fresh copy of ``mods`` (no cached images)."""
    fresh = _encoder_layer(0)
    with torch.no_grad():
        for p, q in zip(_params(fresh), _params(mods)):
            p.copy_(q)
    xx = x.detach().clone().requires_grad_()
    _layer_loss(fresh, xx, gy).backward()
    return [xx.grad] + [p.grad for p in _params(fresh)]


def test_stale_weight_images():
    """A graph captured after eager steps filled the packed-image caches
    re-forms the images on every replay: weights changed in place between
    replays (param.add_, an eager optimizer step) are the weights the replay
    computes with; an eager call after replays that stepped the weights inside
    the graph computes with the stepped weights."""
    mods = _encoder_layer(0)
    params = _params(mods)
    x = torch.randn(2, 700, 80, device=DEV, requires_grad=True)
    gy = torch.randn(2, 700, 80, device=DEV)

    def zero():
        for p in params:
            p.grad = None
        x.grad = None

    def grads():
        return [x.grad.clone()] + [p.grad.clone() for p in params]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):      # warm: every image cached on the weights
            zero()
            _layer_loss(mods, x, gy).backward()
    torch.cuda.current_stream().wait_stream(s)
    zero()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _layer_loss(mods, x, gy).backward()
    graph.replay()
    torch.cuda.synchronize()
    _compare(grads(), _eager_grads(mods, x, gy), True, "replay")
    # in-place change between replays
    g = torch.Generator(device=DEV).manual_seed(5)
    with torch.no_grad():
        for p in params:
            p.add_(torch.randn(p.shape, generator=g, device=DEV) * 0.05)
    graph.replay()
    torch.cuda.synchronize()
    _compare(grads(), _eager_grads(mods, x, gy), True, "after add_")
    # an eager optimizer step between replays (reads the graph's gradients)
    torch.optim.SGD(params, lr=0.5).step()
    graph.replay()
    torch.cuda.synchronize()
    _compare(grads(), _eager_grads(mods, x, gy), True, "after opt.step")
    del graph

    # the optimizer step inside the graph: replays move the weights, not
    # their version counters.  An eager call after replays would cache images
    # at the versions it finds; the next replays leave those versions as they
    # are, so the eager call after them must not read that cache
    opt = torch.optim.SGD(params, lr=0.5)
    zero()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _layer_loss(mods, x, gy).backward()
        opt.step()
    for what in ("eager after replays", "eager after more replays"):
        for _ in range(3):
            graph.replay()
        torch.cuda.synchronize()
        want = _eager_grads(mods, x, gy)
        zero()
        _layer_loss(mods, x, gy).backward()
        _compare(grads(), want, True, what)


def _bp_inputs(st, seed):
    """Seeded BackwardProjection inputs at the shapes of ``st``."""
    c = st.c
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(st.B, st.N, c["C"], st.H, st.W, generator=g)
    depth = torch.rand(st.B, st.N, st.D, st.H, st.W, generator=g)
    depth = depth / depth.sum(2, keepdim=True)
    lss = torch.randn(st.B, c["C"], *c["bev"], generator=g) * 0.1
    return [feat.to(DEV)], lss.to(DEV), depth.to(DEV), st.make_inputs(seed)["cam"]


def test_inference_after_training_replays():
    """Validation under no_grad between replays of a captured training step:
    the sampling_offsets + attention_weights pair (``linear_pair``'s cache)
    and the learned positional encoding (``_pos_cache``) are formed from the
    parameters the replays stepped, as a fresh module with the same state
    forms them."""
    from fbbev_b200.registry import build_head
    import bench
    st = Step("small", "sgd", 1e-2)
    feats, lss, depth, cam = _bp_inputs(st, 41)

    def validate(bp):
        with torch.no_grad():
            return bp(feats, None, lss_bev=lss, cam_params=cam,
                      pred_img_depth=depth)

    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        validate(st.bp)                 # fills the inference caches
        graph = st.capture()
        outs = []
        for i in range(2):
            for j in range(2):
                st.load_inputs(j)
                graph.replay()
            torch.cuda.synchronize()
            outs.append(validate(st.bp).clone())
        fresh = build_head(bench.bp_config(st.c)).to(DEV).eval()
        fresh.load_state_dict(st.bp.state_dict())
        want = validate(fresh)
    finally:
        torch.use_deterministic_algorithms(False)
    for p in st.bp.parameters():
        assert torch.isfinite(p).all()
    assert not torch.equal(outs[0], outs[1])   # the replays moved the weights
    assert torch.equal(outs[1], want), (outs[1] - want).abs().max().item()


def test_inference_capture_keeps_the_cache():
    """With gradients off a capture reads the cached image: the graph treats
    the weights as constants until ``invalidate`` and a new capture."""
    from fbbev_b200.ops import linear as lin
    torch.manual_seed(3)
    w = torch.randn(80, 80, device=DEV) / 80 ** 0.5
    x = torch.randn(1000, 80, device=DEV)
    with torch.no_grad():
        want0 = lin.linear_fused(x, w)          # fills the cache
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = lin.linear_fused(x, w)
        w.mul_(-1.0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, want0)
        assert torch.equal(lin.linear_fused(x, w), -want0)   # eager repacks
        lin.invalidate(w)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            y = lin.linear_fused(x, w)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, -want0)


if __name__ == "__main__":
    # child process of test_replay_equals_eager_deterministic
    assert sys.argv[1] == "replay"
    size, det = sys.argv[2], bool(int(sys.argv[3]))
    print(json.dumps({o: check_replay(size, o, det) for o in ("sgd", "adamw")}))
