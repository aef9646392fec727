"""GPU checks of the restart gradient (``TemporalFusion(restart_grad=True)``):
the adjoint of the history warp (fbbev_history_warp_bwd) against float64
autograd over identity, translated, rotated, flipped, scaled, partly and fully
outside and singular flows; the module on every training route (eager,
two-frame, full) against the reference's golden and the float64 oracle of the
reference's own graph; the default left bitwise unchanged; determinism, no
host sync, the profiler; two ranks under SyncBatchNorm."""
import math
import traceback
from datetime import timedelta

import pytest
import torch
import torch.nn.functional as F

from history_train_full_ref import full_train_ref64
from history_train_ref import module_params64
from test_history_fuse_gpu import (kernel_names, launches, make_fusion,
                                   record_state, step_inputs)
from test_history_restart_grad_cpu import warp_adjoint64
from test_history_train_gpu import (ATOL, GRAD_RTOL, MARGIN, OUT_ATOL,
                                    SUM_RTOL, loss_weight, module_grads)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ADJ = "warp_adjoint_gather_kernel"
ROUTES = ("eager", "two", "full")


# -- the adjoint on its own ---------------------------------------------------
def _fma(a, b, c):
    # fp32 fma: the product is exact in float64, one rounding to fp32 after
    return (a.double() * b.double() + c.double()).float()


def kernel_coords(flow, Z, H, W):
    """The fp32 source coordinates (ix, iy, iz) history_corners computes, op
    for op: the grid the forward samples."""
    n = flow.shape[0]
    z, y, x = torch.meshgrid(*(torch.arange(s, dtype=torch.float32, device=DEV)
                               for s in (Z, H, W)), indexing="ij")
    f = flow.float().reshape(n, 1, 1, 1, 16)
    out = []
    for row, size in ((0, W), (1, H), (2, Z)):
        r = [f[..., 4 * row + k] for k in range(4)]
        p = _fma(r[2], z, _fma(r[1], y, r[0] * x)) + r[3]
        s = torch.tensor(float(size - 1), device=DEV)
        g = p / s * 2.0 - 1.0
        out.append((g + 1.0) / 2.0 * s)
    return out


def adjoint_exact64(G, flow):
    """warp^T G in float64 at the forward's own fp32 coordinates: the exact
    transpose of what the kernel samples."""
    n, C, Z, H, W = G.shape
    ix, iy, iz = kernel_coords(flow, Z, H, W)
    grid = torch.stack([ix.double() / (W - 1) * 2 - 1,
                        iy.double() / (H - 1) * 2 - 1,
                        iz.double() / (Z - 1) * 2 - 1], -1)
    x = torch.zeros(G.shape, dtype=torch.float64, device=DEV,
                    requires_grad=True)
    y = F.grid_sample(x, grid, align_corners=True, mode="bilinear")
    return torch.autograd.grad(y, x, G)[0]


def flows(n, Z, H, W, kind, seed):
    """(n, 4, 4) voxel-index flows of one kind (fp32)."""
    g = torch.Generator().manual_seed(seed)
    out = torch.eye(4, dtype=torch.float64).repeat(n, 1, 1)
    ctr = torch.tensor([(W - 1) / 2, (H - 1) / 2, (Z - 1) / 2],
                       dtype=torch.float64)
    for b in range(n):
        m = torch.eye(3, dtype=torch.float64)
        t = torch.zeros(3, dtype=torch.float64)
        if kind == "integer":
            t = torch.tensor([2.0, -3.0, 1.0]) * (1 if b % 2 else -1)
        elif kind == "fractional":
            t = (torch.rand(3, generator=g, dtype=torch.float64) - 0.5) * 4
        elif kind in ("rotation", "bda"):
            a = float(torch.rand(1, generator=g)) * 2 * math.pi
            m[:2, :2] = torch.tensor([[math.cos(a), -math.sin(a)],
                                      [math.sin(a), math.cos(a)]])
            if kind == "bda":
                flip = torch.diag(torch.tensor([-1.0 if b % 2 else 1.0,
                                                1.0 if b % 2 else -1.0, 1.0],
                                               dtype=torch.float64))
                m = m @ flip * (0.95 + 0.1 * b)
            t = (torch.rand(3, generator=g, dtype=torch.float64) - 0.5) * 2
            t[2] *= 0.2
        elif kind == "partly_outside":
            t = torch.tensor([W / 2 + 0.3, -H / 3 - 0.7, 0.4])
        elif kind == "fully_outside":
            t = torch.tensor([3.0 * W, 0.5, 0.0])
        elif kind == "singular":
            if b % 2:   # rank 1: every voxel onto one line
                m = torch.tensor([[0.7, 0.3, 0.0], [0.35, 0.15, 0.0],
                                  [0.0, 0.0, 0.0]], dtype=torch.float64)
            else:       # rank 0: every voxel onto one point
                m = torch.zeros(3, 3, dtype=torch.float64)
            t = ctr + 0.25
        if kind not in ("identity", "integer", "fractional", "partly_outside",
                        "fully_outside", "singular"):
            t = t + ctr - m @ ctr       # about the volume's centre
        out[b, :3, :3] = m
        out[b, :3, 3] = t
    return out.float().to(DEV)


def run_adjoint(g, flow, mask, C, accumulate=False, base=None):
    from fbbev_b200.view_transformation.temporal_fusion import \
        history_warp_bwd
    n, _, Z, H, W = g.shape
    dst = (torch.randn(n, C, Z, H, W, device=DEV) if base is None
           else base.clone())
    before = dst.clone()
    history_warp_bwd(g, flow, mask, dst, accumulate=accumulate)
    return dst, before


def check_adjoint(n, C, T, zyx, kind, mask, seed, accumulate=False):
    Z, H, W = zyx
    gen = torch.Generator(device=DEV).manual_seed(seed)
    g = torch.randn(n, T * C, Z, H, W, device=DEV, generator=gen)
    flow = flows(n, Z, H, W, kind, seed)
    got, before = run_adjoint(g, flow, mask, C, accumulate)
    G = g.double().view(n, T, C, Z, H, W).sum(1)
    exact = adjoint_exact64(G, flow)
    plain = warp_adjoint64(G, flow.double())
    for b in range(n):
        if not mask[b]:
            assert torch.equal(got[b].view(torch.int32),
                               before[b].view(torch.int32)), (kind, b)
            continue
        want = exact[b] + (before[b].double() if accumulate else 0)
        err = float((got[b].double() - want).abs().max())
        bar = 1e-5 * max(1.0, float(want.abs().max()))
        assert err <= bar, (kind, b, err, bar)
        # against history_warp_cpu's float64 coordinates: the forward's own
        # fp32 coordinate rounding (up to ~1e-5 voxel) comes on top
        want = plain[b] + (before[b].double() if accumulate else 0)
        err = float((got[b].double() - want).abs().max())
        assert err <= 1e-4 * max(1.0, float(want.abs().max())), (kind, b, err)


KINDS = ("identity", "integer", "fractional", "rotation", "bda",
         "partly_outside", "fully_outside", "singular")


@pytest.mark.parametrize("kind", KINDS)
def test_adjoint_small_ragged(kind):
    for n, mask, zyx in ((1, [True], (3, 7, 9)),
                         (2, [True, True], (5, 6, 11)),
                         (3, [False, True, True], (3, 9, 5))):
        check_adjoint(n, 4, 3, zyx, kind, mask, seed=n)
        check_adjoint(n, 4, 1, zyx, kind, mask[::-1], seed=n + 7,
                      accumulate=True)


@pytest.mark.parametrize("kind", ("identity", "fractional", "rotation", "bda",
                                  "partly_outside"))
def test_adjoint_full_size(kind):
    check_adjoint(2, 80, 16, (8, 100, 100), kind, [True, False], seed=3)


def test_adjoint_deterministic_and_batch_independent():
    """Two runs bitwise equal; a sample alone gives the bits it gets inside a
    batch of three, for both entry points."""
    from fbbev_b200 import _lib
    from fbbev_b200.view_transformation.temporal_fusion import (_pack,
                                                                _restart_term)
    C, T, zyx = 80, 16, (8, 40, 40)
    Z, H, W = zyx
    gen = torch.Generator(device=DEV).manual_seed(5)
    g = torch.randn(3, T * C, Z, H, W, device=DEV, generator=gen)
    flow = flows(3, Z, H, W, "bda", 5)
    base = torch.randn(3, C, Z, H, W, device=DEV, generator=gen)
    batch = [run_adjoint(g, flow, [True] * 3, C, True, base)[0]
             for _ in range(2)]
    assert torch.equal(batch[0], batch[1])
    for b in range(3):
        alone, _ = run_adjoint(g[b:b + 1], flow[b:b + 1], [True], C, True,
                               base[b:b + 1])
        assert torch.equal(alone[0], batch[0][b])
    wt = torch.randn(C, C, device=DEV, generator=gen) * 0.1
    wtt = _pack(wt.t(), 80, torch.device(DEV))
    e = g[:, :T * C]
    outs = []
    for _ in range(2):
        d = base.clone()
        _restart_term((flow, bytes([1, 0, 1])), e, T, wtt, d)
        outs.append(d)
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0][1], base[1])
    for b in (0, 2):
        d = base[b:b + 1].clone()
        _restart_term((flow[b:b + 1], bytes([1])), e[b:b + 1], T, wtt, d)
        assert torch.equal(d[0], outs[0][b])
    # against float64: Wt^T warp^T (sum_f e_f)
    r = adjoint_exact64(e.double().view(3, T, C, Z, H, W).sum(1), flow)
    want = base.double() + torch.einsum("kj,nkzyx->njzyx", wt.double(), r)
    for b in (0, 2):
        err = float((outs[0][b].double() - want[b]).abs().max())
        assert err <= 1e-5 * max(1.0, float(want[b].abs().max())), err
    assert _lib.lib().fbbev_abi_version() == 5


# -- the module -----------------------------------------------------------------
@pytest.fixture(autouse=True)
def _no_tf32():
    """The eager route's convolutions in full fp32 (cuDNN would use TF32)."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def warp_at_kernel_coords(history, flow, out, ch_offset):
    """``history_warp_cpu`` in float64 at the fp32 source coordinates the
    warp kernel computes (``kernel_coords``).  Every route's forward samples
    there, bitwise as before this option, so the exact gradient of the
    module is the one at those coordinates.  At history_warp_cpu's float64
    coordinates the restart term would also carry the forward's coordinate
    rounding: up to ~2e-5 voxel at 100 voxels, times the up to eight weights
    each source voxel collects, a few 1e-4 of d curr."""
    n, mc, Z, H, W = history.shape
    ix, iy, iz = kernel_coords(flow.float(), Z, H, W)
    grid = torch.stack([ix.double() / (W - 1) * 2 - 1,
                        iy.double() / (H - 1) * 2 - 1,
                        iz.double() / (Z - 1) * 2 - 1], -1).to(history)
    out[:, ch_offset:ch_offset + mc] = F.grid_sample(
        history, grid, align_corners=True, mode="bilinear")
    return out


# The restart term gathers the gradient of voxels v that sample a source voxel
# s, so a ReLU whose fp32 and float64 inputs straddle zero at v moves d curr at
# s, which the margin mask at s (MARGIN) does not see.  d curr of a restarting
# sample is compared where no voxel that samples s with a non-zero weight has
# a ReLU input within the forward's fp32 error of zero (up to 5e-5, see
# test_history_train_gpu.MARGIN).
REACH_MARGIN = 5e-5


def restart_keep(near, flow, starts):
    """(n, 1, H, W, Z) bool: False at the source voxels of restarting samples
    that a voxel with a ReLU input within REACH_MARGIN of zero samples."""
    bad = (near < REACH_MARGIN).double()[:, None]
    reach = adjoint_exact64(bad, flow)[:, 0] > 0
    ok = ~reach | ~starts.to(reach.device)[:, None, None, None]
    return ok.permute(0, 2, 3, 1)[:, None]


def _oracle_at_kernel_coords():
    import history_train_full_ref
    history_train_full_ref.history_warp_cpu = warp_at_kernel_coords


def fusion(C, T, c_out, zyx, seed, route, do_history=True, restart=True):
    tf = make_fusion(C, T, c_out, zyx, seed, do_history).train()
    if restart is not None:
        tf.restart_grad = restart
    tf.full_frame_kernels = route == "full"
    if route == "eager":
        tf._train_route = lambda *a: False
    return tf


def count_routes(tf):
    calls = {"two": 0, "full": 0}
    for name, key in (("_fuse_train", "two"), ("_fuse_train_full", "full")):
        orig = getattr(tf, name)

        def spy(*a, _o=orig, _k=key):
            calls[_k] += 1
            return _o(*a)
        setattr(tf, name, spy)
    return calls


def run_oracle(C, T, c_out, zyx, n, starts_seq, seed, route, do_history=True):
    """Calls of a restart_grad module on one route against the float64 oracle
    of the reference's own graph (full_train_ref64(restart_grad=True)),
    sampled at the warp kernel's coordinates."""
    tf = fusion(C, T, c_out, zyx, seed, route, do_history)
    rec = record_state(tf)
    calls = count_routes(tf)
    for step, starts in enumerate(starts_seq):
        fresh = step == 0 or all(starts) or not do_history
        curr, metas, bda = step_inputs(n, C, zyx, step, starts, list(range(n)),
                                       seed, shift=6.0)
        curr.requires_grad_()
        p64, stats = module_params64(tf, DEV)
        hist = None if tf.history_bev is None else tf.history_bev.clone()
        tf.zero_grad()
        before = dict(calls)
        out = tf.fuse_history(curr, metas, bda)
        took = {k: calls[k] - before[k] for k in calls}
        want_route = {"eager": {"two": 0, "full": 0},
                      "two": {"two": 1, "full": 0},
                      "full": {"two": int(fresh), "full": int(not fresh)}}
        assert took == want_route[route], (step, took)
        flow, sweep, _, _ = rec[-1]
        c64 = curr.detach().permute(0, 1, 4, 2, 3).double().requires_grad_()
        start = torch.tensor(starts, device=DEV)
        o64, _, _, _, near, _ = full_train_ref64(
            c64, hist, start, flow, sweep, p64, stats, T, True, True,
            restart_grad=True)
        keep = (near >= MARGIN).permute(0, 2, 3, 1)[:, None]
        wgt = loss_weight(out, seed + step) * keep
        (out * wgt).sum().backward()
        (o64 * wgt.permute(0, 1, 4, 2, 3).double()).sum().backward()
        err = float((out.detach().permute(0, 1, 4, 2, 3).double() -
                     o64.detach()).abs().max())
        assert err <= OUT_ATOL, f"step {step}: output {err:.3e}"
        got = module_grads(tf, curr.grad)
        last = full_train_ref64.last
        l1 = {"bt": last["y"].grad.abs().sum((0, 2)),
              "bc": last["y2"].grad.abs().sum((0, 2))}
        want = {k: p64[k].grad for k in ("wt", "bt", "gamma", "beta", "wc",
                                          "bc")}
        want["curr"] = c64.grad.permute(0, 1, 3, 4, 2)
        kc = keep & restart_keep(near, flow, start)
        got["curr"], want["curr"] = got["curr"] * kc, want["curr"] * kc
        errs, bad = {}, {}
        for k, w in want.items():
            diff = (got[k].double() - w).abs()
            errs[k] = float(diff.max() / w.abs().max().clamp_min(1.0))
            s = (float((diff / l1[k].clamp_min(1e-30)).max()) if k in l1
                 else 1.0)
            if errs[k] > GRAD_RTOL[k] and not s <= SUM_RTOL:
                bad[k] = errs[k]
        print(f"{route} n={n} step {step} starts={starts}: "
              f"d curr checked at {float(kc.float().mean()):.2f} of voxels, "
              f"out {err:.2e} "
              + " ".join(f"{k}={v:.1e}" for k, v in errs.items()))
        assert not bad, f"{route} step {step}: relative gradient errors {bad}"
        del c64, o64, near, last, full_train_ref64.last


def _seq(route, n, kind):
    """start_of_sequence per call.  The two-frame route runs with
    do_history = False, so that every call is fresh."""
    if kind == "restart_last":     # starts on; mid-sequence; one restarting
        return [[True] * n, [False] * n, [True] + [False] * (n - 1)]
    return [[False] * n, [False, True, False, False], [False] * n,
            [False, False, True, True]]


@pytest.fixture
def kernel_coords_oracle(monkeypatch):
    import history_train_full_ref
    monkeypatch.setattr(history_train_full_ref, "history_warp_cpu",
                        warp_at_kernel_coords)


@pytest.mark.usefixtures("kernel_coords_oracle")
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("n", [1, 2])
def test_oracle_full_size(route, n):
    run_oracle(80, 16, 160, (8, 100, 100), n, _seq(route, n, "restart_last"),
               seed=60 + n, route=route, do_history=route != "two")


@pytest.mark.usefixtures("kernel_coords_oracle")
@pytest.mark.parametrize("route", ROUTES)
def test_oracle_n4_reduced(route):
    run_oracle(80, 16, 160, (8, 40, 40), 4, _seq(route, 4, "mixed"),
               seed=64, route=route, do_history=route != "two")


@pytest.mark.usefixtures("kernel_coords_oracle")
@pytest.mark.parametrize("route", ("eager", "full"))
def test_oracle_edge_shape(route):
    run_oracle(4, 3, 8, (3, 7, 9), 3, [[True, False, True],
                                       [False, False, False],
                                       [True, True, False]],
               seed=5, route=route)


@pytest.mark.parametrize("route", ROUTES)
def test_module_vs_reference_golden(route):
    """The reference's own fuse_history in train mode over four calls
    (tests/golden/t_fuse_history_train.npz): d curr of every sample,
    restarting ones included.  The two-frame route takes the all-fresh first
    call (both samples start a sequence) and the eager route the rest."""
    import numpy as np
    from conftest import load_golden
    from test_history_train_full_cpu import golden_metas
    from test_temporal_cpu import build_fusion
    g = load_golden("t_fuse_history_train")
    tf = build_fusion(g, DEV).train()
    tf.restart_grad = True
    tf.full_frame_kernels = route == "full"
    if route == "eager":
        tf._train_route = lambda *a: False
    calls = count_routes(tf)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    for step in range(4):
        tf.zero_grad()
        curr = t(g[f"curr{step}"]).requires_grad_()
        out = tf.fuse_history(curr, golden_metas(g, step, DEV),
                              t(g[f"bda{step}"]))
        (out * t(g[f"wgt{step}"])).sum().backward()
        np.testing.assert_allclose(out.detach().cpu().numpy(), g[f"out{step}"],
                                   rtol=0, atol=OUT_ATOL)
        want = g[f"dcurr{step}"]
        bar = GRAD_RTOL["curr"] * max(1.0, float(np.abs(want).max()))
        np.testing.assert_allclose(curr.grad.cpu().numpy(), want, rtol=0,
                                   atol=bar, err_msg=f"{route} step {step}")
    want_calls = {"eager": {"two": 0, "full": 0}, "two": {"two": 1, "full": 0},
                  "full": {"two": 1, "full": 3}}[route]
    assert calls == want_calls, calls


def _step(tf, curr, metas, bda, seed):
    x = curr.clone().requires_grad_()
    n0 = launches()
    out = tf.fuse_history(x, metas, bda)
    (out * loss_weight(out, seed)).sum().backward()
    torch.cuda.synchronize()
    return (launches() - n0, out.detach(), x.grad,
            [p.grad.clone() for p in tf.parameters()],
            [b.clone() for b in tf.buffers()])


@pytest.mark.parametrize("route", ROUTES)
def test_default_unchanged(route):
    """restart_grad unset or False: bitwise the module without the option,
    same launch count.  True on a call without a restart: the same.  True on a
    restart call: every parameter gradient and the non-restarting samples'
    d curr bitwise as with False."""
    C, T, c_out, zyx, n = 16, 3, 24, (3, 9, 10), 3
    do_history = route != "two"
    mods = {k: fusion(C, T, c_out, zyx, 17, route, do_history, restart=r)
            for k, r in (("none", None), ("off", False), ("on", True))}
    seq = [[True, False, True], [False] * 3, [False, True, False]]
    for step, starts in enumerate(seq):
        curr, metas, bda = step_inputs(n, C, zyx, step, starts, [0, 1, 2], 17)
        res = {k: _step(m, curr, metas, bda, step) for k, m in mods.items()}
        ref = res["none"]
        for key in ("off", "on"):
            got = res[key]
            restart = key == "on" and any(starts)
            if not restart:
                assert got[0] == ref[0], (route, step, key)
            else:
                assert got[0] > ref[0], (route, step)
            assert torch.equal(got[1], ref[1])
            for a, b in zip(got[3] + got[4], ref[3] + ref[4]):
                assert torch.equal(a, b), (route, step, key)
            for b in range(n):
                same = torch.equal(got[2][b], ref[2][b])
                assert same == (not (restart and starts[b])), (route, step,
                                                               key, b)


@pytest.mark.parametrize("route", ROUTES)
def test_deterministic_no_sync_profiler(route, monkeypatch):
    """Two runs bitwise equal; the backward of a restart call runs with no
    host sync; the adjoint's kernels run on restart calls only."""
    C, T, c_out, zyx, n = 32, 4, 48, (3, 12, 11), 2
    do_history = route != "two"
    seq = [[True, True], [False, False], [True, False]]
    res = []
    # the eager route's convolutions: cuDNN's deterministic algorithms
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    for rep in range(2):
        tf = fusion(C, T, c_out, zyx, 23, route, do_history)
        out_rep = []
        for step, starts in enumerate(seq):
            curr, metas, bda = step_inputs(n, C, zyx, step, starts, [0, 1], 23)
            x = curr.clone().requires_grad_()
            if rep == 0:
                box = {}

                def call():
                    out = tf.fuse_history(x, metas, bda)
                    loss = (out * loss_weight(out, step)).sum()
                    torch.cuda.synchronize()
                    torch.cuda.set_sync_debug_mode("error")
                    try:
                        loss.backward()
                    finally:
                        torch.cuda.set_sync_debug_mode(0)
                    box["out"] = out.detach()
                names = kernel_names(call)
                assert any(ADJ in k for k in names) == any(starts), (step,
                                                                    names)
                out = box["out"]
            else:
                out = tf.fuse_history(x, metas, bda)
                (out * loss_weight(out, step)).sum().backward()
                out = out.detach()
            out_rep += [out, x.grad] + [p.grad.clone()
                                        for p in tf.parameters()]
            tf.zero_grad()
        res.append(out_rep)
    for a, b in zip(*res):
        assert torch.equal(a, b), route


# -- two ranks under SyncBatchNorm ----------------------------------------------
def _worker(rank, world, init, q, fn, args):
    try:
        torch.cuda.set_device(DEV)
        import torch.distributed as dist
        dist.init_process_group("gloo", init_method=init, rank=rank,
                                world_size=world,
                                timeout=timedelta(seconds=300))
        try:
            torch.backends.cudnn.allow_tf32 = False
            torch.backends.cuda.matmul.allow_tf32 = False
            res = globals()[fn](rank, world, DEV, *args)
        finally:
            dist.destroy_process_group()
        q.put((rank, ("ok", res)))
    except Exception:
        q.put((rank, ("fail", traceback.format_exc())))


def _union_restart(rank, world, dev, n, seed):
    """Three calls per rank: both ranks fresh with every sample starting
    (two-frame route, restart term on both ranks); both mid-sequence (full
    route); rank 0 with sample 0 restarting, rank 1 mid-sequence.  Each call
    against the float64 oracle of the union batch with restart_grad."""
    from test_history_train_dist_gpu import all_gather, sync_fusion
    _oracle_at_kernel_coords()
    C, T, c_out, zyx = 32, 4, 48, (3, 12, 11)
    tf = sync_fusion(C, T, c_out, zyx, seed, dev, do_history=True)
    tf.full_frame_kernels = True
    tf.restart_grad = True
    rec = record_state(tf)
    plan = [[True] * n, [False] * n,
            [True] + [False] * (n - 1) if rank == 0 else [False] * n]
    sl = slice(rank * n, rank * n + n)
    errs = []
    for step, starts in enumerate(plan):
        p64, stats = module_params64(tf, dev)
        hist = None if tf.history_bev is None else tf.history_bev.clone()
        curr, metas, bda = step_inputs(n, C, zyx, step, starts, list(range(n)),
                                       seed * 7 + rank, shift=6.0)
        curr = curr.requires_grad_()
        out = tf.fuse_history(curr, metas, bda)
        flow, sweep, _, _ = rec[-1]
        parts = all_gather((curr.detach().cpu(), None if hist is None
                            else hist.cpu(), torch.tensor(starts),
                            flow.cpu(), sweep.cpu()))
        tf.zero_grad()
        c64 = torch.cat([p[0] for p in parts]).to(dev).permute(
            0, 1, 4, 2, 3).double().requires_grad_()
        h64 = (None if parts[0][1] is None else
               torch.cat([p[1] for p in parts]).to(dev))
        o64, _, _, _, near, _ = full_train_ref64(
            c64, h64, torch.cat([p[2] for p in parts]),
            torch.cat([p[3] for p in parts]).to(dev),
            torch.cat([p[4] for p in parts]).to(dev), p64, stats, T, True,
            True, restart_grad=True)
        keep = (near >= MARGIN).permute(0, 2, 3, 1)[:, None]
        g = torch.Generator().manual_seed(seed + step)
        wgt = torch.randn(o64.permute(0, 1, 3, 4, 2).shape,
                          generator=g).to(dev) * keep
        (o64 * wgt.permute(0, 1, 4, 2, 3).double()).sum().backward()
        (out * wgt[sl]).sum().backward()
        err = float((out.detach().permute(0, 1, 4, 2, 3).double() -
                     o64.detach()[sl]).abs().max())
        assert err <= OUT_ATOL, (step, err)
        got = module_grads(tf, curr.grad)
        k = (keep & restart_keep(near, torch.cat([p[3] for p in parts]).to(dev),
                                 torch.cat([p[2] for p in parts])))[sl]
        want_curr = c64.grad.permute(0, 1, 3, 4, 2)[sl]
        dcurr = float((got["curr"].double() * k - want_curr * k).abs().max()
                      / want_curr.abs().max().clamp_min(1.0))
        assert dcurr <= GRAD_RTOL["curr"], (step, dcurr)
        local = {key: got[key].double().cpu() for key in ("wt", "gamma",
                                                          "beta", "wc")}
        summed = {}
        for other in all_gather(local):
            for key, v in other.items():
                summed[key] = summed.get(key, 0) + v
        for key, v in summed.items():
            w = p64[key].grad.cpu()
            e = float((v - w).abs().max() / w.abs().max().clamp_min(1.0))
            assert e <= GRAD_RTOL[key], (step, key, e)
        errs.append((err, dcurr))
    return errs


def test_two_ranks_restart_matches_union_batch(tmp_path):
    from test_history_train_dist_cpu import run_workers
    res = run_workers(_worker, 2, tmp_path, "_union_restart", (2, 19),
                      timeout=900)
    assert sorted(res) == [0, 1], res
    for r in (0, 1):
        assert res[r][0] == "ok", res[r][1]
    print(res[0][1], res[1][1])
