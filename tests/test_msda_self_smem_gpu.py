"""The shared-memory footprint-tile route of the BEV self-attention sampler
(``msda_self_smem_kernel``, csrc/msda_self_smem.cu) against the flat
global-memory kernel (``fbbev_msda_fused_fwd`` with ``patch_w = 0``), bit for
bit, and against the float64 reference.

The route serves 8 heads x 10 channels, one level, 4 points, one query per
value pixel on a map of at least one staged window (18 x 18 pixels); one query
sits on every pixel, so every case has queries on the four borders and
corners, where the window is shifted inwards and corners off the map read as
zeros."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HEADS, CH, POINTS = 8, 10, 4
KERNEL = "msda_self_smem_kernel"
WINDOW = 18


def _inputs(H, W, bs=1, scale=1.0, sigma=0.3, seed=0, ch=CH):
    """Self-attention call on an H x W map: offsets = (the module's initial
    ring bias, radius p + 1 pixels for point p, + N(0, sigma)) * scale."""
    g = torch.Generator().manual_seed(seed)
    nq = H * W
    value = torch.randn(bs, nq, HEADS, ch, generator=g)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    ref = torch.stack([(xs + 0.5) / W, (ys + 0.5) / H], -1).float().view(
        1, nq, 1, 2).repeat(bs, 1, 1, 1)
    th = torch.arange(HEADS, dtype=torch.float32) * (2.0 * math.pi / HEADS)
    ring = torch.stack([th.cos(), th.sin()], -1)
    ring = ring / ring.abs().max(-1, keepdim=True)[0]
    ring = ring.view(HEADS, 1, 1, 2) * torch.arange(
        1, POINTS + 1, dtype=torch.float32).view(1, 1, POINTS, 1)
    off = (ring + sigma * torch.randn(bs, nq, HEADS, 1, POINTS, 2,
                                      generator=g)) * scale
    lg = torch.randn(bs, nq, HEADS, 1, POINTS, generator=g)
    ss = torch.tensor([[H, W]], dtype=torch.int64)
    ls = torch.zeros(1, dtype=torch.int64)
    return [t.to(DEV) for t in (value, ss, ls, ref, off, lg)]


def _leaving(off, H, W, tile=8, halo=5):
    """Fraction of the in-image samples with a corner outside the staged
    window of their query's tile (the kernel's own test, on the host)."""
    nq = H * W
    q = torch.arange(nq, device=off.device)
    qx, qy = (q % W).view(1, nq, 1, 1, 1), (q // W).view(1, nq, 1, 1, 1)
    px = ((qx + 0.5) / W + off[..., 0] / W) * W - 0.5
    py = ((qy + 0.5) / H + off[..., 1] / H) * H - 0.5
    inimg = (px > -1) & (py > -1) & (px < W) & (py < H)
    xl, yl = px.floor().long(), py.floor().long()
    win = tile + 2 * halo
    x0 = (qx // tile * tile - halo).clamp(0, W - win)
    y0 = (qy // tile * tile - halo).clamp(0, H - win)
    inside = (xl >= x0) & (xl + 1 < x0 + win) & (yl >= y0) & (yl + 1 < y0 + win)
    return float((inimg & ~inside).sum()) / max(1, int(inimg.sum()))


def _kernels(fn):
    """Names of the CUDA kernels ``fn`` launched (the profiler drops a record
    now and then: up to three runs, merged)."""
    from torch.profiler import ProfilerActivity, profile
    seen = set()
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        seen |= {e.name for e in prof.events()}
        if any("fbbev::" in n for n in seen):
            break
    return seen


def _both(args, W):
    from fbbev_b200.ops.ms_deform_attn import ms_deform_attn_fused
    tiled = ms_deform_attn_fused(*args, W)
    flat = ms_deform_attn_fused(*args, 0)
    assert torch.isfinite(flat).all()
    assert torch.equal(tiled, flat), float((tiled - flat).abs().max())
    return tiled


_DISPATCH_NAMES = r"""
import json, sys
sys.path[:0] = sys.argv[1:3]
from fbbev_b200.ops.ms_deform_attn import ms_deform_attn_fused
from test_msda_self_smem_gpu import _inputs, _kernels
print(json.dumps([sorted(_kernels(
    lambda: ms_deform_attn_fused(*_inputs(H, W, ch=ch), pw)))
    for H, W, ch, pw in json.loads(sys.argv[3])]))
"""


def test_dispatch_reaches_the_tile_kernel():
    """8 x 10 self-attention on a map of one window or more runs the tile
    kernel; a smaller map, another head width or patch_w = 0 do not.  The
    profiler names the kernels in a process of its own: in a process that has
    run many other tests, it can stop reporting kernel records at all."""
    import json
    import subprocess
    import sys

    from conftest import ROOT
    cases = [(WINDOW, 40, CH, 40), (200, 200, CH, 200),
             (WINDOW - 1, 40, CH, 40), (40, WINDOW - 1, CH, WINDOW - 1),
             (40, 40, CH, 0), (40, 40, 32, 40)]
    flags = ["-I"] if sys.flags.isolated else \
        ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run(
        [sys.executable, *flags, "-c", _DISPATCH_NAMES, ROOT,
         os.path.dirname(os.path.abspath(__file__)), json.dumps(cases)],
        stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    names = json.loads(res.stdout.splitlines()[-1])
    if not all(any("fbbev::" in n for n in case) for case in names):
        pytest.skip("the profiler reported no library kernel")
    ran = [any(KERNEL in n for n in case) for case in names]
    assert ran == [True, True, False, False, False, False], ran


def test_bench_workload_tensors():
    """The self-attention call of bench.py's fbocc200 step (seeded weights
    and inputs), captured from the module's forward."""
    import bench
    import fbbev_b200.view_transformation.backward_projection as bp_mod
    w = bench.Workload("fbocc200", DEV, seed=0, frames=1)
    calls, orig = [], bp_mod.ms_deform_attn_fused

    def grab(*a, **kw):
        calls.append((a, kw))
        return orig(*a, **kw)
    bp_mod.ms_deform_attn_fused = grab
    try:
        w.step()
    finally:
        bp_mod.ms_deform_attn_fused = orig
    assert len(calls) == 1
    (a, kw), = calls
    assert kw["map_width"] == 200 and a[0].shape == (1, 40000, HEADS, CH)
    _both(a, 200)


@pytest.mark.parametrize("scale,shift,lo,hi", [
    (0.5, 0, 0.0, 0.05), (3.5, 0, 0.4, 0.6), (1.0, 30, 1.0, 1.0)])
def test_samples_leaving_the_window(scale, shift, lo, hi):
    """No sample (but the border ones with a corner off the map), about half
    of them, and every sample (each pushed ``shift`` pixels towards the map's
    middle column) outside the staged window: the result is the flat
    kernel's whichever side served a sample."""
    H = W = 96
    args = _inputs(H, W, scale=scale, seed=3)
    off = args[4]
    qx = (torch.arange(H * W, device=DEV) % W).view(1, H * W, 1, 1, 1)
    off[..., 0] += shift * torch.where(qx < W // 2, 1.0, -1.0)
    frac = _leaving(off, H, W)
    print(f"[self-smem] scale {scale} shift {shift}: {100 * frac:.1f} % of the "
          "in-image samples leave the window")
    assert lo <= frac <= hi, frac
    _both(args, W)


@pytest.mark.parametrize("H,W,bs", [(200, 200, 1), (37, 45, 2), (18, 18, 2),
                                    (19, 131, 1), (5, 40, 2), (64, 64, 3)])
def test_map_sizes(H, W, bs):
    """Maps that are not a multiple of the 8 x 8 tile in either direction,
    exactly one window, fewer rows than a tile (the global patch kernel
    serves it), bs > 1; offsets reach over every border."""
    _both(_inputs(H, W, bs=bs, scale=1.3, seed=H + W), W)


def test_non_finite_offsets():
    """NaN and +-inf offsets in a few rows fail the in-image test as in the
    flat kernel (the sample is skipped) before any window address exists."""
    H, W = 40, 48
    args = _inputs(H, W, bs=2, seed=5)
    off = args[4]
    g = torch.Generator().manual_seed(6)
    rows = torch.randperm(H * W, generator=g)[:64].to(DEV)
    bad = torch.tensor([float("nan"), float("inf"), -float("inf"), 3e38],
                       device=DEV)
    pick = torch.randint(0, 4, off[:, rows].shape, generator=g).to(DEV)
    keep = (torch.rand(off[:, rows].shape, generator=g) < 0.5).to(DEV)
    off[:, rows] = torch.where(keep, off[:, rows], bad[pick])
    assert not torch.isfinite(off).all()
    _both(args, W)


def test_shapes_disagreeing_with_patch_w():
    """patch_w is a scheduling hint: with spatial_shapes of another aspect
    (same pixel count) the samples are still those of spatial_shapes."""
    args = _inputs(40, 60, seed=8)
    _both(args, 60)
    _both(args, 40)       # 60 x 40 tiles over a 40 x 60 map
    _both(args, 100)


def test_against_float64_reference():
    """The attention matrix's own inputs (edge-pinned queries, lattice
    offsets, logits up to +-60) on a 21 x 27 map, forward through the tile
    kernel, against the float64 reference at the matrix's bar."""
    import test_attention_matrix_gpu as M
    from oracle import msda_ref64 as R
    c = M.msda_inputs(977, HEADS, CH, [(21, 27)], self_map=True)
    want = R.msda_fused(*M.msda_ref_args(c, True))
    args = M._gpu(c, ("value", "ss", "ls", "ref", "off", "lg"), ())
    got = _both(args, 27)
    scale = max(1.0, float(want.abs().max()))
    err = float((got.double().cpu() - want).abs().max()) / scale
    print(f"[self-smem] out vs float64: {err:.2e} (bar {M.OUT_BAR:.0e})")
    assert err <= M.OUT_BAR, err
