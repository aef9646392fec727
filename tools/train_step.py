#!/usr/bin/env python
"""Time one training step of a bench.py workload, with the fused attention
backward kernels and with the dense differentiable attention routes, and the
fused step with its optimizer step eagerly and replayed from a CUDA graph.

    python tools/train_step.py [--config fbocc200|bwd_only|...] [--steps K]
                               [--warmup W] [--deterministic]

A step: F and B forward with the context, depth and image features and every
module parameter requiring grad, a fixed seeded weighted sum of both outputs
as the loss, backward().  Prints one JSON line: per arm the median device time
per step (L2 flushed between steps), peak allocated memory and the per-kernel
table of the library's launches, plus the card's name and power limit read in
the same run.  Writes nothing.

--deterministic adds a third arm, ``fused_deterministic``: the fused arm under
torch.use_deterministic_algorithms(True) (the library's *_bwd_det entry
points), timed in the same run as ``fused``.  cuBLAS needs
CUBLAS_WORKSPACE_CONFIG=:4096:8 for that mode; it is set before torch is
imported, and only with this flag.

``graphed``: the fused step plus an SGD ``optimizer.step()``, captured in one
CUDA graph and replayed with new inputs (features, depth and camera
parameters, alternating between two sets) copied into the static buffers
before each replay.  It is timed in the same loop as ``eager``, the same step
run eagerly on the same inputs, the two alternating step by step;
``launch_and_host_ms`` is the difference of their medians.  Its kernel table
comes from torch.profiler (device kernel names, every kernel of the step),
taken after the timed loop.  With --deterministic the pair is also timed
under deterministic algorithms (``graphed_deterministic``).
"""
import argparse
import contextlib
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
if "--deterministic" in sys.argv[1:]:
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import torch  # noqa: E402

import bench  # noqa: E402


@contextlib.contextmanager
def _dense_attention_grad():
    """Train through the dense differentiable attention routes
    (ms_deform_attn_unfused, da_spatial_cross_attention_core_autograd) instead
    of the fused autograd Functions: the comparison arm."""
    from fbbev_b200.ops import ms_deform_attn as ops
    from fbbev_b200.view_transformation import backward_projection as bp_mod

    class _Dense:
        apply = staticmethod(ops.da_spatial_cross_attention_core_autograd)
    saved = (bp_mod.ms_deform_attn_fused_autograd, bp_mod.DaScaFunction)
    bp_mod.ms_deform_attn_fused_autograd = ops.ms_deform_attn_unfused
    bp_mod.DaScaFunction = _Dense
    try:
        yield
    finally:
        bp_mod.ms_deform_attn_fused_autograd, bp_mod.DaScaFunction = saved


def gpu_identity(index):
    """Card name and power limit, read in the run that measures."""
    ident = {"name": torch.cuda.get_device_name(index), "power_limit": None,
             "clocks_max_sm": None}
    try:
        out = subprocess.run(
            ["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm",
             "--format=csv,noheader", "-i", str(index)],
            stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True,
            timeout=20).stdout.strip().split(",")
        ident["power_limit"], ident["clocks_max_sm"] = (s.strip() for s in out)
    except Exception:
        pass
    return ident


@contextlib.contextmanager
def _deterministic_algorithms():
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def train_block(w, steps, warmup, flush, dev, deterministic=False):
    """One training step of the workload, timed: F and B forward with the
    context, depth and image features and every module parameter requiring
    grad, a fixed seeded weighted sum of both outputs as the loss, backward().
    Reported with the fused attention backward and with the dense
    differentiable routes, each as median device time per step (L2 flushed
    between steps), peak allocated memory and the per-kernel table."""
    from fbbev_b200 import _lib
    leaves = [t.detach().clone().requires_grad_()
              for t in [w.feat, w.depth] + list(w.more)]
    feat, depth, more = leaves[0], leaves[1], leaves[2:]
    mods = [m for m in (w.vt, w.bp) if m is not None]
    for m in mods:
        m.requires_grad_(True)
    loss_w = []

    def step():
        for t in leaves:
            t.grad = None
        for m in mods:
            m.zero_grad(set_to_none=True)
        outs = []
        if w.vt is not None:
            outs.append(w.vt(w.cam, feat, depth))
        outs.append(w.bp([feat] + more, None, lss_bev=w.lss,
                         cam_params=w.cam, pred_img_depth=depth))
        if not loss_w:
            g = torch.Generator(device=dev).manual_seed(29)
            loss_w.extend(torch.randn(o.shape, generator=g, device=dev)
                          for o in outs)
        sum((o * k).sum() for o, k in zip(outs, loss_w)).backward()

    def measure():
        for _ in range(max(warmup, 2)):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        times = []
        for _ in range(steps):
            flush.zero_()
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        peak = torch.cuda.max_memory_allocated(dev)
        ms = statistics.median(times)
        ksteps = max(2, min(steps, 5))
        with _lib.KernelTimer() as kt:
            for _ in range(ksteps):
                flush.zero_()
                torch.cuda._sleep(6_000_000)
                step()
            torch.cuda.synchronize()
        rows = bench.kernel_table(kt.records, ms * 1e3, ksteps, {},
                            {"depth_elems": w.depth.numel()})
        return {"step_ms_median": ms, "step_ms_min": min(times),
                "max_memory_allocated_mb": peak / 2**20,
                "kernels": [{"kernel": r["kernel"],
                             "us_per_step": round(r["us_per_step"], 1),
                             "calls_per_step": r["launch_calls_per_step"]}
                            for r in rows]}

    fused = measure()
    with _dense_attention_grad():
        dense = measure()
    line = {"mode": "train", "steps": steps,
            "step": "F + B forward, weighted-sum loss, backward()",
            "fused": fused, "dense_attention_grad": dense,
            "speedup_vs_dense": dense["step_ms_median"] /
            fused["step_ms_median"]}
    if deterministic:
        with _deterministic_algorithms():
            det = measure()
        line["fused_deterministic"] = det
        line["deterministic_vs_fused"] = det["step_ms_median"] / \
            fused["step_ms_median"]
    return line


def _profiler_table(fn, ksteps):
    """Device kernels of ``ksteps`` calls of ``fn``: per kernel name the time
    and launches per step (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ksteps):
            fn()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        r = rows.setdefault(ev.name, [0.0, 0])
        r[0] += ev.device_time_total if hasattr(ev, "device_time_total") \
            else ev.cuda_time_total
        r[1] += 1
    out = [{"kernel": k, "us_per_step": round(us / ksteps, 1),
            "calls_per_step": n / ksteps} for k, (us, n) in rows.items()]
    out.sort(key=lambda r: -r["us_per_step"])
    return out


def graphed_pair(w, steps, warmup, flush, dev):
    """The fused step plus SGD ``optimizer.step()``, eager and replayed from a
    CUDA graph, alternating step by step on the same inputs (two input sets,
    copied into the step's static buffers before each step)."""
    leaves = [t.detach().clone().requires_grad_()
              for t in [w.feat, w.depth] + list(w.more)]
    feat, depth, more = leaves[0], leaves[1], leaves[2:]
    cam = [t.clone() for t in w.cam]
    mods = [m for m in (w.vt, w.bp) if m is not None]
    params = [p for m in mods for p in m.parameters()]
    for m in mods:
        m.requires_grad_(True)
    opt = torch.optim.SGD(params, lr=1e-7)
    g = torch.Generator(device=dev).manual_seed(31)
    flip = torch.diag(torch.tensor([-1.0, 1.0, 1.0], device=dev))
    sets = [[t.detach().clone() for t in leaves] + list(w.cam),
            [t.detach() + 0.01 * torch.randn(t.shape, generator=g, device=dev)
             for t in leaves] + list(w.cam[:5]) + [w.cam[5] @ flip]]
    loss_w = []

    def load(i):
        with torch.no_grad():
            for d, s in zip(leaves + cam, sets[i % 2]):
                d.copy_(s)

    def step():
        outs = []
        if w.vt is not None:
            outs.append(w.vt(cam, feat, depth))
        outs.append(w.bp([feat] + more, None, lss_bev=w.lss, cam_params=cam,
                         pred_img_depth=depth))
        if not loss_w:
            gl = torch.Generator(device=dev).manual_seed(29)
            loss_w.extend(torch.randn(o.shape, generator=gl, device=dev)
                          for o in outs)
        sum((o * k).sum() for o, k in zip(outs, loss_w)).backward()
        opt.step()

    def eager():
        opt.zero_grad(set_to_none=True)
        for t in leaves:
            t.grad = None
        step()

    load(0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(max(warmup, 2)):
            eager()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eager_peak = torch.cuda.max_memory_allocated(dev)
    opt.zero_grad(set_to_none=True)
    for t in leaves:
        t.grad = None
    torch.cuda.reset_peak_memory_stats(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    torch.cuda.synchronize()
    # the graph keeps its own gradient buffers in its pool; eager steps
    # allocate theirs, so the two arms interleave safely
    graph_peak = torch.cuda.max_memory_allocated(dev)
    arms = {"eager": eager, "graphed": graph.replay}
    times = {k: [] for k in arms}
    for i in range(max(warmup, 2)):
        for fn in arms.values():
            load(i)
            fn()
    torch.cuda.synchronize()
    for i in range(steps):
        for name, fn in arms.items():
            load(i)
            flush.zero_()
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    ksteps = max(2, min(steps, 5))
    res = {}
    for name, fn in arms.items():
        res[name] = {
            "step_ms_median": statistics.median(times[name]),
            "step_ms_min": min(times[name]),
            "kernels": _profiler_table(fn, ksteps)}
    res["graphed"]["max_memory_allocated_mb"] = graph_peak / 2**20
    res["eager"]["max_memory_allocated_mb"] = eager_peak / 2**20
    res["launch_and_host_ms"] = res["eager"]["step_ms_median"] - \
        res["graphed"]["step_ms_median"]
    res["step"] = ("F + B forward, weighted-sum loss, backward(), "
                   "SGD optimizer.step(); inputs copied in before each step")
    del graph
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="fbocc200",
                    choices=sorted(c for c in bench.CONFIGS
                                   if bench.CONFIGS[c]["do_b"]))
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--deterministic", action="store_true",
                    help="also time the fused step under "
                    "torch.use_deterministic_algorithms(True)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "train_step.py needs a CUDA device"
    dev = "cuda:0"
    torch.cuda.set_device(0)
    per_rank, _, _ = bench.frames_of(args.config, 1)
    w = bench.Workload(args.config, dev, seed=0, frames=per_rank)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    line = train_block(w, args.steps, args.warmup, flush, dev,
                       args.deterministic)
    line["graphed"] = graphed_pair(w, args.steps, args.warmup, flush, dev)
    if args.deterministic:
        with _deterministic_algorithms():
            line["graphed_deterministic"] = graphed_pair(
                w, args.steps, args.warmup, flush, dev)
    line.update(config=bench.config_dict(args.config, 1), gpu=gpu_identity(0))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
