"""Time the depth supervision at the FB-OCC training size: the reference's
eager expression (get_downsampled_gt_depth + get_depth_loss, depth_net.py:
396-450, evaluated with torch on the GPU) against the kernels
(``fbbev_depth_loss_fwd`` / ``_bwd``), forward plus backward.

    python tools/depth_loss_bench.py [--iters 50] [--out result.json]

B = 4, N = 6, gt 256 x 704, D = 80, ds 16, FB-OCC's depth bins
[2.0, 42.0, 0.5]; a seeded sparse gt (3 % of the pixels carry a depth) and
softmax predictions.  The two routes alternate call by call in one process,
each call after an L2 flush (256 MiB memset), with CUDA events around the
forward and the backward (``torch.autograd.grad``: no accumulation kernel);
the median of ``--iters`` calls is printed.  On the kernel route the
per-entry-point times come from ``KernelTimer``'s events:
``fbbev_depth_loss_fwd`` is the row kernel plus the one-CTA finish kernel.

Achieved bandwidth of the forward: the bytes the algorithm must move (the gt
map, the D predictions of each foreground pixel, the labels and the row
partials) over its time, against the H100 SXM's 3.35 TB/s.  The backward's
bytes: labels, foreground predictions and the dense gradient.  The card's
name, power limit and max SM clock are read in the same run.  Needs a CUDA
device.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
FBOCC = (2.0, 42.0, 0.5)


def card():
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
         "--format=csv,noheader"], stdout=subprocess.PIPE, text=True,
        check=True)
    return out.stdout.strip().splitlines()[0]


def eager_loss(gt, preds, ds, cfg, weight):
    import torch
    import torch.nn.functional as F
    D, h, w = preds.shape[-3:]
    H, W = gt.shape[-2:]
    x = gt.reshape(-1, H // ds, ds, W // ds, ds)
    x = x.permute(0, 1, 3, 2, 4).reshape(-1, ds * ds)
    x = torch.where(x == 0.0, 1e5 * torch.ones_like(x), x)
    t = (torch.min(x, dim=-1).values - (cfg[0] - cfg[2])) / cfg[2]
    t = torch.where((t < D + 1) & (t >= 0.0), t, torch.zeros_like(t))
    onehot = F.one_hot(t.long(), num_classes=D + 1)[:, 1:].float()
    p = preds.reshape(-1, D, h, w).permute(0, 2, 3, 1).reshape(-1, D)
    fg = torch.max(onehot, dim=1).values > 0.0
    s = F.binary_cross_entropy(p[fg], onehot[fg], reduction='none').sum()
    return weight * (s / max(1.0, fg.sum()))


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert args.iters >= 30
    import torch
    assert torch.cuda.is_available(), "depth_loss_bench needs a CUDA device"
    from fbbev_b200 import _lib
    from fbbev_b200.ops.depth_loss import depth_labels, depth_loss

    B, N, H, W, D, ds, wt = 4, 6, 256, 704, 80, 16, 3.0
    BN, h, w = B * N, H // ds, W // ds
    dev = "cuda"
    g = torch.Generator().manual_seed(0)
    hit = torch.rand(BN, H, W, generator=g) < 0.03
    val = torch.rand(BN, H, W, generator=g) * 50.0 - 3.0
    gt = torch.where(hit, val, torch.zeros(())).view(B, N, H, W).to(dev)
    preds = (torch.randn(BN, D, h, w, generator=g) * 3.0).softmax(1)
    preds = preds.view(B, N, D, h, w).to(dev).requires_grad_()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def ev():
        return torch.cuda.Event(enable_timing=True)

    def run_eager():
        e = [ev() for _ in range(3)]
        e[0].record()
        loss = eager_loss(gt, preds, ds, FBOCC, wt)
        e[1].record()
        grad, = torch.autograd.grad(loss, preds)
        e[2].record()
        return e, loss, grad

    def run_kernels(kt):
        e = [ev() for _ in range(3)]
        e[0].record()
        loss = depth_loss(gt, preds, ds, FBOCC, wt)
        e[1].record()
        grad, = torch.autograd.grad(loss, preds)
        e[2].record()
        return e, loss, grad

    # warm-up and agreement check
    _, l_e, g_e = run_eager()
    with _lib.KernelTimer() as kt:
        _, l_k, g_k = run_kernels(kt)
    torch.cuda.synchronize()
    grad_equal = bool(torch.equal(g_e, g_k))
    loss_rel = abs(l_k.item() - l_e.item()) / abs(l_e.item())
    n_fg = int((depth_labels(gt, ds, FBOCC, D) > 0).sum())

    times = {k: [] for k in ("eager_fwd", "eager_bwd", "eager_total",
                             "kern_fwd", "kern_bwd", "kern_total",
                             "fbbev_depth_loss_fwd", "fbbev_depth_loss_bwd")}
    with _lib.KernelTimer() as kt:
        for i in range(args.iters):
            order = ("eager", "kern") if i % 2 == 0 else ("kern", "eager")
            for route in order:
                flush.zero_()
                kt.records.clear()
                e, _, _ = run_eager() if route == "eager" else run_kernels(kt)
                torch.cuda.synchronize()
                times[route + "_fwd"].append(e[0].elapsed_time(e[1]) * 1e3)
                times[route + "_bwd"].append(e[1].elapsed_time(e[2]) * 1e3)
                times[route + "_total"].append(e[0].elapsed_time(e[2]) * 1e3)
                if route == "kern":
                    for name, _, a, b in kt.records:
                        times[name].append(a.elapsed_time(b) * 1e3)
    med = {k: median(v) for k, v in times.items() if v}

    fwd_bytes = BN * H * W * 4 + n_fg * D * 4 + BN * h * w * 4 + BN * h * 12
    bwd_bytes = BN * h * w * 4 + n_fg * D * 4 + BN * D * h * w * 4
    res = dict(
        card=card(), torch_device=torch.cuda.get_device_name(),
        shape=dict(B=B, N=N, H=H, W=W, D=D, ds=ds), n_fg=n_fg,
        iters=args.iters, median_us=med,
        speedup_total=med["eager_total"] / med["kern_total"],
        fwd_algorithmic_bytes=fwd_bytes, bwd_algorithmic_bytes=bwd_bytes,
        fwd_kernel_bw_TBps=fwd_bytes / med["fbbev_depth_loss_fwd"] / 1e6,
        fwd_kernel_share_of_3p35TBps=fwd_bytes / med["fbbev_depth_loss_fwd"]
        / 1e-6 / HBM_PEAK,
        bwd_kernel_bw_TBps=bwd_bytes / med["fbbev_depth_loss_bwd"] / 1e6,
        grad_bitwise_equal=grad_equal, loss_rel_diff=loss_rel)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
