"""Time the dense lift-splat pooling call alone on the bench.py workloads.

    python tools/pool_bench.py [--config fbocc200 unit large frames16]
                               [--iters 50] [--libs A.so B.so --rounds 3]

Per config, the index of ``bench.Workload(config, seed=0)`` is built once
(with the pooling plan the index builder fills, as in a step) and
``fbbev_bev_pool_v2_fwd_dense_planned`` -- both pooling kernels and the side
stream, the row bench.py calls ``bev_pool_v2_fwd_dense_planned`` -- is timed
on it: L2 flushed (256 MiB memset) before each call, the call queued behind a
short spin kernel so that the events bracket device time only, CUDA events
around it, median of ``--iters`` calls.  ``frames16`` is one frame (frame 7)
of the 16-frame workload.  Beside each config it prints the index statistics
that decide the pooling's work split (intervals by length, the interval-sum
rows V, tiles and their long intervals) and the time of a plain device write
of the same volume (``zero_`` of an equal tensor, same flush and median) as
the write ceiling of the card; the card's name, power limit and max SM clock
are printed with the numbers.

With ``--libs`` each library (through ``FBBEV_LIB``) runs in its own process,
alternating, ``--rounds`` times; min / median over the rounds are printed
side by side.  Needs a CUDA device.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
SHORT = 8          # kShortLen in csrc/bev_pool_split.cu


def card():
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
         "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def pick_tile(c):
    """The write kernel's tile (split_pick_tile in csrc/bev_pool_split.cu)."""
    smem = lambda t: (t + 1) * (c + 4) * 4 + 3 * t * 4   # noqa: E731
    if smem(128) <= 40 * 1024:
        return 128
    return 64 if smem(64) <= 45 * 1024 else 32


def workload(config):
    """(depth, feat NHWC, index, shape) of one frame of `config`."""
    import bench
    if config == "frames16":
        w = bench.Workload(config, "cuda", seed=0, frames=16)
        f = 7
        cam = [t[f:f + 1] for t in w.cam]
        depth, feat = w.depth[f:f + 1], w.feat[f:f + 1]
    else:
        w = bench.Workload(config, "cuda", seed=0, frames=1)
        cam, depth, feat = w.cam, w.depth, w.feat
    vt = w.vt
    feat = feat.permute(0, 1, 3, 4, 2).contiguous()
    depth = depth.contiguous()
    shape = vt._bev_feat_shape(depth, feat)
    idx = vt.prepare_index(vt.get_lidar_coor(*cam), pool_channels=shape[-1])
    return depth, feat, idx, shape


def index_stats(idx, shape):
    import torch
    B, Z, Y, X, C = shape
    zyx = Z * Y * X
    n_kept, n_int = (int(v) for v in idx.counts.tolist())
    ln = idx.interval_lengths[:n_int].long()
    rank = idx.ranks_bev[idx.interval_starts[:n_int].long()].long()
    T = pick_tile(C)
    tiles_per_b = -(-zyx // T)
    tile = rank // zyx * tiles_per_b + rank % zyx // T
    long_ = ln > SHORT
    n_tiles = B * tiles_per_b
    nonempty = int(torch.unique(tile).numel())
    long_tiles = int(torch.unique(tile[long_]).numel())
    frac = lambda k: round(float((ln <= k).float().mean()), 4) if n_int else 0.0  # noqa: E731
    return {
        "kept_points": n_kept, "intervals": n_int,
        "len_le_1": frac(1), "len_le_2": frac(2), "len_le_4": frac(4),
        "len_le_8": frac(8), "len_max": int(ln.max()) if n_int else 0,
        "V_MB": round(n_int * C * 4 / 1e6, 1),
        "tile_voxels": T, "tiles": n_tiles, "nonempty_tiles": nonempty,
        "long_intervals": int(long_.sum()),
        "long_points": int(ln[long_].sum()),
        "long_V_MB": round(int(long_.sum()) * C * 4 / 1e6, 2),
        "tiles_with_long": long_tiles,
        "volume_MB": round(B * C * zyx * 4 / 1e6, 1),
    }


def child(configs, iters):
    import torch
    from fbbev_b200.ops.bev_pool_v2 import _dense_forward
    assert torch.cuda.is_available(), "tools/pool_bench.py needs a CUDA device"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def median_us(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(iters):
            flush.zero_()
            torch.cuda._sleep(200_000)     # the call is queued before it runs
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        ts.sort()
        return ts[len(ts) // 2]

    rows = []
    with torch.no_grad():
        for config in configs:
            depth, feat, idx, shape = workload(config)
            args = (depth, feat, idx.ranks_depth, idx.ranks_feat, idx.ranks_bev,
                    shape, idx.interval_starts, idx.interval_lengths,
                    idx.n_intervals_dev, idx.plan)
            us = median_us(lambda: _dense_forward(*args))
            vol = torch.empty(_dense_forward(*args).numel(), device="cuda")
            write_us = median_us(vol.zero_)
            stats = index_stats(idx, shape)
            rows.append({"config": config, "us": round(us, 2),
                         "write_ceiling_us": round(write_us, 2), **stats})
            del vol, args, idx, depth, feat
            torch.cuda.empty_cache()
    print(json.dumps(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+",
                    default=["fbocc200", "unit", "large", "frames16"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--libs", nargs="+", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    assert args.iters >= 30, "median of at least 30 calls"
    if args.child:
        child(args.config, args.iters)
        return
    print("card:", card())
    libs = args.libs or [os.environ.get("FBBEV_LIB", "")]
    runs = {lib: [] for lib in libs}
    for _ in range(args.rounds if args.libs else 1):
        for lib in libs:
            env = dict(os.environ)
            if lib:
                env["FBBEV_LIB"] = os.path.abspath(lib)
            out = subprocess.run(
                [sys.executable, os.path.abspath(__file__), "--child", "--iters",
                 str(args.iters), "--config"] + args.config,
                env=env, stdout=subprocess.PIPE, text=True, check=True)
            runs[lib].append(json.loads(out.stdout.strip().splitlines()[-1]))
    base = runs[libs[0]][0]
    for j, row in enumerate(base):
        print(f"\n{row['config']}: " + ", ".join(
            f"{k} {v}" for k, v in row.items()
            if k not in ("config", "us", "write_ceiling_us")))
        ceil = sorted(r[j]["write_ceiling_us"] for lib in libs
                      for r in runs[lib])
        ceil_med = ceil[len(ceil) // 2]
        print(f"  write ceiling (zero_ of the {row['volume_MB']} MB volume): "
              f"min {ceil[0]:.1f} / median {ceil_med:.1f} us "
              f"({row['volume_MB'] * 1e6 / (ceil_med * 1e-6) / 1e12:.2f} TB/s)")
        for i, lib in enumerate(libs):
            us = sorted(r[j]["us"] for r in runs[lib])
            med = us[len(us) // 2]
            print(f"  lib {i}: pooling min {us[0]:7.1f} / median {med:7.1f} us"
                  f"  = {ceil_med / med:.2f} of the write ceiling"
                  f"  ({row['volume_MB'] * 1e6 / HBM_BPS * 1e6 / med:.2f} of "
                  f"3.35 TB/s for the volume alone)")
    for i, lib in enumerate(libs):
        print(f"lib {i}: {lib or 'default'}")
    print(json.dumps({"card": card(), "libs": libs, "runs": runs}))


if __name__ == "__main__":
    main()
