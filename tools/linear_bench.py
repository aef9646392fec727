"""Time every Linear / FFN call of a bench.py workload in isolation.

    python tools/linear_bench.py [--config fbocc200 bwd_only] [--iters 50]
                                 [--libs A.so B.so --rounds 3]

The calls are discovered by running one step of ``bench.Workload`` with the
C-ABI calls recorded (``_lib.KernelTimer``); each distinct call shape is then
replayed on fresh seeded tensors of the same shapes, row pitches and optional
operands.  Every shape is warmed up first; each timed call is bracketed by
CUDA events with L2 flushed (256 MiB memset) before it, and the median is
reported.  Per call: µs, algorithmic bytes (bench.py's accounting), the share
of the HBM bound at 3.35 TB/s and, for the FFN, the share of the 3xTF32 math
bound at the data sheet's 495 TFLOP/s (a 700 W figure).  The card's name,
power limit and max SM clock are printed with the numbers.

With ``--libs`` each library (through ``FBBEV_LIB``) runs in its own process,
alternating, ``--rounds`` times, and the per-call minimum / median over the
rounds is printed side by side.  Needs a CUDA device.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12
TF32_FLOPS = 495e12
CALLS = ("fbbev_linear_fwd", "fbbev_linear_fwd_split", "fbbev_ffn_fwd")


def card():
    out = subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
         "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, check=True)
    return out.stdout.strip().splitlines()[0]


def discover(config):
    """(name, shape args) of every distinct Linear / FFN call of one step."""
    import torch
    import bench
    from fbbev_b200 import _lib
    w = bench.Workload(config, "cuda", seed=0, frames=1)
    w.step()
    torch.cuda.synchronize()
    with _lib.KernelTimer() as kt:
        w.step()
    torch.cuda.synchronize()
    counts, calls = {}, {}
    for name, a, _, _ in kt.records:
        if name not in CALLS:
            continue
        a = tuple(None if isinstance(v, ctypes.c_void_p) and not v.value else v
                  for v in a)
        key = (name,) + tuple(v if isinstance(v, (int, float)) else v is not None
                              for v in a[:-1])
        counts[key] = counts.get(key, 0) + 1
        calls.setdefault(key, (name, a))
    del w
    return [(name, a, counts[key]) for key, (name, a) in calls.items()]


def replay_args(name, a, g):
    """Fresh tensors for call `a` (same shapes, pitches, optional operands);
    returns (args, keep-alive list)."""
    import torch
    from fbbev_b200 import _lib
    L = _lib.lib()
    keep = []

    def buf(rows, pitch):
        t = torch.randn(rows, pitch, device="cuda", generator=g)
        keep.append(t)
        return _lib.ptr(t)

    def vec(n, present):
        return buf(1, n) if present else None

    def packed(n, k):
        w = torch.randn(n, k, device="cuda", generator=g) / k ** 0.5
        p = torch.empty(L.fbbev_linear_packed_bytes(n, k) // 4, device="cuda")
        _lib.check(L.fbbev_linear_pack(_lib.ptr(w), n, k, _lib.ptr(p), None), "pack")
        keep.append(p)
        return _lib.ptr(p)

    sp = _lib.stream_ptr("cuda")
    if name == "fbbev_linear_fwd":
        (x, ldx, _, b, r, ldr, lw, lb, m, k, n, relu, eps, y, ldy, _) = a
        return (buf(m, ldx), ldx, packed(n, k), vec(n, b), buf(m, ldr) if r else None,
                ldr, vec(n, lw), vec(n, lb), m, k, n, relu, eps, buf(m, ldy), ldy,
                sp), keep
    if name == "fbbev_linear_fwd_split":
        (x, ldx, xa, ldxa, _, b, m, k, n, ns, relu, y0, ldy0, y1, ldy1, _) = a
        return (buf(m, ldx), ldx, buf(m, ldxa) if xa else None, ldxa, packed(n, k),
                vec(n, b), m, k, n, ns, relu, buf(m, ldy0), ldy0,
                buf(m, ldy1) if y1 else None, ldy1, sp), keep
    (x, ldx, _, b1, _, b2, r, ldr, lw, lb, m, e, h, eps, y, ldy, _) = a
    w1 = torch.cat([torch.empty(L.fbbev_linear_packed_bytes(80, e) // 4, device="cuda")
                    for _ in range(h // 80)])
    w1.normal_(generator=g)
    keep.append(w1)
    return (buf(m, ldx), ldx, _lib.ptr(w1), vec(h, b1), packed(e, h), vec(e, b2),
            buf(m, ldr) if r else None, ldr, vec(e, lw), vec(e, lb), m, e, h, eps,
            buf(m, ldy), ldy, sp), keep


def child(configs, iters):
    import torch
    import bench
    from fbbev_b200 import _lib
    assert torch.cuda.is_available(), "tools/linear_bench.py needs a CUDA device"
    L = _lib.lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for config in configs:
        calls = discover(config)
        prepared = [(name, a, n) + replay_args(name, a, g) for name, a, n in calls]
        with torch.no_grad():
            for name, _, _, args, _ in prepared:          # warm every shape
                for _ in range(3):
                    _lib.check(getattr(L, name)(*args), name)
            torch.cuda.synchronize()
            for name, a, n, args, _ in prepared:
                ts = []
                for _ in range(iters):
                    flush.zero_()
                    e0 = torch.cuda.Event(enable_timing=True)
                    e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    rc = getattr(L, name)(*args)
                    e1.record()
                    _lib.check(rc, name)
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1) * 1e3)
                ts.sort()
                us = ts[len(ts) // 2]
                label, nbytes = bench._call_key(name, a, {})
                row = {"config": config, "call": label, "calls_per_step": n,
                       "us": round(us, 2), "bytes": nbytes,
                       "hbm_share": round(nbytes / HBM_BPS * 1e6 / us, 3)}
                if name == "fbbev_ffn_fwd":
                    m, e, h = a[10], a[11], a[12]
                    row["math_share"] = round(
                        3 * 2 * 2 * m * e * h / TF32_FLOPS * 1e6 / us, 3)
                rows.append(row)
    print(json.dumps(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", nargs="+", default=["fbocc200", "bwd_only"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--libs", nargs="+", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
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
    print(f"{'config':9} {'call':58} {'n':>2} " +
          " ".join(f"{'us min/med ' + str(i):>18} {'hbm':>5}" for i in range(len(libs))) +
          "  math")
    for j, row in enumerate(base):
        cells = []
        for lib in libs:
            us = sorted(r[j]["us"] for r in runs[lib])
            med = us[len(us) // 2]
            cells.append(f"{us[0]:8.1f}/{med:8.1f} "
                         f"{row['bytes'] / HBM_BPS * 1e6 / med:5.2f}")
        math = ""
        if "math_share" in row:
            med = sorted(r[j]["us"] for r in runs[libs[-1]])[len(runs[libs[-1]]) // 2]
            math = f"{row['math_share'] * row['us'] / med:5.2f}"
        print(f"{row['config']:9} {row['call'][:58]:58} {row['calls_per_step']:>2} " +
              " ".join(cells) + "  " + math)
    for i, lib in enumerate(libs):
        print(f"lib {i}: {lib or 'default'}")
    print(json.dumps({"card": card(), "libs": libs, "runs": runs}))


if __name__ == "__main__":
    main()
