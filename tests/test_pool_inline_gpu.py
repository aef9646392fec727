"""The one-shot dense pooling (``fbbev_bev_pool_v2_fwd_dense_planned``), whose
write kernel folds intervals of up to 8 points itself, against the staged pair
(``fbbev_bev_pool_v2_sums_planned`` + ``fbbev_bev_pool_v2_write_planned``),
which folds every interval through the interval-sum rows: the two must agree
bit for bit (signed zeros included) on the bench workloads and on crafted
indexes around the short-interval bound and the 4- / 8- / 16-point groups and
32-point slices of the interval-sum kernel."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHORT = 8   # kShortLen in bev_pool_split.cu


def _both(depth, feat, rd, rf, rb, shape, st, ln, n_int_dev=None,
          n_kept_dev=None, plan=None):
    from fbbev_b200.ops.bev_pool_v2 import (bev_pool_v2_deferred,
                                            bev_pool_v2_dense)
    one = bev_pool_v2_dense(depth, feat, rd, rf, rb, shape, st, ln,
                            n_intervals_dev=n_int_dev, n_kept_dev=n_kept_dev,
                            plan=plan)
    staged = bev_pool_v2_deferred(depth, feat, rd, rf, rb, shape, st, ln,
                                  n_intervals_dev=n_int_dev).materialize()
    torch.cuda.synchronize()
    return one, staged


def _assert_bits(one, staged):
    assert one.shape == staged.shape
    assert torch.equal(one.view(torch.int32), staged.view(torch.int32))


@pytest.mark.parametrize("config", ["unit", "fbocc200", "frames16", "large"])
def test_one_shot_equals_staged_bench_configs(config):
    import bench
    frames = 16 if config == "frames16" else 1
    w = bench.Workload(config, DEV, seed=0, frames=frames)
    vt = w.vt
    feat = w.feat.permute(0, 1, 3, 4, 2)
    shape = vt._bev_feat_shape(w.depth, feat)
    idx = vt.prepare_index(vt.get_lidar_coor(*w.cam), pool_channels=shape[-1])
    one, staged = _both(w.depth, feat, idx.ranks_depth, idx.ranks_feat,
                        idx.ranks_bev, shape, idx.interval_starts,
                        idx.interval_lengths, idx.n_intervals_dev,
                        idx.n_kept_dev, idx.plan)
    _assert_bits(one, staged)
    assert one.abs().sum() > 0


def _crafted(lengths, ranks, c, batch, zyx, seed):
    """Index of intervals `lengths` at the sorted voxel ranks `ranks` (batch
    term included); random feat rows / depth bins, with exact zeros and
    negative depths so that signed-zero products occur."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.as_tensor(lengths, dtype=torch.int32)
    ranks = torch.as_tensor(ranks, dtype=torch.int32)
    assert lengths.numel() == ranks.numel()
    assert ranks.numel() < 2 or bool((ranks[1:] > ranks[:-1]).all())
    n = int(lengths.sum())
    n_feat, n_depth = 257, 311
    feat = torch.randn(n_feat, c, generator=g)
    feat[torch.rand(n_feat, c, generator=g) < 0.05] = 0.0
    depth = torch.randn(n_depth, generator=g)
    depth[::17] = 0.0
    st = torch.zeros(lengths.numel(), dtype=torch.int32)
    if lengths.numel() > 1:
        st[1:] = torch.cumsum(lengths, 0)[:-1].int()
    rb = torch.repeat_interleave(ranks, lengths.long())
    rf = torch.randint(0, n_feat, (n,), generator=g, dtype=torch.int32)
    rd = torch.randint(0, n_depth, (n,), generator=g, dtype=torch.int32)
    z = zyx // 64
    shape = (batch, z, 8, 8, c)
    assert z * 64 == zyx
    return [t.to(DEV) for t in (depth, feat, rd, rf, rb)] + [shape] + \
        [st.to(DEV), lengths.to(DEV)]


def _random_mix(seed, batch, zyx, n_int, p_long):
    rng = np.random.default_rng(seed)
    ranks = np.sort(rng.choice(batch * zyx, n_int, replace=False))
    short = rng.integers(1, SHORT + 2, n_int)          # 1 .. L + 1
    long_ = rng.integers(SHORT + 1, 80, n_int)
    lengths = np.where(rng.random(n_int) < p_long, long_, short)
    return lengths, ranks


@pytest.mark.parametrize("c", [4, 80, 132, 256, 512])
@pytest.mark.parametrize("batch", [1, 3])
def test_one_shot_equals_staged_random_mix(c, batch):
    """Lengths 1 .. L + 1 and some long intervals at random voxels: short
    intervals start at every offset of the point groups and slices."""
    zyx = 64 * 40
    lengths, ranks = _random_mix(c + batch, batch, zyx, 900 * batch, 0.1)
    one, staged = _both(*_crafted(lengths, ranks, c, batch, zyx, seed=c))
    _assert_bits(one, staged)


@pytest.mark.parametrize("c", [4, 80, 132, 512])
def test_one_shot_equals_staged_bound_and_straddle(c):
    """Intervals of exactly L and L + 1 points, and short intervals that
    straddle group and slice boundaries (offsets 3, 7, 15, 30, 31 of a
    32-point slice)."""
    lengths = []
    for lead in (3, 7, 15, 30, 31):
        pad = (-sum(lengths) + lead) % 32    # next interval starts at `lead`
        if pad:
            lengths.append(pad)
        lengths += [SHORT, SHORT + 1, 2, SHORT, 1, SHORT + 1, 5]
    ranks = np.arange(len(lengths)) * 3 + 1
    zyx = 64 * 8
    one, staged = _both(*_crafted(lengths, ranks, c, 1, zyx, seed=7))
    _assert_bits(one, staged)


@pytest.mark.parametrize("c", [4, 80, 512])
def test_one_shot_equals_staged_long_only_and_mixed_tiles(c):
    """Tiles holding only long intervals (every voxel of the first 256 a
    long interval), tiles mixing long and short intervals, short-only tiles
    and empty tiles."""
    long_only = [(v, SHORT + 1 + v % 40) for v in range(256)]
    mixed = [(v, SHORT + 4 if v % 5 == 0 else 1 + v % SHORT)
             for v in range(512, 768, 2)]
    short_only = [(v, 1 + v % SHORT) for v in range(1024, 1280, 3)]
    entries = long_only + mixed + short_only
    ranks = [r for r, _ in entries]
    lengths = [n for _, n in entries]
    zyx = 64 * 32
    one, staged = _both(*_crafted(lengths, ranks, c, 1, zyx, seed=11))
    _assert_bits(one, staged)


def test_one_shot_equals_staged_empty_index():
    zyx = 64 * 4
    args = _crafted([], [], 80, 2, zyx, seed=3)
    one, staged = _both(*args)
    _assert_bits(one, staged)
    assert not one.any()


def test_one_shot_refuses_c_above_512():
    """C > 512 is not a dense-op shape (FBBEV_ERR_UNSUPPORTED): the widest
    interval-sum group (32 points, C > 512) is never the fold's."""
    from fbbev_b200 import _lib
    L = _lib.lib()
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    out = torch.empty(4 * 1024 * 64, device=DEV)
    rc = L.fbbev_bev_pool_v2_fwd_dense_planned(
        None, None, None, None, None, None, None, 0, 0, 1024, 1, 64,
        _lib.ptr(out), _lib.ptr(ws), ws.numel(), _lib.stream_ptr(DEV))
    assert rc != 0
