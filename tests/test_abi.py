"""CPU tests of the drop-in boundary: the C-ABI library loads (no GPU needed)
and exports every symbol include/fbbev_b200.h declares; the product path has no
CPU fallback and never touches oracle/."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "fbbev_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fbbev_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_all_exported():
    from fbbev_b200 import _lib
    names = declared_symbols()
    assert len(names) >= 12
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    assert sorted(_lib.EXPORTED_SYMBOLS) == names


def test_abi_version_and_error_strings():
    from fbbev_b200 import _lib
    L = _lib.lib()
    assert L.fbbev_abi_version() == 5
    assert L.fbbev_error_string(0) == b"ok"
    assert b"workspace" in L.fbbev_error_string(-2)
    assert L.fbbev_bev_pool_v2_dense_workspace_bytes(1, 640000, 1000, 2000, 80) >= 4 * (
        640000 // 32 + 1) + 1000 * 80 * 4
    assert L.fbbev_voxel_prepare_workspace_bytes(1000, 5000) > 0


def test_dense_pool_plan_covers_every_shape():
    """The index builder can fill a dense-pooling plan for any shape; the
    interval-sum rows V (n_int x C floats) are there only on the two-kernel
    path (C <= 512), so a C = 1024 workspace holds the plan tables alone."""
    from fbbev_b200 import _lib
    L = _lib.lib()
    ws = L.fbbev_bev_pool_v2_dense_workspace_bytes
    n_int, n_pts = 1000, 2000
    assert ws(1, 64, n_int, n_pts, 512) >= n_int * 512 * 4
    assert ws(1, 64, n_int, n_pts, 1024) == ws(1, 64, n_int, n_pts, 13)
    # plan tables only: fewer than 4 words per interval, no row of C floats
    assert 0 < ws(1, 64, n_int, n_pts, 1024) < n_int * 4 * 4


def test_no_32_point_interval_sum_group_is_built():
    """C <= 512 on the two-kernel path: the interval-sum kernel is built for
    point groups of 4, 8 and 16 only (the 32-point group spills)."""
    log = os.path.join(ROOT, "build", "csrc", "bev_pool_split.ptxas.log")
    if not os.path.exists(log):
        pytest.skip(f"ptxas log not built: {log}")
    names = set(re.findall(r"_ZN5fbbev20interval_sums_kernelILi(\d+)E",
                           open(log).read()))
    assert names == {"4", "8", "16"}, names


def test_argument_validation_without_gpu():
    """Argument errors are reported before anything is enqueued."""
    from fbbev_b200 import _lib
    L = _lib.lib()
    assert L.fbbev_bev_pool_v2_fwd(None, None, None, None, None, None, None,
                                   -1, 80, None, None) == -1
    assert L.fbbev_bev_pool_v2_fwd(None, None, None, None, None, None, None,
                                   0, 80, None, None) == 0   # empty: no-op
    assert L.fbbev_msda_fwd(None, None, None, None, None, 1, 10, 8, 7, 1, 5,
                            4, None, None) == -1             # NULL pointers
    assert L.fbbev_da_sca_fwd(*([None] * 10), 1, 6, 10, 10, 8, 10, 1, 7, 4,
                              80, None, None, 0, 0, None) == -1  # points % Z != 0
    assert L.fbbev_da_sca_workspace_bytes(2, 6) >= 2 * 6 * 4
    # the index builder refuses a pooling plan without channels
    fake = 1 << 20          # a non-NULL pointer that is never dereferenced
    grid = [_lib.c_floats(v) for v in ([0, 0, 0], [1, 1, 1], [4, 4, 4])]
    need = L.fbbev_voxel_prepare_workspace_bytes(16, 64)
    assert L.fbbev_voxel_prepare(fake, None, 0.0, 1, 1, 1, 4, 4, *grid,
                                 *([fake] * 6), fake, need, 0, fake, 1 << 20,
                                 None) == -3


def test_no_cpu_fallback():
    """Ops refuse CPU tensors instead of silently computing elsewhere."""
    from fbbev_b200 import _lib
    from fbbev_b200.ops.bev_pool_v2 import bev_pool_v2
    d = torch.zeros(1, 1, 2, 2, 2)
    f = torch.zeros(1, 1, 2, 2, 2)
    i = torch.zeros(4, dtype=torch.int32)
    with pytest.raises(_lib.FbbevError):
        bev_pool_v2(d, f, i, i, i, (1, 1, 2, 2, 2), i[:2], i[:2])


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "fb-bev_b200")
    for dirpath, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src,
                                     flags=re.M), fn
                assert "libfbbev_oracle" not in src, fn
