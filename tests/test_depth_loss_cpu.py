"""CPU tests of the depth supervision (csrc/depth_loss.cu, ops/depth_loss.py):
the float64 reference (tests/depth_loss_ref64.py) against the reference's own
golden (tests/golden/d_depth_loss.npz), argument validation of the C ABI
before anything is enqueued, and the ptxas figures of the kernels."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from depth_loss_ref64 import grad_ref64, labels_ref, loss_ref64, onehot_ref

CASES = ("fbocc", "lineage", "ds8")


def _case(name):
    z = load_golden("d_depth_loss")
    return {k.split("/", 1)[1]: v for k, v in z.items()
            if k.startswith(name + "/")}


@pytest.mark.parametrize("case", CASES)
def test_ref64_matches_golden(case):
    c = _case(case)
    D, ds, wt = int(c["D"]), int(c["downsample"]), float(c["loss_weight"])
    labels = labels_ref(c["gt"], ds, tuple(c["depth_cfg"]), D)
    np.testing.assert_array_equal(labels, c["labels"])
    np.testing.assert_array_equal(onehot_ref(labels, D), c["onehot"])
    assert int((labels > 0).sum()) == int(c["n_fg"])
    assert 0 < int(c["n_fg"]) < labels.size      # both kinds of pixel occur
    loss = loss_ref64(labels, c["preds"], D, wt)
    assert abs(loss - float(c["loss"])) <= 1e-5 * abs(loss)
    g = grad_ref64(labels, c["preds"], D, wt)
    assert g.shape == c["grad"].shape
    np.testing.assert_allclose(c["grad"], g, rtol=1e-5, atol=0)


def test_ref64_edge_rules():
    """Zeros become 1e5 (so an all-zero patch is background), a NaN anywhere
    in a patch makes the pixel background, t in [0, 1) is class 0 and
    t in [D, D + 1) is the last bin."""
    cfg, D, ds = (2.0, 42.0, 0.5), 80, 2
    gt = np.zeros((1, 2, 12), np.float32)
    gt[0, 0, 2:4] = [5.0, -0.0]          # patch 1: min 5.0 -> t = 7
    gt[0, 1, 4] = np.nan                 # patch 2: NaN
    gt[0, 0, 5] = 3.0
    gt[0, 0, 6] = 1.9                    # patch 3: t = 0.8 -> class 0
    gt[0, 0, 8] = 41.9                   # patch 4: t = 80.8 -> class 80
    gt[0, 0, 10] = 42.0                  # patch 5: t = 81 -> out of range
    np.testing.assert_array_equal(labels_ref(gt, ds, cfg, D),
                                  [0, 7, 0, 0, 80, 0])
    preds = np.full((1, D, 1, 6), 0.5, np.float32)
    preds[0, :, 0, 1] = 0.0              # log(0) clamps at -100
    labels = labels_ref(gt, ds, cfg, D)
    assert loss_ref64(labels, preds, D, 1.0) == pytest.approx(
        (100.0 + 79 * np.log(2.0) + 79 * 0.0 + np.log(2.0)) / 2)
    g = grad_ref64(labels, preds, D, 1.0)
    assert g[0, 6, 0, 1] == pytest.approx(0.5 * -1.0 / 1e-12)
    assert not g[0, :, 0, [0, 2, 3, 5]].any()


def _lib():
    from fbbev_b200 import _lib
    return _lib.lib()


# arbitrary aligned non-NULL addresses: every call below is refused (or is a
# no-op) before anything touches device memory
P = ctypes.c_void_p(0x10000)
P2 = ctypes.c_void_p(0x20000)


def _fwd(L, gt=P, preds=P, bn=2, H=64, W=176, ds=16, d=80, labels=P,
         loss=P, n_fg=P, ws=P2, ws_bytes=1 << 20):
    return L.fbbev_depth_loss_fwd(gt, preds, bn, H, W, ds, d, 1.5, 0.5, 3.0,
                                  labels, loss, n_fg, ws, ws_bytes, None)


def test_fwd_argument_validation_without_gpu():
    L = _lib()
    assert _fwd(L, H=72) == -1                    # H % ds
    assert _fwd(L, W=170) == -1                   # W % ds
    assert _fwd(L, ds=0) == -1
    assert _fwd(L, d=0) == -1
    assert _fwd(L, d=-3) == -1
    assert _fwd(L, bn=-1) == -1
    for kw in ("gt", "labels", "loss", "n_fg", "ws"):
        assert _fwd(L, **{kw: None}) == -1, kw
    assert _fwd(L, gt=ctypes.c_void_p(0x10002)) == -1         # misaligned
    assert _fwd(L, preds=ctypes.c_void_p(0x10001)) == -1
    assert _fwd(L, ws=ctypes.c_void_p(0x20008)) == -1         # < 16 B aligned
    need = L.fbbev_depth_loss_workspace_bytes(2, 64, 16)
    assert need >= 2 * 4 * (8 + 4)                # a (sum, count) per row
    assert _fwd(L, ws_bytes=need - 1) == -2       # workspace too small
    # labels only: preds, loss, n_fg NULL together
    assert _fwd(L, preds=None) == -1
    assert _fwd(L, preds=None, loss=None) == -1
    # empty batch: a no-op, whatever the pointers
    assert L.fbbev_depth_loss_fwd(None, None, 0, 64, 176, 16, 80, 1.5, 0.5,
                                  3.0, None, None, None, None, 0, None) == 0
    assert L.fbbev_depth_loss_fwd(None, None, 0, 60, 176, 16, 80, 1.5, 0.5,
                                  3.0, None, None, None, None, 0, None) == -1
    assert L.fbbev_depth_loss_workspace_bytes(0, 64, 16) == 0


def test_bwd_argument_validation_without_gpu():
    L = _lib()
    ok = dict(labels=P, preds=P, n_fg=P, g=P, out=P2)

    def bwd(bn=2, h=4, w=11, d=80, **kw):
        a = dict(ok, **kw)
        return L.fbbev_depth_loss_bwd(a["labels"], a["preds"], a["n_fg"],
                                      a["g"], bn, h, w, d, 3.0, a["out"], None)
    for k in ok:
        assert bwd(**{k: None}) == -1, k
    assert bwd(out=ctypes.c_void_p(0x20002)) == -1
    assert bwd(d=0) == -1
    assert bwd(h=0) == -1
    assert bwd(bn=-1) == -1
    assert L.fbbev_depth_loss_bwd(None, None, None, None, 0, 4, 11, 80, 3.0,
                                  None, None) == 0


def test_cpu_tensors_raise():
    from fbbev_b200 import _lib as lib_mod
    from fbbev_b200.ops import depth_loss as dl
    gt = torch.zeros(1, 2, 32, 64)
    preds = torch.full((1, 2, 80, 2, 4), 1 / 80)
    with pytest.raises(lib_mod.FbbevError):
        dl.depth_loss(gt, preds, 16, [2.0, 42.0, 0.5], 3.0)
    with pytest.raises(lib_mod.FbbevError):
        dl.downsampled_gt_depth(gt, 16, [2.0, 42.0, 0.5], 80)


def test_sid_raises_and_state_dict_unchanged():
    from fbbev_b200.view_transformation.depth_net_tail import CM_DepthNetTail
    with pytest.raises(NotImplementedError):
        CM_DepthNetTail(16, 8, grid_config=dict(depth=[2.0, 42.0, 0.5]),
                        sid=True)
    t = CM_DepthNetTail(16, 8, downsample=16,
                        grid_config=dict(depth=[2.0, 42.0, 0.5]),
                        depth_channels=80, loss_depth_weight=3.0)
    assert sorted(t.state_dict()) == ["context_conv.bias",
                                      "context_conv.weight"]


def test_kernels_do_not_spill():
    log = os.path.join(ROOT, "build", "csrc", "depth_loss.ptxas.log")
    if not os.path.exists(log):
        pytest.skip(f"ptxas log not built: {log}")
    text = open(log).read()
    props = re.findall(
        r"Function properties for (_ZN5fbbev\d+depth_loss_\w+)\n"
        r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
        r"(\d+) bytes spill loads", text)
    names = {re.sub(r"_ZN5fbbev\d+", "", n).split("E", 1)[0]
             for n, *_ in props}
    assert names == {"depth_loss_fwd_kernel", "depth_loss_finish_kernel",
                     "depth_loss_bwd_kernel"}, names
    for name, stack, st, ld in props:
        assert (int(stack), int(st), int(ld)) == (0, 0, 0), name
