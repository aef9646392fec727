"""CPU tests of the host-side mirror of the BEVDet-lineage callers and the
depth-net tail (SURVEY.md section 8 f3 / f4): registry names, constructor
contract, state-dict keys, ``get_mlp_input`` against the reference's own output,
and that nothing in them computes on the CPU (the kernels are the product)."""
import numpy as np
import pytest
import torch

from conftest import load_golden

GRID = dict(x=[-40, 40, 4.0], y=[-40, 40, 4.0], z=[-1, 5.4, 3.2],
            depth=[2.0, 42.0, 4.0])


def test_registry_names_and_state_dict_keys():
    """The three necks classes build from the reference's config dicts and
    carry ``depth_net.*`` only (no dx / bx / nx: necks/view_transformer.py:35-58
    registers none)."""
    from fbbev_b200.registry import NECKS
    for name in ("LSSViewTransformer", "LSSViewTransformer2"):
        m = NECKS.build(dict(type=name, grid_config=GRID, input_size=(64, 176),
                             downsample=16, in_channels=16, out_channels=8))
        assert sorted(m.state_dict()) == ["depth_net.bias", "depth_net.weight"]
        assert tuple(m.depth_net.weight.shape) == (m.D + 8, 16, 1, 1)
        assert m.D == 10 and m.initial_flag and not m.accelerate
        assert tuple(m.frustum.shape) == (10, 4, 11, 3)
        assert [int(v) for v in m.grid_size] == [20, 20, 2]
    from fbbev_b200.view_transformation.bevdet_lineage import (
        DEPTH_THRESHOLD, LSSViewTransformer, LSSViewTransformer2)
    assert LSSViewTransformer.depth_threshold is None
    assert LSSViewTransformer2.depth_threshold == DEPTH_THRESHOLD == 0.01


def test_bevdepth_needs_a_depth_net_and_mlp_input_matches_reference():
    from fbbev_b200.view_transformation.bevdet_lineage import \
        LSSViewTransformerBEVDepth
    kw = dict(grid_config=GRID, input_size=(64, 176), downsample=16,
              in_channels=16, out_channels=8)
    with pytest.raises(ValueError):
        LSSViewTransformerBEVDepth(**kw)
    net = torch.nn.Identity()
    m = LSSViewTransformerBEVDepth(depthnet_cfg=dict(module=net), **kw)
    assert m.depth_net is net and m.loss_depth_weight == 3.0
    g = load_golden("l_lss_bevdepth")
    cam = [torch.from_numpy(g[k]) for k in
           ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    np.testing.assert_array_equal(m.get_mlp_input(*cam).numpy(),
                                  g["mlp_input"])          # :1010-1034
    assert m.get_mlp_input(*cam).shape[-1] == 27


def test_cm_tail_adopts_the_reference_state_dict_keys():
    from fbbev_b200.view_transformation.depth_net_tail import CM_DepthNetTail
    g = load_golden("l_cm_tail")
    mid, C = g["ctx_in"].shape[1], g["context"].shape[2]
    tail = CM_DepthNetTail(mid, C)
    assert sorted(tail.state_dict()) == ["context_conv.bias",
                                         "context_conv.weight"]
    # a full CM_DepthNet state dict loads non-strictly (extra keys ignored)
    sd = {"context_conv.weight": torch.from_numpy(g["context_conv_weight"]),
          "context_conv.bias": torch.from_numpy(g["context_conv_bias"]),
          "depth_conv.0.conv1.weight": torch.zeros(1)}
    missing, unexpected = tail.load_state_dict(sd, strict=False)
    assert not missing and unexpected == ["depth_conv.0.conv1.weight"]


def test_no_cpu_fallback_in_the_new_ops():
    """lift_tail / bev_mask_fold / the thresholded index builder refuse CPU
    tensors instead of computing anything there."""
    from fbbev_b200 import _lib
    from fbbev_b200.ops.bev_pool_v2 import voxel_pooling_prepare_v2
    from fbbev_b200.ops.lift_tail import lift_tail
    from fbbev_b200.ops.ms_deform_attn import bev_mask_fold
    with pytest.raises(_lib.FbbevError):
        lift_tail(torch.zeros(1, 4, 2, 2), torch.zeros(1, 3, 2, 2))
    with pytest.raises(_lib.FbbevError):
        bev_mask_fold(torch.zeros(2, 1, 8, 4, dtype=torch.bool),
                      torch.ones(1, 8, dtype=torch.bool))
    with pytest.raises(_lib.FbbevError):
        voxel_pooling_prepare_v2(torch.zeros(1, 1, 2, 2, 2, 3), [0, 0, 0],
                                 [1, 1, 1], [4, 4, 4],
                                 depth=torch.ones(1, 1, 2, 2, 2))


def test_header_declares_the_new_entry_points():
    import os
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(here, "include", "fbbev_b200.h")).read()
    for sym in ("fbbev_ffn_fwd", "fbbev_ffn_supported", "fbbev_lift_tail_fwd",
                "fbbev_voxel_prepare", "fbbev_voxel_prepare_cams",
                "fbbev_bev_mask_fold", "fbbev_bev_mask_fold_workspace_bytes"):
        assert sym + "(" in hdr, sym
        assert hasattr(__import__("fbbev_b200")._lib.lib(), sym)
