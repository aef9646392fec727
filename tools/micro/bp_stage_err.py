"""Per-stage error of BackwardProjection.forward against the golden fixtures
recorded from the reference's own classes: where does the whole-module error
come from?  (development aid; run on the GPU box)"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from bp_common import build_bp, cam_params
from fbbev_b200.view_transformation import backward_projection as bp_mod

DEV = "cuda:0"


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def run(case, fused):
    g, bp = build_bp(case, DEV)
    enc = bp.transformer.encoder
    enc.fused_geometry = fused
    sca = enc.layers[0].attentions[1]
    cap = {}
    orig = sca.forward

    def spy(*a, **k):
        out = orig(*a, **k)
        cap['q'] = a[0]
        cap['ref'] = k['reference_points_cam']
        cap['dep'] = k['bev_query_depth']
        cap['mask'] = k['per_cam_mask_list']
        cap['out'] = out
        return out
    sca.forward = spy
    n_lvl = len(g["level_shapes"])
    mlvl = [t(g[f"feat{i}"]) for i in range(n_lvl)]
    with torch.no_grad():
        out = bp(mlvl, None, lss_bev=t(g["lss_bev"]),
                 cam_params=cam_params(g, DEV), pred_img_depth=t(g["depth"]))
    e = lambda a, b: float(np.abs(a.cpu().numpy().reshape(b.shape) - b).max())
    print(f"{case} fused_geometry={fused}")
    print("  self-attn+LN (sca_query) err", e(cap['q'], g["sca_query"]))
    # the reference's sca output includes the post-norm?  compare shape only
    m = cap['mask'].cpu().numpy()
    gm = g["per_cam_mask"]
    print("  mask flips", int((m != gm).sum()), "of", gm.size)
    dep = cap['dep'].cpu().numpy().reshape(g["bev_query_depth"].shape)
    db = g["dbound"]
    bins = lambda d: np.clip(np.floor((d - np.float32(db[0])) / np.float32(db[2])), 0, 39)
    both = (m & gm)
    bf = (bins(dep)[..., 0] != bins(g["bev_query_depth"])[..., 0]) & both
    print("  depth-bin flips among visible", int(bf.sum()), "of", int(both.sum()))
    rc = cap['ref'].cpu().numpy()
    print("  ref_cam err (visible)", float(np.abs(rc - g["reference_points_cam"])[both].max()))
    print("  final err", e(out, g["out"]))
    # with golden geometry injected
    def spy2(*a, **k):
        k = dict(k)
        k['reference_points_cam'] = t(g["reference_points_cam"])
        k['bev_query_depth'] = t(g["bev_query_depth"])
        k['per_cam_mask_list'] = t(g["per_cam_mask"])
        return orig(*a, **k)
    sca.forward = spy2
    with torch.no_grad():
        out2 = bp(mlvl, None, lss_bev=t(g["lss_bev"]),
                  cam_params=cam_params(g, DEV), pred_img_depth=t(g["depth"]))
    print("  final err with golden geometry", e(out2, g["out"]))
    fused_linear_on = bp_mod._fused_linear_on
    bp_mod._fused_linear_on = lambda x, *dropouts: False
    try:
        with torch.no_grad():
            out3 = bp(mlvl, None, lss_bev=t(g["lss_bev"]),
                      cam_params=cam_params(g, DEV),
                      pred_img_depth=t(g["depth"]))
    finally:
        bp_mod._fused_linear_on = fused_linear_on
    print("  ... and torch Linears", e(out3, g["out"]))
    print("  |out| max", float(np.abs(g["out"]).max()))


for case in ["b_bp_e80_1lvl", "b_bp_e64_3lvl"]:
    for fused in (True, False):
        run(case, fused)
