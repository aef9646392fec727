"""d_depth_loss.npz: the reference's own depth supervision, on CPU --
``get_downsampled_gt_depth`` + ``get_depth_loss`` of CM_DepthNet
(mmdet3d/models/fbbev/modules/depth_net.py:396-450) and of
LSSViewTransformerBEVDepth (mmdet3d/models/necks/view_transformer.py:
1036-1081), with d preds from the reference's autograd.

Both are plain methods; they run on a namespace ``self`` carrying the
attributes they read.  Cases (every key prefixed ``<case>/``):

  fbocc    CM_DepthNet, FB-OCC's depth bins [2.0, 42.0, 0.5] (D = 80), ds 16,
           sparse lidar-like gt (most pixels 0, some out of range)
  lineage  LSSViewTransformerBEVDepth, bins [1.0, 60.0, 1.0] (D = 59), ds 16
  ds8      CM_DepthNet, FB-OCC's bins, ds 8

All steps are powers of two, so the reference's CPU division and torch's CUDA
multiplication by the reciprocal give the same labels (the GPU tests pin the
non-power-of-two case against torch on the GPU).

Run in the build container (needs /root/reference):

    python tests/golden/gen_golden_depth_loss.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import ref_import  # noqa: E402
from gen_golden import _np, save  # noqa: E402
from gen_golden_lineage import load_cm_depth_net, load_necks  # noqa: E402


def lidar_like_gt(B, N, H, W, lo, hi, gen):
    """Sparse depth map: ~6 % of the pixels carry a return, a few of them out
    of [lo, hi), one image row block with none at all, and some exact bin
    edges."""
    gt = torch.zeros(B, N, H, W)
    hit = torch.rand(B, N, H, W, generator=gen) < 0.06
    val = torch.rand(B, N, H, W, generator=gen) * (hi - lo + 12.0) + lo - 4.0
    gt[hit] = val[hit]
    flat = gt.view(-1)
    idx = torch.randperm(flat.numel(), generator=gen)[:24]
    edges = torch.tensor([lo, hi, lo + 0.5, hi - 0.5, lo - 0.5, 0.25] * 4)
    flat[idx] = edges
    gt[0, 0, :H // 4] = 0.0
    return gt


def run_case(cls, self_ns, gt, preds, returns_dict):
    self_ns.get_downsampled_gt_depth = types.MethodType(
        cls.get_downsampled_gt_depth, self_ns)
    onehot = cls.get_downsampled_gt_depth(self_ns, gt)
    p = preds.clone().requires_grad_()
    out = cls.get_depth_loss(self_ns, gt, p)
    loss = out['loss_depth'] if returns_dict else out
    loss.backward()
    has = onehot.max(1).values > 0
    labels = torch.where(has, onehot.argmax(1) + 1, torch.zeros_like(has,
                                                                      dtype=torch.long))
    return dict(gt=_np(gt), preds=_np(preds), onehot=_np(onehot).astype(np.uint8),
                labels=_np(labels).astype(np.int32), loss=_np(loss),
                grad=_np(p.grad), n_fg=np.array(int(has.sum())))


def gen_depth_loss():
    ref_import.install_stubs()
    cm = load_cm_depth_net()
    cm['autocast'] = torch.cuda.amp.autocast_mode.autocast
    CM = cm['CM_DepthNet']
    LSS = load_necks().LSSViewTransformerBEVDepth
    arrays = {}

    def add(case, cfg, ds, D, B, N, H, W, seed, lineage=False):
        g = torch.Generator().manual_seed(seed)
        lo, hi, step = cfg
        gt = lidar_like_gt(B, N, H, W, lo, hi, g)
        h, w = H // ds, W // ds
        logits = torch.randn(B * N, D, h, w, generator=g) * 3.0
        preds = logits.softmax(1)
        grid = dict(depth=list(cfg))
        if lineage:
            self_ns = types.SimpleNamespace(downsample=ds, grid_config=grid,
                                            D=D, loss_depth_weight=3.0)
            res = run_case(LSS, self_ns, gt, preds, False)
        else:
            self_ns = types.SimpleNamespace(downsample=ds, grid_config=grid,
                                            depth_channels=D, D=D, sid=False,
                                            loss_depth_weight=3.0)
            res = run_case(CM, self_ns, gt, preds.view(B, N, D, h, w), True)
        res.update(depth_cfg=np.array(cfg, np.float64), downsample=np.array(ds),
                   D=np.array(D), B=np.array(B), N=np.array(N),
                   loss_weight=np.array(3.0))
        for k, v in res.items():
            arrays[f'{case}/{k}'] = v
        print(case, 'n_fg', int(res['n_fg']), 'of', B * N * h * w,
              'loss', float(res['loss']))

    add('fbocc', (2.0, 42.0, 0.5), 16, 80, 1, 3, 64, 176, 71)
    add('lineage', (1.0, 60.0, 1.0), 16, 59, 2, 2, 64, 128, 72, lineage=True)
    add('ds8', (2.0, 42.0, 0.5), 8, 80, 1, 2, 48, 96, 73)
    save('d_depth_loss', **arrays)


if __name__ == "__main__":
    gen_depth_loss()
