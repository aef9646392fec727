"""Seeded synthetic inputs for the view-transformation hot path.

There is no dataset in this environment, so tests and ``bench.py`` drive the
path with a nuScenes-like 6-camera rig built here.  The camera order, the
test-time image augmentation and the tensor layouts follow the reference's
data pipeline so the tensors have the shapes and value ranges the plugin sees
in FB-OCC:

* camera order  ``CAM_FRONT_LEFT, CAM_FRONT, CAM_FRONT_RIGHT, CAM_BACK_LEFT,
  CAM_BACK, CAM_BACK_RIGHT`` -- occupancy_configs/fb_occ/
  fbocc-r50-cbgs_depth_16f_16x4_20e.py:50-53
* test-time ``post_rot = diag(W_in/1600)``, ``post_tran = (0, -crop_h)`` --
  mmdet3d/datasets/pipelines/loading.py:1076-1087 (``sample_augmentation``)
* ``cam_params = (rots, trans, intrins, post_rots, post_trans, bda)`` --
  mmdet3d/datasets/pipelines/loading.py:1308, 1391-1394

Everything here is plain PyTorch on the requested device; nothing imports the
oracle.
"""
import math

import torch

# nuScenes-like yaw (deg, ego frame x-forward / y-left / z-up) and mounting
# position (m) per camera, in the reference's camera order.
_CAM_YAW_DEG = (55.0, 0.0, -55.0, 110.0, 180.0, -110.0)
_CAM_POS = ((1.5, 0.5, 1.5), (1.7, 0.0, 1.5), (1.5, -0.5, 1.5),
            (1.0, 0.5, 1.5), (0.0, 0.0, 1.5), (1.0, -0.5, 1.5))
_FOCAL = (1266.0, 1266.0, 1266.0, 1266.0, 809.0, 1266.0)

# The named grids of BASELINE.json:configs / SURVEY.md section 8(d).
GRID_CONFIGS = {
    # shipped FB-OCC R50 lift-splat grid (fbocc-r50 config :78-84)
    "fbocc_shipped": dict(x=[-40, 40, 0.8], y=[-40, 40, 0.8],
                          z=[-1, 5.4, 0.8], depth=[2.0, 42.0, 0.5]),
    # configs[1]: 200x200x16 voxel grid, same cameras / depth bins
    "fbocc_200": dict(x=[-40, 40, 0.4], y=[-40, 40, 0.4], z=[-1, 5.4, 0.4],
                      depth=[2.0, 42.0, 0.5]),
    # configs[0]: 1-cam 64x176 feature map, D=59, 128x128x1 BEV
    "unit_128": dict(x=[-51.2, 51.2, 0.8], y=[-51.2, 51.2, 0.8],
                     z=[-5, 3, 8], depth=[1.0, 60.0, 1.0]),
    # configs[4]: 400x400x32, D=118
    "fbocc_400": dict(x=[-40, 40, 0.2], y=[-40, 40, 0.2], z=[-1, 5.4, 0.2],
                      depth=[1.0, 60.0, 0.5]),
}


def make_cam_params(batch=1, n_cams=6, input_size=(256, 704),
                    src_size=(900, 1600), device="cpu", jitter=0.0, seed=0):
    """Build ``(rots, trans, intrins, post_rots, post_trans, bda)``.

    ``jitter`` > 0 perturbs yaw / position per sample so batched frames differ
    (each frame is an independent sample, as in the reference's batch dim).
    """
    g = torch.Generator().manual_seed(seed)
    H_in, W_in = input_size
    H_src, W_src = src_size
    rots = torch.zeros(batch, n_cams, 3, 3)
    trans = torch.zeros(batch, n_cams, 3)
    intr = torch.zeros(batch, n_cams, 3, 3)
    post_rots = torch.zeros(batch, n_cams, 3, 3)
    post_trans = torch.zeros(batch, n_cams, 3)
    resize = float(W_in) / float(W_src)
    new_h = int(H_src * resize)
    crop_h = new_h - H_in
    for b in range(batch):
        for n in range(n_cams):
            k = n % 6
            yaw = math.radians(_CAM_YAW_DEG[k])
            pos = torch.tensor(_CAM_POS[k])
            if jitter > 0:
                yaw += float(torch.randn((), generator=g)) * jitter * 0.05
                pos = pos + torch.randn(3, generator=g) * jitter * 0.1
            s, c = math.sin(yaw), math.cos(yaw)
            # cam->ego: columns are the camera's right / down / forward axes
            rots[b, n] = torch.tensor([[s, 0.0, c], [-c, 0.0, s],
                                       [0.0, -1.0, 0.0]])
            trans[b, n] = pos
            f = _FOCAL[k]
            intr[b, n] = torch.tensor([[f, 0.0, 816.0], [0.0, f, 491.0],
                                       [0.0, 0.0, 1.0]])
            post_rots[b, n] = torch.diag(torch.tensor([resize, resize, 1.0]))
            post_trans[b, n] = torch.tensor([0.0, -float(crop_h), 0.0])
    bda = torch.eye(3).repeat(batch, 1, 1)
    return tuple(t.to(device) for t in
                 (rots, trans, intr, post_rots, post_trans, bda))


# torch's CPU softmax over a dim that is not the innermost one splits the
# inner extent across the intra-op threads, and the vectorised exp rounds
# differently from the scalar loop that finishes each chunk: the same seed gives
# other last bits on a host with another thread count.  The depth maps are
# evaluated with this fixed count, so a seed means the same tensor on every
# (x86, AVX2 / AVX-512) host; it is the count the committed fixtures built from
# these inputs (tests/golden/r_ref_cuda.npz) were recorded with.
SOFTMAX_THREADS = 16


def make_depth_feat(batch, n_cams, D, H, W, C, device="cpu", seed=0):
    """``depth = softmax(randn)`` over D (B,N,D,H,W) and ``feat = randn``
    (B,N,C,H,W) -- the outputs of CM_DepthNet (modules/depth_net.py:335-366)."""
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(batch, n_cams, D, H, W, generator=g)
    threads = torch.get_num_threads()
    torch.set_num_threads(SOFTMAX_THREADS)
    try:
        depth = logits.softmax(dim=2)
    finally:
        torch.set_num_threads(threads)
    g.manual_seed(seed + 1)
    feat = torch.randn(batch, n_cams, C, H, W, generator=g)
    return depth.to(device), feat.to(device)
