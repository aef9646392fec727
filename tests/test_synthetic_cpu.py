"""The seeded synthetic inputs are the same tensors whatever the host's torch
thread count: the goldens recorded from them (r_ref_cuda.npz) and the
benchmark's output dumps compare bit for bit only if they are."""
import pytest
import torch


@pytest.mark.parametrize("shape", [(1, 6, 80, 16, 44), (1, 1, 59, 64, 176),
                                   (1, 6, 118, 32, 88)])
def test_depth_does_not_depend_on_thread_count(shape):
    from fbbev_b200 import synthetic
    before = torch.get_num_threads()
    got = []
    try:
        for k in (1, 3, 8, 16, 32, 64):
            torch.set_num_threads(k)
            depth, feat = synthetic.make_depth_feat(*shape, C=4)
            assert torch.get_num_threads() == k     # restored
            got.append((depth, feat))
    finally:
        torch.set_num_threads(before)
    for depth, feat in got[1:]:
        assert torch.equal(depth, got[0][0])
        assert torch.equal(feat, got[0][1])
