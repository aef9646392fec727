"""CPU tests of the two fused attention backward entry points of the C ABI:
argument errors are reported before anything is enqueued, an empty problem is
a no-op."""


def test_fused_backward_argument_validation_without_gpu():
    from fbbev_b200 import _lib
    L = _lib.lib()
    # fbbev_msda_fused_bwd: 7 inputs, bs n_value heads ch levels nq points,
    # grad_value grad_offsets grad_logits stream
    assert L.fbbev_msda_fused_bwd(*([None] * 7), 1, 10, 8, 10, 1, 5, 4,
                                  None, None, None, None) == -1  # NULL inputs
    assert L.fbbev_msda_fused_bwd(*([None] * 7), 0, 10, 8, 10, 1, 5, 4,
                                  None, None, None, None) == 0   # empty: no-op
    assert L.fbbev_msda_fused_bwd(*([None] * 7), 1, 10, 8, 10, 0, 5, 4,
                                  None, None, None, None) == -1  # no levels
    dbound = _lib.c_floats([2.0, 42.0, 0.5])
    # fbbev_da_sca_bwd: 9 inputs, dbound, grad_out, bs n_cams nq n_value heads
    # ch levels points Z DC, 4 gradients, stream
    def da(bs, points, Z, db=dbound):
        return L.fbbev_da_sca_bwd(*([None] * 9), db, None, bs, 6, 10, 10, 8,
                                  10, 1, points, Z, 80, *([None] * 5))
    assert da(1, 8, 4) == -1            # NULL inputs
    assert da(1, 7, 4) == -1            # points % Z != 0
    assert da(1, 8, 4, None) == -1      # no dbound
    assert da(0, 8, 4) == 0             # empty: no-op
    assert da(0, 7, 4) == -1            # checked before the empty test


def test_python_lists_match_library_without_gpu():
    """FUSED_HEAD_WIDTHS / FUSED_Z_ANCHORS (what fused_grad_supported()
    accepts) are exactly the head widths and Z counts the library's fused
    kernels are built for: the _det entry points report FBBEV_ERR_UNSUPPORTED
    (-3) for any other before their empty-problem test."""
    from fbbev_b200 import _lib
    from fbbev_b200.ops.ms_deform_attn import (FUSED_HEAD_WIDTHS,
                                               FUSED_Z_ANCHORS)
    L = _lib.lib()
    for ch in range(1, 129):
        # fbbev_msda_fused_bwd_det: 7 inputs, bs n_value heads ch levels nq
        # points, 3 gradients, workspace, bytes, stream
        rc = L.fbbev_msda_fused_bwd_det(*([None] * 7), 0, 10, 8, ch, 1, 5, 4,
                                        None, None, None, None, 0, None)
        assert rc == (0 if ch in FUSED_HEAD_WIDTHS else -3), (ch, rc)
    dbound = _lib.c_floats([2.0, 42.0, 0.5])
    for Z in range(1, 17):
        # fbbev_da_sca_bwd_det: 9 inputs, dbound, grad_out, bs n_cams nq
        # n_value heads ch levels points Z DC, 4 gradients, workspace, bytes,
        # stream
        rc = L.fbbev_da_sca_bwd_det(*([None] * 9), dbound, None, 0, 6, 10, 10,
                                    8, 10, 1, 2 * Z, Z, 80, *([None] * 5), 0,
                                    None)
        assert rc == (0 if Z in FUSED_Z_ANCHORS else -3), (Z, rc)
