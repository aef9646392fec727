"""CPU test of ``oracle.gpu_ref.eager_reference_mode``: it routes the backward
projection's Linears to nn.Linear by swapping ``_fused_linear_on`` for the
duration of the block, and restores the module's routes on the way out."""
import pytest
import torch

from oracle import gpu_ref


def test_reference_mode_swaps_and_restores_routes():
    from fbbev_b200.view_transformation import backward_projection as bp
    names = ('_fused_linear_on', 'ms_deform_attn_fused',
             'da_spatial_cross_attention_core')
    before = {n: getattr(bp, n) for n in names}
    x = torch.zeros(4, 8)

    with gpu_ref.eager_reference_mode():
        assert bp._fused_linear_on is not before['_fused_linear_on']
        assert bp._fused_linear_on(x, torch.nn.Dropout(0.)) is False
        assert bp.ms_deform_attn_fused is gpu_ref.msda_fused_eager
    assert {n: getattr(bp, n) for n in names} == before

    with pytest.raises(RuntimeError, match='inside'):
        with gpu_ref.eager_reference_mode():
            assert bp._fused_linear_on is not before['_fused_linear_on']
            raise RuntimeError('inside')
    assert {n: getattr(bp, n) for n in names} == before
