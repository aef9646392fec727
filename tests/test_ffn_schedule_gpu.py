"""The fused FFN kernel (fbbev_ffn_fwd) on the row counts where its work
split changes: 64-row units handed out per CTA, a CTA's last step holding one
warpgroup's unit only, 132-SM waves and more units than CTAs.

Per (M, E, hidden): the float64 bar of tests/test_linear_gpu.py (3e-5) without
a residual, with the residual being x itself and with another tensor; bitwise
repeatability; and row slices, computed alone, equal to the same rows of the
full call bit for bit, so a row's result does not depend on which warpgroup or
CTA computed it.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROWS = [1, 63, 64, 65, 127, 129, 132 * 128 - 64, 132 * 128 + 64, 625 * 64, 40000,
        2 * 132 * 128 + 37]


def _ref(hid64, w2, b2, residual, ln):
    y = F.linear(hid64, w2.double(), b2.double())
    if residual is not None:
        y = y + residual.double()
    return F.layer_norm(y, (w2.shape[0],), ln[0].double(), ln[1].double(), 1e-5)


@pytest.mark.parametrize("h", [80, 160, 320])
@pytest.mark.parametrize("e", [16, 48, 80])
@pytest.mark.parametrize("m", ROWS)
def test_ffn_rows_residuals_and_slices(m, e, h):
    from fbbev_b200.ops.linear import ffn_fused
    g = torch.Generator(device="cuda").manual_seed(m * 7 + e * 3 + h)
    x = torch.randn(m, e, device="cuda", generator=g)
    other = torch.randn(m, e, device="cuda", generator=g)
    w1 = torch.randn(h, e, device="cuda", generator=g) / e ** 0.5
    w2 = torch.randn(e, h, device="cuda", generator=g) / h ** 0.5
    b1 = torch.randn(h, device="cuda", generator=g)
    b2 = torch.randn(e, device="cuda", generator=g)
    ln = (torch.rand(e, device="cuda", generator=g) + 0.5,
          torch.randn(e, device="cuda", generator=g))

    def ffn(rows, residual):
        return ffn_fused(rows, w1, b1, w2, b2, residual=residual, ln_weight=ln[0],
                         ln_bias=ln[1], eps=1e-5)

    with torch.no_grad():
        y_none = ffn(x, None)
        y_self = ffn(x, x)
        y_other = ffn(x, other)
        assert torch.equal(y_self, ffn(x, x))
        cuts = sorted({0, min(1, m), min(63, m), m // 2, max(0, m - 65), m})
        parts = [(a, b, ffn(x[a:b], x[a:b])) for a, b in zip(cuts, cuts[1:])]
    hid64 = F.linear(x.double(), w1.double(), b1.double()).relu()
    for residual, y in ((None, y_none), (x, y_self), (other, y_other)):
        err = (y.double() - _ref(hid64, w2, b2, residual, ln)).abs().max().item()
        assert err < 3e-5, err
    for a, b, part in parts:
        assert torch.equal(part, y_self[a:b]), (a, b)
