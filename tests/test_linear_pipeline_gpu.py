"""Edges of the wgmma Linear pipeline (fbbev_linear_fwd / _split, fbbev_ffn_fwd)
against torch in float64, at the bars of tests/test_linear_gpu.py.

Row counts sit on 64-row tile, 132-SM wave and ring-wrap boundaries; K = 80
runs the resident-weight kernel and K = 256 the streamed one.  Also: strided
row pitches of every operand, the two-output split, row-split invariance and
run-to-run bit equality.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROWS = [1, 63, 64, 65, 127, 129, 132 * 64 - 1, 132 * 64 + 1, 40000, 200000]


def _data(m, k, n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(m, k, device="cuda", generator=g)
    w = torch.randn(n, k, device="cuda", generator=g) / k ** 0.5
    b = torch.randn(n, device="cuda", generator=g)
    return g, x, w, b


def _call(x, w, b, *, residual=None, ln=None, relu=False, y=None, x_add=None,
          y2=None, n_split=None):
    """One fbbev_linear_fwd / fbbev_linear_fwd_split call on arbitrary row
    pitches (every operand a row-strided view)."""
    from fbbev_b200 import _lib
    from fbbev_b200.ops.linear import _pack
    L = _lib.lib()
    (_, _, buf), = _pack(w)
    m, k = x.shape
    n = w.shape[0]
    sp = _lib.stream_ptr(x.device)
    if x_add is not None or y2 is not None:
        ns = n if n_split is None else n_split
        rc = L.fbbev_linear_fwd_split(
            _lib.ptr(x), x.stride(0), _lib.ptr(x_add),
            x_add.stride(0) if x_add is not None else 0, _lib.ptr(buf), _lib.ptr(b),
            m, k, n, ns, int(relu), _lib.ptr(y), y.stride(0), _lib.ptr(y2),
            y2.stride(0) if y2 is not None else 0, sp)
        _lib.check(rc, "fbbev_linear_fwd_split")
    else:
        rc = L.fbbev_linear_fwd(
            _lib.ptr(x), x.stride(0), _lib.ptr(buf), _lib.ptr(b), _lib.ptr(residual),
            residual.stride(0) if residual is not None else 0,
            _lib.ptr(ln[0]) if ln else None, _lib.ptr(ln[1]) if ln else None,
            m, k, n, int(relu), 1e-5, _lib.ptr(y), y.stride(0), sp)
        _lib.check(rc, "fbbev_linear_fwd")


def _ref(x, w, b, residual=None, ln=None, relu=False):
    y = F.linear(x.double(), w.double(), b.double())
    if relu:
        y = y.relu()
    if residual is not None:
        y = y + residual.double()
    if ln is not None:
        y = F.layer_norm(y, (w.shape[0],), ln[0].double(), ln[1].double(), 1e-5)
    return y


@pytest.mark.parametrize("k", [80, 256])
@pytest.mark.parametrize("m", ROWS)
def test_rows_on_tile_wave_and_ring_edges(m, k):
    n = 192
    _, x, w, b = _data(m, k, n, m + k)
    y = torch.full((m, n), float("nan"), device="cuda")
    with torch.no_grad():
        _call(x, w, b, y=y, relu=True)
    err = (y.double() - _ref(x, w, b, relu=True)).abs().max().item()
    assert err < 2e-5, err


@pytest.mark.parametrize("m,k", [(40000, 80), (4097, 44), (1000, 256)])
def test_strided_rows_residual_layernorm(m, k):
    n = 80
    g, x, w, b = _data(m, k, n, 7 + m)
    xs = torch.randn(m, k + 12, device="cuda", generator=g)[:, 4:4 + k]
    xs.copy_(x)
    r = torch.randn(m, n + 20, device="cuda", generator=g)[:, 8:8 + n]
    ln = (torch.rand(n, device="cuda", generator=g) + 0.5,
          torch.randn(n, device="cuda", generator=g))
    yb = torch.full((m, n + 36), 7.0, device="cuda")
    y = yb[:, 16:16 + n]
    with torch.no_grad():
        _call(xs, w, b, residual=r, ln=ln, y=y)
    err = (y.double() - _ref(x, w, b, residual=r, ln=ln)).abs().max().item()
    assert err < 2e-5, err
    assert (yb[:, :16] == 7.0).all() and (yb[:, 16 + n:] == 7.0).all()


@pytest.mark.parametrize("m,k", [(40000, 80), (129, 80), (1000, 256)])
def test_strided_x_add_and_two_outputs(m, k):
    na, nb = 128, 64
    g, x, w, b = _data(m, k, na + nb, 11 + m)
    xa = torch.randn(m, k + 8, device="cuda", generator=g)[:, 4:4 + k]
    ya = torch.full((m, na + 4), 3.0, device="cuda")
    yb = torch.full((m, nb + 12), 3.0, device="cuda")
    with torch.no_grad():
        _call(x, w, b, x_add=xa, y=ya[:, :na], y2=yb[:, 4:4 + nb], n_split=na)
        want = _ref(x + xa, w, b)
        ya0 = torch.empty(m, na, device="cuda")
        yb0 = torch.empty(m, nb, device="cuda")
        _call(x + xa, w, b, y=ya0, y2=yb0, n_split=na)
    assert (ya[:, :na].double() - want[:, :na]).abs().max().item() < 2e-5
    assert (yb[:, 4:4 + nb].double() - want[:, na:]).abs().max().item() < 2e-5
    # x + x_add is one fp32 add in the loader: the same bits as adding first
    assert torch.equal(ya[:, :na], ya0) and torch.equal(yb[:, 4:4 + nb], yb0)
    assert (ya[:, na:] == 3.0).all() and (yb[:, :4] == 3.0).all()


@pytest.mark.parametrize("k", [80, 256])
def test_row_split_invariance_and_repeatability(k):
    m, n = 20000, 96
    g, x, w, b = _data(m, k, n, 5 + k)
    r = torch.randn(m, n, device="cuda", generator=g)
    with torch.no_grad():
        y = torch.empty(m, n, device="cuda")
        _call(x, w, b, residual=r, y=y)
        y_again = torch.empty(m, n, device="cuda")
        _call(x, w, b, residual=r, y=y_again)
        assert torch.equal(y, y_again)
        for a, e in ((0, 1), (63, 64), (65, 8513), (8513, m)):
            part = torch.empty(e - a, n, device="cuda")
            _call(x[a:e], w, b, residual=r[a:e], y=part)
            assert torch.equal(part, y[a:e]), (a, e)


@pytest.mark.parametrize("h", [80, 160, 320])
@pytest.mark.parametrize("e", [16, 48, 80])
def test_ffn_widths(e, h):
    from fbbev_b200.ops.linear import ffn_fused
    m = 132 * 128 + 37
    g = torch.Generator(device="cuda").manual_seed(e * h)
    x = torch.randn(m, e, device="cuda", generator=g)
    w1 = torch.randn(h, e, device="cuda", generator=g) / e ** 0.5
    w2 = torch.randn(e, h, device="cuda", generator=g) / h ** 0.5
    b1 = torch.randn(h, device="cuda", generator=g)
    b2 = torch.randn(e, device="cuda", generator=g)
    ln = (torch.rand(e, device="cuda", generator=g) + 0.5,
          torch.randn(e, device="cuda", generator=g))
    with torch.no_grad():
        y = ffn_fused(x, w1, b1, w2, b2, residual=x, ln_weight=ln[0], ln_bias=ln[1])
        y_again = ffn_fused(x, w1, b1, w2, b2, residual=x, ln_weight=ln[0],
                            ln_bias=ln[1])
    hid = F.linear(x.double(), w1.double(), b1.double()).relu()
    ref = _ref(hid, w2, b2, residual=x, ln=ln)
    assert (y.double() - ref).abs().max().item() < 3e-5
    assert torch.equal(y, y_again)
