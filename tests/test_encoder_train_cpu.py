"""CPU tests of the encoder layer's training route on the fused kernels
(``fbbev_linear_fwd_ln_train``, ``fbbev_ffn_fwd_train``, ``fbbev_ffn_bwd``,
``fbbev_layernorm_bwd``):

- the decompositions the kernels compute, in float64 against torch autograd:
  the FFN's data-path backward as the forward's form with the weights
  transposed and swapped and the ReLU mask taken from ``act``, and the
  LayerNorm backward from the saved x^ and 1 / sigma;
- argument validation of every new entry point (no GPU needed: errors are
  returned before anything is enqueued);
- ptxas resources of the new kernel instantiations."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "build", "csrc")
INVALID, UNSUPPORTED = -1, -3
THREADS, REGISTER_FILE = 256, 65536


def _ffn_fwd_form(x, wa, wb, mask=None, b1=None):
    """``relu(x @ wa.T + b1) @ wb.T`` -- or, with ``mask``, the hidden
    pre-activation masked instead of ReLU'd: the form ``fbbev_ffn_bwd`` runs
    with wa = W2^T, wb = W1^T.  Returns (hidden, out)."""
    h = x @ wa.t()
    if mask is None:
        h = torch.relu(h + (b1 if b1 is not None else 0))
    else:
        h = h * mask
    return h, h @ wb.t()


@pytest.mark.parametrize("identity", ["x", "other", "none"])
@pytest.mark.parametrize("with_ln", [False, True])
def test_ffn_backward_is_the_swapped_forward(identity, with_ln):
    g = torch.Generator().manual_seed(3)
    m, e, hid = 37, 48, 160
    d = dict(dtype=torch.float64)
    x = torch.randn(m, e, generator=g, **d).requires_grad_()
    w1 = (torch.randn(hid, e, generator=g, **d) / e ** 0.5).requires_grad_()
    b1 = (0.1 * torch.randn(hid, generator=g, **d)).requires_grad_()
    w2 = (torch.randn(e, hid, generator=g, **d) / hid ** 0.5).requires_grad_()
    b2 = (0.1 * torch.randn(e, generator=g, **d)).requires_grad_()
    other = torch.randn(m, e, generator=g, **d).requires_grad_()
    gam = (1 + 0.1 * torch.randn(e, generator=g, **d)).requires_grad_()
    bet = (0.1 * torch.randn(e, generator=g, **d)).requires_grad_()
    gy = torch.randn(m, e, generator=g, **d)

    act, out = _ffn_fwd_form(x, w1, w2, b1=b1)
    s = out + b2 + {"x": x, "other": other, "none": 0}[identity]
    y = torch.nn.functional.layer_norm(s, (e,), gam, bet, 1e-5) if with_ln else s
    leaves = [x, w1, b1, w2, b2, other, gam, bet]
    grads = torch.autograd.grad(y, leaves, gy, allow_unused=True)
    ref = dict(zip(["x", "w1", "b1", "w2", "b2", "other", "gam", "bet"], grads))

    with torch.no_grad():
        act = act.detach()
        if with_ln:
            mu = s.mean(-1, keepdim=True)
            rstd = (s.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
            xhat = (s - mu) * rstd
            gg = gam * gy
            dz = rstd * (gg - gg.mean(-1, keepdim=True) -
                         xhat * (gg * xhat).mean(-1, keepdim=True))
            torch.testing.assert_close(ref["gam"], (gy * xhat).sum(0))
            torch.testing.assert_close(ref["bet"], gy.sum(0))
        else:
            dz = gy
        # GEMM1': dz @ (W2^T)^T masked by act > 0; GEMM2': dh @ (W1^T)^T
        dh, dx = _ffn_fwd_form(dz, w2.t(), w1.t(), mask=(act > 0).double())
        if identity == "x":
            dx = dx + dz
        torch.testing.assert_close(ref["x"], dx)
        torch.testing.assert_close(ref["w1"], dh.t() @ x)
        torch.testing.assert_close(ref["b1"], dh.sum(0))
        torch.testing.assert_close(ref["w2"], dz.t() @ act)
        torch.testing.assert_close(ref["b2"], dz.sum(0))
        if identity == "other":
            torch.testing.assert_close(ref["other"], dz)


def test_linear_layernorm_backward_decomposition():
    """dz from x^ / 1 / sigma; dx = dz @ W as a forward Linear of W^T;
    dresidual = dz."""
    g = torch.Generator().manual_seed(5)
    m, k, n = 29, 80, 80
    d = dict(dtype=torch.float64)
    x = torch.randn(m, k, generator=g, **d).requires_grad_()
    w = torch.randn(n, k, generator=g, **d).requires_grad_()
    b = torch.randn(n, generator=g, **d).requires_grad_()
    r = torch.randn(m, n, generator=g, **d).requires_grad_()
    gam = torch.randn(n, generator=g, **d).requires_grad_()
    bet = torch.randn(n, generator=g, **d).requires_grad_()
    gy = torch.randn(m, n, generator=g, **d)
    s = x @ w.t() + b + r
    y = torch.nn.functional.layer_norm(s, (n,), gam, bet, 1e-5)
    gx, gw, gb, gr, ggam, gbet = torch.autograd.grad(y, [x, w, b, r, gam, bet], gy)
    with torch.no_grad():
        rstd = (s.var(-1, unbiased=False, keepdim=True) + 1e-5).rsqrt()
        xhat = (s - s.mean(-1, keepdim=True)) * rstd
        gg = gam * gy
        dz = rstd * (gg - gg.mean(-1, keepdim=True) -
                     xhat * (gg * xhat).mean(-1, keepdim=True))
        torch.testing.assert_close(gx, dz @ w.t().t())
        torch.testing.assert_close(gw, dz.t() @ x)
        torch.testing.assert_close(gb, dz.sum(0))
        torch.testing.assert_close(gr, dz)
        torch.testing.assert_close(ggam, (gy * xhat).sum(0))
        torch.testing.assert_close(gbet, gy.sum(0))


def _lib():
    from fbbev_b200 import _lib
    return _lib.lib()


def _p(i):
    """A fake, 16-byte aligned device address: never dereferenced, because
    every call below is refused before anything is enqueued."""
    return ctypes.c_void_p(4096 * i)


def test_linear_ln_train_argument_validation():
    L = _lib()
    f = L.fbbev_linear_fwd_ln_train
    ok = [_p(1), 80, _p(2), None, None, 0, _p(3), _p(4), 100, 80, 80, 1e-5,
          _p(5), 80, _p(6), _p(7), None]

    def call(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return f(*a)
    assert call(a6=None, a7=None) == INVALID          # the LayerNorm is required
    assert call(a14=None) == INVALID                  # xhat
    assert call(a15=None) == INVALID                  # rstd
    assert call(a0=None) == INVALID
    assert call(a12=None) == INVALID                  # y
    assert call(a14=ctypes.c_void_p(4096 + 4)) == INVALID  # xhat misaligned
    assert call(a10=96) == UNSUPPORTED                # n > 80
    assert call(a9=82, a1=84) == UNSUPPORTED          # k % 4
    assert call(a8=-1) == INVALID
    assert call(a8=0) == 0                            # empty: no-op


def test_ffn_train_argument_validation():
    L = _lib()
    f = L.fbbev_ffn_fwd_train
    ok = [_p(1), 80, _p(2), None, _p(3), None, None, 0, _p(4), _p(5), 100, 80,
          320, 1e-5, _p(6), 80, _p(7), _p(8), _p(9), None]

    def call(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return f(*a)
    assert call(a16=None) == INVALID                  # act
    assert call(a17=None) == INVALID                  # xhat with the LayerNorm
    assert call(a18=None) == INVALID                  # rstd with the LayerNorm
    assert call(a8=None) == INVALID                   # ln_weight without ln_bias
    assert call(a16=ctypes.c_void_p(4096 + 8)) == INVALID
    assert call(a12=400) == UNSUPPORTED               # hidden > 320
    assert call(a11=256, a12=1024, a1=256, a15=256) == UNSUPPORTED
    assert call(a11=84, a1=84, a15=84) == UNSUPPORTED  # embed > 80
    assert call(a10=0) == 0
    # no LayerNorm: xhat / rstd are not needed
    assert call(a8=None, a9=None, a17=None, a18=None, a10=0) == 0

    b = L.fbbev_ffn_bwd
    okb = [_p(1), 80, _p(2), _p(3), _p(4), 1, 100, 80, 320, _p(5), _p(6), 80, None]

    def callb(**kw):
        a = list(okb)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return b(*a)
    assert callb(a2=None) == INVALID                  # act
    assert callb(a9=None) == INVALID                  # dh
    assert callb(a10=None) == INVALID                 # dx
    assert callb(a3=None) == INVALID                  # W2^T pack
    assert callb(a1=78) == INVALID                    # lddz < embed
    assert callb(a11=82) == INVALID                   # lddx % 4
    assert callb(a9=ctypes.c_void_p(4096 + 4)) == INVALID
    assert callb(a8=240 + 40) == UNSUPPORTED          # hidden % 80
    assert callb(a6=-1) == INVALID
    assert callb(a6=0) == 0


def test_layernorm_bwd_argument_validation():
    L = _lib()
    ws = L.fbbev_layernorm_bwd_workspace_bytes
    assert ws(40000, 80) >= 2 * 80 * 4
    assert ws(0, 80) > 0                  # the column sums still run
    assert ws(10, 81) == 0 and ws(10, 0) == 0 and ws(-1, 8) == 0
    assert ws(10 ** 8, 80) == ws(10 ** 7, 80)   # the partial count is bounded
    f = L.fbbev_layernorm_bwd
    need = ws(100, 80)
    ok = [_p(1), 80, _p(2), _p(3), _p(4), 100, 80, _p(5), 80, _p(6), _p(7),
          _p(8), need, None]

    def call(**kw):
        a = list(ok)
        for i, v in kw.items():
            a[int(i[1:])] = v
        return f(*a)
    for i in (0, 2, 3, 4, 7, 9, 10, 11):
        assert call(**{f"a{i}": None}) == INVALID, i
    assert call(a12=need - 1) == INVALID              # workspace too small
    assert call(a1=79) == INVALID                     # ldg < n
    assert call(a8=79) == INVALID                     # lddz < n
    assert call(a6=96, a1=96, a8=96) == UNSUPPORTED   # n > 80
    assert call(a5=-1) == INVALID


def _entries(name):
    log = os.path.join(BUILD, f"{name}.ptxas.log")
    if not os.path.exists(log):
        pytest.skip(f"ptxas log not built: {log}")
    text = open(log).read()
    entries, fn = {}, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and fn:
            entries.setdefault(fn, {})["spill"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m and fn:
            entries.setdefault(fn, {})["regs"] = int(m.group(1))
    return text, entries


def _check(text, entries, names):
    for fn in names:
        e = entries[fn]
        assert e["spill"] == (0, 0), (fn, e)
        assert e["regs"] * THREADS <= REGISTER_FILE, (fn, e)
        bad = [l for l in text.splitlines() if fn in l and
               ("serialized" in l or re.search(r"\(C75(1\d|20)\)", l))]
        assert not bad, "\n".join(bad)


def test_ffn_training_instantiations():
    """kTrainFwd (1) and kBwd (2) for every (pad16(E), K-blocks) the
    inference kernel has."""
    from test_ffn_ptxas import ffn_instantiations
    text, entries = _entries("ffn_tf32")
    want = {t for t in ffn_instantiations() if t[2] > 0}
    found = {}
    for fn in entries:
        m = re.search(r"ffn_tf32_kernelILi(\d+)ELi(\d+)ELi(\d+)E", fn)
        if m and int(m.group(3)) > 0:
            found[tuple(int(v) for v in m.groups())] = fn
    assert set(found) == want, set(found) ^ want
    _check(text, entries, found.values())


def test_linear_stats_and_layernorm_bwd_instantiations():
    text, entries = _entries("linear_tf32")
    found = {}
    for fn in entries:
        m = re.search(r"(linear_tf32_kernel(?:_resident)?)ILi(\d+)ELb1ELb1E", fn)
        if m:
            found[(m.group(1), int(m.group(2)))] = fn
    want = {(k, n) for k in ("linear_tf32_kernel", "linear_tf32_kernel_resident")
            for n in (16, 32, 48, 64, 80)}
    assert set(found) == want, set(found) ^ want
    _check(text, entries, found.values())
    text, entries = _entries("layernorm_bwd")
    names = [fn for fn in entries if "layernorm_bwd" in fn]
    assert len(names) == 2, names
    _check(text, entries, names)
