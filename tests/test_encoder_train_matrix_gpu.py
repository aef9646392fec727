"""Every fused FFN kernel instantiation, the LayerNorm backward and the
LayerNorm-epilogue Linear's backward against float64 on the device, at the
widths and row counts where the kernels' work splits change.

- FFN, ``ffn_tf32_kernel<NP2, KB1, MODE>`` (18 instantiations).  E in ``ES``
  reaches every (NP2, KB1) pair and the last column inside and past each
  16-column pad; every E runs with every hidden width at 131 rows.  Two
  (E, hidden) pairs per instantiation also run on the kernel's split edges:
  1 to 129 rows around one and two 64-row units, 2 S 64 - 64, + 37 and + 64
  (S the SM count; the kernel is one CTA per SM, each walking its run of
  64-row units two per step, and these counts leave some CTA an odd run, so
  warpgroup 1 idles on its last step) and 40000.
  * inference (kInfer): ``ffn_fused`` with residual none / x / other,
    LayerNorm on and off, biases on and off;
  * training forward (kTrainFwd): ``fbbev_ffn_fwd_train``'s y bit-equal to
    the inference kernel's, act, x^ and 1 / sigma against float64;
  * backward (kBwd): ``ffn_train``'s gradients of every leaf in modes x+ln,
    other+ln, x and none, with the float64 chain built as in
    test_encoder_train_gpu.py (the ReLU mask is the kernel's act > 0, and it
    may differ from float64's only within fp32 error of zero); and
    ``fbbev_ffn_bwd`` called directly on row-strided dz and dx, with and
    without add_dz, the columns outside each view left untouched.
- ``fbbev_layernorm_bwd`` with one, two and three of a lane's column slots
  live (n <= 32, <= 64, <= 80), below, at and past its 512-CTA cap
  (m = 512 * 64), with ldg > n and lddz > n: dz, dgamma, dbeta, two calls
  bit-identical, m = 0 giving zero sums.
- ``LinearLNTrainFunction``'s gradients at n in 16..80 and k up to 320 (at
  k = 320 the transposed pack behind dx is two column blocks).
- Census: the ``ffn_tf32_kernel`` instantiations torch.profiler saw == the
  dispatch rule's 18 (``test_ffn_ptxas.ffn_instantiations``).

Every tensor passes ``|got - ref|max <= BAR[quantity] * max(1, |ref|max)``.
Each bar is at least 4x the worst error over the whole matrix, measured on an
NVIDIA H100 80GB HBM3 at a 700 W power limit (in BAR's comments).  Every
column sum, the bias and beta sums behind a LayerNorm included, passes the
same max-relative bar with that headroom, so none needs an L1-relative
fallback.  The worst errors are printed with ``-s``."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_encoder_train_gpu import _ffn_train_raw, _lib, _tensors
from test_ffn_ptxas import ffn_instantiations, ffn_kernel_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
INVALID, UNSUPPORTED = -1, -3

# quantity -> bar, after it the worst error measured per entry point; rstd is
# compared relative per row
BAR = {"y": 3e-5,          # ffn 5.0e-6, ffn_train 4.5e-6, linear_ln 3.5e-6
       "act": 1e-5,        # ffn 1.6e-6
       "xhat": 2e-5,       # ffn 4.3e-6
       "rstd": 3e-5,       # ffn 5.0e-6
       "dh": 1e-5,         # ffn_bwd 1.6e-6
       "dx": 2e-5,         # ffn_bwd 4.5e-6, ffn_train 4.4e-6, linear_ln 2.5e-6
       "dw1": 1e-5,        # ffn_train 1.5e-6
       "db1": 1e-5,        # ffn_train 1.6e-6
       "dw2": 1e-5,        # ffn_train 1.6e-6
       "db2": 1e-5,        # ffn_train 2.2e-6
       "dother": 2e-5,     # ffn_train 3.0e-6
       "dgamma": 3e-5,     # ffn_train 5.5e-6, layernorm_bwd 1.5e-6, linear_ln 2.5e-6
       "dbeta": 1e-5,      # ffn_train 9.4e-7, layernorm_bwd 1.3e-6, linear_ln 7.6e-7
       "dz": 1e-6,         # layernorm_bwd 1.8e-7
       "dw": 2e-5,         # linear_ln 3.0e-6
       "db": 1e-5,         # linear_ln 1.8e-6
       "dresidual": 1e-5}  # linear_ln 2.3e-6

WORST = {}                # (entry, quantity) -> largest error
LAUNCHED = {}             # case id -> ffn_tf32_kernel instantiations seen
STATIC = {}               # case id -> instantiations the case must launch


# ---------------- shapes -------------------------------------------------------
ES = (12, 16, 20, 32, 36, 40, 44, 48, 60, 64, 68, 80)
HIDDEN = (80, 160, 240, 320)
SMALL = 131
# (a, b): a * S * 64 + b rows, S the SM count
EDGE_ROWS = (1, 63, 64, 65, 127, 128, 129, (2, -64), (2, 37), (2, 64), 40000)
# two (E, hidden) pairs per (NP2, KB1)
EDGE_PAIRS = ((12, 80), (16, 320), (20, 160), (32, 240), (36, 320), (40, 80),
              (44, 240), (48, 160), (60, 80), (64, 320), (68, 160), (80, 240))
FFN_CASES = ([(e, h, SMALL) for e in ES for h in HIDDEN] +
             [(e, h, r) for e, h in EDGE_PAIRS for r in EDGE_ROWS])


def _rows(r):
    if isinstance(r, tuple):
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        return r[0] * sms * 64 + r[1]
    return r


def _rid(r):
    return f"{r[0]}S64{r[1]:+d}" if isinstance(r, tuple) else str(r)


def _ffn_id(c):
    return f"e{c[0]}-h{c[1]}-m{_rid(c[2])}"


def _kernel(e):
    """(NP2, KB1) of width e by ffn_tf32.cu's dispatch rule."""
    return (e + 15) // 16 * 16, 2 if e > 40 else 1


# ---------------- checks -------------------------------------------------------
def _cmp(entry, qty, got, ref):
    err = (got.double() - ref).abs().max().item() / max(1.0, ref.abs().max().item())
    WORST[(entry, qty)] = max(WORST.get((entry, qty), 0.0), err)
    assert err <= BAR[qty], (entry, qty, err)


def _untouched(buf, cols):
    """The columns of ``buf`` past ``cols`` still hold the NaN they were
    filled with."""
    assert bool(buf[:, cols:].isnan().all())


def _profiled(cid, static, fn):
    """Runs ``fn`` under torch.profiler and records the ffn_tf32_kernel
    instantiations it launched; returns fn's result.  ``static``: the ones
    the case must launch.  The profiler drops a kernel record now and then:
    when one of them is missing, ``fn`` (side-effect free) runs again under a
    fresh profiler, at most twice, and the records are merged."""
    from torch.profiler import ProfilerActivity, profile
    STATIC[cid] = set(static)
    seen, res = set(), None
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            r = fn()
            torch.cuda.synchronize()
        res = r if res is None else res
        seen |= {ffn_kernel_args(ev.name) for ev in prof.events()} - {None}
        if not seen or STATIC[cid] <= seen:
            break
        print(f"[launched] {cid}: not reported by the profiler: "
              f"{sorted(STATIC[cid] - seen)}, run again")
    LAUNCHED[cid] = seen
    return res


def _seed(e, h, m):
    return 7 * m + 3 * e + h


# ---------------- FFN forward: kInfer, kTrainFwd ----------------------------------
FWD_VARIANTS = [(res, ln, bias) for res in ("none", "x", "other")
                for ln in (False, True) for bias in (True, False)]


@pytest.mark.parametrize("e,h,rows", FFN_CASES, ids=[_ffn_id(c) for c in FFN_CASES])
def test_ffn_forward(e, h, rows):
    from fbbev_b200.ops.linear import ffn_fused
    m = _rows(rows)
    t = _tensors(_seed(e, h, m), m, e, h)
    x = t["x"]

    def args(res, ln, bias):
        return (t["b1"] if bias else None, t["b2"] if bias else None,
                {"none": None, "x": x, "other": t["other"]}[res],
                t["ln"] if ln else None)

    def run():
        out = []
        with torch.no_grad():
            for v in FWD_VARIANTS:
                b1, b2, r, ln = args(*v)
                want = ffn_fused(x, t["w1"], b1, t["w2"], b2, residual=r,
                                 ln_weight=ln[0] if ln else None,
                                 ln_bias=ln[1] if ln else None)
                out.append((want,) + _ffn_train_raw(x, t["w1"], b1, t["w2"], b2, r, ln))
        return out

    np2, kb1 = _kernel(e)
    outs = _profiled(f"fwd-{_ffn_id((e, h, rows))}", {(np2, kb1, 0), (np2, kb1, 1)}, run)
    x64, w164, w264 = x.double(), t["w1"].double(), t["w2"].double()
    for v, (want, y, act, xhat, rstd) in zip(FWD_VARIANTS, outs):
        b1, b2, r, ln = args(*v)
        a64 = F.linear(x64, w164, None if b1 is None else b1.double()).relu()
        s = F.linear(a64, w264, None if b2 is None else b2.double())
        if r is not None:
            s = s + r.double()
        assert torch.equal(y, want), v
        _cmp("ffn", "y", want,
             F.layer_norm(s, (e,), ln[0].double(), ln[1].double(), 1e-5) if ln else s)
        _cmp("ffn", "act", act, a64)
        if ln:
            _cmp("ffn", "xhat", xhat, F.layer_norm(s, (e,), None, None, 1e-5))
            ref_r = (s.var(-1, unbiased=False) + 1e-5).rsqrt()
            _cmp("ffn", "rstd", rstd.double() / ref_r, torch.ones_like(ref_r))


# ---------------- FFN backward: kBwd -------------------------------------------------
MODES = ("x+ln", "other+ln", "x", "none")


def _grad_names(mode):
    return (["dx", "dw1", "db1", "dw2", "db2"] + (["dother"] if mode == "other+ln" else [])
            + (["dgamma", "dbeta"] if mode.endswith("ln") else []))


def _ffn_train_grads(t, mode):
    """ffn_train's output and the gradients of every leaf of ``mode``."""
    from fbbev_b200.ops.linear import ffn_train
    e = t["x"].shape[1]
    x, w1, b1, w2, b2 = (t[k].clone().requires_grad_() for k in ("x", "w1", "b1", "w2", "b2"))
    params = [x, w1, b1, w2, b2]
    other = norm = None
    if mode == "other+ln":
        other = t["other"].clone().requires_grad_()
        params.append(other)
    if mode.endswith("ln"):
        norm = nn.LayerNorm(e).to(DEV)
        norm.weight = nn.Parameter(t["ln"][0].clone())
        norm.bias = nn.Parameter(t["ln"][1].clone())
        params += [norm.weight, norm.bias]
    y = ffn_train(x, w1, b1, w2, b2, identity=other, add_identity=mode != "none", norm=norm)
    return y.detach(), torch.autograd.grad(y, params, t["gy"])


def _ffn_ref_grads(t, mode, mask):
    """The same chain in float64 with the hidden activation masked by
    ``mask``: output, hidden pre-activation, leaf gradients in _grad_names
    order."""
    e = t["x"].shape[1]
    p = {k: t[k].double().requires_grad_() for k in ("x", "w1", "b1", "w2", "b2", "other")}
    hid = F.linear(p["x"], p["w1"], p["b1"])
    u = F.linear(hid * mask, p["w2"], p["b2"])
    if mode in ("x+ln", "x"):
        u = u + p["x"]
    if mode == "other+ln":
        u = u + p["other"]
    leaves = [p[k] for k in ("x", "w1", "b1", "w2", "b2")]
    if mode == "other+ln":
        leaves.append(p["other"])
    s = u
    if mode.endswith("ln"):
        lnw, lnb = (v.double().requires_grad_() for v in t["ln"])
        s = F.layer_norm(u, (e,), lnw, lnb, 1e-5)
        leaves += [lnw, lnb]
    refs = torch.autograd.grad(s, leaves, t["gy"].double())
    return s.detach(), hid.detach(), refs


def _ffn_bwd_raw(dz, act, w1, w2, add_dz, dx):
    """fbbev_ffn_bwd on the (possibly row-strided) views dz and dx -> dh."""
    from fbbev_b200.ops import linear as lin
    L = _lib()
    m, e = dz.shape
    hid = w1.shape[0]
    dh = torch.empty(m, hid, device=DEV)
    (_, _, w1tp), = lin._pack(w1, transpose=True)
    L.check(L.lib().fbbev_ffn_bwd(
        L.ptr(dz), dz.stride(0), L.ptr(act), L.ptr(lin._pack_ffn_w1(w2, transpose=True)),
        L.ptr(w1tp), int(add_dz), m, e, hid, L.ptr(dh), L.ptr(dx), dx.stride(0),
        L.stream_ptr(dz.device)), "fbbev_ffn_bwd")
    return dh


@pytest.mark.parametrize("e,h,rows", FFN_CASES, ids=[_ffn_id(c) for c in FFN_CASES])
def test_ffn_backward(e, h, rows):
    m = _rows(rows)
    t = _tensors(_seed(e, h, m) + 1, m, e, h)
    gen = torch.Generator(device=DEV).manual_seed(_seed(e, h, m) + 2)
    # row-strided dz (pitch e + 4) and dx (pitch e + 8), NaN outside the views
    dzbuf = torch.full((m, e + 4), NAN, device=DEV)
    dzbuf[:, :e] = torch.randn(m, e, device=DEV, generator=gen)
    dz0 = dzbuf.clone()

    def run():
        with torch.no_grad():
            _, act, _, _ = _ffn_train_raw(t["x"], t["w1"], t["b1"], t["w2"], t["b2"],
                                          None, None)
        grads = {mode: _ffn_train_grads(t, mode) for mode in MODES}
        direct = []
        for add_dz in (0, 1):
            dxbuf = torch.full((m, e + 8), NAN, device=DEV)
            direct.append((_ffn_bwd_raw(dzbuf[:, :e], act, t["w1"], t["w2"], add_dz,
                                        dxbuf[:, :e]), dxbuf))
        return act, grads, direct

    np2, kb1 = _kernel(e)
    act, grads, direct = _profiled(f"bwd-{_ffn_id((e, h, rows))}",
                                   {(np2, kb1, 1), (np2, kb1, 2)}, run)
    mask = (act > 0).double()
    for mode in MODES:
        y, got = grads[mode]
        s, hid, refs = _ffn_ref_grads(t, mode, mask)
        _cmp("ffn_train", "y", y, s)
        for name, g, r in zip(_grad_names(mode), got, refs):
            _cmp("ffn_train", name, g, r)
    # the kernel's mask differs from float64's only within fp32 error of zero
    bound = 1e-5 * (t["x"].double().abs() @ t["w1"].double().abs().t() +
                    t["b1"].double().abs())
    diff = (hid > 0) != (mask > 0)
    assert bool((hid[diff].abs() <= bound[diff]).all())

    dz64 = dz0[:, :e].double()
    dh64 = (dz64 @ t["w2"].double()) * mask
    for add_dz, (dh, dxbuf) in zip((0, 1), direct):
        _cmp("ffn_bwd", "dh", dh, dh64)
        _cmp("ffn_bwd", "dx", dxbuf[:, :e], dh64 @ t["w1"].double() + add_dz * dz64)
        _untouched(dxbuf, e)
    assert torch.equal(dzbuf[:, :e], dz0[:, :e])
    _untouched(dzbuf, e)


# ---------------- fbbev_layernorm_bwd ------------------------------------------------
LN_N = (4, 16, 28, 32, 36, 48, 64, 68, 76, 80)
LN_M = (0, 1, 63, 64, 65, 32767, 32768, 32769, 40000, 200000)


def _layernorm_bwd_raw(m, g, xhat, rstd, gamma, dz, dgamma, dbeta, ws=None):
    """fbbev_layernorm_bwd over the first m rows of the buffers -> its return
    code.  The buffers keep at least one row, so m = 0 still passes device
    addresses (torch gives an empty tensor a null data_ptr).  ``ws`` defaults
    to a NaN-filled workspace of the size the library asks for."""
    L = _lib()
    n = xhat.shape[1]
    if ws is None:
        nbytes = L.lib().fbbev_layernorm_bwd_workspace_bytes(m, n)
        ws = torch.full((nbytes // 4,), NAN, device=DEV)
    return L.lib().fbbev_layernorm_bwd(
        L.ptr(g), g.stride(0), L.ptr(xhat), L.ptr(rstd), L.ptr(gamma), m, n, L.ptr(dz),
        dz.stride(0), L.ptr(dgamma), L.ptr(dbeta), L.ptr(ws), 4 * ws.numel(),
        L.stream_ptr(xhat.device))


def _ln_inputs(rows, n, seed):
    """Rows z (float64) of varied scale and offset, the fp32 x^ and 1 / sigma
    the kernel reads, gamma, and g as a view of pitch n + 5 with NaN past
    column n."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    z = (torch.randn(rows, n, device=DEV, generator=gen, dtype=torch.float64) *
         (0.5 + 2 * torch.rand(rows, 1, device=DEV, generator=gen, dtype=torch.float64)) +
         torch.randn(rows, 1, device=DEV, generator=gen, dtype=torch.float64))
    var, mean = torch.var_mean(z, -1, unbiased=False, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    xhat = ((z - mean) * rstd).float()
    gamma = torch.rand(n, device=DEV, generator=gen) + 0.5
    gbuf = torch.full((rows, n + 5), NAN, device=DEV)
    gbuf[:, :n] = torch.randn(rows, n, device=DEV, generator=gen)
    return z, xhat, rstd.view(-1).float(), gamma, gbuf[:, :n]


@pytest.mark.parametrize("m", LN_M)
@pytest.mark.parametrize("n", LN_N)
def test_layernorm_bwd(n, m):
    rows = max(m, 1)
    z, xhat, rstd, gamma, g = _ln_inputs(rows, n, 1000 * n + m)
    outs = []
    for _ in range(2):
        dzbuf = torch.full((rows, n + 3), NAN, device=DEV)
        dgamma = torch.full((n,), NAN, device=DEV)
        dbeta = torch.full((n,), NAN, device=DEV)
        assert _layernorm_bwd_raw(m, g, xhat, rstd, gamma, dzbuf[:, :n], dgamma, dbeta) == 0
        outs.append((dzbuf, dgamma, dbeta))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0))
    dzbuf, dgamma, dbeta = outs[0]
    if m == 0:
        assert bool(dzbuf.isnan().all())
        assert bool((dgamma == 0).all()) and bool((dbeta == 0).all())
        return
    _untouched(dzbuf, n)
    z64 = z.clone().requires_grad_()
    w64 = gamma.double().requires_grad_()
    b64 = torch.zeros(n, device=DEV, dtype=torch.float64, requires_grad=True)
    rz, rg, rb = torch.autograd.grad(F.layer_norm(z64, (n,), w64, b64, 1e-5),
                                     (z64, w64, b64), g.double())
    _cmp("layernorm_bwd", "dz", dzbuf[:, :n], rz)
    _cmp("layernorm_bwd", "dgamma", dgamma, rg)
    _cmp("layernorm_bwd", "dbeta", dbeta, rb)


def test_layernorm_bwd_refusals():
    """n = 84 (past the 80 columns a warp holds) is unsupported; ldg < n is an
    invalid argument.  Both are refused before anything is enqueued."""
    m = 64
    _, xhat, rstd, gamma, g = _ln_inputs(m, 84, 5)
    ws = torch.empty(_lib().lib().fbbev_layernorm_bwd_workspace_bytes(m, 80) // 4,
                     device=DEV)
    dz = torch.full((m, 84), NAN, device=DEV)
    dgb = torch.full((2, 84), NAN, device=DEV)
    assert _layernorm_bwd_raw(m, g, xhat, rstd, gamma, dz, dgb[0], dgb[1], ws) == UNSUPPORTED
    _, xhat, rstd, gamma, g = _ln_inputs(m, 80, 6)
    short = g.as_strided((m, 80), (79, 1))
    assert _layernorm_bwd_raw(m, short, xhat, rstd, gamma, dz[:, :80], dgb[0, :80],
                              dgb[1, :80], ws) == INVALID
    torch.cuda.synchronize()
    assert bool(dz.isnan().all()) and bool(dgb.isnan().all())


# ---------------- LinearLNTrainFunction backward ----------------------------------
LNL_N = (16, 32, 48, 64, 80)
LNL_K = (40, 44, 80, 256, 320)
LNL_CASES = ([(n, k, SMALL) for n in LNL_N for k in LNL_K] +
             [(n, k, 40000) for n in LNL_N for k in (44, 320)])


@pytest.mark.parametrize("n,k,m", LNL_CASES)
def test_linear_ln_gradients(n, k, m):
    from fbbev_b200.ops.linear import linear_ln_train
    gen = torch.Generator(device=DEV).manual_seed(13 * n + k + m)
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    b = torch.randn(n, device=DEV, generator=gen)
    r = torch.randn(m, n, device=DEV, generator=gen)
    lnw = torch.rand(n, device=DEV, generator=gen) + 0.5
    lnb = torch.randn(n, device=DEV, generator=gen)
    gy = torch.randn(m, n, device=DEV, generator=gen)
    for bias in (True, False):
        for res in (True, False):
            leaves = [x, w] + ([b] if bias else []) + ([r] if res else [])
            names = ["dx", "dw"] + (["db"] if bias else []) + (["dresidual"] if res else [])
            p32 = [v.clone().requires_grad_() for v in leaves]
            norm = nn.LayerNorm(n).to(DEV)
            norm.weight, norm.bias = nn.Parameter(lnw.clone()), nn.Parameter(lnb.clone())
            y = linear_ln_train(p32[0], p32[1], p32[2] if bias else None,
                                p32[-1] if res else None, norm)
            got = torch.autograd.grad(y, p32 + [norm.weight, norm.bias], gy)
            p64 = [v.double().requires_grad_() for v in leaves + [lnw, lnb]]
            u = F.linear(p64[0], p64[1], p64[2] if bias else None)
            if res:
                u = u + p64[len(leaves) - 1]
            s = F.layer_norm(u, (n,), p64[-2], p64[-1], 1e-5)
            refs = torch.autograd.grad(s, p64, gy.double())
            _cmp("linear_ln", "y", y, s.detach())
            for name, g, rr in zip(names + ["dgamma", "dbeta"], got, refs):
                _cmp("linear_ln", name, g, rr)


# ---------------- which kernels ran ---------------------------------------------------
def test_every_ffn_instantiation_launched():
    """The union of the ffn_tf32_kernel instantiations the FFN cases launched
    == the dispatch rule's 18.  Skips when the module ran only in part.  When
    the profiler reports no FFN kernel at all, the cases' static table stands
    in (printed)."""
    ids = [f"{kind}-{_ffn_id(c)}" for kind in ("fwd", "bwd") for c in FFN_CASES]
    missing = [i for i in ids if i not in LAUNCHED]
    if missing:
        pytest.skip(f"{len(missing)} FFN cases did not run")
    for (entry, qty), err in sorted(WORST.items()):
        print(f"[matrix-worst] {entry} {qty}: {err:.2e}")
    got = set().union(*LAUNCHED.values())
    if not got:
        print("[matrix] the profiler reported no FFN kernel: checking the static "
              "case -> instantiation table instead")
        got = set().union(*STATIC.values())
    want = ffn_instantiations()
    print(f"[matrix] {len(got & want)} of {len(want)} ffn_tf32_kernel instantiations launched")
    assert got == want, (sorted(want - got), sorted(got - want))
