"""ctypes binding of ``libfbbev_b200.so`` (C ABI: ``include/fbbev_b200.h``).

PyTorch is plumbing here: it owns device memory and streams; every kernel on
the hot path is in the shared library.  There is NO fallback -- if the library
is missing or a call fails, an exception is raised.
"""
import ctypes
import os
import subprocess

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# FBBEV_LIB: kernel-tuning aid, points at a variant build of the same ABI
LIB_PATH = os.environ.get("FBBEV_LIB") or os.path.join(
    _HERE, "lib", "libfbbev_b200.so")
CSRC_DIR = os.path.join(_HERE, "csrc")

_p = ctypes.c_void_p
_i32 = ctypes.c_int32
_i64 = ctypes.c_int64
_sz = ctypes.c_size_t

# name -> (restype, argtypes); mirrors include/fbbev_b200.h declaration order
_SIGNATURES = {
    "fbbev_abi_version": (ctypes.c_int, []),
    "fbbev_debug_launch_count": (ctypes.c_longlong, []),
    "fbbev_error_string": (ctypes.c_char_p, [ctypes.c_int]),
    "fbbev_bev_pool_v2_fwd": (ctypes.c_int, [_p] * 7 + [_i32, _i32, _p, _p]),
    "fbbev_bev_pool_v2_dense_workspace_bytes": (
        _sz, [_i32, _i64, _i32, _i32, _i32]),
    "fbbev_bev_pool_v2_plan": (
        ctypes.c_int,
        [_p, _p, _p, _i32, _p, _i32, _i32, _i32, _i64, _p, _sz, _p]),
    "fbbev_bev_pool_v2_fwd_dense_planned": (
        ctypes.c_int,
        [_p] * 7 + [_i32, _i32, _i32, _i32, _i64, _p, _p, _sz, _p]),
    "fbbev_bev_pool_v2_sums_planned": (
        ctypes.c_int, [_p] * 7 + [_i32, _i32, _i32, _i32, _i64, _p, _sz, _p]),
    "fbbev_bev_pool_v2_zmean_planned": (
        ctypes.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i64, _i32, _p, _p, _sz,
                       _p]),
    "fbbev_bev_pool_v2_write_planned": (
        ctypes.c_int, [_p, _p, _i32, _i32, _i32, _i32, _i64, _i32, _p, _p, _p,
                       _sz, _p]),
    "fbbev_bev_pool_v2_bwd": (ctypes.c_int, [_p] * 8 + [_i32, _i32, _p, _p, _p]),
    "fbbev_bev_pool_v2_bwd_bczyx": (
        ctypes.c_int, [_p] * 8 + [_i32, _i32, _i64, _p, _p, _p]),
    "fbbev_bev_pool_v2_bwd_order_workspace_bytes": (
        _sz, [_i32, _i32, _i32, _i64]),
    "fbbev_bev_pool_v2_bwd_order": (
        ctypes.c_int, [_p] * 5 + [_i32, _i32, _p, _p, _i32, _i32, _i32, _i64,
                                  _p, _sz, _p]),
    "fbbev_bev_pool_v2_bwd_rows": (
        ctypes.c_int, [_p, _i32, _i32, _i64, _i32, _p, _sz, _i32, _i32, _p, _p,
                       _p]),
    "fbbev_bev_pool_v2_bwd_ordered": (
        ctypes.c_int, [_p] * 4 + [_i32, _i32, _i64, _i32, _p, _sz, _i32, _i32,
                                  _p, _p, _p]),
    "fbbev_voxel_prepare_workspace_bytes": (_sz, [_i64, _i64]),
    "fbbev_voxel_prepare": (
        ctypes.c_int, [_p, _p, ctypes.c_float] + [_i32] * 5 + [_p] * 3 +
        [_p] * 6 + [_p, _sz, _i32, _p, _sz, _p]),
    "fbbev_voxel_prepare_cams": (
        ctypes.c_int, [_p] * 8 + [_i32, _p, ctypes.c_float] + [_i32] * 5 +
        [_p] * 3 + [_p] * 6 + [_p, _sz, _i32, _p, _sz, _p]),
    "fbbev_lift_tail_fwd": (
        ctypes.c_int, [_p, _i64, _p, _i64, _i32, _i32, _i32, _i32, _p, _p, _p]),
    "fbbev_bev_mask_fold_workspace_bytes": (_sz, [_i32, _i32]),
    "fbbev_bev_mask_fold": (
        ctypes.c_int, [_p, _p, _i32, _i32, _i32, _i32, _p, _p, _sz, _p]),
    "fbbev_point_sampling": (
        ctypes.c_int, [_p] * 3 + [_i32] * 3 + [_p] * 5 + [_i32] * 3 +
        [ctypes.c_float] * 4 + [_p] * 4),
    "fbbev_bev_query_init": (ctypes.c_int, [_p, _p, _i32, _i32, _i32, _p, _p]),
    "fbbev_tokens_to_map": (ctypes.c_int, [_p, _i32, _i32, _i32, _p, _p]),
    "fbbev_msda_fwd": (ctypes.c_int, [_p] * 5 + [_i32] * 7 + [_p, _p]),
    "fbbev_msda_bwd": (ctypes.c_int, [_p] * 6 + [_i32] * 7 + [_p] * 4),
    "fbbev_msda_fused_fwd": (ctypes.c_int, [_p] * 6 + [_i32] * 8 + [_p, _p]),
    "fbbev_msda_fused_bwd": (ctypes.c_int, [_p] * 7 + [_i32] * 7 + [_p] * 4),
    "fbbev_da_sca_workspace_bytes": (_sz, [_i32, _i32]),
    "fbbev_da_sca_fwd": (ctypes.c_int,
                         [_p] * 10 + [_i32] * 10 + [_p, _p, _sz, _i32, _p]),
    "fbbev_da_sca_prologue": (ctypes.c_int,
                              [_p] + [_i32] * 9 + [_p, _p, _sz, _p]),
    "fbbev_da_sca_bwd": (ctypes.c_int, [_p] * 11 + [_i32] * 10 + [_p] * 5),
    "fbbev_msda_fused_bwd_det_workspace_bytes": (_sz, [_i32] * 5),
    "fbbev_msda_fused_bwd_det": (
        ctypes.c_int, [_p] * 7 + [_i32] * 7 + [_p] * 4 + [_sz, _p]),
    "fbbev_da_sca_bwd_det_workspace_bytes": (_sz, [_i32] * 9),
    "fbbev_da_sca_bwd_det": (
        ctypes.c_int, [_p] * 11 + [_i32] * 10 + [_p] * 5 + [_sz, _p]),
    "fbbev_msda_bwd_det_workspace_bytes": (_sz, [_i32] * 5),
    "fbbev_msda_bwd_det": (
        ctypes.c_int, [_p] * 6 + [_i32] * 7 + [_p] * 4 + [_sz, _p]),
    "fbbev_history_warp": (ctypes.c_int, [_p, _i64, _p] + [_i32] * 5 +
                           [_p, _i32, _i32, _p]),
    "fbbev_history_warp_bwd_workspace_bytes": (_sz, [_i32] * 5),
    "fbbev_history_warp_bwd": (ctypes.c_int, [_p, _i64, _i64, _i32, _p, _p] +
                               [_i32] * 5 + [_p, _i32, _p, _sz, _p]),
    "fbbev_history_fuse_supported": (ctypes.c_int, [_i32, _i32]),
    "fbbev_history_fuse_fwd": (ctypes.c_int, [_p, _i64, _p, _i64] + [_p] * 9 +
                               [_i32] * 7 + [_p, _p, _i32, _p]),
    "fbbev_history_train_workspace_bytes": (_sz, [_i32] * 5),
    "fbbev_history_train_fwd": (ctypes.c_int, [
        _p, _i64, _p, _i64] + [_p] * 11 + [
        ctypes.c_double, ctypes.c_double] + [_i32] * 8 + [_p, _p, _p, _sz, _p]),
    "fbbev_history_train_bwd": (ctypes.c_int, [
        _p, _i64, _p, _i64] + [_p] * 9 + [_i32] * 8 + [_p] * 9 + [_sz, _p]),
    "fbbev_history_train_fwd_local": (ctypes.c_int, [
        _p, _i64, _p, _i64] + [_p] * 4 + [_i32] * 6 + [_p, _p, _sz, _p]),
    "fbbev_history_train_fwd_global": (ctypes.c_int, [
        _p, _i64, _p, _i64] + [_p] * 11 + [
        ctypes.c_double, ctypes.c_double, _p] + [_i32] * 8 + [
        _p, _p, _p, _sz, _p]),
    "fbbev_history_train_bwd_local": (ctypes.c_int, [
        _p, _i64, _p, _i64] + [_p] * 8 + [_i32] * 7 + [_p] * 9 + [_sz, _p]),
    "fbbev_history_train_bwd_global": (ctypes.c_int, [
        _p, _p, _p, _p] + [_i32] * 7 + [_p] * 4 + [_sz, _p]),
    "fbbev_history_train_full_workspace_bytes": (_sz, [_i32] * 6),
    "fbbev_history_train_full_fwd": (ctypes.c_int, [_p, _i64] + [_p] * 11 + [
        ctypes.c_double, ctypes.c_double] + [_i32] * 8 + [_p, _p, _p, _sz, _p]),
    "fbbev_history_train_full_fwd_local": (ctypes.c_int, [_p, _i64] +
                                           [_p] * 4 + [_i32] * 6 +
                                           [_p, _p, _sz, _p]),
    "fbbev_history_train_full_fwd_global": (ctypes.c_int, [_p, _i64] +
                                            [_p] * 11 + [
        ctypes.c_double, ctypes.c_double, _p] + [_i32] * 8 + [
        _p, _p, _p, _sz, _p]),
    "fbbev_history_train_full_bwd_hidden": (ctypes.c_int, [_p, _i64] +
                                            [_p] * 7 + [_i32] * 7 +
                                            [_p, _p, _sz, _p]),
    "fbbev_history_train_full_bwd": (ctypes.c_int, [_p] * 5 + [_i32] * 8 +
                                     [_p] * 6 + [_sz, _p]),
    "fbbev_history_train_full_bwd_local": (ctypes.c_int, [_p] * 3 +
                                           [_i32] * 7 + [_p] * 6 + [_sz, _p]),
    "fbbev_history_train_full_bwd_global": (ctypes.c_int, [_p] * 4 +
                                            [_i32] * 7 + [_p] * 3 + [_sz, _p]),
    "fbbev_history_restart_grad_workspace_bytes": (_sz, [_i32] * 5),
    "fbbev_history_restart_grad_curr": (ctypes.c_int, [
        _p, _i64, _i64, _i32, _p, _p, _p] + [_i32] * 5 + [_p, _p, _sz, _p]),
    "fbbev_linear_packed_bytes": (ctypes.c_size_t, [_i32, _i32]),
    "fbbev_linear_pack": (ctypes.c_int, [_p, _i32, _i32, _p, _p]),
    "fbbev_linear_fwd_split": (ctypes.c_int, [
        _p, _i64, _p, _i64, _p, _p, _i64, _i32, _i32, _i32, _i32, _p, _i64, _p,
        _i64, _p]),
    "fbbev_linear_fwd": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _i64, _p, _p, _i64, _i32, _i32, _i32,
        ctypes.c_float, _p, _i64, _p]),
    "fbbev_ffn_supported": (ctypes.c_int, [_i32, _i32]),
    "fbbev_ffn_fwd": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _i64, _i32, _i32,
        ctypes.c_float, _p, _i64, _p]),
    "fbbev_linear_fwd_ln_train": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _i64, _p, _p, _i64, _i32, _i32, ctypes.c_float,
        _p, _i64, _p, _p, _p]),
    "fbbev_ffn_fwd_train": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _i64, _i32, _i32,
        ctypes.c_float, _p, _i64, _p, _p, _p, _p]),
    "fbbev_ffn_bwd": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _i32, _i64, _i32, _i32, _p, _p, _i64, _p]),
    "fbbev_layernorm_bwd_workspace_bytes": (_sz, [_i64, _i32]),
    "fbbev_layernorm_bwd": (ctypes.c_int, [
        _p, _i64, _p, _p, _p, _i64, _i32, _p, _i64, _p, _p, _p, _sz, _p]),
    "fbbev_depth_loss_workspace_bytes": (_sz, [_i32, _i32, _i32]),
    "fbbev_depth_loss_fwd": (ctypes.c_int, [_p, _p] + [_i32] * 5 + [
        ctypes.c_float] * 3 + [_p, _p, _p, _p, _sz, _p]),
    "fbbev_depth_loss_bwd": (ctypes.c_int, [_p] * 4 + [_i32] * 4 + [
        ctypes.c_float, _p, _p]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

ABI_VERSION = 5
ERR_UNSUPPORTED = -3    # FBBEV_ERR_UNSUPPORTED
_lib = None


class FbbevError(RuntimeError):
    pass


def build(verbose=False):
    """Compile libfbbev_b200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", CSRC_DIR, "-j", str(min(8, os.cpu_count() or 1))]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                         text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise FbbevError("building libfbbev_b200.so failed")
    return LIB_PATH


def lib():
    """Load the library (never builds implicitly; never falls back)."""
    global _lib
    if _proxy is not None and _lib is not None:
        return _proxy
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FbbevError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ "
                f"as g; g.build()'` (or `make -C {CSRC_DIR}`).  The CUDA "
                "library is the product; there is no CPU or eager fallback.")
        _lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
        if _lib.fbbev_abi_version() != ABI_VERSION:
            raise FbbevError("libfbbev_b200.so ABI version mismatch")
    return _lib


class KernelTimer:
    """Diagnostics: bracket every C-ABI launch with CUDA events on the calling
    stream (``with KernelTimer() as t: ...; t.records``).  bench.py uses it to
    report per-kernel times / roofline fractions measured live in the run; it
    is off (zero overhead: ``lib()`` returns the CDLL itself) otherwise."""

    _SKIP = ("fbbev_abi_version", "fbbev_debug_launch_count",
             "fbbev_error_string", "fbbev_linear_packed_bytes",
             "fbbev_bev_pool_v2_dense_workspace_bytes",
             "fbbev_bev_pool_v2_bwd_order_workspace_bytes",
             "fbbev_voxel_prepare_workspace_bytes",
             "fbbev_da_sca_workspace_bytes",
             "fbbev_msda_fused_bwd_det_workspace_bytes",
             "fbbev_da_sca_bwd_det_workspace_bytes",
             "fbbev_msda_bwd_det_workspace_bytes",
             "fbbev_history_fuse_supported",
             "fbbev_history_train_workspace_bytes",
             "fbbev_history_train_full_workspace_bytes",
             "fbbev_history_warp_bwd_workspace_bytes",
             "fbbev_history_restart_grad_workspace_bytes",
             "fbbev_layernorm_bwd_workspace_bytes",
             "fbbev_depth_loss_workspace_bytes")

    def __init__(self):
        self.records = []   # (name, args, start_event, end_event)
        self._real = None

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if name in self._SKIP or not name.startswith("fbbev_"):
            return fn

        def timed(*args):
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args)
            e1.record()
            self.records.append((name, args, e0, e1))
            return rc
        return timed

    def __enter__(self):
        global _proxy
        self._real = lib()
        _proxy = self
        return self

    def __exit__(self, *exc):
        global _proxy
        _proxy = None
        return False


_proxy = None


def check(code, what):
    if code != 0:
        msg = lib().fbbev_error_string(code).decode()
        raise FbbevError(f"{what} failed: {msg} (code {code})")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def stream_ptr(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(*tensors):
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise FbbevError(
                "fb-bev_b200 ops run on CUDA tensors only (no CPU fallback); "
                f"got a tensor on {t.device}")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise FbbevError("all tensors must be on the same CUDA device")
    return dev


def matmul_order_flags(*mats):
    """FBBEV_ORDER_SEQ_* bits for the 3x3 matrix stacks a geometry kernel
    applies per point, one bit per argument.

    torch's broadcast ``M.view(.., 1, 1, 1, 3, 3).matmul(pts)`` rounds each
    output as ``fma(m1, x1, m0*x0) + m2*x2`` -- except when M is ONE
    matrix in the column-major layout ``torch.inverse`` returns: the expand is
    then a stride-0 view, cuBLAS receives op 't' and its kernel for that case
    uses the sequential FMA chain (tools/micro/matmul_order2.py).  The flags
    are derived from the tensors exactly as the eager chain would see them, so
    they must be taken BEFORE any ``.contiguous()``."""
    flags = 0
    for i, m in enumerate(mats):
        if m.numel() == 9 and m.stride(-1) != 1:
            flags |= 1 << i
    return flags


ORDER_EXPLICIT = 8      # FBBEV_ORDER_EXPLICIT
_order_codes = {}


def _dot3_orders(m, x):
    """The 18 fp32 ways to form ``m @ x`` ((.., 3, 3) broadcast against
    (.., 3)), in the code order of ``dot3_code`` (csrc/common.cuh).  An fma
    is evaluated in float64 and rounded once (exact for fp32 operands)."""
    def fma(a, b, c):
        return (a.double() * b.double() + c.double()).float()
    xs = [x[..., j] for j in range(3)]
    for last in range(3):
        a, b = [k for k in range(3) if k != last]
        for inner in range(3):
            for outer in range(2):
                rows = []
                for i in range(3):
                    ma, mb, ml = m[..., i, a], m[..., i, b], m[..., i, last]
                    pa, pb = ma * xs[a], mb * xs[b]
                    s = (pa + pb if inner == 0 else
                         fma(ma, xs[a], pb) if inner == 1 else
                         fma(mb, xs[b], pa))
                    rows.append(s + ml * xs[last] if outer == 0 else
                                fma(ml, xs[last], s))
                yield torch.stack(rows, -1)


def matmul_order_codes(mats, points_shape):
    """``order`` argument of ``fbbev_point_sampling``: FBBEV_ORDER_EXPLICIT
    plus, for each matrix stack, the summation order torch's broadcast
    ``mats[i] @ points[..., None]`` rounds with for this shape and layout on
    this device.  cuBLAS picks the kernel (and so the order) by problem size,
    layout and device, so it is measured: once per (shapes, strides, device),
    on seeded random matrices of the same layout and random points, as the
    order that reproduces every output bit.  Each ``mats[i]`` is given as the
    eager chain views it, e.g. ``inv_bda.view(B, 1, 1, 1, 1, 3, 3)``; call
    outside CUDA-graph capture (the first call per shape runs torch ops)."""
    dev = mats[0].device
    key = (tuple(points_shape), str(dev),
           tuple((tuple(m.shape), m.stride()) for m in mats))
    hit = _order_codes.get(key)
    if hit is not None:
        return hit
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(points_shape, generator=g, device=dev)
    order = ORDER_EXPLICIT
    for i, m in enumerate(mats):
        mp = torch.empty_strided(m.size(), m.stride(), device=dev)
        mp.normal_(generator=g)
        want = mp.matmul(x.unsqueeze(-1)).squeeze(-1)
        hits = [int((v == want).all(-1).sum()) for v in _dot3_orders(mp, x)]
        order |= max(range(len(hits)), key=hits.__getitem__) << (8 + 5 * i)
    _order_codes[key] = order
    return order


def c_floats(vals):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])
