// msda_bwd.cu -- multi-scale deformable attention, backward, for sm_90a.
//
// Drop-in for mmcv `_ext.ms_deform_attn_backward`
//   (call site .../bevformer_utils/multi_scale_deformable_attn_function.py:159-169;
//    arithmetic: mmcv-full 1.5.2 ms_deformable_col2im_gpu_kernel_*, the published
//    Deformable-DETR col2im).
//
// One thread per (batch, query, head): it owns every (level, point) of that head,
// so grad_sampling_loc and grad_attn_weight are plain stores (the reference
// reduces them across CH threads through shared memory); only grad_value, which
// many queries hit, uses red.global.add.f32.  With kDet (deterministic mode,
// msda_det.cuh) the kernels write one record per sample for msda_det_bwd.cu
// instead of the grad_value reductions; all else is the same code.
#include "common.cuh"
#include "msda_det.cuh"

namespace fbbev {

constexpr int kMsdaBwdThreads = 128;

// CH > 0: the head's CH channels of grad_out in registers, the channel loop
// unrolled.  CH == 0: any head width, ch channels walked serially, grad_out
// read per channel.
template <int CH, bool kDet>
__global__ void __launch_bounds__(kMsdaBwdThreads) msda_bwd_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, const float* __restrict__ loc,
    const float* __restrict__ attw, const float* __restrict__ grad_out,
    int64_t n_items, int n_value, int heads, int ch_rt, int levels, int nq,
    int points, float* __restrict__ grad_value, float* __restrict__ grad_loc,
    float* __restrict__ grad_attw, DetSink det) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;
  const int ch = CH > 0 ? CH : ch_rt;
  const int m = (int)(idx % heads);
  const int64_t bq = idx / heads;
  const int b = (int)(bq / nq);
  const int E = heads * ch;
  const float* gptr = grad_out + bq * E + m * ch;
  float go[CH > 0 ? CH : 1];
  if (CH > 0) {
#pragma unroll
    for (int c = 0; c < CH; ++c) go[c] = __ldg(gptr + c);
  }
  const int64_t wbase = idx * levels * points;
  int pcell = 0;  // kDet: padded cells of the levels before l
  for (int l = 0; l < levels; ++l) {
    const int H = (int)__ldg(shapes + 2 * l), W = (int)__ldg(shapes + 2 * l + 1);
    const int64_t voff = ((int64_t)b * n_value + __ldg(lstart + l)) * E + m * ch;
    const float* val = value + voff;
    float* gval = grad_value + voff;
    for (int p = 0; p < points; ++p) {
      const int64_t wi = wbase + (int64_t)l * points + p;
      const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + wi);
      const float wgt = __ldg(attw + wi);
      const float h = pix(xy.y, H), w = pix(xy.x, W);
      if (!in_image(h, w, H, W)) continue;
      const Bilinear bl(h, w);
      if (kDet)
        det.value_record(wi, pcell + bl.padded_cell(W), heads, m, h, w, wgt);
      const int64_t o1 = bl.offset(W, E);
      const int64_t o2 = o1 + E, o3 = o1 + (int64_t)W * E, o4 = o3 + E;
      float g_h = 0.f, g_w = 0.f, g_a = 0.f;
#pragma unroll
      for (int c = 0; c < (CH > 0 ? CH : ch); ++c) {
        const float g = CH > 0 ? go[c] : __ldg(gptr + c);
        const float top = g * wgt;
        float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
        if (bl.ok1(H, W)) { v1 = __ldg(val + o1 + c); if (!kDet) atomicAdd(gval + o1 + c, bl.w1 * top); }
        if (bl.ok2(H, W)) { v2 = __ldg(val + o2 + c); if (!kDet) atomicAdd(gval + o2 + c, bl.w2 * top); }
        if (bl.ok3(H, W)) { v3 = __ldg(val + o3 + c); if (!kDet) atomicAdd(gval + o3 + c, bl.w3 * top); }
        if (bl.ok4(H, W)) { v4 = __ldg(val + o4 + c); if (!kDet) atomicAdd(gval + o4 + c, bl.w4 * top); }
        g_h += (-bl.hw * v1 - bl.lw * v2 + bl.hw * v3 + bl.lw * v4) * top;
        g_w += (-bl.hh * v1 + bl.hh * v2 - bl.lh * v3 + bl.lh * v4) * top;
        g_a += (bl.w1 * v1 + bl.w2 * v2 + bl.w3 * v3 + bl.w4 * v4) * g;
      }
      grad_attw[wi] = g_a;
      reinterpret_cast<float2*>(grad_loc)[wi] =
          make_float2((float)W * g_w, (float)H * g_h);
    }
    pcell += (H + 1) * (W + 1);
  }
}

template <bool kDet>
static int launch_msda_bwd(const float* value, const int64_t* spatial_shapes,
                           const int64_t* level_start, const float* loc,
                           const float* attw, const float* grad_out,
                           int64_t n_items, int n_value, int heads, int ch,
                           int levels, int nq, int points, float* grad_value,
                           float* grad_loc, float* grad_attw,
                           const DetSink& det, cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(n_items, kMsdaBwdThreads);
  count_launch();
  auto launch = [&](auto CH) {
    msda_bwd_kernel<CH.value, kDet><<<grid, kMsdaBwdThreads, 0, st>>>(
        value, spatial_shapes, level_start, loc, attw, grad_out, n_items,
        n_value, heads, ch, levels, nq, points, grad_value, grad_loc,
        grad_attw, det);
  };
  if (!dispatch(HeadWidths(), ch, launch))
    launch(std::integral_constant<int, 0>());
  return launch_status();
}

int msda_bwd_records(const float* value, const int64_t* spatial_shapes,
                     const int64_t* level_start, const float* loc,
                     const float* attw, const float* grad_out, int n_value,
                     int heads, int ch, int levels, int nq, int points,
                     float* grad_loc, float* grad_attw, const DetSink& det,
                     cudaStream_t st) {
  return launch_msda_bwd<true>(value, spatial_shapes, level_start, loc, attw,
                               grad_out, (int64_t)nq * heads, n_value, heads,
                               ch, levels, nq, points, nullptr, grad_loc,
                               grad_attw, det, st);
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API int fbbev_msda_bwd(const float* value, const int64_t* spatial_shapes,
                             const int64_t* level_start, const float* loc,
                             const float* attw, const float* grad_out,
                             int32_t bs, int32_t n_value, int32_t heads,
                             int32_t ch, int32_t levels, int32_t nq,
                             int32_t points, float* grad_value, float* grad_loc,
                             float* grad_attw, fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !loc || !attw ||
      !grad_out || !grad_value || !grad_loc || !grad_attw)
    return FBBEV_ERR_INVALID_ARGUMENT;
  return launch_msda_bwd<false>(value, spatial_shapes, level_start, loc,
                                attw, grad_out, n_items, n_value, heads, ch,
                                levels, nq, points, grad_value, grad_loc,
                                grad_attw, DetSink(), as_stream(stream));
}
