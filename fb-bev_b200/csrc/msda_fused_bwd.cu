// msda_fused_bwd.cu -- backward of the two fused deformable-attention entry
// points of msda_fwd.cu, for sm_90a:
//   fbbev_msda_fused_bwd  backward of fbbev_msda_fused_fwd (self-attention)
//   fbbev_da_sca_bwd      backward of fbbev_da_sca_fwd (depth-aware spatial
//                         cross-attention)
//
// Nothing of the forward is materialised: one thread per (batch, query, head),
// the decomposition of the forward kernels, recomputes the softmax, the
// sampling locations and (cross-attention) the depth weights from the
// forward's inputs, and walks the same (camera,) level, point loops:
//   S = <G, sample>,  grad_w += dw * S,
//   grad_offset += w * dw * (dS/dw_im, dS/dh_im)  (loc = ref + off / W and
//                   w_im = loc * W - 0.5: the W cancels),
//   grad_value corners += w * dw * bilinear_weight * G   (vector reductions),
//   grad_dw[cam, z] += w * S,
// then the softmax backward grad_logit = w * (grad_w - sum(w * grad_w)) on the
// thread's own row.  The offset / logit gradients of a row belong to one thread
// and are plain stores (the cross-attention accumulates them over cameras in
// the output row itself), so they are deterministic; grad_value and
// grad_depth_prob, which many queries hit, use red.global.add.  With kDet
// (deterministic mode, msda_det.cuh) the kernels write records for
// msda_det_bwd.cu instead of those reductions; all else is the same code.
#include "common.cuh"
#include "msda_common.cuh"
#include "msda_det.cuh"

namespace fbbev {

constexpr int kFusedBwdThreads = 128;

// p[0..VW) += s * g[0..VW) with one vector reduction (red.global.add.v4/.v2.f32)
template <int VW>
__device__ __forceinline__ void red_vec(float* p, float s, const float* g);
template <>
__device__ __forceinline__ void red_vec<4>(float* p, float s, const float* g) {
  atomicAdd(reinterpret_cast<float4*>(p),
            make_float4(s * g[0], s * g[1], s * g[2], s * g[3]));
}
template <>
__device__ __forceinline__ void red_vec<2>(float* p, float s, const float* g) {
  atomicAdd(reinterpret_cast<float2*>(p), make_float2(s * g[0], s * g[1]));
}
template <>
__device__ __forceinline__ void red_vec<1>(float* p, float s, const float* g) {
  atomicAdd(p, s * g[0]);
}

// Backward of one bilinear sample of a head (sample_accum's convention): with
// G the upstream gradient of the head's CH channels, returns S = <G, sample>,
// gh = <G, d sample / d h_im> and gw = <G, d sample / d w_im>, and adds
// a * corner_weight * G to the four corners of `gval` (skipped when NULL).
template <int CH>
__device__ __forceinline__ void sample_bwd(const float* __restrict__ val,
                                           float* __restrict__ gval, int H,
                                           int W, int E, float h_im,
                                           float w_im, float a,
                                           const float (&G)[CH], float& S,
                                           float& gh, float& gw) {
  S = gh = gw = 0.f;
  if (!in_image(h_im, w_im, H, W)) return;
  constexpr int VW = VecWidth<CH>::value;
  const Bilinear bl(h_im, w_im);
  // corner flags and offsets spelled out from h_low / w_low rather than
  // okN() / offset(): same values, but ptxas then spills less in the kDet
  // cross-attention instantiations
  const int h_low = bl.h_low, w_low = bl.w_low;
  const int h_high = h_low + 1, w_high = w_low + 1;
  const bool ok1 = h_low >= 0 && w_low >= 0;
  const bool ok2 = h_low >= 0 && w_high <= W - 1;
  const bool ok3 = h_high <= H - 1 && w_low >= 0;
  const bool ok4 = h_high <= H - 1 && w_high <= W - 1;
  const int64_t o1 = ((int64_t)h_low * W + w_low) * E;
  const int64_t o2 = o1 + E, o3 = o1 + (int64_t)W * E, o4 = o3 + E;
#pragma unroll
  for (int c = 0; c < CH; c += VW) {
    float v1[VW], v2[VW], v3[VW], v4[VW];
#pragma unroll
    for (int k = 0; k < VW; ++k) v1[k] = v2[k] = v3[k] = v4[k] = 0.f;
    if (ok1) load_vec<VW>(val + o1 + c, v1);
    if (ok2) load_vec<VW>(val + o2 + c, v2);
    if (ok3) load_vec<VW>(val + o3 + c, v3);
    if (ok4) load_vec<VW>(val + o4 + c, v4);
#pragma unroll
    for (int k = 0; k < VW; ++k) {
      const float g = G[c + k];
      S += g * (bl.w1 * v1[k] + bl.w2 * v2[k] + bl.w3 * v3[k] + bl.w4 * v4[k]);
      gh += g * (-bl.hw * v1[k] - bl.lw * v2[k] + bl.hw * v3[k] + bl.lw * v4[k]);
      gw += g * (-bl.hh * v1[k] + bl.hh * v2[k] - bl.lh * v3[k] + bl.lh * v4[k]);
    }
    if (gval) {
      if (ok1) red_vec<VW>(gval + o1 + c, a * bl.w1, G + c);
      if (ok2) red_vec<VW>(gval + o2 + c, a * bl.w2, G + c);
      if (ok3) red_vec<VW>(gval + o3 + c, a * bl.w3, G + c);
      if (ok4) red_vec<VW>(gval + o4 + c, a * bl.w4, G + c);
    }
  }
}

// Backward of sample_scalar: adds corner_weight * g to the (up to) four
// corners of a [pixel][stride] map.
__device__ __forceinline__ void scatter_scalar(float* __restrict__ gmap, int H,
                                               int W, int stride, float h_im,
                                               float w_im, float g) {
  if (!in_image(h_im, w_im, H, W)) return;
  const Bilinear bl(h_im, w_im);
  float* p1 = gmap + bl.offset(W, stride);
  if (bl.ok1(H, W)) atomicAdd(p1, bl.w1 * g);
  if (bl.ok2(H, W)) atomicAdd(p1 + stride, bl.w2 * g);
  if (bl.ok3(H, W)) atomicAdd(p1 + (int64_t)W * stride, bl.w3 * g);
  if (bl.ok4(H, W)) atomicAdd(p1 + (int64_t)W * stride + stride, bl.w4 * g);
}

// G[0..CH) = grad_out of one head, divided by `cnt`
template <int CH>
__device__ __forceinline__ void load_grad(const float* __restrict__ go,
                                          float cnt, float (&G)[CH]) {
  constexpr int VW = VecWidth<CH>::value;
#pragma unroll
  for (int c = 0; c < CH; c += VW) load_vec<VW>(go + c, G + c);
  if (cnt != 1.f) {
#pragma unroll
    for (int c = 0; c < CH; ++c) G[c] = __fdiv_rn(G[c], cnt);
  }
}

// softmax backward on the thread's own row: gl holds grad_w on entry,
// w * (grad_w - sum_j w_j grad_w_j) on exit
__device__ __forceinline__ void softmax_bwd_row(const float* __restrict__ lg,
                                                float* gl, int n, float mx,
                                                float inv) {
  float dot = 0.f;
#pragma unroll 1
  for (int i = 0; i < n; ++i) dot += expf(__ldg(lg + i) - mx) * inv * gl[i];
#pragma unroll 1
  for (int i = 0; i < n; ++i)
    gl[i] = expf(__ldg(lg + i) - mx) * inv * (gl[i] - dot);
}

// ---------------- backward of fbbev_msda_fused_fwd -------------------------
template <int CH, bool kDet>
__global__ void __launch_bounds__(kFusedBwdThreads) msda_fused_bwd_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, const float* __restrict__ ref,
    const float* __restrict__ offsets, const float* __restrict__ logits,
    const float* __restrict__ grad_out, int64_t n_items, int n_value,
    int heads, int levels, int nq, int points, float* __restrict__ grad_value,
    float* __restrict__ grad_offsets, float* __restrict__ grad_logits,
    DetSink det) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;  // idx = (b*nq + q)*heads + m
  const int m = (int)(idx % heads);
  const int64_t bq = idx / heads;
  const int b = (int)(bq / nq);
  const int E = heads * CH;
  float G[CH];
  load_grad<CH>(grad_out + bq * E + m * CH, 1.f, G);
  const int64_t wbase = idx * levels * points;
  float mx, inv;
  softmax_stats(logits + wbase, levels * points, mx, inv);
  int pcell = 0;  // kDet: padded cells of the levels before l
  for (int l = 0; l < levels; ++l) {
    const int H = (int)__ldg(shapes + 2 * l), W = (int)__ldg(shapes + 2 * l + 1);
    const int64_t voff =
        ((int64_t)b * n_value + __ldg(lstart + l)) * E + m * CH;
    const float2 r =
        __ldg(reinterpret_cast<const float2*>(ref) + bq * levels + l);
#pragma unroll 1
    for (int p = 0; p < points; ++p) {
      const int64_t wi = wbase + (int64_t)l * points + p;
      const float2 off = __ldg(reinterpret_cast<const float2*>(offsets) + wi);
      const float lx = r.x + __fdiv_rn(off.x, (float)W);
      const float ly = r.y + __fdiv_rn(off.y, (float)H);
      const float wgt = expf(__ldg(logits + wi) - mx) * inv;
      const float h_im = pix(ly, H), w_im = pix(lx, W);
      float S, gh, gw;
      sample_bwd<CH>(
          value + voff, !kDet && grad_value ? grad_value + voff : nullptr, H,
          W, E, h_im, w_im, wgt, G, S, gh, gw);
      if (kDet && det.key && in_image(h_im, w_im, H, W))
        det.value_record(wi, pcell + Bilinear(h_im, w_im).padded_cell(W),
                         heads, m, h_im, w_im, wgt);
      if (grad_offsets)
        reinterpret_cast<float2*>(grad_offsets)[wi] =
            make_float2(wgt * gw, wgt * gh);
      if (grad_logits) grad_logits[wi] = S;
    }
    pcell += (H + 1) * (W + 1);
  }
  if (grad_logits)
    softmax_bwd_row(logits + wbase, grad_logits + wbase, levels * points, mx,
                    inv);
}

// ---------------- backward of fbbev_da_sca_fwd -----------------------------
// kDet: one pass (sample, camera det.cam); the items of sample
// det.item0 / (nq * heads) only.  Offset / logit rows are accumulated over the
// passes of the cameras in camera order, exactly as over the camera loop.
template <int CH, int Z, bool kDet>
__global__ void __launch_bounds__(kFusedBwdThreads) da_sca_bwd_kernel(
    const float* __restrict__ value, const float* __restrict__ depth_prob,
    const float* __restrict__ ref_cam, const float* __restrict__ ref_depth,
    const uint8_t* __restrict__ mask, const float* __restrict__ offsets,
    const float* __restrict__ logits, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, DaScaParams P,
    const float* __restrict__ grad_out, float* __restrict__ grad_value,
    float* __restrict__ grad_depth_prob, float* __restrict__ grad_offsets,
    float* __restrict__ grad_logits, DetSink det) {
  const int64_t idx =
      (kDet ? det.item0 : 0) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n_items = kDet ? det.item0 + (int64_t)P.nq * P.heads
                               : (int64_t)P.bs * P.nq * P.heads;
  if (idx >= n_items) return;
  const int m = (int)(idx % P.heads);
  const int64_t bq = idx / P.heads;  // b*nq + q
  const int b = (int)(bq / P.nq);
  const int q = (int)(bq - (int64_t)b * P.nq);
  const int E = P.heads * CH;
  const int LP = P.levels * P.points;
  const int H0 = (int)__ldg(shapes + 0), W0 = (int)__ldg(shapes + 1);
  const int64_t wbase = idx * LP;

  // the forward's camera count (mask bit 0; value 2 is processed, not counted)
  int count = 0, n_first = -1, n_last = -1;
  unsigned any = 0;
  for (int n = 0; n < P.n_cams; ++n) {
    const int64_t rbase = (((int64_t)n * P.bs + b) * P.nq + q) * Z;
    unsigned seen = 0;
#pragma unroll
    for (int z = 0; z < Z; ++z) seen |= __ldg(mask + rbase + z);
    count += (int)(seen & 1u);
    any |= seen;
    if (seen) {
      if (n_first < 0) n_first = n;
      n_last = n;
    }
  }
  if (!any) {  // no camera sees the query: zero offset / logit gradients
    if (kDet && det.cam != 0) return;
    for (int i = 0; i < LP; ++i) {
      if (grad_offsets)
        reinterpret_cast<float2*>(grad_offsets)[wbase + i] =
            make_float2(0.f, 0.f);
      if (grad_logits) grad_logits[wbase + i] = 0.f;
    }
    return;
  }
  float G[CH];
  load_grad<CH>(grad_out + bq * E + m * CH, (float)max(count, 1), G);
  const int64_t item = idx - (kDet ? det.item0 : 0);  // item of the pass
  if (kDet && det.key) {
#pragma unroll
    for (int c = 0; c < CH; ++c) det.G[item * CH + c] = G[c];
  }
  float mx, inv;
  softmax_stats(logits + wbase, LP, mx, inv);
  // the lanes of one query hold its heads side by side when heads divides 32:
  // the depth gradient (a sum over heads) is then reduced with shuffles and
  // scattered once per query; otherwise every head scatters its own share
  const int lane = threadIdx.x & (kWarp - 1);
  const bool shfl = (kWarp % P.heads) == 0;
  const unsigned grp =
      !shfl ? 0u
            : (P.heads == kWarp ? kFull
                                : ((1u << P.heads) - 1u) << (lane & ~(P.heads - 1)));
  bool first = kDet ? det.cam == n_first : true;
  // depth records: one per (query, z), or per (query, head, z) without shuffles
  const int hs_n = shfl ? 1 : P.heads, hs = shfl ? 0 : m;

#pragma unroll 1
  for (int n = kDet ? det.cam : 0; n < (kDet ? det.cam + 1 : P.n_cams); ++n) {
    const int64_t rbase = (((int64_t)n * P.bs + b) * P.nq + q) * Z;
    unsigned seen = 0;
#pragma unroll
    for (int z = 0; z < Z; ++z) seen |= __ldg(mask + rbase + z);
    if (!seen) continue;
    const int bn = b * P.n_cams + n;
    const float* dp = depth_prob + (int64_t)bn * H0 * W0 * P.DC;
    float dw[Z], gdw[Z];
    float2 rxy[Z];
    int bin[Z];
#pragma unroll
    for (int z = 0; z < Z; ++z) {
      rxy[z] = __ldg(reinterpret_cast<const float2*>(ref_cam) + rbase + z);
      bin[z] = depth_bin(__ldg(ref_depth + rbase + z), P.d_min, P.d_step,
                         P.DC);
      dw[z] = sample_scalar(dp + bin[z], H0, W0, P.DC, pix(rxy[z].y, H0),
                            pix(rxy[z].x, W0));
      gdw[z] = 0.f;
    }
    int pcell = 0;  // kDet: padded cells of the levels before l
    for (int l = 0; l < P.levels; ++l) {
      const int H = (int)__ldg(shapes + 2 * l);
      const int W = (int)__ldg(shapes + 2 * l + 1);
      const int64_t voff =
          ((int64_t)bn * P.n_value + __ldg(lstart + l)) * E + m * CH;
      // one copy of the sampling code (not Z unrolled ones, which would
      // multiply the register footprint): the anchor's values are selected
#pragma unroll 1
      for (int p = 0; p < P.points; ++p) {
        const int zp = p % Z;  // point index = p'*Z + z
        float2 rz = rxy[0];
        float dwz = dw[0];
#pragma unroll
        for (int z = 1; z < Z; ++z)
          if (zp == z) { rz = rxy[z]; dwz = dw[z]; }
        const int64_t wi = wbase + (int64_t)l * P.points + p;
        const float2 off =
            __ldg(reinterpret_cast<const float2*>(offsets) + wi);
        const float lx = rz.x + __fdiv_rn(off.x, (float)W);
        const float ly = rz.y + __fdiv_rn(off.y, (float)H);
        const float w = expf(__ldg(logits + wi) - mx) * inv;
        const float a = w * dwz;
        const float h_im = pix(ly, H), w_im = pix(lx, W);
        float S, gh, gw;
        sample_bwd<CH>(
            value + voff, !kDet && grad_value ? grad_value + voff : nullptr,
            H, W, E, h_im, w_im, a, G, S, gh, gw);
        if (kDet && det.key && in_image(h_im, w_im, H, W))
          det.value_record(item * LP + (int64_t)l * P.points + p,
                           pcell + Bilinear(h_im, w_im).padded_cell(W),
                           P.heads, m, h_im, w_im, a);
#pragma unroll
        for (int z = 0; z < Z; ++z)
          if (zp == z) gdw[z] += w * S;
        if (grad_logits) {
          const float t = dwz * S;
          grad_logits[wi] = first ? t : grad_logits[wi] + t;
        }
        if (grad_offsets) {
          float2* go = reinterpret_cast<float2*>(grad_offsets) + wi;
          float2 t = make_float2(a * gw, a * gh);
          if (!first) {
            const float2 o = *go;
            t.x += o.x;
            t.y += o.y;
          }
          *go = t;
        }
      }
      pcell += (H + 1) * (W + 1);
    }
    first = false;
    if (kDet ? det.dkey != nullptr : grad_depth_prob != nullptr) {
      if (shfl) {
#pragma unroll
        for (int z = 0; z < Z; ++z)
          for (int o = P.heads >> 1; o > 0; o >>= 1)
            gdw[z] += __shfl_xor_sync(grp, gdw[z], o);
      }
      if (kDet && (!shfl || m == 0)) {
        // key: (camera, padded cell, bin); slot: ((cam, q, hs), z)
        const int64_t slot = (((int64_t)n * P.nq + q) * hs_n + hs) * Z;
        const int cells = (H0 + 1) * (W0 + 1);
#pragma unroll
        for (int z = 0; z < Z; ++z) {
          const float h_im = pix(rxy[z].y, H0), w_im = pix(rxy[z].x, W0);
          if (in_image(h_im, w_im, H0, W0)) {
            det.dkey[slot + z] = (uint32_t)(
                (n * cells + Bilinear(h_im, w_im).padded_cell(W0)) * P.DC + bin[z]);
            det.drec[slot + z] = make_float3(h_im, w_im, gdw[z]);
          }
        }
      } else if (!shfl || m == 0) {
        float* gdp = grad_depth_prob + (int64_t)bn * H0 * W0 * P.DC;
#pragma unroll
        for (int z = 0; z < Z; ++z)
          scatter_scalar(gdp + bin[z], H0, W0, P.DC, pix(rxy[z].y, H0),
                         pix(rxy[z].x, W0), gdw[z]);
      }
    }
  }
  if (grad_logits && (!kDet || det.cam == n_last))
    softmax_bwd_row(logits + wbase, grad_logits + wbase, LP, mx, inv);
}

template <bool kDet>
static int launch_msda_fused_bwd(
    const float* value, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* ref, const float* offsets,
    const float* logits, const float* grad_out, int64_t n_items, int n_value,
    int heads, int ch, int levels, int nq, int points, float* grad_value,
    float* grad_offsets, float* grad_logits, const DetSink& det,
    cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(n_items, kFusedBwdThreads);
  count_launch();
  if (!dispatch(HeadWidths(), ch, [&](auto CH) {
        msda_fused_bwd_kernel<CH.value, kDet>
            <<<grid, kFusedBwdThreads, 0, st>>>(
                value, spatial_shapes, level_start, ref, offsets, logits,
                grad_out, n_items, n_value, heads, levels, nq, points,
                grad_value, grad_offsets, grad_logits, det);
      }))
    return FBBEV_ERR_UNSUPPORTED;
  return launch_status();
}

template <bool kDet>
static int launch_da_sca_bwd(
    const float* value, const float* depth_prob, const float* ref_cam,
    const float* ref_depth, const uint8_t* mask, const float* offsets,
    const float* logits, const int64_t* spatial_shapes,
    const int64_t* level_start, const DaScaParams& P, int ch, int Z,
    int64_t n_items, const float* grad_out, float* grad_value,
    float* grad_depth_prob, float* grad_offsets, float* grad_logits,
    const DetSink& det, cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(n_items, kFusedBwdThreads);
  count_launch();
  bool launched = false;
  dispatch(HeadWidths(), ch, [&](auto CH) {
    launched = dispatch(ZAnchors(), Z, [&](auto ZV) {
      da_sca_bwd_kernel<CH.value, ZV.value, kDet>
          <<<grid, kFusedBwdThreads, 0, st>>>(
              value, depth_prob, ref_cam, ref_depth, mask, offsets, logits,
              spatial_shapes, level_start, P, grad_out, grad_value,
              grad_depth_prob, grad_offsets, grad_logits, det);
    });
  });
  if (!launched) return FBBEV_ERR_UNSUPPORTED;
  return launch_status();
}

int msda_fused_bwd_records(const float* value, const int64_t* spatial_shapes,
                           const int64_t* level_start, const float* ref,
                           const float* offsets, const float* logits,
                           const float* grad_out, int n_value, int heads,
                           int ch, int levels, int nq, int points,
                           float* grad_offsets, float* grad_logits,
                           const DetSink& det, cudaStream_t st) {
  return launch_msda_fused_bwd<true>(
      value, spatial_shapes, level_start, ref, offsets, logits, grad_out,
      (int64_t)nq * heads, n_value, heads, ch, levels, nq, points, nullptr,
      grad_offsets, grad_logits, det, st);
}

int da_sca_bwd_records(const float* value, const float* depth_prob,
                       const float* ref_cam, const float* ref_depth,
                       const uint8_t* mask, const float* offsets,
                       const float* logits, const int64_t* spatial_shapes,
                       const int64_t* level_start, const DaScaParams& P,
                       int ch, int Z, const float* grad_out,
                       float* grad_offsets, float* grad_logits,
                       const DetSink& det, cudaStream_t st) {
  return launch_da_sca_bwd<true>(
      value, depth_prob, ref_cam, ref_depth, mask, offsets, logits,
      spatial_shapes, level_start, P, ch, Z, (int64_t)P.nq * P.heads,
      grad_out, nullptr, nullptr, grad_offsets, grad_logits, det, st);
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API int fbbev_msda_fused_bwd(
    const float* value, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* ref, const float* offsets,
    const float* logits, const float* grad_out, int32_t bs, int32_t n_value,
    int32_t heads, int32_t ch, int32_t levels, int32_t nq, int32_t points,
    float* grad_value, float* grad_offsets, float* grad_logits,
    fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !ref || !offsets ||
      !logits || !grad_out || !vec_aligned(value, ch) ||
      !vec_aligned(grad_out, ch) || !vec_aligned(grad_value, ch))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return launch_msda_fused_bwd<false>(
      value, spatial_shapes, level_start, ref, offsets, logits, grad_out,
      n_items, n_value, heads, ch, levels, nq, points, grad_value,
      grad_offsets, grad_logits, DetSink(), as_stream(stream));
}

FBBEV_API int fbbev_da_sca_bwd(
    const float* value, const float* depth_prob, const float* ref_cam,
    const float* ref_depth, const uint8_t* mask, const float* offsets,
    const float* logits, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* dbound_host,
    const float* grad_out, int32_t bs, int32_t n_cams, int32_t nq,
    int32_t n_value, int32_t heads, int32_t ch, int32_t levels,
    int32_t points, int32_t Z, int32_t DC, float* grad_value,
    float* grad_depth_prob, float* grad_offsets, float* grad_logits,
    fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_cams <= 0 || n_value <= 0 || heads <= 0 ||
      ch <= 0 || levels <= 0 || points <= 0 || Z <= 0 || DC <= 0 ||
      !dbound_host || points % Z != 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !depth_prob || !ref_cam || !ref_depth || !mask || !offsets ||
      !logits || !spatial_shapes || !level_start || !grad_out ||
      !vec_aligned(value, ch) || !vec_aligned(grad_out, ch) ||
      !vec_aligned(grad_value, ch))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const DaScaParams P = da_sca_params(dbound_host, bs, n_cams, nq, n_value,
                                      heads, levels, points, DC);
  return launch_da_sca_bwd<false>(
      value, depth_prob, ref_cam, ref_depth, mask, offsets, logits,
      spatial_shapes, level_start, P, ch, Z, n_items, grad_out, grad_value,
      grad_depth_prob, grad_offsets, grad_logits, DetSink(),
      as_stream(stream));
}
