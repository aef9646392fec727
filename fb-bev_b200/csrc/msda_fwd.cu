// msda_fwd.cu -- multi-scale deformable attention, forward, for sm_90a.
//
// Three entry points share one sampling core:
//   fbbev_msda_fwd        drop-in for mmcv `_ext.ms_deform_attn_forward`
//                         (call site multi_scale_deformable_attn_function.py:127-133)
//   fbbev_msda_fused_fwd  softmax + sampling-location arithmetic + sampling of
//                         mmcv MultiScaleDeformableAttention.forward (self_attn)
//   fbbev_da_sca_fwd      the whole depth-aware spatial cross-attention between
//                         the input Linears and output_proj
//                         (spatial_cross_attention_depth.py:86-223, 465-601)
//
// Sampling convention (mmcv 1.5.2 ms_deform_attn_im2col_bilinear): pixel =
// loc * size - 0.5; a point contributes iff -1 < h < H and -1 < w < W; bilinear
// with zero padding; out = sum_{level, point} weight * sample.
//
// Work decomposition: one thread per (batch, query, head) holding the head's
// CH output channels in registers.  The reference kernel uses one thread per
// output SCALAR, so every thread recomputes the same location / bilinear
// weights CH times and loads one float per corner; here the location math runs
// once per head and each corner is CH contiguous floats fetched with 128-bit
// (or 64-bit for CH = 10) loads.  `value` is small enough to live in L2 (1.4 MB
// at the shipped size, 23 MB for the 4-level config), so HBM traffic is the
// streamed operands only -- which the two fused entry points shrink further by
// never materialising sampling_locations / normalised weights / the one-hot
// depth tensor.
#include "common.cuh"
#include "da_sca_smem.h"
#include "msda_common.cuh"

namespace fbbev {

constexpr int kMsdaThreads = 128;

// Ten contiguous floats whose address is 8-byte but not always 16-byte aligned
// (head width 10: the chunk of head m starts 40 m bytes into the pixel): three
// loads -- 128 + 128 + 64 bits when the start is 16-byte aligned, 64 + 128 + 128
// otherwise -- instead of five 64-bit ones.  The gathers of these kernels are
// bound by L1 wavefronts (one per distinct line per load instruction), so two
// fewer instructions per 40-byte chunk is 40 % less L1 work.
__device__ __forceinline__ void load10(const float* p, float (&v)[10]) {
  if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p + 4));
    const float2 c = __ldg(reinterpret_cast<const float2*>(p + 8));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    v[8] = c.x; v[9] = c.y;
  } else {
    const float2 a = __ldg(reinterpret_cast<const float2*>(p));
    const float4 b = __ldg(reinterpret_cast<const float4*>(p + 2));
    const float4 c = __ldg(reinterpret_cast<const float4*>(p + 6));
    v[0] = a.x; v[1] = a.y;
    v[2] = b.x; v[3] = b.y; v[4] = b.z; v[5] = b.w;
    v[6] = c.x; v[7] = c.y; v[8] = c.z; v[9] = c.w;
  }
}

// acc[0..CH) += wgt * bilinear(value_level, h_im, w_im) for one head.
// `val` points at element [pixel 0][head m][channel 0] of the level; pixel
// stride is E = heads * ch floats.
template <int CH>
__device__ __forceinline__ void sample_accum(const float* __restrict__ val,
                                             int H, int W, int E, float h_im,
                                             float w_im, float wgt,
                                             float (&acc)[CH]) {
  if (!in_image(h_im, w_im, H, W)) return;
  constexpr int VW = VecWidth<CH>::value;
  const Bilinear bl(h_im, w_im);
  const float* p1 = val + bl.offset(W, E);
  const float* p2 = p1 + E;
  const float* p3 = p1 + (int64_t)W * E;
  const float* p4 = p3 + E;
  if (CH == 10 && (E & 1) == 0 &&
      (reinterpret_cast<uintptr_t>(val) & 7) == 0) {
    float v1[10], v2[10], v3[10], v4[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) v1[k] = v2[k] = v3[k] = v4[k] = 0.f;
    if (bl.ok1(H, W)) load10(p1, v1);
    if (bl.ok2(H, W)) load10(p2, v2);
    if (bl.ok3(H, W)) load10(p3, v3);
    if (bl.ok4(H, W)) load10(p4, v4);
#pragma unroll
    for (int k = 0; k < 10; ++k) {
      const float s =
          bl.w1 * v1[k] + bl.w2 * v2[k] + bl.w3 * v3[k] + bl.w4 * v4[k];
      acc[k] += s * wgt;
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < CH; c += VW) {
    float v1[VW], v2[VW], v3[VW], v4[VW];
#pragma unroll
    for (int k = 0; k < VW; ++k) v1[k] = v2[k] = v3[k] = v4[k] = 0.f;
    if (bl.ok1(H, W)) load_vec<VW>(p1 + c, v1);
    if (bl.ok2(H, W)) load_vec<VW>(p2 + c, v2);
    if (bl.ok3(H, W)) load_vec<VW>(p3 + c, v3);
    if (bl.ok4(H, W)) load_vec<VW>(p4 + c, v4);
#pragma unroll
    for (int k = 0; k < VW; ++k) {
      const float s =
          bl.w1 * v1[k] + bl.w2 * v2[k] + bl.w3 * v3[k] + bl.w4 * v4[k];
      acc[c + k] += s * wgt;
    }
  }
}

template <int CH>
__device__ __forceinline__ void store_head(float* o, const float (&acc)[CH]) {
  constexpr int VW = VecWidth<CH>::value;
#pragma unroll
  for (int c = 0; c < CH; c += VW) {
    if (VW == 4)
      *reinterpret_cast<float4*>(o + c) =
          make_float4(acc[c], acc[c + 1], acc[c + 2], acc[c + 3]);
    else if (VW == 2)
      *reinterpret_cast<float2*>(o + c) = make_float2(acc[c], acc[c + 1]);
    else
      o[c] = acc[c];
  }
}

// ---------------- drop-in ms_deform_attn_forward ---------------------------
template <int CH>
__global__ void __launch_bounds__(kMsdaThreads) msda_fwd_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, const float* __restrict__ loc,
    const float* __restrict__ attw, int64_t n_items, int n_value, int heads,
    int levels, int nq, int points, float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_items) return;  // idx = (b*nq + q)*heads + m
  const int m = (int)(idx % heads);
  const int64_t bq = idx / heads;
  const int b = (int)(bq / nq);
  const int E = heads * CH;
  float acc[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) acc[c] = 0.f;
  const int64_t wbase = idx * levels * points;
  for (int l = 0; l < levels; ++l) {
    const int H = (int)__ldg(shapes + 2 * l), W = (int)__ldg(shapes + 2 * l + 1);
    const float* val =
        value + ((int64_t)b * n_value + __ldg(lstart + l)) * E + m * CH;
    for (int p = 0; p < points; ++p) {
      const int64_t wi = wbase + (int64_t)l * points + p;
      const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + wi);
      const float wgt = __ldg(attw + wi);
      sample_accum<CH>(val, H, W, E, pix(xy.y, H), pix(xy.x, W), wgt, acc);
    }
  }
  store_head<CH>(out + bq * E + m * CH, acc);
}

// Any head width: one thread per output scalar (the reference's own
// decomposition); used when CH is not one of the specialised widths, e.g. the
// depth look-up launch of DA_MSDeformableAttention.forward (ch = depth bins).
__global__ void __launch_bounds__(kMsdaThreads) msda_fwd_generic_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, const float* __restrict__ loc,
    const float* __restrict__ attw, int64_t n_out, int n_value, int heads,
    int ch, int levels, int nq, int points, float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out) return;  // idx = ((b*nq + q)*heads + m)*ch + c
  const int c = (int)(idx % ch);
  const int64_t item = idx / ch;
  const int m = (int)(item % heads);
  const int64_t bq = item / heads;
  const int b = (int)(bq / nq);
  const int E = heads * ch;
  const int64_t wbase = item * levels * points;
  float col = 0.f;
  for (int l = 0; l < levels; ++l) {
    const int H = (int)__ldg(shapes + 2 * l), W = (int)__ldg(shapes + 2 * l + 1);
    const float* val =
        value + ((int64_t)b * n_value + __ldg(lstart + l)) * E + m * ch + c;
    for (int p = 0; p < points; ++p) {
      const int64_t wi = wbase + (int64_t)l * points + p;
      const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + wi);
      col += sample_scalar(val, H, W, E, pix(xy.y, H), pix(xy.x, W)) *
             __ldg(attw + wi);
    }
  }
  out[idx] = col;
}

// ---------------- fused mmcv MultiScaleDeformableAttention core ------------
// PATCH > 0: self-attention over the BEV map itself (one level, one query per
// value pixel).  A block then owns a PATCH x PATCH_Y patch of queries instead of
// a run of a BEV row: every query samples within a few pixels of itself, so the
// square's footprint in `value` is ~4x smaller than a row segment's and stays
// in L1 (ncu on the row mapping: 75 % L1 hit rate, 133 MB of L2 sectors for a
// 12.8 MB map -- the kernel was bound by L2 gathers).
template <int CH, int PATCH, int PATCH_Y>
__global__ void __launch_bounds__(PATCH > 0 ? PATCH * PATCH_Y * 8 : kMsdaThreads)
    msda_fused_fwd_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, const float* __restrict__ ref,
    const float* __restrict__ offsets, const float* __restrict__ logits,
    int64_t n_items, int n_value, int heads, int levels, int nq, int points,
    int patch_w, float* __restrict__ out) {
  int64_t idx;
  if (PATCH > 0) {
    // heads == 8; grid = (patches_x, patches_y, bs)
    const int m = threadIdx.x & 7, ql = threadIdx.x >> 3;
    const int qx = blockIdx.x * PATCH + ql % PATCH;
    const int qy = blockIdx.y * PATCH_Y + ql / PATCH;
    if (qx >= patch_w || qy * patch_w + qx >= nq) return;
    idx = ((int64_t)blockIdx.z * nq + (int64_t)qy * patch_w + qx) * heads + m;
  } else {
    idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_items) return;
  }
  const int m = (int)(idx % heads);
  const int64_t bq = idx / heads;
  const int b = (int)(bq / nq);
  const int E = heads * CH;
  float acc[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) acc[c] = 0.f;
  const int64_t wbase = idx * levels * points;
  float mx, inv;
  softmax_stats(logits + wbase, levels * points, mx, inv);
  for (int l = 0; l < levels; ++l) {
    const int H = (int)__ldg(shapes + 2 * l), W = (int)__ldg(shapes + 2 * l + 1);
    const float* val =
        value + ((int64_t)b * n_value + __ldg(lstart + l)) * E + m * CH;
    const float2 r =
        __ldg(reinterpret_cast<const float2*>(ref) + bq * levels + l);
    for (int p = 0; p < points; ++p) {
      const int64_t wi = wbase + (int64_t)l * points + p;
      const float2 off = __ldg(reinterpret_cast<const float2*>(offsets) + wi);
      // sampling_locations = ref + offsets / (W_l, H_l)
      const float lx = r.x + __fdiv_rn(off.x, (float)W);
      const float ly = r.y + __fdiv_rn(off.y, (float)H);
      const float wgt = expf(__ldg(logits + wi) - mx) * inv;
      sample_accum<CH>(val, H, W, E, pix(ly, H), pix(lx, W), wgt, acc);
    }
  }
  store_head<CH>(out + bq * E + m * CH, acc);
}

// ---------------- fused depth-aware spatial cross-attention ----------------
template <int CH, int Z>
__global__ void __launch_bounds__(kMsdaThreads) da_sca_fwd_kernel(
    const float* __restrict__ value, const float* __restrict__ depth_prob,
    const float* __restrict__ ref_cam, const float* __restrict__ ref_depth,
    const uint8_t* __restrict__ mask, const float* __restrict__ offsets,
    const float* __restrict__ logits, const int64_t* __restrict__ shapes,
    const int64_t* __restrict__ lstart, DaScaParams P,
    float* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n_items = (int64_t)P.bs * P.nq * P.heads;
  if (idx >= n_items) return;
  const int m = (int)(idx % P.heads);
  const int64_t bq = idx / P.heads;  // b*nq + q
  const int b = (int)(bq / P.nq);
  const int q = (int)(bq - (int64_t)b * P.nq);
  const int E = P.heads * CH;
  const int LP = P.levels * P.points;
  const int H0 = (int)__ldg(shapes + 0), W0 = (int)__ldg(shapes + 1);

  float tot[CH];
#pragma unroll
  for (int c = 0; c < CH; ++c) tot[c] = 0.f;
  int count = 0;
  float mx = 0.f, inv = 0.f;
  bool have_softmax = false;
  const int64_t wbase = idx * LP;

  for (int n = 0; n < P.n_cams; ++n) {
    const int64_t rbase = (((int64_t)n * P.bs + b) * P.nq + q) * Z;
    // per_cam_mask[j].sum(-1) > 0 (:165).  Mask bytes: bit 0 = visible and
    // counted; 2 = visible through the empty-camera rule of a bev_mask
    // (fbbev_bev_mask_fold): processed, not counted (:166-167, :213-214)
    unsigned seen = 0;
#pragma unroll
    for (int z = 0; z < Z; ++z) seen |= __ldg(mask + rbase + z);
    if (!seen) continue;
    count += (int)(seen & 1u);
    if (!have_softmax) {
      softmax_stats(logits + wbase, LP, mx, inv);  // :540
      have_softmax = true;
    }
    const int bn = b * P.n_cams + n;
    // depth look-up: prob of the anchor's depth bin, bilinearly sampled at the
    // anchor's image location (:196-199, :584-591)
    float dw[Z];
    float2 rxy[Z];
    const float* dp = depth_prob + (int64_t)bn * H0 * W0 * P.DC;
#pragma unroll
    for (int z = 0; z < Z; ++z) {
      rxy[z] = __ldg(reinterpret_cast<const float2*>(ref_cam) + rbase + z);
      const int bin =
          depth_bin(__ldg(ref_depth + rbase + z), P.d_min, P.d_step, P.DC);
      dw[z] = sample_scalar(dp + bin, H0, W0, P.DC, pix(rxy[z].y, H0),
                            pix(rxy[z].x, W0));
    }
    float acc[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) acc[c] = 0.f;
    for (int l = 0; l < P.levels; ++l) {
      const int H = (int)__ldg(shapes + 2 * l);
      const int W = (int)__ldg(shapes + 2 * l + 1);
      const float* val =
          value + ((int64_t)bn * P.n_value + __ldg(lstart + l)) * E + m * CH;
      for (int pp = 0; pp < P.points; pp += Z) {
#pragma unroll
        for (int z = 0; z < Z; ++z) {  // point index = p*Z + z   (:563-570)
          const int64_t wi = wbase + (int64_t)l * P.points + pp + z;
          const float2 off =
              __ldg(reinterpret_cast<const float2*>(offsets) + wi);
          const float lx = rxy[z].x + __fdiv_rn(off.x, (float)W);
          const float ly = rxy[z].y + __fdiv_rn(off.y, (float)H);
          // attention_weights * depth_weights, no renormalisation (:592)
          const float wgt = (expf(__ldg(logits + wi) - mx) * inv) * dw[z];
          sample_accum<CH>(val, H, W, E, pix(ly, H), pix(lx, W), wgt, acc);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) tot[c] += acc[c];  // slots += queries (:208-211)
  }
  // slots / clamp(count, min=1)   (:213-216)
  const float cnt = (float)max(count, 1);
#pragma unroll
  for (int c = 0; c < CH; ++c) tot[c] = __fdiv_rn(tot[c], cnt);
  store_head<CH>(out + bq * E + m * CH, tot);
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API size_t fbbev_da_sca_workspace_bytes(int32_t bs, int32_t n_cams) {
  if (bs <= 0 || n_cams <= 0) return 0;
  return da_sca_smem_workspace_bytes(bs, n_cams);
}

// The part of fbbev_da_sca_fwd that depends on the mask only (visible-query
// counts per camera, zero-fill of `out`): callable ahead of time, e.g. on the
// stream that produced the mask.  Returns FBBEV_ERR_UNSUPPORTED when the shape
// takes the global-memory kernel (which has no prologue).
FBBEV_API int fbbev_da_sca_prologue(const uint8_t* mask, int32_t bs,
                                    int32_t n_cams, int32_t nq, int32_t n_value,
                                    int32_t heads, int32_t ch, int32_t levels,
                                    int32_t points, int32_t Z, float* out,
                                    void* workspace, size_t workspace_bytes,
                                    fbbev_stream_t stream) {
  if (bs <= 0 || nq <= 0 || n_cams <= 0 || !mask || !out || !workspace)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (workspace_bytes < da_sca_smem_workspace_bytes(bs, n_cams) ||
      !da_sca_smem_eligible(n_cams, n_value, heads, ch, levels, points, Z) ||
      bs * n_cams > 4096 || (reinterpret_cast<uintptr_t>(out) & 15))
    return FBBEV_ERR_UNSUPPORTED;
  return da_sca_smem_launch(nullptr, nullptr, nullptr, nullptr, mask, nullptr,
                            nullptr, nullptr, 0.f, 1.f, bs, n_cams, nq, n_value,
                            1, out, workspace, as_stream(stream), kScaPrologue);
}

FBBEV_API int fbbev_msda_fwd(const float* value, const int64_t* spatial_shapes,
                             const int64_t* level_start, const float* loc,
                             const float* attw, int32_t bs, int32_t n_value,
                             int32_t heads, int32_t ch, int32_t levels,
                             int32_t nq, int32_t points, float* out,
                             fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !loc || !attw || !out)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const unsigned grid = (unsigned)ceil_div64(n_items, kMsdaThreads);
  cudaStream_t st = as_stream(stream);
  count_launch();
  if (!dispatch(HeadWidths(), ch, [&](auto CH) {
        msda_fwd_kernel<CH.value><<<grid, kMsdaThreads, 0, st>>>(
            value, spatial_shapes, level_start, loc, attw, n_items, n_value,
            heads, levels, nq, points, out);
      })) {
    const int64_t n_out = n_items * ch;
    msda_fwd_generic_kernel<<<(unsigned)ceil_div64(n_out, kMsdaThreads),
                              kMsdaThreads, 0, st>>>(
        value, spatial_shapes, level_start, loc, attw, n_out, n_value, heads,
        ch, levels, nq, points, out);
  }
  return launch_status();
}

FBBEV_API int fbbev_msda_fused_fwd(
    const float* value, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* ref, const float* offsets,
    const float* logits, int32_t bs, int32_t n_value, int32_t heads,
    int32_t ch, int32_t levels, int32_t nq, int32_t points, int32_t patch_w,
    float* out, fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0 || patch_w < 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !ref || !offsets ||
      !logits || !out)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const unsigned grid = (unsigned)ceil_div64(n_items, kMsdaThreads);
  cudaStream_t st = as_stream(stream);
  count_launch();
  if (patch_w > 0 && heads == 8 && levels == 1 && nq == n_value &&
      nq % patch_w == 0) {
    // BEV self-attention: 8 x 8 query patches (see the kernel)
    constexpr int kPatch = 8;
    const int rows = nq / patch_w;
    const dim3 pgrid((unsigned)((patch_w + kPatch - 1) / kPatch),
                     (unsigned)((rows + kPatch - 1) / kPatch), (unsigned)bs);
    if (pgrid.y <= 65535 && pgrid.z <= 65535) {
      if (!dispatch(HeadWidths(), ch, [&](auto CH) {
            msda_fused_fwd_kernel<CH.value, kPatch, kPatch>
                <<<pgrid, kPatch * kPatch * 8, 0, st>>>(
                    value, spatial_shapes, level_start, ref, offsets, logits,
                    n_items, n_value, heads, levels, nq, points, patch_w, out);
          }))
        return FBBEV_ERR_UNSUPPORTED;
      return launch_status();
    }
  }
  if (!dispatch(HeadWidths(), ch, [&](auto CH) {
        msda_fused_fwd_kernel<CH.value, 0, 0><<<grid, kMsdaThreads, 0, st>>>(
            value, spatial_shapes, level_start, ref, offsets, logits, n_items,
            n_value, heads, levels, nq, points, 0, out);
      }))
    return FBBEV_ERR_UNSUPPORTED;
  return launch_status();
}

FBBEV_API int fbbev_da_sca_fwd(
    const float* value, const float* depth_prob, const float* ref_cam,
    const float* ref_depth, const uint8_t* mask, const float* offsets,
    const float* logits, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* dbound_host, int32_t bs,
    int32_t n_cams, int32_t nq, int32_t n_value, int32_t heads, int32_t ch,
    int32_t levels, int32_t points, int32_t Z, int32_t DC, float* out,
    void* workspace, size_t workspace_bytes, int32_t prologue_done,
    fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_cams <= 0 || n_value <= 0 || heads <= 0 ||
      ch <= 0 || levels <= 0 || points <= 0 || Z <= 0 || DC <= 0 ||
      !dbound_host || points % Z != 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t n_items = (int64_t)bs * nq * heads;
  if (n_items == 0) return FBBEV_OK;
  if (!value || !depth_prob || !ref_cam || !ref_depth || !mask || !offsets ||
      !logits || !spatial_shapes || !level_start || !out)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const DaScaParams P = da_sca_params(dbound_host, bs, n_cams, nq, n_value,
                                      heads, levels, points, DC);
  const unsigned grid = (unsigned)ceil_div64(n_items, kMsdaThreads);
  cudaStream_t st = as_stream(stream);
  // whole camera map in shared memory when it fits (da_sca_smem.cu)
  if (workspace && workspace_bytes >= da_sca_smem_workspace_bytes(bs, n_cams) &&
      da_sca_smem_eligible(n_cams, n_value, heads, ch, levels, points, Z) &&
      bs * n_cams <= 4096 && (reinterpret_cast<uintptr_t>(value) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0)
    return da_sca_smem_launch(value, depth_prob, ref_cam, ref_depth, mask,
                              offsets, logits, spatial_shapes, P.d_min,
                              P.d_step, bs, n_cams, nq, n_value, DC, out,
                              workspace, st,
                              prologue_done ? kScaMain
                                            : (kScaPrologue | kScaMain));
  if (prologue_done) return FBBEV_ERR_INVALID_ARGUMENT;  // no such stage here
  count_launch();
  bool launched = false;
  dispatch(HeadWidths(), ch, [&](auto CH) {
    launched = dispatch(ZAnchors(), Z, [&](auto ZV) {
      da_sca_fwd_kernel<CH.value, ZV.value><<<grid, kMsdaThreads, 0, st>>>(
          value, depth_prob, ref_cam, ref_depth, mask, offsets, logits,
          spatial_shapes, level_start, P, out);
    });
  });
  if (!launched) return FBBEV_ERR_UNSUPPORTED;
  return launch_status();
}
