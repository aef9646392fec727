// msda_common.cuh -- sampling helpers shared by the deformable-attention kernels
#pragma once
#include <type_traits>

#include "common.cuh"

namespace fbbev {

// A compile-time list of ints.  dispatch(list, v, f) calls
// f(std::integral_constant<int, v>()) when v is in the list and returns
// whether it was; contains(list, v) only asks.
template <int... Vs>
struct IntList {};
template <int... Vs>
constexpr bool contains(IntList<Vs...>, int v) {
  return ((v == Vs) || ...);
}
template <int... Vs, class F>
bool dispatch(IntList<Vs...>, int v, F&& f) {
  return ((v == Vs && (f(std::integral_constant<int, Vs>()), true)) || ...);
}

// Head widths (channels per head) and Z-anchor counts the specialised kernels
// are built for; ops/ms_deform_attn.py mirrors them as FUSED_HEAD_WIDTHS /
// FUSED_Z_ANCHORS (tests/test_fused_backward_abi.py checks that they agree)
using HeadWidths = IntList<4, 8, 10, 16, 20, 32, 64>;
using ZAnchors = IntList<1, 2, 4, 8>;
static inline bool fused_head_width(int ch) {
  return contains(HeadWidths(), ch);
}
static inline bool fused_z(int Z) { return contains(ZAnchors(), Z); }

// mmcv's in-image test of a bilinear sample: -1 < h < H and -1 < w < W
__device__ __forceinline__ bool in_image(float h_im, float w_im, int H, int W) {
  return h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W;
}

// Corner geometry of one bilinear sample, mmcv's arithmetic: corners 1..4 are
// (h_low, w_low), (h_low, w_low + 1), (h_low + 1, w_low), (h_low + 1, w_low + 1)
// with weights w1..w4; okN(H, W) tells whether corner N lies in the H x W
// image.  Every sampler and every deterministic-mode gather takes its weights
// from here, so a record's weight is the twin kernel's weight by construction.
struct Bilinear {
  int h_low, w_low;
  float lh, lw, hh, hw;
  float w1, w2, w3, w4;
  __device__ __forceinline__ Bilinear(float h_im, float w_im) {
    h_low = (int)floorf(h_im);
    w_low = (int)floorf(w_im);
    lh = h_im - (float)h_low;
    lw = w_im - (float)w_low;
    hh = 1.f - lh;
    hw = 1.f - lw;
    w1 = hh * hw;
    w2 = hh * lw;
    w3 = lh * hw;
    w4 = lh * lw;
  }
  __device__ __forceinline__ bool ok1(int, int) const {
    return h_low >= 0 && w_low >= 0;
  }
  __device__ __forceinline__ bool ok2(int, int W) const {
    return h_low >= 0 && w_low + 1 <= W - 1;
  }
  __device__ __forceinline__ bool ok3(int H, int) const {
    return h_low + 1 <= H - 1 && w_low >= 0;
  }
  __device__ __forceinline__ bool ok4(int H, int W) const {
    return h_low + 1 <= H - 1 && w_low + 1 <= W - 1;
  }
  // weight of corner k + 1
  __device__ __forceinline__ float weight(int k) const {
    return k == 0 ? w1 : k == 1 ? w2 : k == 2 ? w3 : w4;
  }
  // offset of corner 1 in a W-wide map of `stride` floats per pixel (corner 2
  // is + stride, corner 3 + W * stride, corner 4 + (W + 1) * stride)
  __device__ __forceinline__ int64_t offset(int W, int stride) const {
    return ((int64_t)h_low * W + w_low) * stride;
  }
  // top-left corner cell in the (H+1) x (W+1) grid padded by one row and
  // column before the image (h_low, w_low >= -1 for an in-image sample); the
  // key of the deterministic backward's records
  __device__ __forceinline__ int padded_cell(int W) const {
    return (h_low + 1) * (W + 1) + w_low + 1;
  }
};

// scalar bilinear (depth look-up): value laid out [pixel][stride] floats
__device__ __forceinline__ float sample_scalar(const float* __restrict__ val,
                                               int H, int W, int stride,
                                               float h_im, float w_im) {
  if (!in_image(h_im, w_im, H, W)) return 0.f;
  const Bilinear bl(h_im, w_im);
  const float* p1 = val + bl.offset(W, stride);
  float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
  if (bl.ok1(H, W)) v1 = __ldg(p1);
  if (bl.ok2(H, W)) v2 = __ldg(p1 + stride);
  if (bl.ok3(H, W)) v3 = __ldg(p1 + (int64_t)W * stride);
  if (bl.ok4(H, W)) v4 = __ldg(p1 + (int64_t)W * stride + stride);
  return bl.w1 * v1 + bl.w2 * v2 + bl.w3 * v3 + bl.w4 * v4;
}

// pixel coordinate of a normalised location: loc * size - 0.5, product rounded
// to fp32 before the subtraction exactly as in mmcv's kernel (no FMA contraction)
__device__ __forceinline__ float pix(float loc, int size) {
  return __fsub_rn(__fmul_rn(loc, (float)size), 0.5f);
}

template <int CH>
struct VecWidth {
  static constexpr int value = (CH % 4 == 0) ? 4 : ((CH % 2 == 0) ? 2 : 1);
};

template <int VW>
__device__ __forceinline__ void load_vec(const float* p, float* v);
template <>
__device__ __forceinline__ void load_vec<4>(const float* p, float* v) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p));
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <>
__device__ __forceinline__ void load_vec<2>(const float* p, float* v) {
  const float2 t = __ldg(reinterpret_cast<const float2*>(p));
  v[0] = t.x; v[1] = t.y;
}
template <>
__device__ __forceinline__ void load_vec<1>(const float* p, float* v) {
  v[0] = __ldg(p);
}

// softmax statistics of one (b,q,head) logit row of n = levels*points entries
__device__ __forceinline__ void softmax_stats(const float* __restrict__ lg,
                                              int n, float& mx, float& inv) {
  mx = -INFINITY;
  for (int i = 0; i < n; ++i) mx = fmaxf(mx, __ldg(lg + i));
  float s = 0.f;
  for (int i = 0; i < n; ++i) s += expf(__ldg(lg + i) - mx);
  inv = 1.f / s;
}

struct DaScaParams {
  float d_min, d_step;
  int bs, n_cams, nq, n_value, heads, levels, points, DC;
};

// dbound = (d_min, d_max, d_step) on the host
static inline DaScaParams da_sca_params(const float* dbound, int bs,
                                        int n_cams, int nq, int n_value,
                                        int heads, int levels, int points,
                                        int DC) {
  return DaScaParams{dbound[0], dbound[2], bs,     n_cams, nq,
                     n_value,   heads,     levels, points, DC};
}

// depth bin of an anchor's depth: clamp(floor((d - d_min) / d_step), 0, DC-1)
__device__ __forceinline__ int depth_bin(float d, float d_min, float d_step,
                                         int DC) {
  float fb = floorf(__fdiv_rn(__fsub_rn(d, d_min), d_step));
  fb = fminf(fmaxf(fb, 0.f), (float)(DC - 1));
  return (int)fb;
}

// alignment the vector loads / reductions of head width ch need
static inline bool vec_aligned(const void* p, int ch) {
  const uintptr_t a = ch % 4 == 0 ? 16 : (ch % 2 == 0 ? 8 : 4);
  return p == nullptr || (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0;
}

}  // namespace fbbev
