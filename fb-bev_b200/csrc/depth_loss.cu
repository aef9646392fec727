// depth_loss.cu -- depth supervision of the lift step: get_depth_loss of
// CM_DepthNet (mmdet3d/models/fbbev/modules/depth_net.py:396-450) and of
// LSSViewTransformerBEVDepth (mmdet3d/models/necks/view_transformer.py:
// 1036-1081), with no host synchronisation.
//
// The reference permutes the whole gt map into (pixel, ds*ds) rows, takes the
// row minimum, one-hot encodes a bin index into an int64 (pixels, D + 1)
// tensor, gathers the foreground rows of labels and predictions with two
// boolean masks (one host sync each), normalises by max(1.0, fg_mask.sum())
// (a third sync) and runs binary_cross_entropy.  Here:
//
//   fwd      one CTA per (image, output row): the ds input rows are read
//            coalesced into per-column minima in shared memory, each output
//            pixel takes the minimum of its ds columns and its class
//            c in [0, D]; the CTA then gathers the D predictions of its
//            foreground pixels (bin-major, so a warp reads consecutive
//            pixels of one bin) and writes one (sum, count) partial.
//   finish   one CTA adds the partials in a fixed order and writes loss and
//            n_fg.  No float atomics: the result does not depend on
//            scheduling, and a row's partial depends on that row alone.
//   bwd      dense d preds, zero at background pixels, one pass.
//
// Arithmetic (each step the fp32 operation torch's CUDA kernels perform):
//   m = min over the patch of (g == 0 ? 1e5 : g), NaN propagating (torch.min)
//   t = (m - c0) * (1 / c1)   -- torch's CUDA true division by a CPU scalar
//                                multiplies by the scalar's fp32 reciprocal
//   c = (t >= 0 && t < D + 1) ? trunc(t) : 0;  foreground: c >= 1, y = [d == c-1]
//   loss element: -max(log p, -100) where y = 1, -max(log1p(-p), -100) else
//   d p = ((g * weight) / n) * (p - y) / max((1 - p) * p, 1e-12)
// The clamps are `a < b ? b : a` (std::max), so a NaN propagates as in torch.
#include "common.cuh"

namespace fbbev {

constexpr int kFwdThreads = 256;
constexpr int kFinishThreads = 512;
constexpr int kBwdThreads = 256;

struct DepthLossFwdParams {
  const float* gt;      // (BN, H, W)
  const float* preds;   // (BN, D, h, w); NULL: labels only
  int32_t* labels;      // (BN, h, w)
  double* part_sum;     // (BN * h)
  int32_t* part_cnt;    // (BN * h)
  int H, W, ds, h, w, D;
  int vec4;
  float c0, inv_c1;
};

__device__ __forceinline__ float patch_value(float g) {
  return g == 0.f ? 1e5f : g;
}
__device__ __forceinline__ float4 patch_value(float4 g) {
  return make_float4(patch_value(g.x), patch_value(g.y), patch_value(g.z),
                     patch_value(g.w));
}

// torch.min semantics: a NaN operand makes the result NaN.
__device__ __forceinline__ float min_nan(float a, float b) {
  return (b < a || b != b) ? b : a;
}

__global__ void __launch_bounds__(kFwdThreads)
depth_loss_fwd_kernel(DepthLossFwdParams P) {
  extern __shared__ float4 s_dyn[];              // 16-byte aligned
  float* s_col = reinterpret_cast<float*>(s_dyn); // W column minima, then w labels
  __shared__ double s_sum[kFwdThreads / kWarp];
  __shared__ int s_cnt[kFwdThreads / kWarp];
  const int row = blockIdx.x;                    // n * h + y
  const int n = row / P.h, y = row % P.h;
  const int tid = threadIdx.x;
  const float* src = P.gt + ((int64_t)n * P.H + (int64_t)y * P.ds) * P.W;
  if (P.vec4) {   // W % 4 == 0 and gt 16-byte aligned: 4 columns per load
    const int W4 = P.W >> 2;
    const float4* src4 = reinterpret_cast<const float4*>(src);
    for (int c4 = tid; c4 < W4; c4 += kFwdThreads) {
      float4 m = patch_value(__ldg(src4 + c4));
#pragma unroll 8
      for (int r = 1; r < P.ds; ++r) {
        const float4 v = patch_value(__ldg(src4 + (int64_t)r * W4 + c4));
        m = make_float4(min_nan(m.x, v.x), min_nan(m.y, v.y), min_nan(m.z, v.z),
                        min_nan(m.w, v.w));
      }
      reinterpret_cast<float4*>(s_col)[c4] = m;
    }
  } else {
    for (int col = tid; col < P.W; col += kFwdThreads) {
      float m = patch_value(__ldg(src + col));
#pragma unroll 8
      for (int r = 1; r < P.ds; ++r)
        m = min_nan(m, patch_value(__ldg(src + (int64_t)r * P.W + col)));
      s_col[col] = m;
    }
  }
  __syncthreads();
  int* s_lab = reinterpret_cast<int*>(s_col + P.W);
  int fg = 0;
  for (int x = tid; x < P.w; x += kFwdThreads) {
    float m = s_col[x * P.ds];
    for (int j = 1; j < P.ds; ++j) m = min_nan(m, s_col[x * P.ds + j]);
    const float t = __fmul_rn(__fsub_rn(m, P.c0), P.inv_c1);
    const int c = (t >= 0.f && t < (float)(P.D + 1)) ? (int)t : 0;
    s_lab[x] = c;
    P.labels[(int64_t)row * P.w + x] = c;
    fg += c > 0;
  }
  if (P.preds == nullptr) return;
  __syncthreads();
  // bin-major walk: element e = d * w + x
  double sum = 0.0;
  const float* pr = P.preds + ((int64_t)n * P.D * P.h + y) * P.w;
  const int64_t bin_stride = (int64_t)P.h * P.w;
  const int n_el = P.D * P.w;
  for (int e = tid; e < n_el; e += kFwdThreads) {
    const int d = e / P.w, x = e - d * P.w;
    const int c = s_lab[x];
    if (c == 0) continue;
    const float p = __ldg(pr + d * bin_stride + x);
    float v;
    if (d == c - 1) {
      v = logf(p);
    } else {
      v = log1pf(-p);
    }
    v = v < -100.f ? -100.f : v;
    sum += (double)(-v);
  }
  // fixed-order block reduction
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_down_sync(kFull, sum, o);
    fg += __shfl_down_sync(kFull, fg, o);
  }
  const int lane = tid & 31, warp = tid >> 5;
  if (lane == 0) { s_sum[warp] = sum; s_cnt[warp] = fg; }
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    int k = 0;
    for (int i = 0; i < kFwdThreads / kWarp; ++i) { s += s_sum[i]; k += s_cnt[i]; }
    P.part_sum[row] = s;
    P.part_cnt[row] = k;
  }
}

__global__ void __launch_bounds__(kFinishThreads)
depth_loss_finish_kernel(const double* part_sum, const int32_t* part_cnt,
                         int rows, float weight, float* loss, int32_t* n_fg) {
  __shared__ double s_sum[kFinishThreads / kWarp];
  __shared__ long long s_cnt[kFinishThreads / kWarp];
  const int tid = threadIdx.x;
  double sum = 0.0;
  long long cnt = 0;
  for (int i = tid; i < rows; i += kFinishThreads) {
    sum += part_sum[i];
    cnt += part_cnt[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_down_sync(kFull, sum, o);
    cnt += __shfl_down_sync(kFull, cnt, o);
  }
  const int lane = tid & 31, warp = tid >> 5;
  if (lane == 0) { s_sum[warp] = sum; s_cnt[warp] = cnt; }
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    long long k = 0;
    for (int i = 0; i < kFinishThreads / kWarp; ++i) { s += s_sum[i]; k += s_cnt[i]; }
    const float nf = (float)(k > 1 ? k : 1);
    *loss = __fmul_rn(__fdiv_rn((float)s, nf), weight);
    *n_fg = (int32_t)k;
  }
}

struct DepthLossBwdParams {
  const int32_t* labels;  // (BN, hw)
  const float* preds;     // (BN, D, hw)
  const int32_t* n_fg;
  const float* grad_loss;
  float* grad_preds;      // (BN, D, hw)
  int rows;               // BN * D
  int hw, D;
  float weight;
};

// blockIdx.x: a chunk of pixels, blockIdx.y (strided): an (image, bin) row
__global__ void __launch_bounds__(kBwdThreads)
depth_loss_bwd_kernel(DepthLossBwdParams P) {
  const int nf = *P.n_fg;
  const float k = __fdiv_rn(__fmul_rn(*P.grad_loss, P.weight),
                            (float)(nf > 1 ? nf : 1));
  const int px = blockIdx.x * kBwdThreads + threadIdx.x;
  if (px >= P.hw) return;
  for (int row = blockIdx.y; row < P.rows; row += gridDim.y) {
    const int n = row / P.D, d = row - n * P.D;
    const int c = __ldg(P.labels + (int64_t)n * P.hw + px);
    const int64_t i = (int64_t)row * P.hw + px;
    float g = 0.f;
    if (c > 0) {
      const float p = __ldg(P.preds + i);
      const float yv = d == c - 1 ? 1.f : 0.f;
      float den = __fmul_rn(__fsub_rn(1.f, p), p);
      den = den < 1e-12f ? 1e-12f : den;
      g = __fdiv_rn(__fmul_rn(k, __fsub_rn(p, yv)), den);
    }
    st_stream(P.grad_preds + i, g);
  }
}

static bool misaligned(const void* p, size_t a) {
  return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0;
}

static size_t part_sum_bytes(int64_t rows) { return (size_t)(rows * 8 + 15) / 16 * 16; }

}  // namespace fbbev

using namespace fbbev;

FBBEV_API size_t fbbev_depth_loss_workspace_bytes(int32_t bn, int32_t H,
                                                  int32_t ds) {
  if (bn < 0 || H < 0 || ds <= 0) return 0;
  const int64_t rows = (int64_t)bn * (H / ds);
  return part_sum_bytes(rows) + (size_t)rows * 4;
}

FBBEV_API int fbbev_depth_loss_fwd(const float* gt, const float* preds,
                                   int32_t bn, int32_t H, int32_t W, int32_t ds,
                                   int32_t d, float c0, float c1, float weight,
                                   int32_t* labels, float* loss, int32_t* n_fg,
                                   void* workspace, size_t workspace_bytes,
                                   fbbev_stream_t stream) {
  if (bn < 0 || H <= 0 || W <= 0 || ds <= 0 || d <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (H % ds != 0 || W % ds != 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (bn == 0) return FBBEV_OK;
  if (!gt || !labels || misaligned(gt, 4) || misaligned(labels, 4))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const bool labels_only = preds == nullptr;
  if (labels_only ? (loss || n_fg)
                  : (!loss || !n_fg || misaligned(preds, 4) || misaligned(loss, 4) ||
                     misaligned(n_fg, 4)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int h = H / ds, w = W / ds;
  const int64_t rows = (int64_t)bn * h;
  if (!labels_only) {
    if (workspace_bytes < fbbev_depth_loss_workspace_bytes(bn, H, ds))
      return FBBEV_ERR_WORKSPACE_TOO_SMALL;
    if (!workspace || misaligned(workspace, 16)) return FBBEV_ERR_INVALID_ARGUMENT;
  }
  const size_t smem = (size_t)W * 4 + (size_t)w * 4;
  if (smem > 48 * 1024 || rows > INT32_MAX || (int64_t)d * h * w > INT32_MAX)
    return FBBEV_ERR_UNSUPPORTED;
  DepthLossFwdParams P;
  P.gt = gt; P.preds = preds; P.labels = labels;
  P.part_sum = labels_only ? nullptr : static_cast<double*>(workspace);
  P.part_cnt = labels_only ? nullptr : reinterpret_cast<int32_t*>(
      static_cast<char*>(workspace) + part_sum_bytes(rows));
  P.H = H; P.W = W; P.ds = ds; P.h = h; P.w = w; P.D = d;
  P.vec4 = W % 4 == 0 && !misaligned(gt, 16);
  P.c0 = c0; P.inv_c1 = 1.f / c1;
  count_launch();
  depth_loss_fwd_kernel<<<(unsigned)rows, kFwdThreads, smem, as_stream(stream)>>>(P);
  int rc = launch_status();
  if (rc != FBBEV_OK || labels_only) return rc;
  count_launch();
  depth_loss_finish_kernel<<<1, kFinishThreads, 0, as_stream(stream)>>>(
      P.part_sum, P.part_cnt, (int)rows, weight, loss, n_fg);
  return launch_status();
}

FBBEV_API int fbbev_depth_loss_bwd(const int32_t* labels, const float* preds,
                                   const int32_t* n_fg, const float* grad_loss,
                                   int32_t bn, int32_t h, int32_t w, int32_t d,
                                   float weight, float* grad_preds,
                                   fbbev_stream_t stream) {
  if (bn < 0 || h <= 0 || w <= 0 || d <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (bn == 0) return FBBEV_OK;
  if (!labels || !preds || !n_fg || !grad_loss || !grad_preds ||
      misaligned(labels, 4) || misaligned(preds, 4) || misaligned(n_fg, 4) ||
      misaligned(grad_loss, 4) || misaligned(grad_preds, 4))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int64_t hw = (int64_t)h * w;
  if (hw > INT32_MAX || (int64_t)d * hw > INT32_MAX) return FBBEV_ERR_UNSUPPORTED;
  if ((int64_t)bn * d > INT32_MAX) return FBBEV_ERR_UNSUPPORTED;
  DepthLossBwdParams P;
  P.labels = labels; P.preds = preds; P.n_fg = n_fg; P.grad_loss = grad_loss;
  P.grad_preds = grad_preds; P.rows = bn * d; P.hw = (int)hw; P.D = d;
  P.weight = weight;
  const dim3 grid((unsigned)ceil_div64(hw, kBwdThreads),
                  (unsigned)(P.rows < 65535 ? P.rows : 65535));
  count_launch();
  depth_loss_bwd_kernel<<<grid, kBwdThreads, 0, as_stream(stream)>>>(P);
  return launch_status();
}
