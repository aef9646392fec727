// bev_pool_fwd.cu -- forward lift-splat voxel pooling for sm_90a.
//
// Replaces (reference paths relative to the NVlabs/FB-BEV checkout):
//   bev_pool_v2_kernel + launcher   mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu:18-45, 120-128
//   bev_pool_v2_forward             mmdet3d/ops/bev_pool_v2/src/bev_pool.cpp:28-55
//   QuickCumsumCuda.forward + the permute/contiguous of bev_pool_v2()
//                                   mmdet3d/ops/bev_pool_v2/bev_pool.py:15-39, 84-90
//
//  * bev_pool_interval_kernel -- exact drop-in for the reference kernel
//    (caller-zeroed (B,Z,Y,X,C) output, arbitrary interval list).  One warp per
//    interval: the warp loads up to 32 (ranks_depth, ranks_feat, depth) triples
//    with one coalesced load each and broadcasts them by shuffle, so index and
//    depth words are read once per interval instead of once per channel
//    (reference: bev_pool_cuda.cu:37-38 re-reads them in every one of C threads).
//  * the dense op -- the op the plugin actually needs: the (B,C,Z,Y,X) volume.
//    On the shapes split_supported() accepts (every shape the model runs) it
//    is the two kernels of bev_pool_split.cu, which write every output element
//    exactly once.  Any other shape takes the interval route: the reference's
//    own sequence (zero fill + the interval kernel above) with its transpose
//    folded into the store address, so it is bit-identical to
//    QuickCumsumCuda + permute(0, 4, 1, 2, 3).
#include "bev_pool_split.h"
#include "common.cuh"

namespace fbbev {

constexpr int kPoolThreads = 256;
constexpr int kPoolWarps = kPoolThreads / kWarp;

// Sum of one interval for this lane's channels {lane, lane+32, ...}.
// Point order == reference order (bev_pool_cuda.cu:36-40), one FMA per point
// (nvcc contracts the reference's `psum += feat * depth` the same way).
template <int NCH>
__device__ __forceinline__ void interval_sum(
    const float* __restrict__ depth, const float* __restrict__ feat,
    const int* __restrict__ ranks_depth, const int* __restrict__ ranks_feat,
    int start, int len, int pitch, int cbound, int lane, float (&acc)[NCH]) {
#pragma unroll
  for (int r = 0; r < NCH; ++r) acc[r] = 0.f;
  for (int base = 0; base < len; base += kWarp) {
    const int n = min(kWarp, len - base);
    float d = 0.f;
    int rf = 0;
    if (lane < n) {
      rf = __ldg(ranks_feat + start + base + lane);
      d = __ldg(depth + __ldg(ranks_depth + start + base + lane));
    }
#pragma unroll 4
    for (int k = 0; k < n; ++k) {
      const float dk = __shfl_sync(kFull, d, k);
      const int rfk = __shfl_sync(kFull, rf, k);
      const float* f = feat + (int64_t)rfk * pitch;
#pragma unroll
      for (int r = 0; r < NCH; ++r) {
        const int ch = lane + kWarp * r;
        if (ch < cbound) acc[r] = fmaf(__ldg(f + ch), dk, acc[r]);
      }
    }
  }
}

// zyx == 0: (B,Z,Y,X,C) output (the drop-in op).  zyx > 0: (B,C,Z,Y,X) output
// of n_vox = B*zyx voxels (the dense op's interval route); ranks outside the
// volume are skipped.  n_intervals_dev (may be null): the live interval count
// on the device, capped by n_intervals.
template <int NCH>
__global__ void __launch_bounds__(kPoolThreads) bev_pool_interval_kernel(
    const float* __restrict__ depth, const float* __restrict__ feat,
    const int* __restrict__ ranks_depth, const int* __restrict__ ranks_feat,
    const int* __restrict__ ranks_bev, const int* __restrict__ interval_starts,
    const int* __restrict__ interval_lengths, int n_intervals,
    const int* __restrict__ n_intervals_dev, int c, int c0, int64_t zyx,
    int64_t n_vox, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t i =
      (int64_t)blockIdx.x * kPoolWarps + (threadIdx.x >> 5);
  const int n = n_intervals_dev ? min(__ldg(n_intervals_dev), n_intervals)
                                : n_intervals;
  if (i >= n) return;
  const int start = __ldg(interval_starts + i);
  const int len = __ldg(interval_lengths + i);
  const int rank = __ldg(ranks_bev + start);
  // c0: first channel handled by this launch (channel chunking for C > 256)
  float* o = out + (int64_t)rank * c + c0;
  int64_t ch_stride = 1;
  if (zyx > 0) {  // element (b, ch, v) at (b*C + ch)*zyx + v
    if (rank < 0 || rank >= n_vox) return;
    const int64_t b = rank / zyx;
    o = out + (b * c + c0) * zyx + (rank - b * zyx);
    ch_stride = zyx;
  }
  float acc[NCH];
  const int cc = min(c - c0, NCH * kWarp);
  interval_sum<NCH>(depth, feat + c0, ranks_depth, ranks_feat, start, len, c,
                    cc, lane, acc);
#pragma unroll
  for (int r = 0; r < NCH; ++r) {
    const int ch = lane + kWarp * r;
    if (ch < cc) o[ch * ch_stride] = acc[r];
  }
}

static int launch_intervals(const float* depth, const float* feat,
                            const int* ranks_depth, const int* ranks_feat,
                            const int* ranks_bev, const int* interval_starts,
                            const int* interval_lengths, int n_intervals,
                            const int* n_intervals_dev, int c, int64_t zyx,
                            int64_t n_vox, float* out, cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(n_intervals, kPoolWarps);
  // channels are processed in chunks of <= 256 (8 per lane)
  for (int c0 = 0; c0 < c; c0 += 256) {
    const int nch = (min(c - c0, 256) + kWarp - 1) / kWarp;
    count_launch();
#define FBBEV_INT_CASE(N)                                                     \
  bev_pool_interval_kernel<N><<<grid, kPoolThreads, 0, st>>>(                 \
      depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_starts,       \
      interval_lengths, n_intervals, n_intervals_dev, c, c0, zyx, n_vox, out)
    if (nch <= 1) FBBEV_INT_CASE(1);
    else if (nch <= 2) FBBEV_INT_CASE(2);
    else if (nch <= 3) FBBEV_INT_CASE(3);
    else if (nch <= 4) FBBEV_INT_CASE(4);
    else FBBEV_INT_CASE(8);
#undef FBBEV_INT_CASE
  }
  return launch_status();
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API int fbbev_bev_pool_v2_fwd(
    const float* depth, const float* feat, const int32_t* ranks_depth,
    const int32_t* ranks_feat, const int32_t* ranks_bev,
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals, int32_t c, float* out, fbbev_stream_t stream) {
  if (n_intervals < 0 || c <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (n_intervals == 0) return FBBEV_OK;
  if (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev ||
      !interval_starts || !interval_lengths || !out)
    return FBBEV_ERR_INVALID_ARGUMENT;
  return launch_intervals(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                          interval_starts, interval_lengths, n_intervals,
                          nullptr, c, 0, 0, out, as_stream(stream));
}

FBBEV_API size_t fbbev_bev_pool_v2_dense_workspace_bytes(
    int32_t batch, int64_t n_voxels_per_sample, int32_t n_intervals_max,
    int32_t n_points, int32_t c) {
  if (batch <= 0 || n_voxels_per_sample <= 0 || n_intervals_max < 0 ||
      n_points < 0 || c <= 0)
    return 0;
  return split_workspace_bytes(batch, n_voxels_per_sample, n_intervals_max,
                               n_points, c);
}

static int dense_check(int32_t n_intervals_max, int32_t n_points, int32_t c,
                       int32_t batch, int64_t zyx, const void* out,
                       const void* workspace, size_t workspace_bytes) {
  if (n_intervals_max < 0 || n_points < n_intervals_max || c <= 0 ||
      batch <= 0 || zyx <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!out || !workspace) return FBBEV_ERR_INVALID_ARGUMENT;
  if (workspace_bytes <
      fbbev_bev_pool_v2_dense_workspace_bytes(batch, zyx, n_intervals_max,
                                              n_points, c))
    return FBBEV_ERR_WORKSPACE_TOO_SMALL;
  return FBBEV_OK;
}

FBBEV_API int fbbev_bev_pool_v2_plan(
    const int32_t* ranks_bev, const int32_t* interval_starts,
    const int32_t* interval_lengths, int32_t n_intervals_max,
    const int32_t* n_intervals_dev, int32_t n_points, int32_t c,
    int32_t batch, int64_t n_voxels_per_sample, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = dense_check(n_intervals_max, n_points, c, batch,
                       n_voxels_per_sample, workspace, workspace,
                       workspace_bytes);
  if (rc) return rc;
  if (n_intervals_max > 0 &&
      (!ranks_bev || !interval_starts || !interval_lengths))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return split_plan(ranks_bev, interval_starts, interval_lengths,
                    n_intervals_max, n_intervals_dev, n_points, c, batch,
                    n_voxels_per_sample, workspace, as_stream(stream));
}

// ---- the dense op in stages (deferred materialisation, FBOCC glue) ---------
FBBEV_API int fbbev_bev_pool_v2_sums_planned(
    const float* depth, const float* feat, const int32_t* ranks_depth,
    const int32_t* ranks_feat, const int32_t* ranks_bev,
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, void* plan, size_t plan_bytes,
    fbbev_stream_t stream) {
  int rc = dense_check(n_intervals_max, n_points, c, batch,
                       n_voxels_per_sample, plan, plan, plan_bytes);
  if (rc) return rc;
  if (!split_supported(c, batch, n_voxels_per_sample))
    return FBBEV_ERR_UNSUPPORTED;
  if (n_intervals_max > 0 &&
      (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev ||
       !interval_starts || !interval_lengths))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return split_launch(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                      interval_starts, interval_lengths, n_intervals_max,
                      n_points, c, batch, n_voxels_per_sample, nullptr, plan,
                      as_stream(stream), kSplitSums);
}

FBBEV_API int fbbev_bev_pool_v2_zmean_planned(
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, int32_t yx, float* lss_tokens, void* plan,
    size_t plan_bytes, fbbev_stream_t stream) {
  int rc = dense_check(n_intervals_max, n_points, c, batch,
                       n_voxels_per_sample, lss_tokens, plan, plan_bytes);
  if (rc) return rc;
  if (!split_supported(c, batch, n_voxels_per_sample))
    return FBBEV_ERR_UNSUPPORTED;
  if (n_intervals_max > 0 && (!interval_starts || !interval_lengths))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return split_zmean(interval_starts, interval_lengths, n_intervals_max,
                     n_points, c, batch, n_voxels_per_sample, yx, lss_tokens,
                     plan, as_stream(stream));
}

FBBEV_API int fbbev_bev_pool_v2_write_planned(
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, int32_t yx, const float* add, float* out,
    void* plan, size_t plan_bytes, fbbev_stream_t stream) {
  int rc = dense_check(n_intervals_max, n_points, c, batch,
                       n_voxels_per_sample, out, plan, plan_bytes);
  if (rc) return rc;
  if (!split_supported(c, batch, n_voxels_per_sample))
    return FBBEV_ERR_UNSUPPORTED;
  if (n_intervals_max > 0 && (!interval_starts || !interval_lengths))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return split_launch(nullptr, nullptr, nullptr, nullptr, nullptr,
                      interval_starts, interval_lengths, n_intervals_max,
                      n_points, c, batch, n_voxels_per_sample, out, plan,
                      as_stream(stream), kSplitWrite, add, yx);
}

FBBEV_API int fbbev_bev_pool_v2_fwd_dense_planned(
    const float* depth, const float* feat, const int32_t* ranks_depth,
    const int32_t* ranks_feat, const int32_t* ranks_bev,
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, float* out, void* plan, size_t plan_bytes,
    fbbev_stream_t stream) {
  int rc = dense_check(n_intervals_max, n_points, c, batch,
                       n_voxels_per_sample, out, plan, plan_bytes);
  if (rc) return rc;
  if (n_intervals_max > 0 &&
      (!depth || !feat || !ranks_depth || !ranks_feat || !ranks_bev ||
       !interval_starts || !interval_lengths))
    return FBBEV_ERR_INVALID_ARGUMENT;
  cudaStream_t st = as_stream(stream);
  const int64_t zyx = n_voxels_per_sample;
  if (split_supported(c, batch, zyx))
    return split_launch(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                        interval_starts, interval_lengths, n_intervals_max,
                        n_points, c, batch, zyx, out, plan, st);
  // interval route: zero fill, then one warp per live interval (the count the
  // plan holds) stores its sums into the (B,C,Z,Y,X) volume
  const int64_t n_vox = (int64_t)batch * zyx;
  count_launch();
  const cudaError_t e =
      cudaMemsetAsync(out, 0, (size_t)n_vox * c * sizeof(float), st);
  if (e != cudaSuccess) return (int)e;
  if (n_intervals_max == 0) return FBBEV_OK;
  const SplitPlanPtrs pp =
      split_plan_ptrs(plan, batch, zyx, n_intervals_max, n_points, c);
  return launch_intervals(depth, feat, ranks_depth, ranks_feat, ranks_bev,
                          interval_starts, interval_lengths, n_intervals_max,
                          pp.meta, c, zyx, n_vox, out, st);
}
