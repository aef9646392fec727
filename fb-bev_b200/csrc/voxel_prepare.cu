// voxel_prepare.cu -- device implementation of voxel_pooling_prepare_v2.
//
// Replaces  mmdet3d/models/fbbev/view_transformation/forward_projection/
//           view_transformer.py:547-605
// (about 25 eager PyTorch ops, a radix sort of ~2e5 keys, three boolean-mask
// compactions and three host synchronisations per forward) with a counting
// sort over voxel ranks that never leaves the device:
//
//   K1 voxelize   rank[p] = voxel rank of point p or -1; hist[rank]++      (:570-589)
//   K2 scan       offset[v] = exclusive prefix of hist; interval list =
//                 occupied voxels in rank order                             (:594-602)
//   K3 scatter    bucket[offset[r] + atomic slot] = p                       (:590-592)
//   K4 order      inside each voxel, place points in ascending point index
//                 (deterministic; == a stable argsort) and emit ranks_bev /
//                 ranks_depth / ranks_feat                                  (:561-568, :603-605)
//
// Integer-path parity rules (SURVEY.md appendix A):
//   * voxelisation is fp32 subtract, fp32 IEEE divide, truncation toward zero
//     (`.long()`), so coordinates in (-1, 0) land in cell 0 and are kept;
//   * the bounds test compares the integer coordinate, converted to float32,
//     against the FLOAT32 grid size;
//   * the rank is formed in exact integer arithmetic (the reference's float32
//     arithmetic is identical below 2^24 voxels and wrong above).
#include <algorithm>

#include "bev_pool_split.h"
#include "common.cuh"

namespace fbbev {

constexpr int kPrepThreads = 256;
constexpr int kScanItems = 8;                       // per thread
constexpr int kScanTile = kPrepThreads * kScanItems;  // per block

struct GridParams {
  float lo[3], iv[3], gs[3];
  int gx, gy, gz;
  // depth-threshold sparsification of the BEVDet lineage
  // (necks/view_transformer.py:556-557: kept &= depth.view(-1) > 0.01); the
  // depth tensor is indexed by the point index itself (ranks_depth == arange)
  const float* depth_prob;  // null: keep every in-grid point
  float depth_thresh;
};

// `.long()` of the CUDA device the reference runs on: cvt.rzi.s64.f32
__device__ __forceinline__ long long trunc_i64(float f) {
  return static_cast<long long>(f);
}

__device__ __forceinline__ void voxelize_point(float x, float y, float z,
                                               int64_t p, int64_t per_b,
                                               const GridParams& g,
                                               int* __restrict__ rank,
                                               int* __restrict__ hist) {
  // __fsub_rn / __fdiv_rn: IEEE round-to-nearest, never contracted or
  // replaced by a reciprocal multiply
  const long long cx = trunc_i64(__fdiv_rn(__fsub_rn(x, g.lo[0]), g.iv[0]));
  const long long cy = trunc_i64(__fdiv_rn(__fsub_rn(y, g.lo[1]), g.iv[1]));
  const long long cz = trunc_i64(__fdiv_rn(__fsub_rn(z, g.lo[2]), g.iv[2]));
  const bool keep = cx >= 0 && (float)cx < g.gs[0] && cy >= 0 &&
                    (float)cy < g.gs[1] && cz >= 0 && (float)cz < g.gs[2] &&
                    cx < g.gx && cy < g.gy && cz < g.gz &&
                    (g.depth_prob == nullptr ||
                     __ldg(g.depth_prob + p) > g.depth_thresh);
  int r = -1;
  if (keep) {
    const int64_t b = (unsigned)p / (unsigned)per_b;   // p, per_b < 2^31
    r = (int)(((b * g.gz + cz) * g.gy + cy) * g.gx + cx);
    atomicAdd(hist + r, 1);
  }
  rank[p] = r;
}

__global__ void __launch_bounds__(kPrepThreads) prep_voxelize_kernel(
    const float* __restrict__ coor, int64_t n_pts, int64_t per_b, GridParams g,
    int* __restrict__ rank, int* __restrict__ hist) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  voxelize_point(__ldg(coor + 3 * p + 0), __ldg(coor + 3 * p + 1),
                 __ldg(coor + 3 * p + 2), p, per_b, g, rank, hist);
}

// Same, but the ego-frame coordinate of point (b, n, d, h, w) is evaluated here
// from the camera matrices instead of being read from a materialised
// (B,N,D,H,W,3) tensor: get_lidar_coor (view_transformer.py:458-498) fused into
// the voxelisation.  The chain is the reference's --
//   p = frustum - post_trans;  p = inv(post_rots) p;  p = (p.x p.z, p.y p.z, p.z);
//   p = (rots inv(K)) p + trans;  p = bda p
// -- in fp32, every 3x3 product in the rounding order torch's broadcast matmul
// has on this device (mat3_apply_ref, common.cuh), so the coordinate -- and the
// voxel it truncates into -- is bit-identical to the eager chain's
// (tests/test_forward_gpu.py::test_fused_geometry_bit_exact).
struct CamGeom {
  const float* us;      // [W]  frustum u (linspace over the input width)
  const float* vs;      // [H]  frustum v
  const float* ds;      // [D]  frustum depth bins
  const float* ipr;     // [B*N][9] inverse(post_rots)
  const float* ptr;     // [B*N][3] post_trans
  const float* comb;    // [B*N][9] rots @ inverse(intrins)
  const float* trn;     // [B*N][3] trans
  const float* bda;     // [B][9]
  int N, D, H, W;
  int order;            // FBBEV_ORDER_SEQ_* bits (see include/fbbev_b200.h)
};

__global__ void __launch_bounds__(kPrepThreads) prep_voxelize_cams_kernel(
    CamGeom cg, int64_t n_pts, int64_t per_b, GridParams g,
    int* __restrict__ rank, int* __restrict__ hist) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  // n_pts < 2^31 (checked by the entry point): 32-bit divisions
  const unsigned pu = (unsigned)p;
  const int w = (int)(pu % (unsigned)cg.W);
  unsigned t = pu / (unsigned)cg.W;
  const int h = (int)(t % (unsigned)cg.H);
  t /= (unsigned)cg.H;
  const int d = (int)(t % (unsigned)cg.D);
  const int64_t bn = t / (unsigned)cg.D;
  const int64_t b = (unsigned)bn / (unsigned)cg.N;
  const float* pt = cg.ptr + bn * 3;
  float x = __fsub_rn(__ldg(cg.us + w), __ldg(pt + 0));
  float y = __fsub_rn(__ldg(cg.vs + h), __ldg(pt + 1));
  float z = __fsub_rn(__ldg(cg.ds + d), __ldg(pt + 2));
  float a, bb, c;
  mat3_apply_ref(cg.ipr + bn * 9, x, y, z, (cg.order & 1) != 0, a, bb, c);
  x = __fmul_rn(a, c);
  y = __fmul_rn(bb, c);
  z = c;
  mat3_apply_ref(cg.comb + bn * 9, x, y, z, (cg.order & 2) != 0, a, bb, c);
  const float* tr = cg.trn + bn * 3;
  a = __fadd_rn(a, __ldg(tr + 0));
  bb = __fadd_rn(bb, __ldg(tr + 1));
  c = __fadd_rn(c, __ldg(tr + 2));
  mat3_apply_ref(cg.bda + b * 9, a, bb, c, (cg.order & 4) != 0, x, y, z);
  voxelize_point(x, y, z, p, per_b, g, rank, hist);
}

// ----- two-quantity exclusive scan over hist: (points, occupied voxels) -----
__device__ __forceinline__ int2 warp_incl_scan(int2 v, int lane) {
#pragma unroll
  for (int o = 1; o < kWarp; o <<= 1) {
    const int a = __shfl_up_sync(kFull, v.x, o);
    const int b = __shfl_up_sync(kFull, v.y, o);
    if (lane >= o) {
      v.x += a;
      v.y += b;
    }
  }
  return v;
}

// inclusive block scan of one int2 per thread; returns block total
__device__ __forceinline__ int2 block_incl_scan(int2& v, int2* wsum) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_incl_scan(v, lane);
  if (lane == 31) wsum[warp] = v;
  __syncthreads();
  if (warp == 0) {
    int2 w = lane < kPrepThreads / kWarp ? wsum[lane] : make_int2(0, 0);
    w = warp_incl_scan(w, lane);
    if (lane < kPrepThreads / kWarp) wsum[lane] = w;
  }
  __syncthreads();
  if (warp > 0) {
    v.x += wsum[warp - 1].x;
    v.y += wsum[warp - 1].y;
  }
  const int2 total = wsum[kPrepThreads / kWarp - 1];
  __syncthreads();
  return total;
}

__global__ void __launch_bounds__(kPrepThreads) prep_scan_reduce_kernel(
    const int* __restrict__ hist, int64_t n_vox, int2* __restrict__ block_sums) {
  __shared__ int2 wsum[kPrepThreads / kWarp];
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  int2 v = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + (int64_t)k * kPrepThreads + threadIdx.x;
    if (i < n_vox) {
      const int h = hist[i];
      v.x += h;
      v.y += h > 0;
    }
  }
  const int2 total = block_incl_scan(v, wsum);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// Plan tables of the dense pooling op (bev_pool_split.cu), filled here when a
// pooling workspace is handed to the index builder: the scan below already
// knows, for every voxel, how many intervals and points precede it --
//   tile_first[t] = intervals before the tile's first voxel,
//   seg_rank[i]   = voxel rank of interval i (the voxel index itself),
//   warp_first[w] = first interval starting at or after point 32 w
// -- which is all split_plan_kernel computes (with a binary search per slice
// and a gap fill per interval) in a launch of its own.
struct PlanOut {
  int *tile_first, *seg_rank, *warp_first, *meta;  // tile_first == null: off
  int T, tiles_per_b, n_warps_max;
  int64_t zyx, n_tiles;
};

// Exclusive prefix of the block totals is formed by every block itself (<= a
// few hundred int2 per block), which removes the single-block spine launch;
// the last block also publishes the totals: counts = {n_kept, n_intervals}.
__global__ void __launch_bounds__(kPrepThreads) prep_scan_apply_kernel(
    const int* __restrict__ hist, int64_t n_vox,
    const int2* __restrict__ block_sums, int* __restrict__ offset,
    int* __restrict__ interval_starts, int* __restrict__ interval_lengths,
    int* __restrict__ counts, PlanOut plan) {
  __shared__ int2 wsum[kPrepThreads / kWarp];
  __shared__ int2 s_prefix;
  {  // prefix of the totals of the blocks before this one
    int2 acc = make_int2(0, 0);
    for (int j = threadIdx.x; j < (int)blockIdx.x; j += kPrepThreads) {
      const int2 t = block_sums[j];
      acc.x += t.x;
      acc.y += t.y;
    }
    const int2 tot = block_incl_scan(acc, wsum);
    if (threadIdx.x == 0) s_prefix = tot;
    __syncthreads();
  }
  const int2 bs = s_prefix;
  // blocked arrangement: thread t owns kScanItems consecutive voxels
  const int64_t base =
      (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  int h[kScanItems];
  int2 v = make_int2(0, 0);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + k;
    h[k] = i < n_vox ? hist[i] : 0;
    v.x += h[k];
    v.y += h[k] > 0;
  }
  const int2 mine = v;
  const int2 block_total = block_incl_scan(v, wsum);
  int run_pts = bs.x + v.x - mine.x;  // exclusive prefix for this thread
  int run_int = bs.y + v.y - mine.y;
  const bool planned = plan.tile_first != nullptr;
  // sample / in-sample voxel of the thread's first item: ONE 64-bit division
  // per thread, then counted along (the tile size is a power of two); the
  // per-item divisions cost 11 us of a 43 us index build
  int64_t pb = 0, plocal = 0;
  if (planned && base < n_vox) {
    pb = base / plan.zyx;
    plocal = base - pb * plan.zyx;
  }
  const int t_mask = plan.T - 1, t_shift = 31 - __clz(plan.T);
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    const int64_t i = base + k;
    if (i < n_vox) {
      offset[i] = run_pts;
      if (planned) {
        if (((int)plocal & t_mask) == 0)
          plan.tile_first[pb * plan.tiles_per_b + (plocal >> t_shift)] = run_int;
        if (++plocal == plan.zyx) { plocal = 0; ++pb; }
      }
      if (h[k] > 0) {
        interval_starts[run_int] = run_pts;   // view_transformer.py:597
        interval_lengths[run_int] = h[k];     // :599-602
        if (planned) {
          plan.seg_rank[run_int] = (int)i;
          // slices w with run_pts < 32 w <= run_pts + h start inside or right
          // after this interval: the first interval at or after them is the
          // next one; a slice that starts exactly here gets this one
          if (run_pts % kWarp == 0 && run_pts / kWarp <= plan.n_warps_max)
            plan.warp_first[run_pts / kWarp] = run_int;
          for (int w = run_pts / kWarp + 1;
               w * kWarp <= run_pts + h[k] && w <= plan.n_warps_max; ++w)
            if (w * kWarp > run_pts && w * kWarp < run_pts + h[k])
              plan.warp_first[w] = run_int + 1;
        }
        run_int++;
      }
      run_pts += h[k];
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    const int n_kept = bs.x + block_total.x, n_int = bs.y + block_total.y;
    counts[0] = n_kept;
    counts[1] = n_int;
    if (planned) {
      const int n_warps = min((n_kept + kWarp - 1) / kWarp, plan.n_warps_max);
      plan.meta[0] = n_int;
      plan.meta[1] = n_kept;
      plan.meta[2] = n_warps;
      plan.tile_first[plan.n_tiles] = n_int;
      plan.warp_first[n_warps] = n_int;  // slices at / past the last point
      if (n_int == 0) plan.warp_first[0] = 0;
    }
  }
}

__global__ void __launch_bounds__(kPrepThreads) prep_scatter_kernel(
    const int* __restrict__ rank, int64_t n_pts, const int* __restrict__ offset,
    int* __restrict__ cursor, int* __restrict__ bucket) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n_pts) return;
  const int r = rank[p];
  if (r < 0) return;
  const int s = atomicAdd(cursor + r, 1);
  bucket[offset[r] + s] = (int)p;
}

// One thread per kept point: its final position inside its voxel's run is the
// number of bucket mates with a smaller point index.
__global__ void __launch_bounds__(kPrepThreads) prep_order_kernel(
    const int* __restrict__ bucket, const int* __restrict__ rank,
    const int* __restrict__ offset, const int* __restrict__ hist,
    const int* __restrict__ counts, int D, int64_t hw,
    int* __restrict__ ranks_bev, int* __restrict__ ranks_depth,
    int* __restrict__ ranks_feat) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= counts[0]) return;
  const int p = bucket[j];
  const int r = rank[p];
  const int s = offset[r];
  const int len = hist[r];
  int pos = 0;
  for (int k = 0; k < len; ++k) pos += bucket[s + k] < p;
  const int dst = s + pos;
  ranks_bev[dst] = r;
  ranks_depth[dst] = p;  // arange(num_points), view_transformer.py:561-562
  // arange(num_points // D).reshape(B,N,1,H,W).expand(B,N,D,H,W), :563-568
  const unsigned bn = (unsigned)p / (unsigned)(D * hw);   // D * hw <= n_pts < 2^31
  ranks_feat[dst] = (int)(bn * (unsigned)hw + (unsigned)p % (unsigned)hw);
}

struct PrepWorkspace {
  int* rank;      // [n_pts]
  int* bucket;    // [n_pts]
  int* hist;      // [n_vox]
  int* cursor;    // [n_vox]   (hist and cursor are contiguous: one memset)
  int* offset;    // [n_vox]
  int2* block_sums;  // [n_scan_blocks]
};

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t prep_layout(int64_t n_pts, int64_t n_vox, char* base,
                          PrepWorkspace* w) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes, 256);
    return p;
  };
  const int64_t n_scan_blocks = ceil_div64(n_vox, kScanTile);
  char* rank = take((size_t)n_pts * 4);
  char* bucket = take((size_t)n_pts * 4);
  char* hist = take((size_t)n_vox * 2 * 4);  // hist | cursor
  char* offset = take((size_t)n_vox * 4);
  char* bsum = take((size_t)n_scan_blocks * sizeof(int2));
  if (w) {
    w->rank = reinterpret_cast<int*>(rank);
    w->bucket = reinterpret_cast<int*>(bucket);
    w->hist = reinterpret_cast<int*>(hist);
    w->cursor = w->hist + n_vox;
    w->offset = reinterpret_cast<int*>(offset);
    w->block_sums = reinterpret_cast<int2*>(bsum);
  }
  return off;
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API size_t fbbev_voxel_prepare_workspace_bytes(int64_t n_points,
                                                     int64_t n_voxels_total) {
  if (n_points <= 0 || n_voxels_total <= 0) return 0;
  return prep_layout(n_points, n_voxels_total, nullptr, nullptr);
}

// coor != NULL: voxelise the given coordinates; else evaluate them from *cg.
static int voxel_prepare_impl(
    const float* coor, const CamGeom* cg, int32_t B, int32_t N, int32_t D,
    int32_t H, int32_t W, const float* lo_host, const float* iv_host,
    const float* gs_host, int32_t* ranks_bev, int32_t* ranks_depth,
    int32_t* ranks_feat, int32_t* interval_starts, int32_t* interval_lengths,
    int32_t* counts, void* workspace, size_t workspace_bytes,
    int32_t pool_c, void* pool_plan, size_t pool_plan_bytes,
    const float* depth_prob, float depth_thresh, fbbev_stream_t stream) {
  if (B <= 0 || N <= 0 || D <= 0 || H <= 0 || W <= 0 || !lo_host || !iv_host ||
      !gs_host)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((!coor && !cg) || !ranks_bev || !ranks_depth || !ranks_feat ||
      !interval_starts || !interval_lengths || !counts || !workspace)
    return FBBEV_ERR_INVALID_ARGUMENT;
  GridParams g;
  for (int k = 0; k < 3; ++k) {
    g.lo[k] = lo_host[k];
    g.iv[k] = iv_host[k];
    g.gs[k] = gs_host[k];
    if (!(gs_host[k] >= 1.f) || gs_host[k] > 1e9f)
      return FBBEV_ERR_INVALID_ARGUMENT;
  }
  g.gx = (int)gs_host[0];  // int(self.grid_size[i]), view_transformer.py:537-538
  g.gy = (int)gs_host[1];
  g.gz = (int)gs_host[2];
  g.depth_prob = depth_prob;
  g.depth_thresh = depth_thresh;
  const int64_t n_pts = (int64_t)B * N * D * H * W;
  const int64_t n_vox = (int64_t)B * g.gx * g.gy * g.gz;
  if (n_pts > INT32_MAX || n_vox > INT32_MAX) return FBBEV_ERR_UNSUPPORTED;
  PrepWorkspace w;
  const size_t need =
      prep_layout(n_pts, n_vox, static_cast<char*>(workspace), &w);
  if (workspace_bytes < need) return FBBEV_ERR_WORKSPACE_TOO_SMALL;
  PlanOut plan;
  plan.tile_first = nullptr;
  if (pool_plan) {
    const int64_t zyx = (int64_t)g.gx * g.gy * g.gz;
    const int cap = (int)std::min<int64_t>(n_pts, n_vox);
    if (pool_c <= 0) return FBBEV_ERR_UNSUPPORTED;
    if (pool_plan_bytes < fbbev_bev_pool_v2_dense_workspace_bytes(
                              B, zyx, cap, (int32_t)n_pts, pool_c))
      return FBBEV_ERR_WORKSPACE_TOO_SMALL;
    const SplitPlanPtrs pp =
        split_plan_ptrs(pool_plan, B, zyx, cap, (int)n_pts, pool_c);
    plan.tile_first = pp.tile_first; plan.seg_rank = pp.seg_rank;
    plan.warp_first = pp.warp_first; plan.meta = pp.meta;
    plan.T = pp.T; plan.tiles_per_b = pp.tiles_per_b;
    plan.n_warps_max = pp.n_warps_max;
    plan.zyx = zyx; plan.n_tiles = pp.n_tiles;
  }
  cudaStream_t st = as_stream(stream);

  cudaError_t e = cudaMemsetAsync(w.hist, 0, (size_t)n_vox * 2 * 4, st);
  if (e != cudaSuccess) return (int)e;
  const unsigned pt_grid = (unsigned)ceil_div64(n_pts, kPrepThreads);
  const int n_scan_blocks = (int)ceil_div64(n_vox, kScanTile);
  count_launch(5);
  if (coor)
    prep_voxelize_kernel<<<pt_grid, kPrepThreads, 0, st>>>(
        coor, n_pts, (int64_t)N * D * H * W, g, w.rank, w.hist);
  else
    prep_voxelize_cams_kernel<<<pt_grid, kPrepThreads, 0, st>>>(
        *cg, n_pts, (int64_t)N * D * H * W, g, w.rank, w.hist);
  prep_scan_reduce_kernel<<<n_scan_blocks, kPrepThreads, 0, st>>>(
      w.hist, n_vox, w.block_sums);
  prep_scan_apply_kernel<<<n_scan_blocks, kPrepThreads, 0, st>>>(
      w.hist, n_vox, w.block_sums, w.offset, interval_starts,
      interval_lengths, counts, plan);
  prep_scatter_kernel<<<pt_grid, kPrepThreads, 0, st>>>(
      w.rank, n_pts, w.offset, w.cursor, w.bucket);
  prep_order_kernel<<<pt_grid, kPrepThreads, 0, st>>>(
      w.bucket, w.rank, w.offset, w.hist, counts, D, (int64_t)H * W, ranks_bev,
      ranks_depth, ranks_feat);
  return launch_status();
}

FBBEV_API int fbbev_voxel_prepare(
    const float* coor, const float* depth_prob, float depth_thresh, int32_t B,
    int32_t N, int32_t D, int32_t H, int32_t W, const float* lo_host,
    const float* iv_host, const float* gs_host, int32_t* ranks_bev,
    int32_t* ranks_depth, int32_t* ranks_feat, int32_t* interval_starts,
    int32_t* interval_lengths, int32_t* counts, void* workspace,
    size_t workspace_bytes, int32_t pool_c, void* pool_plan,
    size_t pool_plan_bytes, fbbev_stream_t stream) {
  if (!coor) return FBBEV_ERR_INVALID_ARGUMENT;
  return voxel_prepare_impl(coor, nullptr, B, N, D, H, W, lo_host, iv_host,
                            gs_host, ranks_bev, ranks_depth, ranks_feat,
                            interval_starts, interval_lengths, counts,
                            workspace, workspace_bytes, pool_c, pool_plan,
                            pool_plan_bytes, depth_prob, depth_thresh, stream);
}

FBBEV_API int fbbev_voxel_prepare_cams(
    const float* frustum_u, const float* frustum_v, const float* frustum_d,
    const float* inv_post_rots, const float* post_trans, const float* cam2ego,
    const float* trans, const float* bda, int32_t order_flags,
    const float* depth_prob, float depth_thresh, int32_t B, int32_t N,
    int32_t D, int32_t H, int32_t W, const float* lo_host,
    const float* iv_host, const float* gs_host, int32_t* ranks_bev,
    int32_t* ranks_depth, int32_t* ranks_feat, int32_t* interval_starts,
    int32_t* interval_lengths, int32_t* counts, void* workspace,
    size_t workspace_bytes, int32_t pool_c, void* pool_plan,
    size_t pool_plan_bytes, fbbev_stream_t stream) {
  if (!frustum_u || !frustum_v || !frustum_d || !inv_post_rots ||
      !post_trans || !cam2ego || !trans || !bda)
    return FBBEV_ERR_INVALID_ARGUMENT;
  CamGeom cg;
  cg.us = frustum_u; cg.vs = frustum_v; cg.ds = frustum_d;
  cg.ipr = inv_post_rots; cg.ptr = post_trans; cg.comb = cam2ego;
  cg.trn = trans; cg.bda = bda;
  cg.N = N; cg.D = D; cg.H = H; cg.W = W;
  cg.order = order_flags;
  return voxel_prepare_impl(nullptr, &cg, B, N, D, H, W, lo_host, iv_host,
                            gs_host, ranks_bev, ranks_depth, ranks_feat,
                            interval_starts, interval_lengths, counts,
                            workspace, workspace_bytes, pool_c, pool_plan,
                            pool_plan_bytes, depth_prob, depth_thresh, stream);
}
