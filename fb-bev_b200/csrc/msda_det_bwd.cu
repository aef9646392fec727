// msda_det_bwd.cu -- deterministic backward of the deformable-attention ops,
// for sm_90a:
//   fbbev_msda_fused_bwd_det  twin of fbbev_msda_fused_bwd
//   fbbev_da_sca_bwd_det      twin of fbbev_da_sca_bwd
//   fbbev_msda_bwd_det        twin of fbbev_msda_bwd
//
// No float is accumulated with atomics.  Per pass (one sample; for the
// cross-attention's value gradient one (sample, camera) pair):
//   1. emit: the twin's per-(query, head) kernel runs with records instead of
//      reductions (msda_det.cuh).  Record slots are fixed by the sample's
//      indices; slots without an in-image sample keep kNoKey.
//   2. order: stable LSD radix sort of the keys, 8-bit digits.  A warp tile
//      ranks its keys with __match_any_sync in slot order, so equal keys keep
//      slot order and the cost does not depend on how many share a key.  Then
//      the [begin, end) range of every cell.
//   3. gather: one thread per gradient element sums the records of its four
//      neighbouring cells -- corner k = 0..3 in turn, the element being the
//      (k >> 1, k & 1) corner of the samples of cell (y - (k >> 1),
//      x - (k & 1)), each cell in sorted (= slot) order -- adding the twin's
//      rounded products left to right from +0, and stores once.
#include <cub/block/block_scan.cuh>

#include "common.cuh"
#include "msda_det.cuh"

namespace fbbev {

constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kTileChunks = 32;               // 32-key chunks per warp tile
constexpr int kTile = kWarp * kTileChunks;    // keys per warp tile
constexpr int kSortWarps = 4;                 // warp tiles per block
constexpr int kScanThreads = 1024, kScanItems = 8;
constexpr int kScanSeg = kScanThreads * kScanItems;
constexpr int kGatherThreads = 256;

using BlockScan = cub::BlockScan<int, kScanThreads>;

// ---------------- stable LSD radix sort ------------------------------------
// digit histogram of every warp tile, digit-major: hist[d * tiles + t]
__global__ void __launch_bounds__(kSortWarps * kWarp) radix_hist_kernel(
    const uint32_t* __restrict__ keys, int64_t n, int shift, int64_t tiles,
    int* __restrict__ hist) {
  __shared__ int cnt[kSortWarps][kRadix];
  const int w = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  const int64_t t = (int64_t)blockIdx.x * kSortWarps + w;
  if (t >= tiles) return;
  for (int d = lane; d < kRadix; d += kWarp) cnt[w][d] = 0;
  __syncwarp();
  for (int c = 0; c < kTileChunks; ++c) {
    const int64_t i = t * kTile + c * kWarp + lane;
    const unsigned d =
        i < n ? (__ldg(keys + i) >> shift) & (kRadix - 1) : (unsigned)kRadix;
    const unsigned peers = __match_any_sync(kFull, d);
    if (d < kRadix && lane == __ffs(peers) - 1) cnt[w][d] += __popc(peers);
    __syncwarp();
  }
  for (int d = lane; d < kRadix; d += kWarp) hist[d * tiles + t] = cnt[w][d];
}

__device__ __forceinline__ void scan_load(const int* a, int64_t n, int64_t i0,
                                          int (&v)[kScanItems]) {
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) v[k] = i0 + k < n ? a[i0 + k] : 0;
}
__device__ __forceinline__ void scan_store(int* a, int64_t n, int64_t i0,
                                           const int (&v)[kScanItems],
                                           int add) {
#pragma unroll
  for (int k = 0; k < kScanItems; ++k)
    if (i0 + k < n) a[i0 + k] = v[k] + add;
}

// exclusive scan of a[0..n) in place: segment totals, their scan (one
// block), then every segment
__global__ void __launch_bounds__(kScanThreads) scan_totals_kernel(
    const int* __restrict__ a, int64_t n, int* __restrict__ tot) {
  __shared__ BlockScan::TempStorage tmp;
  int v[kScanItems], agg;
  scan_load(a, n, blockIdx.x * (int64_t)kScanSeg + threadIdx.x * kScanItems, v);
  BlockScan(tmp).ExclusiveSum(v, v, agg);
  if (threadIdx.x == 0) tot[blockIdx.x] = agg;
}
__global__ void __launch_bounds__(kScanThreads) scan_block_kernel(
    int* __restrict__ tot, int64_t n) {
  __shared__ BlockScan::TempStorage tmp;
  int carry = 0;
  for (int64_t s = 0; s < n; s += kScanSeg) {
    int v[kScanItems], agg;
    const int64_t i0 = s + threadIdx.x * kScanItems;
    scan_load(tot, n, i0, v);
    BlockScan(tmp).ExclusiveSum(v, v, agg);
    scan_store(tot, n, i0, v, carry);
    carry += agg;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(
    int* __restrict__ a, int64_t n, const int* __restrict__ tot) {
  __shared__ BlockScan::TempStorage tmp;
  int v[kScanItems], agg;
  const int64_t i0 = blockIdx.x * (int64_t)kScanSeg + threadIdx.x * kScanItems;
  scan_load(a, n, i0, v);
  BlockScan(tmp).ExclusiveSum(v, v, agg);
  scan_store(a, n, i0, v, tot[blockIdx.x]);
}

// stable scatter by digit: keys of a tile in slot order, equal digits ranked
// by lane inside a chunk (vals_in NULL: the slot index itself)
__global__ void __launch_bounds__(kSortWarps * kWarp) radix_scatter_kernel(
    const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
    int64_t n, int shift, int64_t tiles, const int* __restrict__ offs,
    uint32_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out) {
  __shared__ int base[kSortWarps][kRadix];
  const int w = threadIdx.x / kWarp, lane = threadIdx.x % kWarp;
  const int64_t t = (int64_t)blockIdx.x * kSortWarps + w;
  if (t >= tiles) return;
  for (int d = lane; d < kRadix; d += kWarp) base[w][d] = offs[d * tiles + t];
  __syncwarp();
  const unsigned below = (1u << lane) - 1u;
  for (int c = 0; c < kTileChunks; ++c) {
    const int64_t i = t * kTile + c * kWarp + lane;
    const bool ok = i < n;
    const uint32_t key = ok ? __ldg(keys_in + i) : 0u;
    const unsigned d = ok ? (key >> shift) & (kRadix - 1) : (unsigned)kRadix;
    const unsigned peers = __match_any_sync(kFull, d);
    if (ok) {
      const int pos = base[w][d] + __popc(peers & below);
      keys_out[pos] = key;
      vals_out[pos] = vals_in ? __ldg(vals_in + i) : (uint32_t)i;
    }
    __syncwarp();
    if (ok && lane == __ffs(peers) - 1) base[w][d] += __popc(peers);
    __syncwarp();
  }
}

// [begin, end) of every key present in the sorted keys (others stay {0, 0})
__global__ void cell_range_kernel(const uint32_t* __restrict__ sk, int64_t n,
                                  int64_t n_keys, int2* __restrict__ range) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = sk[i];
  if (k >= n_keys) return;
  if (i == 0 || sk[i - 1] != k) range[k].x = (int)i;
  if (i == n - 1 || sk[i + 1] != k) range[k].y = (int)(i + 1);
}

// ---------------- gather ----------------------------------------------------
// The weight of corner k = 2 * dy + dx of a record is Bilinear's, as in the
// twin kernel that wrote the record.
//
// grad_value of one (n_value, heads, ch) map.  Record r belongs to grad row
// r / LP of G (nq, heads*ch).  kFusedArith: the product (a * w) * g of
// sample_bwd (msda_fused_bwd.cu); otherwise w * (g * a) of msda_bwd.cu.
template <bool kFusedArith>
__global__ void __launch_bounds__(kGatherThreads) gather_value_kernel(
    const int64_t* __restrict__ shapes, const int64_t* __restrict__ lstart,
    int levels, int n_value, int heads, int ch, int LP,
    const int2* __restrict__ range, const uint32_t* __restrict__ order,
    const float3* __restrict__ rec, const float* __restrict__ G,
    float* __restrict__ gval) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int E = heads * ch;
  if (idx >= (int64_t)n_value * E) return;
  const int c = (int)(idx % ch), m = (int)((idx / ch) % heads);
  const int v = (int)(idx / E);
  int l = 0, pcell = 0;
  while (l + 1 < levels && v >= (int)__ldg(lstart + l + 1)) {
    pcell += ((int)__ldg(shapes + 2 * l) + 1) * ((int)__ldg(shapes + 2 * l + 1) + 1);
    ++l;
  }
  const int W = (int)__ldg(shapes + 2 * l + 1);
  const int px = v - (int)__ldg(lstart + l), y = px / W, x = px - y * W;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int2 rg =
        range[(pcell + (y + 1 - (k >> 1)) * (W + 1) + x + 1 - (k & 1)) * heads +
              m];
    for (int j = rg.x; j < rg.y; ++j) {
      const uint32_t r = __ldg(order + j);
      const float3 R = rec[r];
      const float wk = Bilinear(R.x, R.y).weight(k);
      const float g = __ldg(G + (int64_t)(r / LP) * ch + c);
      acc = __fadd_rn(acc, kFusedArith ? __fmul_rn(__fmul_rn(R.z, wk), g)
                                       : __fmul_rn(wk, __fmul_rn(g, R.z)));
    }
  }
  gval[idx] = acc;
}

// grad_depth_prob of sample b, (n_cams, H0*W0, DC).  Products w * g as
// scatter_scalar (msda_fused_bwd.cu).
__global__ void __launch_bounds__(kGatherThreads) gather_depth_kernel(
    const int64_t* __restrict__ shapes, int b, int n_cams, int DC, const int2* __restrict__ range, const uint32_t* __restrict__ order,
    const float3* __restrict__ rec, float* __restrict__ gdp) {
  const int H0 = (int)__ldg(shapes), W0 = (int)__ldg(shapes + 1);
  const int64_t per_cam = (int64_t)H0 * W0 * DC;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_cams * per_cam) return;
  const int n = (int)(idx / per_cam);
  const int d = (int)(idx % DC);
  const int px = (int)((idx % per_cam) / DC), y = px / W0, x = px - y * W0;
  const int cells = (H0 + 1) * (W0 + 1);
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int2 rg =
        range[(int64_t)(n * cells + (y + 1 - (k >> 1)) * (W0 + 1) + x + 1 -
                        (k & 1)) * DC + d];
    for (int j = rg.x; j < rg.y; ++j) {
      const float3 R = rec[__ldg(order + j)];
      acc = __fadd_rn(acc,
                      __fmul_rn(Bilinear(R.x, R.y).weight(k), R.z));
    }
  }
  gdp[(int64_t)b * n_cams * per_cam + idx] = acc;
}

// ---------------- workspace -------------------------------------------------
// One record set: n slots, keys < n_keys (kNoKey for empty slots).
struct RecordSet {
  int64_t n = 0, n_keys = 0;
  uint32_t *key = nullptr, *key2 = nullptr, *val = nullptr, *val2 = nullptr;
  float3* rec = nullptr;
  int* hist = nullptr;
  int* tot = nullptr;
  int2* range = nullptr;
  int64_t tiles() const { return ceil_div64(n, kTile); }
};

struct Carver {  // base == nullptr: sizes only
  char* base;
  size_t off = 0;
  template <class T>
  T* take(int64_t count) {
    off = (off + 255) & ~size_t(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += (size_t)count * sizeof(T);
    return p;
  }
};

static void carve_set(Carver& c, RecordSet& s, int64_t n, int64_t n_keys) {
  s.n = n;
  s.n_keys = n_keys;
  const int64_t m = (int64_t)kRadix * s.tiles();
  s.key = c.take<uint32_t>(n);
  s.key2 = c.take<uint32_t>(n);
  s.val = c.take<uint32_t>(n);
  s.val2 = c.take<uint32_t>(n);
  s.rec = c.take<float3>(n);
  s.hist = c.take<int>(m);
  s.tot = c.take<int>(ceil_div64(m, kScanSeg));
  s.range = c.take<int2>(n_keys);
}

// Record sets of a call, from sizes only.  n_cams == 0: the self-attention /
// drop-in op (value records only); otherwise the cross-attention (value
// records of one (sample, camera) pair, G, depth records of one sample).
struct DetLayout {
  RecordSet v, d;
  float* G = nullptr;
  size_t bytes = 0;
};
static inline int depth_heads(int heads) { return kWarp % heads ? heads : 1; }
static DetLayout det_layout(void* ws, int n_cams, int nq, int n_value,
                            int heads, int ch, int levels, int points, int Z,
                            int DC) {
  DetLayout L;
  // (H+1)(W+1) <= 2 H W + 2 for H, W >= 1: cells of all levels
  const int64_t cells = 2 * (int64_t)n_value + 2 * levels;
  char* base = ws ? reinterpret_cast<char*>(
                        (reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255))
                  : nullptr;
  Carver c{base};
  carve_set(c, L.v, (int64_t)nq * heads * levels * points, cells * heads);
  if (n_cams > 0) {
    L.G = c.take<float>((int64_t)nq * heads * ch);
    carve_set(c, L.d, (int64_t)n_cams * nq * depth_heads(heads) * Z,
              (int64_t)n_cams * (2 * (int64_t)n_value + 2) * DC);
  }
  L.bytes = c.off + 255;  // room to align the caller's pointer
  return L;
}

static bool set_fits(const RecordSet& s) {
  return s.n < (int64_t(1) << 31) && s.n_keys < (int64_t(1) << 31);
}

// Sorts a filled record set; returns the slot order, with set.range filled.
static const uint32_t* sort_records(RecordSet& s, cudaStream_t st) {
  int bits = 1;
  while ((int64_t(1) << bits) <= s.n_keys) ++bits;  // kNoKey's low bits above
  const int64_t tiles = s.tiles(), m = (int64_t)kRadix * tiles;
  const int64_t nseg = ceil_div64(m, kScanSeg);
  const unsigned sort_grid = (unsigned)ceil_div64(tiles, kSortWarps);
  uint32_t *kin = s.key, *kout = s.key2, *vin = nullptr, *vout = s.val;
  for (int shift = 0; shift < bits; shift += kRadixBits) {
    radix_hist_kernel<<<sort_grid, kSortWarps * kWarp, 0, st>>>(
        kin, s.n, shift, tiles, s.hist);
    scan_totals_kernel<<<(unsigned)nseg, kScanThreads, 0, st>>>(s.hist, m,
                                                                s.tot);
    scan_block_kernel<<<1, kScanThreads, 0, st>>>(s.tot, nseg);
    scan_apply_kernel<<<(unsigned)nseg, kScanThreads, 0, st>>>(s.hist, m,
                                                               s.tot);
    radix_scatter_kernel<<<sort_grid, kSortWarps * kWarp, 0, st>>>(
        kin, vin, s.n, shift, tiles, s.hist, kout, vout);
    count_launch(5);
    uint32_t* k = kin;
    kin = kout;
    kout = k;
    vin = vout;
    vout = vout == s.val ? s.val2 : s.val;
  }
  cudaMemsetAsync(s.range, 0, s.n_keys * sizeof(int2), st);
  cell_range_kernel<<<(unsigned)ceil_div64(s.n, kGatherThreads),
                      kGatherThreads, 0, st>>>(kin, s.n, s.n_keys, s.range);
  count_launch();
  return vin;
}

static void clear_keys(const RecordSet& s, cudaStream_t st) {
  cudaMemsetAsync(s.key, 0xff, s.n * sizeof(uint32_t), st);
}

template <bool kFusedArith>
static void gather_value(const RecordSet& s, const uint32_t* order,
                         const int64_t* shapes, const int64_t* lstart,
                         int levels, int n_value, int heads, int ch,
                         int points, const float* G, float* gval,
                         cudaStream_t st) {
  const int64_t n = (int64_t)n_value * heads * ch;
  gather_value_kernel<kFusedArith>
      <<<(unsigned)ceil_div64(n, kGatherThreads), kGatherThreads, 0, st>>>(
          shapes, lstart, levels, n_value, heads, ch, levels * points,
          s.range, order, s.rec, G, gval);
  count_launch();
}

static int check_workspace(const DetLayout& L, const void* ws, size_t bytes) {
  if (!set_fits(L.v) || !set_fits(L.d)) return FBBEV_ERR_UNSUPPORTED;
  return !ws || bytes < L.bytes ? FBBEV_ERR_WORKSPACE_TOO_SMALL : FBBEV_OK;
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API size_t fbbev_msda_fused_bwd_det_workspace_bytes(
    int32_t nq, int32_t n_value, int32_t heads, int32_t levels,
    int32_t points) {
  if (nq <= 0 || n_value <= 0 || heads <= 0 || levels <= 0 || points <= 0)
    return 0;
  return det_layout(nullptr, 0, nq, n_value, heads, 0, levels, points, 0, 0)
      .bytes;
}

FBBEV_API size_t fbbev_msda_bwd_det_workspace_bytes(int32_t nq,
                                                    int32_t n_value,
                                                    int32_t heads,
                                                    int32_t levels,
                                                    int32_t points) {
  return fbbev_msda_fused_bwd_det_workspace_bytes(nq, n_value, heads, levels,
                                                  points);
}

FBBEV_API size_t fbbev_da_sca_bwd_det_workspace_bytes(
    int32_t n_cams, int32_t nq, int32_t n_value, int32_t heads, int32_t ch,
    int32_t levels, int32_t points, int32_t Z, int32_t DC) {
  if (n_cams <= 0 || nq <= 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0 || Z <= 0 || DC <= 0)
    return 0;
  return det_layout(nullptr, n_cams, nq, n_value, heads, ch, levels, points,
                    Z, DC)
      .bytes;
}

FBBEV_API int fbbev_msda_fused_bwd_det(
    const float* value, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* ref, const float* offsets,
    const float* logits, const float* grad_out, int32_t bs, int32_t n_value,
    int32_t heads, int32_t ch, int32_t levels, int32_t nq, int32_t points,
    float* grad_value, float* grad_offsets, float* grad_logits,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fused_head_width(ch)) return FBBEV_ERR_UNSUPPORTED;
  if ((int64_t)bs * nq == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !ref || !offsets ||
      !logits || !grad_out || !vec_aligned(value, ch) ||
      !vec_aligned(grad_out, ch))
    return FBBEV_ERR_INVALID_ARGUMENT;
  DetLayout L = det_layout(grad_value ? workspace : nullptr, 0, nq, n_value,
                           heads, ch, levels, points, 0, 0);
  if (grad_value) {
    const int rc = check_workspace(L, workspace, workspace_bytes);
    if (rc != FBBEV_OK) return rc;
  }
  cudaStream_t st = as_stream(stream);
  const int E = heads * ch, LP = levels * points;
  for (int b = 0; b < bs; ++b) {
    const int64_t qb = (int64_t)b * nq;
    DetSink det;
    if (grad_value) {
      clear_keys(L.v, st);
      det.key = L.v.key;
      det.rec = L.v.rec;
    }
    const int rc = msda_fused_bwd_records(
        value + (int64_t)b * n_value * E, spatial_shapes, level_start,
        ref + qb * levels * 2, offsets + qb * heads * LP * 2,
        logits + qb * heads * LP, grad_out + qb * E, n_value, heads, ch,
        levels, nq, points,
        grad_offsets ? grad_offsets + qb * heads * LP * 2 : nullptr,
        grad_logits ? grad_logits + qb * heads * LP : nullptr, det, st);
    if (rc != FBBEV_OK) return rc;
    if (grad_value)
      gather_value<true>(L.v, sort_records(L.v, st), spatial_shapes,
                         level_start, levels, n_value, heads, ch, points,
                         grad_out + qb * E,
                         grad_value + (int64_t)b * n_value * E, st);
  }
  return launch_status();
}

FBBEV_API int fbbev_msda_bwd_det(
    const float* value, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* loc, const float* attw,
    const float* grad_out, int32_t bs, int32_t n_value, int32_t heads,
    int32_t ch, int32_t levels, int32_t nq, int32_t points, float* grad_value,
    float* grad_loc, float* grad_attw, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_value <= 0 || heads <= 0 || ch <= 0 ||
      levels <= 0 || points <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((int64_t)bs * nq == 0) return FBBEV_OK;
  if (!value || !spatial_shapes || !level_start || !loc || !attw ||
      !grad_out || !grad_value || !grad_loc || !grad_attw)
    return FBBEV_ERR_INVALID_ARGUMENT;
  DetLayout L = det_layout(workspace, 0, nq, n_value, heads, ch, levels,
                           points, 0, 0);
  const int rc0 = check_workspace(L, workspace, workspace_bytes);
  if (rc0 != FBBEV_OK) return rc0;
  cudaStream_t st = as_stream(stream);
  const int E = heads * ch, LP = levels * points;
  for (int b = 0; b < bs; ++b) {
    const int64_t qb = (int64_t)b * nq;
    DetSink det;
    clear_keys(L.v, st);
    det.key = L.v.key;
    det.rec = L.v.rec;
    const int rc = msda_bwd_records(
        value + (int64_t)b * n_value * E, spatial_shapes, level_start,
        loc + qb * heads * LP * 2, attw + qb * heads * LP, grad_out + qb * E,
        n_value, heads, ch, levels, nq, points,
        grad_loc + qb * heads * LP * 2, grad_attw + qb * heads * LP, det, st);
    if (rc != FBBEV_OK) return rc;
    gather_value<false>(L.v, sort_records(L.v, st), spatial_shapes,
                        level_start, levels, n_value, heads, ch, points,
                        grad_out + qb * E,
                        grad_value + (int64_t)b * n_value * E, st);
  }
  return launch_status();
}

FBBEV_API int fbbev_da_sca_bwd_det(
    const float* value, const float* depth_prob, const float* ref_cam,
    const float* ref_depth, const uint8_t* mask, const float* offsets,
    const float* logits, const int64_t* spatial_shapes,
    const int64_t* level_start, const float* dbound_host,
    const float* grad_out, int32_t bs, int32_t n_cams, int32_t nq,
    int32_t n_value, int32_t heads, int32_t ch, int32_t levels,
    int32_t points, int32_t Z, int32_t DC, float* grad_value,
    float* grad_depth_prob, float* grad_offsets, float* grad_logits,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  if (bs < 0 || nq < 0 || n_cams <= 0 || n_value <= 0 || heads <= 0 ||
      ch <= 0 || levels <= 0 || points <= 0 || Z <= 0 || DC <= 0 ||
      !dbound_host || points % Z != 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fused_head_width(ch) || !fused_z(Z)) return FBBEV_ERR_UNSUPPORTED;
  if ((int64_t)bs * nq == 0) return FBBEV_OK;
  if (!value || !depth_prob || !ref_cam || !ref_depth || !mask || !offsets ||
      !logits || !spatial_shapes || !level_start || !grad_out ||
      !vec_aligned(value, ch) || !vec_aligned(grad_out, ch))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const bool gv = grad_value != nullptr, gd = grad_depth_prob != nullptr;
  DetLayout L = det_layout(gv || gd ? workspace : nullptr, n_cams, nq,
                           n_value, heads, ch, levels, points, Z, DC);
  if (gv || gd) {
    const int rc = check_workspace(L, workspace, workspace_bytes);
    if (rc != FBBEV_OK) return rc;
  }
  const DaScaParams P = da_sca_params(dbound_host, bs, n_cams, nq, n_value,
                                      heads, levels, points, DC);
  cudaStream_t st = as_stream(stream);
  const int E = heads * ch;
  for (int b = 0; b < bs; ++b) {
    if (gd) clear_keys(L.d, st);
    for (int n = 0; n < n_cams; ++n) {
      DetSink det;
      det.item0 = (int64_t)b * nq * heads;
      det.cam = n;
      if (gv) {
        clear_keys(L.v, st);
        det.key = L.v.key;
        det.rec = L.v.rec;
        det.G = L.G;
      }
      if (gd) {
        det.dkey = L.d.key;
        det.drec = L.d.rec;
      }
      const int rc = da_sca_bwd_records(
          value, depth_prob, ref_cam, ref_depth, mask, offsets, logits,
          spatial_shapes, level_start, P, ch, Z, grad_out, grad_offsets,
          grad_logits, det, st);
      if (rc != FBBEV_OK) return rc;
      if (gv)
        gather_value<true>(
            L.v, sort_records(L.v, st), spatial_shapes, level_start, levels,
            n_value, heads, ch, points, L.G,
            grad_value + ((int64_t)b * n_cams + n) * n_value * E, st);
    }
    if (gd) {
      const uint32_t* order = sort_records(L.d, st);
      const int64_t n_out = (int64_t)n_cams * n_value * DC;  // >= H0*W0
      gather_depth_kernel<<<(unsigned)ceil_div64(n_out, kGatherThreads),
                            kGatherThreads, 0, st>>>(
          spatial_shapes, b, n_cams, DC, L.d.range, order, L.d.rec,
          grad_depth_prob);
      count_launch();
    }
  }
  return launch_status();
}
