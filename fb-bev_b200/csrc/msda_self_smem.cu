// msda_self_smem.cu -- BEV self-attention sampler (the fused core of mmcv
// MultiScaleDeformableAttention.forward) gathering from a shared-memory
// footprint tile (sm_90a).
//
// Same arithmetic, bit for bit, as msda_fused_fwd_kernel (msda_fwd.cu).  That
// kernel is bound by L1 wavefronts: a thread is one (query, head) and every
// corner of every sample is a 40-byte gather, so the 32 lanes of a load point
// at up to 32 different 128-byte lines and L1 serves one line per wavefront.
// The samples of a query lie within a few pixels of the query's own pixel (the
// offset bias is a ring of radius <= 4 pixels, plus a learned term), so here
//
//   * a CTA owns a kTx x kTy rectangle of queries and stages the value pixels
//     of that rectangle grown by kR pixels on each side -- shifted inwards at
//     the map's borders so that the window always has its full size -- with
//     one 1-D bulk copy per window row on one mbarrier;
//   * lane = (query slot, head), four queries of a BEV row per warp; the
//     offsets / logits rows are plain coalesced loads issued before the wait on
//     the barrier, the softmax over the points stays in registers;
//   * a sample whose four corners lie in the window gathers with LDS.64: with
//     the 80-float pixel pitch the eight head chunks of a pixel fall into
//     disjoint banks and odd / even pixels are 16 banks apart (da_sca_smem.cu);
//     the window's row pitch is a whole number of pixels and a load instruction
//     serves one corner, so only the pixel parity within that corner matters;
//   * any other sample (learned offsets are unbounded; corners off the map at
//     the borders) loads the same corners from global memory, absent corners as
//     zeros, and runs through the same arithmetic: the result does not depend
//     on which side served it.
//
// Selected from the shape by fbbev_msda_fused_fwd: 8 heads x 10 channels, one
// level, 4 points, one query per value pixel, a map at least one window wide
// and high.  Every other shape keeps the global-memory kernels.
#include "msda_self_smem.h"

#include "bulk.cuh"
#include "common.cuh"
#include "msda_common.cuh"

namespace fbbev {

constexpr int kCH = 10, kHeads = 8, kE = 80, kPts = 4;
// queries per CTA and halo; the window is (kTx + 2 kR) x (kTy + 2 kR) pixels
constexpr int kTx = 8, kTy = 8, kR = 5;
constexpr int kWx = kTx + 2 * kR, kWy = kTy + 2 * kR;
constexpr int kThreads = kTx * kTy * kHeads;
constexpr int kTileBytes = kWx * kWy * kE * 4;
// 103,680 B of tile and 64 registers x 512 threads: two CTAs per SM, one
// staging its window while the other gathers
constexpr int kCtasPerSm = 2;
static_assert(kTx % 4 == 0, "a warp is four queries of one BEV row");
static_assert(kThreads <= 1024 && kWy <= 32, "one CTA, one copy per lane");

// acc += wgt * sample, the corners at p1..p4 (channel 0 of the lane's head);
// from global memory a corner outside the map reads as zeros
template <bool SMEM>
__device__ __forceinline__ void gather_accum(const Bilinear& bl, const float* p1,
                                             const float* p2, const float* p3,
                                             const float* p4, int H, int W,
                                             float wgt, float (&acc)[kCH]) {
  const float2 zero = make_float2(0.f, 0.f);
  const bool ok1 = SMEM || bl.ok1(H, W), ok2 = SMEM || bl.ok2(H, W);
  const bool ok3 = SMEM || bl.ok3(H, W), ok4 = SMEM || bl.ok4(H, W);
#pragma unroll
  for (int c = 0; c < kCH; c += 2) {
    const float2 v1 = ok1 ? ld2<SMEM>(p1 + c) : zero;
    const float2 v2 = ok2 ? ld2<SMEM>(p2 + c) : zero;
    const float2 v3 = ok3 ? ld2<SMEM>(p3 + c) : zero;
    const float2 v4 = ok4 ? ld2<SMEM>(p4 + c) : zero;
    acc[c] += bl.blend(v1.x, v2.x, v3.x, v4.x) * wgt;
    acc[c + 1] += bl.blend(v1.y, v2.y, v3.y, v4.y) * wgt;
  }
}

// grid = (ceil(W / kTx), ceil(nq / W / kTy), bs); W = the map's width as the
// caller's patch_w, nq = n_value = H * W
__global__ void __launch_bounds__(kThreads, kCtasPerSm) msda_self_smem_kernel(
    const float* __restrict__ value, const int64_t* __restrict__ shapes,
    const float* __restrict__ ref, const float* __restrict__ offsets,
    const float* __restrict__ logits, int nq, int W, float* __restrict__ out) {
  extern __shared__ __align__(128) float tile[];
  __shared__ uint64_t bar;
  const int H = nq / W;
  const int tx0 = blockIdx.x * kTx, ty0 = blockIdx.y * kTy;
  // the window: the tile and its halo, shifted to lie inside the map
  const int x0 = min(max(tx0 - kR, 0), W - kWx);
  const int y0 = min(max(ty0 - kR, 0), H - kWy);
  const float* vmap = value + (int64_t)blockIdx.z * nq * kE;

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(&bar), 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0)
      mbar_arrive_expect_tx(smem_u32(&bar), kTileBytes);
    __syncwarp();
    // a window row is a contiguous run of kWx pixels of the map
    if (threadIdx.x < kWy)
      bulk_g2s(smem_u32(tile + threadIdx.x * kWx * kE),
               vmap + ((int64_t)(y0 + threadIdx.x) * W + x0) * kE, kWx * kE * 4,
               smem_u32(&bar));
  }

  const int m = threadIdx.x & 7, ql = threadIdx.x >> 3;
  const int qx = tx0 + ql % kTx, qy = ty0 + ql / kTx;
  // thread 0 (the tile's first query) always stays and waits for the copies,
  // so the CTA outlives them
  if (qx >= W || qy >= H) return;
  const int64_t bq = (int64_t)blockIdx.z * nq + qy * W + qx;
  const int64_t item = bq * kHeads + m;

  // sampling geometry from spatial_shapes as in the global kernels; the window
  // only serves a map that is the W-wide map the queries are laid out on
  const int Hs = (int)__ldg(shapes), Ws = (int)__ldg(shapes + 1);
  const bool window_ok = Hs == H && Ws == W;
  const float2 r = __ldg(reinterpret_cast<const float2*>(ref) + bq);
  const float4 lg4 = __ldg(reinterpret_cast<const float4*>(logits) + item);
  const float4 oa = __ldg(reinterpret_cast<const float4*>(offsets) + 2 * item);
  const float4 ob =
      __ldg(reinterpret_cast<const float4*>(offsets) + 2 * item + 1);
  const float lg[kPts] = {lg4.x, lg4.y, lg4.z, lg4.w};
  const float ox[kPts] = {oa.x, oa.z, ob.x, ob.z};
  const float oy[kPts] = {oa.y, oa.w, ob.y, ob.w};

  // softmax over the points, the statistics of softmax_stats in its order
  float mx = -INFINITY;
#pragma unroll
  for (int p = 0; p < kPts; ++p) mx = fmaxf(mx, lg[p]);
  float wgt[kPts], s = 0.f;
#pragma unroll
  for (int p = 0; p < kPts; ++p) {
    wgt[p] = expf(lg[p] - mx);
    s += wgt[p];
  }
  const float inv = 1.f / s;
  float h_im[kPts], w_im[kPts];
#pragma unroll
  for (int p = 0; p < kPts; ++p) {
    wgt[p] *= inv;
    // sampling_locations = ref + offsets / (W, H)
    w_im[p] = pix(r.x + __fdiv_rn(ox[p], (float)Ws), Ws);
    h_im[p] = pix(r.y + __fdiv_rn(oy[p], (float)Hs), Hs);
  }

  float acc[kCH];
#pragma unroll
  for (int c = 0; c < kCH; ++c) acc[c] = 0.f;
  const float* smap = tile + m * kCH;
  const float* gmap = vmap + m * kCH;
  mbar_wait(smem_u32(&bar), 0);
#pragma unroll
  for (int p = 0; p < kPts; ++p) {
    // NaN and +-inf locations fail this test as in the global kernels; past
    // it -1 <= h_low < Hs and -1 <= w_low < Ws, and the window test below comes
    // before any shared-memory address is formed
    if (!in_image(h_im[p], w_im[p], Hs, Ws)) continue;
    const Bilinear bl(h_im[p], w_im[p]);
    const int wy = bl.h_low - y0, wx = bl.w_low - x0;
    if (window_ok && (unsigned)wy < (unsigned)(kWy - 1) &&
        (unsigned)wx < (unsigned)(kWx - 1)) {
      const float* p1 = smap + (wy * kWx + wx) * kE;
      gather_accum<true>(bl, p1, p1 + kE, p1 + kWx * kE, p1 + (kWx + 1) * kE,
                         Hs, Ws, wgt[p], acc);
    } else {
      const float* p1 = gmap + bl.offset(Ws, kE);
      const float* p3 = p1 + (int64_t)Ws * kE;
      gather_accum<false>(bl, p1, p1 + kE, p3, p3 + kE, Hs, Ws, wgt[p], acc);
    }
  }
  float2* o = reinterpret_cast<float2*>(out + bq * kE + m * kCH);
#pragma unroll
  for (int c = 0; c < kCH / 2; ++c)
    o[c] = make_float2(acc[2 * c], acc[2 * c + 1]);
}

bool msda_self_smem_eligible(int bs, int n_value, int heads, int ch, int levels,
                             int nq, int points, int patch_w) {
  return bs <= 65535 && heads == kHeads && ch == kCH && levels == 1 && points == kPts &&
         patch_w >= kWx && nq == n_value && nq % patch_w == 0 &&
         nq / patch_w >= kWy && (nq / patch_w + kTy - 1) / kTy <= 65535;
}

int msda_self_smem_launch(const float* value, const int64_t* shapes,
                          const float* ref, const float* offsets,
                          const float* logits, int bs, int nq, int patch_w,
                          float* out, cudaStream_t st) {
  // per device, so on every launch
  const cudaError_t attr = cudaFuncSetAttribute(
      msda_self_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
      kTileBytes);
  if (attr != cudaSuccess) return static_cast<int>(attr);
  const dim3 grid((unsigned)((patch_w + kTx - 1) / kTx),
                  (unsigned)((nq / patch_w + kTy - 1) / kTy), (unsigned)bs);
  msda_self_smem_kernel<<<grid, kThreads, kTileBytes, st>>>(
      value, shapes, ref, offsets, logits, nq, patch_w, out);
  return launch_status();
}

}  // namespace fbbev
