// ffn_tf32.cu -- the encoder layer's FFN as ONE Hopper tensor-core kernel:
//
//     y = LayerNorm( residual + W2 . relu(W1 . x + b1) + b2 )
//
// What it replaces: mmcv `FFN` (Linear -> ReLU -> Linear, identity add) and the
// `norm` that follows it in the reference's operation order
// (bevformer_encoder.py:251-377, config ffn_cfgs / operation_order).  The
// reference runs two cuBLAS GEMMs, three element-wise kernels and a LayerNorm
// kernel, with the 40000 x 320 hidden activation (51 MB) written to and read
// back from memory in between.  Here the hidden tile never leaves the SM:
//
//   X       the CTA's 128 rows of x, split hi / lo (3xTF32, see wgmma.cuh),
//           stay in shared memory for the whole tile
//   GEMM1   per 80-column hidden chunk: H[128 x 80] = X . W1_chunk^T, one
//           wgmma accumulator per warpgroup (64 rows each)
//   convert + b1, ReLU, hi / lo split of the accumulator registers into a
//           shared-memory A tile (K-major core-matrix layout)
//   GEMM2   Y[128 x E] += H_chunk . W2[:, chunk]^T, accumulator in registers
//           across all chunks
//   finish  + b2 + residual, LayerNorm over the quad that holds each row,
//           column-pair stores
//
// The grid is persistent (one CTA per SM), each CTA looping over 128-row
// tiles.  The weights stream through a two-slot ring of 25.6 KB stages (one
// 1-D bulk copy each, in the order the tensor cores consume them: the
// K-blocks of W1 chunk c, then the two K-blocks of W2 that chunk c feeds; the
// sequence runs on across the CTA's tiles).  Each stage is one full-width
// wgmma per operand pair and k8 step; a slot is refilled as soon as the MMAs
// of the stage before have drained (wgmma.wait_group 1), so the tensor cores
// drain only at the hidden-chunk conversion.  The next tile's X rows are
// loaded into registers during the last chunk and stored once its GEMM1 has
// read the current tile.
// Shared memory: X tile hi / lo (<= 80 KB) | hidden tile hi / lo (80 KB) |
// weight ring (2 x 25.6 KB) | mbarriers | b1, b2, gamma, beta (2.2 KB).
//
// Shapes: E <= 80, E % 4 == 0; hidden % 80 == 0, hidden <= 320.
#include "common.cuh"
#include "wgmma.cuh"

namespace fbbev {
namespace ffn {

constexpr int kChunks = kKB / 4;        // 16-byte chunks of a row per K-block
constexpr int kTileM = 128;
constexpr int kAPart = kTileM * kKB * 4;            // bytes of A_hi (== A_lo)
constexpr int kABlock = 2 * kAPart;                 // one K-block, hi + lo
constexpr int kAChunkStride = (kTileM / 8) * 128;   // bytes between K chunks
constexpr int kThreads = 256;           // two warpgroups
constexpr int kHC = 80;                 // hidden columns per GEMM1 chunk
constexpr int kMaxE = 80;
constexpr int kMaxHidden = 320;
constexpr int kWStage = 2 * kHC * kKB * 4;          // >= 2 * pad16(E) * kKB * 4
constexpr int kXBytes = 2 * kABlock;                // E <= 80: two K-blocks
constexpr int kHBytes = (kHC / kKB) * kABlock;
constexpr int kCv = kMaxHidden + 3 * kMaxE;         // b1 | b2 | gamma | beta
constexpr int kSmem = kXBytes + kHBytes + 2 * kWStage + 16 + kCv * 4;

struct Params {
  const float* x;         // [M][E]
  const float* w1p;       // hidden / 80 blocks, each fbbev_linear_pack(80 rows, E)
  const float* b1;        // [hidden] or null
  const float* w2p;       // fbbev_linear_pack(E rows, hidden)
  const float* b2;        // [E] or null
  const float* residual;  // [M][E] or null
  const float* gamma;     // [E] or null (no LayerNorm)
  const float* beta;
  float* y;               // [M][E]
  int M, E, n_kb1, n_hc;
  int64_t ldx, ldr, ldy;
  float eps;
};

// A-tile offset (bytes) of element (row, col) of a [128 x 40 k] block image
__device__ __forceinline__ uint32_t a_off(int row, int col) {
  return (uint32_t)((col >> 2) * (kTileM / 8) + (row >> 3)) * 128u + (row & 7) * 16u +
         (col & 3) * 4u;
}

// finish of one tile on the GEMM2 accumulator: + b2 + residual, LayerNorm,
// column-pair stores; `rbase` is the thread's first row, q = lane % 4.  b2 /
// gamma / beta come from shared memory (`cv`, zero past E) and the residual
// loads are issued together from always-valid addresses (see linear_epilogue).
template <int NP2>
__device__ __forceinline__ void ffn_finish(const Params& p, const float (&acc2)[NP2 / 2],
                                           const float* cv, int rbase, int q) {
  const float* b2 = cv + kMaxHidden;
  const float* gamma = b2 + kMaxE;
  const float* beta = gamma + kMaxE;
  const int E = p.E;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rbase + 8 * h;
    const bool row_ok = row < p.M;
    float t[NP2 / 4];
    float2 r[NP2 / 8];
    if (p.residual) {
#pragma unroll
      for (int J = 0; J < NP2 / 8; ++J) {
        const int col = 8 * J + 2 * q;
        const float* src = row_ok && col < E ? p.residual + (size_t)row * p.ldr + col
                                             : p.residual;
        r[J] = __ldg(reinterpret_cast<const float2*>(src));
      }
    }
#pragma unroll
    for (int J = 0; J < NP2 / 8; ++J) {
      const int col = 8 * J + 2 * q;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float u = acc2[4 * J + 2 * h + e];
        if (p.b2) u += b2[col + e];  // columns >= E are neither reduced nor stored
        t[2 * J + e] = u;
      }
      if (p.residual) {
        t[2 * J] += r[J].x;
        t[2 * J + 1] += r[J].y;
      }
    }
    if (p.gamma) {
      float sum = 0.f;
#pragma unroll
      for (int J = 0; J < NP2 / 8; ++J)
        if (8 * J + 2 * q < E) sum += t[2 * J] + t[2 * J + 1];
      sum += __shfl_xor_sync(kFull, sum, 1);
      sum += __shfl_xor_sync(kFull, sum, 2);
      const float mean = sum / (float)E;
      float sq = 0.f;
#pragma unroll
      for (int J = 0; J < NP2 / 8; ++J)
        if (8 * J + 2 * q < E) {
          const float a = t[2 * J] - mean, b = t[2 * J + 1] - mean;
          sq += a * a + b * b;
        }
      sq += __shfl_xor_sync(kFull, sq, 1);
      sq += __shfl_xor_sync(kFull, sq, 2);
      const float rstd = rsqrtf(sq / (float)E + p.eps);
#pragma unroll
      for (int J = 0; J < NP2 / 8; ++J) {
        const int col = 8 * J + 2 * q;
        if (col < E) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
            t[2 * J + e] = fmaf((t[2 * J + e] - mean) * rstd, gamma[col + e],
                                beta[col + e]);
        }
      }
    }
    if (!row_ok) continue;
#pragma unroll
    for (int J = 0; J < NP2 / 8; ++J) {
      const int col = 8 * J + 2 * q;
      if (col < E)
        *reinterpret_cast<float2*>(p.y + (size_t)row * p.ldy + col) =
            make_float2(t[2 * J], t[2 * J + 1]);
    }
  }
}

template <int NP2>
__global__ void __launch_bounds__(kThreads, 1) ffn_tf32_kernel(const Params p) {
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* xs = smem;
  unsigned char* hs = smem + kXBytes;
  const uint32_t xs_a = smem_u32(xs), hs_a = smem_u32(hs);
  const uint32_t ws_a = hs_a + kHBytes;
  const uint32_t bar = ws_a + 2 * kWStage;
  // b1 | b2 | gamma | beta, zero past hidden / E: read by every tile
  float* cv = reinterpret_cast<float*>(hs + kHBytes + 2 * kWStage + 16);
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 8u, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < kCv; i += kThreads) {
    const int j = i < kMaxHidden ? i : (i - kMaxHidden) % kMaxE;
    const float* v = i < kMaxHidden ? p.b1
                     : i < kMaxHidden + kMaxE ? p.b2
                     : i < kMaxHidden + 2 * kMaxE ? p.gamma : p.beta;
    const int n = i < kMaxHidden ? p.n_hc * kHC : p.E;
    cv[i] = v && j < n ? __ldg(v + j) : 0.f;
  }
  __syncthreads();

  // tiles blockIdx.x, + gridDim.x, ... (the grid is never larger than the
  // tile count); the weight stages of all of them form one sequence
  const int n_tiles = (p.M + kTileM - 1) / kTileM;
  const int per_c = p.n_kb1 + kHC / kKB;   // weight stages per hidden chunk
  const int per_tile = p.n_hc * per_c;
  const int total = ((n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1) * per_tile;
  auto issue_w = [&](int i) {
    if (tid != 0 || i >= total) return;
    const int t = i % per_tile;
    const int c = t / per_c, j = t - c * per_c;
    const float* src;
    uint32_t bytes;
    if (j < p.n_kb1) {
      src = p.w1p + (size_t)(c * p.n_kb1 + j) * (kWStage / 4);
      bytes = kWStage;
    } else {
      const int kb = c * (kHC / kKB) + (j - p.n_kb1);
      src = p.w2p + (size_t)kb * (2 * NP2 * kKB);
      bytes = 2u * NP2 * kKB * 4u;
    }
    const uint32_t s = i & 1;
    mbar_arrive_expect_tx(bar + 8u * s, bytes);
    bulk_g2s(ws_a + s * kWStage, src, bytes, bar + 8u * s);
  };
  issue_w(0);
  issue_w(1);

  // X tile -> hi / lo images (columns >= E are zero): loaded into registers,
  // then stored, so the next tile's loads overlap the current tile's tail
  float4 xv[kXBytes / kABlock][5];
  auto load_x = [&](int row0) {
#pragma unroll
    for (int kb = 0; kb < kXBytes / kABlock; ++kb)
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const int idx = tid + kThreads * i;
        const int r = idx / kChunks, ch = idx - r * kChunks;
        const int g = row0 + r, col = kb * kKB + 4 * ch;
        xv[kb][i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kb < p.n_kb1 && g < p.M && col < p.E)
          xv[kb][i] = __ldg(reinterpret_cast<const float4*>(p.x + (size_t)g * p.ldx + col));
      }
  };
  auto store_x = [&]() {
#pragma unroll
    for (int kb = 0; kb < kXBytes / kABlock; ++kb) {
      if (kb >= p.n_kb1) break;
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        const int idx = tid + kThreads * i;
        const int r = idx / kChunks, ch = idx - r * kChunks;
        const float4 v = xv[kb][i];
        float4 hi;
        hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
        const float4 lo = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
        unsigned char* a = xs + (size_t)kb * kABlock + a_off(r, 4 * ch);
        *reinterpret_cast<float4*>(a) = hi;
        *reinterpret_cast<float4*>(a + kAPart) = lo;
      }
    }
  };
  load_x(blockIdx.x * kTileM);
  store_x();
  fence_proxy_async();
  __syncthreads();

  const int rl = wg * 64 + wq * 16 + (lane >> 2);   // tile row of acc[.. + 0 / 1]
  int it = 0;
  // after issuing stage `it`'s wgmma's: once stage it - 1's have drained (both
  // warpgroups), its slot takes stage it + 1 while stage it's MMAs run
  auto next_stage = [&]() {
    wgmma_commit();
    wgmma_wait<1>();
    __syncthreads();
    if (it >= 1) issue_w(it + 1);
    ++it;
  };
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int row0 = tile * kTileM;
    const bool more = tile + (int)gridDim.x < n_tiles;
    float acc2[NP2 / 2];  // written first by a scale-d = 0 MMA, never zeroed
    for (int c = 0; c < p.n_hc; ++c) {
      float acc1[kHC / 2];
      for (int j = 0; j < p.n_kb1; ++j) {
        const uint32_t s = it & 1;
        mbar_wait(bar + 8u * s, (it >> 1) & 1u);
        const uint32_t a_hi = xs_a + j * kABlock + wg * 1024u;
        const uint32_t w_hi = ws_a + s * kWStage;
        wgmma_fence();
        wg_kblock_3xtf32<kHC>(acc1, a_hi, a_hi + kAPart, kAChunkStride, w_hi,
                              w_hi + kHC * kKB * 4, kHC * 16, j > 0);
        next_stage();
      }
      wgmma_wait<0>();
      acc_fence(acc1);
      // the last chunk's GEMM1 has read the X tile: the next tile's loads start
      if (c == p.n_hc - 1 && more) load_x(row0 + (int)gridDim.x * kTileM);
      // hidden chunk: + b1, ReLU, hi / lo split -> this warpgroup's rows of hs
#pragma unroll
      for (int J = 0; J < kHC / 8; ++J) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * J + 2 * q + e;
            float v = acc1[4 * J + 2 * h + e];
            if (p.b1) v += cv[c * kHC + col];
            v = fmaxf(v, 0.f);
            const float hi = tf32_hi(v);
            unsigned char* a = hs + (size_t)(col / kKB) * kABlock + a_off(rl + 8 * h, col % kKB);
            *reinterpret_cast<float*>(a) = hi;
            *reinterpret_cast<float*>(a + kAPart) = v - hi;
          }
        }
      }
      fence_proxy_async();
      __syncthreads();
      for (int j = 0; j < kHC / kKB; ++j) {
        const uint32_t s = it & 1;
        mbar_wait(bar + 8u * s, (it >> 1) & 1u);
        const uint32_t a_hi = hs_a + j * kABlock + wg * 1024u;
        const uint32_t w_hi = ws_a + s * kWStage;
        wgmma_fence();
        wg_kblock_3xtf32<NP2>(acc2, a_hi, a_hi + kAPart, kAChunkStride, w_hi,
                              w_hi + NP2 * kKB * 4, NP2 * 16, c > 0 || j > 0);
        next_stage();
      }
    }
    // both warpgroups are past the last GEMM1 (the __syncthreads above)
    if (more) store_x();
    wgmma_wait<0>();
    acc_fence(acc2);
    ffn_finish<NP2>(p, acc2, cv, row0 + rl, q);
    fence_proxy_async();
    __syncthreads();
  }
}

static inline int pad16(int n) { return (n + 15) / 16 * 16; }

template <int NP2>
static int launch(const Params& p, int tiles, cudaStream_t st) {
  static int resident = 0;  // CTAs that fit on the device at once
  if (!resident) {
    cudaError_t e = cudaFuncSetAttribute(
        ffn_tf32_kernel<NP2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return (int)e;
    e = resident_ctas(ffn_tf32_kernel<NP2>, kThreads, kSmem, &resident);
    if (e != cudaSuccess) return (int)e;
  }
  ffn_tf32_kernel<NP2><<<tiles < resident ? tiles : resident, kThreads, kSmem, st>>>(p);
  return launch_status();
}

}  // namespace ffn
}  // namespace fbbev

using namespace fbbev;

FBBEV_API int fbbev_ffn_supported(int32_t embed, int32_t hidden) {
  return embed > 0 && embed <= ffn::kMaxE && embed % 4 == 0 && hidden > 0 &&
                 hidden % ffn::kHC == 0 && hidden <= ffn::kMaxHidden
             ? 1
             : 0;
}

FBBEV_API int fbbev_ffn_fwd(const float* x, int64_t ldx, const float* w1_packed,
                            const float* b1, const float* w2_packed,
                            const float* b2, const float* residual, int64_t ldr,
                            const float* ln_weight, const float* ln_bias,
                            int64_t m, int32_t embed, int32_t hidden,
                            float ln_eps, float* y, int64_t ldy,
                            fbbev_stream_t stream) {
  if (!x || !w1_packed || !w2_packed || !y || m < 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((ln_weight == nullptr) != (ln_bias == nullptr))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fbbev_ffn_supported(embed, hidden) || m > (int64_t)1 << 30)
    return FBBEV_ERR_UNSUPPORTED;
  if (ldx < embed || ldy < embed || (residual && ldr < embed) || ldx % 4 ||
      ldy % 4 || (residual && ldr % 4))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
       reinterpret_cast<uintptr_t>(w1_packed) |
       reinterpret_cast<uintptr_t>(w2_packed) |
       reinterpret_cast<uintptr_t>(residual)) & 15)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (m == 0) return FBBEV_OK;
  ffn::Params p;
  p.x = x; p.w1p = w1_packed; p.b1 = b1; p.w2p = w2_packed; p.b2 = b2;
  p.residual = residual; p.gamma = ln_weight; p.beta = ln_bias; p.y = y;
  p.M = (int)m; p.E = embed;
  p.n_kb1 = (embed + kKB - 1) / kKB;
  p.n_hc = hidden / ffn::kHC;
  p.ldx = ldx; p.ldr = ldr; p.ldy = ldy; p.eps = ln_eps;
  const int tiles = (int)ceil_div64(m, ffn::kTileM);
  cudaStream_t st = as_stream(stream);
  count_launch();
  switch (ffn::pad16(embed)) {
    case 16: return ffn::launch<16>(p, tiles, st);
    case 32: return ffn::launch<32>(p, tiles, st);
    case 48: return ffn::launch<48>(p, tiles, st);
    case 64: return ffn::launch<64>(p, tiles, st);
    default: return ffn::launch<80>(p, tiles, st);
  }
}
