// linear_tf32.cu -- the row-wise Linears of the backward projection on the
// Hopper tensor cores (wgmma.mma_async, accumulators in registers), fp32 in /
// fp32 out.
//
// What it replaces: every nn.Linear of the BEVFormer encoder layer the reference
// builds for the backward projection -- sampling_offsets / attention_weights /
// value_proj / output_proj of the self- and cross-attention
// (spatial_cross_attention_depth.py:420-427, mmcv MultiScaleDeformableAttention)
// and the FFN (bevformer_encoder.py:251-377 op order) -- together with what
// follows each of them row by row: bias, ReLU, the residual add and the
// LayerNorm(embed_dims).  The reference runs them as cuBLAS fp32 GEMMs plus
// separate elementwise / LayerNorm kernels.
//
// Numerics: the 1e-4 parity bar excludes plain TF32 (10-bit mantissa), so every
// product is formed as 3xTF32 (see wg_kblock_3xtf32, wgmma.cuh): three
// wgmma.mma_async kind tf32 per k8 step into the same fp32 accumulator.
//
// Two kernels, chosen by the shape: for 40 < K <= 80 (every K of the encoder
// layer) linear_tf32_kernel_resident keeps the weights in shared memory and
// forms the A operands in registers (described at the kernel); every other K
// runs linear_tf32_kernel, which streams the weights per K-block.
//
// linear_tf32_kernel: a persistent grid (as many CTAs as are resident at
// once), each CTA looping over 128-row tiles; two warpgroups (rows 0-63 /
// 64-127 of the tile).  The CTA's work is a sequence of steps, one per (tile, 40-float
// K-block), through two shared-memory stages.  In step g each warpgroup issues
// the full-width wgmma's of stage g & 1 (the tile's first with scale-d = 0),
// then, once step g - 1's MMAs have drained, the CTA refills the other stage
// for step g + 1 while step g's run: one thread starts the 1-D bulk copy (TMA)
// of the pre-packed weight block, completion on an mbarrier; all 256 threads
// split the X rows they loaded one step earlier into hi / lo (K-major
// core-matrix layout) and issue the global loads of step g + 2.  So the X
// loads of the next tile are in flight during the MMAs and the epilogue of
// this one.  The epilogue works on the accumulator registers: bias, ReLU,
// residual, LayerNorm, stores of column pairs (optionally two outputs: a
// column split, for two Linears that share their input).
#include "common.cuh"
#include "wgmma.cuh"

namespace fbbev {

constexpr int kChunks = kKB / 4;                 // 16-byte chunks per row
constexpr int kTileM = kATileM;
constexpr int kLinThreads = 256;                 // two warpgroups
constexpr int kMaxN = 192;
constexpr int kMaxLnN = 80;  // widest LayerNorm row (the encoder's embed_dims)

// ------------------------------ weight packing -------------------------------
// W [N][K] row-major -> [k-block][hi, lo][chunk 0..9][Npad / 8][8 rows][4]:
// exactly the shared-memory image of one stage, so a stage's weights are one
// contiguous bulk copy.  Rows >= N and columns >= K are zero.
__global__ void linear_pack_kernel(const float* __restrict__ w, int n, int k,
                                   int npad, int n_kb, float* __restrict__ out) {
  const int64_t total = (int64_t)n_kb * kChunks * npad;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int row = (int)(i % npad);
    const int ch = (int)((i / npad) % kChunks);
    const int kb = (int)(i / ((int64_t)npad * kChunks));
    float hi[4], lo[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = kb * kKB + ch * 4 + j;
      const float v = (row < n && col < k) ? w[(int64_t)row * k + col] : 0.f;
      tf32_split(v, hi[j], lo[j]);
    }
    const int64_t part = (int64_t)kChunks * npad * 4;  // floats of one hi / lo part
    const int64_t off =
        (int64_t)kb * 2 * part + (int64_t)ch * npad * 4 + (row / 8) * 32 + (row % 8) * 4;
    *reinterpret_cast<float4*>(out + off) = make_float4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<float4*>(out + off + part) =
        make_float4(lo[0], lo[1], lo[2], lo[3]);
  }
}

// -------------------------------- the kernel ---------------------------------
struct LinearParams {
  const float* x;         // [M][K]
  const float* x_add;     // [M][K] or null: the GEMM input is x + x_add
  const float* wp;        // packed weights
  const float* bias;      // [N] or null
  const float* residual;  // [M][N] or null
  const float* gamma;     // LayerNorm weight [N] or null
  const float* beta;      // LayerNorm bias [N] or null
  float* y;               // [M][N]
  int M, K, N, n_kb, relu;
  int64_t ldx, ldr, ldy;  // row strides in floats
  int64_t ldxa;           // row stride of x_add
  // optional second output: columns [n_split, N) go to y2 (row stride ldy2)
  float* y2;
  int64_t ldy2;
  int n_split;
  float eps;
  // resident-weight kernel: ring stages per warpgroup and the stage layout
  // (bytes: X rows at 0, x_add rows at xa_off, residual rows at res_off)
  int stages;
  uint32_t stage_bytes, xa_off, res_off;
  // STATS (training forward, fbbev_linear_fwd_ln_train): the normalised rows
  // x^ ([M][N], dense) and 1 / sigma per row ([M]) for the LayerNorm backward
  float* xhat;
  float* rstd;
};

// Epilogue of one tile on the accumulator registers: bias, ReLU, residual,
// LayerNorm (the four lanes of a quad hold one row: two shuffles per
// reduction), column-pair stores (optionally split over two outputs).  `rbase`
// is the thread's first row, q = lane % 4.  `cv` holds bias / gamma / beta
// ([3][NPAD], zero past N) in shared memory.  `res(h, col)` returns residual
// columns col, col + 1 of row rbase + 8 h; it is called from always-valid
// addresses and in batches: a load that sits in a branch in front of its use
// costs a full memory round trip per column pair.  STATS (with LN) also stores
// x^ = (t - mean) / sigma, the value multiplied by gamma, and 1 / sigma.
template <int NPAD, bool LN, bool STATS, typename Res>
__device__ __forceinline__ void linear_epilogue(const LinearParams& p,
                                                const float (&acc)[NPAD / 2],
                                                const float* cv, int rbase, int q,
                                                Res res) {
  constexpr int kBatch = 8;  // residual column pairs in flight per thread
  const int N = p.N;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rbase + 8 * h;
    const bool row_ok = row < p.M;
    float t[NPAD / 4];
#pragma unroll
    for (int J = 0; J < NPAD / 8; ++J) {
      const int col = 8 * J + 2 * q;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        float u = acc[4 * J + 2 * h + e];
        if (p.bias) u += cv[col + e];
        if (p.relu) u = fmaxf(u, 0.f);
        t[2 * J + e] = u;  // columns >= N are neither reduced nor stored
      }
    }
    if (p.residual) {
#pragma unroll
      for (int J0 = 0; J0 < NPAD / 8; J0 += kBatch) {
        float2 r[kBatch];
#pragma unroll
        for (int b = 0; b < kBatch && J0 + b < NPAD / 8; ++b)
          r[b] = res(h, 8 * (J0 + b) + 2 * q);
#pragma unroll
        for (int b = 0; b < kBatch && J0 + b < NPAD / 8; ++b) {
          t[2 * (J0 + b)] += r[b].x;
          t[2 * (J0 + b) + 1] += r[b].y;
        }
      }
    }
    if (LN) {
      // two-pass statistics over the N valid columns; a quad holds the row
      float sum = 0.f;
#pragma unroll
      for (int J = 0; J < NPAD / 8; ++J)
        if (8 * J + 2 * q < N) sum += t[2 * J] + t[2 * J + 1];
      sum += __shfl_xor_sync(kFull, sum, 1);
      sum += __shfl_xor_sync(kFull, sum, 2);
      const float mean = sum / (float)N;
      float sq = 0.f;
#pragma unroll
      for (int J = 0; J < NPAD / 8; ++J)
        if (8 * J + 2 * q < N) {
          const float a = t[2 * J] - mean, b = t[2 * J + 1] - mean;
          sq += a * a + b * b;
        }
      sq += __shfl_xor_sync(kFull, sq, 1);
      sq += __shfl_xor_sync(kFull, sq, 2);
      const float rstd = rsqrtf(sq / (float)N + p.eps);
      float xs[STATS ? NPAD / 4 : 1];
#pragma unroll
      for (int J = 0; J < NPAD / 8; ++J) {
        const int col = 8 * J + 2 * q;
        if (col < N) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float xh = (t[2 * J + e] - mean) * rstd;
            if (STATS) xs[2 * J + e] = xh;
            t[2 * J + e] = fmaf(xh, cv[NPAD + col + e], cv[2 * NPAD + col + e]);
          }
        }
      }
      if (STATS && row_ok) {
        if (q == 0) p.rstd[row] = rstd;
#pragma unroll
        for (int J = 0; J < NPAD / 8; ++J) {
          const int col = 8 * J + 2 * q;
          if (col < N)
            *reinterpret_cast<float2*>(p.xhat + (size_t)row * N + col) =
                make_float2(xs[2 * J], xs[2 * J + 1]);
        }
      }
    }
    if (!row_ok) continue;
#pragma unroll
    for (int J = 0; J < NPAD / 8; ++J) {
      const int col = 8 * J + 2 * q;
      if (col >= N) continue;
      float* dst = col < p.n_split ? p.y + (size_t)row * p.ldy + col
                                   : p.y2 + (size_t)row * p.ldy2 + (col - p.n_split);
      *reinterpret_cast<float2*>(dst) = make_float2(t[2 * J], t[2 * J + 1]);
    }
  }
}

template <int NPAD, bool LN, bool STATS>
__global__ void __launch_bounds__(kLinThreads, 1)
    linear_tf32_kernel(const LinearParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr uint32_t w_part = kb_part(NPAD);              // bytes of W_hi
  constexpr uint32_t stage_bytes = 2u * kAPart + 2u * w_part;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar = smem_u32(smem + 2 * stage_bytes);   // [2] weight stages
  float* cv = reinterpret_cast<float*>(smem + 2 * stage_bytes + 16);  // [3][NPAD]
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_init(bar + 8u, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < 3 * NPAD; i += kLinThreads) {
    const int c = i % NPAD;
    const float* v = i < NPAD ? p.bias : (i < 2 * NPAD ? p.gamma : p.beta);
    cv[i] = v && c < p.N ? __ldg(v + c) : 0.f;
  }
  __syncthreads();

  // The CTA's steps: (tile, K-block) pairs, tiles blockIdx.x, + gridDim.x, ...
  // (the grid is never larger than the tile count); step g uses stage g & 1.
  const int n_kb = p.n_kb;
  const int n_tiles = (p.M + kTileM - 1) / kTileM;
  const int n_steps = (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x * n_kb + n_kb;
  auto issue_w = [&](int g) {
    if (tid == 0 && g < n_steps) {
      const uint32_t s = g & 1;
      mbar_arrive_expect_tx(bar + 8u * s, 2u * w_part);
      bulk_g2s(smem_base + s * stage_bytes + 2u * kAPart,
               p.wp + (size_t)(g % n_kb) * (2u * w_part / 4u), 2u * w_part, bar + 8u * s);
    }
  };
  // X block of step g: 128 rows x 10 chunks of 4 floats, 5 chunks per thread
  float4 v[5];
  auto load_x = [&](int g) {
    if (g >= n_steps) return;
    const int kb = g % n_kb;
    const int row0 = ((int)blockIdx.x + g / n_kb * (int)gridDim.x) * kTileM;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int idx = tid + kLinThreads * i;
      const int r = idx / kChunks, ch = idx - r * kChunks;
      const int g_row = row0 + r, col = kb * kKB + 4 * ch;
      const bool ok = g_row < p.M && col < p.K;
      v[i] = ok ? __ldg(reinterpret_cast<const float4*>(p.x + (size_t)g_row * p.ldx + col))
                : make_float4(0.f, 0.f, 0.f, 0.f);
      if (p.x_add && ok) {  // query + query_pos in the loader (one fp32 add, as torch)
        const float4 a = __ldg(
            reinterpret_cast<const float4*>(p.x_add + (size_t)g_row * p.ldxa + col));
        v[i].x = __fadd_rn(v[i].x, a.x);
        v[i].y = __fadd_rn(v[i].y, a.y);
        v[i].z = __fadd_rn(v[i].z, a.z);
        v[i].w = __fadd_rn(v[i].w, a.w);
      }
    }
  };
  // hi / lo split of the loaded block into stage g & 1 (K-major core matrices)
  auto store_x = [&](int g) {
    if (g >= n_steps) return;
    unsigned char* a_st = smem + (size_t)(g & 1) * stage_bytes;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const int idx = tid + kLinThreads * i;
      const int r = idx / kChunks, ch = idx - r * kChunks;
      const float4 x = v[i];
      float4 hi, lo;
      tf32_split(x.x, hi.x, lo.x);
      tf32_split(x.y, hi.y, lo.y);
      tf32_split(x.z, hi.z, lo.z);
      tf32_split(x.w, hi.w, lo.w);
      const uint32_t off = a_off(r, 4 * ch);
      *reinterpret_cast<float4*>(a_st + off) = hi;
      *reinterpret_cast<float4*>(a_st + off + kAPart) = lo;
    }
  };

  issue_w(0);
  issue_w(1);
  load_x(0);
  store_x(0);
  load_x(1);
  fence_proxy_async();
  __syncthreads();

  float acc[NPAD / 2];  // written first by a scale-d = 0 MMA, never zeroed
  int kb = 0, tile = blockIdx.x;
  for (int g = 0; g < n_steps; ++g) {
    const uint32_t s = g & 1;
    mbar_wait<true>(bar + 8u * s, (g >> 1) & 1u);
    const uint32_t a_hi = smem_base + s * stage_bytes + wg * 1024u;  // 8 row groups
    const uint32_t w_hi = smem_base + s * stage_bytes + 2u * kAPart;
    wgmma_fence();
    wg_kblock_3xtf32<NPAD>(acc, a_hi, a_hi + kAPart, kAChunkStride, w_hi,
                           w_hi + w_part, kb_chunk(NPAD), kb > 0);
    wgmma_commit();
    // step g - 1's MMAs (both warpgroups) have read stage s ^ 1: refill it
    // with step g + 1 while step g's MMAs run, and start the loads of g + 2
    wgmma_wait<1>();
    __syncthreads();
    if (g >= 1) issue_w(g + 1);
    store_x(g + 1);
    load_x(g + 2);
    if (kb == n_kb - 1) {
      wgmma_wait<0>();
      acc_fence(acc);
      const int rbase = tile * kTileM + wg * 64 + wq * 16 + (lane >> 2);
      linear_epilogue<NPAD, LN, STATS>(p, acc, cv, rbase, lane & 3, [&](int h, int col) {
        const int row = rbase + 8 * h;
        const float* src = row < p.M && col < p.N ? p.residual + (size_t)row * p.ldr + col
                                                  : p.residual;
        return __ldg(reinterpret_cast<const float2*>(src));
      });
      kb = 0;
      tile += gridDim.x;
    } else {
      ++kb;
    }
    fence_proxy_async();
    __syncthreads();
  }
  wgmma_wait<0>();  // nothing is pending (the last step ends in an epilogue)
}

// --------------------- resident-weight kernel (40 < K <= 80) ---------------------
// The packed weights (two K-blocks, hi + lo: 10 KB per 16 columns) are copied
// into shared memory once per CTA.  Each warpgroup works on its own 64-row
// tiles (the CTA's tiles alternate between the two), so one warpgroup's
// epilogue overlaps the other's MMAs and nothing synchronises the CTA after
// the set-up.  A tile's rows are staged raw (fp32) in a per-warpgroup ring of
// p.stages stages; within a stage each warp owns the 16 rows its A fragments
// and accumulator rows cover, and fetches them itself: one 1-D bulk copy per
// row and operand (X, x_add, residual), completion on the warp's own
// mbarrier.  A warp reads only its own rows, so a stage needs no "empty"
// barrier: the warp refills it as soon as it has read it -- right after the A
// fragments are in registers when there is no residual, after the epilogue
// otherwise.  The A operand is formed in registers: x (+ x_add, one fp32 add
// as torch), split hi / lo, and the same three MMAs per k8 step as
// wg_kblock_3xtf32 (wg_kblock_3xtf32_rs).  X rows have a pitch of 84 floats,
// which makes the fragment loads free of bank conflicts; residual rows have
// NPAD + 8 (conflict-free float2 loads).
constexpr int kRTileM = 64;
constexpr int kXPitch = 84;
constexpr int kMaxResidentK = 2 * kKB;
constexpr int kMaxStages = 4;
constexpr int kSmemLimit = 227 * 1024;  // opt-in shared memory per CTA (sm_90)

template <int NPAD>
constexpr uint32_t resident_w_bytes() { return 2u * 2u * kb_part(NPAD); }

// The MMAs of one 64-row tile over its two K-blocks, A from the raw stage in
// registers: v = x + x_add (one fp32 add), split hi / lo, columns >= K zero.
// A K-block's fragments are formed before its fence, so the next block's
// shared-memory loads overlap the MMAs of this one.
template <int NPAD>
__device__ __forceinline__ void resident_mma(float (&acc)[NPAD / 2], const float* xs,
                                             const float* xa, int xa_pitch, int rl, int q,
                                             int K, uint32_t w_base) {
  constexpr uint32_t w_part = kb_part(NPAD);
  uint32_t a_hi[2][kKSteps][4], a_lo[2][kKSteps][4];
#pragma unroll
  for (int kb = 0; kb < 2; ++kb) {
#pragma unroll
    for (int k = 0; k < kKSteps; ++k)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = rl + 8 * (e & 1), c = kb * kKB + 8 * k + q + 4 * (e >> 1);
        float v = __fadd_rn(xs[r * kXPitch + c], xa[r * xa_pitch + c]);
        v = c < K ? v : 0.f;
        tf32_split(v, a_hi[kb][k][e], a_lo[kb][k][e]);
      }
    wgmma_fence();
    const uint32_t b_hi = w_base + kb * 2u * w_part;
    wg_kblock_3xtf32_rs<NPAD>(acc, a_hi[kb], a_lo[kb], b_hi, b_hi + w_part, kb_chunk(NPAD),
                              kb > 0);
  }
}

template <int NPAD, bool LN, bool STATS>
__global__ void __launch_bounds__(kLinThreads, 1)
    linear_tf32_kernel_resident(const LinearParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int kResPitch = NPAD + 8;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int S = p.stages;
  const uint32_t ring_bytes = 2u * S * p.stage_bytes;
  unsigned char* ring = smem + resident_w_bytes<NPAD>() + wg * S * p.stage_bytes;
  // mbarriers: [0] weights, then [warpgroup][stage][warp]
  const uint32_t bars = smem_u32(smem + resident_w_bytes<NPAD>() + ring_bytes);
  const uint32_t warp_bar = bars + 8u * (1 + wg * S * 4 + wq);  // + 32 s for stage s
  float* cv = reinterpret_cast<float*>(smem + resident_w_bytes<NPAD>() + ring_bytes +
                                       8 * (1 + 8 * S));  // [3][NPAD]
  float* neg_zero = cv + 3 * NPAD;                         // [kMaxResidentK]
  if (tid == 0) {
    for (int i = 0; i <= 8 * S; ++i) mbar_init(bars + 8u * i, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < 3 * NPAD; i += kLinThreads) {
    const int c = i % NPAD;
    const float* v = i < NPAD ? p.bias : (i < 2 * NPAD ? p.gamma : p.beta);
    cv[i] = v && c < p.N ? __ldg(v + c) : 0.f;
  }
  if (tid < kMaxResidentK) neg_zero[tid] = -0.f;
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bars, resident_w_bytes<NPAD>());
    bulk_g2s(smem_u32(smem), p.wp, resident_w_bytes<NPAD>(), bars);
  }

  // this warpgroup's tiles: blockIdx.x + j gridDim.x for j = wg, wg + 2, ...
  // (the grid is never larger than the tile count)
  const int n_tiles = (p.M + kRTileM - 1) / kRTileM;
  const int n_cta = (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1;
  const int n_it = (n_cta - wg + 1) / 2;
  const int K = p.K;
  const uint32_t x_bytes = 4u * K;
  const uint32_t row_bytes = x_bytes * (p.x_add ? 2u : 1u) + (p.residual ? 4u * p.N : 0u);
  // warp-collective: stage the warp's 16 rows of tile iteration i
  auto fill = [&](int i) {
    if (i >= n_it) return;
    const int s = i % S;
    const int row0 = ((int)blockIdx.x + (2 * i + wg) * (int)gridDim.x) * kRTileM + 16 * wq;
    const int rows = min(16, p.M - row0);  // may be <= 0 in the last tile
    const uint32_t bar = warp_bar + 32u * s;
    __syncwarp();
    fence_proxy_async();  // the warp's reads of this stage before the copies' writes
    if (lane == 0) mbar_arrive_expect_tx(bar, rows > 0 ? rows * row_bytes : 0u);
    __syncwarp();
    if (lane < rows) {
      const int r = row0 + lane, lr = 16 * wq + lane;
      unsigned char* st = ring + s * p.stage_bytes;
      bulk_g2s(smem_u32(st + lr * kXPitch * 4), p.x + (size_t)r * p.ldx, x_bytes, bar);
      if (p.x_add)
        bulk_g2s(smem_u32(st + p.xa_off + lr * kXPitch * 4), p.x_add + (size_t)r * p.ldxa,
                 x_bytes, bar);
      if (p.residual)
        bulk_g2s(smem_u32(st + p.res_off + lr * kResPitch * 4),
                 p.residual + (size_t)r * p.ldr, 4u * p.N, bar);
    }
  };
  for (int i = 0; i < S; ++i) fill(i);
  mbar_wait<true>(bars, 0);

  const int rl = 16 * wq + (lane >> 2);  // stage row of acc[.. + 0 / 1]
  const int q = lane & 3;
  const uint32_t w_base = smem_u32(smem);
  float acc[NPAD / 2];  // written first by a scale-d = 0 MMA, never zeroed
  for (int i = 0; i < n_it; ++i) {
    const int s = i % S;
    mbar_wait<true>(warp_bar + 32u * s, (uint32_t)(i / S) & 1u);
    const unsigned char* st = ring + s * p.stage_bytes;
    const float* xs = reinterpret_cast<const float*>(st);
    // no x_add: add the row of -0 (x + -0 == x for every x), so the loads
    // that define the A registers sit in no branch (ptxas would serialise the
    // MMAs, C7520)
    const float* xa = p.x_add ? reinterpret_cast<const float*>(st + p.xa_off) : neg_zero;
    const int xa_pitch = p.x_add ? kXPitch : 0;
    resident_mma<NPAD>(acc, xs, xa, xa_pitch, rl, q, K, w_base);
    wgmma_commit();
    if (!p.residual) fill(i + S);  // the stage is in registers: refill it now
    wgmma_wait<0>();
    acc_fence(acc);
    const float* rs = reinterpret_cast<const float*>(st + p.res_off);
    const int tile = (int)blockIdx.x + (2 * i + wg) * (int)gridDim.x;
    linear_epilogue<NPAD, LN, STATS>(p, acc, cv, tile * kRTileM + rl, q, [&](int h, int col) {
      return *reinterpret_cast<const float2*>(rs + (rl + 8 * h) * kResPitch + col);
    });
    if (p.residual) fill(i + S);
  }
}

static inline int pad16(int n) { return (n + 15) / 16 * 16; }
static inline int n_kblocks(int k) { return (k + kKB - 1) / kKB; }

// Ring stages per warpgroup of the resident-weight kernel for this call, or
// 0 (the streamed kernel runs) when the weights are not exactly two K-blocks
// (40 < K <= 80) or they and one stage per warpgroup do not fit.
static int resident_layout(LinearParams& p, int npad) {
  if (p.n_kb != 2) return 0;
  const uint32_t x_rows = kRTileM * kXPitch * 4;
  p.xa_off = x_rows;
  p.res_off = p.x_add ? 2 * x_rows : x_rows;
  p.stage_bytes = p.res_off + (p.residual ? kRTileM * (npad + 8) * 4 : 0);
  const int fixed = 2 * 2 * kb_part(npad) + 8 * (1 + 8 * kMaxStages) +
                    (3 * npad + kMaxResidentK) * 4;
  const int s = (kSmemLimit - fixed) / (2 * (int)p.stage_bytes);
  return s < kMaxStages ? s : kMaxStages;
}

template <int NPAD, bool LN, bool STATS>
static int launch_linear_t(const LinearParams& p, cudaStream_t st) {
  if (p.stages > 0) {
    static int resident = 0;  // CTAs that fit on the device at once
    auto kern = linear_tf32_kernel_resident<NPAD, LN, STATS>;
    if (!resident) {
      cudaError_t e = cudaFuncSetAttribute(
          kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
      if (e != cudaSuccess) return (int)e;
      e = resident_ctas(kern, kLinThreads, kSmemLimit, &resident);
      if (e != cudaSuccess) return (int)e;
    }
    const size_t smem = resident_w_bytes<NPAD>() + 2 * (size_t)p.stages * p.stage_bytes +
                        8 * (1 + 8 * p.stages) + (3 * NPAD + kMaxResidentK) * 4;
    const int tiles = (int)ceil_div64(p.M, kRTileM);
    kern<<<tiles < resident ? tiles : resident, kLinThreads, smem, st>>>(p);
    return launch_status();
  }
  constexpr size_t smem =
      2 * (2 * (size_t)kAPart + 2 * (size_t)kb_part(NPAD)) + 16 + 3 * NPAD * 4;
  static int resident = 0;  // CTAs that fit on the device at once
  auto kern = linear_tf32_kernel<NPAD, LN, STATS>;
  if (!resident) {
    cudaError_t e = cudaFuncSetAttribute(
        kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    e = resident_ctas(kern, kLinThreads, smem, &resident);
    if (e != cudaSuccess) return (int)e;
  }
  const int tiles = (int)ceil_div64(p.M, kTileM);
  kern<<<tiles < resident ? tiles : resident, kLinThreads, smem, st>>>(p);
  return launch_status();
}

template <bool LN>
static int launch_linear(const LinearParams& p, int npad, cudaStream_t st) {
  switch (npad) {
    case 16: return launch_linear_t<16, LN, false>(p, st);
    case 32: return launch_linear_t<32, LN, false>(p, st);
    case 48: return launch_linear_t<48, LN, false>(p, st);
    case 64: return launch_linear_t<64, LN, false>(p, st);
    case 80: return launch_linear_t<80, LN, false>(p, st);
    case 96: return launch_linear_t<96, LN, false>(p, st);
    case 112: return launch_linear_t<112, LN, false>(p, st);
    case 128: return launch_linear_t<128, LN, false>(p, st);
    case 144: return launch_linear_t<144, LN, false>(p, st);
    case 160: return launch_linear_t<160, LN, false>(p, st);
    case 176: return launch_linear_t<176, LN, false>(p, st);
    case 192: return launch_linear_t<192, LN, false>(p, st);
    default: return FBBEV_ERR_UNSUPPORTED;
  }
}

// the LayerNorm training forward: rows of up to kMaxLnN columns
static int launch_linear_stats(const LinearParams& p, int npad, cudaStream_t st) {
  switch (npad) {
    case 16: return launch_linear_t<16, true, true>(p, st);
    case 32: return launch_linear_t<32, true, true>(p, st);
    case 48: return launch_linear_t<48, true, true>(p, st);
    case 64: return launch_linear_t<64, true, true>(p, st);
    case 80: return launch_linear_t<80, true, true>(p, st);
    default: return FBBEV_ERR_UNSUPPORTED;
  }
}

}  // namespace fbbev

using namespace fbbev;

FBBEV_API size_t fbbev_linear_packed_bytes(int32_t n, int32_t k) {
  if (n <= 0 || k <= 0) return 0;
  return (size_t)n_kblocks(k) * 2 * kKB * pad16(n) * sizeof(float);
}

FBBEV_API int fbbev_linear_pack(const float* weight, int32_t n, int32_t k,
                                float* packed, fbbev_stream_t stream) {
  if (!weight || !packed || n <= 0 || k <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (reinterpret_cast<uintptr_t>(packed) & 15) return FBBEV_ERR_INVALID_ARGUMENT;
  const int npad = pad16(n), nkb = n_kblocks(k);
  const int64_t total = (int64_t)nkb * kChunks * npad;
  count_launch();
  linear_pack_kernel<<<(unsigned)ceil_div64(total, 256), 256, 0,
                       as_stream(stream)>>>(weight, n, k, npad, nkb, packed);
  return launch_status();
}

static int linear_run(const float* x, int64_t ldx, const float* x_add,
                      int64_t ldxa, const float* packed, const float* bias, const float* residual, int64_t ldr,
                      const float* ln_weight, const float* ln_bias, int64_t m,
                      int32_t k, int32_t n, int32_t relu, float ln_eps, float* y,
                      int64_t ldy, float* y2, int64_t ldy2, int32_t n_split,
                      fbbev_stream_t stream, float* xhat = nullptr,
                      float* rstd = nullptr) {
  if (!x || !packed || !y || m < 0 || k <= 0 || n <= 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((ln_weight == nullptr) != (ln_bias == nullptr))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (k % 4 != 0 || n % 4 != 0 || n > kMaxN || m > (int64_t)1 << 30)
    return FBBEV_ERR_UNSUPPORTED;
  if (ldx < k || ldy < n_split || (residual && ldr < n) || ldx % 4 || ldy % 4 ||
      (residual && ldr % 4))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n_split < n &&
      (!y2 || n_split <= 0 || n_split % 4 || ldy2 < n - n_split || ldy2 % 4 ||
       ln_weight || (reinterpret_cast<uintptr_t>(y2) & 15)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y) |
       reinterpret_cast<uintptr_t>(packed) |
       reinterpret_cast<uintptr_t>(residual) |
       reinterpret_cast<uintptr_t>(x_add)) & 15)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (x_add && (ldxa < k || ldxa % 4)) return FBBEV_ERR_INVALID_ARGUMENT;
  const bool ln = ln_weight != nullptr;
  const bool stats = xhat != nullptr;
  if (stats && (!ln || !rstd || relu || (reinterpret_cast<uintptr_t>(xhat) & 15)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (m == 0) return FBBEV_OK;
  LinearParams p;
  p.x = x; p.x_add = x_add; p.ldxa = ldxa; p.wp = packed; p.bias = bias; p.residual = residual;
  p.gamma = ln_weight; p.beta = ln_bias; p.y = y;
  p.y2 = y2; p.ldy2 = ldy2; p.n_split = n_split;
  p.M = (int)m; p.K = k; p.N = n; p.n_kb = n_kblocks(k);
  p.relu = relu; p.eps = ln_eps;
  p.ldx = ldx; p.ldr = ldr; p.ldy = ldy;
  p.xhat = xhat; p.rstd = rstd;
  if (ln && n > kMaxLnN) return FBBEV_ERR_UNSUPPORTED;
  p.stages = resident_layout(p, pad16(n));
  cudaStream_t st = as_stream(stream);
  count_launch();
  if (stats) return launch_linear_stats(p, pad16(n), st);
  return ln ? launch_linear<true>(p, pad16(n), st) : launch_linear<false>(p, pad16(n), st);
}

FBBEV_API int fbbev_linear_fwd(const float* x, int64_t ldx, const float* packed,
                               const float* bias, const float* residual,
                               int64_t ldr, const float* ln_weight,
                               const float* ln_bias, int64_t m, int32_t k,
                               int32_t n, int32_t relu, float ln_eps, float* y,
                               int64_t ldy, fbbev_stream_t stream) {
  return linear_run(x, ldx, nullptr, 0, packed, bias, residual, ldr, ln_weight,
                    ln_bias, m, k, n, relu, ln_eps, y, ldy, nullptr, 0, n, stream);
}

FBBEV_API int fbbev_linear_fwd_split(const float* x, int64_t ldx,
                                     const float* x_add, int64_t ldx_add,
                                     const float* packed, const float* bias,
                                     int64_t m, int32_t k, int32_t n,
                                     int32_t n_split, int32_t relu, float* y0,
                                     int64_t ldy0, float* y1, int64_t ldy1,
                                     fbbev_stream_t stream) {
  return linear_run(x, ldx, x_add, ldx_add, packed, bias, nullptr, 0, nullptr,
                    nullptr, m, k, n, relu, 0.f, y0, ldy0, y1, ldy1, n_split,
                    stream);
}

FBBEV_API int fbbev_linear_fwd_ln_train(const float* x, int64_t ldx, const float* packed,
                                        const float* bias, const float* residual,
                                        int64_t ldr, const float* ln_weight,
                                        const float* ln_bias, int64_t m, int32_t k,
                                        int32_t n, float ln_eps, float* y, int64_t ldy,
                                        float* xhat, float* rstd, fbbev_stream_t stream) {
  if (!ln_weight || !xhat || !rstd) return FBBEV_ERR_INVALID_ARGUMENT;
  if (n > kMaxLnN) return FBBEV_ERR_UNSUPPORTED;
  return linear_run(x, ldx, nullptr, 0, packed, bias, residual, ldr, ln_weight, ln_bias,
                    m, k, n, 0, ln_eps, y, ldy, nullptr, 0, n, stream, xhat, rstd);
}
