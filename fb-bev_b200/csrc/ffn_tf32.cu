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
//   X       a warpgroup's 64 rows of x, raw fp32 in shared memory (one 1-D bulk
//           copy per row, 84-float pitch: conflict-free fragment loads), split
//           hi / lo (3xTF32, see wgmma.cuh) into GEMM1's register A fragments
//           one K-block at a time
//   GEMM1   per 80-column hidden chunk: H[64 x 80] = X . W1_chunk^T, A from
//           registers, accumulator in registers
//   convert + b1, ReLU, hi / lo split of the accumulator registers into the
//           warpgroup's rows of a shared-memory A tile (K-major core matrices)
//   GEMM2   Y[64 x E] += H_chunk . W2[:, chunk]^T, accumulator in registers
//           across all chunks
//   finish  + b2 + residual, LayerNorm over the quad that holds each row,
//           column-pair stores
//
// The arithmetic is that of a plain chunk-by-chunk loop: per k8 step the three
// products of wg_kblock_3xtf32 in its order, chunks into the GEMM2 accumulator
// in hidden order (register A fragments give the same bits as the
// shared-memory image of the same values).
//
// Work: rows are handed out in 64-row units, a contiguous run of
// floor / ceil(units / grid) per CTA (at M = 40000: 625 units, 4 or 5 per
// CTA, so the call lasts 2.5 steps of 128 rows rather than 3).  A CTA walks its
// run two units per step, warpgroup w taking the step's unit w; when the run
// is odd, warpgroup 1 sits out the last step.
//
// Weights stream through a four-slot ring of 25.6 KB stages (one 1-D bulk
// copy each, in the order the MMAs are issued: per chunk the K-blocks of W1,
// then the two of W2; the sequence runs on across the CTA's steps).  Both
// warpgroups read every stage.  A slot has a "full" mbarrier (tx count) and an
// arrival counter: each warp arrives once the MMAs reading the slot have
// drained, and the warp whose arrival is the eighth refills the slot with the
// stage four places on ("last one out refills": no producer warp, no warp
// waits for a slot to empty).  Nothing synchronises the CTA after set-up; a
// warpgroup's H rows need only a 128-thread named barrier, and each warp waits
// for its own X rows on its own mbarrier.
//
// A warpgroup's chunk g, with GEMM2(g - 1) in flight on entry:
//   issue GEMM1(g) (fragments formed per K-block, behind GEMM2(g - 1))
//   wait for GEMM2(g - 1) only, release W2(g - 1): its slots refill while
//     GEMM1(g) runs
//   wait for GEMM1(g), release W1(g); at a tile edge, finish the previous tile
//   convert g into H, named barrier, issue GEMM2(g)
// Each refill has about one GEMM's MMAs to land in.  The finish and the
// conversion run with the warpgroup's MMAs drained: an accumulator read while
// any wgmma is in flight makes ptxas serialise every MMA (C7514), and a second
// GEMM1 accumulator queued through the conversion does not fit the registers
// beside the fragments at E > 40 (C7512).
//
// Shared memory: X rows (128 x 84 floats, 42 KB) | hidden tile hi / lo
// (80 KB) | weight ring (4 x 25.6 KB) | mbarriers, counters | b1, b2, gamma,
// beta (2.2 KB).
//
// Shapes: E <= 80, E % 4 == 0; hidden % 80 == 0, hidden <= 320.
//
// Training (MODE, a template flag: kInfer is the inference kernel unchanged):
//   kTrainFwd  the same arithmetic; the conversion also stores the hidden
//              activation relu(x . W1^T + b1) (`act`, m x hidden), and the
//              finish stores the normalised row x^ (exactly the value the
//              epilogue multiplies by gamma) and 1 / sigma per row
//   kBwd       the data path of the backward: with W2^T packed in W1's place
//              and W1^T in W2's, x = dz gives GEMM1' dA = dz . W2, the
//              conversion masks it by act > 0 (read from `act`) instead of
//              + b1 / ReLU and stores dh, GEMM2' accumulates dx = dh . W1;
//              the finish adds dz itself when it is passed as the residual
#include "common.cuh"
#include "wgmma.cuh"

namespace fbbev {
namespace ffn {

constexpr int kTileM = kATileM;
constexpr int kUnitM = 64;              // rows per warpgroup and step
constexpr int kThreads = 256;           // two warpgroups
constexpr int kWarps = kThreads / 32;
constexpr int kHC = 80;                 // hidden columns per GEMM1 chunk
constexpr int kMaxE = 80;
constexpr int kMaxHidden = 320;
constexpr int kXPitch = 84;             // floats per X row: conflict-free fragment loads
constexpr int kSlots = 4;
constexpr int kWStage = 2 * kb_part(kHC);          // >= 2 * kb_part(pad16(E))
constexpr int kXBytes = kTileM * kXPitch * 4;
constexpr int kHBytes = (kHC / kKB) * kABlock;
constexpr int kBarBytes = 8 * (kSlots + kWarps) + 4 * kSlots + 16;
constexpr int kCv = kMaxHidden + 3 * kMaxE;         // b1 | b2 | gamma | beta
constexpr int kSmem = kXBytes + kHBytes + kSlots * kWStage + kBarBytes + kCv * 4;
static_assert(kSmem <= 227 * 1024, "opt-in shared memory per CTA (sm_90)");

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
  int M, E, n_hc;
  int64_t ldx, ldr, ldy;
  float eps;
};

constexpr int kInfer = 0, kTrainFwd = 1, kBwd = 2;

// the training modes' extra pointers (dense rows): kTrainFwd writes h_out =
// act, xhat, rstd; kBwd reads act_in and writes h_out = dh.  A struct of its
// own, so the inference kernel's parameters (and code) stay as they are.
struct TrainParams : Params {
  const float* act_in;    // [M][hidden]
  float* h_out;           // [M][hidden]
  float* xhat;            // [M][E] (LayerNorm only)
  float* rstd;            // [M] (LayerNorm only)
};
template <int MODE> struct ParamsFor { using type = TrainParams; };
template <> struct ParamsFor<kInfer> { using type = Params; };

__device__ __forceinline__ void bar_sync_wg(int wg) {
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}
// shared-memory counter add; acq_rel: the arriving warp's drained MMAs come
// before the arrival, and the refill of the last arriver after all of them
__device__ __forceinline__ uint32_t smem_add_acq_rel(uint32_t addr, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], %2;"
               : "=r"(old)
               : "r"(addr), "r"(v)
               : "memory");
  return old;
}

// finish of one tile on the GEMM2 accumulator: + b2 + residual, LayerNorm,
// column-pair stores; `rbase` is the thread's first row, q = lane % 4.  b2 /
// gamma / beta come from shared memory (`cv`, zero past E) and the residual
// loads are issued together from always-valid addresses (see linear_epilogue).
template <int NP2, int MODE, typename P>
__device__ __forceinline__ void ffn_finish(const P& p, const float (&acc2)[NP2 / 2],
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
    float xs[MODE == kTrainFwd ? NP2 / 4 : 1];
    float2 r[NP2 / 8];
    if (p.residual) {
      // columns past E read the row's last pair (their sums are never used)
      const float* res = p.residual + (row_ok ? (size_t)row * p.ldr : 0);
#pragma unroll
      for (int J = 0; J < NP2 / 8; ++J)
        r[J] = __ldg(reinterpret_cast<const float2*>(res + min(8 * J + 2 * q, E - 2)));
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
          for (int e = 0; e < 2; ++e) {
            const float xh = (t[2 * J + e] - mean) * rstd;
            if constexpr (MODE == kTrainFwd) xs[2 * J + e] = xh;
            t[2 * J + e] = fmaf(xh, gamma[col + e], beta[col + e]);
          }
        }
      }
      if constexpr (MODE == kTrainFwd) {
        if (row_ok) {
          if (q == 0) p.rstd[row] = rstd;
#pragma unroll
          for (int J = 0; J < NP2 / 8; ++J) {
            const int col = 8 * J + 2 * q;
            if (col < E)
              *reinterpret_cast<float2*>(p.xhat + (size_t)row * E + col) =
                  make_float2(xs[2 * J], xs[2 * J + 1]);
          }
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

// NP2 = pad16(E); KB1 = 40-float K-blocks of E (GEMM1's stages per chunk)
template <int NP2, int KB1, int MODE>
__global__ void __launch_bounds__(kThreads, 1)
    ffn_tf32_kernel(const typename ParamsFor<MODE>::type p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int per_c = KB1 + kHC / kKB;              // weight stages per chunk
  const float* xrows = reinterpret_cast<const float*>(smem);
  unsigned char* hs = smem + kXBytes;
  const uint32_t hs_a = smem_u32(hs);
  const uint32_t ws_a = hs_a + kHBytes;
  const uint32_t full = ws_a + kSlots * kWStage;      // [slot]
  const uint32_t xbar = full + 8u * kSlots;           // [warp]
  const uint32_t cnt = xbar + 8u * kWarps;            // [slot] arrival counters
  // b1 | b2 | gamma | beta, zero past hidden / E: read by every tile
  float* cv = reinterpret_cast<float*>(hs + kHBytes + kSlots * kWStage + kBarBytes);
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
  const int warp = tid >> 5;
  if (tid == 0) {
    for (int i = 0; i < kSlots + kWarps; ++i) mbar_init(full + 8u * i, 1);
    fence_mbar_init();
  }
  if (tid < kSlots) reinterpret_cast<uint32_t*>(smem + (cnt - smem_u32(smem)))[tid] = 0u;
  for (int i = tid; i < kCv; i += kThreads) {
    const int j = i < kMaxHidden ? i : (i - kMaxHidden) % kMaxE;
    const float* v = i < kMaxHidden ? p.b1
                     : i < kMaxHidden + kMaxE ? p.b2
                     : i < kMaxHidden + 2 * kMaxE ? p.gamma : p.beta;
    const int n = i < kMaxHidden ? p.n_hc * kHC : p.E;
    cv[i] = v && j < n ? __ldg(v + j) : 0.f;
  }
  // the row copies write columns < E only: the columns past E stay zero
  for (int i = tid; i < kXBytes / 16; i += kThreads)
    reinterpret_cast<float4*>(smem)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();

  // this CTA's units [u0, u0 + n_units): steps of two, unit u0 + 2 s + wg
  const int units = (p.M + kUnitM - 1) / kUnitM;
  const int per = units / (int)gridDim.x, extra = units % (int)gridDim.x;
  const int b = blockIdx.x;
  const int u0 = b * per + min(b, extra);
  const int n_units = per + (b < extra ? 1 : 0);
  const int n_hc = p.n_hc;
  const int n_chunks = (n_units + 1) / 2 * n_hc;          // the CTA's chunk sequence
  const int my_chunks = (wg == 0 ? (n_units + 1) / 2 : n_units / 2) * n_hc;
  // stage sequence, in the order the MMAs are issued: per chunk g the K-blocks
  // of W1(g), then the two of W2(g).  Its length is read from shared memory
  // by the refills, so that it takes no register in the chunk loop.
  volatile int* total = reinterpret_cast<int*>(cv) - 4;
  if (tid == 0) *total = n_chunks * per_c;
  __syncthreads();
  auto issue_w = [&](int i) {
    if (i >= *total) return;
    const int g = i / per_c, t = i - g * per_c, c = g % n_hc;
    const float* src;
    uint32_t bytes;
    if (t < KB1) {
      src = p.w1p + (size_t)(c * KB1 + t) * (kWStage / 4);
      bytes = kWStage;
    } else {
      src = p.w2p + (size_t)(c * (kHC / kKB) + t - KB1) * (2 * NP2 * kKB);
      bytes = 2u * kb_part(NP2);
    }
    const uint32_t s = i % kSlots;
    mbar_arrive_expect_tx(full + 8u * s, bytes);
    bulk_g2s(ws_a + s * kWStage, src, bytes, full + 8u * s);
  };
  if (tid == 0)
    for (int i = 0; i < kSlots; ++i) issue_w(i);

  int it = 0;   // next stage to consume
  int rel = 0;  // next stage to release
  auto wait_stage = [&]() { mbar_wait<true>(full + 8u * (it % kSlots), (it / kSlots) & 1u); };
  // the warp's MMAs on stages [rel, rel + n) have drained: arrive; the eighth
  // arrival refills the slot
  auto release = [&](int n) {
    for (int k = 0; k < n; ++k, ++rel) {
      if (lane == 0) {
        const uint32_t old = smem_add_acq_rel(cnt + 4u * (rel % kSlots), 1u);
        if (old % kWarps == kWarps - 1) issue_w(rel + kSlots);
      }
    }
  };
  // stages this warpgroup does not read: still waited for (so the arrivals of
  // one use of a slot never mix with the next) and released
  auto skip = [&](int n) {
    for (int k = 0; k < n; ++k) {
      wait_stage();
      ++it;
      release(1);
    }
  };

  // the warp's 16 X rows of step s, one bulk copy per row
  const float* xw = xrows + (wg * kUnitM + 16 * wq) * kXPitch;
  const uint32_t xb = xbar + 8u * warp;
  auto fill_x = [&](int s) {
    const int row0 = (u0 + 2 * s + wg) * kUnitM + 16 * wq;
    const int rows = min(16, p.M - row0);  // may be <= 0 in the last unit
    __syncwarp();
    fence_proxy_async();  // the warp's reads of its rows before the copies' writes
    if (lane == 0) mbar_arrive_expect_tx(xb, rows > 0 ? rows * 4u * p.E : 0u);
    __syncwarp();
    if (lane < rows)
      bulk_g2s(smem_u32(xw + lane * kXPitch), p.x + (size_t)(row0 + lane) * p.ldx,
               4u * p.E, xb);
  };
  // GEMM1's A fragments of one K-block of chunk gg's tile (hi / lo, columns
  // >= E zero).  A tile's rows are waited for before its first K-block; after
  // its last chunk's last K-block the warp's rows take the next tile's.
  const int my_steps = my_chunks / n_hc;
  auto frag = [&](uint32_t (&fh)[kKSteps][4], uint32_t (&fl)[kKSteps][4], int kb, int gg) {
    const int s = gg / n_hc, c = gg - s * n_hc;
    if (kb == 0 && c == 0) mbar_wait<true>(xb, s & 1);
#pragma unroll
    for (int k = 0; k < kKSteps; ++k)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int r = (lane >> 2) + 8 * (e & 1), col = kb * kKB + 8 * k + q + 4 * (e >> 1);
        tf32_split(xw[r * kXPitch + col], fh[k][e], fl[k][e]);
      }
    if (kb == KB1 - 1 && c == n_hc - 1 && s + 1 < my_steps) fill_x(s + 1);
  };
  // one K-block of GEMM1, one commit group
  auto gemm1 = [&](float (&acc)[kHC / 2], const uint32_t (&fh)[kKSteps][4],
                   const uint32_t (&fl)[kKSteps][4], int kb) {
    wait_stage();
    const uint32_t w_hi = ws_a + (it % kSlots) * kWStage;
    wgmma_fence();
    wg_kblock_3xtf32_rs<kHC>(acc, fh, fl, w_hi, w_hi + kb_part(kHC), kb_chunk(kHC), kb > 0);
    ++it;
    wgmma_commit();
  };

  const int rl = wg * 64 + wq * 16 + (lane >> 2);   // tile row of acc[.. + 0 / 1]
  unsigned char* const h_base = hs + a_off(rl, 2 * q);
  float acc2[NP2 / 2];  // written first by a scale-d = 0 MMA, never zeroed
  uint32_t f0h[kKSteps][4], f0l[kKSteps][4];  // K-block 0 of GEMM1
  uint32_t f1h[kKSteps][4], f1l[kKSteps][4];  // K-block 1 (E > 40)
  float acc1[kHC / 2];  // GEMM1 of the current chunk
  // chunk g; GEMM2(g - 1) in flight on entry
  auto chunk = [&](int g) {
    const int c = g % n_hc;
    frag(f0h, f0l, 0, g);
    gemm1(acc1, f0h, f0l, 0);
    if (KB1 == 2) {
      frag(f1h, f1l, 1, g);
      gemm1(acc1, f1h, f1l, 1);
    }
    if (g > 0) {
      wgmma_wait<KB1>();  // GEMM2(g - 1) has drained, GEMM1(g) stays queued
      release(kHC / kKB);
    }
    wgmma_wait<0>();
    acc_fence(acc1);
    release(KB1);
    if (c == 0 && g > 0) {
      // (after the full drain: ptxas serialises the MMAs when an accumulator
      // is read while any wgmma is in flight, C7514)
      acc_fence(acc2);
      ffn_finish<NP2, MODE>(p, acc2, cv,
                            (u0 + 2 * (g / n_hc - 1) + wg) * kUnitM + rl - wg * 64, q);
    }
    // hidden chunk: + b1, ReLU, hi / lo split -> this warpgroup's rows of hs
    // (a_off(rl + 8 h, 8 J + 2 q + e) as the thread's base + a constant)
    const float* b1c = cv + c * kHC + 2 * q;
    // training: the thread's rows of act / dh, columns c * 80 + 8 J + 2 q + e
    const int hrow = (u0 + 2 * (g / n_hc) + wg) * kUnitM + rl - wg * 64;
    const size_t hcol = (size_t)c * kHC + 2 * q;
    const int64_t ldh = (int64_t)n_hc * kHC;
    float2 mk[MODE == kBwd ? kHC / 4 : 1];
    if constexpr (MODE == kBwd) {
      // the mask's act rows, loaded together from always-valid addresses
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float* src = p.act_in + (size_t)min(hrow + 8 * h, p.M - 1) * ldh + hcol;
#pragma unroll
        for (int J = 0; J < kHC / 8; ++J)
          mk[2 * J + h] = __ldg(reinterpret_cast<const float2*>(src + 8 * J));
      }
    }
#pragma unroll
    for (int J = 0; J < kHC / 8; ++J) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float vv[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float v = acc1[4 * J + 2 * h + e];
          if constexpr (MODE == kBwd) {
            v = (e ? mk[2 * J + h].y : mk[2 * J + h].x) > 0.f ? v : 0.f;
          } else {
            if (p.b1) v += b1c[8 * J + e];
            v = fmaxf(v, 0.f);
          }
          vv[e] = v;
          unsigned char* a = h_base + (J / kKSteps) * kABlock +
                             (J % kKSteps) * 2 * kAChunkStride + h * 128 + e * 4;
          tf32_split(v, *reinterpret_cast<float*>(a), *reinterpret_cast<float*>(a + kAPart));
        }
        if constexpr (MODE != kInfer) {
          if (hrow + 8 * h < p.M)
            *reinterpret_cast<float2*>(p.h_out + (size_t)(hrow + 8 * h) * ldh + hcol + 8 * J) =
                make_float2(vv[0], vv[1]);
        }
      }
    }
    fence_proxy_async();
    bar_sync_wg(wg);
    // recomputed per chunk: hoisted out of the loop, the 20 descriptors would
    // stay live across it
    uint32_t h_a = hs_a + wg * 1024u;
    asm volatile("" : "+r"(h_a));
#pragma unroll
    for (int j = 0; j < kHC / kKB; ++j) {
      wait_stage();
      const uint32_t a_hi = h_a + j * kABlock;
      const uint32_t w_hi = ws_a + (it % kSlots) * kWStage;
      wgmma_fence();
      wg_kblock_3xtf32<NP2>(acc2, a_hi, a_hi + kAPart, kAChunkStride, w_hi,
                            w_hi + kb_part(NP2), kb_chunk(NP2), c > 0 || j > 0);
      ++it;
    }
    wgmma_commit();
  };

  if (my_chunks > 0) {
    fill_x(0);
    for (int g = 0; g < my_chunks; ++g) chunk(g);
    wgmma_wait<0>();
    acc_fence(acc2);
    release(kHC / kKB);
    ffn_finish<NP2, MODE>(p, acc2, cv,
                          (u0 + 2 * (my_chunks / n_hc - 1) + wg) * kUnitM + rl - wg * 64, q);
  }
  skip(*total - it);
}

static inline int pad16(int n) { return (n + 15) / 16 * 16; }

template <int NP2, int KB1, int MODE>
static int launch(const typename ParamsFor<MODE>::type& p, cudaStream_t st) {
  static int resident = 0;  // CTAs that fit on the device at once
  auto kern = ffn_tf32_kernel<NP2, KB1, MODE>;
  if (!resident) {
    cudaError_t e =
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return (int)e;
    e = resident_ctas(kern, kThreads, kSmem, &resident);
    if (e != cudaSuccess) return (int)e;
  }
  const int steps = (int)ceil_div64(p.M, kTileM);  // two 64-row units per CTA at least
  kern<<<steps < resident ? steps : resident, kThreads, kSmem, st>>>(p);
  return launch_status();
}

template <int MODE>
static int dispatch(const typename ParamsFor<MODE>::type& p, cudaStream_t st) {
  const bool two_kb = p.E > kKB;  // GEMM1 over two 40-float K-blocks
  switch (pad16(p.E)) {
    case 16: return launch<16, 1, MODE>(p, st);
    case 32: return launch<32, 1, MODE>(p, st);
    case 48: return two_kb ? launch<48, 2, MODE>(p, st) : launch<48, 1, MODE>(p, st);
    case 64: return launch<64, 2, MODE>(p, st);
    default: return launch<80, 2, MODE>(p, st);
  }
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

static bool misaligned(const void* a, const void* b = nullptr, const void* c = nullptr,
                       const void* d = nullptr, const void* e = nullptr) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) |
           reinterpret_cast<uintptr_t>(c) | reinterpret_cast<uintptr_t>(d) |
           reinterpret_cast<uintptr_t>(e)) & 15) != 0;
}

// the checks and Params of fbbev_ffn_fwd (and of the training forward)
static int ffn_params(ffn::Params& p, const float* x, int64_t ldx, const float* w1_packed,
                      const float* b1, const float* w2_packed, const float* b2,
                      const float* residual, int64_t ldr, const float* ln_weight,
                      const float* ln_bias, int64_t m, int32_t embed, int32_t hidden,
                      float ln_eps, float* y, int64_t ldy) {
  if (!x || !w1_packed || !w2_packed || !y || m < 0)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((ln_weight == nullptr) != (ln_bias == nullptr))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fbbev_ffn_supported(embed, hidden) || m > (int64_t)1 << 30)
    return FBBEV_ERR_UNSUPPORTED;
  if (ldx < embed || ldy < embed || (residual && ldr < embed) || ldx % 4 ||
      ldy % 4 || (residual && ldr % 4))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (misaligned(x, y, w1_packed, w2_packed, residual)) return FBBEV_ERR_INVALID_ARGUMENT;
  p.x = x; p.w1p = w1_packed; p.b1 = b1; p.w2p = w2_packed; p.b2 = b2;
  p.residual = residual; p.gamma = ln_weight; p.beta = ln_bias; p.y = y;
  p.M = (int)m; p.E = embed;
  p.n_hc = hidden / ffn::kHC;
  p.ldx = ldx; p.ldr = ldr; p.ldy = ldy; p.eps = ln_eps;
  return FBBEV_OK;
}

FBBEV_API int fbbev_ffn_fwd(const float* x, int64_t ldx, const float* w1_packed,
                            const float* b1, const float* w2_packed,
                            const float* b2, const float* residual, int64_t ldr,
                            const float* ln_weight, const float* ln_bias,
                            int64_t m, int32_t embed, int32_t hidden,
                            float ln_eps, float* y, int64_t ldy,
                            fbbev_stream_t stream) {
  ffn::Params p;
  const int rc = ffn_params(p, x, ldx, w1_packed, b1, w2_packed, b2, residual, ldr,
                            ln_weight, ln_bias, m, embed, hidden, ln_eps, y, ldy);
  if (rc != FBBEV_OK || m == 0) return rc;
  count_launch();
  return ffn::dispatch<ffn::kInfer>(p, as_stream(stream));
}

FBBEV_API int fbbev_ffn_fwd_train(const float* x, int64_t ldx, const float* w1_packed,
                                  const float* b1, const float* w2_packed,
                                  const float* b2, const float* residual, int64_t ldr,
                                  const float* ln_weight, const float* ln_bias,
                                  int64_t m, int32_t embed, int32_t hidden,
                                  float ln_eps, float* y, int64_t ldy, float* act,
                                  float* xhat, float* rstd, fbbev_stream_t stream) {
  ffn::TrainParams p;
  const int rc = ffn_params(p, x, ldx, w1_packed, b1, w2_packed, b2, residual, ldr,
                            ln_weight, ln_bias, m, embed, hidden, ln_eps, y, ldy);
  if (rc != FBBEV_OK) return rc;
  if (!act || (ln_weight && (!xhat || !rstd)) || misaligned(act, xhat))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (m == 0) return FBBEV_OK;
  p.act_in = nullptr; p.h_out = act; p.xhat = xhat; p.rstd = rstd;
  count_launch();
  return ffn::dispatch<ffn::kTrainFwd>(p, as_stream(stream));
}

FBBEV_API int fbbev_ffn_bwd(const float* dz, int64_t lddz, const float* act,
                            const float* w2t_packed, const float* w1t_packed,
                            int32_t add_dz, int64_t m, int32_t embed, int32_t hidden,
                            float* dh, float* dx, int64_t lddx, fbbev_stream_t stream) {
  ffn::TrainParams p;
  const int rc = ffn_params(p, dz, lddz, w2t_packed, nullptr, w1t_packed, nullptr,
                            add_dz ? dz : nullptr, lddz, nullptr, nullptr, m, embed,
                            hidden, 0.f, dx, lddx);
  if (rc != FBBEV_OK) return rc;
  if (!act || !dh || misaligned(act, dh)) return FBBEV_ERR_INVALID_ARGUMENT;
  if (m == 0) return FBBEV_OK;
  p.act_in = act; p.h_out = dh; p.xhat = nullptr; p.rstd = nullptr;
  count_launch();
  return ffn::dispatch<ffn::kBwd>(p, as_stream(stream));
}
