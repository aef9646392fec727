// history_train.cu -- the training route of FBOCC.fuse_history for a call in
// which every sample is fresh (no history yet, or start_of_sequence): forward
// and backward of the time conv + BN + ReLU and the keyframe-mixing conv, in
// the two-frame form.
//
// A fresh sample's T history frames are T copies of one warped frame x1 with
// one sweep time, so (notation of DESIGN.md §4, frame 0 = the current frame x0)
//   y_f  = Wt[:, :C] x_f + Wt[:, C] * time_f + bt          f = 0, 1
//   BN   train: mu = (S y_0 + T S y_1) / N, var likewise (frame 1 counted T
//        times, N = n (T+1) Z H W); eval: the running statistics
//   h_f  = relu(gamma (y_f - mu) / sigma + beta)
//   Y2   = Wc_0 h_0 + Wbar h_1 + bc,   Wbar = sum_{f>=1} Wc_f
// and backward from g = dL/dY2
//   d_0  = (Wc_0^T g) [h_0 > 0],  d_1 = (Wbar^T g) [h_1 > 0]  (d_1: the T frames' sum)
//   dbeta = S (d_0 + d_1),  dgamma = S (d_0 xhat_0 + d_1 xhat_1)
//   e_f  = gamma / sigma (d_f - k_f dbeta / N - k_f xhat_f dgamma / N),  k_0 = 1,
//          k_1 = T (train; eval drops the /N terms)
//   dcurr = Wt[:, :C]^T e_0
// The weight gradients are products over the n Z H W voxels of the two-frame
// tensors this file writes (h_0, h_1, e_0, e_1) with g, x0 and x1; the caller
// forms them with library GEMMs.
//
// Every product is one kernel, history_train_gemm_kernel: per 128-voxel tile
// of one sample, acc[128 x N] = sum over segments s of A_s . B_s^T, with A_s a
// channel-major (n, K_s, Z H W) tensor read straight into wgmma A fragments
// (3xTF32, split hi / lo in registers) and all of B resident in shared memory
// (fbbev_linear_pack images, one bulk copy per CTA); grid.y selects the frame.
// The epilogue is a template parameter:
//   kStats   y_f; per-channel fp64 sums of y and y^2          (train-mode BN)
//   kHidden  h_f (and xhat_f) to global memory
//   kOut     acc + bias to global memory                      (Y2, dcurr)
//   kDelta   d_f = acc [h_f > 0] to global memory; fp64 sums of d and d xhat
// Channel sums are reduced across the lanes of a warp by shuffles, accumulated
// per warp in shared memory, summed over the warps and written as one partial
// per CTA; history_train_bn_kernel adds the partials in CTA order.  No float
// atomics anywhere: every output is bitwise reproducible for a given device.
#include "common.cuh"
#include "history_warp_bwd.h"
#include "wgmma.cuh"

namespace fbbev {
namespace htrain {

constexpr int kThreads = 256;   // two warpgroups of 64 rows
constexpr int kTileM = 128;
constexpr int kMaxC = 80;
constexpr int kMaxCout = 160;
constexpr int kMaxGrid = 1024;  // partial-sum slots per frame
constexpr int kSmemLimit = 227 * 1024;
constexpr int kCvLen = 160;     // per-channel constant vectors in shared memory
constexpr int kNumCv = 6;       // bias | time_w | mean | invstd | gamma | beta
constexpr int kRedBytes = (kThreads / 32) * 2 * kMaxC * 8;
constexpr size_t kPartBytes = (size_t)2 * kMaxGrid * 2 * kMaxC * sizeof(double);
constexpr size_t kCoefBytes = 8 * kMaxC * sizeof(float);

enum Epi { kStats = 0, kHidden = 1, kOut = 2, kDelta = 3 };

struct Params {
  const float* a[2][2];       // [frame][segment] (n, k_seg, zhw) A operands
  int64_t a_bstride[2][2];    // floats between samples
  const float* w[2];          // [frame] packed B: n_seg * n_kb K-blocks of N rows
  int n_seg, k_seg, n_kb;
  int zhw, tps, n_tiles, ncol;
  const float* time;          // [n]: time of frame 1 (frame 0: 0)
  const float* bias;          // [ncol] or null
  const float* time_w;        // [C]            (kStats, kHidden)
  const float* stats;         // mean[80] | invstd[80]  (kHidden)
  const float* gamma;         // [C] or null (1)
  const float* beta;          // [C] or null (0)
  float* out[2];              // [frame] (n, ncol, zhw)
  float* out2[2];             // [frame] xhat (kHidden) or null
  const float* h[2];          // [frame] h_f (kDelta)
  const float* xhat[2];       // [frame] xhat_f (kDelta)
  double* part;               // [frame][kMaxGrid][2][kMaxC]  (kStats, kDelta)
  // nf > 0: the full route, grid.y = nf frames of one tensor per operand:
  // A = a[0][0] + b a_bstride + f a_fstride, B = w[0] + f w_fstride, time
  // [b nf + f], out / out2 / xhat [0] + b o_bstride + f o_fstride (floats)
  int nf;
  int64_t a_fstride, w_fstride, o_bstride, o_fstride;
  int accum;                  // kOut: acc + out instead of acc + bias (K-chunks)
};

__device__ __forceinline__ double warp_rows_sum(double v) {
  // lanes that share lane % 4 hold the same columns
  v += __shfl_xor_sync(kFull, v, 4);
  v += __shfl_xor_sync(kFull, v, 8);
  v += __shfl_xor_sync(kFull, v, 16);
  return v;
}

template <int N, int EPI>
__global__ void __launch_bounds__(kThreads, 1) history_train_gemm_kernel(const Params p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int kb_bytes = 2 * kb_part(N);
  const int w_bytes = p.n_seg * p.n_kb * kb_bytes;
  const uint32_t w_a = smem_u32(smem);
  float* cv = reinterpret_cast<float*>(smem + w_bytes);
  double* red = reinterpret_cast<double*>(smem + w_bytes + kNumCv * kCvLen * 4);
  const uint32_t bar = w_a + w_bytes + kNumCv * kCvLen * 4 + kRedBytes;
  const int tid = threadIdx.x, f = blockIdx.y;
  const int fs = p.nf ? 0 : f;  // pointer slot of the frame
  const int wg = tid >> 7, warp = tid >> 5, wq = warp & 3, lane = tid & 31, q = lane & 3;
  const int zhw = p.zhw;
  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < kNumCv * kCvLen; i += kThreads) {
    const int k = i / kCvLen, c = i - k * kCvLen;
    float v = 0.f;
    if (k == 0) {
      if (p.bias && c < p.ncol) v = __ldg(p.bias + c);
    } else if (c < kMaxC && EPI != kOut && c < p.ncol) {
      if (k == 1 && EPI != kDelta) v = __ldg(p.time_w + c);
      if (EPI == kHidden) {
        if (k == 2) v = __ldg(p.stats + c);
        if (k == 3) v = __ldg(p.stats + kMaxC + c);
      }
      if (EPI != kStats) {  // kDelta: the ReLU mask from xhat when h is null
        if (k == 4) v = p.gamma ? __ldg(p.gamma + c) : 1.f;
        if (k == 5) v = p.beta ? __ldg(p.beta + c) : 0.f;
      }
    }
    cv[i] = v;
  }
  for (int i = tid; i < kRedBytes / 8; i += kThreads) red[i] = 0.0;
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar, w_bytes);
    bulk_g2s(w_a, p.w[fs] + (p.nf ? f * p.w_fstride : 0), w_bytes, bar);
  }
  const float* bias = cv;
  const float* time_w = cv + kCvLen;
  const float* mean = cv + 2 * kCvLen;
  const float* invstd = cv + 3 * kCvLen;
  const float* gamma = cv + 4 * kCvLen;
  const float* beta = cv + 5 * kCvLen;
  double* red_w = red + warp * 2 * kMaxC;
  mbar_wait<true>(bar, 0);

  const int rl = wg * 64 + wq * 16 + (lane >> 2);  // tile row of acc[.. + 0 / 1]
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int b = tile / p.tps;
    const int v0 = (tile - b * p.tps) * kTileM;
    const int vr0 = min(v0 + rl, zhw - 1), vr1 = min(v0 + rl + 8, zhw - 1);
    const bool ok0 = v0 + rl < zhw, ok1 = v0 + rl + 8 < zhw;
    float acc[N / 2];  // written first by a scale-d = 0 MMA, never zeroed
    for (int s = 0; s < p.n_seg; ++s) {
      const float* base =
          p.a[fs][s] + (int64_t)b * p.a_bstride[fs][s] + (p.nf ? f * p.a_fstride : 0);
      for (int kb = 0; kb < p.n_kb; ++kb) {
        uint32_t ah[kKSteps][4], al[kKSteps][4];
#pragma unroll
        for (int k = 0; k < kKSteps; ++k)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = kb * kKB + 8 * k + q + 4 * (e >> 1);
            const float v =
                c < p.k_seg ? __ldg(base + (int64_t)c * zhw + ((e & 1) ? vr1 : vr0)) : 0.f;
            tf32_split(v, ah[k][e], al[k][e]);
          }
        wgmma_fence();
        const uint32_t b_kb = w_a + (uint32_t)((s * p.n_kb + kb) * kb_bytes);
        wg_kblock_3xtf32_rs<N>(acc, ah, al, b_kb, b_kb + kb_part(N), kb_chunk(N),
                               (s | kb) != 0);
        wgmma_commit();
        wgmma_wait<0>();
      }
    }
    acc_fence(acc);

    const float st = p.nf ? (p.time ? __ldg(p.time + b * p.nf + f) : 0.f)
                          : (f == 1 && p.time ? __ldg(p.time + b) : 0.f);
    const int64_t row0 =
        p.nf ? b * p.o_bstride + f * p.o_fstride : (int64_t)b * p.ncol * zhw;
    if (EPI == kOut) {
#pragma unroll
      for (int J = 0; J < N / 8; ++J)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * J + 2 * q + e;
            if (col < p.ncol && (h ? ok1 : ok0)) {
              float* o = p.out[fs] + row0 + (int64_t)col * zhw + (h ? vr1 : vr0);
              __stcs(o, acc[4 * J + 2 * h + e] + (p.accum ? *o : bias[col]));
            }
          }
    } else if (EPI == kHidden) {
#pragma unroll
      for (int J = 0; J < N / 8; ++J)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * J + 2 * q + e;
            if (col < p.ncol && (h ? ok1 : ok0)) {
              const float y = acc[4 * J + 2 * h + e] + fmaf(time_w[col], st, bias[col]);
              const float xh = (y - mean[col]) * invstd[col];
              const int64_t o = row0 + (int64_t)col * zhw + (h ? vr1 : vr0);
              p.out[fs][o] = fmaxf(fmaf(gamma[col], xh, beta[col]), 0.f);
              if (p.out2[fs]) p.out2[fs][o] = xh;
            }
          }
    } else {  // kStats, kDelta: per-channel sums
#pragma unroll
      for (int J = 0; J < N / 8; ++J)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * J + 2 * q + e;
          double s1 = 0.0, s2 = 0.0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (col < p.ncol && (h ? ok1 : ok0)) {
              if (EPI == kStats) {
                const double y = acc[4 * J + 2 * h + e] + fmaf(time_w[col], st, bias[col]);
                s1 += y;
                s2 += y * y;
              } else {
                const int64_t o = row0 + (int64_t)col * zhw + (h ? vr1 : vr0);
                const float xh = __ldg(p.xhat[fs] + o);
                // h_f > 0, read back or (h null) as the kHidden epilogue forms it
                const bool live = p.h[fs] ? __ldg(p.h[fs] + o) > 0.f
                                          : fmaf(gamma[col], xh, beta[col]) > 0.f;
                const float d = live ? acc[4 * J + 2 * h + e] : 0.f;
                p.out[fs][o] = d;
                s1 += d;
                s2 += (double)d * xh;
              }
            }
          }
          s1 = warp_rows_sum(s1);
          s2 = warp_rows_sum(s2);
          if (lane < 4) {
            red_w[col] += s1;
            red_w[kMaxC + col] += s2;
          }
        }
    }
  }
  if (EPI == kStats || EPI == kDelta) {
    __syncthreads();
    if (tid < 2 * kMaxC) {
      double s = 0.0;
      for (int w = 0; w < kThreads / 32; ++w) s += red[w * 2 * kMaxC + tid];
      p.part[((size_t)f * kMaxGrid + blockIdx.x) * 2 * kMaxC + tid] = s;
    }
  }
}

// The per-channel step between the passes, one CTA:
//   mode 0 (forward, train-mode BN): batch statistics from the kStats partials
//          (frame 1 counted T times), saved as mean | invstd; running
//          statistics updated as torch does (momentum, or the cumulative
//          average 1 / num_batches_tracked when momentum < 0; unbiased var)
//   mode 1 (forward, eval-mode BN): mean | invstd from the running statistics
//   mode 2 (backward): dbeta, dgamma from the kDelta partials and the
//          coefficients of e_f = p d_f + q_f xhat_f + r_f (coef [p|q0|q1|r0|r1])
// The staged pair splits modes 0 and 2 at their sums, for a BN whose
// statistics span several ranks; each rank exports one fp64 row of 2 C + 1:
//   mode 3 (forward, local):  row [S y_0 + T S y_1 | S y_0^2 + T S y_1^2 | count]
//   mode 4 (forward, global): mode 0 from the world rows summed in rank order
//   mode 5 (backward, local): this rank's dbeta, dgamma and row [dbeta | dgamma | count]
//   mode 6 (backward, global): mode 2's coefficients from the rows summed in rank
//          order (dbeta, dgamma stay local, as torch's SyncBatchNorm returns them)
// Every rank sums the same rows in the same order, so mean, invstd and the
// running statistics are bitwise equal across ranks; with world = 1 the rank's
// own row gives exactly the one-shot modes' values.
struct BnParams {
  const double* part;
  int grid, C, T, mode, train;
  double count, eps, momentum;
  const int64_t* nbt;
  float* running_mean;
  float* running_var;
  float* save;          // mean[80] | invstd[80]
  const float* gamma;
  float* coef;          // 5 x 80
  float* dgamma;
  float* dbeta;
  double* row;          // [2 C + 1]            (modes 3, 5)
  const double* rows;   // [world][2 C + 1]     (modes 4, 6)
  int world;
  int nf;               // > 0: the full route's nf frames, each counted once:
                        // all their partials are summed into the frame-0 sums
};

__device__ __forceinline__ void bn_batch_stats(const BnParams& p, int c, double s1, double s2,
                                               double count) {
  const double mean = s1 / count;
  const double var = fmax(s2 / count - mean * mean, 0.0);
  p.save[c] = (float)mean;
  p.save[kMaxC + c] = (float)(1.0 / sqrt(var + p.eps));
  const double m = p.momentum >= 0.0 ? p.momentum : 1.0 / (double)*p.nbt;
  const double unbiased = count > 1.0 ? var * count / (count - 1.0) : var;
  p.running_mean[c] = (float)((1.0 - m) * p.running_mean[c] + m * mean);
  p.running_var[c] = (float)((1.0 - m) * p.running_var[c] + m * unbiased);
}

__device__ __forceinline__ void bn_coefficients(const BnParams& p, int c, double db, double dg,
                                                double count) {
  const double pc = (p.gamma ? (double)p.gamma[c] : 1.0) * (double)p.save[kMaxC + c];
  p.coef[c] = (float)pc;
  for (int f = 0; f < 2; ++f) {
    const double k = p.train ? (f ? (double)p.T : 1.0) / count : 0.0;
    p.coef[(1 + f) * kMaxC + c] = (float)(-pc * k * dg);
    p.coef[(3 + f) * kMaxC + c] = (float)(-pc * k * db);
  }
}

__global__ void history_train_bn_kernel(const BnParams p) {
  const int c = threadIdx.x;
  if (c >= p.C) return;
  double s[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  if (p.mode != 1 && p.nf) {  // every frame into the frame-0 sums
    double a0 = 0.0, a1 = 0.0;
    for (int f = 0; f < p.nf; ++f)
      for (int i = 0; i < p.grid; ++i) {
        const double* q = p.part + ((size_t)f * kMaxGrid + i) * 2 * kMaxC + c;
        a0 += q[0];
        a1 += q[kMaxC];
      }
    s[0][0] = a0;
    s[0][1] = a1;
  } else if (p.mode != 1) {  // grid = 0 in modes 4 and 6
    for (int f = 0; f < 2; ++f)
      for (int i = 0; i < p.grid; ++i)
        for (int k = 0; k < 2; ++k)
          s[f][k] += p.part[((size_t)f * kMaxGrid + i) * 2 * kMaxC + k * kMaxC + c];
  }
  if (p.mode == 0) {
    bn_batch_stats(p, c, s[0][0] + p.T * s[1][0], s[0][1] + p.T * s[1][1], p.count);
  } else if (p.mode == 1) {
    p.save[c] = p.running_mean[c];
    p.save[kMaxC + c] = (float)(1.0 / sqrt((double)p.running_var[c] + p.eps));
  } else if (p.mode == 2) {
    const double db = s[0][0] + s[1][0], dg = s[0][1] + s[1][1];
    p.dbeta[c] = (float)db;
    p.dgamma[c] = (float)dg;
    bn_coefficients(p, c, db, dg, p.count);
  } else if (p.mode == 3 || p.mode == 5) {
    const bool fwd = p.mode == 3;
    const double r0 = fwd ? s[0][0] + p.T * s[1][0] : s[0][0] + s[1][0];
    const double r1 = fwd ? s[0][1] + p.T * s[1][1] : s[0][1] + s[1][1];
    p.row[c] = r0;
    p.row[p.C + c] = r1;
    if (c == 0) p.row[2 * p.C] = p.count;
    if (!fwd) {
      p.dbeta[c] = (float)r0;
      p.dgamma[c] = (float)r1;
    }
  } else {  // modes 4, 6
    const int w = 2 * p.C + 1;
    double r0 = p.rows[c], r1 = p.rows[p.C + c], count = p.rows[2 * p.C];
    for (int r = 1; r < p.world; ++r) {
      r0 += p.rows[(size_t)r * w + c];
      r1 += p.rows[(size_t)r * w + p.C + c];
      count += p.rows[(size_t)r * w + 2 * p.C];
    }
    if (p.mode == 4)
      bn_batch_stats(p, c, r0, r1, count);
    else
      bn_coefficients(p, c, r0, r1, count);
  }
}

// e_f = p d_f + q_f xhat_f + r_f, in place over d_f; grid.y = frame.  The
// tensors hold cs channels per sample (C, or the full route's (T+1) C with
// grid.y = 1: every frame takes q_0, r_0)
__global__ void history_train_e_kernel(float* e0, float* e1, const float* x0, const float* x1,
                                       const float* coef, int C, int cs, int zhw,
                                       int64_t total) {
  const int f = blockIdx.y;
  float* e = f ? e1 : e0;
  const float* xh = f ? x1 : x0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)((i / zhw) % cs) % C;
    e[i] = fmaf(__ldg(coef + c), e[i],
                fmaf(__ldg(coef + (1 + f) * kMaxC + c), __ldg(xh + i),
                     __ldg(coef + (3 + f) * kMaxC + c)));
  }
}

// One persistent launch: grid.x = min(tiles, resident CTAs, kMaxGrid), grid.y =
// frames.  *grid receives grid.x (the partial-sum slots a kStats / kDelta
// launch fills).
template <int N, int EPI>
static int launch_gemm(const Params& p, int frames, cudaStream_t st, int* grid = nullptr) {
  auto kern = history_train_gemm_kernel<N, EPI>;
  // CTAs resident at once, per number of resident weight K-blocks (the only
  // thing the shared memory depends on; n_seg * n_kb <= 2 * 4)
  static int resident[9] = {};
  const int blocks = p.n_seg * p.n_kb;
  const int smem = blocks * 2 * kb_part(N) + kNumCv * kCvLen * 4 + kRedBytes + 16;
  if (blocks > 8 || smem > kSmemLimit) return FBBEV_ERR_UNSUPPORTED;
  if (!resident[blocks]) {
    cudaError_t e =
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemLimit);
    if (e == cudaSuccess) e = resident_ctas(kern, kThreads, smem, &resident[blocks]);
    if (e != cudaSuccess) return (int)e;
  }
  int g = p.n_tiles < resident[blocks] ? p.n_tiles : resident[blocks];
  if (g > kMaxGrid) g = kMaxGrid;
  if (grid) *grid = g;
  count_launch();
  kern<<<dim3(g, frames), kThreads, smem, st>>>(p);
  return launch_status();
}

static Params base_params(int n, int zhw) {
  Params p = {};
  p.zhw = zhw;
  p.tps = (int)ceil_div64(zhw, kTileM);
  p.n_tiles = n * p.tps;
  return p;
}

static int launch_bn(const BnParams& b, cudaStream_t st) {
  count_launch();
  history_train_bn_kernel<<<1, 128, 0, st>>>(b);
  return launch_status();
}

}  // namespace htrain
}  // namespace fbbev

using namespace fbbev;
using namespace fbbev::htrain;

FBBEV_API size_t fbbev_history_train_workspace_bytes(int32_t n, int32_t c, int32_t Z,
                                                     int32_t H, int32_t W) {
  if (n < 0 || c <= 0 || Z <= 0 || H <= 0 || W <= 0) return 0;
  return kPartBytes + kCoefBytes + (size_t)2 * n * c * Z * H * W * sizeof(float);
}

static int check_shape(int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H,
                       int32_t W) {
  if (n < 0 || T < 1 || Z <= 0 || H <= 0 || W <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fbbev_history_fuse_supported(c, c_out)) return FBBEV_ERR_UNSUPPORTED;
  const int64_t zhw = (int64_t)Z * H * W;
  if (zhw >= ((int64_t)1 << 31) || n > 65535 ||
      n * ceil_div64(zhw, kTileM) >= ((int64_t)1 << 31))
    return FBBEV_ERR_UNSUPPORTED;
  return FBBEV_OK;
}

static bool aligned16(const void* a) { return (reinterpret_cast<uintptr_t>(a) & 15) == 0; }

FBBEV_API int fbbev_history_train_fwd(
    const float* x0, int64_t x0_batch_stride, const float* x1, int64_t x1_batch_stride,
    const float* time, const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wc_packed, const float* bias_c, const float* gamma, const float* beta,
    float* running_mean, float* running_var, const int64_t* num_batches_tracked,
    double momentum, double eps, int32_t train, int32_t n, int32_t T, int32_t c,
    int32_t c_out, int32_t Z, int32_t H, int32_t W, float* out, float* save,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = check_shape(n, T, c, c_out, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  const int zhw = Z * H * W;
  if (x0_batch_stride < (int64_t)c * zhw || x1_batch_stride < (int64_t)c * zhw)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n == 0) return FBBEV_OK;
  if (!x0 || !x1 || !time || !wt_packed || !bias_t || !time_w || !wc_packed || !bias_c ||
      !running_mean || !running_var || !out || !save || !workspace ||
      (train && !num_batches_tracked))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!aligned16(wt_packed) || !aligned16(wc_packed) || !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_workspace_bytes(n, c, Z, H, W))
    return FBBEV_ERR_INVALID_ARGUMENT;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  float* h0 = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes + kCoefBytes);
  float* h1 = h0 + (size_t)n * c * zhw;

  Params g = base_params(n, zhw);  // y_f / h_f = f(x_f . Wt^T), frames 0 and 1
  g.a[0][0] = x0; g.a_bstride[0][0] = x0_batch_stride;
  g.a[1][0] = x1; g.a_bstride[1][0] = x1_batch_stride;
  g.w[0] = g.w[1] = wt_packed;
  g.n_seg = 1; g.k_seg = c; g.n_kb = (c + kKB - 1) / kKB; g.ncol = c;
  g.time = time; g.bias = bias_t; g.time_w = time_w;
  BnParams b = {};
  b.C = c; b.T = T; b.eps = eps; b.momentum = momentum; b.nbt = num_batches_tracked;
  b.running_mean = running_mean; b.running_var = running_var; b.save = save;
  b.count = (double)n * (T + 1) * zhw;
  if (train) {
    g.part = part;
    if ((rc = launch_gemm<kMaxC, kStats>(g, 2, st, &b.grid)) != FBBEV_OK) return rc;
    b.part = part;
    b.mode = 0;
  } else {
    b.mode = 1;
  }
  if ((rc = launch_bn(b, st)) != FBBEV_OK) return rc;
  g.stats = save; g.gamma = gamma; g.beta = beta;
  g.out[0] = h0; g.out[1] = h1;
  if ((rc = launch_gemm<kMaxC, kHidden>(g, 2, st)) != FBBEV_OK) return rc;

  Params y = base_params(n, zhw);  // Y2 = [h_0 | h_1] . [Wc_0 | Wbar]^T + bc
  y.a[0][0] = h0; y.a[0][1] = h1;
  y.a_bstride[0][0] = y.a_bstride[0][1] = (int64_t)c * zhw;
  y.w[0] = wc_packed;
  y.n_seg = 2; y.k_seg = c; y.n_kb = (c + kKB - 1) / kKB; y.ncol = c_out;
  y.bias = bias_c; y.out[0] = out;
  return c_out > kMaxC ? launch_gemm<kMaxCout, kOut>(y, 1, st)
                       : launch_gemm<kMaxC, kOut>(y, 1, st);
}

FBBEV_API int fbbev_history_train_bwd(
    const float* x0, int64_t x0_batch_stride, const float* x1, int64_t x1_batch_stride,
    const float* time, const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wct_packed, const float* wtt_packed, const float* gamma, const float* beta,
    const float* save, int32_t train, int32_t n, int32_t T, int32_t c, int32_t c_out,
    int32_t Z, int32_t H, int32_t W, const float* grad_out, float* h0, float* h1, float* e0,
    float* e1, float* grad_curr, float* grad_gamma, float* grad_beta, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = check_shape(n, T, c, c_out, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  const int zhw = Z * H * W;
  if (x0_batch_stride < (int64_t)c * zhw || x1_batch_stride < (int64_t)c * zhw)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n == 0) return FBBEV_OK;
  if (!x0 || !x1 || !time || !wt_packed || !bias_t || !time_w || !wct_packed ||
      (grad_curr && !wtt_packed) || !save || !grad_out || !h0 || !h1 || !e0 || !e1 ||
      !grad_gamma || !grad_beta || !workspace)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (!aligned16(wt_packed) || !aligned16(wct_packed) ||
      (grad_curr && !aligned16(wtt_packed)) || !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_workspace_bytes(n, c, Z, H, W))
    return FBBEV_ERR_INVALID_ARGUMENT;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  float* coef = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes);
  float* xh0 = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes + kCoefBytes);
  float* xh1 = xh0 + (size_t)n * c * zhw;
  const int64_t dense = (int64_t)c * zhw;

  Params g = base_params(n, zhw);  // recompute h_f, xhat_f
  g.a[0][0] = x0; g.a_bstride[0][0] = x0_batch_stride;
  g.a[1][0] = x1; g.a_bstride[1][0] = x1_batch_stride;
  g.w[0] = g.w[1] = wt_packed;
  g.n_seg = 1; g.k_seg = c; g.n_kb = (c + kKB - 1) / kKB; g.ncol = c;
  g.time = time; g.bias = bias_t; g.time_w = time_w;
  g.stats = save; g.gamma = gamma; g.beta = beta;
  g.out[0] = h0; g.out[1] = h1; g.out2[0] = xh0; g.out2[1] = xh1;
  if ((rc = launch_gemm<kMaxC, kHidden>(g, 2, st)) != FBBEV_OK) return rc;

  Params d = base_params(n, zhw);  // d_f = (Wc_f^T g) [h_f > 0] into e_f; sums
  const size_t wct_floats = fbbev_linear_packed_bytes(kMaxC, c_out) / sizeof(float);
  d.a[0][0] = d.a[1][0] = grad_out;
  d.a_bstride[0][0] = d.a_bstride[1][0] = (int64_t)c_out * zhw;
  d.w[0] = wct_packed; d.w[1] = wct_packed + wct_floats;
  d.n_seg = 1; d.k_seg = c_out; d.n_kb = (c_out + kKB - 1) / kKB; d.ncol = c;
  d.out[0] = e0; d.out[1] = e1; d.h[0] = h0; d.h[1] = h1; d.xhat[0] = xh0; d.xhat[1] = xh1;
  d.part = part;
  BnParams b = {};
  b.C = c; b.T = T; b.mode = 2; b.train = train; b.save = const_cast<float*>(save);  // read only in mode 2
  b.gamma = gamma;
  b.count = (double)n * (T + 1) * zhw; b.part = part; b.coef = coef;
  b.dgamma = grad_gamma; b.dbeta = grad_beta;
  rc = launch_gemm<kMaxC, kDelta>(d, 2, st, &b.grid);
  if (rc == FBBEV_OK) rc = launch_bn(b, st);
  if (rc != FBBEV_OK) return rc;

  const int64_t total = (int64_t)n * dense;
  count_launch();
  const int64_t blocks = ceil_div64(total, 256);
  history_train_e_kernel<<<dim3((unsigned)(blocks < 4096 ? blocks : 4096), 2), 256, 0, st>>>(e0, e1, xh0, xh1, coef, c, c, zhw, total);
  if ((rc = launch_status()) != FBBEV_OK) return rc;
  if (!grad_curr) return FBBEV_OK;

  Params x = base_params(n, zhw);  // dcurr = e_0 . Wt[:, :C]
  x.a[0][0] = e0; x.a_bstride[0][0] = dense;
  x.w[0] = wtt_packed;
  x.n_seg = 1; x.k_seg = c; x.n_kb = (c + kKB - 1) / kKB; x.ncol = c;
  x.out[0] = grad_curr;
  return launch_gemm<kMaxC, kOut>(x, 1, st);
}

// -- the staged pair, for a time BN whose statistics span several ranks ------
// Each pass is split at its one statistics step (modes 3 / 4 and 5 / 6 of
// history_train_bn_kernel); the caller gathers the ranks' rows in between.

static Params frame_params(const float* x0, int64_t x0_batch_stride, const float* x1,
                           int64_t x1_batch_stride, const float* time, const float* wt_packed,
                           const float* bias_t, const float* time_w, int n, int c, int zhw) {
  Params g = base_params(n, zhw);  // y_f = x_f . Wt^T + time_f Wt[:, c] + bt, f = 0, 1
  g.a[0][0] = x0; g.a_bstride[0][0] = x0_batch_stride;
  g.a[1][0] = x1; g.a_bstride[1][0] = x1_batch_stride;
  g.w[0] = g.w[1] = wt_packed;
  g.n_seg = 1; g.k_seg = c; g.n_kb = (c + kKB - 1) / kKB; g.ncol = c;
  g.time = time; g.bias = bias_t; g.time_w = time_w;
  return g;
}

static int check_frames(const float* x0, int64_t x0_batch_stride, const float* x1,
                        int64_t x1_batch_stride, const float* time, const float* wt_packed,
                        const float* bias_t, const float* time_w, int32_t n, int32_t T,
                        int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
                        const void* workspace, size_t workspace_bytes) {
  const int rc = check_shape(n, T, c, c_out, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  const int64_t dense = (int64_t)c * Z * H * W;
  if (x0_batch_stride < dense || x1_batch_stride < dense || !workspace ||
      !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_workspace_bytes(n, c, Z, H, W))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n > 0 && (!x0 || !x1 || !time || !wt_packed || !bias_t || !time_w ||
                !aligned16(wt_packed)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return FBBEV_OK;
}

FBBEV_API int fbbev_history_train_fwd_local(
    const float* x0, int64_t x0_batch_stride, const float* x1, int64_t x1_batch_stride,
    const float* time, const float* wt_packed, const float* bias_t, const float* time_w,
    int32_t n, int32_t T, int32_t c, int32_t Z, int32_t H, int32_t W, double* row,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  if (!row) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_frames(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                        time_w, n, T, c, c, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  BnParams b = {};
  b.C = c; b.T = T; b.mode = 3; b.part = part; b.row = row;
  b.count = (double)n * (T + 1) * zhw;
  if (n > 0) {  // n = 0: a zero row (no partials)
    Params g = frame_params(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                            time_w, n, c, zhw);
    g.part = part;
    if ((rc = launch_gemm<kMaxC, kStats>(g, 2, st, &b.grid)) != FBBEV_OK) return rc;
  }
  return launch_bn(b, st);
}

FBBEV_API int fbbev_history_train_fwd_global(
    const float* x0, int64_t x0_batch_stride, const float* x1, int64_t x1_batch_stride,
    const float* time, const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wc_packed, const float* bias_c, const float* gamma, const float* beta,
    float* running_mean, float* running_var, const int64_t* num_batches_tracked,
    double momentum, double eps, const double* rows, int32_t world, int32_t n, int32_t T,
    int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W, float* out, float* save,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  if (world < 1 || !rows) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_frames(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                        time_w, n, T, c, c_out, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (!running_mean || !running_var || !num_batches_tracked || !save ||
      (n > 0 && (!wc_packed || !bias_c || !out || !aligned16(wc_packed))))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  BnParams b = {};
  b.C = c; b.T = T; b.mode = 4; b.rows = rows; b.world = world;
  b.eps = eps; b.momentum = momentum; b.nbt = num_batches_tracked;
  b.running_mean = running_mean; b.running_var = running_var; b.save = save;
  if ((rc = launch_bn(b, st)) != FBBEV_OK || n == 0) return rc;

  float* h0 = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes + kCoefBytes);
  float* h1 = h0 + (size_t)n * c * zhw;
  Params g = frame_params(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                          time_w, n, c, zhw);
  g.stats = save; g.gamma = gamma; g.beta = beta;
  g.out[0] = h0; g.out[1] = h1;
  if ((rc = launch_gemm<kMaxC, kHidden>(g, 2, st)) != FBBEV_OK) return rc;

  Params y = base_params(n, zhw);  // Y2 = [h_0 | h_1] . [Wc_0 | Wbar]^T + bc
  y.a[0][0] = h0; y.a[0][1] = h1;
  y.a_bstride[0][0] = y.a_bstride[0][1] = (int64_t)c * zhw;
  y.w[0] = wc_packed;
  y.n_seg = 2; y.k_seg = c; y.n_kb = (c + kKB - 1) / kKB; y.ncol = c_out;
  y.bias = bias_c; y.out[0] = out;
  return c_out > kMaxC ? launch_gemm<kMaxCout, kOut>(y, 1, st)
                       : launch_gemm<kMaxC, kOut>(y, 1, st);
}

FBBEV_API int fbbev_history_train_bwd_local(
    const float* x0, int64_t x0_batch_stride, const float* x1, int64_t x1_batch_stride,
    const float* time, const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wct_packed, const float* gamma, const float* beta, const float* save,
    int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
    const float* grad_out, float* h0, float* h1, float* e0, float* e1, float* grad_gamma,
    float* grad_beta, double* row, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (!row) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_frames(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                        time_w, n, T, c, c_out, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (!save || !grad_gamma || !grad_beta ||
      (n > 0 && (!wct_packed || !grad_out || !h0 || !h1 || !e0 || !e1 ||
                 !aligned16(wct_packed))))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  float* xh0 = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes + kCoefBytes);
  float* xh1 = xh0 + (size_t)n * c * zhw;
  BnParams b = {};
  b.C = c; b.T = T; b.mode = 5; b.part = part; b.row = row;
  b.count = (double)n * (T + 1) * zhw;
  b.dgamma = grad_gamma; b.dbeta = grad_beta;
  if (n > 0) {
    Params g = frame_params(x0, x0_batch_stride, x1, x1_batch_stride, time, wt_packed, bias_t,
                            time_w, n, c, zhw);  // recompute h_f, xhat_f
    g.stats = save; g.gamma = gamma; g.beta = beta;
    g.out[0] = h0; g.out[1] = h1; g.out2[0] = xh0; g.out2[1] = xh1;
    if ((rc = launch_gemm<kMaxC, kHidden>(g, 2, st)) != FBBEV_OK) return rc;

    Params d = base_params(n, zhw);  // d_f = (Wc_f^T g) [h_f > 0] into e_f; sums
    const size_t wct_floats = fbbev_linear_packed_bytes(kMaxC, c_out) / sizeof(float);
    d.a[0][0] = d.a[1][0] = grad_out;
    d.a_bstride[0][0] = d.a_bstride[1][0] = (int64_t)c_out * zhw;
    d.w[0] = wct_packed; d.w[1] = wct_packed + wct_floats;
    d.n_seg = 1; d.k_seg = c_out; d.n_kb = (c_out + kKB - 1) / kKB; d.ncol = c;
    d.out[0] = e0; d.out[1] = e1; d.h[0] = h0; d.h[1] = h1; d.xhat[0] = xh0; d.xhat[1] = xh1;
    d.part = part;
    if ((rc = launch_gemm<kMaxC, kDelta>(d, 2, st, &b.grid)) != FBBEV_OK) return rc;
  }
  return launch_bn(b, st);
}

FBBEV_API int fbbev_history_train_bwd_global(
    const float* wtt_packed, const float* gamma, const float* save, const double* rows,
    int32_t world, int32_t n, int32_t T, int32_t c, int32_t Z, int32_t H, int32_t W, float* e0,
    float* e1, float* grad_curr, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (world < 1 || !rows) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_shape(n, T, c, c, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  if (!save || !workspace || !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_workspace_bytes(n, c, Z, H, W) ||
      (n > 0 && (!e0 || !e1 || (grad_curr && (!wtt_packed || !aligned16(wtt_packed))))))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  float* coef = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes);
  float* xh0 = reinterpret_cast<float*>(static_cast<char*>(workspace) + kPartBytes + kCoefBytes);
  float* xh1 = xh0 + (size_t)n * c * zhw;
  BnParams b = {};
  b.C = c; b.T = T; b.mode = 6; b.train = 1; b.rows = rows; b.world = world;
  b.save = const_cast<float*>(save);  // read only in mode 6
  b.gamma = gamma; b.coef = coef;
  if ((rc = launch_bn(b, st)) != FBBEV_OK || n == 0) return rc;

  const int64_t dense = (int64_t)c * zhw;
  const int64_t total = (int64_t)n * dense;
  count_launch();
  const int64_t blocks = ceil_div64(total, 256);
  history_train_e_kernel<<<dim3((unsigned)(blocks < 4096 ? blocks : 4096), 2), 256, 0, st>>>(
      e0, e1, xh0, xh1, coef, c, c, zhw, total);
  if ((rc = launch_status()) != FBBEV_OK) return rc;
  if (!grad_curr) return FBBEV_OK;

  Params x = base_params(n, zhw);  // dcurr = e_0 . Wt[:, :C]
  x.a[0][0] = e0; x.a_bstride[0][0] = dense;
  x.w[0] = wtt_packed;
  x.n_seg = 1; x.k_seg = c; x.n_kb = (c + kKB - 1) / kKB; x.ncol = c;
  x.out[0] = grad_curr;
  return launch_gemm<kMaxC, kOut>(x, 1, st);
}

// -- the full route: every sample's T + 1 frames, fresh or not -----------------
// The frames are channel slices [f c, (f+1) c) of one (n, (T+1) c, Z, H, W)
// tensor (the concatenation buffer), time is (n, T+1), and every frame is
// counted once in the statistics; the GEMM, BN and e kernels are those of the
// two-frame route with grid.y = T + 1 (Params::nf, BnParams::nf).  The cat
// conv's K = (T+1) c does not fit in shared memory: it runs as K-chunks of two
// frames, each a two-segment kOut launch with the two-frame route's resident
// B, accumulating into out.  Workspace: per-frame partial slots | coef | one
// (n, (T+1) c, Z H W) tensor (h_f in the forward, xhat_f in the backward).

static size_t full_part_bytes(int T) {
  return (size_t)(T + 1) * kMaxGrid * 2 * kMaxC * sizeof(double);
}

static float* full_coef(void* ws, int T) {
  return reinterpret_cast<float*>(static_cast<char*>(ws) + full_part_bytes(T));
}

static float* full_frames_buf(void* ws, int T) {
  return reinterpret_cast<float*>(static_cast<char*>(ws) + full_part_bytes(T) + kCoefBytes);
}

FBBEV_API size_t fbbev_history_train_full_workspace_bytes(int32_t n, int32_t T, int32_t c,
                                                          int32_t Z, int32_t H, int32_t W) {
  if (n < 0 || T < 1 || T >= 65535 || c <= 0 || Z <= 0 || H <= 0 || W <= 0) return 0;
  return full_part_bytes(T) + kCoefBytes +
         (size_t)n * (T + 1) * c * Z * H * W * sizeof(float);
}

static int check_full(const float* x, int64_t x_batch_stride, const float* time,
                      const float* wt_packed, const float* bias_t, const float* time_w,
                      int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H,
                      int32_t W, const void* workspace, size_t workspace_bytes) {
  const int rc = check_shape(n, T, c, c_out, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  if (T >= 65535) return FBBEV_ERR_UNSUPPORTED;  // grid.y = T + 1
  if (x_batch_stride < (int64_t)(T + 1) * c * Z * H * W || !workspace ||
      !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_full_workspace_bytes(n, T, c, Z, H, W))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n > 0 && (!x || !time || !wt_packed || !bias_t || !time_w || !aligned16(wt_packed)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return FBBEV_OK;
}

// y_f = x_f . Wt^T + time_f Wt[:, c] + bt over the T + 1 frames; h_f, xhat_f
// and d_f, e_f laid out as x, densely
static Params full_frame_params(const float* x, int64_t x_batch_stride, const float* time,
                                const float* wt_packed, const float* bias_t,
                                const float* time_w, int n, int T, int c, int zhw) {
  Params g = base_params(n, zhw);
  g.nf = T + 1;
  g.a[0][0] = x; g.a_bstride[0][0] = x_batch_stride; g.a_fstride = (int64_t)c * zhw;
  g.w[0] = wt_packed;
  g.n_seg = 1; g.k_seg = c; g.n_kb = (c + kKB - 1) / kKB; g.ncol = c;
  g.time = time; g.bias = bias_t; g.time_w = time_w;
  g.o_bstride = (int64_t)(T + 1) * c * zhw; g.o_fstride = (int64_t)c * zhw;
  return g;
}

// Y2 = sum_f h_f . Wc_f^T + bc: two frames per launch, the first launch
// adding bc, the others adding out
static int full_cat_conv(const float* h, const float* wc_packed, const float* bias_c, int n,
                         int T, int c, int c_out, int zhw, float* out, cudaStream_t st) {
  const int F = T + 1;
  const size_t per = fbbev_linear_packed_bytes(c_out > kMaxC ? kMaxCout : kMaxC, c) / sizeof(float);
  const int64_t dense = (int64_t)c * zhw;
  for (int f0 = 0; f0 < F; f0 += 2) {
    Params y = base_params(n, zhw);
    y.n_seg = F - f0 < 2 ? F - f0 : 2;
    for (int s = 0; s < y.n_seg; ++s) {
      y.a[0][s] = h + (f0 + s) * dense;
      y.a_bstride[0][s] = F * dense;
    }
    y.w[0] = wc_packed + f0 * per;
    y.k_seg = c; y.n_kb = (c + kKB - 1) / kKB; y.ncol = c_out;
    y.bias = bias_c; y.out[0] = out; y.accum = f0 > 0;
    const int rc = c_out > kMaxC ? launch_gemm<kMaxCout, kOut>(y, 1, st)
                                 : launch_gemm<kMaxC, kOut>(y, 1, st);
    if (rc != FBBEV_OK) return rc;
  }
  return FBBEV_OK;
}

static int full_fwd_tail(const Params& frames, const float* save, const float* gamma,
                         const float* beta, const float* wc_packed, const float* bias_c, int n,
                         int T, int c, int c_out, int zhw, float* out, void* workspace,
                         cudaStream_t st) {
  Params g = frames;
  float* h = full_frames_buf(workspace, T);
  g.stats = save; g.gamma = gamma; g.beta = beta; g.out[0] = h;
  int rc = launch_gemm<kMaxC, kHidden>(g, T + 1, st);
  if (rc != FBBEV_OK) return rc;
  return full_cat_conv(h, wc_packed, bias_c, n, T, c, c_out, zhw, out, st);
}

FBBEV_API int fbbev_history_train_full_fwd(
    const float* x, int64_t x_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wc_packed, const float* bias_c,
    const float* gamma, const float* beta, float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps, int32_t train, int32_t n,
    int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W, float* out,
    float* save, void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = check_full(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, c_out, Z, H,
                      W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (n == 0) return FBBEV_OK;
  if (!wc_packed || !bias_c || !running_mean || !running_var || !out || !save ||
      !aligned16(wc_packed) || (train && !num_batches_tracked))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  Params g = full_frame_params(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, zhw);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.eps = eps; b.momentum = momentum;
  b.nbt = num_batches_tracked; b.running_mean = running_mean; b.running_var = running_var;
  b.save = save; b.count = (double)n * (T + 1) * zhw;
  if (train) {
    Params s = g;
    s.part = part;
    if ((rc = launch_gemm<kMaxC, kStats>(s, T + 1, st, &b.grid)) != FBBEV_OK) return rc;
    b.part = part;
    b.mode = 0;
  } else {
    b.mode = 1;
  }
  if ((rc = launch_bn(b, st)) != FBBEV_OK) return rc;
  return full_fwd_tail(g, save, gamma, beta, wc_packed, bias_c, n, T, c, c_out, zhw, out,
                       workspace, st);
}

FBBEV_API int fbbev_history_train_full_fwd_local(
    const float* x, int64_t x_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, int32_t n, int32_t T, int32_t c, int32_t Z,
    int32_t H, int32_t W, double* row, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (!row) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_full(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, c, Z, H, W,
                      workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  double* part = static_cast<double*>(workspace);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.mode = 3; b.part = part; b.row = row;
  b.count = (double)n * (T + 1) * zhw;
  if (n > 0) {
    Params g =
        full_frame_params(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, zhw);
    g.part = part;
    if ((rc = launch_gemm<kMaxC, kStats>(g, T + 1, st, &b.grid)) != FBBEV_OK) return rc;
  }
  return launch_bn(b, st);
}

FBBEV_API int fbbev_history_train_full_fwd_global(
    const float* x, int64_t x_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wc_packed, const float* bias_c,
    const float* gamma, const float* beta, float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps, const double* rows,
    int32_t world, int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H,
    int32_t W, float* out, float* save, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (world < 1 || !rows) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_full(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, c_out, Z, H,
                      W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (!running_mean || !running_var || !num_batches_tracked || !save ||
      (n > 0 && (!wc_packed || !bias_c || !out || !aligned16(wc_packed))))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.mode = 4; b.rows = rows; b.world = world;
  b.eps = eps; b.momentum = momentum; b.nbt = num_batches_tracked;
  b.running_mean = running_mean; b.running_var = running_var; b.save = save;
  if ((rc = launch_bn(b, st)) != FBBEV_OK || n == 0) return rc;
  Params g = full_frame_params(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, zhw);
  return full_fwd_tail(g, save, gamma, beta, wc_packed, bias_c, n, T, c, c_out, zhw, out,
                       workspace, st);
}

FBBEV_API int fbbev_history_train_full_bwd_hidden(
    const float* x, int64_t x_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* gamma, const float* beta,
    const float* save, int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H,
    int32_t W, float* h, void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = check_full(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, c_out, Z, H,
                      W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (n == 0) return FBBEV_OK;
  if (!save || !h) return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  Params g = full_frame_params(x, x_batch_stride, time, wt_packed, bias_t, time_w, n, T, c, zhw);
  g.stats = save; g.gamma = gamma; g.beta = beta;
  g.out[0] = h; g.out2[0] = full_frames_buf(workspace, T);
  return launch_gemm<kMaxC, kHidden>(g, T + 1, as_stream(stream));
}

static int check_full_bwd(int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H,
                          int32_t W, const void* workspace, size_t workspace_bytes) {
  const int rc = check_shape(n, T, c, c_out, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  if (T >= 65535) return FBBEV_ERR_UNSUPPORTED;
  if (!workspace || !aligned16(workspace) ||
      workspace_bytes < fbbev_history_train_full_workspace_bytes(n, T, c, Z, H, W))
    return FBBEV_ERR_INVALID_ARGUMENT;
  return FBBEV_OK;
}

// d_f = (Wc_f^T g) [h_f > 0] into e for every frame, with the mask taken from
// the xhat_f of _bwd_hidden; the sums into the per-frame slots
static int full_delta(const float* wct_packed, const float* gamma, const float* beta, int n,
                      int T, int c, int c_out, int zhw, const float* grad_out, float* e,
                      void* workspace, cudaStream_t st, int* grid) {
  Params d = base_params(n, zhw);
  d.nf = T + 1;
  d.a[0][0] = grad_out; d.a_bstride[0][0] = (int64_t)c_out * zhw;
  d.w[0] = wct_packed; d.w_fstride = fbbev_linear_packed_bytes(kMaxC, c_out) / sizeof(float);
  d.n_seg = 1; d.k_seg = c_out; d.n_kb = (c_out + kKB - 1) / kKB; d.ncol = c;
  d.gamma = gamma; d.beta = beta;
  d.out[0] = e; d.xhat[0] = full_frames_buf(workspace, T);
  d.o_bstride = (int64_t)(T + 1) * c * zhw; d.o_fstride = (int64_t)c * zhw;
  d.part = static_cast<double*>(workspace);
  return launch_gemm<kMaxC, kDelta>(d, T + 1, st, grid);
}

// e_f from d_f over every frame, then dcurr = e_0 . Wt[:, :c]
static int full_e_and_curr(const float* wtt_packed, int n, int T, int c, int zhw, float* e,
                           float* grad_curr, void* workspace, cudaStream_t st) {
  const int64_t total = (int64_t)n * (T + 1) * c * zhw;
  const float* xh = full_frames_buf(workspace, T);
  count_launch();
  const int64_t blocks = ceil_div64(total, 256);
  history_train_e_kernel<<<dim3((unsigned)(blocks < 4096 ? blocks : 4096), 1), 256, 0, st>>>(
      e, e, xh, xh, full_coef(workspace, T), c, (T + 1) * c, zhw, total);
  int rc = launch_status();
  if (rc != FBBEV_OK || !grad_curr) return rc;
  Params x = base_params(n, zhw);
  x.a[0][0] = e; x.a_bstride[0][0] = (int64_t)(T + 1) * c * zhw;
  x.w[0] = wtt_packed;
  x.n_seg = 1; x.k_seg = c; x.n_kb = (c + kKB - 1) / kKB; x.ncol = c;
  x.out[0] = grad_curr;
  return launch_gemm<kMaxC, kOut>(x, 1, st);
}

FBBEV_API int fbbev_history_train_full_bwd(
    const float* wct_packed, const float* wtt_packed, const float* gamma, const float* beta,
    const float* save, int32_t train, int32_t n, int32_t T, int32_t c, int32_t c_out,
    int32_t Z, int32_t H, int32_t W, const float* grad_out, float* e, float* grad_curr,
    float* grad_gamma, float* grad_beta, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  int rc = check_full_bwd(n, T, c, c_out, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (n == 0) return FBBEV_OK;
  if (!wct_packed || !aligned16(wct_packed) || (grad_curr && (!wtt_packed || !aligned16(wtt_packed))) ||
      !save || !grad_out || !e || !grad_gamma || !grad_beta)
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.mode = 2; b.train = train;
  b.save = const_cast<float*>(save);  // read only in mode 2
  b.gamma = gamma; b.count = (double)n * (T + 1) * zhw;
  b.part = static_cast<double*>(workspace); b.coef = full_coef(workspace, T);
  b.dgamma = grad_gamma; b.dbeta = grad_beta;
  rc = full_delta(wct_packed, gamma, beta, n, T, c, c_out, zhw, grad_out, e, workspace, st,
                  &b.grid);
  if (rc == FBBEV_OK) rc = launch_bn(b, st);
  if (rc != FBBEV_OK) return rc;
  return full_e_and_curr(wtt_packed, n, T, c, zhw, e, grad_curr, workspace, st);
}

FBBEV_API int fbbev_history_train_full_bwd_local(
    const float* wct_packed, const float* gamma, const float* beta, int32_t n, int32_t T,
    int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W, const float* grad_out, float* e,
    float* grad_gamma, float* grad_beta, double* row, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream) {
  if (!row) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_full_bwd(n, T, c, c_out, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (!grad_gamma || !grad_beta ||
      (n > 0 && (!wct_packed || !aligned16(wct_packed) || !grad_out || !e)))
    return FBBEV_ERR_INVALID_ARGUMENT;
  const int zhw = Z * H * W;
  cudaStream_t st = as_stream(stream);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.mode = 5; b.part = static_cast<double*>(workspace);
  b.row = row; b.count = (double)n * (T + 1) * zhw;
  b.dgamma = grad_gamma; b.dbeta = grad_beta;
  if (n > 0 &&
      (rc = full_delta(wct_packed, gamma, beta, n, T, c, c_out, zhw, grad_out, e, workspace, st,
                       &b.grid)) != FBBEV_OK)
    return rc;
  return launch_bn(b, st);
}

FBBEV_API int fbbev_history_train_full_bwd_global(
    const float* wtt_packed, const float* gamma, const float* save, const double* rows,
    int32_t world, int32_t n, int32_t T, int32_t c, int32_t Z, int32_t H, int32_t W, float* e,
    float* grad_curr, void* workspace, size_t workspace_bytes, fbbev_stream_t stream) {
  if (world < 1 || !rows) return FBBEV_ERR_INVALID_ARGUMENT;
  int rc = check_full_bwd(n, T, c, c, Z, H, W, workspace, workspace_bytes);
  if (rc != FBBEV_OK) return rc;
  if (!save || (n > 0 && (!e || (grad_curr && (!wtt_packed || !aligned16(wtt_packed))))))
    return FBBEV_ERR_INVALID_ARGUMENT;
  cudaStream_t st = as_stream(stream);
  BnParams b = {};
  b.C = c; b.T = T; b.nf = T + 1; b.mode = 6; b.train = 1; b.rows = rows; b.world = world;
  b.save = const_cast<float*>(save);  // read only in mode 6
  b.gamma = gamma; b.coef = full_coef(workspace, T);
  if ((rc = launch_bn(b, st)) != FBBEV_OK || n == 0) return rc;
  return full_e_and_curr(wtt_packed, n, T, c, Z * H * W, e, grad_curr, workspace, st);
}

// -- the restart term: the reference's gradient through its restart write -----
// A sample that starts a sequence has the grad-carrying current frame as its T
// history frames (fbocc.py:255), so d curr gains Wt[:, :c]^T warp^T (sum_{f>=1}
// e_f).  The warp acts per channel and Wt per voxel, so the two commute: the
// adjoint runs on the e_f the backward already wrote (history_warp_bwd.cu),
// then one kOut launch per restarting sample adds Wt^T R into its d curr.
// Workspace: R (c, Z H W) | the adjoint's.
static size_t restart_r_bytes(int c, int64_t zhw) {
  return ((size_t)c * zhw * sizeof(float) + 255) & ~size_t(255);
}

FBBEV_API size_t fbbev_history_restart_grad_workspace_bytes(int32_t c, int32_t Z, int32_t H,
                                                            int32_t W, int32_t frames) {
  const size_t adj = fbbev_history_warp_bwd_workspace_bytes(c, Z, H, W, frames);
  return adj ? restart_r_bytes(c, (int64_t)Z * H * W) + adj : 0;
}

FBBEV_API int fbbev_history_restart_grad_curr(
    const float* e, int64_t e_batch_stride, int64_t e_frame_stride, int32_t frames,
    const uint8_t* mask, const float* flow, const float* wtt_packed, int32_t n, int32_t c,
    int32_t Z, int32_t H, int32_t W, float* grad_curr, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream) {
  int rc = check_shape(n, 1, c, c, Z, H, W);
  if (rc != FBBEV_OK) return rc;
  const int64_t zhw = (int64_t)Z * H * W, dense = (int64_t)c * zhw;
  if (frames < 1 || (frames > 1 && e_frame_stride < dense) ||
      e_batch_stride < (int64_t)(frames - 1) * e_frame_stride + dense)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (zhw > kWarpAdjMaxVoxels) return FBBEV_ERR_UNSUPPORTED;
  if (n == 0) return FBBEV_OK;
  if (!e || !mask || !flow || !wtt_packed || !grad_curr || !workspace ||
      !aligned16(wtt_packed) || !aligned16(workspace) ||
      workspace_bytes < fbbev_history_restart_grad_workspace_bytes(c, Z, H, W, frames))
    return FBBEV_ERR_INVALID_ARGUMENT;
  cudaStream_t st = as_stream(stream);
  float* r = static_cast<float*>(workspace);
  void* adj = static_cast<char*>(workspace) + restart_r_bytes(c, zhw);
  for (int b = 0; b < n; ++b) {
    if (!mask[b]) continue;
    rc = warp_adjoint(e + b * e_batch_stride, e_frame_stride, frames, flow + 16 * b, c, Z, H,
                      W, r, 0, adj, st);
    if (rc != FBBEV_OK) return rc;
    Params x = base_params(1, (int)zhw);  // d curr[b] += R . Wt[:, :c]
    x.a[0][0] = r; x.a_bstride[0][0] = dense;
    x.w[0] = wtt_packed;
    x.n_seg = 1; x.k_seg = c; x.n_kb = (c + kKB - 1) / kKB; x.ncol = c;
    x.out[0] = grad_curr + b * dense; x.accum = 1;
    if ((rc = launch_gemm<kMaxC, kOut>(x, 1, st)) != FBBEV_OK) return rc;
  }
  return FBBEV_OK;
}
