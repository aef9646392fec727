// history_fuse.cu -- the whole data path of FBOCC.fuse_history after the
// state update, inference only, as ONE Hopper tensor-core kernel.
//
// What it replaces (mmdet3d/models/fbbev/detectors/fbocc.py:263-317): the
// trilinear warp of the history, torch.cat with the current frame, the
// sweep-time channel, history_keyframe_time_conv (Conv3d 1x1x1 (C+1) -> C, BN,
// ReLU) over all T + 1 frames, history_keyframe_cat_conv (Conv3d 1x1x1
// (T+1) C -> C_out, BN, ReLU) and the closing permute().clone().  Every
// intermediate of that chain (the 17-frame stack is 435 MB per sample at the
// FB-OCC size) goes through memory there; here nothing but the next history
// and the output is written.
//
// Per 128-voxel tile of one sample (BN in eval mode folded into both convs on
// the host; frame f = 0 is the current frame, f >= 1 history slot f - 1):
//
//   Y = 0
//   for f in 0..T:
//     A_f = curr (f = 0) | history_sample of history slot f - 1 under the flow
//     H_f = relu(A_f . Wt'^T + bias_t' + Wt'[:, C] * 0.5 sweep[b, f])
//     Y  += H_f . Wc'[:, f C : (f+1) C]^T
//     (next history given, f < T) write A_f into its channels [f C, (f+1) C)
//   out = relu(Y + bias_c')
//
// A fresh sample (no history yet, or start_of_sequence) has T copies of the
// current frame as history, all with one sweep time: every history frame gives
// the same H, so Y = H_0 . Wc_0^T + H_w . (sum_{f>=1} Wc_f)^T -- two frames of
// work, with the summed weights packed beside Wc'.
//
// Organisation (as ffn_tf32.cu): persistent grid, two warpgroups of 64 rows,
// 3xTF32 wgmma with fp32 accumulators.
//   GEMM1   A_f formed in registers (gathered, split hi / lo), Wt' resident in
//           shared memory (two K-blocks, hi + lo, 51.2 KB); N = 80
//   H tile  relu(acc + bias) split hi / lo into shared memory (80 KB)
//   GEMM2   Y[64 x 80 per half] += H_f . Wc'_f^T; the weights stream through a
//           two-slot ring of 25.6 KB stages (80 output rows x one 40-float
//           K-block, hi + lo; one 1-D bulk copy each) in consumption order;
//           C_out > 80 runs as two 80-column halves
// The corner offsets and weights of the tile's voxels (history_corners, the
// same function history_warp_kernel calls) are computed once per tile into
// shared memory (8 KB): every frame of the tile samples at the same locations.
// They are read from there at each sample rather than held in registers, which
// GEMM1's A fragments and the two accumulators leave no room for.
#include "common.cuh"
#include "history_common.cuh"
#include "wgmma.cuh"

namespace fbbev {
namespace hfuse {

constexpr int kThreads = 256;        // two warpgroups
constexpr int kTileM = kATileM;
constexpr int kMaxC = 80;            // GEMM1 width (Wt' rows padded to 80)
constexpr int kHalf = 80;            // GEMM2 columns per half
constexpr int kMaxCout = 2 * kHalf;
constexpr int kWPart = kb_part(kHalf);             // bytes of one hi / lo part of a stage
constexpr int kWStage = 2 * kWPart;                // 25.6 KB
constexpr int kCv = 2 * kMaxC + kMaxCout;          // bias_t | time_w | bias_c
// shared memory: Wt' | H tile | weight ring | corner table | constants | mbarriers
constexpr int kOffH = 2 * kWStage;
constexpr int kOffRing = kOffH + 2 * kABlock;
constexpr int kOffTab = kOffRing + 2 * kWStage;
constexpr int kOffCv = kOffTab + kTileM * 8 * 8;
constexpr int kOffBar = kOffCv + kCv * 4;
constexpr int kSmem = kOffBar + 32;

struct Params {
  const float* curr;      // (n, C, Z, H, W), samples curr_bstride floats apart
  const float* hist;      // (n, T C, Z, H, W) or null (every sample fresh)
  const uint8_t* fresh;   // [n]
  const float* flow;      // (n, 4, 4)
  const float* sweep;     // (n, T + 1)
  const float* wt;        // fbbev_linear_pack(Wt'[:, :C] padded to 80 rows, k = C)
  const float* wc;        // per frame f and half h: pack(Wc'_f rows 80h.., k = C)
  const float* wc_sum;    // the same for sum_{f>=1} Wc'_f
  const float* bias_t;    // [C]
  const float* time_w;    // [C] = Wt'[:, C]
  const float* bias_c;    // [C_out]
  float* out;             // (n, C_out, Z, H, W)
  float* next;            // (n, next_ch, Z, H, W) or null
  int64_t curr_bstride, hist_bstride, next_bstride;
  int T, C, Cout, Z, H, W, zhw, n_kb, tps, n_tiles;
};

__device__ __forceinline__ bool is_fresh(const Params& p, int b) {
  return !p.hist || __ldg(p.fresh + b) != 0;
}

template <int NH>
__global__ void __launch_bounds__(kThreads, 1) history_fuse_kernel(const Params p) {
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t wt_a = smem_u32(smem);
  const uint32_t hs_a = wt_a + kOffH, ws_a = wt_a + kOffRing;
  unsigned char* hs = smem + kOffH;
  int* tab_off = reinterpret_cast<int*>(smem + kOffTab);                   // [8][128]
  float* tab_w = reinterpret_cast<float*>(smem + kOffTab + kTileM * 8 * 4);  // [8][128]
  float* cv = reinterpret_cast<float*>(smem + kOffCv);
  const float* bias_t = cv;
  const float* time_w = cv + kMaxC;
  const float* bias_c = cv + 2 * kMaxC;
  const uint32_t bar_wt = wt_a + kOffBar, bar = bar_wt + 8u;  // Wt' | ring slots 0, 1
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
  const int T = p.T, C = p.C, n_kb = p.n_kb, zhw = p.zhw;
  if (tid == 0) {
    mbar_init(bar_wt, 1);
    mbar_init(bar, 1);
    mbar_init(bar + 8u, 1);
    fence_mbar_init();
  }
  for (int i = tid; i < kCv; i += kThreads) {
    float v = 0.f;
    if (i < kMaxC) {
      if (i < C) v = __ldg(p.bias_t + i);
    } else if (i < 2 * kMaxC) {
      if (i - kMaxC < C) v = __ldg(p.time_w + i - kMaxC);
    } else if (i - 2 * kMaxC < p.Cout) {
      v = __ldg(p.bias_c + i - 2 * kMaxC);
    }
    cv[i] = v;
  }
  __syncthreads();

  // Weight stages in consumption order: tiles blockIdx.x, + gridDim.x, ...
  // (the grid is never larger than the tile count), frames of the tile, halves,
  // K-blocks.  Thread 0 walks that sequence with its own cursor.
  const int per_frame = NH * n_kb;
  int pt = blockIdx.x, ps = 0, pj = 0;
  uint32_t pi = 0;
  auto issue_w = [&]() {
    if (tid != 0 || pt >= p.n_tiles) return;
    const bool fr = is_fresh(p, pt / p.tps);
    const float* src = fr && ps == 1 ? p.wc_sum + (size_t)pj * (kWStage / 4)
                                     : p.wc + (size_t)(ps * per_frame + pj) * (kWStage / 4);
    const uint32_t s = pi & 1;
    mbar_arrive_expect_tx(bar + 8u * s, kWStage);
    bulk_g2s(ws_a + s * kWStage, src, kWStage, bar + 8u * s);
    ++pi;
    if (++pj == per_frame) {
      pj = 0;
      if (++ps == (fr ? 2 : T + 1)) {
        ps = 0;
        pt += gridDim.x;
      }
    }
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_wt, n_kb * kWStage);
    bulk_g2s(wt_a, p.wt, n_kb * kWStage, bar_wt);
  }
  issue_w();
  issue_w();
  mbar_wait<true>(bar_wt, 0);

  const int rl = wg * 64 + wq * 16 + (lane >> 2);  // tile row of acc[.. + 0 / 1]
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    const int b = tile / p.tps;
    const int v0 = (tile - b * p.tps) * kTileM;
    const bool fresh = is_fresh(p, b);
    const int nf = fresh ? 2 : T + 1;
    // corner table (the previous tile's gathers are behind a __syncthreads)
    if (tid < kTileM) {
      const int v = v0 + tid;
      float wgt[8];
      int64_t off[8];
      if (v < zhw) {
        history_corners(p.flow + b * 16, v % p.W, (v / p.W) % p.H, v / (p.W * p.H), p.W,
                        p.H, p.Z, wgt, off);
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          wgt[k] = 0.f;
          off[k] = 0;
        }
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        tab_off[k * kTileM + tid] = (int)off[k];
        tab_w[k * kTileM + tid] = wgt[k];
      }
    }
    __syncthreads();
    const int vr0 = min(v0 + rl, zhw - 1), vr1 = min(v0 + rl + 8, zhw - 1);
    const bool ok0 = v0 + rl < zhw, ok1 = v0 + rl + 8 < zhw;
    const float* cur_b = p.curr + (int64_t)b * p.curr_bstride;
    float* next_b = p.next ? p.next + (int64_t)b * p.next_bstride : nullptr;

    float acc2[NH][kHalf / 2];  // written first by a scale-d = 0 MMA, never zeroed
    for (int s = 0; s < nf; ++s) {
      const float* base = s == 0 || fresh
                              ? cur_b
                              : p.hist + (int64_t)b * p.hist_bstride + (int64_t)(s - 1) * C * zhw;
      const float st = 0.5f * __ldg(p.sweep + (int64_t)b * (T + 1) + s);
      // next-history frames this A fills: f = s, or 1..T-1 for a fresh sample
      const int f_end = fresh && s == 1 ? T : min(s + 1, T);
      float acc1[kMaxC / 2];
      for (int kb = 0; kb < n_kb; ++kb) {
        float a[kKSteps][4];
#pragma unroll
        for (int k = 0; k < kKSteps; ++k)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int h = e & 1;
            const int c = kb * kKB + 8 * k + q + 4 * (e >> 1);
            const float* src = base + (int64_t)min(c, C - 1) * zhw;
            float v;
            if (s == 0) {
              v = __ldg(src + (h ? vr1 : vr0));
            } else {
              float cw[8];
              int co[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                cw[j] = tab_w[j * kTileM + rl + 8 * h];
                co[j] = tab_off[j * kTileM + rl + 8 * h];
              }
              v = history_sample(src, cw, co);
            }
            a[k][e] = c < C ? v : 0.f;
          }
        if (next_b && s < f_end) {
#pragma unroll
          for (int k = 0; k < kKSteps; ++k)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int h = e & 1;
              const int c = kb * kKB + 8 * k + q + 4 * (e >> 1);
              if (c < C && (h ? ok1 : ok0))
                for (int f = s; f < f_end; ++f)
                  __stcs(next_b + (int64_t)(f * C + c) * zhw + (h ? vr1 : vr0), a[k][e]);
            }
        }
        uint32_t ah[kKSteps][4], al[kKSteps][4];
#pragma unroll
        for (int k = 0; k < kKSteps; ++k)
#pragma unroll
          for (int e = 0; e < 4; ++e) tf32_split(a[k][e], ah[k][e], al[k][e]);
        wgmma_fence();
        const uint32_t b_hi = wt_a + kb * kWStage;
        wg_kblock_3xtf32_rs<kMaxC>(acc1, ah, al, b_hi, b_hi + kWPart, kb_chunk(kMaxC), kb > 0);
        wgmma_commit();
        // also drains the previous frame's GEMM2: the H tile is free after this
        wgmma_wait<0>();
      }
      acc_fence(acc1);
      // H_f = relu(acc + bias_t' + time_w * 0.5 sweep), hi / lo -> this
      // warpgroup's rows of the H tile (columns >= C are zero)
#pragma unroll
      for (int J = 0; J < kMaxC / 8; ++J) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * J + 2 * q + e;
            const float v = fmaxf(acc1[4 * J + 2 * h + e] + fmaf(time_w[col], st, bias_t[col]), 0.f);
            unsigned char* d = hs + (size_t)(col / kKB) * kABlock + a_off(rl + 8 * h, col % kKB);
            tf32_split(v, *reinterpret_cast<float*>(d), *reinterpret_cast<float*>(d + kAPart));
          }
        }
      }
      fence_proxy_async();
      __syncthreads();
#pragma unroll
      for (int h = 0; h < NH; ++h) {
        for (int kb = 0; kb < n_kb; ++kb) {
          const uint32_t sl = it & 1;
          mbar_wait<true>(bar + 8u * sl, (it >> 1) & 1u);
          const uint32_t a_hi = hs_a + kb * kABlock + wg * 1024u;
          const uint32_t w_hi = ws_a + sl * kWStage;
          wgmma_fence();
          wg_kblock_3xtf32<kHalf>(acc2[h], a_hi, a_hi + kAPart, kAChunkStride, w_hi,
                                  w_hi + kWPart, kb_chunk(kHalf), s > 0 || kb > 0);
          // once the previous stage's MMAs have drained (both warpgroups), its
          // slot takes the stage after this one
          wgmma_commit();
          wgmma_wait<1>();
          __syncthreads();
          if (it >= 1) issue_w();
          ++it;
        }
      }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < NH; ++h) acc_fence(acc2[h]);
    // out = relu(Y + bias_c'), (n, C_out, Z, H, W)
    float* out_b = p.out + (int64_t)b * p.Cout * zhw;
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int J = 0; J < kHalf / 8; ++J)
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = kHalf * h + 8 * J + 2 * q + e;
            if (col < p.Cout && (r ? ok1 : ok0))
              __stcs(out_b + (int64_t)col * zhw + (r ? vr1 : vr0),
                     fmaxf(acc2[h][4 * J + 2 * r + e] + bias_c[col], 0.f));
          }
  }
}

template <int NH>
static int launch(const Params& p, cudaStream_t st) {
  static int resident = 0;  // CTAs that fit on the device at once
  if (!resident) {
    cudaError_t e = cudaFuncSetAttribute(history_fuse_kernel<NH>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return (int)e;
    e = resident_ctas(history_fuse_kernel<NH>, kThreads, kSmem, &resident);
    if (e != cudaSuccess) return (int)e;
  }
  history_fuse_kernel<NH>
      <<<p.n_tiles < resident ? p.n_tiles : resident, kThreads, kSmem, st>>>(p);
  return launch_status();
}

}  // namespace hfuse
}  // namespace fbbev

using namespace fbbev;

FBBEV_API int fbbev_history_fuse_supported(int32_t c, int32_t c_out) {
  return c >= 4 && c <= hfuse::kMaxC && c % 4 == 0 && c_out >= 4 &&
                 c_out <= hfuse::kMaxCout && c_out % 4 == 0
             ? 1
             : 0;
}

FBBEV_API int fbbev_history_fuse_fwd(
    const float* curr, int64_t curr_batch_stride, const float* history,
    int64_t history_batch_stride, const uint8_t* fresh, const float* flow,
    const float* sweep, const float* wt_packed, const float* wc_packed,
    const float* wc_sum_packed, const float* bias_t, const float* time_w,
    const float* bias_c, int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z,
    int32_t H, int32_t W, float* out, float* next_history, int32_t next_channels,
    fbbev_stream_t stream) {
  if (n < 0 || T < 1 || Z <= 0 || H <= 0 || W <= 0) return FBBEV_ERR_INVALID_ARGUMENT;
  if (!fbbev_history_fuse_supported(c, c_out)) return FBBEV_ERR_UNSUPPORTED;
  const int64_t zhw = (int64_t)Z * H * W;
  const int64_t tps = ceil_div64(zhw, hfuse::kTileM);
  if (zhw >= ((int64_t)1 << 31) || n > 65535 || n * tps >= ((int64_t)1 << 31))
    return FBBEV_ERR_UNSUPPORTED;
  if (curr_batch_stride < c * zhw ||
      (history && history_batch_stride < (int64_t)T * c * zhw) ||
      (next_history && next_channels < T * c))
    return FBBEV_ERR_INVALID_ARGUMENT;
  if (n == 0) return FBBEV_OK;
  if (!curr || !fresh || !flow || !sweep || !wt_packed || !wc_packed || !wc_sum_packed ||
      !bias_t || !time_w || !bias_c || !out)
    return FBBEV_ERR_INVALID_ARGUMENT;
  if ((reinterpret_cast<uintptr_t>(wt_packed) | reinterpret_cast<uintptr_t>(wc_packed) |
       reinterpret_cast<uintptr_t>(wc_sum_packed)) & 15)
    return FBBEV_ERR_INVALID_ARGUMENT;
  hfuse::Params p;
  p.curr = curr; p.hist = history; p.fresh = fresh; p.flow = flow; p.sweep = sweep;
  p.wt = wt_packed; p.wc = wc_packed; p.wc_sum = wc_sum_packed;
  p.bias_t = bias_t; p.time_w = time_w; p.bias_c = bias_c;
  p.out = out; p.next = next_history;
  p.curr_bstride = curr_batch_stride;
  p.hist_bstride = history_batch_stride;
  p.next_bstride = (int64_t)next_channels * zhw;
  p.T = T; p.C = c; p.Cout = c_out; p.Z = Z; p.H = H; p.W = W;
  p.zhw = (int)zhw;
  p.n_kb = (c + kKB - 1) / kKB;
  p.tps = (int)tps;
  p.n_tiles = (int)(n * tps);
  cudaStream_t st = as_stream(stream);
  count_launch();
  return c_out > hfuse::kHalf ? hfuse::launch<2>(p, st) : hfuse::launch<1>(p, st);
}
