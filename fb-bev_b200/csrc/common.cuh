// common.cuh -- shared helpers for the sm_90a kernels behind libfbbev_b200.so
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/fbbev_b200.h"

#define FBBEV_API extern "C" __attribute__((visibility("default")))

namespace fbbev {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

static inline cudaStream_t as_stream(fbbev_stream_t s) {
  return reinterpret_cast<cudaStream_t>(s);
}

// Returns the pending launch error (positive cudaError_t) or 0.
static inline int launch_status() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? FBBEV_OK : static_cast<int>(e);
}

// Diagnostics only: cumulative number of kernel launches issued by this library
// (bench.py reports it as `gpu_launches`).  Defined in capi.cu.
void count_launch(int n = 1);

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Number of CTAs of `kern` that are resident on the current device at once:
// the grid of a persistent kernel.
template <typename Kernel>
static inline cudaError_t resident_ctas(Kernel kern, int threads, size_t smem,
                                        int* ctas) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess)
    e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess)
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem);
  if (e == cudaSuccess && per_sm < 1) e = cudaErrorInvalidConfiguration;
  if (e == cudaSuccess) *ctas = sms * per_sm;
  return e;
}

// Streaming (evict-first) 128-bit / 32-bit stores for write-once outputs.
__device__ __forceinline__ void st_stream(float4* p, const float4& v) {
  __stcs(p, v);
}
__device__ __forceinline__ void st_stream(float* p, float v) { __stcs(p, v); }

// y = M x for a row-major 3x3 M, in the rounding order torch's broadcast
// (..,3,3) @ (..,3,1) matmul has (torch 2.11 / cuBLAS 12.8; identified by
// tools/micro/matmul_order2.py over all 18 FMA / non-FMA association orders):
//   y_i = fma(m_i1, x_1, m_i0 * x_0) + m_i2 * x_2            (batched 'n' kernel)
// and, when `seq` is set, the sequential FMA chain
//   y_i = fma(m_i2, x_2, fma(m_i1, x_1, m_i0 * x_0))
// which cuBLAS uses for a single column-major matrix broadcast over the batch
// (torch.inverse returns column-major; with one matrix in total the expand is a
// stride-0 view and the transposed layout reaches cuBLAS as op 't').
__device__ __forceinline__ float dot3_ref(float m0, float m1, float m2, float x,
                                          float y, float z, bool seq) {
  const float s = __fmaf_rn(m1, y, __fmul_rn(m0, x));
  return seq ? __fmaf_rn(m2, z, s) : __fadd_rn(s, __fmul_rn(m2, z));
}
// y = m . x with the three products summed in one of the 18 fp32 orders
// (FBBEV_ORDER_EXPLICIT, include/fbbev_b200.h): code = 6 last + 2 inner + outer;
// `last` is the index added last, a < b the other two; inner 0: p_a + p_b,
// 1: fma(m_a, x_a, p_b), 2: fma(m_b, x_b, p_a); outer 0: s + p_last,
// 1: fma(m_last, x_last, s).  Code 16 is dot3_ref(seq = false), 17 seq = true.
__device__ __forceinline__ float dot3_code(float m0, float m1, float m2, float x0,
                                           float x1, float x2, int code) {
  const int last = code / 6, inner = (code >> 1) % 3;
  // operands picked by selects (no runtime-indexed arrays: they would live in
  // local memory)
  const float ma = last == 0 ? m1 : m0, xa = last == 0 ? x1 : x0;
  const float mb = last == 2 ? m1 : m2, xb = last == 2 ? x1 : x2;
  const float ml = last == 0 ? m0 : (last == 1 ? m1 : m2);
  const float xl = last == 0 ? x0 : (last == 1 ? x1 : x2);
  const float pa = __fmul_rn(ma, xa), pb = __fmul_rn(mb, xb);
  const float s = inner == 0 ? __fadd_rn(pa, pb)
                  : inner == 1 ? __fmaf_rn(ma, xa, pb)
                               : __fmaf_rn(mb, xb, pa);
  return (code & 1) ? __fmaf_rn(ml, xl, s) : __fadd_rn(s, __fmul_rn(ml, xl));
}
__device__ __forceinline__ void mat3_apply_code(const float* __restrict__ m,
                                                float x, float y, float z,
                                                int code, float& ox, float& oy,
                                                float& oz) {
  ox = dot3_code(__ldg(m + 0), __ldg(m + 1), __ldg(m + 2), x, y, z, code);
  oy = dot3_code(__ldg(m + 3), __ldg(m + 4), __ldg(m + 5), x, y, z, code);
  oz = dot3_code(__ldg(m + 6), __ldg(m + 7), __ldg(m + 8), x, y, z, code);
}
// the i-th stack's order: an explicit code, or seq / non-seq by flag bit i
__device__ __forceinline__ int order_code(int order, int i) {
  if (order & FBBEV_ORDER_EXPLICIT) return (order >> (8 + 5 * i)) & 31;
  return (order >> i) & 1 ? 17 : 16;
}
__device__ __forceinline__ void mat3_apply_ref(const float* __restrict__ m,
                                               float x, float y, float z,
                                               bool seq, float& ox, float& oy,
                                               float& oz) {
  ox = dot3_ref(__ldg(m + 0), __ldg(m + 1), __ldg(m + 2), x, y, z, seq);
  oy = dot3_ref(__ldg(m + 3), __ldg(m + 4), __ldg(m + 5), x, y, z, seq);
  oz = dot3_ref(__ldg(m + 6), __ldg(m + 7), __ldg(m + 8), x, y, z, seq);
}

}  // namespace fbbev
