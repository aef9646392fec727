// wgmma.cuh -- the 3xTF32 layer of the Hopper tensor-core kernels
// (linear_tf32.cu, ffn_tf32.cu, history_fuse.cu, history_train.cu): warpgroup
// MMA (wgmma.mma_async, tf32) with shared-memory matrix descriptors (K-major,
// no swizzle) or with A from registers, the shared-memory operand images and
// hi / lo split they read, and the 3xTF32 K-block products the kernels are
// built on.  mbarriers and bulk copies come from bulk.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "bulk.cuh"

namespace fbbev {

// ------------------------------- PTX wrappers --------------------------------
// generic-proxy shared-memory writes -> visible to wgmma / bulk copies
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// K-major operand without swizzle: 8-row x 16-byte core matrices; `lbo` bytes
// between the two K-adjacent core matrices of one k8 step, `sbo` bytes between
// 8-row groups (wgmma matrix descriptor, layout type 0 = no swizzle).
__device__ __forceinline__ uint64_t smem_desc(uint32_t addr, uint32_t lbo,
                                              uint32_t sbo) {
  return (uint64_t)((addr >> 4) & 0x3FFFu) |
         ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32);
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator accesses across wgmma issue / wait
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// The accumulator of an m64nNk8 f32 wgmma is N / 2 registers per thread:
// FBBEV_ACC_N is their PTX operand list "%0, %1, ..., %(N/2 - 1)" and
// FBBEV_ACC_OPS_N the matching "+f"(d[0]), ..., "+f"(d[N/2 - 1]).
#define FBBEV_D8(i)                                                                 \
  "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]),       \
      "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define FBBEV_ACC_16 "%0, %1, %2, %3, %4, %5, %6, %7"
#define FBBEV_ACC_32 FBBEV_ACC_16 ", %8, %9, %10, %11, %12, %13, %14, %15"
#define FBBEV_ACC_48 FBBEV_ACC_32 ", %16, %17, %18, %19, %20, %21, %22, %23"
#define FBBEV_ACC_64 FBBEV_ACC_48 ", %24, %25, %26, %27, %28, %29, %30, %31"
#define FBBEV_ACC_80 FBBEV_ACC_64 ", %32, %33, %34, %35, %36, %37, %38, %39"
#define FBBEV_ACC_96 FBBEV_ACC_80 ", %40, %41, %42, %43, %44, %45, %46, %47"
#define FBBEV_ACC_112 FBBEV_ACC_96 ", %48, %49, %50, %51, %52, %53, %54, %55"
#define FBBEV_ACC_128 FBBEV_ACC_112 ", %56, %57, %58, %59, %60, %61, %62, %63"
#define FBBEV_ACC_144 FBBEV_ACC_128 ", %64, %65, %66, %67, %68, %69, %70, %71"
#define FBBEV_ACC_160 FBBEV_ACC_144 ", %72, %73, %74, %75, %76, %77, %78, %79"
#define FBBEV_ACC_176 FBBEV_ACC_160 ", %80, %81, %82, %83, %84, %85, %86, %87"
#define FBBEV_ACC_192 FBBEV_ACC_176 ", %88, %89, %90, %91, %92, %93, %94, %95"
#define FBBEV_ACC_OPS_16 FBBEV_D8(0)
#define FBBEV_ACC_OPS_32 FBBEV_ACC_OPS_16, FBBEV_D8(8)
#define FBBEV_ACC_OPS_48 FBBEV_ACC_OPS_32, FBBEV_D8(16)
#define FBBEV_ACC_OPS_64 FBBEV_ACC_OPS_48, FBBEV_D8(24)
#define FBBEV_ACC_OPS_80 FBBEV_ACC_OPS_64, FBBEV_D8(32)
#define FBBEV_ACC_OPS_96 FBBEV_ACC_OPS_80, FBBEV_D8(40)
#define FBBEV_ACC_OPS_112 FBBEV_ACC_OPS_96, FBBEV_D8(48)
#define FBBEV_ACC_OPS_128 FBBEV_ACC_OPS_112, FBBEV_D8(56)
#define FBBEV_ACC_OPS_144 FBBEV_ACC_OPS_128, FBBEV_D8(64)
#define FBBEV_ACC_OPS_160 FBBEV_ACC_OPS_144, FBBEV_D8(72)
#define FBBEV_ACC_OPS_176 FBBEV_ACC_OPS_160, FBBEV_D8(80)
#define FBBEV_ACC_OPS_192 FBBEV_ACC_OPS_176, FBBEV_D8(88)
// The widths the kernels use, each with the operand numbers N/2 ... N/2 + 5
// that follow its accumulator.
#define FBBEV_WGMMA_WIDTHS(X)     \
  X(16, 8, 9, 10, 11, 12, 13)     \
  X(32, 16, 17, 18, 19, 20, 21)   \
  X(48, 24, 25, 26, 27, 28, 29)   \
  X(64, 32, 33, 34, 35, 36, 37)   \
  X(80, 40, 41, 42, 43, 44, 45)   \
  X(96, 48, 49, 50, 51, 52, 53)   \
  X(112, 56, 57, 58, 59, 60, 61)  \
  X(128, 64, 65, 66, 67, 68, 69)  \
  X(144, 72, 73, 74, 75, 76, 77)  \
  X(160, 80, 81, 82, 83, 84, 85)  \
  X(176, 88, 89, 90, 91, 92, 93)  \
  X(192, 96, 97, 98, 99, 100, 101)

// D[64 x N] = A[64 x 8] . B[N x 8]^T + (scale_d ? D : 0), tf32 operands from
// shared memory, one instruction for the full width (N a multiple of 16, up to
// 192).  Issuing a tile's first MMA with scale_d = 0 instead of zeroing D keeps
// every write to the accumulator registers inside the wgmma pipeline, so
// ptxas need not serialise the MMAs (C7515).
#define FBBEV_WGMMA_SS(W, m0, m1, m2, m3, m4, m5)                                     \
  if constexpr (N == W)                                                               \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #m2 ", 0;\n\t"              \
                 "wgmma.mma_async.sync.aligned.m64n" #W "k8.f32.tf32.tf32 {"          \
                 FBBEV_ACC_##W "}, %" #m0 ", %" #m1 ", p, 1, 1;\n\t}"                 \
                 : FBBEV_ACC_OPS_##W                                                  \
                 : "l"(da), "l"(db), "r"(scale_d)                                     \
                 : "memory");
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db,
                                           uint32_t scale_d) {
  static_assert(N % 16 == 0 && N >= 16 && N <= 192, "wgmma_tf32: N");
  FBBEV_WGMMA_WIDTHS(FBBEV_WGMMA_SS)
}

// The same product with A from registers: the m64k8 tf32 A fragment of a
// warp is rows 16 (warp % 4) + lane / 4 (+ 8 for a[1], a[3]) and columns
// lane % 4 (+ 4 for a[2], a[3]) of the k8 step.  A wgmma.fence must separate
// the writes of `a` from the instruction, and `a` must stay unchanged until
// the instruction has completed (wgmma.wait_group).
#define FBBEV_WGMMA_RS(W, m0, m1, m2, m3, m4, m5)                                     \
  if constexpr (N == W)                                                               \
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #m5 ", 0;\n\t"              \
                 "wgmma.mma_async.sync.aligned.m64n" #W "k8.f32.tf32.tf32 {"          \
                 FBBEV_ACC_##W "}, {%" #m0 ", %" #m1 ", %" #m2 ", %" #m3 "}, %" #m4   \
                 ", p, 1, 1;\n\t}"                                                    \
                 : FBBEV_ACC_OPS_##W                                                  \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d)  \
                 : "memory");
template <int N>
__device__ __forceinline__ void wgmma_tf32_rs(float* d, const uint32_t (&a)[4],
                                              uint64_t db, uint32_t scale_d) {
  static_assert(N % 16 == 0 && N >= 16 && N <= 192, "wgmma_tf32_rs: N");
  FBBEV_WGMMA_WIDTHS(FBBEV_WGMMA_RS)
}

// ------------------------------ operand images -------------------------------
// 3xTF32 split of an fp32 value: hi = the upper 19 bits (exactly a tf32),
// lo = the exact fp32 remainder.  x.w ~= x_hi.w_hi + x_lo.w_hi + x_hi.w_lo
// (relative error ~2^-21), which the 1e-4 parity bar needs; plain tf32 is not
// enough.
__device__ __forceinline__ void tf32_split(float v, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
  lo = v - hi;
}
// the same into the b32 registers of a wgmma A fragment
__device__ __forceinline__ void tf32_split(float v, uint32_t& hi, uint32_t& lo) {
  float h, l;
  tf32_split(v, h, l);
  hi = __float_as_uint(h);
  lo = __float_as_uint(l);
}

// Shared-memory image of one 40-float K-block of an operand of `rows` rows (a
// multiple of 16), as the kernels store A tiles and fbbev_linear_pack stores
// weights: [hi, lo][10 chunks of 4 floats][rows / 8][8 rows][4 floats];
// kb_chunk(rows) bytes between chunks, 128 between row groups, and a k8 step
// is two chunks.
constexpr int kKB = 40;            // floats of K per block
constexpr int kKSteps = kKB / 8;   // k8 steps per block
constexpr int kb_part(int rows) { return rows * kKB * 4; }  // bytes of hi (== lo)
constexpr int kb_chunk(int rows) { return rows * 16; }

// The A tile of the kernels that stage A in shared memory: 128 rows, a
// warpgroup's 64 rows 1024 bytes (8 row groups) into each part.
constexpr int kATileM = 128;
constexpr int kAPart = kb_part(kATileM);          // bytes of A_hi (== A_lo)
constexpr int kABlock = 2 * kAPart;               // one K-block, hi + lo
constexpr int kAChunkStride = kb_chunk(kATileM);  // bytes between K chunks
// byte offset of element (row, col) of A_hi
__device__ __forceinline__ uint32_t a_off(int row, int col) {
  return (uint32_t)((col >> 2) * (kATileM / 8) + (row >> 3)) * 128u + (row & 7) * 16u +
         (col & 3) * 4u;
}

// ----------------------------- 3xTF32 products ------------------------------
// acc[64 x NPAD] (+)= A[64 x 40] . B[NPAD x 40]^T for one warpgroup, as three
// full-width tf32 products per k8 step (hi.hi, lo.hi, hi.lo) into the same
// accumulator; `accumulate` == 0 starts the accumulator with this K-block.
// Accumulator layout (wgmma m64nN, f32): acc[4 J + 2 h + e] is row
// 16 (warp % 4) + lane / 4 + 8 h, column 8 J + 2 (lane % 4) + e.
template <int NPAD>
__device__ __forceinline__ void wg_kblock_3xtf32(float (&acc)[NPAD / 2],
                                                 uint32_t a_hi, uint32_t a_lo,
                                                 uint32_t a_chunk, uint32_t b_hi,
                                                 uint32_t b_lo, uint32_t b_chunk,
                                                 uint32_t accumulate) {
  static_assert(NPAD % 16 == 0 && NPAD >= 16 && NPAD <= 256, "NPAD");
#pragma unroll
  for (int k = 0; k < kKSteps; ++k) {
    const uint64_t dah = smem_desc(a_hi + 2u * k * a_chunk, a_chunk, 128);
    const uint64_t dal = smem_desc(a_lo + 2u * k * a_chunk, a_chunk, 128);
    const uint64_t dbh = smem_desc(b_hi + 2u * k * b_chunk, b_chunk, 128);
    const uint64_t dbl = smem_desc(b_lo + 2u * k * b_chunk, b_chunk, 128);
    wgmma_tf32<NPAD>(acc, dah, dbh, k == 0 ? accumulate : 1u);
    wgmma_tf32<NPAD>(acc, dal, dbh, 1u);
    wgmma_tf32<NPAD>(acc, dah, dbl, 1u);
  }
}

// The same product with A from registers: ah / al are the hi / lo fragments
// (tf32_split, layout of wgmma_tf32_rs) of the K-block's five k8 steps.  The
// caller fences them (wgmma_fence) and keeps them until the MMAs complete.
template <int NPAD>
__device__ __forceinline__ void wg_kblock_3xtf32_rs(float (&acc)[NPAD / 2],
                                                    const uint32_t (&ah)[kKSteps][4],
                                                    const uint32_t (&al)[kKSteps][4],
                                                    uint32_t b_hi, uint32_t b_lo,
                                                    uint32_t b_chunk, uint32_t accumulate) {
  static_assert(NPAD % 16 == 0 && NPAD >= 16 && NPAD <= 256, "NPAD");
#pragma unroll
  for (int k = 0; k < kKSteps; ++k) {
    const uint64_t dbh = smem_desc(b_hi + 2u * k * b_chunk, b_chunk, 128);
    const uint64_t dbl = smem_desc(b_lo + 2u * k * b_chunk, b_chunk, 128);
    wgmma_tf32_rs<NPAD>(acc, ah[k], dbh, k == 0 ? accumulate : 1u);
    wgmma_tf32_rs<NPAD>(acc, al[k], dbh, 1u);
    wgmma_tf32_rs<NPAD>(acc, ah[k], dbl, 1u);
  }
}

}  // namespace fbbev
