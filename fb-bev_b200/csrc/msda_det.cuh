// msda_det.cuh -- records of the deterministic deformable-attention backward
// (msda_det_bwd.cu).  In deterministic mode the per-(batch, query, head)
// backward kernels of msda_bwd.cu / msda_fused_bwd.cu run unchanged except
// that, instead of adding into grad_value / grad_depth_prob with atomics, they
// write one record per bilinear sample: a key naming the sample's top-left
// corner cell and (h_im, w_im, coefficient).  msda_det_bwd.cu sorts the
// records by key (stable, so the order inside a cell is record-index order)
// and every gradient element gathers its four neighbouring cells in a fixed
// order with one plain store.
#pragma once
#include "msda_common.cuh"

namespace fbbev {

// key of a record slot that holds no sample; sorts after every real key
constexpr uint32_t kNoKey = 0xffffffffu;

// Where one pass of a backward kernel writes its records.  A pass is one
// sample (self-attention, drop-in op) or one (sample, camera) pair
// (cross-attention); record indices are local to it.
struct DetSink {
  uint32_t* key = nullptr;   // value-gradient record keys (NULL: none)
  float3* rec = nullptr;     // (h_im, w_im, coefficient)
  uint32_t* dkey = nullptr;  // depth-gradient record keys (NULL: none)
  float3* drec = nullptr;    // (h_im, w_im, head-summed depth gradient)
  float* G = nullptr;        // cross-attention: grad_out / camera count
                             // (nq, heads*ch) of the pass's sample
  int64_t item0 = 0;         // cross-attention: first (b, q, head) item
  int cam = 0;               // cross-attention: camera of the pass

  // value-gradient record r of an in-image sample of head m; `cell` is the
  // sample's padded cell (Bilinear::padded_cell) plus the padded cells of the
  // levels before its own, the key head-minor
  __device__ __forceinline__ void value_record(int64_t r, int cell, int heads,
                                               int m, float h_im, float w_im,
                                               float coef) const {
    key[r] = (uint32_t)(cell * heads + m);
    rec[r] = make_float3(h_im, w_im, coef);
  }
};

// One record pass of the backward kernels (launchers in msda_fused_bwd.cu and
// msda_bwd.cu).  Pointers are those of the pass's sample; the cross-attention
// takes the whole batch and picks its pass from det.item0 / det.cam.
int msda_fused_bwd_records(const float* value, const int64_t* spatial_shapes,
                           const int64_t* level_start, const float* ref,
                           const float* offsets, const float* logits,
                           const float* grad_out, int n_value, int heads,
                           int ch, int levels, int nq, int points,
                           float* grad_offsets, float* grad_logits,
                           const DetSink& det, cudaStream_t st);
int da_sca_bwd_records(const float* value, const float* depth_prob,
                       const float* ref_cam, const float* ref_depth,
                       const uint8_t* mask, const float* offsets,
                       const float* logits, const int64_t* spatial_shapes,
                       const int64_t* level_start, const DaScaParams& P,
                       int ch, int Z, const float* grad_out,
                       float* grad_offsets, float* grad_logits,
                       const DetSink& det, cudaStream_t st);
int msda_bwd_records(const float* value, const int64_t* spatial_shapes,
                     const int64_t* level_start, const float* loc,
                     const float* attw, const float* grad_out, int n_value,
                     int heads, int ch, int levels, int nq, int points,
                     float* grad_loc, float* grad_attw, const DetSink& det,
                     cudaStream_t st);

}  // namespace fbbev
