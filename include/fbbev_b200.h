/*
 * fbbev_b200.h -- C ABI of libfbbev_b200.so: the H100 (sm_90a) implementation
 * of the FB-BEV / FB-OCC forward-backward view-transformation hot path.
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes only; every pointer is a DEVICE pointer unless
 *     the parameter name ends in `_host`;
 *   - the caller owns every buffer including workspaces; nothing is allocated,
 *     no host<->device synchronisation happens inside a call, and all work is
 *     enqueued on `stream` (a cudaStream_t; NULL = legacy default stream);
 *   - return value: 0 on success, a negative FBBEV_ERR_* for argument errors,
 *     or a positive cudaError_t raised while enqueuing.  Nothing throws.
 *   - re-entrant per stream; no global mutable state.
 *
 * Each entry point names the reference interface it replaces (paths relative
 * to the NVlabs/FB-BEV checkout).  INTEGRATION.md shows the reference-side
 * binding for each.
 */
#ifndef FBBEV_B200_H_
#define FBBEV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FBBEV_OK 0
#define FBBEV_ERR_INVALID_ARGUMENT (-1)
#define FBBEV_ERR_WORKSPACE_TOO_SMALL (-2)
#define FBBEV_ERR_UNSUPPORTED (-3)

#define FBBEV_ABI_VERSION 5

typedef void* fbbev_stream_t; /* cudaStream_t */

int fbbev_abi_version(void);
/* Diagnostics: cumulative number of kernel launches issued by this library. */
long long fbbev_debug_launch_count(void);
/* Static string for a return code of any entry point. */
const char* fbbev_error_string(int code);

/* =====================================================================
 * F -- lift-splat voxel pooling (bev_pool_v2)
 * ===================================================================== */

/*
 * Drop-in for `bev_pool_v2_ext.bev_pool_v2_forward`
 *   mmdet3d/ops/bev_pool_v2/src/bev_pool.cpp:28-55 (launcher
 *   bev_pool_cuda.cu:120-128, kernel :18-45).
 * depth (B,N,D,H,W) fp32; feat (B,N,H,W,C) fp32; index arrays int32;
 * out (B,Z,Y,X,C) fp32, ZERO-FILLED BY THE CALLER as in bev_pool.py:25.
 * Semantics identical to the reference for arbitrary interval lists: one
 * plain store of the interval sum to voxel ranks_bev[interval_starts[i]].
 * Differences: 64-bit offsets (the reference overflows int32 when
 * B*Z*Y*X*C >= 2^31) and the caller's stream instead of the legacy stream.
 */
int fbbev_bev_pool_v2_fwd(const float* depth, const float* feat,
                          const int32_t* ranks_depth,
                          const int32_t* ranks_feat, const int32_t* ranks_bev,
                          const int32_t* interval_starts,
                          const int32_t* interval_lengths, int32_t n_intervals,
                          int32_t c, float* out, fbbev_stream_t stream);

/*
 * Fused replacement for the whole reference op
 *   `bev_pool_v2()` = QuickCumsumCuda.forward + permute(0,4,1,2,3).contiguous()
 *   mmdet3d/ops/bev_pool_v2/bev_pool.py:15-39, 84-90.
 * Writes EVERY element of out exactly once, directly in the op's final
 * (B,C,Z,Y,X) layout: no caller-side memset, no transpose pass.
 *
 * Precondition (what voxel_pooling_prepare_v2 always produces,
 * view_transformer.py:590-602): intervals are listed in non-decreasing order
 * of their voxel rank ranks_bev[interval_starts[i]], one interval per voxel.
 * Out-of-range ranks are ignored (memory-safe).
 *
 * Two calls:
 *   _plan     builds the tile table of a given (index, C) into `workspace`
 *             (>= fbbev_bev_pool_v2_dense_workspace_bytes(...) bytes);
 *   _planned  runs the pooling kernels from it.  The workspace doubles as
 *             their scratch, so `_planned` writes it as well: one workspace
 *             per concurrent stream.
 * A caller that reuses an index (static camera rig, `accelerate=True`,
 * view_transformer.py:261-283) plans once; fbbev_voxel_prepare(_cams) can
 * fill the plan while it builds the index, so no `_plan` launch is needed.
 *
 * n_intervals_dev: optional device int32 holding the live interval count
 *   (<= n_intervals_max); NULL means n_intervals_max is the count.  This lets
 *   the prepare -> pool chain run without a host sync / under CUDA graphs.
 * n_points = number of entries in ranks_bev / ranks_depth / ranks_feat (an
 *   upper bound of the kept points when the buffers are over-allocated).
 * n_voxels_per_sample = Z*Y*X.
 * Any C > 0 and volume.  Two kernels write every element once when
 * C % 4 == 0, Z*Y*X % 4 == 0, 4 <= C <= 512 and B*Z*Y*X < 2^31 (every shape
 * the model runs; out must then be 16-byte aligned); any other shape is
 * zero-filled and then written by the drop-in kernel above, its (B,Z,Y,X,C)
 * store address transposed to (B,C,Z,Y,X), so its output is bit-identical to
 * fbbev_bev_pool_v2_fwd + permute(0,4,1,2,3).
 */
size_t fbbev_bev_pool_v2_dense_workspace_bytes(int32_t batch,
                                               int64_t n_voxels_per_sample,
                                               int32_t n_intervals_max,
                                               int32_t n_points, int32_t c);
int fbbev_bev_pool_v2_plan(const int32_t* ranks_bev,
                           const int32_t* interval_starts,
                           const int32_t* interval_lengths,
                           int32_t n_intervals_max,
                           const int32_t* n_intervals_dev, int32_t n_points,
                           int32_t c, int32_t batch,
                           int64_t n_voxels_per_sample, void* workspace,
                           size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_bev_pool_v2_fwd_dense_planned(
    const float* depth, const float* feat, const int32_t* ranks_depth,
    const int32_t* ranks_feat, const int32_t* ranks_bev,
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, float* out, void* plan, size_t plan_bytes,
    fbbev_stream_t stream);

/*
 * The dense op in stages, for FBOCC's glue around the two projections
 * (mmdet3d/models/fbbev/detectors/fbocc.py:339, 357-366):
 *     bev_feat = forward_projection(...)                       # dense volume
 *     refined  = backward_projection(..., lss_bev=bev_feat.mean(-1), ...)
 *     bev_feat = refined[..., None] + bev_feat                 # re-add
 * reads the 204.8 MB volume twice and writes it twice.  After
 * fbbev_bev_pool_v2_plan on the same workspace:
 *   _sums_planned   runs the interval-sum stage only (V / X rows in the plan);
 *   _zmean_planned  writes bev_feat.mean(-1) as a TOKEN-major map
 *                   lss_tokens (B, Y*X, C) from the interval sums (one warp
 *                   per (b, y, x) sums its Z voxels in z order: the same
 *                   bits on every run);
 *                   yx = Y*X;
 *   _write_planned  materialises the (B,C,Z,Y,X) volume, adding `add` (may be
 *                   NULL; (B, C, Y*X), e.g. the refined BEV) to every Z slice
 *                   on the way out -- the volume is written exactly once.
 * Requirements: a shape the dense op runs with two kernels (C % 4 == 0,
 * (Z*Y*X) % 4 == 0, 4 <= C <= 512, B*Z*Y*X < 2^31) and yx % 4 == 0;
 * FBBEV_ERR_UNSUPPORTED otherwise (use the one-shot op and eager glue).
 */
int fbbev_bev_pool_v2_sums_planned(
    const float* depth, const float* feat, const int32_t* ranks_depth,
    const int32_t* ranks_feat, const int32_t* ranks_bev,
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, void* plan, size_t plan_bytes,
    fbbev_stream_t stream);
int fbbev_bev_pool_v2_zmean_planned(
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, int32_t yx, float* lss_tokens, void* plan,
    size_t plan_bytes, fbbev_stream_t stream);
int fbbev_bev_pool_v2_write_planned(
    const int32_t* interval_starts, const int32_t* interval_lengths,
    int32_t n_intervals_max, int32_t n_points, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, int32_t yx, const float* add, float* out,
    void* plan, size_t plan_bytes, fbbev_stream_t stream);

/*
 * Drop-in for `bev_pool_v2_ext.bev_pool_v2_backward`
 *   mmdet3d/ops/bev_pool_v2/src/bev_pool.cpp:72-102 (kernel
 *   bev_pool_cuda.cu:64-118).  Intervals are runs of equal ranks_feat
 *   (bev_pool.py:45-55).  out_grad (B,Z,Y,X,C); depth_grad / feat_grad
 *   zero-filled by the caller (bev_pool.py:65-66).  Any C > 0, as the
 *   forward: up to 512 channels in one launch, wider rows in launches of 512
 *   channels whose depth dot products add to the first one's.
 */
int fbbev_bev_pool_v2_bwd(const float* out_grad, const float* depth,
                          const float* feat, const int32_t* ranks_depth,
                          const int32_t* ranks_feat, const int32_t* ranks_bev,
                          const int32_t* interval_starts,
                          const int32_t* interval_lengths, int32_t n_intervals,
                          int32_t c, float* depth_grad, float* feat_grad,
                          fbbev_stream_t stream);

/*
 * Same contract as fbbev_bev_pool_v2_bwd, but out_grad is (B,C,Z,Y,X) -- the
 * layout of the tensor `bev_pool_v2()` returns (bev_pool.py:89), i.e. the
 * gradient as autograd delivers it -- so the full-volume transpose copy the
 * reference performs first (`out_grad.contiguous()`, bev_pool.py:67) is skipped.
 */
int fbbev_bev_pool_v2_bwd_bczyx(
    const float* out_grad, const float* depth, const float* feat,
    const int32_t* ranks_depth, const int32_t* ranks_feat,
    const int32_t* ranks_bev, const int32_t* interval_starts,
    const int32_t* interval_lengths, int32_t n_intervals, int32_t c,
    int64_t n_voxels_per_sample, float* depth_grad, float* feat_grad,
    fbbev_stream_t stream);

/*
 * The backward of the dense op without a host sync, for training
 *   (QuickCumsumCuda.backward, mmdet3d/ops/bev_pool_v2/bev_pool.py:42-81, and
 *   the gradient of FBOCC's glue, mmdet3d/models/fbbev/detectors/
 *   fbocc.py:357-366).  Three stages:
 *   _order    once per index: sorts the kept points stably by ranks_feat on
 *             the device (the order of bev_pool.py:45-55's stable sort) and
 *             maps every point and voxel to its interval.  The live counts
 *             come from n_kept_dev / n_intervals_dev (NULL: n_points /
 *             n_intervals_max); ranks_feat must be < n_pix = B*N*H*W.
 *             `order` holds the result: >=
 *             fbbev_bev_pool_v2_bwd_order_workspace_bytes(...) bytes, read by
 *             the two stages below, which take the same n_points, n_pix, c,
 *             batch and n_voxels_per_sample.
 *   _rows     grad_rows[i][c] = out_grad[b, c, voxel of interval i] for every
 *             live interval (grad_rows: n_intervals_max rows of c floats; the
 *             rows of dead intervals are not written), out_grad (B,C,Z,Y,X)
 *             read once, tile by tile.  grad_sum_z (may be NULL): (B, C, yx)
 *             = out_grad summed over Z in z order from +0 (the gradient of
 *             the re-add `refined[..., None] + bev_feat`); yx = Y*X, or Z*Y*X
 *             when no Z sum is wanted.  out_grad and grad_sum_z 16-byte
 *             aligned.
 *   _ordered  depth_grad / feat_grad from the rows, bit-identical to
 *             fbbev_bev_pool_v2_bwd_bczyx on the stably feature-sorted
 *             intervals (both run C <= 512 in one pass).  grad_lss_tokens (may be NULL): the gradient of
 *             bev_feat.mean(-1) as a token-major (B, yx, C) map, added to
 *             every row on load as torch's mean backward and gradient sum
 *             round it (g + g_lss * (1/Z), Z = n_voxels_per_sample / yx).
 *             grad_rows may be NULL when grad_lss_tokens is given (the
 *             volume itself has no gradient: rows are g_lss * (1/Z) alone).
 *             feat_grad is written in full; depth_grad is zero-filled by the
 *             caller (only the slots of kept points are written).
 * No host sync and no float atomics: the same bits on every run.
 * Shapes: those the dense op runs with two kernels (C % 4 == 0,
 * Z*Y*X % 4 == 0, 4 <= C <= 512, B*Z*Y*X < 2^31); FBBEV_ERR_UNSUPPORTED,
 * before anything is enqueued, for any other (use fbbev_bev_pool_v2_bwd_bczyx).
 * batch == 0 is a no-op.
 * FBOCC's glue under autograd runs the sequence sums_planned -> zmean_planned
 * -> (backward projection) -> write_planned(add) forward and _rows with
 * grad_sum_z (the re-add's gradient of `refined`) -> _ordered with
 * grad_lss_tokens backward: the volume's gradient is read once.
 */
size_t fbbev_bev_pool_v2_bwd_order_workspace_bytes(
    int32_t n_points, int32_t n_pix, int32_t batch,
    int64_t n_voxels_per_sample);
int fbbev_bev_pool_v2_bwd_order(
    const int32_t* ranks_depth, const int32_t* ranks_feat,
    const int32_t* ranks_bev, const int32_t* interval_starts,
    const int32_t* interval_lengths, int32_t n_points,
    int32_t n_intervals_max, const int32_t* n_kept_dev,
    const int32_t* n_intervals_dev, int32_t n_pix, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, void* order, size_t order_bytes,
    fbbev_stream_t stream);
int fbbev_bev_pool_v2_bwd_rows(
    const float* out_grad, int32_t c, int32_t batch,
    int64_t n_voxels_per_sample, int32_t yx, const void* order,
    size_t order_bytes, int32_t n_points, int32_t n_pix, float* grad_rows,
    float* grad_sum_z, fbbev_stream_t stream);
int fbbev_bev_pool_v2_bwd_ordered(
    const float* grad_rows, const float* grad_lss_tokens, const float* depth,
    const float* feat, int32_t c, int32_t batch, int64_t n_voxels_per_sample,
    int32_t yx, const void* order, size_t order_bytes, int32_t n_points,
    int32_t n_pix, float* depth_grad, float* feat_grad,
    fbbev_stream_t stream);

/*
 * Device implementation of `voxel_pooling_prepare_v2`
 *   mmdet3d/models/fbbev/view_transformation/forward_projection/
 *   view_transformer.py:547-605  (integer path, bit-exact).
 * coor (B,N,D,H,W,3) fp32 ego-frame points from get_lidar_coor (:458-498).
 * lo/iv/gs: grid lower bound, interval and FLOAT32 grid size (:384-387).
 * Outputs (each sized for B*N*D*H*W entries): ranks_bev / ranks_depth /
 * ranks_feat sorted by voxel rank, ascending point index inside a voxel
 * (a stable sort; the reference's argsort order inside a voxel is
 * unspecified), interval_starts / interval_lengths; counts[0] = n_kept,
 * counts[1] = n_intervals (device int32[2]).
 * Voxel rank is computed in exact integer arithmetic; the reference computes
 * it in float32 (:586-589), which is identical while B*Z*Y*X < 2^24.
 * Requires B*Z*Y*X < 2^31 and B*N*D*H*W < 2^31.
 *
 * depth_prob (may be NULL: no threshold) adds the depth-threshold
 * sparsification of the BEVDet-lineage transformer
 *   mmdet3d/models/necks/view_transformer.py:520-578 (LSSViewTransformer2.
 *   voxel_pooling_prepare_v2: `kept = kept & (depth.view(-1) > 0.01)`, :556-557)
 *   and its cached-index form (:645-678: the geometric index filtered by
 *   `(depth.view(-1) > 0.01)[self.kept]` on every forward):
 * depth_prob (B,N,D,H,W) fp32 -- the tensor the pooling op will read, indexed
 * by the point index (ranks_depth == arange); a point is kept when
 * depth_prob[p] > depth_thresh (strict, as the reference).
 *
 * pool_plan (may be NULL): a dense-pooling workspace of
 * fbbev_bev_pool_v2_dense_workspace_bytes(B, Z*Y*X, min(n_points, B*Z*Y*X),
 * n_points, pool_c) bytes.  When given, the scan over the voxel histogram also
 * fills the pooling plan (what fbbev_bev_pool_v2_plan computes in a launch of
 * its own), so the index can go straight to fbbev_bev_pool_v2_fwd_dense_planned
 * / _sums_planned with the same workspace and n_intervals_max = min(n_points,
 * B*Z*Y*X).  A plan needs pool_c > 0, else FBBEV_ERR_UNSUPPORTED.
 * Argument errors are reported before anything is enqueued.
 */
size_t fbbev_voxel_prepare_workspace_bytes(int64_t n_points,
                                           int64_t n_voxels_total);
int fbbev_voxel_prepare(
    const float* coor, const float* depth_prob, float depth_thresh, int32_t B,
    int32_t N, int32_t D, int32_t H, int32_t W, const float* lo_host,
    const float* iv_host, const float* gs_host, int32_t* ranks_bev,
    int32_t* ranks_depth, int32_t* ranks_feat, int32_t* interval_starts,
    int32_t* interval_lengths, int32_t* counts, void* workspace,
    size_t workspace_bytes, int32_t pool_c, void* pool_plan,
    size_t pool_plan_bytes, fbbev_stream_t stream);

/*
 * fbbev_voxel_prepare with get_lidar_coor fused in
 *   (view_transformer.py:458-498 + 547-605): the (B,N,D,H,W,3) coordinate tensor
 *   is never materialised.  frustum_u [W], frustum_v [H], frustum_d [D] are the
 *   three axes of the frustum template (create_frustum, :389-411);
 *   inv_post_rots = inverse(post_rots) (B*N,3,3); cam2ego = rots @ inverse(K)
 *   (B*N,3,3) -- the two tiny products the reference also forms before touching
 *   the points (:483-491); post_trans, trans (B*N,3); bda (B,3,3).
 * The per-point chain is evaluated in fp32 in the rounding order the reference's
 * eager chain has on this device (torch broadcast matmul -> cuBLAS): per output
 * row fma(m1, x1, m0*x0) + m2*x2, or -- FBBEV_ORDER_SEQ_* bit set -- the
 * sequential chain fma(m2, x2, fma(m1, x1, m0*x0)) cuBLAS uses when ONE
 * column-major matrix (the layout torch.inverse returns) is broadcast over the
 * whole batch.  order_flags: bit 0 inv_post_rots, bit 1 cam2ego, bit 2 bda.
 * The index is bit-identical to fbbev_voxel_prepare on get_lidar_coor's output.
 * Everything else (depth_prob, pool_plan) as fbbev_voxel_prepare.
 */
#define FBBEV_ORDER_SEQ_A 1
#define FBBEV_ORDER_SEQ_B 2
#define FBBEV_ORDER_SEQ_C 4
/* fbbev_point_sampling only: with this bit set, bits [8 + 5 i, 13 + 5 i) hold
 * the summation order of matrix stack i (0 inv_bda, 1 ego2cam, 2 post_rots) as
 * code = 6 last + 2 inner + outer (csrc/common.cuh, dot3_code): one of the 18
 * fp32 ways to sum three products with or without FMA.  torch's broadcast
 * matmul picks its cuBLAS kernel -- and with it the order -- by problem size
 * and device, so the caller finds the code for each shape (see
 * _lib.matmul_order_codes). */
#define FBBEV_ORDER_EXPLICIT 8
int fbbev_voxel_prepare_cams(
    const float* frustum_u, const float* frustum_v, const float* frustum_d,
    const float* inv_post_rots, const float* post_trans, const float* cam2ego,
    const float* trans, const float* bda, int32_t order_flags,
    const float* depth_prob, float depth_thresh, int32_t B, int32_t N,
    int32_t D, int32_t H, int32_t W, const float* lo_host,
    const float* iv_host, const float* gs_host, int32_t* ranks_bev,
    int32_t* ranks_depth, int32_t* ranks_feat, int32_t* interval_starts,
    int32_t* interval_lengths, int32_t* counts, void* workspace,
    size_t workspace_bytes, int32_t pool_c, void* pool_plan,
    size_t pool_plan_bytes, fbbev_stream_t stream);

/*
 * The tail of the depth net as the PRODUCER of the pooling op's inputs
 * (SURVEY.md section 8 f4 / f3):
 *   CM_DepthNet.forward   mmdet3d/models/fbbev/modules/depth_net.py:359-363
 *       depth = depth.softmax(dim=1); context.view(B, N, C, H, W)
 *   LSSViewTransformer / LSSViewTransformer2 / LSSViewTransformerBEVDepth.forward
 *       mmdet3d/models/necks/view_transformer.py:313-321, 710-718, 1094-1096
 *       depth_digit = x[:, :D]; tran_feat = x[:, D:D+C]; depth = softmax(dim=1)
 *   + the `feat.permute(0,1,3,4,2)` / `feat.contiguous()` transposing copy inside
 *     the pooling op (view_transformer.py:530, bev_pool.py:19).
 * depth_logits: image n, bin k, pixel p at [n * logits_image_stride + k*hw + p]
 * (NCHW with its own image stride, so a channel slice of a wider tensor works);
 * context likewise with c channels.  Either may be NULL (that half is skipped).
 * depth_out (bn, d, hw) = softmax over the d bins (max / sum of expf / divide,
 * as torch); feat_out (bn, hw, c) = context transposed to pixel-major -- the
 * (B,N,H,W,C) layout `bev_pool_v2` reads.  One launch.
 */
int fbbev_lift_tail_fwd(const float* depth_logits, int64_t logits_image_stride,
                        const float* context, int64_t context_image_stride,
                        int32_t bn, int32_t d, int32_t c, int32_t hw,
                        float* depth_out, float* feat_out,
                        fbbev_stream_t stream);

/* =====================================================================
 * B -- BEV -> image depth-aware spatial cross-attention (MSDeformAttn)
 * ===================================================================== */

/*
 * One-kernel `bevformer_encoder.point_sampling`
 *   .../backward_projection/bevformer_utils/bevformer_encoder.py:92-120.
 * X [nX], Y [nY], Z [nZ]: voxel-centre coordinates per axis (get_reference_points
 * '3d', :64-70); inv_bda = inverse(bda) (B,3,3); ego2cam = inverse(rots @
 * inverse(K)) (B*N,3,3); trans, post_trans (B*N,3); post_rots (B*N,3,3);
 * (w_in, h_in) = data_config input_size; eps = 1e-5 and one_minus_eps =
 * (float)(1.0 - 1e-5), the two scalars of the visibility test (:113-117).
 * order_flags as for fbbev_voxel_prepare_cams: bit 0 inv_bda, bit 1 ego2cam,
 * bit 2 post_rots.  The image-plane normalisation multiplies by (1 / w_in),
 * (1 / h_in) as torch's CUDA `tensor /= python_scalar` does.
 * Outputs in the reference's layouts: ref_cam (N,B,nY*nX,nZ,2), depth
 * (N,B,nY*nX,nZ), mask (N,B,nY*nX,nZ) uint8; bit-identical to the eager chain.
 */
int fbbev_point_sampling(
    const float* X, const float* Y, const float* Z, int32_t nX, int32_t nY,
    int32_t nZ, const float* inv_bda, const float* trans, const float* ego2cam,
    const float* post_rots, const float* post_trans, int32_t order_flags,
    int32_t B, int32_t N, float w_in, float h_in, float eps,
    float one_minus_eps, float* ref_cam, float* depth, uint8_t* mask,
    fbbev_stream_t stream);

/*
 * BEV queries of `BackwardProjection.forward`
 *   .../backward_projection/backward_projection.py:93-97:
 *   out[b, q, :] = embedding[q, :] + lss_bev[b, :, q]   (lss_bev may be NULL)
 * embedding (nq, E) = bev_embedding.weight; lss_bev (bs, E, bev_h*bev_w) = the
 * lift-splat BEV, channel-major; out (bs, nq, E) contiguous (the reference's
 * (nq, bs, E) tensor is its permuted view).  One pass, one fp32 add per element.
 */
int fbbev_bev_query_init(const float* embedding, const float* lss_bev,
                         int32_t bs, int32_t nq, int32_t E, float* out,
                         fbbev_stream_t stream);

/*
 * out[b, e, q] = tokens[b, q, e]: the last line of `BackwardProjection.forward`
 *   (backward_projection.py:131-133: bev.permute(0, 2, 1).view(bs, -1, bev_h,
 *   bev_w).contiguous()).  tokens (bs, nq, E), out (bs, E, nq), both dense fp32,
 *   16-byte aligned; nq % 4 == 0 and E % 4 == 0, else FBBEV_ERR_UNSUPPORTED.
 */
int fbbev_tokens_to_map(const float* tokens, int32_t bs, int32_t nq, int32_t E,
                        float* out, fbbev_stream_t stream);

/*
 * Drop-in for `ext_module.ms_deform_attn_forward` (mmcv-full 1.5.2 `_ext`)
 *   call site: .../backward_projection/bevformer_utils/
 *   multi_scale_deformable_attn_function.py:127-133.
 * value (bs, n_value, heads, ch) fp32; spatial_shapes (levels,2) and
 * level_start (levels) are DEVICE int64 as in the reference
 * (bevformer.py:108-111); loc (bs,nq,heads,levels,points,2) as (x,y) in
 * [0,1]; attw (bs,nq,heads,levels,points); out (bs,nq,heads*ch).
 * No im2col_step restriction.  For ch in {4, 8, 10, 16, 20, 32, 64}, value /
 * out aligned to the head's vector width (16 bytes for ch % 4 == 0, 8 for
 * even ch), else FBBEV_ERR_INVALID_ARGUMENT.
 */
int fbbev_msda_fwd(const float* value, const int64_t* spatial_shapes,
                   const int64_t* level_start, const float* loc,
                   const float* attw, int32_t bs, int32_t n_value,
                   int32_t heads, int32_t ch, int32_t levels, int32_t nq,
                   int32_t points, float* out, fbbev_stream_t stream);

/*
 * Drop-in for `ext_module.ms_deform_attn_backward`
 *   call site: multi_scale_deformable_attn_function.py:159-169.
 * grad_value / grad_loc / grad_attw zero-filled by the caller (:155-157).
 */
int fbbev_msda_bwd(const float* value, const int64_t* spatial_shapes,
                   const int64_t* level_start, const float* loc,
                   const float* attw, const float* grad_out, int32_t bs,
                   int32_t n_value, int32_t heads, int32_t ch, int32_t levels,
                   int32_t nq, int32_t points, float* grad_value,
                   float* grad_loc, float* grad_attw, fbbev_stream_t stream);

/*
 * Fused core of mmcv `MultiScaleDeformableAttention.forward` (the encoder
 * layer's self_attn, fbocc-r50 config :176-180): softmax over levels*points,
 * sampling_locations = ref + offsets / (W_l, H_l), bilinear sampling and
 * weighted sum in one kernel -- `loc` / normalised `attw` never touch HBM.
 * ref (bs,nq,levels,2); offsets (bs,nq,heads,levels,points,2) = raw output of
 * the sampling_offsets Linear; logits (bs,nq,heads,levels,points) = raw output
 * of the attention_weights Linear; out (bs,nq,heads*ch).
 * patch_w: 0, or -- for self-attention over the map itself (levels == 1, nq ==
 * n_value, 8 heads) -- the map width W: query q = y * W + x then sits on value
 * pixel (y, x) and blocks own 8x8 query squares (L1-resident footprint) instead
 * of runs of a row; at ch == 10, 4 points and a map of at least 18 x 18 pixels
 * the square's footprint is staged in shared memory (msda_self_smem.cu; needs
 * value, offsets, logits and out 16-byte aligned, else the 8x8 global kernel
 * runs).  Results do not depend on it.
 * value / out aligned to the head's vector width (16 bytes for ch % 4 == 0,
 * 8 for even ch), else FBBEV_ERR_INVALID_ARGUMENT.
 */
int fbbev_msda_fused_fwd(const float* value, const int64_t* spatial_shapes,
                         const int64_t* level_start, const float* ref,
                         const float* offsets, const float* logits, int32_t bs,
                         int32_t n_value, int32_t heads, int32_t ch,
                         int32_t levels, int32_t nq, int32_t points,
                         int32_t patch_w, float* out, fbbev_stream_t stream);

/*
 * Backward of fbbev_msda_fused_fwd (same arguments without patch_w, plus
 * grad_out (bs,nq,heads*ch)).  Everything is recomputed from the forward's
 * inputs; nothing in between is materialised.
 * grad_value (bs,n_value,heads,ch): accumulated with atomics (vector
 *   reductions; summation order not fixed), ZERO-FILLED BY THE CALLER;
 * grad_offsets (bs,nq,heads,levels,points,2), grad_logits
 *   (bs,nq,heads,levels,points): every element written by the call.
 * reference_points get no gradient.  Any grad pointer may be NULL: that
 * gradient is not computed.  value / grad_out / grad_value aligned to the
 * head's vector width (16 bytes for ch % 4 == 0, 8 for even ch).
 * Head widths outside {4, 8, 10, 16, 20, 32, 64}: FBBEV_ERR_UNSUPPORTED.
 */
int fbbev_msda_fused_bwd(const float* value, const int64_t* spatial_shapes,
                         const int64_t* level_start, const float* ref,
                         const float* offsets, const float* logits,
                         const float* grad_out, int32_t bs, int32_t n_value,
                         int32_t heads, int32_t ch, int32_t levels,
                         int32_t nq, int32_t points, float* grad_value,
                         float* grad_offsets, float* grad_logits,
                         fbbev_stream_t stream);

/*
 * Fused depth-aware spatial cross-attention: everything between the three
 * input Linears and `output_proj` of
 *   DA_SpatialCrossAttention.forward   spatial_cross_attention_depth.py:86-223
 *   DA_MSDeformableAttention.forward   spatial_cross_attention_depth.py:465-601
 * i.e. per-camera query selection (:156-169), rebatch (:173-186), depth bin
 * one-hot (:196-199), softmax (:540), sampling locations (:554-570), the depth
 * look-up MSDA launch (:584-591), depth re-weighting (:592), the main MSDA
 * launch (:593-595), scatter-add over cameras (:208-211) and the division by
 * the per-query camera count (:213-216).
 *
 * value      (bs*n_cams, n_value, heads, ch)  value_proj(feat), camera-major
 *            inside a sample (row = b*n_cams + cam), as at :188-191
 * depth_prob (bs*n_cams, H0*W0, DC)  pred_img_depth flattened as at :131-133
 * ref_cam    (n_cams, bs, nq, Z, 2)  reference_points_cam (bevformer_encoder.py:117)
 * ref_depth  (n_cams, bs, nq, Z)     bev_query_depth (:120)
 * mask       (n_cams, bs, nq, Z) uint8   per_cam_mask_list (:118)
 * offsets    (bs, nq, heads, levels, points, 2)  raw sampling_offsets(query)
 * logits     (bs, nq, heads, levels, points)     raw attention_weights(query)
 *   (both Linears act row-wise, so evaluating them once per BEV query equals
 *    the reference's evaluation on the re-batched copies)
 * points = num_points (all Z anchors), Z = num_Z_anchors, point index
 *   = p*Z + z (:563-570, :590).
 * dbound_host = (d_min, d_max, d_step) (:196); DC = depth bins.
 * out        (bs, nq, heads*ch) = slots / clamp(count, 1), the tensor the
 *            reference feeds to output_proj (:219).
 * bev_mask (:156-159): pass the output of fbbev_bev_mask_fold as `mask`.
 * Mask bytes: 0 = not visible; bit 0 set = visible and counted in the camera
 * mean; 2 = visible but not counted (the reference's empty-camera rule).
 *
 * workspace (fbbev_da_sca_workspace_bytes(bs, n_cams) bytes, may be NULL):
 * with it, and when one camera's value map fits in shared memory (n_value *
 * heads * ch * 4 <= ~220 KB; 8 heads x 10 channels, 1 level, 8 points, 4
 * anchors -- the FB-OCC head), the camera-resident kernel of da_sca_smem.cu
 * runs: a CTA stages its camera's map with TMA bulk copies and serves the
 * queries that camera sees from shared memory; contributions of several
 * cameras to one query are combined with red.global.add on the zero-filled
 * output (the order of these <= n_cams additions is not fixed).  Without a
 * workspace, or for other shapes, the one-thread-per-(query, head) kernel
 * gathers from global memory.  value / out aligned to the head's vector
 * width (16 bytes for ch % 4 == 0, 8 for even ch), else
 * FBBEV_ERR_INVALID_ARGUMENT.
 */
size_t fbbev_da_sca_workspace_bytes(int32_t bs, int32_t n_cams);
int fbbev_da_sca_fwd(const float* value, const float* depth_prob,
                     const float* ref_cam, const float* ref_depth,
                     const uint8_t* mask, const float* offsets,
                     const float* logits, const int64_t* spatial_shapes,
                     const int64_t* level_start, const float* dbound_host,
                     int32_t bs, int32_t n_cams, int32_t nq, int32_t n_value,
                     int32_t heads, int32_t ch, int32_t levels, int32_t points,
                     int32_t Z, int32_t DC, float* out, void* workspace,
                     size_t workspace_bytes, int32_t prologue_done,
                     fbbev_stream_t stream);
/* The mask-only part of fbbev_da_sca_fwd's camera-resident path (per-camera
 * visible-query counts into `workspace`, zero-fill of `out`), callable ahead of
 * time -- e.g. on the stream that produced the mask, beside the self-attention.
 * Pass the same `out` / `workspace` to fbbev_da_sca_fwd with prologue_done = 1.
 * FBBEV_ERR_UNSUPPORTED when the shape takes the global-memory kernel. */
int fbbev_da_sca_prologue(const uint8_t* mask, int32_t bs, int32_t n_cams,
                          int32_t nq, int32_t n_value, int32_t heads,
                          int32_t ch, int32_t levels, int32_t points, int32_t Z,
                          float* out, void* workspace, size_t workspace_bytes,
                          fbbev_stream_t stream);

/*
 * Backward of fbbev_da_sca_fwd: same inputs and mask encoding (the camera
 * count of a query is taken from mask bit 0 exactly as in the forward), plus
 * grad_out (bs,nq,heads*ch).  One thread per (sample, query, head) recomputes
 * softmax, locations and depth weights and walks the cameras that see the
 * query; the pairs no camera sees cost nothing.
 * grad_value (bs*n_cams,n_value,heads,ch) and grad_depth_prob
 *   (bs*n_cams,H0*W0,DC): accumulated with atomics, ZERO-FILLED BY THE CALLER;
 * grad_offsets / grad_logits: every element written (zeros for queries no
 *   camera sees).
 * ref_cam / ref_depth / mask get no gradient.  NULL grad pointers are skipped
 * (e.g. a frozen depth net: no depth atomics at all).  Alignment as for
 * fbbev_msda_fused_bwd.  Head widths outside {4, 8, 10, 16, 20, 32, 64} and
 * Z outside {1, 2, 4, 8}: FBBEV_ERR_UNSUPPORTED.
 */
int fbbev_da_sca_bwd(const float* value, const float* depth_prob,
                     const float* ref_cam, const float* ref_depth,
                     const uint8_t* mask, const float* offsets,
                     const float* logits, const int64_t* spatial_shapes,
                     const int64_t* level_start, const float* dbound_host,
                     const float* grad_out, int32_t bs, int32_t n_cams,
                     int32_t nq, int32_t n_value, int32_t heads, int32_t ch,
                     int32_t levels, int32_t points, int32_t Z, int32_t DC,
                     float* grad_value, float* grad_depth_prob,
                     float* grad_offsets, float* grad_logits,
                     fbbev_stream_t stream);

/*
 * Deterministic twins of the three attention backward entry points
 * (msda_det_bwd.cu): the arguments of fbbev_msda_fused_bwd / fbbev_da_sca_bwd
 * / fbbev_msda_bwd plus a caller-owned workspace of at least
 * fbbev_*_bwd_det_workspace_bytes(...) bytes (sizes only; 0 for an empty
 * problem), FBBEV_ERR_WORKSPACE_TOO_SMALL when it is short.  No float is
 * accumulated with atomics, and every output is a function of the inputs
 * alone: bit-identical across runs and processes on one GPU model, and
 * independent of bs (each sample is computed by itself).
 *   - grad_offsets / grad_loc, grad_logits / grad_attw: the twin's per-thread
 *     arithmetic, bit-identical to the twin's result.
 *   - grad_value and grad_depth_prob are written whole, each element once
 *     (no zero-fill needed).  Element (pixel (y, x), head, channel) -- or
 *     (camera, pixel (y, x), depth bin) -- is the sum, from +0 and left to
 *     right in fp32, of the twin's rounded per-sample products, ordered by
 *       1. corner k = 0, 1, 2, 3: the samples whose top-left corner cell
 *          (h_low, w_low) is (y - (k >> 1), x - (k & 1)), i.e. the element
 *          is their corner k (weights hh*hw, hh*lw, lh*hw, lh*lw);
 *       2. within a cell, the sample index: (query, point) for grad_value
 *          (head and level are the element's), (query, z) for grad_depth_prob
 *          -- (query, head, z) when heads does not divide 32, where the twin
 *          scatters each head's share; otherwise the head sum of the twin's
 *          shuffle reduction.
 *     Products: (a * w) * g for the fused samplers, w * (g * attw) for
 *     fbbev_msda_bwd, w * g_depth for the depth look-up.
 * Workspace (each array rounded up to 256 B, plus 255 B): per record set of
 * n slots and K cell keys, 28 n + 1024 ceil(n / 1024) + 8 K bytes (+ scan
 * totals); value records n = nq*heads*levels*points, K = heads*(2*n_value +
 * 2*levels); the cross-attention adds G (4*nq*heads*ch) and depth records
 * n = n_cams*nq*(32 % heads ? heads : 1)*Z, K = n_cams*(2*n_value + 2)*DC.
 * fbbev_msda_bwd_det takes any ch; the others the twin's head widths / Z.
 */
size_t fbbev_msda_fused_bwd_det_workspace_bytes(int32_t nq, int32_t n_value,
                                                int32_t heads, int32_t levels,
                                                int32_t points);
int fbbev_msda_fused_bwd_det(const float* value, const int64_t* spatial_shapes,
                             const int64_t* level_start, const float* ref,
                             const float* offsets, const float* logits,
                             const float* grad_out, int32_t bs,
                             int32_t n_value, int32_t heads, int32_t ch,
                             int32_t levels, int32_t nq, int32_t points,
                             float* grad_value, float* grad_offsets,
                             float* grad_logits, void* workspace,
                             size_t workspace_bytes, fbbev_stream_t stream);
size_t fbbev_da_sca_bwd_det_workspace_bytes(int32_t n_cams, int32_t nq,
                                            int32_t n_value, int32_t heads,
                                            int32_t ch, int32_t levels,
                                            int32_t points, int32_t Z,
                                            int32_t DC);
int fbbev_da_sca_bwd_det(const float* value, const float* depth_prob,
                         const float* ref_cam, const float* ref_depth,
                         const uint8_t* mask, const float* offsets,
                         const float* logits, const int64_t* spatial_shapes,
                         const int64_t* level_start, const float* dbound_host,
                         const float* grad_out, int32_t bs, int32_t n_cams,
                         int32_t nq, int32_t n_value, int32_t heads,
                         int32_t ch, int32_t levels, int32_t points, int32_t Z,
                         int32_t DC, float* grad_value, float* grad_depth_prob,
                         float* grad_offsets, float* grad_logits,
                         void* workspace, size_t workspace_bytes,
                         fbbev_stream_t stream);
size_t fbbev_msda_bwd_det_workspace_bytes(int32_t nq, int32_t n_value,
                                          int32_t heads, int32_t levels,
                                          int32_t points);
int fbbev_msda_bwd_det(const float* value, const int64_t* spatial_shapes,
                       const int64_t* level_start, const float* loc,
                       const float* attw, const float* grad_out, int32_t bs,
                       int32_t n_value, int32_t heads, int32_t ch,
                       int32_t levels, int32_t nq, int32_t points,
                       float* grad_value, float* grad_loc, float* grad_attw,
                       void* workspace, size_t workspace_bytes,
                       fbbev_stream_t stream);

/*
 * `per_cam_mask_list & bev_mask[None, :, :, None]` with the reference's
 * empty-camera rule (spatial_cross_attention_depth.py:156-169, 213-214) as a
 * device-side pass, so a bev_mask no longer forces the per-camera nonzero() /
 * re-batching loops (6*bs host synchronisations per layer in the reference).
 * mask (n_cams, bs, nq, Z) uint8/bool; bev_mask (bs, nq) uint8/bool; mask_out
 * (n_cams, bs, nq, Z) uint8 in the encoding fbbev_da_sca_fwd documents:
 * 1 where mask & bev_mask; for a (sample, camera) pair that sees no query under
 * the masked list, the anchors of the FIRST query it sees at all get 2.
 */
size_t fbbev_bev_mask_fold_workspace_bytes(int32_t bs, int32_t n_cams);
int fbbev_bev_mask_fold(const uint8_t* mask, const uint8_t* bev_mask,
                        int32_t bs, int32_t n_cams, int32_t nq, int32_t Z,
                        uint8_t* mask_out, void* workspace,
                        size_t workspace_bytes, fbbev_stream_t stream);

/* ---- row-wise Linear (+ bias, ReLU, residual, LayerNorm) on wgmma -----------
 * Replaces the nn.Linear / LayerNorm / residual chain of the reference's
 * encoder layer for the backward projection: sampling_offsets,
 * attention_weights, value_proj, output_proj
 * (spatial_cross_attention_depth.py:420-427, 226-233; mmcv
 * MultiScaleDeformableAttention), mmcv FFN and the `norm` entries of
 * operation_order (bevformer_encoder.py:251-377), which the reference runs as
 * cuBLAS fp32 GEMMs plus separate elementwise kernels.
 *
 *   y = LN( act( x . W^T + bias ) + residual )
 *
 * x (m, k) fp32 with row stride ldx floats, W (n, k) as in nn.Linear.weight,
 * y (m, n) with row stride ldy (a column block of a wider output is allowed);
 * bias / residual (m, n; row stride ldr) / ln_weight+ln_bias (n) are optional
 * (NULL), relu != 0
 * applies ReLU before the residual.  fp32 in and out; products are formed as
 * 3xTF32 on the tensor cores (error ~1e-6 relative, inside the 1e-4 bar; plain
 * TF32 is not).  Weights are packed once (hi / lo split in the shared-memory
 * layout of the kernel) with fbbev_linear_pack into fbbev_linear_packed_bytes
 * bytes; k % 4 == 0, n % 4 == 0, n <= 192 (split wider layers over n), n <= 80
 * with the LayerNorm epilogue (whole rows stay in shared memory),
 * 16-byte aligned pointers; otherwise FBBEV_ERR_UNSUPPORTED /
 * FBBEV_ERR_INVALID_ARGUMENT.
 */
size_t fbbev_linear_packed_bytes(int32_t n, int32_t k);
int fbbev_linear_pack(const float* weight, int32_t n, int32_t k, float* packed,
                      fbbev_stream_t stream);
int fbbev_linear_fwd(const float* x, int64_t ldx, const float* packed,
                     const float* bias, const float* residual, int64_t ldr,
                     const float* ln_weight, const float* ln_bias, int64_t m,
                     int32_t k, int32_t n, int32_t relu, float ln_eps, float* y,
                     int64_t ldy, fbbev_stream_t stream);

/* Two Linears that read the same x as ONE launch: `packed` / `bias` hold the
 * row-concatenated weight (n = n0 + n1 rows, n <= 192) and bias; output columns
 * [0, n_split) go to y0 (row stride ldy0), [n_split, n) to y1 (ldy1), each dense.
 * This is sampling_offsets + attention_weights of both attention modules
 * (spatial_cross_attention_depth.py:420-424, 533-540): they act on the same
 * query and feed one sampling kernel.  No residual / LayerNorm here.
 * x_add (may be NULL; row stride ldx_add): the GEMM input is x + x_add, formed
 * in the loader with one fp32 add per element -- `query = query + query_pos`
 * of both attention modules (spatial_cross_attention_depth.py:117-118, mmcv
 * MultiScaleDeformableAttention.forward) without a separate pass. */
int fbbev_linear_fwd_split(const float* x, int64_t ldx, const float* x_add,
                           int64_t ldx_add, const float* packed,
                           const float* bias, int64_t m, int32_t k, int32_t n,
                           int32_t n_split, int32_t relu, float* y0,
                           int64_t ldy0, float* y1, int64_t ldy1,
                           fbbev_stream_t stream);

/*
 * The encoder layer's FFN and the LayerNorm after it as ONE kernel:
 *     y = LN( residual + W2 . relu(W1 . x + b1) + b2 )
 * mmcv `FFN` (two Linears, ReLU, identity add; fbocc-r50 config ffn_cfgs) and
 * the following `norm` of operation_order (bevformer_encoder.py:251-377).  The
 * hidden activation (m x hidden) lives in registers / shared memory only.
 * w1_packed: hidden / 80 consecutive blocks, block c = fbbev_linear_pack of
 *   rows [80 c, 80 c + 80) of W1 (hidden, embed) -- i.e. fbbev_linear_pack(n = 80,
 *   k = embed) per block, fbbev_linear_packed_bytes(80, embed) bytes each;
 * w2_packed: fbbev_linear_pack(W2 (embed, hidden)).
 * b1 (hidden), b2 (embed), residual (m, embed; row stride ldr), ln_weight /
 * ln_bias (embed) may be NULL.  embed <= 80, embed % 4 == 0, hidden % 80 == 0,
 * hidden <= 320 (fbbev_ffn_supported); FBBEV_ERR_UNSUPPORTED otherwise (use
 * fbbev_linear_fwd per Linear).  Numerics as fbbev_linear_fwd (3xTF32).
 */
int fbbev_ffn_supported(int32_t embed, int32_t hidden);
int fbbev_ffn_fwd(const float* x, int64_t ldx, const float* w1_packed,
                  const float* b1, const float* w2_packed, const float* b2,
                  const float* residual, int64_t ldr, const float* ln_weight,
                  const float* ln_bias, int64_t m, int32_t embed,
                  int32_t hidden, float ln_eps, float* y, int64_t ldy,
                  fbbev_stream_t stream);

/* ---- training of the encoder layer's fused ops -------------------------------
 * Replaces, under autograd, the torch LayerNorm after output_proj and the
 * FFN's two Linears + ReLU + identity add + LayerNorm
 * (bevformer_encoder.py:251-377 operation_order; mmcv FFN), which the
 * reference trains as nn.Linear / nn.LayerNorm with the hidden activation and
 * the LayerNorm input in memory.
 *
 * fbbev_linear_fwd_ln_train: fbbev_linear_fwd with a LayerNorm (ln_weight /
 * ln_bias required, no ReLU, n <= 80) that also writes what the backward needs:
 * xhat (m, n; dense) = the normalised row exactly as the epilogue multiplies it
 * by ln_weight, and rstd (m) = 1 / sqrt(var + eps).  y is bit-identical to
 * fbbev_linear_fwd on the same inputs.
 *
 * fbbev_ffn_fwd_train: fbbev_ffn_fwd that also writes act (m, hidden; dense)
 * = relu(x . W1^T + b1) as the kernel holds it in fp32, and, with the
 * LayerNorm, xhat (m, embed; dense) and rstd (m) as above.  y is
 * bit-identical to fbbev_ffn_fwd.
 *
 * fbbev_ffn_bwd: the FFN's data-path backward in one kernel (the forward's
 * structure with the weights transposed and swapped):
 *     dh = (dz . W2) * [act > 0]      (written: dW1 = dh^T x needs it)
 *     dx = dh . W1 (+ dz when add_dz: the identity is the FFN's own input)
 * w2t_packed: W2^T (hidden, embed) packed as w1_packed of fbbev_ffn_fwd
 * (hidden / 80 blocks of fbbev_linear_pack(80, embed)); w1t_packed:
 * fbbev_linear_pack of W1^T (embed, hidden).  dz (m, embed; row stride lddz),
 * act (m, hidden; dense) from fbbev_ffn_fwd_train, dh (m, hidden; dense),
 * dx (m, embed; row stride lddx).  Shapes as fbbev_ffn_supported.  The weight
 * and bias gradients are left to the caller's GEMMs.
 *
 * fbbev_layernorm_bwd: for rows of n <= 80, from the upstream gradient g
 * (row stride ldg), xhat and rstd of the training forwards and gamma (n):
 *     dz = rstd (gamma g - mean(gamma g) - xhat mean(gamma g xhat))
 *     dgamma = sum_rows g xhat       dbeta = sum_rows g
 * dz has row stride lddz.  The column sums are per-CTA partials in
 * `workspace` (fbbev_layernorm_bwd_workspace_bytes(m, n) bytes) added in a
 * fixed order: no float atomics, the result is reproducible bit for bit.
 *
 * All four check their arguments before anything is enqueued; 16-byte aligned
 * pointers (xhat, act, dh included).
 */
int fbbev_linear_fwd_ln_train(const float* x, int64_t ldx, const float* packed,
                              const float* bias, const float* residual,
                              int64_t ldr, const float* ln_weight,
                              const float* ln_bias, int64_t m, int32_t k,
                              int32_t n, float ln_eps, float* y, int64_t ldy,
                              float* xhat, float* rstd, fbbev_stream_t stream);
int fbbev_ffn_fwd_train(const float* x, int64_t ldx, const float* w1_packed,
                        const float* b1, const float* w2_packed, const float* b2,
                        const float* residual, int64_t ldr,
                        const float* ln_weight, const float* ln_bias, int64_t m,
                        int32_t embed, int32_t hidden, float ln_eps, float* y,
                        int64_t ldy, float* act, float* xhat, float* rstd,
                        fbbev_stream_t stream);
int fbbev_ffn_bwd(const float* dz, int64_t lddz, const float* act,
                  const float* w2t_packed, const float* w1t_packed,
                  int32_t add_dz, int64_t m, int32_t embed, int32_t hidden,
                  float* dh, float* dx, int64_t lddx, fbbev_stream_t stream);
size_t fbbev_layernorm_bwd_workspace_bytes(int64_t m, int32_t n);
int fbbev_layernorm_bwd(const float* g, int64_t ldg, const float* xhat,
                        const float* rstd, const float* gamma, int64_t m,
                        int32_t n, float* dz, int64_t lddz, float* dgamma,
                        float* dbeta, void* workspace, size_t workspace_bytes,
                        fbbev_stream_t stream);

/* =====================================================================
 * T -- temporal fusion of the BEV / voxel history (the stage after the path)
 * ===================================================================== */

/*
 * The sampling half of `FBOCC.fuse_history`
 *   mmdet3d/models/fbbev/detectors/fbocc.py:207-319, `generate_grid` :170-205:
 *   grid = rt_flow @ (x, y, z, 1); normalise; F.grid_sample(history, grid,
 *   align_corners=True, bilinear, zeros); torch.cat([curr_bev, sampled], 1)
 * as one pass.  history (n, mc, Z, H, W) fp32 = the T previous frames stacked
 * along channels, samples history_batch_stride floats apart (>= mc*Z*H*W: the
 * history may be a channel slice of the previous step's concatenation buffer); flow (n, 4, 4) row-major = inverse(feat2bev) @ history_augs @
 * curr_to_prev_ego_rt @ inverse(forward_augs) @ feat2bev (:196-197), mapping
 * voxel indices (x, y, z, 1) of the current frame to voxel indices of the
 * history; out (n, c_total, Z, H, W): the warped history is written into
 * channels [ch_offset, ch_offset + mc) -- pass the concatenation buffer and
 * ch_offset = C so that no torch.cat copy is needed.  The 5-D grid tensor is
 * never materialised.
 */
int fbbev_history_warp(const float* history, int64_t history_batch_stride,
                       const float* flow, int32_t n, int32_t mc, int32_t Z,
                       int32_t H, int32_t W, float* out, int32_t c_total,
                       int32_t ch_offset, fbbev_stream_t stream);

/*
 * The adjoint (input gradient) of fbbev_history_warp, summed over frames that
 * share one flow:
 *   grad_src[b] (+)= warp_b^T ( sum_{f < frames} grad[b, f] )
 * for every sample b whose mask byte is set.  This is the gradient the
 * reference's restart write (fbocc.py:255) sends from the T warped copies of a
 * restarting sample back to its current frame.
 * grad: frame f of sample b is the (c, Z, H, W) dense block at grad + b
 *   grad_batch_stride + f grad_frame_stride (floats; the frame stride is
 *   ignored for frames == 1); flow (n, 4, 4) as for fbbev_history_warp;
 * mask [n] bytes in HOST memory, or NULL for every sample; other samples of
 *   grad_src are not touched;
 * grad_src (n, c, Z, H, W) dense: overwritten (accumulate == 0) or added to.
 * The exact transpose of the fp32 forward: the same corner offsets and
 * weights; a corner outside the volume adds nothing.  Frames are summed first,
 * in f order from +0.  Deterministic: every output element is written once,
 * as a sum in an order fixed by the sample's own flow (not by the grid, n or
 * the other samples); no float atomics.  Any finite flow, singular ones
 * included.  Enqueues a few kernels per masked sample, never synchronises.
 * workspace: fbbev_history_warp_bwd_workspace_bytes(c, Z, H, W, frames)
 * bytes, 16-byte aligned (0: invalid shape).  Z*H*W < 2^28, else
 * FBBEV_ERR_UNSUPPORTED.
 */
size_t fbbev_history_warp_bwd_workspace_bytes(int32_t c, int32_t Z, int32_t H,
                                              int32_t W, int32_t frames);
int fbbev_history_warp_bwd(const float* grad, int64_t grad_batch_stride,
                           int64_t grad_frame_stride, int32_t frames,
                           const uint8_t* mask, const float* flow, int32_t n,
                           int32_t c, int32_t Z, int32_t H, int32_t W,
                           float* grad_src, int32_t accumulate,
                           void* workspace, size_t workspace_bytes,
                           fbbev_stream_t stream);

/*
 * The whole data path of `FBOCC.fuse_history` after its state update, for
 * inference (BN in eval mode, no autograd), as ONE kernel:
 *   mmdet3d/models/fbbev/detectors/fbocc.py:263-317: grid_sample of the
 *   history, torch.cat with the current frame and the sweep-time channel,
 *   history_keyframe_time_conv (Conv3d 1x1x1 (C+1) -> C, BN, ReLU) over the
 *   T + 1 frames, history_keyframe_cat_conv (Conv3d 1x1x1 (T+1) C -> C_out,
 *   BN, ReLU), permute().clone().
 * curr (n, c, Z, H, W) fp32, samples curr_batch_stride floats apart;
 * history (n, T c, Z, H, W), history_batch_stride floats apart, or NULL when
 *   there is none yet (every sample is then fresh);
 * fresh [n] (1 byte each): sample b has no history of its own (first call or
 *   start_of_sequence): its T history frames are read as copies of curr[b];
 * flow (n, 4, 4) as for fbbev_history_warp; sweep (n, T + 1) the frames'
 *   sweep times (frame 0 = current);
 * BN folded into the convs (W' = W g / sqrt(var + eps), b' = (b - mean) g /
 *   sqrt(var + eps) + beta), fp32:
 *   wt_packed    fbbev_linear_pack of Wt'[:, :c] zero-padded to 80 rows (k = c);
 *   wc_packed    for frame f = 0..T, then half h (output rows [80 h, 80 h + 80)
 *                zero-padded to 80 rows): fbbev_linear_pack(80, c) of
 *                Wc'[rows, f c : (f+1) c], fbbev_linear_packed_bytes(80, c) each,
 *                halves = 1 for c_out <= 80, else 2;
 *   wc_sum_packed the same for sum_{f>=1} Wc'_f (one frame);
 *   bias_t [c] = b_t'; time_w [c] = Wt'[:, c] (the sweep-time column);
 *   bias_c [c_out] = b_c'.
 * out (n, c_out, Z, H, W) dense.  next_history (n, next_channels, Z, H, W) or
 * NULL: channels [f c, (f+1) c) receive frame f's input for f = 0..T-1 (the
 * current frame, then the warped history), bit-identical to what
 * fbbev_history_warp writes; other channels are not touched.
 * Shapes: fbbev_history_fuse_supported(c, c_out) (c % 4 == 0, 4 <= c <= 80,
 * c_out % 4 == 0, 4 <= c_out <= 160), T >= 1, Z*H*W < 2^31, n <= 65535;
 * FBBEV_ERR_UNSUPPORTED otherwise.  Numerics: 3xTF32 (as fbbev_linear_fwd).
 */
int fbbev_history_fuse_supported(int32_t c, int32_t c_out);
int fbbev_history_fuse_fwd(const float* curr, int64_t curr_batch_stride,
                           const float* history, int64_t history_batch_stride,
                           const uint8_t* fresh, const float* flow,
                           const float* sweep, const float* wt_packed,
                           const float* wc_packed, const float* wc_sum_packed,
                           const float* bias_t, const float* time_w,
                           const float* bias_c, int32_t n, int32_t T, int32_t c,
                           int32_t c_out, int32_t Z, int32_t H, int32_t W,
                           float* out, float* next_history,
                           int32_t next_channels, fbbev_stream_t stream);

/* -- training route of FBOCC.fuse_history, every sample fresh ---------------
 * A call in which every sample is fresh (no history yet, or
 * start_of_sequence) has T history frames that are T copies of one warped
 * frame x1 with one sweep time.  Forward and backward of the time conv + BN +
 * ReLU and of the keyframe-mixing conv (before its BN) then need two frames:
 *   y_f = Wt[:, :c] x_f + Wt[:, c] time_f + bt  (time_0 = 0, time_1 = time[b]),
 *   h_f = relu(gamma (y_f - mean) invstd + beta),
 *   out = Wc_0 h_0 + Wbar h_1 + bc,  Wbar = sum_{f>=1} Wc_f.
 * x0, x1 (n, c, Z, H, W) fp32, dense inside a sample, samples *_batch_stride
 * floats apart; time [n] = freq * sweep time of the history frames.
 * Packed weights (fbbev_linear_pack images, 16-byte aligned):
 *   wt_packed   Wt[:, :c] zero-padded to 80 rows, k = c;
 *   wc_packed   Wc_0 then Wbar, each zero-padded to 80 rows (c_out <= 80) or
 *               160 rows, k = c;
 *   wct_packed  Wc_0^T then Wbar^T, each zero-padded to 80 rows, k = c_out;
 *   wtt_packed  Wt[:, :c]^T zero-padded to 80 rows, k = c.
 * train != 0: the time BN uses the batch statistics, with frame 1 counted T
 * times over N = n (T+1) Z H W values, and updates running_mean / running_var
 * as torch does (momentum, or 1 / *num_batches_tracked when momentum < 0; the
 * caller increments num_batches_tracked first; unbiased variance).  train == 0:
 * the running statistics.  save [160] receives mean[80] | invstd[80], the
 * statistics the backward needs.  out (n, c_out, Z, H, W) dense.
 * Backward from grad_out (n, c_out, Z, H, W) dense: h0, h1 (the recomputed
 * h_f) and e0, e1 (the gradients at the time conv's output, e1 summed over the
 * T history frames), each (n, c, Z, H, W) dense, for the weight gradients;
 * grad_curr (n, c, Z, H, W) dense or NULL; grad_gamma, grad_beta [c].
 * workspace: fbbev_history_train_workspace_bytes(n, c, Z, H, W) bytes,
 * 16-byte aligned, no other state.  Shapes as fbbev_history_fuse_supported.
 * Numerics: 3xTF32 products, fp64 channel sums reduced in a fixed order (no
 * float atomics: bitwise reproducible).
 */
size_t fbbev_history_train_workspace_bytes(int32_t n, int32_t c, int32_t Z,
                                           int32_t H, int32_t W);
int fbbev_history_train_fwd(
    const float* x0, int64_t x0_batch_stride, const float* x1,
    int64_t x1_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wc_packed,
    const float* bias_c, const float* gamma, const float* beta,
    float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps,
    int32_t train, int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z,
    int32_t H, int32_t W, float* out, float* save, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_bwd(
    const float* x0, int64_t x0_batch_stride, const float* x1,
    int64_t x1_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wct_packed,
    const float* wtt_packed, const float* gamma, const float* beta,
    const float* save, int32_t train, int32_t n, int32_t T, int32_t c,
    int32_t c_out, int32_t Z, int32_t H, int32_t W, const float* grad_out,
    float* h0, float* h1, float* e0, float* e1, float* grad_curr,
    float* grad_gamma, float* grad_beta, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream);

/* The same two passes with a train-mode time BN whose statistics span several
 * ranks (torch's SyncBatchNorm): each pass is split at its one statistics
 * step into a local half, which writes this rank's fp64 row, and a global
 * half, which takes every rank's row.  Between the halves the caller gathers
 * the rows of all ranks into rows [world][2 c + 1] (rank r's row at r (2 c +
 * 1)); the global half adds them on the device in rank order 0..world-1, so
 * every rank that passes the same rows gets bitwise the same mean, invstd and
 * running statistics.  Arguments are those of fbbev_history_train_fwd / _bwd
 * (train is implied).
 *   _fwd_local   row [2 c + 1] = [S1 | S2 | count]: S1[ch] = sum of y_0 + T
 *                sum of y_1 over this rank's voxels, S2 likewise of y^2,
 *                count = n (T+1) Z H W.
 *   _fwd_global  mean and biased variance from the summed rows over the
 *                summed count -> save; running statistics updated with the
 *                unbiased variance (N / (N - 1), N the global count); out.
 *   _bwd_local   h0, h1, e0, e1 (e_f = the masked d_f until _bwd_global),
 *                this rank's grad_gamma / grad_beta (rank-local, as torch
 *                returns them) and row [sum d | sum d xhat | count].
 *   _bwd_global  e0, e1 from the summed rows and the global count, then
 *                grad_curr (NULL: skipped).
 * Both halves of a pass take the same workspace of
 * fbbev_history_train_workspace_bytes(n, c, Z, H, W) bytes, and nothing may
 * use it between them (the backward keeps xhat_f there).  n = 0 is allowed:
 * the local halves write a zero row (and zero grad_gamma / grad_beta), the
 * global halves update only the statistics.  With world = 1 and rows = the
 * rank's own row, the staged pair computes bit for bit what the one-shot
 * entry point computes.  world < 1 or rows / row NULL:
 * FBBEV_ERR_INVALID_ARGUMENT, checked before anything else.
 */
int fbbev_history_train_fwd_local(
    const float* x0, int64_t x0_batch_stride, const float* x1,
    int64_t x1_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, int32_t n, int32_t T, int32_t c,
    int32_t Z, int32_t H, int32_t W, double* row, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_fwd_global(
    const float* x0, int64_t x0_batch_stride, const float* x1,
    int64_t x1_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wc_packed,
    const float* bias_c, const float* gamma, const float* beta,
    float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps,
    const double* rows, int32_t world, int32_t n, int32_t T, int32_t c,
    int32_t c_out, int32_t Z, int32_t H, int32_t W, float* out, float* save,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_bwd_local(
    const float* x0, int64_t x0_batch_stride, const float* x1,
    int64_t x1_batch_stride, const float* time, const float* wt_packed,
    const float* bias_t, const float* time_w, const float* wct_packed,
    const float* gamma, const float* beta, const float* save, int32_t n,
    int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
    const float* grad_out, float* h0, float* h1, float* e0, float* e1,
    float* grad_gamma, float* grad_beta, double* row, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_bwd_global(
    const float* wtt_packed, const float* gamma, const float* save,
    const double* rows, int32_t world, int32_t n, int32_t T, int32_t c,
    int32_t Z, int32_t H, int32_t W, float* e0, float* e1, float* grad_curr,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream);

/* -- training route of FBOCC.fuse_history, every sample's T + 1 frames --------
 * The same data path for any sample, fresh or carrying history, over all F =
 * T + 1 frames as the caller materialised them:
 *   y_f = Wt[:, :c] x_f + Wt[:, c] time[b, f] + bt,   f = 0..T,
 *   h_f = relu(gamma (y_f - mean) invstd + beta),  out = sum_f Wc_f h_f + bc,
 * every frame counted once in the batch statistics (N = n F Z H W).
 * x (n, F c, Z, H, W) fp32: frame f is the channel slice [f c, (f+1) c), dense
 * inside a sample, samples x_batch_stride floats apart (the concatenation
 * buffer of the history warp); time (n, F) dense = freq * sweep times.
 * Packed weights (fbbev_linear_pack images, 16-byte aligned):
 *   wt_packed   as the two-frame route;
 *   wc_packed   Wc_0 .. Wc_T, each zero-padded to 80 rows (c_out <= 80) or
 *               160 rows, k = c;
 *   wct_packed  Wc_0^T .. Wc_T^T, each zero-padded to 80 rows, k = c_out;
 *   wtt_packed  as the two-frame route.
 * train, the statistics, save, out: as fbbev_history_train_fwd.
 * The backward is two calls on one workspace, with nothing else using it in
 * between: _bwd_hidden writes h (n, F c, Z, H, W) dense, the recomputed h_f
 * the caller needs for dWc = sum g h^T, and keeps xhat_f in the workspace;
 * _bwd (or the staged _bwd_local / _bwd_global) then writes e (n, F c, Z, H,
 * W) dense, the gradient at the time conv's output of every frame (e may be
 * the h buffer: it is not read), grad_curr = Wt[:, :c]^T e_0 (NULL: skipped),
 * grad_gamma and grad_beta.  The staged halves follow the two-frame route's
 * rules, with rows in the same [S1 | S2 | count] / [sum d | sum d xhat |
 * count] format, so ranks on either route gather into one call.
 * workspace: fbbev_history_train_full_workspace_bytes(n, T, c, Z, H, W)
 * bytes, 16-byte aligned.  Shapes as fbbev_history_fuse_supported, T < 65535.
 */
size_t fbbev_history_train_full_workspace_bytes(int32_t n, int32_t T, int32_t c,
                                                int32_t Z, int32_t H, int32_t W);
int fbbev_history_train_full_fwd(
    const float* x, int64_t x_batch_stride, const float* time,
    const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wc_packed, const float* bias_c, const float* gamma,
    const float* beta, float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps,
    int32_t train, int32_t n, int32_t T, int32_t c, int32_t c_out, int32_t Z,
    int32_t H, int32_t W, float* out, float* save, void* workspace,
    size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_full_fwd_local(
    const float* x, int64_t x_batch_stride, const float* time,
    const float* wt_packed, const float* bias_t, const float* time_w,
    int32_t n, int32_t T, int32_t c, int32_t Z, int32_t H, int32_t W,
    double* row, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream);
int fbbev_history_train_full_fwd_global(
    const float* x, int64_t x_batch_stride, const float* time,
    const float* wt_packed, const float* bias_t, const float* time_w,
    const float* wc_packed, const float* bias_c, const float* gamma,
    const float* beta, float* running_mean, float* running_var,
    const int64_t* num_batches_tracked, double momentum, double eps,
    const double* rows, int32_t world, int32_t n, int32_t T, int32_t c,
    int32_t c_out, int32_t Z, int32_t H, int32_t W, float* out, float* save,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_full_bwd_hidden(
    const float* x, int64_t x_batch_stride, const float* time,
    const float* wt_packed, const float* bias_t, const float* time_w,
    const float* gamma, const float* beta, const float* save, int32_t n,
    int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
    float* h, void* workspace, size_t workspace_bytes, fbbev_stream_t stream);
int fbbev_history_train_full_bwd(
    const float* wct_packed, const float* wtt_packed, const float* gamma,
    const float* beta, const float* save, int32_t train, int32_t n, int32_t T,
    int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
    const float* grad_out, float* e, float* grad_curr, float* grad_gamma,
    float* grad_beta, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream);
int fbbev_history_train_full_bwd_local(
    const float* wct_packed, const float* gamma, const float* beta, int32_t n,
    int32_t T, int32_t c, int32_t c_out, int32_t Z, int32_t H, int32_t W,
    const float* grad_out, float* e, float* grad_gamma, float* grad_beta,
    double* row, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream);
int fbbev_history_train_full_bwd_global(
    const float* wtt_packed, const float* gamma, const float* save,
    const double* rows, int32_t world, int32_t n, int32_t T, int32_t c,
    int32_t Z, int32_t H, int32_t W, float* e, float* grad_curr,
    void* workspace, size_t workspace_bytes, fbbev_stream_t stream);

/* -- the restart term of both kernel routes ----------------------------------
 * The reference's restart write (fbocc.py:255) makes a restarting sample's T
 * history frames warped copies of its grad-carrying current frame, so its d
 * curr gains
 *   grad_curr[b] += Wt[:, :c]^T warp_b^T ( sum_{f < frames} e[b, f] )
 * for every sample b whose mask byte is set (the warp acts per channel, Wt
 * per voxel: the two commute).  e: the gradients at the time conv's output of
 * the history frames, as the backward wrote them: the two-frame route's e1
 * (frames = 1: it already sums the T copies), or frames 1..T of the full
 * route's e (e + c Z H W, frame stride c Z H W, batch stride (T+1) c Z H W).
 * Frame layout, flow and mask (HOST bytes, not NULL) as fbbev_history_warp_bwd;
 * wtt_packed as fbbev_history_train_bwd; grad_curr (n, c, Z, H, W) dense, the
 * backward's d curr, added to (other samples not touched).  Deterministic as
 * fbbev_history_warp_bwd; the product is the routes' 3xTF32 kernel.
 * workspace: fbbev_history_restart_grad_workspace_bytes(c, Z, H, W, frames)
 * bytes, 16-byte aligned.  Shapes: c as fbbev_history_fuse_supported(c, c),
 * Z*H*W < 2^28.
 */
size_t fbbev_history_restart_grad_workspace_bytes(int32_t c, int32_t Z,
                                                  int32_t H, int32_t W,
                                                  int32_t frames);
int fbbev_history_restart_grad_curr(
    const float* e, int64_t e_batch_stride, int64_t e_frame_stride,
    int32_t frames, const uint8_t* mask, const float* flow,
    const float* wtt_packed, int32_t n, int32_t c, int32_t Z, int32_t H,
    int32_t W, float* grad_curr, void* workspace, size_t workspace_bytes,
    fbbev_stream_t stream);

/* =====================================================================
 * D -- depth supervision of the lift step (the training loss on `depth`)
 * ===================================================================== */

/*
 * Replaces get_downsampled_gt_depth + get_depth_loss of CM_DepthNet
 *   mmdet3d/models/fbbev/modules/depth_net.py:396-450
 * and of LSSViewTransformerBEVDepth
 *   mmdet3d/models/necks/view_transformer.py:1036-1081
 * (sid = False) with no host synchronisation.
 * gt (bn, H, W) fp32 dense; preds (bn, d, h, w) fp32 dense, h = H / ds,
 * w = W / ds (CM's (B, N, D, h, w) is the same memory).
 *   m     = min over the ds x ds patch of (g == 0 ? 1e5 : g), NaN propagating
 *   t     = (m - c0) * (1 / c1)     fp32, as torch's CUDA division by a scalar
 *   label = (0 <= t < d + 1) ? trunc(t) : 0             class in [0, d]
 * with c0 = (float)(lo - step) (difference in double), c1 = (float)step of
 * grid_config['depth'] = [lo, hi, step].  Pixels with label >= 1 are
 * foreground, one-hot at bin label - 1.
 *   loss = weight * (S / max(1, n_fg)),  S = sum over foreground pixels and
 *   all d bins of torch's binary_cross_entropy element (logs clamped at -100)
 * Outputs: labels (bn, h, w) int32 -- the only per-pixel state the backward
 * needs; loss (0-d fp32) and n_fg (0-d int32) on the device.  The sum is
 * deterministic (per-row partials in the workspace, added in a fixed order;
 * no float atomics).
 * preds == NULL computes labels only (loss, n_fg and the workspace unused,
 * loss and n_fg must be NULL).
 * workspace: fbbev_depth_loss_workspace_bytes(bn, H, ds) bytes, 16-byte
 * aligned.  Errors: H or W not a multiple of ds, d <= 0, NULL or misaligned
 * pointers.  bn == 0 is a no-op.  W <= 12288 (else FBBEV_ERR_UNSUPPORTED).
 */
size_t fbbev_depth_loss_workspace_bytes(int32_t bn, int32_t H, int32_t ds);
int fbbev_depth_loss_fwd(const float* gt, const float* preds, int32_t bn,
                         int32_t H, int32_t W, int32_t ds, int32_t d, float c0,
                         float c1, float weight, int32_t* labels, float* loss,
                         int32_t* n_fg, void* workspace,
                         size_t workspace_bytes, fbbev_stream_t stream);
/*
 * d preds of fbbev_depth_loss_fwd's loss, dense (bn, d, h, w), 0 at
 * background pixels; grad_loss: device fp32 scalar (the upstream gradient),
 * n_fg as the forward wrote it.  In the reference's autograd order:
 *   k = (grad_loss * weight) / max(1, n_fg)
 *   grad_preds = k * (p - y) / max((1 - p) * p, 1e-12)
 * each an IEEE fp32 operation.  bn == 0 is a no-op.
 */
int fbbev_depth_loss_bwd(const int32_t* labels, const float* preds,
                         const int32_t* n_fg, const float* grad_loss,
                         int32_t bn, int32_t h, int32_t w, int32_t d,
                         float weight, float* grad_preds,
                         fbbev_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* FBBEV_B200_H_ */
