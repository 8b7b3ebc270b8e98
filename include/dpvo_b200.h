/*
 * dpvo_b200.h -- C-ABI of the H100-native DPVO update hot path.
 *
 * Every entry point takes plain device pointers, sizes/strides and a CUDA stream and
 * returns an int status (DPVO_OK == 0).  No torch types cross this boundary.  The three
 * torch-extension shims (cuda_corr / cuda_ba / lietorch_backends, see dpvo_b200/csrc/shim.cpp)
 * adapt torch::Tensor -> these calls and keep the reference's pybind names and signatures.
 *
 * Reference interfaces replaced (paths relative to the princeton-vl/DPVO tree):
 *   cuda_corr          dpvo/altcorr/correlation.cpp:57-62, correlation_kernel.cu:193-333
 *   cuda_ba            dpvo/fastba/ba.cpp:183-188, ba_cuda.cu:433-617
 *   lietorch_backends  dpvo/lietorch/src/lietorch.cpp:286-316, lietorch_gpu.cu:298-601
 *   Update operator    dpvo/net.py:27-92, dpvo/blocks.py:15-48 (pieces: LayerNorm, SoftAgg, GEMMs)
 *
 * All pointers are DEVICE pointers unless stated otherwise.  `stream` is a cudaStream_t
 * passed as void* (NULL = legacy default stream).  Kernels are compiled for sm_90a only;
 * there is no CPU fallback: a call on a machine without a usable device returns DPVO_ERR_CUDA.
 */
#ifndef DPVO_B200_H
#define DPVO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ------------------------------------------------------------------- */
#define DPVO_OK               0
#define DPVO_ERR_INVALID      1   /* bad argument (null pointer, negative size, bad dtype) */
#define DPVO_ERR_UNSUPPORTED  2   /* valid request outside what this build implements      */
#define DPVO_ERR_CUDA         3   /* CUDA runtime error; see dpvo_last_error()             */
#define DPVO_ERR_WORKSPACE    4   /* workspace too small                                   */

/* ---- element types (match at::ScalarType semantics, not values) --------------------- */
#define DPVO_F16  0
#define DPVO_F32  1
#define DPVO_F64  2
#define DPVO_BF16 3

/* ---- Lie group ids: lietorch/include/dispatch.h:12-32 -------------------------------- */
#define DPVO_SO3   1
#define DPVO_RXSO3 2
#define DPVO_SE3   3
#define DPVO_SIM3  4

const char* dpvo_version(void);
/* Thread-local text of the last non-OK status produced by this library. */
const char* dpvo_last_error(void);
/* Number of kernel launches issued by this library since process start (all entry points). */
int64_t dpvo_launch_count(void);

/* ======================================================================================
 * cuda_corr  (altcorr)
 * ====================================================================================== */

/*
 * cuda_corr.forward -- correlation_kernel.cu:193-233 (kernel :82-136 + bilinear blend :221-230
 * + permute :232), fused into one launch.
 *
 *   fmap1   logical [B, S1, C, P, P]   patch features, indexed by ii[m]   (gmap)
 *   fmap2   logical [B, S2, C, H2, W2] frame features, indexed by jj[m]   (pyramid level)
 *   coords  contiguous fp32 [B, M, 2, P, P]   (x, y) per patch pixel
 *   ii, jj  int64 [M]
 *   out     logical [B, M, 2R+1 (x offset), 2R+1 (y offset), P, P], element (b,m,xo,yo,i,j)
 *           stored at out[((((b*M+m)*(2R+1)+xo)*(2R+1)+yo)*P+i)*P+j) * out_elem_stride].
 *           out_elem_stride = 1 gives the reference's (contiguous) result; 2 lets two pyramid
 *           levels interleave into the [B, M, 882] layout DPVO.corr builds with torch.stack
 *           (dpvo/dpvo.py:207).
 *   fmapX_strides: element strides of the 5 logical dims (any layout; channels-last, i.e.
 *           stride[2] == 1, is the fast path for fp16).
 *   dtype   element type of fmap1, fmap2 and out (F16 / F32 / F64 / BF16).
 * Out-of-image taps contribute exactly 0 (correlation_kernel.cu:121-122).  Accumulation is
 * fp32 (fp64 for F64) -- the reference accumulates in the input type (:121).
 */
int dpvo_corr_forward(const void* fmap1, const int64_t* fmap1_strides,
                      const void* fmap2, const int64_t* fmap2_strides,
                      const float* coords, const int64_t* ii, const int64_t* jj,
                      void* out, int64_t out_elem_stride,
                      int dtype, int B, int M, int C, int P,
                      int S1, int S2, int H2, int W2, int radius, void* stream);

/*
 * Two-level fused form of DPVO.corr (dpvo/dpvo.py:200-207): level 0 samples fmap2_l0 at coords,
 * level 1 samples fmap2_l1 at coords / lvl1_div (4 in DPVO), result written as
 * out[B, M, 2R+1, 2R+1, P, P, 2] (level innermost) == torch.stack([c0, c1], -1).  Consecutive
 * (b, m) rows are out_row_stride elements apart (>= 2*(2R+1)^2*P^2, even; 896 pads the 882 features of
 * DPVO to the k-block of the first dense layer -- padding columns are not written).
 */
int dpvo_corr_forward_pyramid2(const void* fmap1, const int64_t* fmap1_strides,
                               const void* fmap2_l0, const int64_t* l0_strides, int H0, int W0,
                               const void* fmap2_l1, const int64_t* l1_strides, int H1, int W1,
                               float lvl1_div,
                               const float* coords, const int64_t* ii, const int64_t* jj,
                               void* out, int64_t out_row_stride,
                               int dtype, int B, int M, int C, int P,
                               int S1, int S2, int radius,
                               void* workspace, int64_t workspace_bytes, void* stream);
/* Scratch for the binned path of dpvo_corr_forward_pyramid2 (per-bin counters and edge lists of the level-1
 * regions and the level-0 wgmma/TMA kernel, and the list of edges whose nine tap windows fit no box, finished by the
 * mma.sync kernel).  workspace may be NULL: the call then runs the mma.sync kernel for every edge.  S1 / S2 are the
 * slot counts of the patch-feature and frame-feature rings (extents of the TMA tensor maps and of the bins). */
int64_t dpvo_corr_pyramid2_workspace_bytes(int64_t M);

/*
 * cuda_corr.backward -- correlation_kernel.cu:236-286 (bilinear-transpose :252-269 + kernel
 * :139-190) fused.  grad is logical [B, M, 2R+1(x), 2R+1(y), P, P], contiguous, element type
 * grad_dtype (fp32, or the feature dtype).  fmap1_grad / fmap2_grad are shaped like fmap1 /
 * fmap2 with the given element strides (torch::zeros_like keeps the input layout) and MUST be
 * zero-filled by the caller; gradients are accumulated with atomics as in the reference, but
 * one atomic per touched (pixel, channel) instead of one per tap.  No gradient w.r.t. coords.
 */
int dpvo_corr_backward(const void* fmap1, const int64_t* fmap1_strides,
                       const void* fmap2, const int64_t* fmap2_strides,
                       const float* coords, const int64_t* ii, const int64_t* jj,
                       const void* grad, int grad_dtype,
                       void* fmap1_grad, const int64_t* fmap1_grad_strides,
                       void* fmap2_grad, const int64_t* fmap2_grad_strides,
                       int dtype, int B, int M, int C, int P,
                       int S1, int S2, int H2, int W2, int radius, void* stream);

/*
 * cuda_corr.patchify_forward -- correlation_kernel.cu:288-307 (kernel :16-47).
 *   net [B, C, H, W] (strided), coords fp32 [B, M, 2] contiguous,
 *   patches [B, M, C, D, D] contiguous with D = 2R+2, zero where the window leaves the map.
 * The whole output is written (no pre-zeroing needed).
 */
int dpvo_patchify_forward(const void* net, const int64_t* net_strides, const float* coords,
                          void* patches, int dtype, int B, int M, int C, int H, int W,
                          int radius, void* stream);

/*
 * cuda_corr.patchify_backward -- correlation_kernel.cu:310-333 (kernel :49-80).
 *   gradient [B, M, C, D, D] contiguous; net_grad [B, C, H, W] contiguous, zero-filled by caller.
 */
int dpvo_patchify_backward(const void* gradient, const float* coords, void* net_grad,
                           int dtype, int B, int M, int C, int H, int W, int radius,
                           void* stream);

/* ======================================================================================
 * patch-graph index structure (replaces torch::_unique + CPU stable_sort in ba.cpp:59-97,
 * torch.unique in blocks.py:41 and torch::_unique in ba_cuda.cu:447)
 * ====================================================================================== */

/*
 * Group E edges by the pair key (key_a[e], key_b[e]) (key_b may be NULL -> key_a alone); the
 * members of a group are ordered by (sec[e], e) (sec may be NULL -> ordered by e).  For
 * |key_b| < mul this is the same partition as the scalar key key_a*mul + key_b that
 * Update.forward builds (net.py:88: ii*12345 + jj).
 * Outputs (all device):
 *   order[E]          int32 edge ids sorted by (key_a, key_b, sec, e)
 *   group_of[E]       int32 dense group id of every edge; groups numbered by ascending key
 *   group_start[E+1]  int32 CSR offsets into order (entries [0..G] are written)
 *   group_key_a[E], group_key_b[E]  int64 keys of every group ([0..G-1] written; key_b may be NULL)
 *   n_groups[1]       int32 G
 * workspace: dpvo_group_workspace_bytes(E) bytes.  Deterministic: stable radix sort, integer
 * atomics only.
 */
int64_t dpvo_group_workspace_bytes(int64_t E);
int dpvo_group_edges(const int64_t* key_a, const int64_t* key_b, const int64_t* sec, int64_t E,
                     int32_t* order, int32_t* group_of, int32_t* group_start,
                     int64_t* group_key_a, int64_t* group_key_b, int32_t* n_groups,
                     void* workspace, int64_t workspace_bytes, void* stream);
/*
 * Two groupings of the same E edges in ONE cooperative launch (the kernel is bound by grid-barrier latency, so
 * the second problem costs nothing): what one update needs -- by patch (kk, NULL, jj) for fastba.neighbors
 * (ba.cpp:59-97) / agg_kk, and by frame pair (ii, jj, NULL) for agg_ij (net.py:87-88) and the BA pose blocks.
 * Arguments as dpvo_group_edges, suffixed 0 / 1; each problem has its own workspace of workspace_bytes_each.
 */
int dpvo_group_edges_pair(const int64_t* key_a0, const int64_t* key_b0, const int64_t* sec0,
                          int32_t* order0, int32_t* group_of0, int32_t* group_start0,
                          int64_t* group_key_a0, int64_t* group_key_b0, int32_t* n_groups0, void* workspace0,
                          const int64_t* key_a1, const int64_t* key_b1, const int64_t* sec1,
                          int32_t* order1, int32_t* group_of1, int32_t* group_start1,
                          int64_t* group_key_a1, int64_t* group_key_b1, int32_t* n_groups1, void* workspace1,
                          int64_t E, int64_t workspace_bytes_each, void* stream);

/*
 * neighbors from an existing grouping keyed by the edge's patch and ordered by target frame
 * (dpvo_group_edges(kk, NULL, jj, ...)): ix/jx = previous/next edge of the same group, -1 at ends.
 */
int dpvo_neighbors_from_groups(const int32_t* order, const int32_t* group_of, int64_t E,
                               int64_t* ix, int64_t* jx, void* stream);

/*
 * cuda_ba.neighbors -- ba.cpp:59-97.  For every edge e: ix[e] = the edge preceding e and
 * jx[e] = the edge following e among the edges with the same ii value, ordered by
 * (jj, original position) (std::stable_sort semantics); -1 at the ends.  int64 outputs.
 * workspace: dpvo_neighbors_workspace_bytes(E).
 */
int64_t dpvo_neighbors_workspace_bytes(int64_t E);
int dpvo_neighbors(const int64_t* ii, const int64_t* jj, int64_t E,
                   int64_t* ix, int64_t* jx,
                   void* workspace, int64_t workspace_bytes, void* stream);

/* ======================================================================================
 * cuda_ba  (fastba)
 * ====================================================================================== */

/*
 * cuda_ba.forward, eff_impl == false -- ba_cuda.cu:433-582.  `iterations` Gauss-Newton steps
 * over poses [t0, t1) and the inverse depth of every patch referenced by kk, IN PLACE.
 *   poses      fp32 [n_poses, 7]  (tx ty tz qx qy qz qw)
 *   patches    fp32 [n_patches, 3, P, P]
 *   intrinsics fp32 [>=1, 4]  (row 0 is used for every edge: ba_cuda.cu:253-259)
 *   target, weight fp32 [E, 2];  lmbda fp32 [1];  ii, jj, kk int64 [E]
 * Damping S += I*(1e-4*S + 1) (:560), Q = 1/(C + lmbda) (:519), retractions :157-229.
 * Requires t1 - t0 <= 32 (dense 6N x 6N system held on chip); t1 - t0 == 0 is the
 * structure-only branch (:521-531).  workspace: dpvo_ba_workspace_bytes(E, t1 - t0).
 */
int64_t dpvo_ba_workspace_bytes(int64_t E, int n_free_poses);
int dpvo_ba_forward(float* poses, float* patches, const float* intrinsics,
                    const float* target, const float* weight, const float* lmbda,
                    const int64_t* ii, const int64_t* jj, const int64_t* kk,
                    int64_t E, int64_t n_poses, int64_t n_patches, int P,
                    int t0, int t1, int iterations,
                    void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Same Gauss-Newton iterations on groupings the caller already holds (the update operator builds
 * exactly these two per update): kk grouping = dpvo_group_edges(kk, NULL, [jj]) -> k_order, k_start,
 * k_key (= sorted unique patch ids), k_n;  pair grouping = dpvo_group_edges(ii, jj, NULL) -> p_order,
 * p_start, p_key_i, p_key_j, p_n.  workspace: dpvo_ba_grouped_workspace_bytes(E, t1 - t0).
 */
int64_t dpvo_ba_grouped_workspace_bytes(int64_t E, int n_free_poses);
int dpvo_ba_forward_grouped(float* poses, float* patches, const float* intrinsics,
                            const float* target, const float* weight, const float* lmbda,
                            const int64_t* ii, const int64_t* jj, const int64_t* kk,
                            int64_t E, int P, int t0, int t1, int iterations,
                            const int32_t* k_order, const int32_t* k_start, const int64_t* k_key, const int32_t* k_n,
                            const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                            const int64_t* p_key_j, const int32_t* p_n,
                            void* workspace, int64_t workspace_bytes, void* stream);

/*
 * B independent sliding windows in one launch sequence (two launches per iteration for the whole batch).  Stream b owns
 * frames [b F, (b+1) F) and patches [b F M, (b+1) F M) of poses / patches / intrinsics (F = frames_per_stream,
 * M = patches_per_frame); its window is [t0[b], t1[b]) in global frame numbers (host arrays), and row b F of
 * intrinsics is its camera.  The groupings are the dpvo_ba_forward_grouped ones, built over the concatenation of the
 * streams' edges; each stream's group range is found on the device (no host synchronisation, graph-capturable).  No
 * edge may join two streams.  A stream with t1[b] == t0[b] or without edges is left untouched.  Every t1 - t0 <= 12
 * runs the fast path for the whole batch, otherwise the general path does; t1 - t0 > 32 is DPVO_ERR_UNSUPPORTED,
 * B > 64 too.  Each stream's result is that of dpvo_ba_forward_grouped on the stream alone, with one exception: a
 * stream with an empty window (t1[b] == t0[b]) keeps its depths, where dpvo_ba_forward_grouped runs its
 * structure-only (depth-only) step.
 * workspace: dpvo_ba_batched_workspace_bytes(E, B, max_b (t1[b] - t0[b])) on the current device.
 */
int64_t dpvo_ba_batched_workspace_bytes(int64_t E, int B, int max_free_poses);
int dpvo_ba_forward_batched(float* poses, float* patches, const float* intrinsics,
                            const float* target, const float* weight, const float* lmbda,
                            const int64_t* ii, const int64_t* jj, const int64_t* kk,
                            int64_t E, int P, int B, int frames_per_stream, int patches_per_frame,
                            const int* t0, const int* t1, int iterations,
                            const int32_t* k_order, const int32_t* k_start, const int64_t* k_key, const int32_t* k_n,
                            const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                            const int64_t* p_key_j, const int32_t* p_n,
                            void* workspace, int64_t workspace_bytes, void* stream);

/*
 * Wide windows / cuda_ba.forward(..., eff_impl=True) -- replaces dpvo/fastba/block_e.cu:38-299 (EfficentE) and
 * the eff_impl branch of ba_cuda.cu:495-563.  For any number of free poses N = t1 - t0: one call assembles
 *     S = B - E diag(Q) E^T + I o (1e-4 S + 1)   fp32 [6N, 6N]  and   y = v - E diag(Q) u   fp32 [6N]
 * (the block-sparse pose/depth coupling E is never materialised: one CTA per source frame forms its dense
 * product in shared memory); the caller solves S dX = y (dense Cholesky -- a library call, as in the reference,
 * ba_cuda.cu:547-549) and hands dX to dpvo_ba_wide_update, which back-substitutes the depths, retracts patches
 * and poses in place.  Requires the DPVO patch numbering kk = frame * PPF + slot (as block_e.cu does) and the
 * (ii, jj) pair grouping of dpvo_group_edges(ii, jj, NULL).  `status` is a zero-initialised device int:
 * after the stream has drained, 1 = a frame is observed from more frames than fit on chip, 2 = a patch id lies
 * outside its frame's slot range; the results are then invalid.
 */
int dpvo_ba_wide_system(float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
                        const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int PPF,
                        int t0, int t1, const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                        const int64_t* p_key_j, const int32_t* p_n, float* S, float* y, int* status, void* stream);
int dpvo_ba_wide_update(float* poses, float* patches, const float* intrinsics, const float* target, const float* weight,
                        const float* lmbda, const int64_t* ii, const int64_t* jj, const int64_t* kk, int64_t E, int P, int PPF,
                        int t0, int t1, const int32_t* p_order, const int32_t* p_start, const int64_t* p_key_i,
                        const int64_t* p_key_j, const int32_t* p_n, const float* dX, int* status, void* stream);

/*
 * cuda_ba.solve_system -- ba.cpp:120-180 (pose-graph optimisation of the loop-closure back end,
 * loop_closure/optim_utils.py:229): normal equations of r relative-pose residuals with 7x7 Jacobian blocks,
 *     A = J^T J  (fp64 [7n, 7n]),  b = -J^T res  (fp64 [7n]),  A.diag += lm * A.diag + ep.
 * The reference builds them in an Eigen sparse matrix on the CPU; here one kernel scatters the four 7x7 block
 * products of every residual.  The caller solves the leading 7*freen x 7*freen system (dense Cholesky).
 * J_i, J_j fp32 [r, 7, 7], res fp32 [r, 7], ii, jj int64 [r] (ii != jj), A and b zeroed by the call.
 */
int dpvo_posegraph_system(const float* J_i, const float* J_j, const int64_t* ii, const int64_t* jj, const float* res,
                          int64_t r, int64_t n, double ep, double lm, double* A, double* b, void* stream);

/*
 * cuda_ba.reproject -- ba_cuda.cu:585-617 (kernel :379-429): coords fp32 [E, 2, P, P].
 * clamp_depth = 0 reproduces the kernel (divide by raw Z, :422-423, intrinsics row 0);
 * clamp_depth = 1 reproduces pops.transform (projective_ops.py:53-68: Z clamped to >= 0.1 in
 * proj :43, per-edge intrinsics rows ii / jj), the form DPVO.reproject feeds to corr.
 */
int dpvo_reproject(const float* poses, const float* patches, const float* intrinsics,
                   const int64_t* ii, const int64_t* jj, const int64_t* kk,
                   float* coords, int64_t E, int P, int clamp_depth, void* stream);

/* ======================================================================================
 * lietorch_backends
 * ====================================================================================== */
/*
 * One entry per pybind function of lietorch.cpp:286-316.  group = DPVO_SO3..DPVO_SIM3,
 * dtype = DPVO_F32 / DPVO_F64, n = batch (number of group elements), all tensors contiguous
 * [n, dim].  Embedding widths: SO3 4, RxSO3 5, SE3 7, Sim3 8; tangent widths 3, 4, 6, 7.
 * Backward functions follow lietorch_gpu.cu:32-256 (left-tangent gradients; gradients w.r.t.
 * group elements have the embedding width with the components past the tangent width 0).
 * All four groups are implemented: SO3 / SE3 with register-specialised operators, RxSO3 / Sim3 (rxso3.h, sim3.h) with the
 * generic small-matrix operators of csrc/lie_scaled.cuh.
 */
int dpvo_lie_exp(int group, int dtype, const void* a, void* X, int64_t n, void* stream);
int dpvo_lie_exp_backward(int group, int dtype, const void* grad, const void* a, void* da,
                          int64_t n, void* stream);
int dpvo_lie_log(int group, int dtype, const void* X, void* a, int64_t n, void* stream);
int dpvo_lie_log_backward(int group, int dtype, const void* grad, const void* X, void* dX,
                          int64_t n, void* stream);
int dpvo_lie_inv(int group, int dtype, const void* X, void* Y, int64_t n, void* stream);
int dpvo_lie_inv_backward(int group, int dtype, const void* grad, const void* X, void* dX,
                          int64_t n, void* stream);
int dpvo_lie_mul(int group, int dtype, const void* X, const void* Y, void* Z, int64_t n,
                 void* stream);
int dpvo_lie_mul_backward(int group, int dtype, const void* grad, const void* X, const void* Y,
                          void* dX, void* dY, int64_t n, void* stream);
int dpvo_lie_adj(int group, int dtype, const void* X, const void* a, void* b, int64_t n,
                 void* stream);
int dpvo_lie_adj_backward(int group, int dtype, const void* grad, const void* X, const void* a,
                          void* dX, void* da, int64_t n, void* stream);
int dpvo_lie_adjT(int group, int dtype, const void* X, const void* a, void* b, int64_t n,
                  void* stream);
int dpvo_lie_adjT_backward(int group, int dtype, const void* grad, const void* X, const void* a,
                           void* dX, void* da, int64_t n, void* stream);
int dpvo_lie_act(int group, int dtype, const void* X, const void* p, void* q, int64_t n,
                 void* stream);
int dpvo_lie_act_backward(int group, int dtype, const void* grad, const void* X, const void* p,
                          void* dX, void* dp, int64_t n, void* stream);
int dpvo_lie_act4(int group, int dtype, const void* X, const void* p, void* q, int64_t n,
                  void* stream);
int dpvo_lie_act4_backward(int group, int dtype, const void* grad, const void* X, const void* p,
                           void* dX, void* dp, int64_t n, void* stream);
int dpvo_lie_as_matrix(int group, int dtype, const void* X, void* T, int64_t n, void* stream);
int dpvo_lie_projector(int group, int dtype, const void* X, void* Pm, int64_t n, void* stream);
int dpvo_lie_jinv(int group, int dtype, const void* X, const void* a, void* b, int64_t n,
                  void* stream);

/* ======================================================================================
 * Update operator building blocks (dpvo/net.py:27-92, dpvo/blocks.py:15-48)
 * ====================================================================================== */

/*
 * y[r, :] = LayerNorm(a[r] + b[r] + c[r]) * gamma + beta, optionally followed by ReLU
 * (b, c optional, may be NULL).  rows x dim, dim % 128 == 0, dim <= 1024; eps as given (1e-3 in
 * Update: net.py:41,47,49,57).  a/b/c element types in_dtypes[3] (F16/F32); gamma/beta fp32;
 * statistics in fp32.  Result written as fp32 (y32) and/or fp16 (y16) in the same pass.
 * b_index (optional, int64 [rows]): operand b is read from row b_index[r] -- the context gather
 * `imap[:, kk % (M*pmem)]` of dpvo.py:334 folded into the pass.
 * c_scale (optional, fp16 [rows, dim] with row stride ld_c_scale): operand c enters as c_scale * c, i.e. the
 * GatedResidual x + gate * res (blocks.py:28-29) that precedes the second LayerNorm of the GRU is folded in.
 * y32 may alias a (rows are read completely before they are written).
 */
int dpvo_add_layernorm(const void* a, const void* b, const void* c, const int* in_dtypes,
                       const int64_t* b_index, const void* c_scale, int64_t ld_c_scale,
                       const float* gamma, const float* beta, float eps,
                       void* y32, void* y16, int relu, int64_t rows, int dim, void* stream);

/* Neighbour gather with mask (net.py:81-85): y[e, :] = (idx[e] >= 0) ? x[idx[e], :] : 0. */
int dpvo_gather_rows_masked(const void* x, int x_dtype, const int64_t* idx,
                            void* y, int y_dtype, int64_t rows, int dim, void* stream);

/*
 * net32[e, :] += u[src(e), :] with src(e) = e (group_of == NULL; residual adds of net.py:84-85)
 * or src(e) = group_of[e] (the `[:, jx]` expand of blocks.py:46 fused with net.py:87-88).
 * net32 fp32 in place; optional fp16 copy of the result in net16.
 */
int dpvo_residual_add(void* net32, const void* u, int u_dtype, const int32_t* group_of, void* net16,
                      int64_t rows, int dim, void* stream);
/* net16[e, :] = fp16( net32[e, :] + u[src(e), :] ) without touching net32: the operand of the next dense layer when the
 * consumer of the fp32 state (dpvo_update_gru_heads) adds u[src] itself -- one pass over the fp32 state less */
int dpvo_residual_sum16(const void* net32, const void* u, int u_dtype, const int32_t* group_of, void* net16,
                        int64_t rows, int dim, void* stream);

/* GatedResidual (blocks.py:28-29): y32 = x32 + sigmoid(gate16) * res16; optional relu(y) as fp16. */
int dpvo_gated_residual(const void* x32, const void* gate16, const void* res16, void* y32, void* y16_relu,
                        int64_t rows, int dim, void* stream);

/*
 * SoftAgg reduction (blocks.py:40-43; torch_scatter 2.1.2 scatter_softmax + scatter_sum):
 *   y[g, c] = sum_{e in g} f[e, c] * exp(gl[e, c] - max_g) / sum_{e in g} exp(gl[e, c] - max_g)
 * over the CSR of dpvo_group_edges (order, group_start; G read from n_groups on the device).
 * f, gl fp16 [E, dim] with row stride ld elements (so both may be column blocks of one [E, 2*dim]
 * GEMM output); y fp16 [G, dim]; max_groups bounds the launch.  fp32 math, one pass.
 */
int dpvo_softagg_reduce(const void* f16, const void* g16, int64_t ld, const int32_t* order, const int32_t* group_start,
                        const int32_t* n_groups, int64_t max_groups, void* y16, int dim, void* stream);

/*
 * SoftAgg f|g layer fused with its reduction (blocks.py:31-43): y as dpvo_softagg_reduce computes it from
 *   f = fp16(x Wf^T + bf), gl = fp16(x Wg^T + bg)
 * without the [E, 2*dim] layer output.  x16 fp16 [E, dim] (row stride ldx, rows 16-byte aligned) is read in the
 * sorted order of the CSR (order, group_of, group_start; G read from n_groups on the device).  w16 fp16 [2*dim, dim]
 * and bias fp32 [2*dim] hold the f and g rows interleaved by 96-channel slice: rows 192 s .. 192 s + 95 are
 * Wf rows 96 s .. 96 s + 95, rows 192 s + 96 .. 192 s + 191 are Wg rows 96 s .. 96 s + 95.  y fp16 [max_groups, dim];
 * rows G .. max_groups - 1 are zero.  dim = 384.  workspace: dpvo_softagg_fused_workspace_bytes(E) bytes
 * (partial results of the groups that span more than one 64-row tile).  Two launches give bit-identical results.
 */
int64_t dpvo_softagg_fused_workspace_bytes(int64_t E);
int dpvo_softagg_fused(const void* x16, int64_t ldx, const int32_t* order, const int32_t* group_of,
                       const int32_t* group_start, const int32_t* n_groups, const void* w16, const float* bias,
                       int64_t E, int64_t max_groups, void* y16, void* workspace, int64_t workspace_bytes,
                       int dim, void* stream);

/*
 * The two output heads (net.py:62-71, 92): delta = Wd relu(net) + bd, weight = sigmoid(Ww relu(net) + bw).
 * W4 fp32 [4, dim] = rows (Wd[0], Wd[1], Ww[0], Ww[1]); b4 fp32 [4]; delta, weight fp32 [rows, 2].
 * coords (optional, fp32 [rows, 2, P, P]): when given, `delta` receives the BA target
 * coords[:, :, P/2, P/2] + delta directly (dpvo.py:341).
 * gate16 / res16 (optional, fp16 [rows, dim], row strides ld_gate / ld_res): the heads read net32 + gate16 * res16
 * and that sum is written back to net32 -- the last GatedResidual of the GRU folded into this pass.
 */
int dpvo_update_heads(void* net32, const void* gate16, int64_t ld_gate, const void* res16, int64_t ld_res,
                      const float* W4, const float* b4, const float* coords, int P,
                      float* delta, float* weight, int64_t rows, int dim, void* stream);

/*
 * Dense layer on tensor cores (wgmma, fp16 operands, fp32 accumulation in registers):
 *   Y = epilogue( X[rows, K] @ W[N, K]^T + bias[N] )
 * X, W fp16 row-major (K contiguous, rows 16-byte aligned), bias fp32 (may be NULL).
 * gather (optional, int64 [rows]): row r of X is read from X[gather[r]], or taken as zero when
 * gather[r] < 0 -- the masked neighbour gather of net.py:81-85 folded into the operand load.
 * Epilogues:
 *   DPVO_EPI_NONE      y = acc + bias
 *   DPVO_EPI_RELU      y = relu(acc + bias)
 *   DPVO_EPI_SIGMOID   y = sigmoid(acc + bias)
 *   DPVO_EPI_RESADD    y = res + acc + bias                       (res: [rows, N], F16/F32, stride ldres)
 *   DPVO_EPI_GATEDRES  y = res + gate * (acc + bias)              (gate: [rows, N] fp16, stride ldgate)
 *   DPVO_EPI_SIGMOID_RELU  columns [0, N/2): sigmoid(acc + bias), columns [N/2, N): relu(acc + bias) -- two layers that
 *                      share their input stacked into one GEMM (gate and first residual layer of GatedResidual, blocks.py:17-29)
 * Y dtype y_dtype (F16 or F32), row stride ldy; Y16 (optional) receives an fp16 copy of the same
 * result (row stride ldy16) so a following layer can consume it without another pass.  Y may alias
 * res.  K % 64 == 0 (pad 882 -> 896 with zeros), N % 32 == 0.  Row tails are handled.
 */
#define DPVO_EPI_NONE     0
#define DPVO_EPI_RELU     1
#define DPVO_EPI_SIGMOID  2
#define DPVO_EPI_RESADD   3
#define DPVO_EPI_GATEDRES 4
#define DPVO_EPI_SIGMOID_RELU 5
int dpvo_linear_f16(const void* X, int64_t ldx, const int64_t* gather, const void* W, int64_t ldw,
                    const float* bias, const void* res, int res_dtype, int64_t ldres,
                    const void* gate, int64_t ldgate, void* Y, int y_dtype, int64_t ldy,
                    void* Y16, int64_t ldy16,
                    int64_t rows, int N, int K, int epilogue, void* stream);

/* ---- Update operator, fused layer chains (dpvo_b200/csrc/chain.cu) -------------------------------------------------
 * The row-local stretches of Update.forward (dpvo/net.py:74-92) as one wgmma kernel each: a 64-edge tile runs
 * through every dense layer of the stretch on chip (operand tile in shared memory, fp32 accumulator in registers),
 * LayerNorm / gating / heads in the epilogues.  DIM = 384 (net.py:24), E = edges, all weights fp16 row-major
 * [out, in], all parameters fp32, `net32` is the fp32 recurrent state [E, 384] updated IN PLACE.
 *
 * dpvo_update_corr_norm   (net.py:76-77, corr = net.py:66-72)
 *     net32 <- LN_norm( net32 + inp16[inp_index ? inp_index[e] : e] + corr.5( relu( LN_corr.3( corr.2( relu( corr.0(corr16) ) ) ) ) ) )
 *     corr16 [E, 896] fp16 (882 correlation features zero padded to 896; row stride ld_corr halves), W0 = corr.0.weight padded
 *     to [384, 896], W25 = rows of corr.2.weight then corr.5.weight [768, 384],
 *     params = corr.0.bias | corr.2.bias | corr.3.weight | corr.3.bias | corr.5.bias | norm.weight | norm.bias (7 x 384).
 *     net16 [E, 384] receives the fp16 copy of the new state (operand of the next layer).
 * dpvo_update_neighbor_mlp  (net.py:83-85, one call for c1 with ix and one for c2 with jx)
 *     net32 <- net32 + c.2( relu( c.0( mask * net16_in[index] ) ) ),  index[e] = -1 masks the row (mask = 0)
 *     Wab = rows of c.0.weight then c.2.weight [768, 384], params = c.0.bias | c.2.bias.  net16_out != net16_in.
 * dpvo_update_gru_heads  (net.py:88-92, blocks.py:15-29)
 *     x = LN_gru.0( net32 + hkk16[group_kk[e]] + hij16[group_of[e]] );  y = x + gate1(x) * res1(x);  z = LN_gru.2(y);
 *     net32 <- z + gate2(z) * res2(z)        (net.py:87-88: the two SoftAgg results are added here, not in a pass of their own)
 *     delta = d(net32) (+ centre of coords when given: the BA target of dpvo.py:341), weight = w(net32)
 *     W6 = rows of gru.1.gate.0 | gru.1.res.0 | gru.1.res.2 | gru.3.gate.0 | gru.3.res.0 | gru.3.res.2 weights [2304, 384],
 *     params = gru.0.weight | gru.0.bias | b(gate1) | b(res1.0) | b(res1.2) | gru.2.weight | gru.2.bias | b(gate2) | b(res2.0) |
 *              b(res2.2) | d.1.weight[2,384] | w.1.weight[2,384] | d.1.bias[2] | w.1.bias[2]          (14 x 384 + 4 floats)
 *     hij16 [G, 384] fp16 / group_of int32 [E], hkk16 [G', 384] fp16 / group_kk int32 [E]: each pair may be NULL (nothing
 *     added).  coords [E, 2, P, P] fp32 or NULL.
 *     delta, weight [E, 2] fp32.  workspace: dpvo_update_gru_workspace_bytes() bytes (row-private scratch, L2 resident).
 */
int dpvo_update_corr_norm(const void* corr16, int64_t ld_corr, const void* W0, const void* W25, const float* params,
                          float* net32, const void* inp16, const int64_t* inp_index, void* net16, int64_t E, void* stream);
int dpvo_update_neighbor_mlp(const void* net16_in, const int64_t* index, const void* Wab, const float* params,
                             float* net32, void* net16_out, int64_t E, void* stream);
int64_t dpvo_update_gru_workspace_bytes(void);
int dpvo_update_gru_heads(float* net32, const void* hij16, const int32_t* group_of, const void* hkk16, const int32_t* group_kk,
                          const void* W6, const float* params, const float* coords, int P, float* delta, float* weight,
                          void* workspace, int64_t E, void* stream);

/* ---- Device-resident patch-graph bookkeeping (dpvo_b200/csrc/pgraph.cu) ---------------------------------------------
 * Fixed-capacity edge arrays ii, jj, kk (int64 [cap]) + active (uint8 [cap]) replace the reference's growing /
 * shrinking tensors (dpvo/dpvo.py:215-238 append_factors / remove_factors, :282-286 keyframe renumbering) so that a
 * captured CUDA graph of update() survives topology changes.  A parked slot holds the dummy edge (ii = jj = dummy_frame,
 * kk = dummy_patch: a reserved frame / patch no real edge uses), so parked edges form their own groups in every
 * grouping and never mix with real ones; the caller multiplies the confidence weights by `active` before bundle
 * adjustment.  All decisions read device scalars: no host synchronisation, graph capturable.
 *   dpvo_pgraph_remove   rule 0: park active edges whose patch frame kk / M < *frame - param          (dpvo.py:300, 306)
 *                        rule 1: park edges with ii == *frame or jj == *frame, then for the survivors
 *                                ii > k: kk -= M, ii -= 1;  jj > k: jj -= 1                            (dpvo.py:282-286)
 *                        enable (device int32, may be NULL): 0 turns the call into a no-op (keyframe decision on device)
 *   dpvo_pgraph_append   new edges fill the parked slots in index order; state (fp32 [cap, 384] row-major, may be NULL):
 *                        the rows of the new edges are zeroed (dpvo.py:220-221); slot_of_new (int32 [n_new], required with
 *                        state) receives the slot of every new edge, -1 if the store is full (*overflow is then set to 1)
 *   dpvo_pgraph_new_edges  the (2 r - 1) M edges DPVO adds for frame *n - 1 in steady state (n >= r): __edges_forw then
 *                        __edges_back of dpvo.py:362-375, as (ii = source frame, jj = target frame, kk = patch)
 * n_active: device int32 running count of active edges (integer atomics).
 */
int dpvo_pgraph_remove(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, int rule,
                       const int64_t* frame, int64_t param, const int32_t* enable, int64_t dummy_frame,
                       int64_t dummy_patch, int M, int32_t* n_active, void* stream);
int dpvo_pgraph_append(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t cap, const int64_t* new_ii,
                       const int64_t* new_jj, const int64_t* new_kk, int64_t n_new, const int32_t* enable,
                       float* state, int32_t* slot_of_new, int32_t* n_active, int32_t* overflow, void* stream);
int dpvo_pgraph_new_edges(const int64_t* n_dev, int M, int r, int64_t* ii, int64_t* jj, int64_t* kk, void* stream);

/* ---- Proximity loop closure (dpvo_b200/csrc/loop.cu) ----------------------------------------------------------------
 * The DPV-SLAM back end of dpvo/patchgraph.py:56-91 and dpvo/dpvo.py:223-326, 449-455 on the fixed-capacity store.
 * Candidates: targets j in [n - freq, n - kf_index), sources i in [max(l - max_age, 0), l), l = n - removal, laid out
 * as J = freq - kf_index rows of max_age slots: slot (j - (n - freq)) * max_age + (i - max(l - max_age, 0)).  n and
 * last_ba are device int64 scalars; a proposal runs only when n - *last_ba >= freq (dpvo.py:449-450).
 *   dpvo_loop_candidates  J * max_age, the length of `scores` (0 for a bad range)
 *   dpvo_loop_scores   fp32 [J * max_age]: mean over the valid patches of frame i of the centre-pixel flow
 *                      0.5 |full - origin| + 0.5 |translation only - origin| (valid: Z > 0.2), if more than 0.75 M are
 *                      valid; +inf otherwise, for a slot outside the range and for every slot when no proposal is due.
 *                      A fixed-order reduction: two launches give identical bits.
 *   dpvo_loop_select   reduce_edges (loop_closure/optim_utils.py:23-61): slots with score < thresh in ascending
 *                      (score, slot), skip j - i < 30 and suppressed pairs, accept and suppress (i +- 1, j), at most
 *                      max_pairs.  pairs int64 [max_pairs, 2] = (i, j) in acceptance order, *n_pairs their count (0 when no
 *                      proposal ran); *last_ba = n when one was accepted.  The M edges of accepted pair p go to slots
 *                      p M + m of the loop region (ii, jj, kk, active, state: its first `region` slots), state rows zeroed;
 *                      *n_active counts the new edges, *overflow is set if a slot still held an active edge.
 *                      (freq - kf_index) * max_age > 16384 is DPVO_ERR_UNSUPPORTED.
 *   dpvo_pgraph_remove_store  the third removal rule: park the active edges with
 *                      kk / M < n - removal && !((jj - ii) > 30 && jj > n - opt_window)   (dpvo.py:300-310)
 *                      and keep each one's (ii, jj, kk, target [2], weight [2]) in the inactive store (capacity s_cap,
 *                      fp32 target / weight [cap, 2]).  The store fills from its end: the edges of one call are placed in
 *                      slot order below those of the previous calls, so the used part is [s_cap - *s_count, s_cap).  Edges
 *                      beyond the capacity are dropped and *s_overflow is set.
 *   dpvo_loop_flags    flags int64 [4]: 1 + the offset of the last active edge in slots [normal, cap) (0 without one);
 *                      1 if an active edge has ii < n - removal - 1
 *                      (dpvo.py:348); the minimum active ii (INT64_MAX without one); *s_count (0 if s_count is NULL)
 *   dpvo_loop_normalize  PatchGraph.normalize (patchgraph.py:84-91) for frames [0, n): depths / mean depth, translations
 *                      * mean depth, every pose rebased on pose 0.  patches fp32 [>= n M, 3, P, P], poses fp32 [>= n, 7]
 *   dpvo_loop_normalize_deltas  the same, and the translations of the n_delta relative poses of a keyframe delta table
 *                      (fp32 [n_delta, 7], dpvo_keyframe_*) * mean depth as well (dP.scale(s), patchgraph.py:89-90).
 *                      dpvo_loop_normalize is this call with no table.
 */
int64_t dpvo_loop_candidates(int max_age, int freq, int kf_index);
int dpvo_loop_scores(const float* poses, const float* patches, const float* intrinsics, const int64_t* n_dev,
                     const int64_t* last_ba, int M, int removal, int max_age, int freq, int kf_index,
                     float* scores, void* stream);
int dpvo_loop_select(const float* scores, const int64_t* n_dev, int64_t* last_ba, int M, int removal, int max_age,
                     int freq, int kf_index, float thresh, int max_pairs, int64_t* pairs, int32_t* n_pairs,
                     int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, int64_t region, float* state,
                     int32_t* n_active, int32_t* overflow, void* stream);
int dpvo_pgraph_remove_store(int64_t* ii, int64_t* jj, int64_t* kk, uint8_t* active, const float* target,
                             const float* weight, int64_t cap, const int64_t* n_dev, int removal, int opt_window,
                             const int32_t* enable, int64_t dummy_frame, int64_t dummy_patch, int M,
                             int32_t* n_active, int64_t* s_ii, int64_t* s_jj, int64_t* s_kk, float* s_target,
                             float* s_weight, int64_t s_cap, int32_t* s_count, int32_t* s_overflow, void* stream);
int dpvo_loop_flags(const int64_t* ii, const uint8_t* active, int64_t cap, int64_t normal, int64_t n, int removal,
                    const int32_t* s_count, int64_t* flags, void* stream);
int dpvo_loop_normalize(float* poses, float* patches, int64_t n, int M, int P, void* stream);
int dpvo_loop_normalize_deltas(float* poses, float* patches, int64_t n, int M, int P, float* delta, int64_t n_delta,
                               void* stream);

/* ---- Keyframe culling (dpvo_b200/csrc/keyframe.cu) ------------------------------------------------------------------
 * DPVO.keyframe (dpvo/dpvo.py:257-300) and get_pose / terminate (:166-198) for B >= 1 streams of F frame slots each
 * (one stream: B = 1).  Stream b's frames are [b F, (b + 1) F) of poses fp32 [B F, 7], patches fp32 [B F M, 3, 3, 3] and
 * intrinsics fp32 [B F, 4]; edges carry these global numbers.  Per stream, on the device: n int64 [B] (local frame
 * counts), tstamp int64 [B, F] (the timestamp of every frame slot), counter int64 [B] (the next timestamp), and a delta
 * table of T >= F timestamps: delta fp32 [B, T, 7] (relative poses) with delta_src int64 [B, T] (their source
 * timestamp, < 0 where nothing is recorded).  KI = keyframe_index >= 1.
 *   dpvo_keyframe_motion  stream b's edges are slots [b slots, (b + 1) slots) of ii / jj / kk / active.  With
 *                      i = n - KI - 1, j = n - KI + 1, k = n - KI: m = mean(i, j) + mean(j, i), each the fp64 mean of the
 *                      flow_mag (beta = 0.5) of all 9 pixels of every active edge of that (ii, jj), validity ignored; an
 *                      empty set gives NaN.  flag int32 [B] = (m / 2 < thresh), k int64 [B] = b F + k (global, the
 *                      frame for dpvo_pgraph_remove rule 1), m fp64 [B].  Under the flag: delta[tstamp[k]] =
 *                      P_k P_{k-1}^-1 with source tstamp[k - 1] (*overflow [b] = 1 if tstamp[k] >= T), and n[b] -= 1.
 *                      64 CTAs per stream write partial sums to workspace (dpvo_keyframe_motion_workspace_bytes(B)
 *                      bytes), one thread per stream adds them in order: two launches give identical bits.
 *   dpvo_keyframe_shift  under flag[b]: for t = k .. n - 2 (KI - 1 launches, one per step, in that order), slot t + 1 ->
 *                      slot t of each of the nbuf (<= 9) buffers.  Buffer q's slot t of stream b is the row_bytes[q]
 *                      bytes at bases[q] + (b rows[q] + t mod rows[q]) row_bytes[q]: rows = F for per-frame buffers,
 *                      mem / pmem for the rings.  rows[q] < KI and row_bytes not a positive multiple of 4 are rejected.
 *   dpvo_keyframe_shift_bytes  dpvo_keyframe_shift for slots of any positive byte count at any alignment (a buffer whose
 *                      slots 4 does not divide is copied one byte per thread), e.g. the colours uint8 [F, M, 3].
 *   dpvo_keyframe_count  mode 0 (add_frame, dpvo.py:400, 440): tstamp[n - 1] = counter, counter += 1.  mode 1
 *                      (skip_frame, :441-444): delta[counter] = identity with source counter - 1, counter += 1.  A
 *                      timestamp outside the table sets overflow[b].
 *   dpvo_keyframe_trajectory  out fp32 [B, T, 7]: for t < counter, pose(t)^-1 where pose(t) is the pose of the live
 *                      frame with tstamp t, else dP_t pose(src_t) (terminate()'s poses.inv()).  map int32 [B, T] is
 *                      scratch.  A chain of stream b that meets an unrecorded timestamp writes NaN and sets error[b]
 *                      (int32 [B]).
 */
int dpvo_keyframe_motion(const float* poses, const float* patches, const float* intrinsics, int64_t F, int B,
                         const int64_t* ii, const int64_t* jj, const int64_t* kk, const uint8_t* active, int64_t slots,
                         int64_t* n, const int64_t* tstamp, float* delta, int64_t* delta_src, int64_t T, int ki,
                         double thresh, int32_t* flag, int64_t* k, double* m, int32_t* overflow, void* workspace,
                         int64_t workspace_bytes, void* stream);
int64_t dpvo_keyframe_motion_workspace_bytes(int B);
int dpvo_keyframe_shift(void* const* bases, const int64_t* row_bytes, const int64_t* rows, int nbuf, int64_t F, int B,
                        int ki, const int32_t* flag, const int64_t* k, void* stream);
int dpvo_keyframe_shift_bytes(void* const* bases, const int64_t* row_bytes, const int64_t* rows, int nbuf, int64_t F,
                              int B, int ki, const int32_t* flag, const int64_t* k, void* stream);
int dpvo_keyframe_count(int mode, const int64_t* n, int64_t* tstamp, int64_t F, int B, int64_t* counter, float* delta,
                        int64_t* delta_src, int64_t T, int32_t* overflow, void* stream);
int dpvo_keyframe_trajectory(const float* poses, const int64_t* tstamp, const int64_t* n, int64_t F, int B,
                             const float* delta, const int64_t* delta_src, int64_t T, const int64_t* counter,
                             int32_t* map, float* out, int32_t* error, void* stream);

/* ---- Frame encoders (dpvo_b200/csrc/encoder.cu) ---------------------------------------------------------------------
 * BasicEncoder4 (extractor.py:200-264) as used by Patchifier (net.py:95-157) for inference: fnet (instance norm after
 * every convolution but the last, output 128) and inet (no norm, output 384).  Activations are NHWC fp16, convolutions
 * run on the tensor cores with fp32 accumulation and round their output to fp16.
 *
 * Packed weights (FrameEncoder.pack()):
 *   w16  fp16 blob: for encoder e = fnet, inet and layer l = 0..10 in the order
 *          conv1 (stem), layer1.0.conv1, layer1.0.conv2, layer1.1.conv1, layer1.1.conv2, layer2.0.conv1,
 *          layer2.0.downsample.0, layer2.0.conv2, layer2.1.conv1, layer2.1.conv2, conv2 (output)
 *        the layer's weight W[cout][cin][ky][kx] as [tap = ky*k + kx][cin / 8][cout][cin % 8], back to back.  The stem
 *        is one tap with K = (cin*7 + ky)*7 + kx (147, zero-padded to 160) in place of cin.
 *   b32  fp32 [2][11][384]: the biases, zero-padded.
 *
 * dpvo_encoder_conv: one layer for nenc (1 or 2) encoders, io[e] describing encoder e.  shape is a DPVO_ENC_* value.
 *   prologue: stem: x is the uint8 image [3, H, W] with element strides x_strides (c, y, x), normalised as
 *                   fp16(2 (x / 255) - 0.5) (dpvo.py:389).
 *             otherwise x is fp16 NHWC [H, W, cin] dense and is transformed as
 *                   x' = relu?((x - mean) * rstd)    (x_stats [2][cin] = (mean, rstd), or NULL for none; x_relu)
 *                   skip given: x' = relu(skip' + x'),  skip' = relu?((skip - mean) * rstd) by skip_stats / skip_relu
 *             out-of-image taps read 0 after the transform.  joined (3x3 layers with skip): x' of every pixel is also
 *             written there, fp16 NHWC [H, W, cin].
 *   epilogue: y = fp16((conv(x') + bias) * scale), pixel strides y_sy, y_sx, channel stride 1.
 *             pool (optional): fp16 4x4 average of y (F.avg_pool2d order), strides pool_sy, pool_sx.
 *             stats (optional, cout <= 64): [2][cout] (mean, 1/sqrt(var + 1e-5)) of the fp16 y over the image.
 *   workspace: dpvo_encoder_conv_workspace_bytes(shape, H, W) bytes when any stats are requested.
 *   Output size: (H + 2 (k/2) - k) / s + 1.  No float atomics: two launches give identical bits.
 *
 * dpvo_encode_frame: both encoders over one uint8 image [3, H, W] (element strides s_c, s_y, s_x), about a dozen
 * launches, writing a new frame's slots directly (all channels-last, channel stride 1):
 *   fmap1  fp16 [h, w, 128]     fnet(image) / 4                      (pixel strides f1_sy, f1_sx)
 *   fmap2  fp16 [h/4, w/4, 128] F.avg_pool2d(fmap1, 4, 4)            (f2_sy, f2_sx)
 *   imap   fp16 [M, 384]        inet(image) / 4 at the centroids      (row stride i_sm)
 *   gmap   fp16 [M, 3, 3, 128]  the 3x3 windows of fmap1 at the centroids (strides g_sm, g_sy, g_sx)
 *   patches fp32 [M, 3, 3, 3]   (x + dx, y + dy, 1) around each centroid, contiguous
 * coords fp32 [M, 2] (x, y) integer centroids.  h, w = the encoder output size of H, W.
 * workspace: dpvo_encode_frame_workspace_bytes(H, W) bytes (activations, statistics).
 * It is the B = 1 case of dpvo_encode_frames.
 *
 * dpvo_encode_frames: B (1..64) images in one pass, the same launches as one image: image b is uint8 [3, H, W] at
 * images + b s_b (element strides s_c, s_y, s_x: a stacked [B, 3, H, W] tensor or its permuted [B, H, W, 3] view).
 * Each image is encoded with its own instance-norm statistics, and its slots are bit-identical to dpvo_encode_frame of
 * that image alone.  The destinations are rows of rings (element strides between rows: f1_sr, f2_sr, g_sm, i_sm, 27):
 *   fmap1 / fmap2  row frame_row[b] of rings of frame_rows rows
 *   gmap / imap    rows [feat_row[b], feat_row[b] + M) of rings of feat_rows rows
 *   patches        rows [patch_row[b], patch_row[b] + M) of a [patch_rows, 3, 3, 3] buffer
 * The row lists are host int64 [B]; a row outside its ring, or two images writing a common row, is rejected.
 * coords fp32 [B, M, 2].  depth fp32 [B, M] (the patches' third channel), or NULL for 1.
 * workspace: dpvo_encode_frames_workspace_bytes(B, H, W) bytes, B blocks of dpvo_encode_frame_workspace_bytes(H, W).
 * One strided memset and 12 launches for any B; no host synchronisation (graph-capturable).
 *
 * dpvo_encode_frames_colors: dpvo_encode_frames that also writes the viewer colours (dpvo.py:392-404), uint8 rows
 * [patch_row[b], patch_row[b] + M) of colors [patch_rows, 3] (the patches' rows; pg.colors_'s [F, M, 3] layout):
 *   colors[m][c] = uint8((clr[2 - c] + 0.5) * 127.5),  clr = the bilinear patchify (altcorr/correlation.py:51-66) of
 *   2 (image * fp32(1 / 255)) - 0.5 at 4 (coords[m] + 0.5), pixels outside the image 0, each step one fp32 operation
 *   rounded to nearest, the cast truncating.  Same launches as dpvo_encode_frames; colors must not be NULL.
 */
#define DPVO_ENC_STEM        0   /* 7x7/2, 3 -> 32   */
#define DPVO_ENC_C3_32       1   /* 3x3/1, 32 -> 32  */
#define DPVO_ENC_C3S2_32_64  2   /* 3x3/2, 32 -> 64  */
#define DPVO_ENC_C1S2_32_64  3   /* 1x1/2, 32 -> 64  */
#define DPVO_ENC_C3_64       4   /* 3x3/1, 64 -> 64  */
#define DPVO_ENC_OUT_128     5   /* 1x1/1, 64 -> 128 */
#define DPVO_ENC_OUT_384     6   /* 1x1/1, 64 -> 384 */

typedef struct dpvo_encoder_conv_io {
  const void* x;
  int64_t x_strides[3];
  const float* x_stats;
  int x_relu;
  const void* skip;
  const float* skip_stats;
  int skip_relu;
  void* joined;
  const void* w;
  const float* bias;
  void* y;
  int64_t y_sy, y_sx;
  void* pool;
  int64_t pool_sy, pool_sx;
  float* stats;
  float scale;
} dpvo_encoder_conv_io;

int64_t dpvo_encoder_conv_workspace_bytes(int shape, int H, int W);
int dpvo_encoder_conv(int shape, int H, int W, int nenc, const dpvo_encoder_conv_io* io, void* workspace,
                      int64_t workspace_bytes, void* stream);
int64_t dpvo_encode_frame_workspace_bytes(int H, int W);
int dpvo_encode_frame(const uint8_t* image, int64_t s_c, int64_t s_y, int64_t s_x, int H, int W,
                      const void* w16, const float* b32, const float* coords, int M,
                      void* fmap1, int64_t f1_sy, int64_t f1_sx, void* fmap2, int64_t f2_sy, int64_t f2_sx,
                      void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm,
                      float* patches, void* workspace, int64_t workspace_bytes, void* stream);
int64_t dpvo_encode_frames_workspace_bytes(int B, int H, int W);
int dpvo_encode_frames(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H, int W,
                       const void* w16, const float* b32, const float* coords, int M,
                       void* fmap1, int64_t f1_sr, int64_t f1_sy, int64_t f1_sx,
                       void* fmap2, int64_t f2_sr, int64_t f2_sy, int64_t f2_sx, int64_t frame_rows,
                       void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm, int64_t feat_rows,
                       float* patches, int64_t patch_rows,
                       const int64_t* frame_row, const int64_t* feat_row, const int64_t* patch_row,
                       const float* depth, void* workspace, int64_t workspace_bytes, void* stream);

int dpvo_encode_frames_colors(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H, int W,
                              const void* w16, const float* b32, const float* coords, int M,
                              void* fmap1, int64_t f1_sr, int64_t f1_sy, int64_t f1_sx,
                              void* fmap2, int64_t f2_sr, int64_t f2_sy, int64_t f2_sx, int64_t frame_rows,
                              void* gmap, int64_t g_sm, int64_t g_sy, int64_t g_sx, void* imap, int64_t i_sm, int64_t feat_rows,
                              float* patches, int64_t patch_rows,
                              const int64_t* frame_row, const int64_t* feat_row, const int64_t* patch_row,
                              const float* depth, uint8_t* colors, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- Camera-image preparation (dpvo_b200/csrc/undistort.cu) ---------------------------------------------------------
 * dpvo_undistort_frames: the image preparation of the reference's readers (dpvo/stream.py:image_stream / video_stream,
 * evaluate_tum.py:tum_image_stream) for B (1..64) uint8 images of one raw size H x W in one launch:
 *   cv2.undistort(image, K, (k1, k2, p1, p2, k3)), then, with half, cv2.resize(fx = fy = 0.5, INTER_AREA), then the
 *   crop window rows [y0, y0 + Ho) x columns [x0, x0 + Wo) of the (halved) image.
 * Image b is [3, H, W] at images + b s_b with element strides s_c, s_y, s_x (a stacked [B, 3, H, W] tensor or its
 * permuted [B, H, W, 3] view); its window goes to out + b o_sb, element strides o_sy, o_sx, o_sc (e.g. [B, Ho, Wo, 3]).
 * Channels are processed alike (BGR stays BGR).  Image b is undistorted with cameras[b] (host array, passed by value:
 * a captured graph keeps it).  The arithmetic is OpenCV's exact integer specification (DESIGN §3.8): the float64
 * map rounded to 1/32 pixel, the fixed-point bilinear with 2^15 weight sums and zeros outside the image, the 2 x 2
 * average (sum + 2) >> 2.  A camera without coefficients maps every pixel onto itself (crop, and halve if asked).
 * Rejected (DPVO_ERR_INVALID): B outside 1..64, a non-finite or non-positive focal length, a non-finite principal point
 * or coefficient, halving an odd-sized image, a window outside the (halved) image, an empty window.
 * No workspace, no atomics, no host synchronisation (graph-capturable).
 */
typedef struct dpvo_camera {
  double fx, fy, cx, cy;           /* pinhole intrinsics of the raw image, pixels */
  double k1, k2, p1, p2, k3;       /* OpenCV's radial (k1, k2, k3) and tangential (p1, p2) coefficients */
} dpvo_camera;

int dpvo_undistort_frames(const uint8_t* images, int64_t s_b, int64_t s_c, int64_t s_y, int64_t s_x, int B, int H, int W,
                          const dpvo_camera* cameras, int half, int y0, int x0, int Ho, int Wo, uint8_t* out,
                          int64_t o_sb, int64_t o_sy, int64_t o_sx, int64_t o_sc, void* stream);

/* ---- Map (dpvo_b200/csrc/map.cu) --------------------------------------------------------------------------------------
 * dpvo_point_cloud: the points of DPVO.update (dpvo.py:358-360) for B (1..64) streams of F frame slots and M patches per
 * frame.  Stream b's frames are [b F, (b + 1) F) of poses fp32 [B F, 7] and intrinsics fp32 [B F, 4], its patches
 * [b F M, (b + 1) F M) of patches fp32 [B F M, 3, 3, 3] and its points the same rows of points fp32 [B F M, 3].  n is a
 * host int64 [B] (each stream's frame count, passed by value: a captured graph keeps it).  Rows [0, n[b] M) of stream b
 * get pops.point_cloud's centre point of each patch,
 *   X = ((x - cx) / fx, (y - cy) / fy, 1, d),  P = act4(pose^-1, X),  point = P.xyz / P.w
 * with the lietorch SE3 operators (pose^-1 rounded to fp32 and loaded again, as SE3.inv() then act4 do); the rows above
 * are not written.  One launch, one thread per patch.
 */
int dpvo_point_cloud(const float* poses, const float* patches, const float* intrinsics, int64_t F, int M, int B,
                     const int64_t* n, float* points, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DPVO_B200_H */
