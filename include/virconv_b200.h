/*
 * virconv_b200 — C ABI of the H100 (sm_90a) sparse-convolution hot path of VirConv.
 *
 * The reference (hailanyi/VirConv) has no FFI of its own for this path: every sparse operator is a
 * call into the third-party Python package spconv 2.1 (`import spconv.pytorch as spconv`,
 * pcdet/utils/spconv_utils.py:33-36).  Each entry point below therefore cites the reference CALL
 * SITE (file:line under /root/reference) whose spconv work it replaces; the Python classes in
 * `virconv_b200/spconv_compat.py` re-create the spconv.pytorch surface on top of these calls
 * (binding shown in INTEGRATION.md).
 *
 * Contract (SURVEY §8b):
 *   - plain pointers + sizes; all pointers are DEVICE pointers unless marked "host";
 *   - the caller (PyTorch) owns every input, output and workspace buffer; the library never
 *     allocates, frees or retains a pointer past the call;
 *   - all work is enqueued on the cudaStream_t passed as `stream`; no hidden device sync,
 *     re-entrant, one host thread per device;
 *   - return 0 on success, <0 on error (message: vc_last_error(), thread-local); no exceptions,
 *     no exit();
 *   - row-major everywhere: features [N, C]; indices [N, 1+ndim] int32 = (batch, z, y, x) or
 *     (batch, u, v); conv weight in spconv-2.x layout [C_out, K, C_in] with K = prod(kernel) and
 *     offsets numbered z-major (k = (kz*Ky+ky)*Kx+kx), see detector3d_template.py:358-370;
 *   - a rulebook is a NEIGHBOUR TABLE nbr[K, N_out] int32: input row feeding output row o through
 *     kernel offset k, or -1 (canonical form, SURVEY §8a-R; oracle/rulebook.py is the definition).
 */
#ifndef VIRCONV_B200_H
#define VIRCONV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VC_OK 0
#define VC_ERR_INVALID (-1)      /* bad argument */
#define VC_ERR_CUDA (-2)         /* CUDA runtime error (launch / config) */
#define VC_ERR_WORKSPACE (-3)    /* workspace too small */
#define VC_ERR_UNSUPPORTED (-4)  /* channel count / ndim not compiled in */
#define VC_ERR_PIPELINE (-5)     /* a tensor-core kernel's mbarrier wait timed out earlier (err_flag set): results invalid */

#define VC_MAX_NDIM 3
#define VC_TILE_ROWS 128         /* output rows per CTA tile in the conv kernels (BN partial granularity) */

typedef void* vc_stream_t;       /* cudaStream_t */

int vc_version(void);
const char* vc_last_error(void);
/* number of kernels this library has launched so far in this process (bench.py's gpu_launches) */
long long vc_launch_count(void);
/* BatchNorm backward as ONE cooperative launch (reduction, grid-wide barrier, apply; default on) or as two launches (0). */
int vc_set_bn_fused(int enable);
/* BatchNorm + ReLU of the tensor-core conv forward inside the conv's own launch (1, the default; cooperative: conv, grid-wide
 * barrier, apply) or as a separate apply kernel (0).  Read when a forward is enqueued (a captured graph keeps its choice). */
int vc_set_conv_bn_fused(int enable);
/* Tensor-core conv kernel selector: accepts 1 (the persistent kernel, csrc/conv_tc2.cu, the only one); else VC_ERR_INVALID. */
int vc_set_tc_variant(int variant);
/* A/B aid for the persistent tensor-core conv kernel (conv_tc2.cu): CTAs per SM, 0 = automatic (two when each still gets a
 * ring of >= 2 stages in half the shared memory), 1 or 2 = forced.  The cooperative conv + BN grid keeps one CTA per SM
 * unless 2 is forced or no index kernel runs beside it (the plan executor's static mode with side streams, which enqueues
 * the whole index phase before the first feature kernel). */
int vc_conv_tc2_config(int ctas_per_sm);
/* Host-only: the shared-memory plan the persistent tensor-core conv takes for a cin -> cout layer with K offsets under the
 * current vc_conv_tc2_config, for a launch that takes BatchNorm channel sums (bn_sums != 0: the forward of a conv + BN layer,
 * whose epilogue needs a staging buffer) or not (a dgrad, a plain forward).  out[0] = ring stages, out[1] = 1 when all K
 * weight slices stay resident in shared memory (else they stream with the ring), out[2] = CTAs per SM, out[3] = dynamic
 * shared memory per CTA in bytes. */
int vc_conv_tc2_plan(int cin, int cout, int K, int bn_sums, int32_t* out);
/* The plan executor's weight-gradient launches (csrc/wgrad_tc3.cu): variant must be 1 (the only kernel); max_ctas > 0 caps
 * the CTAs of each launch, over all its passes; 0, the default: half the SMs for each pass, so that each CTA shares its
 * SM with a dgrad CTA of the main stream. */
int vc_conv_wgrad_tc3_config(int variant, int max_ctas);
/* Host-only: the grid of the tensor-core wgrad launch over n_rows output rows of a cin -> cout layer with K offsets under a
 * CTA cap of max_ctas >= 1.  out[0] = CTAs per pass (0 when n_rows is 0: nothing is launched), out[1] = passes (groups of
 * kernel offsets whose accumulators fit the registers, blockIdx.y).  out[0] * out[1] <= max_ctas whenever
 * out[1] <= max_ctas; a launch with more passes than the cap takes one CTA per pass. */
int vc_wgrad_launch_geometry(int cin, int cout, int K, int n_rows, int max_ctas, int32_t* out);

/* ------------------------------------------------------------------------------------------------
 * Rulebooks.  Replaces spconv `ops.get_indice_pairs`, reached from every conv call site:
 * spconv_backbone.py:89 (SubMConv3d), :113 (SubMConv2d on image indices built at :217-222),
 * :92-93 and :563-564 (SparseConv3d).
 * ---------------------------------------------------------------------------------------------- */

/* Submanifold: output rows == input rows.  Hash table of linearised coordinates (lowest row wins on
 * duplicate coordinates), 1 thread per (row, offset) probe, per-offset pair counts through a
 * shared-memory histogram.  ws >= vc_subm_rulebook_ws_bytes(n). */
size_t vc_subm_rulebook_ws_bytes(int n);
int vc_subm_rulebook(const int32_t* indices, int n, int ndim, int batch_size,
                     const int32_t* spatial_shape /*host[ndim]*/, const int32_t* ksize /*host[ndim]*/,
                     const int32_t* dilation /*host[ndim]*/, int32_t* nbr /*[K,n]*/,
                     int32_t* pair_num /*[K], may be NULL*/, void* ws, size_t ws_bytes, vc_stream_t stream);

/* Regular (strided) sparse conv, two phases because the output row count is data dependent.
 *   count: marks every reachable output cell in a bitmap over the OUTPUT grid and ranks it (prefix sum
 *          of popcounts) -> *n_out_dev; also writes out_shape (host).  Output rows are therefore
 *          ordered by ascending linear index, batch most significant (voxel_query_utils.py:85-91 needs
 *          batch-contiguous rows).
 *   fill : after the caller has read n_out and allocated, emits out_indices, nbr_fwd[K,n_out],
 *          nbr_bwd[K,n] (output row per input row; the dgrad table) and pair counts.
 * The same `ws` (>= vc_conv_rulebook_ws_bytes) must be passed to both calls, untouched in between. */
size_t vc_conv_rulebook_ws_bytes(int ndim, int batch_size, const int32_t* out_shape /*host[ndim]*/);
int vc_conv_out_shape(int ndim, const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                      const int32_t* padding, const int32_t* dilation, int32_t* out_shape /*host[ndim]*/);
int vc_conv_rulebook_count(const int32_t* indices, int n, int ndim, int batch_size,
                           const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                           const int32_t* padding, const int32_t* dilation,
                           int32_t* n_out_dev /*device int32[1]*/, void* ws, size_t ws_bytes, vc_stream_t stream);
int vc_conv_rulebook_fill(const int32_t* indices, int n, int ndim, int batch_size,
                          const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                          const int32_t* padding, const int32_t* dilation, int n_out,
                          int32_t* out_indices /*[n_out,1+ndim]*/, int32_t* nbr_fwd /*[K,n_out]*/,
                          int32_t* nbr_bwd /*[K,n]*/, int32_t* pair_num /*[K], may be NULL*/,
                          void* ws, size_t ws_bytes, vc_stream_t stream);

/* spconv-style `indice_pairs [2,K,n]` (-1 padded) + `indice_pair_num [K]` from a neighbour table, each
 * offset's pairs ordered by ascending output row.  Only for API parity / tests; the conv kernels
 * consume the neighbour table directly. */
int vc_pairs_from_nbr(const int32_t* nbr, int K, int n, int32_t* pairs /*[2,K,n]*/,
                      int32_t* pair_num /*[K]*/, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Convolution (output-stationary implicit gather-GEMM).  Replaces spconv `ops.indice_conv` and its
 * autograd backward for the same call sites.  fp32 in / fp32 accumulate / fp32 out.
 * Supported channel counts: cin, cout in {8,16,32,64} (SURVEY Appendix A).
 * fwd / dgrad take a workspace of vc_conv_ws_bytes(cin, cout, K) for the re-laid-out weights
 * ([K, C_in, C_out] for forward, [K, C_out, C_in] for dgrad), rebuilt on every call.
 * ---------------------------------------------------------------------------------------------- */
size_t vc_conv_ws_bytes(int cin, int cout, int K);

/* out[o, co] = sum_k sum_ci in[nbr[k,o], ci] * w[co, k, ci].
 * bn_sums (may be NULL): [2, cout] float64 accumulator the kernel ADDS the output's channel sums (sum x,
 * sum x^2) to, for the BatchNorm1d that follows every conv (spconv_backbone.py:101-105); caller zeroes it. */
int vc_conv_fwd_f32(const float* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                    int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, vc_stream_t stream);

/* din[i, ci] = sum_k sum_co dout[nbr_t[k,i], co] * w[co, kk, ci],  kk = mirror ? K-1-k : k.
 * nbr_t is the table indexed by INPUT row: the rulebook's nbr_bwd for a regular conv, or the
 * submanifold table itself with mirror=1 (valid when coordinates are unique). */
int vc_conv_dgrad_f32(const float* dout, const float* w, const int32_t* nbr_t, float* din, int n_in, int cin,
                      int cout, int K, int mirror, void* ws, size_t ws_bytes, vc_stream_t stream);

/* din[nbr[k,o], :] += dout[o, :] @ w[:, k, :]  with float atomics; din must be zeroed by the caller.
 * Needed for the 2-D image branch, whose table is many-to-one (duplicate pixel coordinates). */
int vc_conv_dgrad_scatter_f32(const float* dout, const float* w, const int32_t* nbr, float* din, int n_out,
                              int cin, int cout, int K, void* ws, size_t ws_bytes, vc_stream_t stream);

/* dw[co, k, ci] = sum_o in[nbr[k,o], ci] * dout[o, co].  Deterministic two-pass reduction.
 * ws >= vc_conv_wgrad_ws_bytes(n_out, cin, cout, K). */
size_t vc_conv_wgrad_ws_bytes(int n_out, int cin, int cout, int K);
int vc_conv_wgrad_f32(const float* in, const float* dout, const int32_t* nbr, float* dw, int n_out, int cin,
                      int cout, int K, void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * bf16 tensor-core variants of forward / dgrad / wgrad (wgmma, fp32 accumulators in registers).  Same
 * tables, fp32 weights (converted per call) and fp32 outputs; the GATHERED operand (input features for
 * forward, output gradients for dgrad) is bf16 [N, C] row major — vc_cast_f32_bf16 makes it.
 * cin, cout in {8,16,32,64} for forward, gather dgrad and wgrad; {16,32,64} for the scatter dgrad.
 * ws >= vc_conv_tc_ws_bytes(cin, cout, K) for forward and both dgrads.  err_flag (device int32, may be
 * NULL) is set non-zero if a pipeline wait ever times out (bounded wait instead of a hang); results are
 * then invalid.
 * ---------------------------------------------------------------------------------------------- */
int vc_cast_f32_bf16(const float* in, void* out_bf16, long long n_elements /* multiple of 4 */, vc_stream_t stream);
size_t vc_conv_tc_ws_bytes(int cin, int cout, int K);
int vc_conv_fwd_tc(const void* in_bf16, const float* w, const int32_t* nbr, float* out, int n_out, int cin, int cout,
                   int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* vc_conv_fwd_tc over input rows of pitch in_ld bf16 elements (>= cin, multiple of 8): `in` may be a column slice of a
 * wider matrix, as the plan executor reads an in-place concat; the other columns are never read. */
int vc_conv_fwd_tc_ld(const void* in_bf16, int in_ld, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                      int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* din[nbr[k,o], :] += dout[o, :] @ w[:, k, :] on tensor cores, for many-to-one tables (image branch); din zeroed by the
 * caller; the dout tile is contiguous, the result is scattered with 8-byte vector reductions. */
int vc_conv_dgrad_scatter_tc(const void* dout_bf16, const float* w, const int32_t* nbr, float* din, int n_out, int cin,
                             int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
int vc_conv_dgrad_tc(const void* dout_bf16, const float* w, const int32_t* nbr_t, float* din, int n_in, int cin,
                     int cout, int K, int mirror, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* dw[co,k,ci] = sum_o in[nbr[k,o],ci] * dout[o,co] on tensor cores: both operands bf16 (MN-major wgmma), 128/cin
 * kernel offsets stacked along the MMA M dimension, accumulators resident in registers across all tiles of a
 * persistent CTA, which adds them into one fp32 image with vector reductions: the summation order, and so the last
 * bits of dw, vary from run to run.  One CTA per SM for each pass of offset groups.  ws >= vc_conv_wgrad_tc_ws_bytes(...). */
size_t vc_conv_wgrad_tc_ws_bytes(int n_out, int cin, int cout, int K);
int vc_conv_wgrad_tc(const void* in_bf16, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out, int cin,
                     int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Deterministic variants (the plan executor's mode under torch.use_deterministic_algorithms): no float atomics, every
 * reduction in an order fixed by the data alone, so the results are bit-identical from run to run and for every grid
 * size / CTA cap.
 * ---------------------------------------------------------------------------------------------- */
/* Conv forward (precision 0: fp32 `in`, gather_gemm_kernel; 1: bf16 `in`, the persistent tensor-core kernel) with the
 * BatchNorm channel sums: every 128-row tile writes its float64 partial [2, cout], then the partials are added in tile
 * order into bn_sums [2, cout] (overwritten, not accumulated).  cin, cout in {8,16,32,64}.
 * ws >= vc_conv_fwd_det_ws_bytes(n_out, cin, cout, K). */
size_t vc_conv_fwd_det_ws_bytes(int n_out, int cin, int cout, int K);
int vc_conv_fwd_det(int precision, const void* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin, int cout,
                    int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* Conv forward on tensor cores followed by BatchNorm + ReLU (vc_bn_apply_relu_f32's arithmetic), as the plan executor runs
 * it: with vc_set_conv_bn_fused(1) in ONE cooperative launch (a grid-wide barrier between the conv and the apply), else the
 * conv, then the apply kernel; both give the same bits.  x [n_out, cout]: the conv's fp32 output (kept for backward);
 * y / y_bf16 (either may be NULL) at row pitches y_ld / yb_ld (multiples of 4, >= cout: a column slice of a wider matrix).
 * n_dev (optional, device int): the row count, n_out is then the capacity and the output rows [count, n_out) are zeroed.
 * deterministic: the BN sums from per-128-row-tile partials added in tile order (vc_conv_fwd_det).  cin, cout in
 * {8,16,32,64}.  ws >= vc_conv_bn_relu_tc_ws_bytes(n_out, cin, cout, K). */
size_t vc_conv_bn_relu_tc_ws_bytes(int n_out, int cin, int cout, int K);
int vc_conv_bn_relu_tc(const void* in_bf16, const float* w, const int32_t* nbr, float* x, int n_out, const int32_t* n_dev, int cin,
                       int cout, int K, int deterministic, const float* gamma, const float* beta, float* running_mean,
                       float* running_var, long long* num_batches_tracked, float momentum, float eps, int training, float* y,
                       int y_ld, void* y_bf16, int yb_ld, float* stats_out, void* ws, size_t ws_bytes, int32_t* err_flag,
                       vc_stream_t stream);
/* vc_conv_wgrad_tc with the rows split into 32 runs of consecutive 128-row tiles (from n_out alone); a CTA claims whole
 * runs, each run's sum goes to its own fp32 image, and the images are added in run order.  The CTA cap of
 * vc_conv_wgrad_tc3_config applies (0: one CTA per SM for each pass, as vc_conv_wgrad_tc).  ws >= vc_conv_wgrad_tc_det_ws_bytes(...) (32 images). */
size_t vc_conv_wgrad_tc_det_ws_bytes(int n_out, int cin, int cout, int K);
int vc_conv_wgrad_tc_det(const void* in_bf16, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out, int cin,
                         int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* vc_conv_wgrad_tc_det over input rows of pitch in_ld bf16 elements (>= cin, multiple of 8), as vc_conv_fwd_tc_ld. */
int vc_conv_wgrad_tc_det_ld(const void* in_bf16, int in_ld, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out,
                            int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream);
/* vc_bn_relu_bwd_f32 with (sum g, sum g*xhat) reduced per 512-row chunk into float64 partials (ws) and added in chunk order
 * (vc_set_bn_fused selects one cooperative launch or two, with the same result).  ws >= vc_bn_bwd_det_ws_bytes(n, c). */
size_t vc_bn_bwd_det_ws_bytes(int n, int c);
int vc_bn_relu_bwd_det_f32(const float* dy, const float* x, const float* gamma, const float* stats, float* dx, void* dx_bf16,
                           float* dgamma, float* dbeta, int n, int c, int training, void* ws, size_t ws_bytes, vc_stream_t stream);
/* vc_subm_rulebook plus rep [n]: the lowest row at each row's own coordinate (the row itself when it lies outside the grid)
 * — the groups of rows the many-to-one 2-D tables merge. */
int vc_subm_rulebook_rep(const int32_t* indices, int n, int ndim, int batch_size, const int32_t* spatial_shape,
                         const int32_t* ksize, const int32_t* dilation, int32_t* nbr, int32_t* pair_num, int32_t* rep, void* ws,
                         size_t ws_bytes, vc_stream_t stream);
/* Input gradient of a many-to-one submanifold table (odd kernel sizes) in gather form, OVERWRITING din [n, cin]:
 *   din[i] = W_c^T dout[i] + [rep[i] == i] sum_{k != c} W_k^T S[p(i) - delta_k],
 * S[p] = the sum of dout over the rows at pixel p in ascending row order — equal to vc_conv_dgrad_scatter_* up to the
 * summation order.  The rows are grouped by rep with integer atomics, each group sorted, and the result comes from one
 * mirrored gather dgrad over [dout; S] (fp32: gather_gemm_kernel; tc: bf16 dout and S, the persistent tensor-core kernel).
 * n_dev (device int32, may be NULL): rows below it are valid, n is the capacity (table tail -1, din tail 0).
 * ws >= vc_conv_dgrad_gather2d_ws_bytes(n, cin, cout, K). */
size_t vc_conv_dgrad_gather2d_ws_bytes(int n, int cin, int cout, int K);
int vc_conv_dgrad_gather2d_f32(const float* dout, const float* w, const int32_t* nbr, const int32_t* rep, float* din, int n,
                               const int32_t* n_dev, int cin, int cout, int K, void* ws, size_t ws_bytes, vc_stream_t stream);
int vc_conv_dgrad_gather2d_tc(const void* dout_bf16, const float* w, const int32_t* nbr, const int32_t* rep, float* din, int n,
                              const int32_t* n_dev, int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag,
                              vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * BatchNorm1d(eps, momentum) + ReLU over the active rows.  Replaces the `norm_fn(out_channels)`,
 * `nn.ReLU()` members of every `spconv.SparseSequential` (spconv_backbone.py:101-105, :160, :561-567).
 * ---------------------------------------------------------------------------------------------- */

/* y = relu(BN(x)) in one pass.  training != 0: batch statistics from `sums` (the [2,c] float64 accumulator the conv
 * filled): mean, biased var -> scale = gamma*invstd, shift = beta - mean*scale; running_mean / running_var updated in
 * place with the unbiased variance and *num_batches_tracked (int64, may be NULL) incremented — torch.nn.BatchNorm1d
 * semantics.  training == 0: statistics from the running buffers.  stats_out [4,c] = scale, shift, mean, invstd is
 * kept for backward.  y_bf16 (may be NULL): bf16 shadow of y = the next conv's tensor-core operand.  In place
 * (y == x) allowed.  The ReLU is torch.relu's: a NaN stays NaN. */
int vc_bn_apply_relu_f32(const float* x, const double* sums, int n_rows, int c, const float* gamma, const float* beta,
                         float* running_mean, float* running_var, long long* num_batches_tracked, float momentum,
                         float eps, int training, float* y, void* y_bf16, float* stats_out, int relu, vc_stream_t stream);
/* Backward of y = relu(gamma*(x-mean)*invstd + beta), stats = the forward's stats_out:
 *   g = dy * !(y <= 0) (a NaN y passes dy, as torch's threshold_backward); dbeta = sum g; dgamma = sum g*xhat;
 *   train: dx = gamma*invstd*(g - dbeta/n - xhat*dgamma/n);   eval: dx = gamma*invstd*g.
 * bsums: [2,c] float64 scratch accumulator, zeroed by the caller.  dx_bf16 (may be NULL): bf16 shadow of dx. */
int vc_bn_relu_bwd_f32(const float* dy, const float* x, const float* y, const float* gamma, const float* stats,
                       float* dx, void* dx_bf16, float* dgamma, float* dbeta, int n, int c, int training,
                       double* bsums, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Voxel index -> image pixel index.  Replaces `index2uv` + `index2points` + the per-sample
 * `X_TRANS.backward_with_param` / `Calibration.lidar_to_rect_cuda` / `rect_to_img_cuda` loop
 * (spconv_backbone.py:8-24, :54-83; X_transform.py:139-154; calibration_kitti.py:120-153).
 * params: [batch_size, 28] float32 per sample:
 *   [0..11]  M = V2C^T @ R0^T  (4x3, row major)        [12..19] first two columns of P2^T (4x2)
 *   [20] has_transform  [21] scale  [22] flip  [23] cos(-rot)  [24] sin(-rot)  [25..27] unused
 * grid: 6 floats (vx, vy, vz, min_x, min_y, min_z) = voxel size * stride and range min + half voxel.
 * uv_out [n,3] int32 = (batch, clamp(u,0,u_max-1)/stride, clamp(v,0,v_max-1)/stride).
 * ---------------------------------------------------------------------------------------------- */
int vc_index2uv(const int32_t* indices /*[n,4] b,z,y,x*/, int n, int batch_size, const float* params,
                const float* grid /*host[6]*/, int stride, int u_max, int v_max, int32_t* uv_out,
                vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Hash-grid voxelisation + MeanVFE.  Replaces `VoxelGeneratorWrapper.generate` -> spconv
 * `Point2VoxelCPU3d.point_to_voxel` (pcdet/datasets/processor/data_processor.py:43-59, called :156,:173) and
 * `MeanVFE.forward` (pcdet/models/backbones_3d/vfe/mean_vfe.py:39-58) with identical results.
 * points [n, 1+c] float32 rows (batch, x, y, z, features...), samples contiguous in ascending batch order (what
 * `collate_batch` produces, dataset.py:349-353).  Per sample: voxels in order of first appearance, at most max_voxels,
 * at most max_points (<= 8) points per voxel in point order.  Outputs (capacity batch_size*max_voxels rows):
 * out_features [*, c] = per-voxel mean (last channel = max over the zero-padded slots if vfe_max_last),
 * out_coords [*, 4] = (b, z, y, x), out_num [*], optional out_voxels [*, max_points, c] (caller zeroes), *n_out_dev.
 * pc_range host[6] = (x0,y0,z0,x1,y1,z1), voxel_size host[3].  ws >= vc_voxelize_ws_bytes(...).
 * ---------------------------------------------------------------------------------------------- */
size_t vc_voxelize_ws_bytes(int n_points, int batch_size, int max_points);
int vc_voxelize_mean(const float* points, int n_points, int c, int batch_size, const float* pc_range,
                     const float* voxel_size, int max_points, int max_voxels, int vfe_max_last, float* out_features,
                     int32_t* out_coords, int32_t* out_num, float* out_voxels /*may be NULL*/, int32_t* n_out_dev,
                     void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * StVD input point discard.  Replaces `DatasetTemplate.partition` + `DatasetTemplate.input_point_discard`
 * (pcdet/datasets/dataset.py:120-189; applied to the virtual points of every frame at :275-290): bin_num range bins
 * along x of width max_dis/bin_num (last bin open-ended, x < 0 / NaN in no bin), emitted far -> near, the nearest bins
 * randomly subsampled.  The random draws stay on the host so that they come from the same numpy generator, in the same
 * order, as the reference's (virconv_b200/preprocess.py); the device does the order-preserving partition and the gather.
 *   vc_stvd_partition: points [n, c] fp32 (x in column 0) -> totals_dev[16] = points per bin, and in ws the per-bin point
 *                      lists (original order inside a bin).
 *   vc_stvd_gather   : segs host [n_seg][4] = (bin, out_base, count, sel_base): output rows [out_base, out_base+count)
 *                      are the bin's points with in-bin ranks sel_dev[sel_base + r] (sel_base < 0: rank r itself).
 * ws >= vc_stvd_ws_bytes(n), the same buffer for both calls.
 * ---------------------------------------------------------------------------------------------- */
size_t vc_stvd_ws_bytes(int n_points);
int vc_stvd_partition(const float* points, int n, int c, int bin_num, double max_dis, int32_t* totals_dev /*[16]*/,
                      void* ws, size_t ws_bytes, vc_stream_t stream);
int vc_stvd_gather(const float* points, int n, int c, const int32_t* segs /*host*/, int n_seg, const int32_t* sel_dev,
                   float* out /*[n_out, c]*/, int n_out, void* ws, size_t ws_bytes, vc_stream_t stream);

/* The input front end with the draws on the device, no host read (graph-capturable), csrc/stvd.cu.  points [cap, w] fp32
 * collated rows (b, x, y, z, ..., indicator), scenes contiguous and ascending, *n_dev (may be NULL: cap) valid rows;
 * indicator 1 = virtual, 2 = LiDAR, anything else and b outside [0, batch_size) is dropped.  Per scene, the virtual points go
 * through the StVD input discard (bin_num bins of width max_dis / bin_num, the reference's position / per_bin arithmetic in
 * float64; a subsampled bin keeps its `per_bin` smallest (u, row), u = word 0 of Philox4x32-10 with counter
 * (row, 0, 1, draw) and key (seed & 0xffffffff, seed >> 32), seed = *seed_dev, in row order), then
 *   later_fusion 0: out_points = [LiDAR, kept virtual bins far -> near] per scene, column 4 (intensity) divided by 10;
 *   later_fusion 1: out_points = LiDAR, out_mm = kept virtual bins far -> near;
 * rows outside pc_range (host[6], x and y, bounds inclusive) dropped; shuffle != 0: each scene's block of each stream
 * permuted by a Philox-keyed Feistel bijection (counter domain 2).  src_* (may be NULL) = the input row of every output row.
 * n_out_dev[2] = rows written per stream; tails: batch column -1, zeros, source -1.  status_dev[B]: bit 0 = the scene has
 * no virtual point (the reference divides by zero); bit 1 = the scenes of the batch are not contiguous and ascending, and
 * nothing was kept.  *overflow_dev = max(*overflow_dev, rows that did not fit).
 * ws >= vc_stvd_input_ws_bytes(cap, batch_size).  A memset and 22 launches. */
size_t vc_stvd_input_ws_bytes(int cap, int batch_size);
int vc_stvd_input_front_end(const float* points, int cap, const int32_t* n_dev /*may be NULL*/, int w, int batch_size, int bin_num,
                            double max_dis, double rate, const float* pc_range /*host[6]*/, int later_fusion, int shuffle,
                            const int64_t* seed_dev, int draw, float* out_points, int32_t* src_points /*may be NULL*/,
                            int cap_points, float* out_mm, int32_t* src_mm /*may be NULL*/, int cap_mm,
                            int32_t* n_out_dev /*[2]*/, int32_t* status_dev /*[B]*/, int32_t* overflow_dev /*[1], may be NULL*/,
                            void* ws, size_t ws_bytes, vc_stream_t stream);

/* StVD layer discard (`layer_voxel_discard`, spconv_backbone.py:134-147) with the subset drawn on the device, no host read
 * (graph-capturable), csrc/stvd_layer.cu.  Over n rows (n_dev != NULL: *n_dev valid rows of a capacity-n buffer) at discard
 * site `site`: k = int(n_valid * (1 - rate)) evaluated in float64; the kept rows are the k rows with the smallest (u_i, i),
 * u_i = keys[i] (keys != NULL, uint32) or word 0 of Philox4x32-10 with counter (i, site, 0, 0) and key
 * (seed & 0xffffffff, seed >> 32), seed = *seed_dev (int64).  -> keep [n] = the kept rows in ascending order, tail -1;
 * *kept_dev = k; pos [n] (may be NULL) = a row's position in keep or -1.  The same result on every run.
 * ws >= vc_stvd_layer_keep_ws_bytes(n).  A memset and seven launches. */
size_t vc_stvd_layer_keep_ws_bytes(int cap);
int vc_stvd_layer_keep(const uint32_t* keys /*may be NULL*/, const int64_t* seed_dev /*may be NULL with keys*/, int site, int n,
                       const int32_t* n_dev /*may be NULL*/, double rate, int32_t* keep, int32_t* kept_dev /*[1]*/,
                       int32_t* pos /*may be NULL*/, void* ws, size_t ws_bytes, vc_stream_t stream);

/* `generate_voxel2pinds` (pcdet/utils/spconv_utils.py:13-21): dense [B, *spatial_shape] int32 map voxel -> row, -1 where
 * empty (the RoI head's look-up table, ted_head.py:527,625). */
int vc_voxel2pinds(const int32_t* indices, int n, int ndim, int batch_size, const int32_t* spatial_shape, int32_t* out,
                   vc_stream_t stream);

/* `SparseConvTensor.dense()` (height_compression.py:29): out [B, C, *shape] must be zeroed by the caller. */
int vc_dense_f32(const float* features, const int32_t* indices, int n, int c, int ndim, int batch_size,
                 const int32_t* spatial_shape, float* out, vc_stream_t stream);
/* Gradient of dense(): dfeatures[n, c] = dout[b, c, coords]. */
int vc_dense_bwd_f32(const float* dout, const int32_t* indices, int n, int c, int ndim, int batch_size,
                     const int32_t* spatial_shape, float* dfeatures, vc_stream_t stream);

/* Row-counted forms of the three calls above for a static-mode (capacity-sized) tensor: `cap` rows of indices / features,
 * n_dev (device int32[1]) the valid ones.  Rows at or past *n_dev are skipped (their -1 index tail is never used as an
 * address); the dense() gradient of those rows is zero.  Otherwise the same results as vc_voxel2pinds / vc_dense_f32 /
 * vc_dense_bwd_f32 on the valid rows. */
int vc_voxel2pinds_rows(const int32_t* indices, int cap, const int32_t* n_dev, int ndim, int batch_size,
                        const int32_t* spatial_shape, int32_t* out, vc_stream_t stream);
int vc_dense_rows_f32(const float* features, const int32_t* indices, int cap, const int32_t* n_dev, int c, int ndim,
                      int batch_size, const int32_t* spatial_shape, float* out, vc_stream_t stream);
int vc_dense_rows_bwd_f32(const float* dout, const int32_t* indices, int cap, const int32_t* n_dev, int c, int ndim,
                          int batch_size, const int32_t* spatial_shape, float* dfeatures, vc_stream_t stream);

/* Test-time x-batching of the ROT_NUM transformed copies (spconv_backbone.py:339-471, csrc/xbatch.cu), no host read:
 *   vc_xbatch_pack : R copies (host arrays of R device pointers: features [caps[i], c] fp32, coordinates [caps[i], 4] int32
 *                    (b, z, y, x), row counts n_dev[i] int32[1]) -> out [cap_out >= sum(caps)]: the valid rows of copy 0,
 *                    copy 1, ... in order (= torch.cat of the exact rows) with x += i * W; zero feature / -1 coordinate
 *                    tail; *n_out_dev = the total.  One launch.
 *   vc_xbatch_split: the device form of `decompose_tensor` (:314-337).  A published tensor (features [cap, c] fp32, c in
 *                    {16, 32, 64} else VC_ERR_UNSUPPORTED; indices [cap, 4] int32; *n_dev valid rows) of a grid of x extent
 *                    Wt -> R outputs of capacity cap (host arrays of R device pointers).  q = Wt / 4; output i = the rows
 *                    with i*q < x < (i+1)*q (strict: the x == i*q column is in no copy, :325) in the parent's order, with
 *                    x -= i*q; zero feature / -1 index tail; *n_out_dev[i] its rows.  ws >= vc_xbatch_split_ws_bytes(cap, R).
 *                    Three launches (tile counts of every copy, one scan, ballot-ranked emit).
 * R outside [1, 4] -> VC_ERR_INVALID (the reference's x-batching factor is 4, :360). */
int vc_xbatch_pack(const float* const* features, const int32_t* const* coords, const int32_t* const* n_dev,
                   const int32_t* caps /*host [R]*/, int R, int c, int W, int cap_out, float* out_features, int32_t* out_coords,
                   int32_t* n_out_dev, vc_stream_t stream);
size_t vc_xbatch_split_ws_bytes(int cap, int R);
int vc_xbatch_split(const float* features, const int32_t* indices, int cap, const int32_t* n_dev, int c, int Wt, int R,
                    float* const* out_features, int32_t* const* out_indices, int32_t* const* n_out_dev, void* ws, size_t ws_bytes,
                    vc_stream_t stream);

/* NRConv channel concat (spconv_backbone.py:227): out[:, :ca] = a, out[:, ca:] = b, plus an optional bf16 shadow. */
int vc_cat2_f32(const float* a, const float* b, float* out, void* out_bf16 /*may be NULL*/, int n, int ca, int cb,
                vc_stream_t stream);

/* Mean over the valid rows of a [cap_rows, c] fp32 matrix (c % 4 == 0): n_dev (device int32[1], may be NULL: all cap_rows
 * rows) is the row count.  Deterministic: float64 partials added in a fixed order that depends on (cap_rows, c) only.
 * ws >= vc_masked_mean_ws_bytes().  The backward writes the whole [cap_rows, c] gradient: g / (n*c) on the first n rows,
 * zeros on the rest (g: device float32[1]). */
size_t vc_masked_mean_ws_bytes(void);
int vc_masked_mean_f32(const float* x, long long cap_rows, int c, const int32_t* n_dev, float* out /*device [1]*/, void* ws,
                       size_t ws_bytes, vc_stream_t stream);
int vc_masked_mean_bwd_f32(const float* g, long long cap_rows, int c, const int32_t* n_dev, float* dx, vc_stream_t stream);

/* Row gather for StVD layer discard (spconv_backbone.py:134-147): out[r] = in[rows[r]]. */
int vc_gather_rows(const void* in, const int32_t* rows, void* out, int n_rows, int row_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Voxel-RoI pooling primitives: the stacked pointnet2 ops the RoI head runs on x_conv3 / x_conv4 (ted_head.py:496-552).
 * Same arguments, layouts and results as the reference launchers they replace:
 *   vc_voxel_query       <- voxel_query_kernel_launcher_stack (pointnet2_stack/src/voxel_query_gpu.cu:92-113) plus the
 *                           `idx[empty_ball_mask] = 0` of VoxelQuery.forward (voxel_query_utils.py:38-39): idx [M, nsample]
 *                           = the first nsample rows found scanning the (2r+1)^3 cells around new_coords (b,z,y,x) in
 *                           z-major order whose centre xyz lies within `radius` of new_xyz, padded with the first hit;
 *                           empty_mask [M] uint8 = 1 and idx row = 0 where nothing was found.  point_indices: dense
 *                           [B, R1, R2, R3] voxel -> row map (vc_voxel2pinds).
 *   vc_group_points      <- group_points_kernel_launcher_stack (group_points_gpu.cu:106-125): out [M, C, nsample] =
 *                           features[start(batch of m) + idx[m, s], c], idx batch-local.
 *   vc_group_points_grad <- group_points_grad_kernel_launcher_stack (:47-68): grad_features (zeroed by the caller)
 *                           += grad_out, float atomics.
 * ---------------------------------------------------------------------------------------------- */
int vc_voxel_query(int M, int R1, int R2, int R3, int nsample, float radius, int z_range, int y_range, int x_range,
                   const float* new_xyz, const float* xyz, const int32_t* new_coords, const int32_t* point_indices,
                   int32_t* idx, unsigned char* empty_mask, vc_stream_t stream);
int vc_group_points(int B, int M, int C, int nsample, const float* features, const int32_t* features_batch_cnt,
                    const int32_t* idx, const int32_t* idx_batch_cnt, float* out, vc_stream_t stream);
int vc_group_points_grad(int B, int M, int C, int N, int nsample, const float* grad_out, const int32_t* idx,
                         const int32_t* idx_batch_cnt, const int32_t* features_batch_cnt, float* grad_features,
                         vc_stream_t stream);
/* Deterministic form of vc_group_points_grad (rule D4 of csrc/voxel_pool.cu): no float atomics; grad_features [N, C] is
 * written (every row, zero where no slot points): grad_features[row, c] = the fp32 sum over the slots (m, s) of that global
 * row, in ascending (m, s), of grad_out[m, c, s].  The same bits on every run, whatever the grid.
 * ws >= vc_group_points_grad_det_ws_bytes(M, N, nsample).  No host read. */
size_t vc_group_points_grad_det_ws_bytes(int M, int N, int nsample);
int vc_group_points_grad_det(int B, int M, int C, int N, int nsample, const float* grad_out, const int32_t* idx,
                             const int32_t* idx_batch_cnt, const int32_t* features_batch_cnt, float* grad_features, void* ws,
                             size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Fused voxel-RoI grid pooling: one grouper of `NeighborVoxelSAModuleMSG.forward` (voxel_pool_modules.py:70-130) between
 * `mlps_in[k]` and `mlps_out[k]` — query, grouping, position MLP Conv2d(3->C) + BatchNorm2d, add, ReLU, max over the
 * samples — without any [M, C, nsample] tensor.  csrc/voxel_pool.cu states the rules.  C in {16, 32, 64} and
 * nsample <= VC_VOXEL_POOL_MAX_NSAMPLE, anything else -> VC_ERR_UNSUPPORTED.  No call reads the device on the host.
 *   vc_voxel_pool_query <- vc_voxel_query (same idx [M, nsample] of GLOBAL rows and empty_mask [M]), plus, when moments is
 *                          not NULL, moments[9] (float64, zeroed by the caller) += sum over all M * nsample slots of
 *                          r = xyz[idx] - new_xyz (zero for empty balls): rx, ry, rz, rx rx, rx ry, rx rz, ry ry, ry rz, rz rz.
 *   vc_voxel_pool_bn_fold  one launch, one thread per channel: the position branch's BatchNorm2d over n = M * nsample
 *                          slots.  Train mode: mean = W E[r], biased var = diag(W Cov(r) W^T) from the moments,
 *                          *num_batches_tracked += 1, running stats updated (momentum < 0: cumulative average, unbiased
 *                          var n/(n-1)); eval mode: the running stats.  -> scale / shift [C] fp32 of the folded affine map,
 *                          stat [C, 2] float64 = mean, invstd.  w_pos [C, 3].
 *   vc_voxel_pool_bn_grad  one launch: dw [C, 3], dgamma, dbeta [C] fp32 from sums (vc_voxel_pool_bwd), the moments (train
 *                          mode: the BN coupling term over all n slots) and stat.
 *   vc_voxel_pool_fwd   <- pooled [M, C] fp32 = max_s ReLU(features_in[idx[m, s]] + scale * (w_pos r) + shift) and
 *                          argmax [M, C] uint8 = the first slot attaining it; w_pos [C, 3], scale / shift [C] = the
 *                          BatchNorm2d of the position branch folded into an affine map.
 *   vc_voxel_pool_bwd   <- grad_features_in [N, C] (accumulated, float atomics) += grad_pooled * [pooled > 0] at the argmax
 *                          row of non-empty balls; sums [C, 4] (float64, zeroed by the caller) += per channel sum dy and
 *                          sum dy * r (x, y, z) over the argmax slots, dy = grad_pooled * [pooled > 0].
 * ---------------------------------------------------------------------------------------------- */
#define VC_VOXEL_POOL_MAX_NSAMPLE 64
int vc_voxel_pool_query(int M, int R1, int R2, int R3, int nsample, float radius, int z_range, int y_range, int x_range,
                        const float* new_xyz, const float* xyz, const int32_t* new_coords, const int32_t* point_indices,
                        int32_t* idx, unsigned char* empty_mask, double* moments /*may be NULL*/, vc_stream_t stream);
int vc_voxel_pool_bn_fold(int C, long long n, int training, const double* moments /*NULL in eval mode*/, const float* w_pos,
                          const float* gamma, const float* beta, float* running_mean, float* running_var,
                          long long* num_batches_tracked, double eps, double momentum, float* scale, float* shift,
                          double* stat, vc_stream_t stream);
int vc_voxel_pool_bn_grad(int C, long long n, int training, const double* sums, const double* moments, const float* w_pos,
                          const float* gamma, const double* stat, float* dw, float* dgamma, float* dbeta, vc_stream_t stream);
/* SyncBatchNorm2d as the position branch's BatchNorm over several ranks (train mode): the caller all-reduces
 * [moments (9), n] (float64, n = the rank's M * nsample) and passes the sum as moments10 — statistics and the running update
 * then come from the union of the ranks' slots.  vc_voxel_pool_bn_grad_sync: sums and moments are the rank's own, gsums
 * [C, 4] the all-reduced sums and n_glob the all-reduced slot count (moments10[9]); the coupling term of dw takes the global
 * mean of dy and of dy*xhat, dgamma / dbeta stay local (torch's SyncBatchNorm backward). */
int vc_voxel_pool_bn_fold_sync(int C, int training, const double* moments10, const float* w_pos, const float* gamma,
                               const float* beta, float* running_mean, float* running_var, long long* num_batches_tracked,
                               double eps, double momentum, float* scale, float* shift, double* stat, vc_stream_t stream);
int vc_voxel_pool_bn_grad_sync(int C, const double* n_glob, const double* sums, const double* gsums, const double* moments,
                               const float* w_pos, const float* gamma, const double* stat, float* dw, float* dgamma,
                               float* dbeta, vc_stream_t stream);
int vc_voxel_pool_fwd(int M, int C, int nsample, const float* features_in, const float* xyz, const float* new_xyz,
                      const int32_t* idx, const unsigned char* empty_mask, const float* w_pos, const float* scale,
                      const float* shift, float* pooled, unsigned char* argmax, vc_stream_t stream);
int vc_voxel_pool_bwd(int M, int C, int N, int nsample, const float* grad_pooled, const float* pooled,
                      const unsigned char* argmax, const int32_t* idx, const unsigned char* empty_mask, const float* xyz,
                      const float* new_xyz, float* grad_features_in, double* sums, vc_stream_t stream);
/* Deterministic mode (rules D1-D3 of csrc/voxel_pool.cu): no float atomics, every sum in an order fixed by the data.
 *   vc_voxel_pool_query_det  <- vc_voxel_pool_query with moments[9] WRITTEN (not accumulated; required) from per-256-point
 *                               partials added in chunk order.  ws >= vc_voxel_pool_query_det_ws_bytes(M).
 *   vc_voxel_pool_bwd_det    <- grad_features_in [N, C] WRITTEN (every row; an fp32 sum per row in ascending query point over
 *                               the inverse slot map) and sums [C, 4] WRITTEN (per-256-point partials in chunk order).
 *                               ws >= vc_voxel_pool_bwd_det_ws_bytes(M, C, N, nsample); N <= 2^20 rows.
 *   vc_voxel_pool_det_config    caps the CTAs of their grid-stride kernels (0, the default: 8 per SM); the results do not
 *                               depend on it. */
int vc_voxel_pool_det_config(int max_ctas);
size_t vc_voxel_pool_query_det_ws_bytes(int M);
int vc_voxel_pool_query_det(int M, int R1, int R2, int R3, int nsample, float radius, int z_range, int y_range, int x_range,
                            const float* new_xyz, const float* xyz, const int32_t* new_coords, const int32_t* point_indices,
                            int32_t* idx, unsigned char* empty_mask, double* moments, void* ws, size_t ws_bytes,
                            vc_stream_t stream);
size_t vc_voxel_pool_bwd_det_ws_bytes(int M, int C, int N, int nsample);
int vc_voxel_pool_bwd_det(int M, int C, int N, int nsample, const float* grad_pooled, const float* pooled,
                          const unsigned char* argmax, const int32_t* idx, const unsigned char* empty_mask, const float* xyz,
                          const float* new_xyz, float* grad_features_in, double* sums, void* ws, size_t ws_bytes,
                          vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Rotated-box IoU and NMS of the detector heads: the reference's `iou3d_nms_cuda` extension (pcdet/ops/iou3d_nms), whose
 * rules csrc/iou3d_nms.cu states.  Boxes are (x, y, z, dx, dy, dz, heading) fp32; the pairwise calls take [n, 7] row-major.
 *   vc_boxes_overlap_bev  <- boxesoverlapLauncher (iou3d_nms_kernel.cu:378-387): out [na, nb] = BEV intersection area.
 *   vc_boxes_iou_bev      <- boxesioubevLauncher (:389-398): out [na, nb] = BEV IoU.
 *   vc_boxes_iou3d        <- boxesoverlapLauncher + the torch glue of iou3d_nms_utils.boxes_iou3d_gpu (:67-100), fused:
 *                            out [na, nb] = 3-D IoU.
 *   vc_boxes_iou_bev_host <- boxes_iou_bev_cpu (iou3d_cpu.cpp:232-252): HOST pointers, no GPU needed; bit-identical to
 *                            vc_boxes_iou_bev (shared geometry code).
 *   vc_nms_boxes          <- nmsLauncher / nmsNormalLauncher plus the host side of nms_gpu / nms_normal_gpu
 *                            (iou3d_nms.cpp:90-186), batched over segments and without a host read:
 *                            boxes [batch, n_max, ld] (ld >= 7, columns 0..6 used; each segment sorted by descending
 *                            score), counts [batch] device int32 = valid rows per segment (clamped to [0, n_max]),
 *                            normal != 0: axis-aligned IoU (heading ignored).  Box j is dropped when an earlier kept box
 *                            has IoU > thresh with it; at most post_max boxes are kept.  keep [batch, post_max] int32 =
 *                            kept row indices in order, tail -1; num_keep [batch] int32.  Two launches (upper-triangle
 *                            suppression mask into ws, then the greedy pass on the device), graph-capturable.
 *                            ws >= vc_nms_ws_bytes(batch, n_max); n_max > VC_NMS_MAX_BOXES -> VC_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
#define VC_NMS_MAX_BOXES 16384
int vc_boxes_overlap_bev(const float* boxes_a, int na, const float* boxes_b, int nb, float* out, vc_stream_t stream);
int vc_boxes_iou_bev(const float* boxes_a, int na, const float* boxes_b, int nb, float* out, vc_stream_t stream);
int vc_boxes_iou3d(const float* boxes_a, int na, const float* boxes_b, int nb, float* out, vc_stream_t stream);
int vc_boxes_iou_bev_host(const float* boxes_a /*host*/, int na, const float* boxes_b /*host*/, int nb, float* out /*host*/);
size_t vc_nms_ws_bytes(int batch, int n_max);
int vc_nms_boxes(const float* boxes, int batch, int n_max, int ld, const int32_t* counts, float thresh, int normal,
                 int post_max, int32_t* keep, int32_t* num_keep, void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Anchor-head targets of the RPN (AnchorHeadSingle), whose rules csrc/anchor_targets.cu states.  No call reads the
 * device on the host; both are graph-capturable.
 *   vc_anchor_mask    <- AnchorHeadSingle.get_anchor_mask (anchor_head_single.py:75-115): points [n_points, ld] fp32
 *                        (column 1 = x, column 2 = y, all scenes together), min_x / min_y = point_cloud_range[0:2],
 *                        inv_stride = 1.0f / float(round(voxel_size * 80)) -> mask [H, W] uint8 (0 / 1).  coarse
 *                        [H/10 * W/10] uint8 is scratch, zeroed by the caller.  Two launches.
 *   vc_anchor_targets <- AxisAlignedTargetAssigner.assign_targets (axis_aligned_target_assigner.py:46-243; POS_FRACTION
 *                        < 0, MATCH_HEIGHT False, not multihead, NORM_BY_NUM_EXAMPLES False) for all scenes and anchor
 *                        sets in one grid: anchors [N, 7] in the output order with anchor_set [N] int32 in [0, n_sets);
 *                        matched / unmatched [n_sets] HOST fp32 thresholds; gt [B, M, ld] (ld >= 8, class in the last
 *                        column); name_sets [n_names] HOST = bitmask of the anchor sets whose class name is class_names[k]
 *                        -> labels [B, N] int32, targets [B, N, 7], reg_weights [B, N], gt_ious [B, N] fp32, every element
 *                        written.  ws >= vc_anchor_targets_ws_bytes(B, n_sets, M); M > VC_ANCHOR_MAX_GT ->
 *                        VC_ERR_UNSUPPORTED.  A memset and two launches.
 * ---------------------------------------------------------------------------------------------- */
#define VC_ANCHOR_MAX_GT 512
#define VC_ANCHOR_MAX_SETS 8
#define VC_ANCHOR_MAX_NAMES 32
int vc_anchor_mask(const float* points, int n_points, int ld, float min_x, float min_y, float inv_stride, int H, int W,
                   unsigned char* coarse, unsigned char* mask, vc_stream_t stream);
size_t vc_anchor_targets_ws_bytes(int B, int n_sets, int M);
int vc_anchor_targets(const float* anchors, const int32_t* anchor_set, int N, int n_sets, const float* matched /*host*/,
                      const float* unmatched /*host*/, const float* gt, int B, int M, int ld, const int32_t* name_sets /*host*/,
                      int n_names, int32_t* labels, float* targets, float* reg_weights, float* gt_ious, void* ws,
                      size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * RoI target sampling of the two-stage head (TEDMHead), whose rules csrc/roi_targets.cu states.  No host read;
 * graph-capturable.
 *   vc_roi_targets <- ProposalTargetLayer.forward (roi_heads/target_assigner/proposal_target_layer.py:32-353;
 *                     SAMPLE_ROI_BY_EACH_CLASS True, CLS_SCORE_TYPE roi_iou_x) plus the canonical transform of
 *                     RoIHeadTemplate.assign_targets (roi_head_template.py:133-158), all scenes in one call:
 *                     rois [B, M, ldr] (ldr >= 7), roi_scores [B, M] fp32, roi_labels [B, M] int64, gt [B, G, ldg]
 *                     (ldg >= 8, class in the last column); per-class HOST float64 thresholds [n_cls] as the config
 *                     gives them (REG_FG_THRESH, CLS_FG_THRESH, CLS_BG_THRESH; HARD_SAMPLING_THRESH / _RATIO, read only
 *                     with hard_sampling != 0), CLS_BG_THRESH_LO, R = ROI_PER_IMAGE, F = int(round(FG_RATIO * R)),
 *                     HARD_BG_RATIO; uniforms in [0, 1): u_fg [B, ld_ufg >= max(M, R)], u_bg [B, R], u_hs [n_cls]
 *                     -> rois [B, R, ldr], gt_of_rois_src / gt_of_rois [B, R, ldg], gt_iou_of_rois / roi_scores
 *                     [B, R] fp32, roi_labels / reg_valid_mask [B, R] int64, rcnn_cls_labels [B, R] fp32, every element
 *                     written; status [1] int32 = number of scenes with neither foreground nor background RoIs (the
 *                     reference raises there; their rows are zero).  ws >= vc_roi_targets_ws_bytes(B, M, G) (G does
 *                     not change the size).  M > VC_ROI_TARGETS_MAX_ROIS, G > VC_ROI_TARGETS_MAX_GT or
 *                     ldg > VC_ROI_TARGETS_MAX_LDG -> VC_ERR_UNSUPPORTED.  A memset and two launches.
 * ---------------------------------------------------------------------------------------------- */
#define VC_ROI_TARGETS_MAX_ROIS 4096
#define VC_ROI_TARGETS_MAX_GT 512
#define VC_ROI_TARGETS_MAX_LDG 16
#define VC_ROI_TARGETS_MAX_CLASSES 16
size_t vc_roi_targets_ws_bytes(int B, int M, int G);
int vc_roi_targets(const float* rois, const float* roi_scores, const int64_t* roi_labels, int B, int M, int ldr,
                   const float* gt, int G, int ldg, int n_cls, const double* reg_fg /*host*/, const double* cls_fg /*host*/,
                   const double* cls_bg /*host*/, double cls_bg_lo, const double* hs_thresh /*host*/,
                   const double* hs_ratio /*host*/, int hard_sampling, int R, int F, double hard_bg_ratio,
                   const float* u_fg, int ld_ufg, const float* u_bg, const float* u_hs, float* o_rois, float* o_gt_src,
                   float* o_gt, float* o_iou, float* o_scores, int64_t* o_labels, int64_t* o_reg, float* o_cls,
                   int32_t* status, void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Training losses of the detector heads with their gradients, whose rules csrc/head_losses.cu states.  No host read;
 * graph-capturable; losses and gradients are bit-identical run to run (fixed-order float64 sums, no float atomics).
 *   vc_rpn_loss  <- AnchorHeadTemplate.get_loss (anchor_head_template.py:178-333; OD_LOSS off, WeightedSmoothL1Loss,
 *                   one head, 7 codes): cls_preds [B, N, n_cls], box_preds [B, N, 7], dir_cls_preds [B, N, n_bins] or
 *                   NULL (no direction term), labels [B, N] int32, reg_targets [B, N, 7], anchors [N, 7] (shared by all
 *                   scenes; read only for the direction target), all fp32 contiguous; alpha / gamma of the focal loss,
 *                   beta of the smooth-L1, code_weights HOST [7], the cls / loc / dir loss weights, DIR_OFFSET ->
 *                   losses [4] fp32 = (cls, loc, dir, total) as the reference's tb values; g_cls / g_box / g_dir = d total
 *                   / d each prediction (shapes of the inputs), every element written.  ws >= vc_rpn_loss_ws_bytes(B, N).
 *                   A memset and two launches.
 *   vc_rcnn_loss <- RoIHeadTemplate.get_loss (roi_head_template.py:161-291; CLS_LOSS BinaryCrossEntropy, REG_LOSS
 *                   smooth-l1): K <= VC_RCNN_MAX_BRANCHES branches from a HOST table, each n rows of rcnn_cls [n, 1],
 *                   rcnn_reg [n, 7], its targets rois [n, ldr], gt_of_rois (canonical) / gt_of_rois_src [n, ldg],
 *                   reg_valid_mask int64 [n], rcnn_cls_labels fp32 [n], and a weight; several branches may share one
 *                   target set.  corner != 0: CORNER_LOSS_REGULARIZATION.  -> losses [K * 4 + 1] fp32 = per branch
 *                   (cls, reg, corner, bb), then the weighted total (the reference's rcnn_loss); g_cls [n] / g_reg [n, 7]
 *                   per branch = d total / d rcnn_cls / rcnn_reg, every element written.  The table is copied into the
 *                   launch's parameters: no host-to-device copy.  ws >= vc_rcnn_loss_ws_bytes(K).  A memset and one
 *                   launch (one CTA per branch).
 * ---------------------------------------------------------------------------------------------- */
#define VC_RCNN_MAX_BRANCHES 18
typedef struct vc_rcnn_branch {
    const float* rcnn_cls;
    const float* rcnn_reg;
    const float* rois;
    const float* gt_of_rois;
    const float* gt_of_rois_src;
    const int64_t* reg_valid_mask;
    const float* rcnn_cls_labels;
    float* g_cls;
    float* g_reg;
    int n, ldr, ldg;
    float weight;
} vc_rcnn_branch;
size_t vc_rpn_loss_ws_bytes(int B, int N);
int vc_rpn_loss(const float* cls_preds, const float* box_preds, const float* dir_cls_preds, const int32_t* labels,
                const float* reg_targets, const float* anchors, int B, int N, int n_cls, int n_bins, double alpha,
                double gamma, double beta, const double* code_weights /*host[7]*/, double cls_weight, double loc_weight,
                double dir_weight, double dir_offset, float* losses, float* g_cls, float* g_box, float* g_dir, void* ws,
                size_t ws_bytes, vc_stream_t stream);
size_t vc_rcnn_loss_ws_bytes(int K);
int vc_rcnn_loss(const vc_rcnn_branch* branches /*host[K]*/, int K, double beta, const double* code_weights /*host[7]*/,
                 double cls_weight, double reg_weight, double corner_weight, int corner, float* losses, void* ws,
                 size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Part-score RoI pooling of TEDMHead's PART branch (VirConv-T / -S), whose rules csrc/part_pool.cu states.  No host
 * read; graph-capturable; the backward is bit-identical run to run (fixed-order sums, no float atomics).
 *   vc_part_pool_fwd <- TEDMHead.obtain_conf_preds (ted_head.py:425-448) with gen_sample_grid and
 *                       bilinear_interpolate_torch_gridsample (:110-156), all scenes in one call: parts [B, S*S, H, W]
 *                       and rois [B, N, ld] (ld >= 7) fp32 contiguous, grid size S, GRID_OFFSETS (ox, oy), spatial scale
 *                       1 / FEATMAP_STRIDE -> out [B * N] fp32 (torch.cat(confi), scene-major).  One launch.
 *   vc_part_pool_bwd <- its gradient with respect to the part map: g [B * N] (d loss / d out) -> dparts [B, S*S, H, W],
 *                       every element written.  ws >= vc_part_pool_bwd_ws_bytes(B, N, S) (0 today: the tap records stay
 *                       in shared memory).  One launch.
 *   N > VC_PART_POOL_MAX_ROIS or S outside [2, VC_PART_POOL_MAX_GRID] -> VC_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
#define VC_PART_POOL_MAX_ROIS 1024
#define VC_PART_POOL_MAX_GRID 16
int vc_part_pool_fwd(const float* parts, const float* rois, int B, int N, int ld, int S, int H, int W, float ox, float oy,
                     float scale, float* out, vc_stream_t stream);
size_t vc_part_pool_bwd_ws_bytes(int B, int N, int S);
int vc_part_pool_bwd(const float* rois, const float* g, int B, int N, int ld, int S, int H, int W, float ox, float oy,
                     float scale, float* dparts, void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * RoI grid points of TEDMHead.roi_grid_pool / roi_grid_pool_mm, whose rules csrc/roi_grid.cu states.  No host read;
 * graph-capturable; every operation rounds once in fp32, as torch's elementwise kernels do.
 *   vc_roi_grid_points <- get_global_grid_points_of_roi (ted_head.py:652-673) and the voxel coordinates of the grid
 *                         points (:481-485, :528-532) for all scenes and S feature sources in one launch: rois [B, N, ld]
 *                         (ld >= 7) fp32 contiguous, grid size G (1..64), range3 = point_cloud_range[0:3] and voxel3 =
 *                         voxel_size as float32 (host), strides [S] (host, >= 1) -> new_xyz [B*N*G^3, 3] fp32 and
 *                         new_coords [S, B*N*G^3, 4] int32 as (b, x, y, z).
 *   S > VC_ROI_GRID_MAX_SOURCES -> VC_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
#define VC_ROI_GRID_MAX_SOURCES 4
int vc_roi_grid_points(const float* rois, int B, int N, int ld, int G, const float* range3, const float* voxel3,
                       const int32_t* strides, int S, float* new_xyz, int* new_coords, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Box decoding of the heads and TEDMHead's cascade stage transforms, whose rules csrc/box_decode.cu states.  One launch
 * per call, all scenes in one grid; no host read; graph-capturable; every fp32 operation rounds once, as torch's
 * elementwise kernels do.  All tensors fp32, contiguous, on the device.
 *   vc_anchor_decode     <- AnchorHeadTemplate.generate_predicted_boxes (anchor_head_template.py:335-382), ResidualCoder
 *                           with 7 codes: box_preds [B, A, 7], dir_cls [B, A, NB] (NULL: no direction classifier),
 *                           anchors [A, 7] shared by the scenes, DIR_OFFSET, DIR_LIMIT_OFFSET and period = 2 pi /
 *                           NUM_DIR_BINS as float32 -> out [B, A, 7].
 *   vc_anchor_decode_bwd <- its gradient with respect to box_preds: grad [B, A, 7] -> dbox [B, A, 7].
 *   vc_roi_decode        <- RoIHeadTemplate.generate_predicted_boxes (roi_head_template.py:294-324): box_preds [B*N, 7],
 *                           rois [B, N, ld] (ld >= 7) -> out [B, N, 7].
 *   vc_roi_decode_bwd    <- its gradient with respect to box_preds: grad [B, N, 7] -> dbox [B*N, 7].
 *   vc_box_xtrans        <- TEDMHead.roi_x_trans / roi_score_trans / pred_x_trans (ted_head.py:675-746) over
 *                           X_TRANS.backward_with_param / forward_with_param (X_transform.py:49-154): boxes [B, N, ld]
 *                           (ld >= 7), transform_param [B, R, 3] (rotation, flip, scale) -> out [B, N, ld]: the backward
 *                           transform of stage from_stage, then the forward transform of stage to_stage; a stage < 0 is
 *                           skipped.  Columns beyond 7 are copied.
 * ---------------------------------------------------------------------------------------------- */
int vc_anchor_decode(const float* box_preds, const float* dir_cls, const float* anchors, int B, int A, int NB,
                     float dir_offset, float dir_limit_offset, float period, float* out, vc_stream_t stream);
int vc_anchor_decode_bwd(const float* grad, const float* box_preds, const float* anchors, int B, int A, int with_dir,
                         float* dbox, vc_stream_t stream);
int vc_roi_decode(const float* box_preds, const float* rois, int B, int N, int ld, float* out, vc_stream_t stream);
int vc_roi_decode_bwd(const float* grad, const float* box_preds, const float* rois, int B, int N, int ld, float* dbox,
                      vc_stream_t stream);
int vc_box_xtrans(const float* boxes, const float* transform_param, int B, int N, int ld, int R, int from_stage,
                  int to_stage, float* out, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Parameter update of the adam_onecycle / adam_cosin step (csrc/optim.cu): what the reference's loop does after
 * loss.backward() (tools/train_utils/train_utils.py:50-52: clip_grad_norm_, OptimWrapper.step of fastai_optim.py:132-149
 * over torch.optim.Adam) for EVERY parameter tensor in two launches.  No host read, no allocation; graph-capturable;
 * bit-identical run to run and for every max_ctas (fixed-order float64 norm, no float atomics).
 *   segs    device [n_segs]: one entry per parameter tensor, fp32 throughout.  g == NULL: a trainable parameter that got no
 *           gradient; it takes no part in the norm and is decayed only.
 *   chunks  device [n_chunks]: the tensors cut into pieces of at most VC_OPTIM_CHUNK elements (off a multiple of 4), made
 *           by the caller once from the element counts.
 *   hyper   device float64[5]: lr, beta1 (the CURRENT momentum), beta2, eps, wd.
 *   counters device int64[2]: t = steps applied so far, and steps skipped.  The call advances one of them.
 *   guards  HOST array of n_guards (<= VC_OPTIM_MAX_GUARDS) device int32 words, read by the norm pass.
 *   status  device, written by the norm pass: total_norm = sqrt(sum g^2); clip_coef = min(1, max_norm / (total_norm + 1e-6))
 *           (1 when max_norm < 0: no clipping); apply = total_norm is finite and every guard word is zero; then the step's
 *           scalars, formed in float64 and rounded to fp32 once.
 * With apply == 0 nothing is written to p, m, v or t and `skipped` grows by one.  Otherwise, per element, with
 * gh = clip_coef * g and t counting this step:
 *   p <- p * (1 - wd * lr);  m <- m + (1 - beta1) * (gh - m);  v <- beta2 * v + (1 - beta2) * gh^2;
 *   p <- p - lr / (1 - beta1^t) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps).
 * The gradients are never written.  ws >= vc_optim_ws_bytes(n_chunks), ZEROED by the caller before the first call and
 * left alone afterwards (the norm pass's ticket resets itself).  max_ctas > 0 caps both grids (0: one CTA per chunk).
 * ---------------------------------------------------------------------------------------------- */
#define VC_OPTIM_CHUNK 4096
#define VC_OPTIM_MAX_GUARDS 8
typedef struct {
    float* p;
    const float* g; /* may be NULL */
    float* m;       /* exp_avg */
    float* v;       /* exp_avg_sq */
    long long n;
} vc_optim_seg;
typedef struct {
    int32_t seg;
    int32_t len;
    long long off;
} vc_optim_chunk;
typedef struct {
    double total_norm, clip_coef;
    int32_t apply;
    float clip, decay, step_size, bc2_sqrt, eps, w1, beta2, w2;
    int32_t pad[3];
} vc_optim_status; /* 64 bytes */
size_t vc_optim_ws_bytes(int n_chunks);
int vc_optim_step(const vc_optim_seg* segs, int n_segs, const vc_optim_chunk* chunks, int n_chunks, double max_norm,
                  const int32_t* const* guards /*host[n_guards]*/, int n_guards, const double* hyper, long long* counters,
                  vc_optim_status* status, int max_ctas, void* ws, size_t ws_bytes, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Plan executor: a whole backbone forward / backward in ONE call.  Replaces the Python layer loop of
 * `VirConvL8x.forward` (spconv_backbone.py:609-699), `NRConvBlock.forward` (:207-229) and the two streams of
 * `VirConv8x.forward` (:339-535) together with autograd's reverse walk over them: the host side of ~100 operator
 * calls per step becomes native.  The caller describes the layer graph once as a PLAN:
 *   ops_i [n_ops, 24] int32, ops_f [n_ops, 8] float32, one row per op, executed in order:
 *     [0] kind  1 SUBM_RB   index set a            -> rulebook c            ([21] = 1 if coordinates are unique)
 *               2 CONV_RB   index set a            -> index set b, rulebook c   (host reads the row count once)
 *               3 INDEX2UV  3-D index set a        -> 2-D index set b       ([6],[7] = image shape, [21] stride,
 *                                                                            [22] u_max, [23] v_max, ops_f[0..5] = grid)
 *               4 CBR       features a, rulebook c -> features b            conv + BatchNorm1d + ReLU of layer [20]
 *                                                                            ([18] cin, [19] cout, [21] = input needs grad)
 *               5 CAT       features a, features b -> features c            channel concat
 *               6 DISCARD   index set a, features [18] -> index set b, features [19]   StVD layer discard at site c
 *                                                                            (vc_stvd_layer_keep: selection and index gather
 *                                                                            on the index stream, feature gather on main;
 *                                                                            [6],[7] = float64 rate, low / high 32 bits)
 *     [1] stream (0 main: feature ops, 1 side: index ops, 2 second side stream: the image branch's index ops)
 *     [2..4] a, b, c   [5] ndim   [6..8] kernel size
 *     [9..11] stride   [12..14] padding   [15..17] dilation
 *   layer_ptrs [n_layers, 9] uint64: weight, gamma, beta, running_mean, running_var, num_batches_tracked, then the
 *   caller's gradient buffers d_weight, d_gamma, d_beta (written by vc_exec_backward); layer_f [n_layers, 2] = eps, momentum.
 *   Feature slot 0 / index set 0 are the network input (feats0 [n0, c0] fp32, idx0 [n0, 4] int32, shape0 host[3]).
 * Memory: every activation, rulebook and scratch buffer is carved out of `arena` (bump allocation, nothing reused
 * inside a step; VC_ERR_WORKSPACE if it is too small).  `state` (>= vc_exec_state_bytes(), host) receives the buffer
 * addresses and row counts that vc_exec_backward and vc_exec_query read; the library keeps nothing else between calls
 * (apart from a pool of CUDA events for cross-stream ordering).  `pinned_host`: >= 16 int32 of page-locked host memory
 * for the row-count read-backs.  precision 0 = fp32 kernels, 1 = bf16 tensor-core kernels where channels allow.
 * Index ops run on side_stream (may be NULL = single stream), those of stream 2 on side2_stream (may be NULL: then on
 * side_stream); on return every later use of main_stream is ordered
 * after all of the step's work.  side_waits_main != 0: the side stream first waits for everything already queued on
 * main_stream (always safe).  0: the caller guarantees idx0 / proj_params are valid in side_stream order and that the
 * arena may be written from side_stream right away (e.g. it was allocated there) — the index ops of this step then
 * overlap the previous step's backward.
 * Static mode (n0_dev != NULL): nothing in the call reads a device value on the host, so the whole forward (and the
 * backward that follows it) can be captured into a CUDA graph (SURVEY §8b "CUDA-graph-capturable").  n0 is then the
 * CAPACITY of feats0 / idx0, *n0_dev the number of valid rows; caps[i] (host, indexed by index-set id) is the row
 * capacity of the strided convs' output sets; every data-dependent row count stays in device memory
 * (vc_exec_query(state, 2, id)[6] = its address), published buffers have capacity rows with a zero / -1 tail, and a row
 * count that does not fit its capacity is clamped and reported as max() into *overflow_flag (device int32; zero it
 * before the step, re-run with larger capacities when it is non-zero afterwards).  Use side_waits_main = 1 under capture.
 * flags: bits 8-9 = phase (static mode only).  0 enqueues the whole forward, 1 ONLY the index operators (rulebooks,
 * projections), 2 ONLY the feature operators (weight images, conv + BN + ReLU, concat) over the arena phase 1 filled: call
 * both with the same arguments, so they allocate the same addresses and leave the same state (graph.PipelinedStep runs
 * the index phase of step t+1 beside the feature phase of step t).  Bit 2 = deterministic mode, recorded in the state
 * for the backward: the BN sums of the conv forward per 128-row tile and of BN backward per 512-row chunk, the
 * tensor-core wgrad per row run (32 images per layer), all added in a fixed order, and the many-to-one 2-D tables'
 * input gradient in gather form (vc_conv_dgrad_gather2d_*; timing kinds 8 / 9) — published features, indices, BN
 * running statistics and gradients are then bit-identical from run to run.  Other bits are ignored (callers pass
 * bit 0 = 1).
 * ---------------------------------------------------------------------------------------------- */
size_t vc_exec_state_bytes(void);
int vc_exec_forward(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                    int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0, const int32_t* shape0 /*host[3]*/,
                    int batch_size, const float* proj_params /*device [B,28], may be NULL without INDEX2UV ops*/,
                    int training, int precision, int flags, void* arena, size_t arena_bytes,
                    int32_t* pinned_host, int32_t* err_flag, void* state, size_t state_bytes, vc_stream_t main_stream,
                    vc_stream_t side_stream, int side_waits_main, const int32_t* caps /*host, may be NULL*/,
                    const int32_t* n0_dev /*device, NULL = exact mode*/, int32_t* overflow_flag /*device*/,
                    vc_stream_t side2_stream /*may be NULL: ops planned for stream 2 (image branch) then share side_stream*/);
/* vc_exec_forward plus the seed of the plan's DISCARD ops (device int64[1], read on the index stream); vc_exec_forward is
 * this call with rng_seed_dev = NULL, which a plan with a DISCARD op rejects.  In exact mode a discard that keeps no row
 * fails (VC_ERR_INVALID, naming the site); in static mode its output set has the input's capacity. */
int vc_exec_forward_seeded(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                           int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0, const int32_t* shape0,
                           int batch_size, const float* proj_params, int training, int precision, int flags, void* arena,
                           size_t arena_bytes, int32_t* pinned_host, int32_t* err_flag, void* state, size_t state_bytes,
                           vc_stream_t main_stream, vc_stream_t side_stream, int side_waits_main, const int32_t* caps,
                           const int32_t* n0_dev, int32_t* overflow_flag, vc_stream_t side2_stream,
                           const int64_t* rng_seed_dev /*may be NULL without DISCARD ops*/);
/* Reverse walk.  pub_slots [n_pub]: feature slots whose gradients come from outside (the published tensors), ext_grads
 * [n_pub]: device pointers to those gradients ([rows, c] fp32 contiguous, read only) or 0.  Writes d_weight / d_gamma /
 * d_beta of every layer (zeros where nothing flowed back).  Same arena as the forward (it continues allocating).
 * wgrad_stream (may be NULL): the weight-gradient kernels go there, concurrent with the BN-backward / dgrad chain on
 * `stream`; `stream` is joined with it before the call returns. */
int vc_exec_backward(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                     int n_layers, const int32_t* pub_slots, const uint64_t* ext_grads, int n_pub, void* arena,
                     size_t arena_bytes, int32_t* err_flag, void* state, vc_stream_t stream, vc_stream_t wgrad_stream);
/* SyncBatchNorm across ranks (torch.nn.SyncBatchNorm semantics; training mode only — eval uses the running statistics).
 * vc_exec_forward_sync / vc_exec_backward_sync are vc_exec_forward_seeded / vc_exec_backward plus a caller-owned float64
 * exchange buffer `xchg`, host slot offsets xchg_off [n_layers, 2] (in doubles: forward slot, backward slot of each layer)
 * and a host callback.  With exchange_fn NULL (world size 1) they are the plain calls.  Otherwise every conv + BN layer runs
 * conv with epilogue sums -> exchange -> BN apply (never the fused conv + BN launch), and its BN backward runs reduce ->
 * exchange -> element-wise apply:
 *   forward slot  [sum x (cout), sum x^2 (cout), row count] — the count written by a kernel (static mode: from the device
 *                 count); after the exchange the statistics divide by the all-reduced count, the running statistics use it
 *                 for the unbiased variance;
 *   backward slot [sum g (cout), sum g*xhat (cout)] — the local d_gamma / d_beta are written before the exchange and stay
 *                 local; dx takes the all-reduced sums and the forward slot's global count.
 * exchange_fn(user, layer, direction 0 forward / 1 backward, slot, n doubles) is called on the host at each exchange point
 * and must enqueue the in-place sum of the slot over all ranks on main_stream / `stream` (under CUDA-graph capture it runs
 * once, at capture time); non-zero return fails the call.  Every rank makes the same calls in the same order.  In the
 * deterministic mode the local sums keep their fixed order.  The backward reads the forward slots: same buffer. */
typedef int (*vc_bn_exchange_fn)(void* user, int layer, int direction, double* slot, int n);
int vc_exec_forward_sync(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                         int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0, const int32_t* shape0,
                         int batch_size, const float* proj_params, int training, int precision, int flags, void* arena,
                         size_t arena_bytes, int32_t* pinned_host, int32_t* err_flag, void* state, size_t state_bytes,
                         vc_stream_t main_stream, vc_stream_t side_stream, int side_waits_main, const int32_t* caps,
                         const int32_t* n0_dev, int32_t* overflow_flag, vc_stream_t side2_stream, const int64_t* rng_seed_dev,
                         double* xchg, const int64_t* xchg_off /*host*/, vc_bn_exchange_fn exchange_fn, void* exchange_user);
int vc_exec_backward_sync(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                          int n_layers, const int32_t* pub_slots, const uint64_t* ext_grads, int n_pub, void* arena,
                          size_t arena_bytes, int32_t* err_flag, void* state, vc_stream_t stream, vc_stream_t wgrad_stream,
                          double* xchg, const int64_t* xchg_off, vc_bn_exchange_fn exchange_fn, void* exchange_user);
/* Read a state blob.  what 0: out[0] = arena bytes in use, out[1] = of them, the deterministic mode's partials, tables and
 * operands, out[2] = deterministic mode;  1 (feature slot id): f32 ptr, bf16 ptr, rows, c, row pitch of f32 / bf16,
 * gradient ptr, row pitch of the gradient (after vc_exec_backward: the slot's final input gradient; a published slot no
 * layer reads keeps the caller's ext_grads pointer);  2 (index set): idx ptr, n, ndim, shape[3];  3 (rulebook): nbr,
 * nbr_bwd, pair_num ptrs, K, n_in, n_out, subm, unique;  4 (layer): x ptr, y ptr, stats ptr, forward runs on the tensor
 * cores, rulebook id, in slot, out slot;  5 (op index of a DISCARD): keep ptr, kept rows (exact mode; static mode: the
 * capacity), kept_dev ptr, n_in, site;  6 (layer, after vc_exec_backward): the upstream gradient ptr vc_exec_backward read
 * and its row pitch, the BN backward's fp32 dx ptr (0 where no fp32 kernel reads it) and bf16 dx ptr (0 in fp32 mode),
 * then the forward, weight-gradient and input-gradient kinds (vc_exec_timing_read's kinds, -1: no input gradient); all
 * pointers 0 where nothing flowed back into the layer.  The arena is never reused inside a step, so every pointer stays
 * valid until the arena is released.  out: >= 8 int64 (host). */
int vc_exec_query(const void* state, int what, int id, long long* out);
/* Optional per-launch timing of the conv kernels (bench.py's roofline pass): vc_exec_timing(1) clears and arms it,
 * vc_exec_timing_read synchronises and returns up to max_records (ms, [kind, layer]) records; kind 0 fwd f32, 1 fwd tc,
 * 2 dgrad f32, 3 dgrad tc, 4 dgrad scatter f32, 5 wgrad f32, 6 wgrad tc, 7 dgrad scatter tc, 8 dgrad gather2d f32,
 * 9 dgrad gather2d tc. */
int vc_exec_timing(int enable);
int vc_exec_timing_read(float* ms_out, int32_t* kind_layer_out, int max_records);

/* ---- gradient all-reduce over NVLink peer memory (SURVEY 8e; replaces DistributedDataParallel's NCCL all-reduce of
 * tools/train.py:140-141 for the backbone's one flat 1.7 MB gradient buffer) ----
 * Every rank owns a SYMMETRIC fp32 buffer of 2 * n_pad floats and a symmetric array of vc_allreduce_peer_flag_words(world)
 * zero-initialised uint32 flags, both mapped into every peer (torch.distributed._symmetric_memory); peer_bufs / peer_flags are
 * HOST arrays of `world` device addresses: where rank r's buffer / flags are mapped in THIS process.  One call per step on every
 * rank with the same, strictly increasing `epoch` (first call: 1): grads[i] <- scale * sum over ranks of grads[i], in place.
 * A peer that does not show up within 4 s sets *err_flag (0x400 + peer) instead of hanging the GPU. */
int vc_allreduce_peer_flag_words(int world);
int vc_allreduce_peer_f32(const uint64_t* peer_bufs, const uint64_t* peer_flags, int rank, int world, float* grads, long long n,
                          long long n_pad, unsigned epoch, float scale, int32_t* err_flag, vc_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * KITTI evaluation (csrc/kitti_eval.cu, geometry in csrc/kitti_eval_geom.cuh): what kitti_object_eval_python/eval.py's
 * eval_class computes for the three metrics of get_official_eval_result, over a whole evaluation set in nine launches.
 * Packed input (double, VC_KE_ROW per object, one upload):
 *   GT row  : bbox x0 y0 x1 y1, alpha, location x y z, dimensions l h w, rotation_y, truncated, occluded,
 *             class id (car 0, pedestrian 1, cyclist 2, van 3, person_sitting 4, truck 5, other -1), DontCare (1 / 0)
 *   DT row  : bbox x0 y0 x1 y1, alpha, location x y z, dimensions l h w, rotation_y, score, class id, 0, 0
 *   offs    : int64 [3][F + 1]: the frames' first GT row, first detection row and first overlap pair
 *             (pair_off[f + 1] - pair_off[f] = n_gt[f] * n_dt[f])
 *   lane_mo : double [L] min overlap per lane, L = 3 * C * 3 * K, lane = ((metric * C + class) * 3 + difficulty) * K + k
 *   vc_kitti_overlaps   <- one metric's per-frame [n_dt, n_gt] blocks (0 image, 1 BEV, 2 3-D) into ov [n_pair]
 *   vc_kitti_rotate_iou <- rotate_iou_gpu_eval (rotate_iou.py:295): boxes [N, 5], qboxes [K, 5] float32 -> out [N, K]
 *   vc_kitti_eval       <- eval_class for metrics 0, 1, 2: ov [3][n_pair] and, per lane, out[lane * VC_KE_LANE_W ..]:
 *                          [0] the number of thresholds T, [1, 42) the thresholds, [42, 206) tp, fp, fn, similarity per
 *                          threshold, [206, 247) precision, [247, 288) recall, [288, 329) orientation (eval_class's
 *                          arrays, running max applied).  classes: host array of C class ids.
 * ---------------------------------------------------------------------------------------------- */
#define VC_KE_ROW 16
#define VC_KE_SAMPLES 41
#define VC_KE_LANE_W 329
#define VC_KE_MAX_CLASSES 6
#define VC_KE_MAX_OVERLAPS 10
int vc_kitti_overlaps(const double* gt, const double* dt, const long long* offs, int F, long long n_pair, int metric,
                      double* ov, vc_stream_t stream);
int vc_kitti_rotate_iou(const float* boxes, const float* qboxes, int N, int K, int criterion, float* out,
                        vc_stream_t stream);
size_t vc_kitti_eval_ws_bytes(int F, int NG, int ND, int C, int K);
int vc_kitti_eval(const double* gt, const double* dt, const long long* offs, const double* lane_mo, int F, int NG, int ND,
                  long long n_pair, int C, const int* classes, int K, int compute_aos, double* ov, double* out, void* ws,
                  size_t ws_bytes, vc_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* VIRCONV_B200_H */
