// Shared helpers for the virconv_b200 sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/virconv_b200.h"

namespace vc {

void set_error(const char* fmt, ...);
void count_launch();  // bumps the counter behind vc_launch_count()

#define VC_CHECK_ARG(cond, ...)                 \
    do {                                        \
        if (!(cond)) {                          \
            vc::set_error(__VA_ARGS__);         \
            return VC_ERR_INVALID;              \
        }                                       \
    } while (0)

#define VC_CUDA(expr)                                                                          \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            vc::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return VC_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

#define VC_LAUNCH_CHECK()          \
    do {                           \
        vc::count_launch();        \
        VC_CUDA(cudaGetLastError()); \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

struct Geom {  // conv geometry, passed by value to kernels
    int ndim;
    int K;
    int batch;                   // batch size: rows with a batch index outside [0, batch) or coordinates outside `shape` are ignored
    int shape[VC_MAX_NDIM];      // input spatial shape
    int oshape[VC_MAX_NDIM];     // output spatial shape
    int ksize[VC_MAX_NDIM];
    int stride[VC_MAX_NDIM];
    int pad[VC_MAX_NDIM];
    int dil[VC_MAX_NDIM];
};

__device__ __forceinline__ uint32_t mix64(uint64_t k) {  // murmur3 finaliser
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdULL;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ULL;
    k ^= k >> 33;
    return (uint32_t)k;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
    uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    int sz = valid ? 16 : 0;  // src-size 0 => 16 bytes of zeros
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(sz));
}
// same, destination given as a 32-bit shared-space address (saves the generic->shared conversion per copy)
__device__ __forceinline__ void cp_async16_s(uint32_t smem_addr, const void* gsrc, bool valid) {
    int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_addr), "l"(gsrc), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// Stage the tile's slice nbr[k0 .. k0+kcount) x [base, base+128) of a neighbour table into shared memory.  Loads are
// issued in batches of 8 independent LDGs per thread (a plain `nbr_s[i] = nbr[...]` loop serialises one global-memory
// round trip per iteration: ~20 dependent round trips for K = 27, which was most of a conv CTA's prologue).
template <int THREADS, int BATCH = 8>
__device__ __forceinline__ void stage_nbr_tile(const int32_t* __restrict__ nbr, int n_rows, int k0, int kcount, int base,
                                               int* nbr_s) {
    const int total = kcount * 128;
    for (int i0 = threadIdx.x; i0 < total; i0 += THREADS * BATCH) {
        int v[BATCH];
#pragma unroll
        for (int j = 0; j < BATCH; ++j) {
            const int i = i0 + j * THREADS;
            const int k = i >> 7, row = base + (i & 127);
            v[j] = (i < total && row < n_rows) ? __ldg(nbr + (size_t)(k0 + k) * n_rows + row) : -1;
        }
#pragma unroll
        for (int j = 0; j < BATCH; ++j) {
            const int i = i0 + j * THREADS;
            if (i < total) nbr_s[i] = v[j];
        }
    }
}

// ---- shared between rulebook.cu and executor.cu ----
// `n_dev` (optional): the row count lives in device memory and `n` / `n_out` are capacities (static mode, graph capturable)
int subm_rulebook_dev(const int32_t* indices, int n, const int* n_dev, int ndim, int batch_size, const int32_t* spatial_shape,
                      const int32_t* ksize, const int32_t* dilation, int32_t* nbr, int32_t* pair_num, void* ws, size_t ws_bytes,
                      cudaStream_t stream, int32_t* rep = nullptr,   // rep (optional): [n] lowest row at each row's coordinate
                      bool unique = false);   // every coordinate held by one row: half the probes (the table is its own transpose)
// where a strided conv's output bitmap and its ranks lie in the workspace of its chain (conv_chain_rank)
struct ConvRank {
    const uint32_t *bitmap, *word_rank, *block_sum;
};
// L chained strided convs (rulebook.cu header: each level's input set is the previous level's output set; a single strided
// conv is a chain of one): every level's output set from the first input set, in one mark + scan pass and one emit
constexpr int CONV_CHAIN_MAX = 4;
struct ConvChain {
    int L, ndim, batch;
    const int32_t* shape0;   // input spatial shape of level 0; level l + 1's is level l's output shape
    const int32_t *ksize[CONV_CHAIN_MAX], *stride[CONV_CHAIN_MAX], *pad[CONV_CHAIN_MAX], *dil[CONV_CHAIN_MAX];
};
bool conv_chain_composable(const ConvChain& ch);   // 1 <= L <= CONV_CHAIN_MAX, dilation 1 everywhere when L >= 2
size_t conv_chain_ws_bytes(const ConvChain& ch);
ConvRank conv_chain_rank(const ConvChain& ch, const void* ws, int level);
// n_out_dev [L]: each level's row count; caps (NULL: no clamp) [L]: capacities, a larger count is clamped and reported
int conv_chain_count_dev(const ConvChain& ch, const int32_t* indices, int n, const int* n_dev, int32_t* n_out_dev, const int* caps,
                         int* overflow, void* ws, size_t ws_bytes, cudaStream_t stream);
// out_idx [L]: output index buffers of caps[l] rows
int conv_chain_emit_dev(const ConvChain& ch, int32_t* const* out_idx, const int* caps, void* ws, size_t ws_bytes, cudaStream_t stream);

// The per-stage index work of up to IDX_BATCH_MAX stages, one launch per kind (rulebook.cu, misc.cu): the same results as
// one call per stage (subm_rulebook_dev and vc_conv_rulebook_fill are batches of one).  The caller owns the buffers and
// clears them first (so that the regions of all stages can be cleared together): hash tables to 0xFF, a mirrored table's
// rows k > centre to -1, pair counts to 0, nbr_fwd to -1.
constexpr int IDX_BATCH_MAX = 4;
bool subm_sym(int ndim, const int32_t* ksize, bool unique);   // the mirrored probe (half the offsets, rows k > centre pre-filled)
struct SubmStage {   // one submanifold rulebook (subm_rulebook_dev); table: vc_subm_rulebook_ws_bytes(n) bytes
    const int32_t* idx;
    int n;
    const int* n_dev;
    int ndim;
    const int32_t *shape, *ksize, *dil;
    int32_t *nbr, *pair_num;
    void* table;
    size_t table_bytes;
    int32_t* rep;    // optional [n]: lowest row at each row's coordinate (the stage then probes every offset)
};
int subm_rulebook_batch_dev(const SubmStage* st, int n_st, int batch_size, bool unique, cudaStream_t stream);
struct TablesStage {  // one strided conv's tables (nbr_bwd, pair counts, nbr_fwd scattered from the input rows)
    const int32_t* idx;
    int n;
    const int* n_dev;
    int ndim;
    const int32_t *shape, *ksize, *stride, *pad, *dil;
    int n_out;
    ConvRank rank;
    int32_t *nbr_fwd, *nbr_bwd, *pair_num;   // nbr_fwd NULL: written by conv_fwd_lookup_batch_dev instead
};
int conv_tables_batch_dev(const TablesStage* st, int n_st, int batch_size, cudaStream_t stream);
// Over chain levels (conv_chain_rank): a level's rows are its bitmap's set bits in rank order, so a cell's row is its rank,
// and a rank at or past the level's held rows (n, or *n_dev) is absent.
struct SubmLookupStage {   // one submanifold rulebook over a chain level's output set, `rank` that level's bitmap
    const int32_t* idx;
    int n;
    const int* n_dev;
    int ndim;
    const int32_t *shape, *ksize, *dil;
    ConvRank rank;
    int32_t *nbr, *pair_num;
};
int subm_lookup_batch_dev(const SubmLookupStage* st, int n_st, int batch_size, cudaStream_t stream);
struct FwdLookupStage {    // nbr_fwd of a chained strided conv whose input set is the chain level `in_rank`
    const int32_t* out_idx;          // the conv's output rows
    int n_out;
    const int* n_out_dev;
    int n_in;                        // the input level's held rows
    const int* n_in_dev;
    ConvRank in_rank;
    int ndim;
    const int32_t *shape, *ksize, *stride, *pad, *dil;   // shape: the input level's
    int32_t* nbr_fwd;
};
int conv_fwd_lookup_batch_dev(const FwdLookupStage* st, int n_st, int batch_size, cudaStream_t stream);
struct UVStage {     // one projection (index2uv_dev)
    const int32_t* idx;
    int n;
    const int* n_dev;
    const float* grid;
    int stride, u_max, v_max;
    int32_t* uv;
};
int index2uv_batch_dev(const UVStage* st, int n_st, int batch_size, const float* params, cudaStream_t stream);

// ---- bn.cu / misc.cu internals used by the plan executor (device row counts, strided outputs) ----
int bn_apply_relu_dev(const float* x, const double* sums, int n_rows, const int* n_dev, int c, const float* gamma,
                      const float* beta, float* running_mean, float* running_var, long long* num_batches_tracked, float momentum,
                      float eps, int training, float* y, int y_ld, void* y_bf16, int yb_ld, float* stats_out, int relu,
                      int tail_zero, cudaStream_t stream, const double* n_glob = nullptr);
// part (deterministic mode, else NULL): [cdiv(n, BN_DET_ROWS), 2, c] float64 chunk partials, summed in chunk order
int bn_relu_bwd_dev(const float* dy, int dy_ld, const float* x, const float* gamma, const float* stats, float* dx, void* dx_bf16,
                    float* dgamma, float* dbeta, int n, const int* n_dev, int c, int training, double* bsums, int tail_zero,
                    cudaStream_t stream, double* part = nullptr);
// deterministic BN sums: sums [2, c] = the per-part partials part [cdiv(rows, rows_per_part), 2, c] added in part order
int bn_sums_reduce_dev(const double* part, int cap_rows, const int* n_dev, int rows_per_part, int c, double* sums,
                       cudaStream_t stream);
static constexpr int BN_DET_ROWS = 512;   // rows per chunk of the deterministic BN backward reduction
// SyncBatchNorm exchange (executor.cu): local sums into a rank's float64 slot before the all-reduce, and the backward split
// around it (bn.cu states the layouts); n_glob: device float64, the row count over all ranks
int bn_sync_pack_dev(const double* sums, int c, int n_rows, const int* n_dev, double* slot, float* dgamma, float* dbeta,
                     cudaStream_t stream);
int bn_relu_bwd_local_dev(const float* dy, int dy_ld, const float* x, const float* stats, int n, const int* n_dev, int c,
                          double* bsums, double* part, float* dgamma, float* dbeta, double* slot, cudaStream_t stream);
int bn_relu_bwd_apply_dev(const float* dy, int dy_ld, const float* x, const float* gamma, const float* stats,
                          const double* bsums, const double* n_glob, float* dx, void* dx_bf16, int n, const int* n_dev, int c,
                          int tail_zero, cudaStream_t stream);
int cat2_dev(const float* a, const float* b, float* out, void* out_bf16, int n, const int* n_dev, int ca, int cb, cudaStream_t stream);
int index2uv_dev(const int32_t* indices, int n, const int* n_dev, int batch_size, const float* params, const float* grid,
                 int stride, int u_max, int v_max, int32_t* uv_out, cudaStream_t stream);

// ---- stvd_layer.cu internals used by the plan executor (StVD layer discard) ----
// out[r] = keep[r] >= 0 ? in[keep[r]] : 0 for r < rows (fp32 and / or bf16; either may be NULL), in [*, c] dense, c % 4 == 0
int stvd_gather_feats_dev(const float* in, int c, const int32_t* keep, int rows, float* out, void* out_bf16, cudaStream_t st);
// out[r] = keep[r] >= 0 ? in[keep[r]] : -1 (rows of `cols` int32)
int stvd_gather_idx_dev(const int32_t* in, int cols, const int32_t* keep, int rows, int32_t* out, cudaStream_t st);
// dx[i] = pos[i] >= 0 ? dy[pos[i]] : 0 for i < n_in, row pitches dy_ld / dx_ld
int stvd_grad_dev(const float* dy, int dy_ld, int c, const int32_t* pos, int n_in, float* dx, int dx_ld, cudaStream_t st);

// ---- shared between conv_tc.cu, conv_tc2.cu and executor.cu ----
struct TcPrepEntry {
    const float* w;   // parameter, spconv layout [C_out, K, C_in]
    void* img;        // bf16 UMMA image, K * cin * cout elements
    int cin, cout, K;
    int mode;         // 0 forward image, 1 dgrad image
    int mirror;       // dgrad: kernel offsets mirrored (submanifold table re-used as its own transpose)
    int layout;       // 0: core-matrix image of the scatter dgrad (tc_scatter_kernel); 1: swizzled + padded to 16 (conv_tc2.cu)
    int first;        // element prefix (filled by tc_prep_images)
};
static constexpr int TC_PREP_MAX = 64;
struct TcPrepTable {
    TcPrepEntry e[TC_PREP_MAX];
    int n, total;
};
int tc_prep_images(TcPrepTable& t, cudaStream_t stream);
// ---- conv_tc.cu (tensor-core scatter dgrad of many-to-one tables) ----
static inline bool tc_scatter_ch_ok(int c) { return c == 16 || c == 32 || c == 64; }
int tc_scatter_with_image(int kc, int nr, const void* dout_bf16, const void* wimg, const int32_t* nbr, float* din, int n_out,
                          int K, int* err, cudaStream_t stream, int din_ld = 0);   // din_ld: row pitch of din (0: nr)
// fp32 scatter dgrad (vc_conv_dgrad_scatter_f32) into a din of row pitch din_ld (>= cin, multiple of 4)
int conv_dgrad_scatter_f32_ld(const float* dout, const float* w, const int32_t* nbr, float* din, int din_ld, int n_out, int cin,
                              int cout, int K, void* ws, size_t ws_bytes, cudaStream_t stream);
// ---- gather2d.cu (deterministic input gradient of the many-to-one 2-D tables) ----
// Groups of rows sharing a coordinate, from rep (vc_subm_rulebook_rep), and the gather table over U = [dout; S] (2 cap rows):
// nbr_g[centre][i] = i, nbr_g[k][i] = cap + nbr[k][i] for a representative i (rep[i] == i), else -1.
struct G2Prep {
    int32_t *nbr_g, *cnt, *off, *rows, *cur, *tot;   // cnt / off / rows: the rows of representative r's group, ascending
};
size_t gather2d_prep_bytes(int cap, int K);
G2Prep gather2d_carve(void* ws, int cap, int K);
int gather2d_prep_dev(const int32_t* nbr, const int32_t* rep, int K, int cap, const int* n_dev, const G2Prep& P, cudaStream_t st);
// U rows [cap + r] = sum of g over group r in ascending row order (fp32 sums; g fp32 or bf16, out fp32 and / or bf16)
int gather2d_sum_dev(const float* g, const void* g_bf16, int c, const G2Prep& P, int cap, const int* n_dev, float* u,
                     void* u_bf16, cudaStream_t st);
// The same grouping for E elements over G groups (the deterministic voxel-RoI pooling's inverse slot map): the caller fills
// key[E] (group of each element, < 0: none); slot_groups_dev leaves rows[off[r] .. off[r] + cnt[r]) = the elements of group
// r in ascending order, by integer work only.  Long groups are merge-sorted, one block each (max_ctas > 0 caps the grid).
struct SlotGroups {
    int32_t *key, *rows, *scratch, *cnt, *cur, *nbig, *off, *big, *tot;
};
size_t slot_groups_bytes(int E, int G);
SlotGroups slot_groups_carve(void* ws, int E, int G);
int slot_groups_dev(int E, int G, const SlotGroups& P, int max_ctas, cudaStream_t st);
extern int g_pool_det_ctas;   // vc_voxel_pool_det_config: CTA cap of the deterministic voxel-pooling kernels (0: automatic)
// dst[r, :] (row pitch ld) += src[r, :] (dense [cap, c]) for r below the row count
int add_rows_ld_dev(float* dst, int ld, const float* src, int cap, const int* n_dev, int c, cudaStream_t st);

// ---- conv_tc2.cu (persistent tensor-core conv: forward and gather dgrad) ----
int num_sms();   // of the current device
// BatchNorm + ReLU run by a forward conv launch itself, after a grid-wide barrier (the arguments of bn_apply_relu_dev; relu on)
struct BnTail {
    const float *gamma, *beta;
    float *running_mean, *running_var;
    long long* nbt;          // num_batches_tracked (may be NULL)
    float momentum, eps;
    int training;
    double* sums;            // [2, c] channel sums: zeroed by the caller (deterministic mode: written from the tile partials)
    float* y;                // fp32 output (may be NULL), row pitch y_ld
    int y_ld;
    void* yb;                // bf16 shadow (may be NULL), row pitch yb_ld
    int yb_ld;
    float* stats;            // [4, c] scale, shift, mean, invstd
    int tail_zero;           // zero the output rows [count, capacity)
    int* bar;                // grid-barrier counter, zeroed by the caller
};
extern int g_conv_bn_fused;  // vc_set_conv_bn_fused; cleared for good when the device refuses the cooperative launch
size_t tc_image_bytes(int cin, int cout, int K, int layout);
bool tc2_ch_ok(int c);
int tc2_conv(int kc, int nr, const void* in_bf16, const void* wimg, const int32_t* nbr, long long pitch, float* out, int n_rows,
             const int* n_dev, int K, double* bn_sums, int* err, cudaStream_t stream, const float* addend,
             int* tile_counter = nullptr, int flags = 0,   // flags: bit 0 sparse offsets (strided dgrad), bit 1 no index kernel
                                                           // beside it (the conv + BN grid takes 2 CTAs/SM), bit 2 zeros
                                                           // in out's rows [*n_dev, n_rows)
             int in_ld = 0,                                // row pitch of in_bf16 (0: kc)
             double* bn_part = nullptr,                    // deterministic BN sums: [tiles, 2, nr] per 128-row tile (bn_sums NULL)
             const BnTail* bn = nullptr,                   // forward only: BN + ReLU in the same launch when g_conv_bn_fused
             bool* bn_done = nullptr);                     // set when it ran (else the caller launches the apply)
// fp32 gather conv forward (vc_conv_fwd_f32) whose BN channel sums go to bn_part [tiles, 2, cout] per 128-row tile instead
int conv_fwd_f32_part(const float* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin, int cout, int K,
                      double* bn_part, void* ws, size_t ws_bytes, cudaStream_t stream);

// ---- wgrad_tc3.cu (persistent tensor-core wgrad) ----
extern int g_wgrad3_ctas;
// det_chunks > 0 (deterministic mode): scratch holds det_chunks partial images [det_chunks][K][cin][cout], zero on entry; the
// 128-row tiles are split into det_chunks runs of consecutive tiles (from the row count alone), a CTA claims whole runs and
// writes each run's sum into its own image, so the result does not depend on the grid or the schedule
int tc3_wgrad(int cin, int cout, const void* in_bf16, const void* dout_bf16, const int32_t* nbr, long long pitch, float* scratch,
              int n_rows, const int* n_dev, int K, int* err, cudaStream_t stream, int* tile_counter, int max_ctas,
              int in_ld = 0,    // row pitch of in_bf16 (0: cin)
              int det_chunks = 0);
static constexpr int WGRAD_DET_CHUNKS = 32;
int wgrad3_passes(int cin, int cout, int K);
struct WgradFinEntry {
    const float* scratch;   // [n_part][K][cin][cout] accumulated by tc3_wgrad
    float* dw;              // parameter layout [cout][K][cin]
    int cin, cout, K, first;
    int n_part;             // partial images added in order (1, or WGRAD_DET_CHUNKS in deterministic mode)
};
static constexpr int WGRAD_FIN_MAX = 64;
struct WgradFinTable {
    WgradFinEntry e[WGRAD_FIN_MAX];
    int n, total;
};
int wgrad_finalize(WgradFinTable& t, cudaStream_t stream);

// ReLU with torch's rules, shared by every kernel that applies one (bn_common.cuh, voxel_pool.cu):
// forward, torch.relu: NaN stays NaN (fmaxf alone would return 0), -0.0 becomes +0
__device__ __forceinline__ float relu_nan(float v) { return v != v ? v : fmaxf(v, 0.f); }
// backward, torch's threshold_backward: the gradient passes unless the activation is <= 0, so it passes at NaN
__device__ __forceinline__ float relu_grad(float pre, float g) { return pre <= 0.f ? 0.f : g; }

}  // namespace vc
