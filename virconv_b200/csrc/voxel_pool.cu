// Fused voxel-RoI grid pooling of TEDMHead (SURVEY §8f row 3) — sm_90a.
//
// Replaces, per grouper k, everything `NeighborVoxelSAModuleMSG.forward` (pcdet/ops/pointnet2/pointnet2_stack/
// voxel_pool_modules.py:70-130) does between `mlps_in[k]` and `mlps_out[k]`: the voxel query, the grouping of features and
// relative positions into [M, C, nsample] tensors, the position MLP Conv2d(3->C, no bias) + BatchNorm2d, the add, the ReLU
// and max_pool2d over the samples.  Nothing of size [M, C, nsample] is materialised, forward or backward.
//
// The reference's rules, kept here:
//   1. new_coords arrive as [b, z, y, x] (the module reorders its [b, x, y, z] input, :84, before calling in).
//   2. Query: exactly vc_voxel_query (shared device code, voxel_query.cuh): the first nsample hits in z-major scan order
//      within the radius, remaining slots filled with the first hit, an empty ball flagged.  idx holds the GLOBAL rows of
//      voxel2point_indices; the reference's round trip through batch-local ids (voxel_query_utils.py:85-91) gives the same
//      rows whenever new_coords[:, 0] agrees with new_xyz_batch_cnt, which is how TEDMHead builds them.
//   3. Per slot s of query point m: r = xyz[row] - new_xyz[m] in fp32 and f = features_in[row]; both are zero for an empty
//      ball (:99, :105).
//   4. Position branch p = BN2d(W_pos r).  Because the conv has no bias, the train-mode statistics over all M * nsample slots
//      (duplicated fill slots and the zeros of empty balls included) follow exactly from the moments of r:
//      mean = W E[r], var = diag(W Cov(r) W^T) (biased).  The query pass accumulates the nine moments
//      (sum r, sum r r^T) in float64; pool_bn_fold_kernel turns them into the statistics, updates the running ones and
//      folds BN into p = scale * (W r) + shift.  Eval mode folds the running statistics.
//   5. v = ReLU(f + p) (relu_nan: NaN stays NaN); pooled[m, c] = max_s v, argmax = the FIRST slot attaining it, or the
//      LAST NaN slot if any (max_pool2d's rule: a slot replaces the maximum when it is larger or NaN).
//   6. Backward: dy = g * [!(pooled <= 0)] at the argmax slot (relu_grad: a NaN maximum passes g).  The feature gradient
//      goes to features_in[row(m, argmax)] for non-empty balls only (the reference zeroes the grouped features of empty balls in place, :99).  The position branch
//      needs only the per-channel sums  sum dy  and  sum dy * r  over the argmax slots (dy is zero everywhere else); with the
//      forward moments they give dW_pos, dgamma, dbeta including the train-mode BN coupling term (pool_bn_grad_kernel).
//      No gradient flows to xyz / new_xyz.
// Limits compiled in: C in {16, 32, 64}, nsample <= 64 (argmax is stored as uint8); anything else -> VC_ERR_UNSUPPORTED.
//
// Deterministic mode (vc_voxel_pool_query_det, vc_voxel_pool_bwd_det; vc_group_points_grad_det in roi_pool.cu): no float
// atomics, every sum in an order fixed by the data alone — never by the grid, the CTA count or the scheduler:
//   D1 moments.  The query points are cut into chunks of DET_CHUNK = 256 consecutive points (a constant).  A point's nine
//      float64 moments are summed over its slots s = lane, lane + 32 per lane, then over the lanes by a fixed xor butterfly;
//      a chunk's points are added by a fixed shared-memory tree into the chunk's own partial; the partials are added in
//      chunk order in float64.  pool_bn_fold_kernel's arithmetic is unchanged.
//   D2 feature gradient.  grad_features_in[r, c] = the fp32 sum, in ascending m and from 0.0, of
//      dy[m, c] = grad_pooled[m, c] * [!(pooled[m, c] <= 0)] over the non-empty m with idx[m, argmax[m, c]] == r; plain adds
//      (a sequential float32 sum on the CPU gives the same bits).  Every row of [0, N) is written, zero where no slot points.
//   D3 channel sums.  The [C, 4] float64 sums of dy and dy * r are partials per chunk of DET_CHUNK query points (a fixed
//      per-thread assignment, a fixed butterfly and a fixed order over the warps), added in chunk order.
//      pool_bn_grad_kernel is unchanged.
//   D4 group_points_grad.  grad_features[row, c] = the fp32 sum over the slots (m, s) of that global row (batch offset
//      from features_batch_cnt + local idx), in ascending (m, s), of grad_out[m, c, s]; the fill slots that repeat the
//      first hit are included, as in the reference.
// D2 and D4 walk the inverse slot map: the slots (m, s) grouped by the row they point at, each group in ascending
// m * nsample + s, built once per call from idx with integer atomics, a scan, a place step and a per-group sort
// (slot_groups_dev, gather2d.cu; long groups are merge-sorted, never in quadratic time).  D2 adds dy[m, c] only at the slot
// s == argmax[m, c] of each listed (m, s), so each (m, c) counts once even where fill slots repeat a row.
#include "voxel_query.cuh"

namespace vc {
namespace {

constexpr int PQ_WARPS = 8;      // query pass: warps per block
constexpr int PB_THREADS = 256;  // pooling passes: threads per block

__global__ void __launch_bounds__(PQ_WARPS * 32) pool_query_kernel(int M, int R1, int R2, int R3, int nsample, float radius,
                                                                   int z_range, int y_range, int x_range,
                                                                   const float* __restrict__ new_xyz,
                                                                   const float* __restrict__ xyz,
                                                                   const int* __restrict__ new_coords,
                                                                   const int* __restrict__ point_indices,
                                                                   int* __restrict__ idx, unsigned char* __restrict__ empty,
                                                                   double* __restrict__ moments) {
    __shared__ double red[PQ_WARPS][9];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // moments: sum rx, ry, rz, then sum rx rx, rx ry, rx rz, ry ry, ry rz, rz rz
    double acc[9];
#pragma unroll
    for (int k = 0; k < 9; k++) acc[k] = 0.0;
    for (int pt = blockIdx.x * PQ_WARPS + warp; pt < M; pt += gridDim.x * PQ_WARPS) {
        const int first = voxel_query_warp(pt, lane, R1, R2, R3, nsample, radius, z_range, y_range, x_range, new_xyz, xyz,
                                           new_coords, point_indices, idx);
        if (lane == 0) empty[pt] = first < 0 ? 1 : 0;
        if (moments && first >= 0) {     // an empty ball's slots have r = 0
            __syncwarp();                // the slots written by the other lanes
            const float nx = new_xyz[pt * 3 + 0], ny = new_xyz[pt * 3 + 1], nz = new_xyz[pt * 3 + 2];
            for (int s = lane; s < nsample; s += 32) {
                const int row = idx[(size_t)pt * nsample + s];
                const float rx = __ldg(xyz + row * 3 + 0) - nx, ry = __ldg(xyz + row * 3 + 1) - ny, rz = __ldg(xyz + row * 3 + 2) - nz;
                const double x = rx, y = ry, z = rz;
                acc[0] += x; acc[1] += y; acc[2] += z;
                acc[3] += x * x; acc[4] += x * y; acc[5] += x * z;
                acc[6] += y * y; acc[7] += y * z; acc[8] += z * z;
            }
        }
    }
    if (!moments) return;
#pragma unroll
    for (int k = 0; k < 9; k++) {
        double v = acc[k];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) red[warp][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < 9) {
        double v = 0.0;
        for (int w = 0; w < PQ_WARPS; w++) v += red[w][threadIdx.x];
        atomicAdd(moments + threadIdx.x, v);
    }
}

// lanes of a warp over the channels of one query point: LPP lanes per point (32 / LPP points per warp), CPL channels per
// lane (c = sub + j * LPP, so the lanes of a point read one feature row coalesced)
template <int C>
struct Lanes {
    static constexpr int LPP = C < 32 ? C : 32;
    static constexpr int CPL = C / LPP;
};

template <int C>
__global__ void __launch_bounds__(PB_THREADS) pool_fwd_kernel(int M, int nsample, const float* __restrict__ features_in,
                                                             const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                                                             const int* __restrict__ idx, const unsigned char* __restrict__ empty,
                                                             const float* __restrict__ w_pos, const float* __restrict__ scale,
                                                             const float* __restrict__ shift, float* __restrict__ pooled,
                                                             unsigned char* __restrict__ argmax) {
    using L = Lanes<C>;
    const int t = blockIdx.x * PB_THREADS + threadIdx.x;
    const int pt = t / L::LPP, sub = t % L::LPP;
    if (pt >= M) return;
    float w0[L::CPL], w1[L::CPL], w2[L::CPL], sc[L::CPL], sh[L::CPL], best[L::CPL];
    int arg[L::CPL];
#pragma unroll
    for (int j = 0; j < L::CPL; j++) {
        const int c = sub + j * L::LPP;
        w0[j] = __ldg(w_pos + c * 3 + 0); w1[j] = __ldg(w_pos + c * 3 + 1); w2[j] = __ldg(w_pos + c * 3 + 2);
        sc[j] = __ldg(scale + c); sh[j] = __ldg(shift + c);
        best[j] = -INFINITY; arg[j] = 0;
    }
    const bool emp = empty[pt] != 0;
    const float nx = new_xyz[pt * 3 + 0], ny = new_xyz[pt * 3 + 1], nz = new_xyz[pt * 3 + 2];
    const int* rows = idx + (size_t)pt * nsample;
#pragma unroll 4
    for (int s = 0; s < nsample; s++) {
        float rx = 0.f, ry = 0.f, rz = 0.f;
        float f[L::CPL];
#pragma unroll
        for (int j = 0; j < L::CPL; j++) f[j] = 0.f;
        if (!emp) {
            const int row = __ldg(rows + s);
            rx = __ldg(xyz + row * 3 + 0) - nx; ry = __ldg(xyz + row * 3 + 1) - ny; rz = __ldg(xyz + row * 3 + 2) - nz;
#pragma unroll
            for (int j = 0; j < L::CPL; j++) f[j] = __ldg(features_in + (size_t)row * C + sub + j * L::LPP);
        }
#pragma unroll
        for (int j = 0; j < L::CPL; j++) {
            const float x = w0[j] * rx + w1[j] * ry + w2[j] * rz;
            const float v = relu_nan(f[j] + (sc[j] * x + sh[j]));
            if (v > best[j] || v != v) { best[j] = v; arg[j] = s; }
        }
    }
#pragma unroll
    for (int j = 0; j < L::CPL; j++) {
        const size_t o = (size_t)pt * C + sub + j * L::LPP;
        pooled[o] = best[j];
        argmax[o] = (unsigned char)arg[j];
    }
}

template <int C>
__global__ void __launch_bounds__(PB_THREADS) pool_bwd_kernel(int M, int nsample, const float* __restrict__ grad_pooled,
                                                             const float* __restrict__ pooled,
                                                             const unsigned char* __restrict__ argmax,
                                                             const int* __restrict__ idx, const unsigned char* __restrict__ empty,
                                                             const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                                                             float* __restrict__ grad_features_in, double* __restrict__ sums) {
    using L = Lanes<C>;
    constexpr int WARPS = PB_THREADS / 32;
    __shared__ double red[WARPS][C][4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = threadIdx.x % L::LPP;
    double acc[L::CPL][4];
#pragma unroll
    for (int j = 0; j < L::CPL; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
    const int step = gridDim.x * (PB_THREADS / L::LPP);
    for (int pt = (blockIdx.x * PB_THREADS + threadIdx.x) / L::LPP; pt < M; pt += step) {
        const bool emp = empty[pt] != 0;
        const float nx = new_xyz[pt * 3 + 0], ny = new_xyz[pt * 3 + 1], nz = new_xyz[pt * 3 + 2];
#pragma unroll
        for (int j = 0; j < L::CPL; j++) {
            const size_t o = (size_t)pt * C + sub + j * L::LPP;
            const float dy = relu_grad(pooled[o], grad_pooled[o]);
            if (dy == 0.f) continue;
            acc[j][0] += dy;
            if (emp) continue;
            const int row = idx[(size_t)pt * nsample + argmax[o]];
            atomicAdd(grad_features_in + (size_t)row * C + sub + j * L::LPP, dy);
            const float rx = __ldg(xyz + row * 3 + 0) - nx, ry = __ldg(xyz + row * 3 + 1) - ny, rz = __ldg(xyz + row * 3 + 2) - nz;
            acc[j][1] += (double)dy * rx; acc[j][2] += (double)dy * ry; acc[j][3] += (double)dy * rz;
        }
    }
    // the PPW points of a warp share channels: fold them, then the warps of the block, then one atomic per value
#pragma unroll
    for (int j = 0; j < L::CPL; j++)
#pragma unroll
        for (int k = 0; k < 4; k++) {
            double v = acc[j][k];
            for (int o = L::LPP; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane < L::LPP) red[warp][sub + j * L::LPP][k] = v;
        }
    __syncthreads();
    for (int q = threadIdx.x; q < C * 4; q += PB_THREADS) {
        double v = 0.0;
        for (int w = 0; w < WARPS; w++) v += red[w][q / 4][q % 4];
        atomicAdd(sums + q, v);
    }
}

// moments m[9] -> E[r] (3) and Cov(r) (3 x 3) over n slots
__device__ __forceinline__ void moments_to_cov(const double* __restrict__ m, double n, double er[3], double cov[3][3]) {
    const double s[3][3] = {{m[3], m[4], m[5]}, {m[4], m[6], m[7]}, {m[5], m[7], m[8]}};
    for (int i = 0; i < 3; i++) er[i] = m[i] / n;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) cov[i][j] = s[i][j] / n - er[i] * er[j];
}

// one thread per channel: the BatchNorm2d of the position branch (rule 4), folded; running statistics as torch's
// _BatchNorm (momentum < 0: cumulative average); stat [C, 2] = mean, invstd for the backward
__global__ void pool_bn_fold_kernel(int C, double n, const double* __restrict__ n_dev, int training, const double* __restrict__ moments,
                                    const float* __restrict__ w_pos, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, float* __restrict__ running_mean,
                                    float* __restrict__ running_var, long long* __restrict__ num_batches_tracked, double eps,
                                    double momentum, float* __restrict__ scale, float* __restrict__ shift,
                                    double* __restrict__ stat) {
    const int c = threadIdx.x;
    if (n_dev != nullptr) n = *n_dev;   // (SyncBatchNorm: the slot count over all ranks)
    const long long nbt = training ? num_batches_tracked[0] + 1 : 0;
    __syncthreads();
    if (training && c == 0) num_batches_tracked[0] = nbt;
    if (c >= C) return;
    double mean, var;
    if (training) {
        double er[3], cov[3][3];
        moments_to_cov(moments, n, er, cov);
        const double w[3] = {w_pos[c * 3 + 0], w_pos[c * 3 + 1], w_pos[c * 3 + 2]};
        mean = w[0] * er[0] + w[1] * er[1] + w[2] * er[2];
        var = 0.0;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) var += w[i] * cov[i][j] * w[j];
        var = var > 0.0 ? var : 0.0;
        const double f = momentum < 0.0 ? 1.0 / (double)nbt : momentum;
        running_mean[c] = (float)((1.0 - f) * running_mean[c] + f * mean);
        running_var[c] = (float)((1.0 - f) * running_var[c] + f * var * n / (n > 1.0 ? n - 1.0 : 1.0));
    } else {
        mean = running_mean[c];
        var = running_var[c];
    }
    const double invstd = 1.0 / sqrt(var + eps);
    const double sc = gamma[c] * invstd;
    scale[c] = (float)sc;
    shift[c] = (float)(beta[c] - mean * sc);
    stat[c * 2 + 0] = mean;
    stat[c * 2 + 1] = invstd;
}

// one thread per channel: dW_pos, dgamma, dbeta from the per-channel sums of the pooling backward (rule 6)
// gsums / n_dev (SyncBatchNorm, else NULL): the all-reduced sums and slot count; sums and moments stay the rank's own
__global__ void pool_bn_grad_kernel(int C, double n, const double* __restrict__ n_dev, int training, const double* __restrict__ sums,
                                    const double* __restrict__ gsums, const double* __restrict__ moments, const float* __restrict__ w_pos,
                                    const float* __restrict__ gamma, const double* __restrict__ stat, float* __restrict__ dw,
                                    float* __restrict__ dgamma, float* __restrict__ dbeta) {
    const int c = threadIdx.x;
    if (c >= C) return;
    const double w[3] = {w_pos[c * 3 + 0], w_pos[c * 3 + 1], w_pos[c * 3 + 2]};
    const double mean = stat[c * 2 + 0], invstd = stat[c * 2 + 1];
    const double sdy = sums[c * 4 + 0], sdyr[3] = {sums[c * 4 + 1], sums[c * 4 + 2], sums[c * 4 + 3]};
    // x = w r before BN, xhat = (x - mean) invstd:  dbeta = sum dy, dgamma = sum dy xhat
    const double dg = (sdyr[0] * w[0] + sdyr[1] * w[1] + sdyr[2] * w[2] - mean * sdy) * invstd;
    const double* gs = gsums != nullptr ? gsums : sums;
    const double gsdy = gs[c * 4 + 0];
    const double gdg = gsums != nullptr ? (gs[c * 4 + 1] * w[0] + gs[c * 4 + 2] * w[1] + gs[c * 4 + 3] * w[2] - mean * gsdy) * invstd : dg;
    if (n_dev != nullptr) n = *n_dev;
    const double k = gamma[c] * invstd;
    for (int j = 0; j < 3; j++) {
        double d = sdyr[j];
        if (training) {
            // dx = gamma invstd (dy - sum dy / n - xhat sum dy xhat / n) over all n slots, dW = sum dx r, with
            // sum xhat r_j = invstd (sum_i (sum r_j r_i) w_i - mean sum r_j)
            const double s[3][3] = {{moments[3], moments[4], moments[5]}, {moments[4], moments[6], moments[7]},
                                    {moments[5], moments[7], moments[8]}};
            const double sxr = (s[j][0] * w[0] + s[j][1] * w[1] + s[j][2] * w[2] - mean * moments[j]) * invstd;
            d = d - gsdy / n * moments[j] - gdg / n * sxr;
        }
        dw[c * 3 + j] = (float)(k * d);
    }
    dgamma[c] = (float)dg;
    dbeta[c] = (float)sdy;
}

// ---- deterministic mode (D1 - D3) ----
constexpr int DET_CHUNK = 256;   // query points per partial of D1 and D3: a constant, never derived from the grid

__device__ __forceinline__ int det_chunks(int M) { return (M + DET_CHUNK - 1) / DET_CHUNK; }

// D1: the query of vc_voxel_pool_query, and part[chunk][9] = the chunk's moments (fixed order, see the file header)
__global__ void __launch_bounds__(PQ_WARPS * 32) pool_query_det_kernel(int M, int R1, int R2, int R3, int nsample, float radius,
                                                                       int z_range, int y_range, int x_range,
                                                                       const float* __restrict__ new_xyz,
                                                                       const float* __restrict__ xyz,
                                                                       const int* __restrict__ new_coords,
                                                                       const int* __restrict__ point_indices,
                                                                       int* __restrict__ idx, unsigned char* __restrict__ empty,
                                                                       double* __restrict__ part) {
    __shared__ double pm[DET_CHUNK][9];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int chunks = det_chunks(M);
    for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        for (int p = warp; p < DET_CHUNK; p += PQ_WARPS) {
            const int pt = ch * DET_CHUNK + p;   // warp-uniform
            double acc[9];
#pragma unroll
            for (int k = 0; k < 9; k++) acc[k] = 0.0;
            if (pt < M) {
                const int first = voxel_query_warp(pt, lane, R1, R2, R3, nsample, radius, z_range, y_range, x_range, new_xyz,
                                                   xyz, new_coords, point_indices, idx);
                if (lane == 0) empty[pt] = first < 0 ? 1 : 0;
                if (first >= 0) {
                    __syncwarp();
                    const float nx = new_xyz[pt * 3 + 0], ny = new_xyz[pt * 3 + 1], nz = new_xyz[pt * 3 + 2];
                    for (int s = lane; s < nsample; s += 32) {
                        const int row = idx[(size_t)pt * nsample + s];
                        const float rx = __ldg(xyz + row * 3 + 0) - nx, ry = __ldg(xyz + row * 3 + 1) - ny,
                                    rz = __ldg(xyz + row * 3 + 2) - nz;
                        const double x = rx, y = ry, z = rz;
                        acc[0] += x; acc[1] += y; acc[2] += z;
                        acc[3] += x * x; acc[4] += x * y; acc[5] += x * z;
                        acc[6] += y * y; acc[7] += y * z; acc[8] += z * z;
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < 9; k++) {
                double v = acc[k];
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == 0) pm[p][k] = v;
            }
        }
        __syncthreads();
        for (int st = DET_CHUNK / 2; st > 0; st >>= 1) {
            for (int q = threadIdx.x; q < st * 9; q += blockDim.x) pm[q / 9][q % 9] += pm[q / 9 + st][q % 9];
            __syncthreads();
        }
        if (threadIdx.x < 9) part[(size_t)ch * 9 + threadIdx.x] = pm[0][threadIdx.x];
        __syncthreads();
    }
}

// out[q] = sum over the chunks, in chunk order, of part[chunk][q] (float64; one thread per value)
__global__ void chunk_sum_kernel(const double* __restrict__ part, int chunks, int width, double* __restrict__ out) {
    const int q = threadIdx.x;
    if (q >= width) return;
    double v = 0.0;
    for (int ch = 0; ch < chunks; ch++) v += part[(size_t)ch * width + q];
    out[q] = v;
}

// D1 / D2 / D4: the slot keys of the fused pooling: the global row of (m, s), -1 for an empty ball (or a row outside [0, N))
__global__ void pool_slot_key_kernel(int E, int N, int nsample, const int* __restrict__ idx,
                                     const unsigned char* __restrict__ empty, int32_t* __restrict__ key) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= E) return;
    const int row = idx[t];
    key[t] = (empty[t / nsample] == 0 && row >= 0 && row < N) ? row : -1;
}

// D2: one row per LPP lanes, its slot list walked in ascending (m, s); every row of [0, N) written
template <int C>
__global__ void __launch_bounds__(PB_THREADS) pool_grad_rows_det_kernel(int N, int nsample, const float* __restrict__ grad_pooled,
                                                                       const float* __restrict__ pooled,
                                                                       const unsigned char* __restrict__ argmax,
                                                                       const int* __restrict__ cnt, const int* __restrict__ off,
                                                                       const int32_t* __restrict__ slots,
                                                                       float* __restrict__ grad_features_in) {
    using L = Lanes<C>;
    const int t = blockIdx.x * PB_THREADS + threadIdx.x;
    const int r = t / L::LPP, sub = t % L::LPP;
    if (r >= N) return;
    float acc[L::CPL];
#pragma unroll
    for (int j = 0; j < L::CPL; j++) acc[j] = 0.f;
    const int n = cnt[r];
    const int32_t* p = slots + off[r];
    for (int i = 0; i < n; i++) {
        const int slot = __ldg(p + i);
        const int m = slot / nsample, s = slot - m * nsample;
#pragma unroll
        for (int j = 0; j < L::CPL; j++) {
            const size_t o = (size_t)m * C + sub + j * L::LPP;
            if (__ldg(argmax + o) == s) acc[j] = __fadd_rn(acc[j], relu_grad(__ldg(pooled + o), __ldg(grad_pooled + o)));
        }
    }
#pragma unroll
    for (int j = 0; j < L::CPL; j++) grad_features_in[(size_t)r * C + sub + j * L::LPP] = acc[j];
}

// D3: part[chunk][C][4] = the chunk's per-channel sums of dy and dy * r (the terms of pool_bwd_kernel, fixed order)
template <int C>
__global__ void __launch_bounds__(PB_THREADS) pool_sums_det_kernel(int M, int nsample, const float* __restrict__ grad_pooled,
                                                                  const float* __restrict__ pooled,
                                                                  const unsigned char* __restrict__ argmax,
                                                                  const int* __restrict__ idx, const unsigned char* __restrict__ empty,
                                                                  const float* __restrict__ xyz, const float* __restrict__ new_xyz,
                                                                  double* __restrict__ part) {
    using L = Lanes<C>;
    constexpr int WARPS = PB_THREADS / 32, PPB = PB_THREADS / L::LPP;
    __shared__ double red[WARPS][C][4];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = threadIdx.x % L::LPP, pl = threadIdx.x / L::LPP;
    const int chunks = det_chunks(M);
    for (int ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        double acc[L::CPL][4];
#pragma unroll
        for (int j = 0; j < L::CPL; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
        const int end = min(M, (ch + 1) * DET_CHUNK);
        for (int pt = ch * DET_CHUNK + pl; pt < end; pt += PPB) {
            const bool emp = empty[pt] != 0;
            const float nx = new_xyz[pt * 3 + 0], ny = new_xyz[pt * 3 + 1], nz = new_xyz[pt * 3 + 2];
#pragma unroll
            for (int j = 0; j < L::CPL; j++) {
                const size_t o = (size_t)pt * C + sub + j * L::LPP;
                const float dy = relu_grad(pooled[o], grad_pooled[o]);
                if (dy == 0.f) continue;
                acc[j][0] += dy;
                if (emp) continue;
                const int row = idx[(size_t)pt * nsample + argmax[o]];
                const float rx = __ldg(xyz + row * 3 + 0) - nx, ry = __ldg(xyz + row * 3 + 1) - ny, rz = __ldg(xyz + row * 3 + 2) - nz;
                acc[j][1] += (double)dy * rx; acc[j][2] += (double)dy * ry; acc[j][3] += (double)dy * rz;
            }
        }
#pragma unroll
        for (int j = 0; j < L::CPL; j++)
#pragma unroll
            for (int k = 0; k < 4; k++) {
                double v = acc[j][k];
                for (int o = L::LPP; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane < L::LPP) red[warp][sub + j * L::LPP][k] = v;
            }
        __syncthreads();
        for (int q = threadIdx.x; q < C * 4; q += PB_THREADS) {
            double v = 0.0;
            for (int w = 0; w < WARPS; w++) v += red[w][q / 4][q % 4];
            part[(size_t)ch * C * 4 + q] = v;
        }
        __syncthreads();
    }
}

int pool_grid_cap(int per_sm) {
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return per_sm * sms;
}

// grid of the deterministic grid-stride kernels: the work's own size, capped at 8 CTAs per SM or vc_voxel_pool_det_config
int det_grid(long long need) {
    const int cap = g_pool_det_ctas > 0 ? g_pool_det_ctas : pool_grid_cap(8);
    return need < 1 ? 1 : (need < cap ? (int)need : cap);
}

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

bool channels_supported(int C) { return C == 16 || C == 32 || C == 64; }

}  // namespace

int g_pool_det_ctas = 0;

}  // namespace vc

using namespace vc;

extern "C" int vc_voxel_pool_det_config(int max_ctas) {
    VC_CHECK_ARG(max_ctas >= 0, "vc_voxel_pool_det_config: max_ctas %d < 0", max_ctas);
    g_pool_det_ctas = max_ctas;
    return VC_OK;
}

extern "C" int vc_voxel_pool_query(int M, int R1, int R2, int R3, int nsample, float radius, int z_range, int y_range,
                                   int x_range, const float* new_xyz, const float* xyz, const int32_t* new_coords,
                                   const int32_t* point_indices, int32_t* idx, unsigned char* empty_mask, double* moments,
                                   vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(M >= 0 && R1 > 0 && R2 > 0 && R3 > 0 && nsample > 0 && z_range >= 0 && y_range >= 0 && x_range >= 0,
                 "bad voxel_pool_query arguments");
    if (nsample > VC_VOXEL_POOL_MAX_NSAMPLE) {
        set_error("voxel_pool_query: nsample %d > %d is not compiled in", nsample, VC_VOXEL_POOL_MAX_NSAMPLE);
        return VC_ERR_UNSUPPORTED;
    }
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(new_xyz && xyz && new_coords && point_indices && idx && empty_mask, "null pointer");
    const int blocks = cdiv(M, PQ_WARPS) < pool_grid_cap(8) ? cdiv(M, PQ_WARPS) : pool_grid_cap(8);
    pool_query_kernel<<<blocks, PQ_WARPS * 32, 0, stream>>>(M, R1, R2, R3, nsample, radius, z_range, y_range, x_range, new_xyz,
                                                            xyz, new_coords, point_indices, idx, empty_mask, moments);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_bn_fold(int C, long long n, int training, const double* moments, const float* w_pos,
                                     const float* gamma, const float* beta, float* running_mean, float* running_var,
                                     long long* num_batches_tracked, double eps, double momentum, float* scale, float* shift,
                                     double* stat, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(C > 0 && C <= 1024 && n > 0, "bad voxel_pool_bn_fold arguments");
    VC_CHECK_ARG(w_pos && gamma && beta && running_mean && running_var && scale && shift && stat, "null pointer");
    VC_CHECK_ARG(!training || (moments && num_batches_tracked), "train mode needs moments and num_batches_tracked");
    pool_bn_fold_kernel<<<1, (C + 31) / 32 * 32, 0, stream>>>(C, (double)n, nullptr, training, moments, w_pos, gamma, beta, running_mean,
                                                              running_var, num_batches_tracked, eps, momentum, scale, shift,
                                                              stat);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_bn_grad(int C, long long n, int training, const double* sums, const double* moments,
                                     const float* w_pos, const float* gamma, const double* stat, float* dw, float* dgamma,
                                     float* dbeta, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(C > 0 && C <= 1024 && n > 0, "bad voxel_pool_bn_grad arguments");
    VC_CHECK_ARG(sums && w_pos && gamma && stat && dw && dgamma && dbeta && (!training || moments), "null pointer");
    pool_bn_grad_kernel<<<1, (C + 31) / 32 * 32, 0, stream>>>(C, (double)n, nullptr, training, sums, nullptr, moments, w_pos, gamma,
                                                              stat, dw, dgamma, dbeta);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_bn_fold_sync(int C, int training, const double* moments10, const float* w_pos, const float* gamma,
                                          const float* beta, float* running_mean, float* running_var,
                                          long long* num_batches_tracked, double eps, double momentum, float* scale, float* shift,
                                          double* stat, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(C > 0 && C <= 1024 && training, "bad voxel_pool_bn_fold_sync arguments (train mode only)");
    VC_CHECK_ARG(moments10 && num_batches_tracked && w_pos && gamma && beta && running_mean && running_var && scale && shift && stat,
                 "null pointer");
    pool_bn_fold_kernel<<<1, (C + 31) / 32 * 32, 0, stream>>>(C, 1.0, moments10 + 9, training, moments10, w_pos, gamma, beta,
                                                              running_mean, running_var, num_batches_tracked, eps, momentum, scale,
                                                              shift, stat);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_bn_grad_sync(int C, const double* n_glob, const double* sums, const double* gsums,
                                          const double* moments, const float* w_pos, const float* gamma, const double* stat,
                                          float* dw, float* dgamma, float* dbeta, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(C > 0 && C <= 1024, "bad voxel_pool_bn_grad_sync arguments");
    VC_CHECK_ARG(n_glob && sums && gsums && moments && w_pos && gamma && stat && dw && dgamma && dbeta, "null pointer");
    pool_bn_grad_kernel<<<1, (C + 31) / 32 * 32, 0, stream>>>(C, 1.0, n_glob, 1, sums, gsums, moments, w_pos, gamma, stat, dw,
                                                              dgamma, dbeta);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_fwd(int M, int C, int nsample, const float* features_in, const float* xyz, const float* new_xyz,
                                 const int32_t* idx, const unsigned char* empty_mask, const float* w_pos, const float* scale,
                                 const float* shift, float* pooled, unsigned char* argmax, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(M >= 0 && C > 0 && nsample > 0, "bad voxel_pool_fwd arguments");
    if (!channels_supported(C) || nsample > VC_VOXEL_POOL_MAX_NSAMPLE) {
        set_error("voxel_pool_fwd: C = %d, nsample = %d is not compiled in (C in {16, 32, 64}, nsample <= %d)", C, nsample,
                  VC_VOXEL_POOL_MAX_NSAMPLE);
        return VC_ERR_UNSUPPORTED;
    }
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(features_in && xyz && new_xyz && idx && empty_mask && w_pos && scale && shift && pooled && argmax,
                 "null pointer");
    const int lpp = C < 32 ? C : 32;
    const int blocks = cdiv((long long)M * lpp, PB_THREADS);
#define VC_POOL_FWD(CC)                                                                                                \
    pool_fwd_kernel<CC><<<blocks, PB_THREADS, 0, stream>>>(M, nsample, features_in, xyz, new_xyz, idx, empty_mask, w_pos, \
                                                           scale, shift, pooled, argmax)
    if (C == 16) VC_POOL_FWD(16);
    else if (C == 32) VC_POOL_FWD(32);
    else VC_POOL_FWD(64);
#undef VC_POOL_FWD
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel_pool_bwd(int M, int C, int N, int nsample, const float* grad_pooled, const float* pooled,
                                 const unsigned char* argmax, const int32_t* idx, const unsigned char* empty_mask,
                                 const float* xyz, const float* new_xyz, float* grad_features_in, double* sums,
                                 vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(M >= 0 && C > 0 && N >= 0 && nsample > 0, "bad voxel_pool_bwd arguments");
    if (!channels_supported(C) || nsample > VC_VOXEL_POOL_MAX_NSAMPLE) {
        set_error("voxel_pool_bwd: C = %d, nsample = %d is not compiled in (C in {16, 32, 64}, nsample <= %d)", C, nsample,
                  VC_VOXEL_POOL_MAX_NSAMPLE);
        return VC_ERR_UNSUPPORTED;
    }
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(grad_pooled && pooled && argmax && idx && empty_mask && xyz && new_xyz && grad_features_in && sums,
                 "null pointer");
    const int lpp = C < 32 ? C : 32;
    const int need = cdiv((long long)M * lpp, PB_THREADS), cap = pool_grid_cap(8);
    const int blocks = need < cap ? need : cap;
#define VC_POOL_BWD(CC)                                                                                              \
    pool_bwd_kernel<CC><<<blocks, PB_THREADS, 0, stream>>>(M, nsample, grad_pooled, pooled, argmax, idx, empty_mask, xyz, \
                                                           new_xyz, grad_features_in, sums)
    if (C == 16) VC_POOL_BWD(16);
    else if (C == 32) VC_POOL_BWD(32);
    else VC_POOL_BWD(64);
#undef VC_POOL_BWD
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_voxel_pool_query_det_ws_bytes(int M) {
    return M > 0 ? al256((size_t)cdiv(M, DET_CHUNK) * 9 * sizeof(double)) : 256;
}

extern "C" int vc_voxel_pool_query_det(int M, int R1, int R2, int R3, int nsample, float radius, int z_range, int y_range,
                                       int x_range, const float* new_xyz, const float* xyz, const int32_t* new_coords,
                                       const int32_t* point_indices, int32_t* idx, unsigned char* empty_mask, double* moments,
                                       void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(M >= 0 && R1 > 0 && R2 > 0 && R3 > 0 && nsample > 0 && z_range >= 0 && y_range >= 0 && x_range >= 0,
                 "bad voxel_pool_query_det arguments");
    if (nsample > VC_VOXEL_POOL_MAX_NSAMPLE) {
        set_error("voxel_pool_query_det: nsample %d > %d is not compiled in", nsample, VC_VOXEL_POOL_MAX_NSAMPLE);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(moments != nullptr, "voxel_pool_query_det: moments is NULL");
    if (M == 0) {
        VC_CUDA(cudaMemsetAsync(moments, 0, 9 * sizeof(double), stream));
        return VC_OK;
    }
    VC_CHECK_ARG(new_xyz && xyz && new_coords && point_indices && idx && empty_mask && ws, "null pointer");
    if (ws_bytes < vc_voxel_pool_query_det_ws_bytes(M)) {
        set_error("voxel_pool_query_det workspace %zu < %zu", ws_bytes, vc_voxel_pool_query_det_ws_bytes(M));
        return VC_ERR_WORKSPACE;
    }
    const int chunks = cdiv(M, DET_CHUNK);
    double* part = (double*)ws;
    pool_query_det_kernel<<<det_grid(chunks), PQ_WARPS * 32, 0, stream>>>(M, R1, R2, R3, nsample, radius, z_range, y_range,
                                                                         x_range, new_xyz, xyz, new_coords, point_indices,
                                                                         idx, empty_mask, part);
    VC_LAUNCH_CHECK();
    chunk_sum_kernel<<<1, 32, 0, stream>>>(part, chunks, 9, moments);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_voxel_pool_bwd_det_ws_bytes(int M, int C, int N, int nsample) {
    if (M < 0 || C <= 0 || N < 0 || nsample <= 0) return 0;
    return slot_groups_bytes(M * nsample, N) + al256((size_t)cdiv(M, DET_CHUNK) * C * 4 * sizeof(double));
}

extern "C" int vc_voxel_pool_bwd_det(int M, int C, int N, int nsample, const float* grad_pooled, const float* pooled,
                                     const unsigned char* argmax, const int32_t* idx, const unsigned char* empty_mask,
                                     const float* xyz, const float* new_xyz, float* grad_features_in, double* sums, void* ws,
                                     size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(M >= 0 && C > 0 && N >= 0 && nsample > 0, "bad voxel_pool_bwd_det arguments");
    if (!channels_supported(C) || nsample > VC_VOXEL_POOL_MAX_NSAMPLE) {
        set_error("voxel_pool_bwd_det: C = %d, nsample = %d is not compiled in (C in {16, 32, 64}, nsample <= %d)", C, nsample,
                  VC_VOXEL_POOL_MAX_NSAMPLE);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG((long long)M * nsample <= 0x7fffffffLL, "voxel_pool_bwd_det: %d x %d slots", M, nsample);
    VC_CHECK_ARG(sums && (N == 0 || grad_features_in), "null pointer");
    if (M == 0) {
        if (N > 0) VC_CUDA(cudaMemsetAsync(grad_features_in, 0, (size_t)N * C * sizeof(float), stream));
        VC_CUDA(cudaMemsetAsync(sums, 0, (size_t)C * 4 * sizeof(double), stream));
        return VC_OK;
    }
    VC_CHECK_ARG(grad_pooled && pooled && argmax && idx && empty_mask && xyz && new_xyz && ws, "null pointer");
    if (ws_bytes < vc_voxel_pool_bwd_det_ws_bytes(M, C, N, nsample)) {
        set_error("voxel_pool_bwd_det workspace %zu < %zu", ws_bytes, vc_voxel_pool_bwd_det_ws_bytes(M, C, N, nsample));
        return VC_ERR_WORKSPACE;
    }
    const int E = M * nsample, chunks = cdiv(M, DET_CHUNK), lpp = C < 32 ? C : 32;
    const SlotGroups P = slot_groups_carve(ws, E, N);
    double* part = (double*)((char*)ws + slot_groups_bytes(E, N));
    if (N > 0) {
        pool_slot_key_kernel<<<cdiv(E, 256), 256, 0, stream>>>(E, N, nsample, idx, empty_mask, P.key);
        VC_LAUNCH_CHECK();
        const int rc = slot_groups_dev(E, N, P, g_pool_det_ctas, stream);
        if (rc) return rc;
    }
#define VC_POOL_BWD_DET(CC)                                                                                                  \
    do {                                                                                                                     \
        if (N > 0) {                                                                                                         \
            pool_grad_rows_det_kernel<CC><<<cdiv((long long)N * lpp, PB_THREADS), PB_THREADS, 0, stream>>>(                  \
                N, nsample, grad_pooled, pooled, argmax, P.cnt, P.off, P.rows, grad_features_in);                            \
            VC_LAUNCH_CHECK();                                                                                               \
        }                                                                                                                    \
        pool_sums_det_kernel<CC><<<det_grid(chunks), PB_THREADS, 0, stream>>>(M, nsample, grad_pooled, pooled, argmax, idx,   \
                                                                              empty_mask, xyz, new_xyz, part);               \
        VC_LAUNCH_CHECK();                                                                                                   \
    } while (0)
    if (C == 16) VC_POOL_BWD_DET(16);
    else if (C == 32) VC_POOL_BWD_DET(32);
    else VC_POOL_BWD_DET(64);
#undef VC_POOL_BWD_DET
    chunk_sum_kernel<<<1, C * 4, 0, stream>>>(part, chunks, C * 4, sums);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
