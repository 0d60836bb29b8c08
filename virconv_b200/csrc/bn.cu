// BatchNorm1d(eps, momentum) + ReLU over the active rows of a sparse tensor — sm_90a.
//
// Replaces the `norm_fn(out_channels)` / `nn.ReLU()` members of every spconv.SparseSequential
// (spconv_backbone.py:101-105, :160 eps=1e-3 momentum=0.01, :561-567).  HBM-bound elementwise work.
//
// Statistics never get their own pass: the conv epilogue adds each tile's channel sums (sum x, sum x^2) into a
// [2, C] float64 accumulator with atomics, and the apply kernel below derives mean / invstd / scale / shift from
// it per thread (block 0 also publishes them for backward and updates the running statistics).  Backward is two
// kernels: a reduce that accumulates (sum g, sum g*xhat) the same way, and an apply that derives its per-channel
// coefficients from those sums.  The float64 accumulators make the fp32-rounded results independent of the
// atomic arrival order for all practical purposes (each addend is an fp32 tile partial, < 2^12 of them).
#include <cooperative_groups.h>

#include "bn_common.cuh"

namespace vc {

// y = relu(x*scale + shift); train: statistics from `sums`, eval: from the running buffers.
// stats_out [4, c] = scale, shift, mean, invstd (block 0).  grid-stride over float4 with stride % (c/4) == 0.
__global__ void __launch_bounds__(256) bn_apply_relu_kernel(
    const float4* __restrict__ x, const double* __restrict__ sums, int n_rows, const int* __restrict__ n_dev, int c,
    const float* __restrict__ gamma, const float* __restrict__ beta, float* running_mean, float* running_var,
    long long* num_batches_tracked, float momentum, float eps, int training, float4* __restrict__ y, int y_ld4,
    uint2* __restrict__ y_bf16, int yb_ld4, float* __restrict__ stats_out, int relu, int tail_zero,
    const double* __restrict__ n_glob) {
    // n_glob (SyncBatchNorm, else NULL): the row count over all ranks the statistics divide by, sums then being the
    // all-reduced ones.
    // n_dev (static mode): the row count lives in device memory, n_rows is the capacity of the buffers; with tail_zero the
    // rows [count, capacity) of the outputs are written as zeros (published tensors keep a defined tail).
    // y_ld4 / yb_ld4: row pitch of the outputs in float4 / uint2 units (>= c/4: the output may be a column slice of a
    // wider matrix — the concat of an NRConv block is written in place, spconv_backbone.py:227).
    const int cap_rows = n_rows;
    if (n_dev != nullptr) n_rows = min(n_rows, __ldg(n_dev));
    const int c4 = c / 4;
    const size_t n4 = (size_t)n_rows * c4;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const int cg = (int)(i0 % c4);
    __shared__ float sc_s[128], sh_s[128];
    if (threadIdx.x < c)   // one thread per channel derives scale / shift (float64 once per block, not per thread)
        bn_channel(training ? sums[threadIdx.x] : 0.0, training ? sums[c + threadIdx.x] : 0.0, threadIdx.x, c,
                   n_glob != nullptr ? (int)__ldg(n_glob) : n_rows, gamma, beta,
                   running_mean, running_var, momentum, eps, training, sc_s, sh_s, blockIdx.x == 0, stats_out);
    if (training && blockIdx.x == 0 && threadIdx.x == 0 && num_batches_tracked != nullptr) *num_batches_tracked += 1;
    __syncthreads();
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sc[j] = sc_s[cg * 4 + j];
        sh[j] = sh_s[cg * 4 + j];
    }
    const bool dense = y_ld4 == c4 && yb_ld4 == c4;
    for (size_t i = i0; i < n4; i += stride) {
        const float4 v = bn_relu4(x[i], sc, sh, relu);
        const size_t r = i / c4;
        const size_t oy = dense ? i : r * y_ld4 + cg, ob = dense ? i : r * yb_ld4 + cg;
        if (y != nullptr) y[oy] = v;
        if (y_bf16 != nullptr) y_bf16[ob] = pack_bf16x4(v);   // shadow copy: the next conv's tensor-core operand
    }
    if (tail_zero && cap_rows > n_rows) {
        const size_t t4 = (size_t)cap_rows * c4;
        for (size_t i = n4 + i0; i < t4; i += stride) {
            const size_t r = i / c4;
            if (y != nullptr) y[r * y_ld4 + cg] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (y_bf16 != nullptr) y_bf16[r * yb_ld4 + cg] = make_uint2(0u, 0u);
        }
    }
}

// ---- deterministic mode (torch.use_deterministic_algorithms): fixed-order float64 reductions ------------------------------
// Partials are keyed by a unit of work that does not depend on the launch (a conv's 128-row tile, a BN_DET_ROWS chunk of
// rows); they are summed in that unit's order, so the result is bit-identical for every grid size and every schedule.

// sums[j] = sum over parts p < n_parts of part[p][j], j < 2c: one block per column, thread t takes parts t, t + 256, ...
// in ascending order, then a fixed tree.  n_parts = cdiv(rows, rows_per_part), rows from n_dev when given.
__global__ void __launch_bounds__(256) bn_sums_reduce_kernel(const double* __restrict__ part, int cap_rows, const int* __restrict__ n_dev,
                                                             int rows_per_part, int c, double* __restrict__ sums) {
    __shared__ double red[256];
    const int rows = n_dev != nullptr ? min(cap_rows, __ldg(n_dev)) : cap_rows;
    const int n_parts = (rows + rows_per_part - 1) / rows_per_part;
    const double v = bn_sums_column(part, n_parts, c, blockIdx.x, red);
    if (threadIdx.x == 0) sums[blockIdx.x] = v;
}

// BN backward, deterministic: chunk ch = rows [ch * BN_DET_ROWS, ...) -> part[ch][2][c] = (sum g, sum g*xhat) in float64.
// Thread (cg, rl) takes rows rl, rl + rowlanes, ... of the chunk; the row lanes are added in lane order.  Needs
// rowlanes * 2 * c floats of shared memory (shf) and a __syncthreads-uniform call.
__device__ __forceinline__ void bn_bwd_chunk_partials(const float4* __restrict__ dy, int dy_ld4, const float4* __restrict__ x,
                                                      const float* __restrict__ stats, int n, int c, double* __restrict__ part,
                                                      float* shf) {
    const int c4 = c / 4, cg = threadIdx.x % c4, rl = threadIdx.x / c4, rowlanes = blockDim.x / c4;
    const float4 sc = reinterpret_cast<const float4*>(stats)[cg];
    const float4 sh = reinterpret_cast<const float4*>(stats + c)[cg];
    const float4 m = reinterpret_cast<const float4*>(stats + 2 * c)[cg];
    const float4 is = reinterpret_cast<const float4*>(stats + 3 * c)[cg];
    const int n_chunks = (n + BN_DET_ROWS - 1) / BN_DET_ROWS;
    for (int chk = blockIdx.x; chk < n_chunks; chk += gridDim.x) {
        const int end = min(n, (chk + 1) * BN_DET_ROWS);
        float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
        for (int row = chk * BN_DET_ROWS + rl; row < end; row += rowlanes) {
            const size_t i = (size_t)row * c4 + cg;
            float4 g = dy[(size_t)row * dy_ld4 + cg], xx = x[i];
            g.x = relu_grad(fmaf(xx.x, sc.x, sh.x), g.x); g.y = relu_grad(fmaf(xx.y, sc.y, sh.y), g.y);
            g.z = relu_grad(fmaf(xx.z, sc.z, sh.z), g.z); g.w = relu_grad(fmaf(xx.w, sc.w, sh.w), g.w);
            s[0] += g.x; s[1] += g.y; s[2] += g.z; s[3] += g.w;
            q[0] = fmaf(g.x, (xx.x - m.x) * is.x, q[0]); q[1] = fmaf(g.y, (xx.y - m.y) * is.y, q[1]);
            q[2] = fmaf(g.z, (xx.z - m.z) * is.z, q[2]); q[3] = fmaf(g.w, (xx.w - m.w) * is.w, q[3]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            shf[(rl * 2 + 0) * c + cg * 4 + j] = s[j];
            shf[(rl * 2 + 1) * c + cg * 4 + j] = q[j];
        }
        __syncthreads();
        if (threadIdx.x < 2 * c) {
            const int which = threadIdx.x / c, ch = threadIdx.x % c;
            double v = 0.0;
            for (int l = 0; l < rowlanes; ++l) v += (double)shf[(l * 2 + which) * c + ch];
            part[(size_t)chk * 2 * c + which * c + ch] = v;
        }
        __syncthreads();
    }
}

// (S, Q) of every channel from the chunk partials, the same in every block: thread t adds chunks sub, sub + nsub, ... of
// column t % 2c (sub = t / 2c), the subs are then added in order.  dsh: 256 doubles of shared memory.  Returns through
// S_out / Q_out for threads < c.
__device__ __forceinline__ void bn_bwd_sum_partials(const double* __restrict__ part, int n, int c, double* dsh, double& S_out,
                                                    double& Q_out) {
    const int n_chunks = (n + BN_DET_ROWS - 1) / BN_DET_ROWS;
    const int cols = 2 * c, nsub = blockDim.x / cols;
    const int col = threadIdx.x % cols, sub = threadIdx.x / cols;
    double v = 0.0;
    if (sub < nsub)
        for (int chk = sub; chk < n_chunks; chk += nsub) v += __ldcg(part + (size_t)chk * cols + col);
    dsh[threadIdx.x] = v;
    __syncthreads();
    if (threadIdx.x < c) {
        double S = 0.0, Q = 0.0;
        for (int u = 0; u < nsub; ++u) {
            S += dsh[u * cols + threadIdx.x];
            Q += dsh[u * cols + c + threadIdx.x];
        }
        S_out = S;
        Q_out = Q;
    }
    __syncthreads();
}

// backward pass 1: sum g and sum g*xhat over rows, g = dy*!(y<=0) (relu_grad: a NaN activation passes the gradient, as
// torch's threshold_backward does); block partial -> float64 atomics on bsums [2, c]
// (the ReLU mask is recomputed from x with the forward's own scale / shift and fmaf: bit-identical to testing y,
//  so the activation itself is not read again; dy may be a column slice of a wider matrix: row pitch dy_ld4 float4)
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const float4* __restrict__ dy, int dy_ld4, const float4* __restrict__ x,
                                                            const float* __restrict__ stats, int n, const int* __restrict__ n_dev,
                                                            int c, double* __restrict__ bsums, double* __restrict__ part) {
    extern __shared__ float shf[];  // [rowlanes][2][c]
    if (n_dev != nullptr) n = min(n, __ldg(n_dev));
    if (part != nullptr) {          // deterministic: per-chunk partials, summed by the apply kernel
        bn_bwd_chunk_partials(dy, dy_ld4, x, stats, n, c, part, shf);
        return;
    }
    const int c4 = c / 4;
    const int cg = threadIdx.x % c4, rl = threadIdx.x / c4, rowlanes = blockDim.x / c4;
    const float4 sc = reinterpret_cast<const float4*>(stats)[cg];
    const float4 sh = reinterpret_cast<const float4*>(stats + c)[cg];
    const float4 m = reinterpret_cast<const float4*>(stats + 2 * c)[cg];
    const float4 is = reinterpret_cast<const float4*>(stats + 3 * c)[cg];
    float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
    for (int row = blockIdx.x * rowlanes + rl; row < n; row += gridDim.x * rowlanes) {
        size_t i = (size_t)row * c4 + cg;
        float4 g = dy[(size_t)row * dy_ld4 + cg], xx = x[i];
        g.x = relu_grad(fmaf(xx.x, sc.x, sh.x), g.x); g.y = relu_grad(fmaf(xx.y, sc.y, sh.y), g.y);
        g.z = relu_grad(fmaf(xx.z, sc.z, sh.z), g.z); g.w = relu_grad(fmaf(xx.w, sc.w, sh.w), g.w);
        s[0] += g.x; s[1] += g.y; s[2] += g.z; s[3] += g.w;
        q[0] = fmaf(g.x, (xx.x - m.x) * is.x, q[0]); q[1] = fmaf(g.y, (xx.y - m.y) * is.y, q[1]);
        q[2] = fmaf(g.z, (xx.z - m.z) * is.z, q[2]); q[3] = fmaf(g.w, (xx.w - m.w) * is.w, q[3]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        shf[(rl * 2 + 0) * c + cg * 4 + j] = s[j];
        shf[(rl * 2 + 1) * c + cg * 4 + j] = q[j];
    }
    __syncthreads();
    if (threadIdx.x < 2 * c) {
        int which = threadIdx.x / c, ch = threadIdx.x % c;
        float v = 0.f;
        for (int l = 0; l < rowlanes; ++l) v += shf[(l * 2 + which) * c + ch];
        atomicAdd(bsums + which * c + ch, (double)v);
    }
}

// backward pass 2:  train: dx = gi*(g - S/n - xhat*Q/n);  eval: dx = gi*g;   gi = gamma*invstd
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float4* __restrict__ dy, int dy_ld4, const float4* __restrict__ x,
                                                           const float* __restrict__ gamma,
                                                           const float* __restrict__ stats,
                                                           const double* __restrict__ bsums, int n_rows,
                                                           const int* __restrict__ n_dev, int c, int training,
                                                           float4* __restrict__ dx, uint2* __restrict__ dx_bf16,
                                                           float* __restrict__ dgamma, float* __restrict__ dbeta, int tail_zero,
                                                           const double* __restrict__ part, const double* __restrict__ n_glob) {
    // n_glob (SyncBatchNorm, else NULL): bsums are the all-reduced sums, *n_glob the row count over all ranks; dgamma /
    // dbeta are then NULL (the local ones were written before the exchange)
    const int cap_rows = n_rows;
    if (n_dev != nullptr) n_rows = min(n_rows, __ldg(n_dev));
    const int c4 = c / 4;
    const size_t n4 = (size_t)n_rows * c4;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const int cg = (int)(i0 % c4);
    __shared__ float a_s[128], b_s[128], d_s[128];
    __shared__ double dsh[256];
    double S = 0.0, Q = 0.0;
    if (part != nullptr) bn_bwd_sum_partials(part, n_rows, c, dsh, S, Q);
    if (threadIdx.x < c) {
        const int ch = threadIdx.x;
        if (part == nullptr) {
            S = bsums[ch];
            Q = bsums[c + ch];
        }
        const float mean = stats[2 * c + ch], invstd = stats[3 * c + ch];
        const float gi = gamma[ch] * invstd;
        if (training) {
            const double nn = n_glob != nullptr ? __ldg(n_glob) : (double)(n_rows > 0 ? n_rows : 1);
            const float k1 = (float)(Q / nn) * invstd;
            a_s[ch] = gi;
            b_s[ch] = -gi * k1;
            d_s[ch] = gi * (k1 * mean - (float)(S / nn));
        } else {
            a_s[ch] = gi;
            b_s[ch] = 0.f;
            d_s[ch] = 0.f;
        }
        if (blockIdx.x == 0 && dgamma != nullptr) {
            dbeta[ch] = (float)S;
            dgamma[ch] = (float)Q;
        }
    }
    __syncthreads();
    float a[4], b[4], d[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        a[j] = a_s[cg * 4 + j];
        b[j] = b_s[cg * 4 + j];
        d[j] = d_s[cg * 4 + j];
    }
    const float4 sc = reinterpret_cast<const float4*>(stats)[cg];
    const float4 sh = reinterpret_cast<const float4*>(stats + c)[cg];
    for (size_t i = i0; i < n4; i += stride) {
        float4 g = dy[dy_ld4 == c4 ? i : (i / c4) * dy_ld4 + cg], xx = x[i], r;
        g.x = relu_grad(fmaf(xx.x, sc.x, sh.x), g.x); g.y = relu_grad(fmaf(xx.y, sc.y, sh.y), g.y);
        g.z = relu_grad(fmaf(xx.z, sc.z, sh.z), g.z); g.w = relu_grad(fmaf(xx.w, sc.w, sh.w), g.w);
        // (eval: b = d = 0 and x does not enter dx, so a NaN x gives gi * g as torch does, not 0 * NaN; 0 is the value
        // fmaf(0, x, 0) has for every finite x)
        r.x = fmaf(a[0], g.x, training ? fmaf(b[0], xx.x, d[0]) : 0.f); r.y = fmaf(a[1], g.y, training ? fmaf(b[1], xx.y, d[1]) : 0.f);
        r.z = fmaf(a[2], g.z, training ? fmaf(b[2], xx.z, d[2]) : 0.f); r.w = fmaf(a[3], g.w, training ? fmaf(b[3], xx.w, d[3]) : 0.f);
        if (dx != nullptr) dx[i] = r;
        if (dx_bf16 != nullptr) dx_bf16[i] = pack_bf16x4(r);
    }
    if (tail_zero && cap_rows > n_rows) {
        // static mode: rows between the count and the capacity are operands of the tensor-core wgrad tiles (multiplied by
        // zero-filled gathers): they must be finite
        const size_t t4 = (size_t)cap_rows * c4;
        for (size_t i = n4 + i0; i < t4; i += stride) {
            if (dx != nullptr) dx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (dx_bf16 != nullptr) dx_bf16[i] = make_uint2(0u, 0u);
        }
    }
}

// SyncBatchNorm: a rank's local sums [2, c] into its exchange slot before the all-reduce.  Forward (dgamma == NULL):
// slot = [sum x (c), sum x^2 (c), row count] (the count from n_dev in static mode).  Backward: slot = [sum g (c),
// sum g*xhat (c)], and the local dbeta / dgamma (which stay local: DDP averages them) are written from the same sums.
__global__ void __launch_bounds__(256) bn_sync_pack_kernel(const double* __restrict__ sums, int c, int n_rows,
                                                           const int* __restrict__ n_dev, double* __restrict__ slot,
                                                           float* __restrict__ dgamma, float* __restrict__ dbeta) {
    for (int j = threadIdx.x; j < 2 * c; j += blockDim.x) {
        const double v = sums[j];
        slot[j] = v;
        if (dgamma != nullptr) (j < c ? dbeta[j] : dgamma[j - c]) = (float)v;
    }
    if (dgamma == nullptr && threadIdx.x == 0) slot[2 * c] = (double)(n_dev != nullptr ? min(n_rows, __ldg(n_dev)) : n_rows);
}

// backward, both passes in ONE cooperative launch (grid-wide barrier between the reduction and the apply): 20 launches fewer per
// step than reduce + apply, and the second read of dy / x comes out of L2.  Same arithmetic as the two kernels above.
__global__ void __launch_bounds__(256) bn_bwd_fused_kernel(const float4* __restrict__ dy, int dy_ld4, const float4* __restrict__ x,
                                                           const float* __restrict__ gamma, const float* __restrict__ stats,
                                                           double* __restrict__ bsums, int n_rows, const int* __restrict__ n_dev, int c,
                                                           int training, float4* __restrict__ dx, uint2* __restrict__ dx_bf16,
                                                           float* __restrict__ dgamma, float* __restrict__ dbeta, int tail_zero,
                                                           double* __restrict__ part) {
    extern __shared__ float shf[];  // [rowlanes][2][c]
    const int cap_rows = n_rows;
    if (n_dev != nullptr) n_rows = min(n_rows, __ldg(n_dev));
    const int c4 = c / 4;
    if (part != nullptr) {          // deterministic: per-chunk partials, summed in chunk order after the barrier
        bn_bwd_chunk_partials(dy, dy_ld4, x, stats, n_rows, c, part, shf);
    } else {
        const int cg = threadIdx.x % c4, rl = threadIdx.x / c4, rowlanes = blockDim.x / c4;
        const float4 sc = reinterpret_cast<const float4*>(stats)[cg];
        const float4 sh = reinterpret_cast<const float4*>(stats + c)[cg];
        const float4 m = reinterpret_cast<const float4*>(stats + 2 * c)[cg];
        const float4 is = reinterpret_cast<const float4*>(stats + 3 * c)[cg];
        float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
        for (int row = blockIdx.x * rowlanes + rl; row < n_rows; row += gridDim.x * rowlanes) {
            size_t i = (size_t)row * c4 + cg;
            float4 g = dy[(size_t)row * dy_ld4 + cg], xx = x[i];
            g.x = relu_grad(fmaf(xx.x, sc.x, sh.x), g.x); g.y = relu_grad(fmaf(xx.y, sc.y, sh.y), g.y);
            g.z = relu_grad(fmaf(xx.z, sc.z, sh.z), g.z); g.w = relu_grad(fmaf(xx.w, sc.w, sh.w), g.w);
            s[0] += g.x; s[1] += g.y; s[2] += g.z; s[3] += g.w;
            q[0] = fmaf(g.x, (xx.x - m.x) * is.x, q[0]); q[1] = fmaf(g.y, (xx.y - m.y) * is.y, q[1]);
            q[2] = fmaf(g.z, (xx.z - m.z) * is.z, q[2]); q[3] = fmaf(g.w, (xx.w - m.w) * is.w, q[3]);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            shf[(rl * 2 + 0) * c + cg * 4 + j] = s[j];
            shf[(rl * 2 + 1) * c + cg * 4 + j] = q[j];
        }
        __syncthreads();
        if (threadIdx.x < 2 * c) {
            int which = threadIdx.x / c, ch = threadIdx.x % c;
            float v = 0.f;
            for (int l = 0; l < rowlanes; ++l) v += shf[(l * 2 + which) * c + ch];
            atomicAdd(bsums + which * c + ch, (double)v);
        }
    }
    __threadfence();
    cooperative_groups::this_grid().sync();
    const size_t n4 = (size_t)n_rows * c4;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const int cg = (int)(i0 % c4);
    float* a_s = shf;                 // (the reduction's staging is dead: reuse it)
    float* b_s = shf + 128;
    float* d_s = shf + 256;
    __syncthreads();
    double S = 0.0, Q = 0.0;
    if (part != nullptr) bn_bwd_sum_partials(part, n_rows, c, reinterpret_cast<double*>(shf + 512), S, Q);
    if (threadIdx.x < c) {
        const int ch = threadIdx.x;
        if (part == nullptr) {
            S = __ldcg(bsums + ch);
            Q = __ldcg(bsums + c + ch);
        }
        const float mean = stats[2 * c + ch], invstd = stats[3 * c + ch];
        const float gi = gamma[ch] * invstd;
        if (training) {
            const double nn = (double)(n_rows > 0 ? n_rows : 1);
            const float k1 = (float)(Q / nn) * invstd;
            a_s[ch] = gi;
            b_s[ch] = -gi * k1;
            d_s[ch] = gi * (k1 * mean - (float)(S / nn));
        } else {
            a_s[ch] = gi;
            b_s[ch] = 0.f;
            d_s[ch] = 0.f;
        }
        if (blockIdx.x == 0) {
            dbeta[ch] = (float)S;
            dgamma[ch] = (float)Q;
        }
    }
    __syncthreads();
    float a[4], b[4], d[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        a[j] = a_s[cg * 4 + j];
        b[j] = b_s[cg * 4 + j];
        d[j] = d_s[cg * 4 + j];
    }
    const float4 sc = reinterpret_cast<const float4*>(stats)[cg];
    const float4 sh = reinterpret_cast<const float4*>(stats + c)[cg];
    for (size_t i = i0; i < n4; i += stride) {
        float4 g = dy[dy_ld4 == c4 ? i : (i / c4) * dy_ld4 + cg], xx = x[i], r;
        g.x = relu_grad(fmaf(xx.x, sc.x, sh.x), g.x); g.y = relu_grad(fmaf(xx.y, sc.y, sh.y), g.y);
        g.z = relu_grad(fmaf(xx.z, sc.z, sh.z), g.z); g.w = relu_grad(fmaf(xx.w, sc.w, sh.w), g.w);
        // (eval: b = d = 0 and x does not enter dx, so a NaN x gives gi * g as torch does, not 0 * NaN; 0 is the value
        // fmaf(0, x, 0) has for every finite x)
        r.x = fmaf(a[0], g.x, training ? fmaf(b[0], xx.x, d[0]) : 0.f); r.y = fmaf(a[1], g.y, training ? fmaf(b[1], xx.y, d[1]) : 0.f);
        r.z = fmaf(a[2], g.z, training ? fmaf(b[2], xx.z, d[2]) : 0.f); r.w = fmaf(a[3], g.w, training ? fmaf(b[3], xx.w, d[3]) : 0.f);
        if (dx != nullptr) dx[i] = r;
        if (dx_bf16 != nullptr) dx_bf16[i] = pack_bf16x4(r);
    }
    if (tail_zero && cap_rows > n_rows) {
        const size_t t4 = (size_t)cap_rows * c4;
        for (size_t i = n4 + i0; i < t4; i += stride) {
            if (dx != nullptr) dx[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (dx_bf16 != nullptr) dx_bf16[i] = make_uint2(0u, 0u);
        }
    }
}

int g_bn_fused = 1;     // 1: reduce + apply in one cooperative launch; 0: two launches (vc_set_bn_fused)

static bool c_ok(int c) { return c > 0 && c % 4 == 0 && c <= 128; }

static int ew_blocks(size_t n4) {
    size_t b = (n4 + 255) / 256;
    if (b > 132 * 16) b = 132 * 16;
    return (int)(b < 1 ? 1 : b);
}

}  // namespace vc

using namespace vc;

// internal entry points (plan executor): device row count, strided outputs / gradients, optional outputs
int vc::bn_apply_relu_dev(const float* x, const double* sums, int n_rows, const int* n_dev, int c, const float* gamma,
                          const float* beta, float* running_mean, float* running_var, long long* num_batches_tracked,
                          float momentum, float eps, int training, float* y, int y_ld, void* y_bf16, int yb_ld,
                          float* stats_out, int relu, int tail_zero, cudaStream_t stream, const double* n_glob) {
    VC_CHECK_ARG(c_ok(c) && n_rows >= 0, "bad bn args c=%d rows=%d", c, n_rows);
    VC_CHECK_ARG(gamma && beta && running_mean && running_var && stats_out, "null pointer");
    VC_CHECK_ARG(!training || sums, "training-mode BN needs the conv's channel sums");
    VC_CHECK_ARG(!training || n_rows > 0 || n_glob, "training-mode BN over zero rows");
    VC_CHECK_ARG(n_rows == 0 || (x && (y || y_bf16)), "null pointer");
    VC_CHECK_ARG(y_ld % 4 == 0 && yb_ld % 4 == 0 && y_ld >= c && yb_ld >= c, "bad output pitch");
    bn_apply_relu_kernel<<<dim3(ew_blocks((size_t)n_rows * c / 4)), dim3(256), 0, stream>>>((const float4*)x, sums, n_rows, n_dev,
        c, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, training, (float4*)y, y_ld / 4,
        (uint2*)y_bf16, yb_ld / 4, stats_out, relu, tail_zero, n_glob);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int vc::bn_relu_bwd_dev(const float* dy, int dy_ld, const float* x, const float* gamma, const float* stats, float* dx,
                        void* dx_bf16, float* dgamma, float* dbeta, int n, const int* n_dev, int c, int training,
                        double* bsums, int tail_zero, cudaStream_t stream, double* part) {
    VC_CHECK_ARG(c_ok(c) && n >= 0, "bad args n=%d c=%d", n, c);
    VC_CHECK_ARG(dgamma && dbeta && bsums && stats && gamma, "null pointer");
    VC_CHECK_ARG(dy_ld % 4 == 0 && dy_ld >= c, "bad gradient pitch");
    if (n > 0 && g_bn_fused) {
        VC_CHECK_ARG(dy && x && (dx || dx_bf16), "null pointer");
        // the grid must be co-resident for the grid-wide barrier: <= 2 blocks per SM (the row loop and the apply loop stride)
        static int max_blocks = 0;
        if (max_blocks == 0) {
            int dev = 0, sms = 132, per_sm = 0;
            cudaGetDevice(&dev);
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bn_bwd_fused_kernel, 256, 8192) != cudaSuccess || per_sm < 1) per_sm = 1;
            max_blocks = sms * (per_sm < 2 ? per_sm : 2);
        }
        const int c4 = c / 4, rowlanes = 256 / c4;
        int blocks = (n + rowlanes - 1) / rowlanes;
        if (blocks > max_blocks) blocks = max_blocks;
        // (>= 512 floats + 256 doubles: the apply phase's coefficients and, in deterministic mode, the partial sums)
        const size_t smem = (size_t)rowlanes * 2 * c * sizeof(float) < 4096 ? 4096 : (size_t)rowlanes * 2 * c * sizeof(float);
        const float4* dy4 = (const float4*)dy;
        const float4* x4 = (const float4*)x;
        int dy_ld4 = dy_ld / 4;
        float4* dx4 = (float4*)dx;
        uint2* dxb = (uint2*)dx_bf16;
        void* args[] = {&dy4, &dy_ld4, &x4, &gamma, &stats, &bsums, &n, &n_dev, &c, &training, &dx4, &dxb, &dgamma, &dbeta, &tail_zero,
                        &part};
        const cudaError_t ce = cudaLaunchCooperativeKernel((const void*)bn_bwd_fused_kernel, dim3(blocks), dim3(256), args, smem, stream);
        if (ce == cudaSuccess) {
            vc::count_launch();
            return VC_OK;
        }
        // (a device / driver configuration without cooperative launches: fall back to the two-kernel form for good)
        cudaGetLastError();
        g_bn_fused = 0;
    }
    if (n > 0) {
        VC_CHECK_ARG(dy && x && (dx || dx_bf16), "null pointer");
        int c4 = c / 4;
        int rowlanes = 256 / c4;
        int blocks = (n + rowlanes - 1) / rowlanes;
        if (blocks > 296) blocks = 296;
        size_t smem = (size_t)rowlanes * 2 * c * sizeof(float);
        bn_bwd_reduce_kernel<<<dim3(blocks), dim3(256), smem, stream>>>((const float4*)dy, dy_ld / 4, (const float4*)x, stats, n,
            n_dev, c, bsums, part);
        VC_LAUNCH_CHECK();
    }
    bn_bwd_apply_kernel<<<dim3(ew_blocks((size_t)n * c / 4)), dim3(256), 0, stream>>>((const float4*)dy, dy_ld / 4,
        (const float4*)x, gamma, stats, bsums, n, n_dev, c, training, (float4*)dx, (uint2*)dx_bf16, dgamma, dbeta, tail_zero,
        (const double*)part, nullptr);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int vc::bn_sync_pack_dev(const double* sums, int c, int n_rows, const int* n_dev, double* slot, float* dgamma, float* dbeta,
                         cudaStream_t stream) {
    VC_CHECK_ARG(c_ok(c) && n_rows >= 0 && sums && slot && (dgamma == nullptr) == (dbeta == nullptr), "bad bn exchange args");
    bn_sync_pack_kernel<<<1, 256, 0, stream>>>(sums, c, n_rows, n_dev, slot, dgamma, dbeta);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// SyncBatchNorm backward, first half: the local (sum g, sum g*xhat) into bsums [2, c] (zeroed by the caller; deterministic
// mode: chunk partials `part`, added in chunk order), then the local dbeta / dgamma and the exchange slot [2c]
int vc::bn_relu_bwd_local_dev(const float* dy, int dy_ld, const float* x, const float* stats, int n, const int* n_dev, int c,
                              double* bsums, double* part, float* dgamma, float* dbeta, double* slot, cudaStream_t stream) {
    VC_CHECK_ARG(c_ok(c) && n >= 0 && bsums && stats && dgamma && dbeta && slot, "bad args n=%d c=%d", n, c);
    VC_CHECK_ARG(dy_ld % 4 == 0 && dy_ld >= c, "bad gradient pitch");
    if (n > 0) {
        VC_CHECK_ARG(dy && x, "null pointer");
        const int c4 = c / 4, rowlanes = 256 / c4;
        int blocks = (n + rowlanes - 1) / rowlanes;
        if (blocks > 296) blocks = 296;
        bn_bwd_reduce_kernel<<<dim3(blocks), dim3(256), (size_t)rowlanes * 2 * c * sizeof(float), stream>>>(
            (const float4*)dy, dy_ld / 4, (const float4*)x, stats, n, n_dev, c, bsums, part);
        VC_LAUNCH_CHECK();
        if (part != nullptr) {
            const int rc = bn_sums_reduce_dev(part, n, n_dev, BN_DET_ROWS, c, bsums, stream);
            if (rc) return rc;
        }
    }
    return bn_sync_pack_dev(bsums, c, n, n_dev, slot, dgamma, dbeta, stream);
}

// second half, after the exchange: dx from the all-reduced sums and the global row count n_glob (device float64)
int vc::bn_relu_bwd_apply_dev(const float* dy, int dy_ld, const float* x, const float* gamma, const float* stats,
                              const double* bsums, const double* n_glob, float* dx, void* dx_bf16, int n, const int* n_dev, int c,
                              int tail_zero, cudaStream_t stream) {
    VC_CHECK_ARG(c_ok(c) && n >= 0 && bsums && n_glob && stats && gamma, "bad args n=%d c=%d", n, c);
    VC_CHECK_ARG(n == 0 || (dy && x && (dx || dx_bf16)), "null pointer");
    bn_bwd_apply_kernel<<<dim3(ew_blocks((size_t)n * c / 4)), dim3(256), 0, stream>>>((const float4*)dy, dy_ld / 4,
        (const float4*)x, gamma, stats, bsums, n, n_dev, c, 1, (float4*)dx, (uint2*)dx_bf16, nullptr, nullptr, tail_zero,
        nullptr, n_glob);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_bn_apply_relu_f32(const float* x, const double* sums, int n_rows, int c, const float* gamma,
                                    const float* beta, float* running_mean, float* running_var,
                                    long long* num_batches_tracked, float momentum, float eps, int training, float* y,
                                    void* y_bf16, float* stats_out, int relu, vc_stream_t stream_) {
    VC_CHECK_ARG(n_rows == 0 || y, "null pointer");
    return vc::bn_apply_relu_dev(x, sums, n_rows, nullptr, c, gamma, beta, running_mean, running_var, num_batches_tracked, momentum,
                                 eps, training, y, c, y_bf16, c, stats_out, relu, 0, (cudaStream_t)stream_);
}

/* (y is no longer read: the ReLU mask is recomputed from x and the saved scale / shift — kept in the signature) */
extern "C" int vc_bn_relu_bwd_f32(const float* dy, const float* x, const float* y, const float* gamma, const float* stats,
                                  float* dx, void* dx_bf16, float* dgamma, float* dbeta, int n, int c, int training,
                                  double* bsums, vc_stream_t stream_) {
    (void)y;
    VC_CHECK_ARG(n == 0 || dx, "null pointer");
    return vc::bn_relu_bwd_dev(dy, c, x, gamma, stats, dx, dx_bf16, dgamma, dbeta, n, nullptr, c, training, bsums, 0,
                               (cudaStream_t)stream_);
}

int vc::bn_sums_reduce_dev(const double* part, int cap_rows, const int* n_dev, int rows_per_part, int c, double* sums,
                           cudaStream_t stream) {
    VC_CHECK_ARG(c_ok(c) && cap_rows >= 0 && rows_per_part > 0 && part && sums, "bad bn sums args");
    bn_sums_reduce_kernel<<<dim3(2 * c), dim3(256), 0, stream>>>(part, cap_rows, n_dev, rows_per_part, c, sums);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_bn_bwd_det_ws_bytes(int n, int c) {
    return (size_t)((n + BN_DET_ROWS - 1) / BN_DET_ROWS) * 2 * (c > 0 ? c : 0) * sizeof(double);
}

extern "C" int vc_bn_relu_bwd_det_f32(const float* dy, const float* x, const float* gamma, const float* stats, float* dx,
                                      void* dx_bf16, float* dgamma, float* dbeta, int n, int c, int training, void* ws,
                                      size_t ws_bytes, vc_stream_t stream_) {
    VC_CHECK_ARG(n == 0 || dx || dx_bf16, "null pointer");
    VC_CHECK_ARG(ws && ws_bytes >= vc_bn_bwd_det_ws_bytes(n, c), "deterministic BN backward workspace too small");
    return vc::bn_relu_bwd_dev(dy, c, x, gamma, stats, dx, dx_bf16, dgamma, dbeta, n, nullptr, c, training, (double*)ws, 0,
                               (cudaStream_t)stream_, (double*)ws);
}

extern "C" int vc_set_bn_fused(int enable) {
    vc::g_bn_fused = enable ? 1 : 0;
    return VC_OK;
}
