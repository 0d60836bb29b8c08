// StVD layer discard on the device (`layer_voxel_discard`, spconv_backbone.py:134-147) — sm_90a.
//
// The reference keeps `np.random.permutation(n)[:int(n * (1 - rate))]`: a uniformly random k-subset of the rows.  Here
// the subset is drawn on the device, without a host read, so that a step can be captured into a CUDA graph:
//   * key of row i at discard site d: u_i = word 0 of Philox4x32-10 with counter (i, d, 0, 0) and key (seed low word,
//     seed high word), seed = one int64 in device memory (or caller-given uint32 keys);
//   * kept rows: the k rows with the smallest (u_i, i), listed in ascending row order (published tensors stay
//     batch-contiguous), k = int(n * (1 - rate)) in float64 as Python evaluates it.
// Selection is a radix select of the k-th smallest u (four 8-bit digit passes: per-block shared-memory histograms added
// into a global one with integer atomics, every block resolving the digits of the earlier passes itself), then an
// order-preserving compaction: per-tile counts of the rows below / equal to the threshold, one scan over the tiles, and
// ranks from warp ballots — the rows equal to the threshold are taken lowest row first, which is the (u, i) order.  The
// result is the same on every run.
#include <cuda_bf16.h>

#include "common.cuh"
#include "philox.cuh"

namespace vc {
namespace {

constexpr int TILE = 256;           // rows per block of the count / emit passes; threads of every selection kernel
constexpr int SCAN_THREADS = 1024;
constexpr int PASSES = 4;           // 8-bit digits of a 32-bit key

__device__ __forceinline__ int live_rows(const int* n_dev, int cap) {
    if (!n_dev) return cap;
    const int n = *n_dev;
    return n < 0 ? 0 : (n > cap ? cap : n);
}

__device__ __forceinline__ int keep_count(int n, double rate) {   // int(n * (1 - rate)), Python's float64 arithmetic
    const int k = (int)((double)n * (1.0 - rate));
    return k < 0 ? 0 : (k > n ? n : k);
}

// Digits of the k-th smallest key fixed by the histograms of passes [0, passes): -> (prefix, rank still to take among the
// rows whose top 8*passes bits equal prefix).  Every thread of the (TILE-thread) block takes part.
__device__ void resolve(const unsigned* hist, int passes, int k, uint32_t& prefix, int& rem) {
    __shared__ unsigned s_scan[256];
    __shared__ uint32_t s_prefix, s_next_prefix;
    __shared__ int s_rem, s_next_rem;
    const int t = threadIdx.x;
    if (t == 0) {
        s_prefix = 0;
        s_rem = k;
    }
    for (int p = 0; p < passes; ++p) {
        s_scan[t] = hist[p * 256 + t];
        __syncthreads();
        for (int off = 1; off < 256; off <<= 1) {
            const unsigned v = t >= off ? s_scan[t - off] : 0u;
            __syncthreads();
            s_scan[t] += v;
            __syncthreads();
        }
        const unsigned r = (unsigned)s_rem, incl = s_scan[t], excl = t ? s_scan[t - 1] : 0u;
        if (excl < r && r <= incl) {          // exactly one digit holds the r-th smallest
            s_next_prefix = (s_prefix << 8) | (uint32_t)t;
            s_next_rem = (int)(r - excl);
        }
        __syncthreads();
        if (t == 0) {
            s_prefix = s_next_prefix;
            s_rem = s_next_rem;
        }
        __syncthreads();
    }
    __syncthreads();
    prefix = s_prefix;
    rem = s_rem;
}

// exclusive rank of `f` among the TILE threads of the block, and the block's total
__device__ __forceinline__ int block_rank(bool f, int& total) {
    __shared__ int s_w[TILE / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    __syncthreads();
    if (lane == 0) s_w[w] = __popc(m);
    __syncthreads();
    int off = 0, tot = 0;
#pragma unroll
    for (int j = 0; j < TILE / 32; ++j) {
        off += j < w ? s_w[j] : 0;
        tot += s_w[j];
    }
    total = tot;
    return off + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(TILE) stvd_hist_kernel(const uint32_t* __restrict__ keys, const int64_t* __restrict__ seed,
                                                         uint32_t site, int cap, const int* __restrict__ n_dev, double rate,
                                                         uint32_t* __restrict__ u, unsigned* __restrict__ hist, int pass) {
    const int n = live_rows(n_dev, cap), k = keep_count(n, rate);
    if (k == 0) return;
    uint32_t prefix;
    int rem;
    resolve(hist, pass, k, prefix, rem);
    __shared__ unsigned h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int shift = 24 - 8 * pass;
    uint32_t k0 = 0, k1 = 0;
    if (pass == 0 && !keys) {
        const uint64_t s = (uint64_t)*seed;
        k0 = (uint32_t)s;
        k1 = (uint32_t)(s >> 32);
    }
    for (int i = blockIdx.x * TILE + threadIdx.x; i < n; i += gridDim.x * TILE) {
        uint32_t v;
        if (pass == 0) {
            v = keys ? keys[i] : philox_word0((uint32_t)i, site, 0u, 0u, k0, k1);
            u[i] = v;
        } else {
            v = u[i];
        }
        if (pass == 0 || (v >> (shift + 8)) == prefix) atomicAdd(&h[(v >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (h[threadIdx.x]) atomicAdd(&hist[pass * 256 + threadIdx.x], h[threadIdx.x]);
}

// per tile: rows below / equal to the threshold key; block 0 records (k, threshold, rank among the equal rows)
__global__ void __launch_bounds__(TILE) stvd_count_kernel(const uint32_t* __restrict__ u, int cap, const int* __restrict__ n_dev,
                                                          double rate, const unsigned* __restrict__ hist, int* __restrict__ blk_lt,
                                                          int* __restrict__ blk_eq, int* __restrict__ sel, int32_t* __restrict__ kept_dev) {
    const int n = live_rows(n_dev, cap), k = keep_count(n, rate);
    uint32_t thr = 0;
    int rem = 0;
    if (k > 0) resolve(hist, PASSES, k, thr, rem);
    const int i = blockIdx.x * TILE + threadIdx.x;
    const uint32_t v = (k > 0 && i < n) ? u[i] : 0u;
    const int c_lt = __syncthreads_count(k > 0 && i < n && v < thr);
    const int c_eq = __syncthreads_count(k > 0 && i < n && v == thr);
    if (threadIdx.x == 0) {
        blk_lt[blockIdx.x] = c_lt;
        blk_eq[blockIdx.x] = c_eq;
        if (blockIdx.x == 0) {
            sel[0] = k;
            sel[1] = (int)thr;
            sel[2] = rem;
            *kept_dev = k;
        }
    }
}

// one block: eq_base[b] = equal rows in tiles before b; keep_base[b] = kept rows in tiles before b (in place)
__global__ void __launch_bounds__(SCAN_THREADS) stvd_scan_kernel(int nb, const int* __restrict__ sel, int* __restrict__ blk_lt,
                                                                 int* __restrict__ blk_eq) {
    __shared__ int s_w[SCAN_THREADS / 32];
    __shared__ int s_carry[2];
    const int rem = sel[2], lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_carry[0] = s_carry[1] = 0;
    __syncthreads();
    for (int base = 0; base < nb; base += SCAN_THREADS) {
        const int b = base + threadIdx.x;
        int vals[2] = {b < nb ? blk_eq[b] : 0, 0};
        int excl[2];
        for (int pass = 0; pass < 2; ++pass) {
            int x = vals[pass];
            for (int off = 1; off < 32; off <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, off);
                if (lane >= off) x += y;
            }
            if (lane == 31) s_w[w] = x;
            __syncthreads();
            int woff = 0, tot = 0;
            for (int j = 0; j < SCAN_THREADS / 32; ++j) {
                woff += j < w ? s_w[j] : 0;
                tot += s_w[j];
            }
            excl[pass] = s_carry[pass] + woff + x - vals[pass];
            __syncthreads();
            if (threadIdx.x == 0) s_carry[pass] += tot;
            if (pass == 0) {   // kept rows of tile b: all below the threshold plus its share of the equal ones
                int take = rem - excl[0];
                take = take < 0 ? 0 : (take > vals[0] ? vals[0] : take);
                vals[1] = (b < nb ? blk_lt[b] : 0) + take;
            }
            __syncthreads();
        }
        if (b < nb) {
            blk_eq[b] = excl[0];
            blk_lt[b] = excl[1];
        }
    }
}

__global__ void __launch_bounds__(TILE) stvd_emit_kernel(const uint32_t* __restrict__ u, int cap, const int* __restrict__ n_dev,
                                                         const int* __restrict__ sel, const int* __restrict__ keep_base,
                                                         const int* __restrict__ eq_base, int32_t* __restrict__ keep,
                                                         int32_t* __restrict__ pos) {
    const int n = live_rows(n_dev, cap), k = sel[0], rem = sel[2];
    const uint32_t thr = (uint32_t)sel[1];
    const int i = blockIdx.x * TILE + threadIdx.x;
    const bool live = k > 0 && i < n;
    const uint32_t v = live ? u[i] : 0u;
    const bool lt = live && v < thr, eq = live && v == thr;
    int tot;
    const int eq_rank = eq_base[blockIdx.x] + block_rank(eq, tot);
    const bool kp = lt || (eq && eq_rank < rem);
    const int r = keep_base[blockIdx.x] + block_rank(kp, tot);
    if (i < cap) {
        if (kp) keep[r] = i;
        if (i >= k) keep[i] = -1;
        if (pos) pos[i] = kp ? r : -1;
    }
}

// out rows r < rows: keep[r] >= 0 ? in[keep[r]] : 0 (fp32 and / or its bf16 rounding), c % 4 == 0
__global__ void __launch_bounds__(256) stvd_gather_feats_kernel(const float4* __restrict__ in, int c4, const int32_t* __restrict__ keep,
                                                                int rows, float4* __restrict__ out, __nv_bfloat162* __restrict__ outb) {
    const size_t total = (size_t)rows * c4, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const size_t r = e / c4;
        const int c = (int)(e % c4);
        const int src = keep[r];
        const float4 v = src >= 0 ? in[(size_t)src * c4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
        if (out) out[e] = v;
        if (outb) {
            outb[2 * e] = __floats2bfloat162_rn(v.x, v.y);
            outb[2 * e + 1] = __floats2bfloat162_rn(v.z, v.w);
        }
    }
}

__global__ void __launch_bounds__(256) stvd_gather_idx_kernel(const int32_t* __restrict__ in, int cols, const int32_t* __restrict__ keep,
                                                              int rows, int32_t* __restrict__ out) {
    const size_t total = (size_t)rows * cols, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const size_t r = e / cols;
        const int src = keep[r];
        out[e] = src >= 0 ? in[(size_t)src * cols + (e % cols)] : -1;
    }
}

// dx[i] = pos[i] >= 0 ? dy[pos[i]] : 0 — every input row written once, no atomics
__global__ void __launch_bounds__(256) stvd_grad_kernel(const float4* __restrict__ dy, int dy_ld4, int c4, const int32_t* __restrict__ pos,
                                                        int n_in, float4* __restrict__ dx, int dx_ld4) {
    const size_t total = (size_t)n_in * c4, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const size_t i = e / c4;
        const int c = (int)(e % c4);
        const int p = pos[i];
        dx[i * dx_ld4 + c] = p >= 0 ? dy[(size_t)p * dy_ld4 + c] : make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

int ew_blocks(size_t n) {
    size_t b = (n + 255) / 256;
    if (b > 132 * 8) b = 132 * 8;
    return (int)(b < 1 ? 1 : b);
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

int stvd_gather_feats_dev(const float* in, int c, const int32_t* keep, int rows, float* out, void* out_bf16, cudaStream_t st) {
    VC_CHECK_ARG(c % 4 == 0, "StVD layer discard: %d channels (multiple of 4 expected)", c);
    if (rows <= 0 || (!out && !out_bf16)) return VC_OK;
    stvd_gather_feats_kernel<<<ew_blocks((size_t)rows * (c / 4)), 256, 0, st>>>((const float4*)in, c / 4, keep, rows, (float4*)out,
                                                                               (__nv_bfloat162*)out_bf16);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int stvd_gather_idx_dev(const int32_t* in, int cols, const int32_t* keep, int rows, int32_t* out, cudaStream_t st) {
    if (rows <= 0) return VC_OK;
    stvd_gather_idx_kernel<<<ew_blocks((size_t)rows * cols), 256, 0, st>>>(in, cols, keep, rows, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int stvd_grad_dev(const float* dy, int dy_ld, int c, const int32_t* pos, int n_in, float* dx, int dx_ld, cudaStream_t st) {
    VC_CHECK_ARG(c % 4 == 0 && dy_ld % 4 == 0 && dx_ld % 4 == 0, "StVD layer discard backward: pitches must be multiples of 4");
    if (n_in <= 0) return VC_OK;
    stvd_grad_kernel<<<ew_blocks((size_t)n_in * (c / 4)), 256, 0, st>>>((const float4*)dy, dy_ld / 4, c / 4, pos, n_in, (float4*)dx,
                                                                       dx_ld / 4);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_stvd_layer_keep_ws_bytes(int cap) {
    const size_t n = cap > 0 ? (size_t)cap : 0, nb = (n + TILE - 1) / TILE;
    return align256(PASSES * 256 * 4) + align256(4 * 4) + 2 * align256(nb * 4) + align256(n * 4);
}

extern "C" int vc_stvd_layer_keep(const uint32_t* keys, const int64_t* seed_dev, int site, int n, const int32_t* n_dev, double rate,
                                  int32_t* keep, int32_t* kept_dev, int32_t* pos, void* ws, size_t ws_bytes, vc_stream_t stream) {
    VC_CHECK_ARG(n >= 0 && site >= 0 && kept_dev, "vc_stvd_layer_keep: n %d, site %d, kept_dev %p", n, site, (void*)kept_dev);
    VC_CHECK_ARG(rate >= 0.0 && rate <= 1.0, "vc_stvd_layer_keep: rate %g outside [0, 1]", rate);
    VC_CHECK_ARG(keys || seed_dev, "vc_stvd_layer_keep: neither keys nor a seed");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) {
        VC_CUDA(cudaMemsetAsync(kept_dev, 0, 4, st));
        return VC_OK;
    }
    VC_CHECK_ARG(keep && ws && ws_bytes >= vc_stvd_layer_keep_ws_bytes(n), "vc_stvd_layer_keep: keep / workspace (%zu < %zu bytes)",
                 ws_bytes, vc_stvd_layer_keep_ws_bytes(n));
    const int nb = (n + TILE - 1) / TILE;
    char* p = (char*)ws;
    unsigned* hist = (unsigned*)p;
    p += align256(PASSES * 256 * 4);
    int* sel = (int*)p;
    p += align256(4 * 4);
    int* blk_lt = (int*)p;
    p += align256((size_t)nb * 4);
    int* blk_eq = (int*)p;
    p += align256((size_t)nb * 4);
    uint32_t* u = (uint32_t*)p;
    VC_CUDA(cudaMemsetAsync(hist, 0, PASSES * 256 * 4, st));
    const int hist_grid = nb < num_sms() * 4 ? nb : num_sms() * 4;
    for (int pass = 0; pass < PASSES; ++pass) {
        stvd_hist_kernel<<<hist_grid, TILE, 0, st>>>(keys, seed_dev, (uint32_t)site, n, n_dev, rate, u, hist, pass);
        VC_LAUNCH_CHECK();
    }
    stvd_count_kernel<<<nb, TILE, 0, st>>>(u, n, n_dev, rate, hist, blk_lt, blk_eq, sel, kept_dev);
    VC_LAUNCH_CHECK();
    stvd_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(nb, sel, blk_lt, blk_eq);
    VC_LAUNCH_CHECK();
    stvd_emit_kernel<<<nb, TILE, 0, st>>>(u, n, n_dev, sel, blk_lt, blk_eq, keep, pos);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
