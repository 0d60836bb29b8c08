// fp32 sparse convolution kernels (forward, dgrad, wgrad) — output-stationary implicit gather-GEMM, sm_90a.
//
// Replaces spconv `ops.indice_conv` (+ backward) behind spconv_backbone.py:89,92-93,113,563-564.
// This is the 1e-4-parity path: fp32 operands, fp32 FMA accumulation on the CUDA cores.
//
// Tiling (gather_gemm): one CTA = 128 output rows x all C_out, 256 threads; per kernel offset k the CTA
// gathers the 128 neighbour rows in[nbr[k,o], :] (16-byte cp.async chunks, zero-fill for missing
// neighbours) and the [C_in, C_out] slice of the pre-transposed weights into shared memory, double
// buffered, and accumulates an (RT x 4) register micro-tile per thread.  Offsets with no neighbour in the
// tile are skipped entirely; a warp whose 16 rows have no neighbour at k skips the math.
// Each output row is written exactly once -> algorithmic bytes = N_in*C_in*4 + N_out*C_out*4 + K*N_out*4
// (neighbour table) + K*C_in*C_out*4 (SURVEY §8d), FLOPs = 2*P*C_in*C_out.
#include <type_traits>

#include "common.cuh"

namespace vc {

static constexpr int TM = VC_TILE_ROWS;
static constexpr int TCM_ROWS = 128;
static constexpr int NTHREADS = 256;
static constexpr int MAXK = 32;

template <int CI, int CO>
struct Cfg {
    static constexpr int NCG = CO / 4;                 // column groups (float4 of outputs)
    static constexpr int NRG = NTHREADS / NCG;         // row groups
    static constexpr int RT = TM / NRG;                // rows per thread
    static constexpr int PAD = (NCG >= 8) ? 0 : 4;     // breaks LDS.128 bank conflicts when few column groups
    static constexpr int AS = CI + PAD;                // A row stride in floats
    static constexpr int CPR = CI / 4;                 // 16-byte chunks per gathered row
    static constexpr int A_FLOATS = TM * AS;
    static constexpr int W_FLOATS = CI * CO;
    static constexpr size_t smem_gather(int K) { return (size_t)(2 * A_FLOATS + 2 * W_FLOATS) * 4 + (size_t)K * TM * 4; }
    static constexpr size_t smem_scatter(int K) { return (size_t)(A_FLOATS + 2 * W_FLOATS) * 4 + (size_t)K * TM * 4; }
};

// wt layouts: mode 0 (forward)  wt[k][ci][co] = w[co][k][ci]
//             mode 1 (dgrad)    wt[k][co][ci] = w[co][kk][ci], kk = mirror ? K-1-k : k
__global__ void prep_weights_kernel(const float* __restrict__ w, float* __restrict__ wt, int cin, int cout, int K,
                                    int mode, int mirror) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int total = K * cin * cout;
    if (i >= total) return;
    if (mode == 0) {
        int co = i % cout, ci = (i / cout) % cin, k = i / (cout * cin);
        wt[i] = w[((size_t)co * K + k) * cin + ci];
    } else {
        int ci = i % cin, co = (i / cin) % cout, k = i / (cin * cout);
        int kk = mirror ? (K - 1 - k) : k;
        wt[i] = w[((size_t)co * K + kk) * cin + ci];
    }
}

// shared prologue: stage nbr[:, tile] and build the list of offsets that touch this tile
__device__ __forceinline__ int stage_nbr(const int32_t* __restrict__ nbr, int n_rows, int K, int base, int* nbr_s,
                                         int* klist, unsigned* kmask) {
    if (threadIdx.x == 0) *kmask = 0u;
    static_assert(TM == 128, "stage_nbr_tile assumes 128-row tiles");
    stage_nbr_tile<NTHREADS>(nbr, n_rows, 0, K, base, nbr_s);
    __syncthreads();
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = warp; k < K; k += NTHREADS / 32) {
        bool any = false;
#pragma unroll
        for (int j = 0; j < TM / 32; ++j) any |= nbr_s[k * TM + j * 32 + lane] >= 0;
        if (__any_sync(0xffffffffu, any) && lane == 0) atomicOr(kmask, 1u << k);
    }
    __syncthreads();
    unsigned m = *kmask;
    if (threadIdx.x == 0) {
        int c = 0;
        for (int k = 0; k < K; ++k)
            if (m >> k & 1u) klist[c++] = k;
    }
    __syncthreads();
    return __popc(m);
}

template <int CI, int CO>
__device__ __forceinline__ void issue_w(const float* __restrict__ wt, int k, float* Ws) {
    constexpr int NCH = CI * CO / 4;
    const float* src = wt + (size_t)k * CI * CO;
    for (int q = threadIdx.x; q < NCH; q += NTHREADS) cp_async16(Ws + q * 4, src + q * 4, true);
}

template <int CI, int CO>
__device__ __forceinline__ void issue_gather(const float* __restrict__ in, const int* nbr_k, float* As) {
    using C = Cfg<CI, CO>;
#pragma unroll
    for (int j = 0; j < TM * C::CPR / NTHREADS; ++j) {
        int q = threadIdx.x + j * NTHREADS;
        int r = q / C::CPR, c = q % C::CPR;
        int src_row = nbr_k[r];
        const float* src = in + (size_t)(src_row < 0 ? 0 : src_row) * CI + c * 4;
        cp_async16(As + r * C::AS + c * 4, src, src_row >= 0);
    }
}

template <int CI, int CO>
__device__ __forceinline__ void tile_mac(const float* As, const float* Ws, int row0, int tx, float (&acc)[Cfg<CI, CO>::RT][4]) {
    using C = Cfg<CI, CO>;
#pragma unroll 2
    for (int c4 = 0; c4 < CI / 4; ++c4) {
        float4 a[C::RT];
#pragma unroll
        for (int r = 0; r < C::RT; ++r) a[r] = *reinterpret_cast<const float4*>(As + (row0 + r) * C::AS + c4 * 4);
        float4 w0 = *reinterpret_cast<const float4*>(Ws + (c4 * 4 + 0) * CO + tx * 4);
        float4 w1 = *reinterpret_cast<const float4*>(Ws + (c4 * 4 + 1) * CO + tx * 4);
        float4 w2 = *reinterpret_cast<const float4*>(Ws + (c4 * 4 + 2) * CO + tx * 4);
        float4 w3 = *reinterpret_cast<const float4*>(Ws + (c4 * 4 + 3) * CO + tx * 4);
#pragma unroll
        for (int r = 0; r < C::RT; ++r) {
            acc[r][0] = fmaf(a[r].x, w0.x, acc[r][0]); acc[r][1] = fmaf(a[r].x, w0.y, acc[r][1]);
            acc[r][2] = fmaf(a[r].x, w0.z, acc[r][2]); acc[r][3] = fmaf(a[r].x, w0.w, acc[r][3]);
            acc[r][0] = fmaf(a[r].y, w1.x, acc[r][0]); acc[r][1] = fmaf(a[r].y, w1.y, acc[r][1]);
            acc[r][2] = fmaf(a[r].y, w1.z, acc[r][2]); acc[r][3] = fmaf(a[r].y, w1.w, acc[r][3]);
            acc[r][0] = fmaf(a[r].z, w2.x, acc[r][0]); acc[r][1] = fmaf(a[r].z, w2.y, acc[r][1]);
            acc[r][2] = fmaf(a[r].z, w2.z, acc[r][2]); acc[r][3] = fmaf(a[r].z, w2.w, acc[r][3]);
            acc[r][0] = fmaf(a[r].w, w3.x, acc[r][0]); acc[r][1] = fmaf(a[r].w, w3.y, acc[r][1]);
            acc[r][2] = fmaf(a[r].w, w3.z, acc[r][2]); acc[r][3] = fmaf(a[r].w, w3.w, acc[r][3]);
        }
    }
}

// out[o, :] = sum_k in[nbr[k,o], :] @ wt[k]          (forward, and dgrad through the transposed table)
template <int CI, int CO>
__global__ void __launch_bounds__(NTHREADS, (Cfg<CI, CO>::RT >= 8) ? 2 : 3)
gather_gemm_kernel(const float* __restrict__ in, const float* __restrict__ wt, const int32_t* __restrict__ nbr,
                   float* __restrict__ out, int n_out, int K, double* __restrict__ bn_sums, double* __restrict__ bn_part) {
    using C = Cfg<CI, CO>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* As = reinterpret_cast<float*>(smem_raw);         // [2][TM][AS]
    float* Ws = As + 2 * C::A_FLOATS;                       // [2][CI][CO]
    int* nbr_s = reinterpret_cast<int*>(Ws + 2 * C::W_FLOATS);  // [K][TM]
    __shared__ int klist[MAXK];
    __shared__ unsigned kmask;
    __shared__ float red[NTHREADS / 32][2][CO];

    const int base = blockIdx.x * TM;
    const int nk = stage_nbr(nbr, n_out, K, base, nbr_s, klist, &kmask);

    const int tx = threadIdx.x % C::NCG, ty = threadIdx.x / C::NCG;
    const int row0 = ty * C::RT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc[C::RT][4];
#pragma unroll
    for (int r = 0; r < C::RT; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;

    if (nk > 0) {
        int k0 = klist[0];
        issue_gather<CI, CO>(in, nbr_s + k0 * TM, As);
        issue_w<CI, CO>(wt, k0, Ws);
        cp_async_commit();
    }
    for (int t = 0; t < nk; ++t) {
        cp_async_wait<0>();
        __syncthreads();
        const int k = klist[t];
        if (t + 1 < nk) {
            int kn = klist[t + 1];
            issue_gather<CI, CO>(in, nbr_s + kn * TM, As + ((t + 1) & 1) * C::A_FLOATS);
            issue_w<CI, CO>(wt, kn, Ws + ((t + 1) & 1) * C::W_FLOATS);
            cp_async_commit();
        }
        // the 16 rows this warp owns: skip the math if none has a neighbour at k
        bool mine = nbr_s[k * TM + warp * 16 + (lane & 15)] >= 0;
        if (__any_sync(0xffffffffu, mine))
            tile_mac<CI, CO>(As + (t & 1) * C::A_FLOATS, Ws + (t & 1) * C::W_FLOATS, row0, tx, acc);
    }

    float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int r = 0; r < C::RT; ++r) {
        int row = base + row0 + r;
        if (row < n_out) {
            *reinterpret_cast<float4*>(out + (size_t)row * CO + tx * 4) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s[j] += acc[r][j];
                q[j] = fmaf(acc[r][j], acc[r][j], q[j]);
            }
        }
    }
    if (bn_sums != nullptr || bn_part != nullptr) {  // tile's channel sums for the BatchNorm that follows -> float64 [2, CO]
#pragma unroll
        for (int off = C::NCG; off < 32; off <<= 1) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s[j] += __shfl_xor_sync(0xffffffffu, s[j], off);
                q[j] += __shfl_xor_sync(0xffffffffu, q[j], off);
            }
        }
        if (lane < C::NCG) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                red[warp][0][tx * 4 + j] = s[j];
                red[warp][1][tx * 4 + j] = q[j];
            }
        }
        __syncthreads();
        if (threadIdx.x < 2 * CO) {
            int which = threadIdx.x / CO, ch = threadIdx.x % CO;
            float v = 0.f;
#pragma unroll
            for (int w = 0; w < NTHREADS / 32; ++w) v += red[w][which][ch];
            if (bn_part != nullptr)   // deterministic mode: one partial per tile, added in tile order by bn_sums_reduce_dev
                bn_part[((size_t)blockIdx.x * 2 + which) * CO + ch] = (double)v;
            else
                atomicAdd(bn_sums + which * CO + ch, (double)v);
        }
    }
}

// din[nbr[k,o], :] += dout[o, :] @ wt[k]     (many-to-one tables: float atomics; din row pitch out_ld)
template <int CI, int CO>
__global__ void __launch_bounds__(NTHREADS, 2)
scatter_gemm_kernel(const float* __restrict__ in, const float* __restrict__ wt, const int32_t* __restrict__ nbr,
                    float* __restrict__ out, int out_ld, int n_rows, int K) {
    using C = Cfg<CI, CO>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* As = reinterpret_cast<float*>(smem_raw);         // [TM][AS]  rows of `in` (contiguous tile)
    float* Ws = As + C::A_FLOATS;                           // [2][CI][CO]
    int* nbr_s = reinterpret_cast<int*>(Ws + 2 * C::W_FLOATS);
    __shared__ int klist[MAXK];
    __shared__ unsigned kmask;

    const int base = blockIdx.x * TM;
    const int nk = stage_nbr(nbr, n_rows, K, base, nbr_s, klist, &kmask);
    if (nk == 0) return;
    const int tx = threadIdx.x % C::NCG, ty = threadIdx.x / C::NCG;
    const int row0 = ty * C::RT;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

#pragma unroll
    for (int j = 0; j < TM * C::CPR / NTHREADS; ++j) {
        int qd = threadIdx.x + j * NTHREADS;
        int r = qd / C::CPR, c = qd % C::CPR;
        bool ok = base + r < n_rows;
        cp_async16(As + r * C::AS + c * 4, in + (size_t)(ok ? base + r : 0) * CI + c * 4, ok);
    }
    issue_w<CI, CO>(wt, klist[0], Ws);
    cp_async_commit();
    for (int t = 0; t < nk; ++t) {
        cp_async_wait<0>();
        __syncthreads();
        const int k = klist[t];
        if (t + 1 < nk) {
            issue_w<CI, CO>(wt, klist[t + 1], Ws + ((t + 1) & 1) * C::W_FLOATS);
            cp_async_commit();
        }
        bool mine = nbr_s[k * TM + warp * 16 + (lane & 15)] >= 0;
        if (!__any_sync(0xffffffffu, mine)) continue;
        float acc[C::RT][4];
#pragma unroll
        for (int r = 0; r < C::RT; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;
        tile_mac<CI, CO>(As, Ws + (t & 1) * C::W_FLOATS, row0, tx, acc);
#pragma unroll
        for (int r = 0; r < C::RT; ++r) {
            int dst = nbr_s[k * TM + row0 + r];
            if (dst >= 0) {
                float* p = out + (size_t)dst * out_ld + tx * 4;
                // one 16-byte vector reduction (sm_90+) instead of four scalar atomics: a quarter of the L2 atomic operations
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(acc[r][0]), "f"(acc[r][1]),
                             "f"(acc[r][2]), "f"(acc[r][3])
                             : "memory");
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// wgrad: grid (K, R).  CTA (k, r) reduces  in[nbr[k,o], :]^T @ dout[o, :]  over its chunk of output rows
// into a [CI, CO] register tile; partials [R, K, CI, CO] are then summed in a fixed order (deterministic)
// and written in the parameter's own layout [CO, K, CI].
// ------------------------------------------------------------------------------------------------
static constexpr int WG_WIN = 256;  // candidate rows per window (one per thread)

template <int CI, int CO>
struct WCfg {
    static constexpr int NCG = CO / 4;
    static constexpr int ACTIVE = (CI * NCG < NTHREADS) ? CI * NCG : NTHREADS;  // threads covering one [CI, CO] tile
    static constexpr int REP = NTHREADS / ACTIVE;  // replicas: each takes every REP-th pair (small channel counts)
    static constexpr int NIG = ACTIVE / NCG;       // ci groups
    static constexpr int RI = CI / NIG;            // ci rows per thread (1,2,4)
    static constexpr size_t smem = (size_t)WG_WIN * (CI + CO) * 4 + 2 * WG_WIN * 4;
};

template <int CI, int CO>
__global__ void __launch_bounds__(NTHREADS, 2)
wgrad_kernel(const float* __restrict__ in, const float* __restrict__ dout, const int32_t* __restrict__ nbr,
             float* __restrict__ partial, int n_out, int K, int rows_per_chunk) {
    using W = WCfg<CI, CO>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* As = reinterpret_cast<float*>(smem_raw);  // [WG_WIN][CI]
    float* Bs = As + WG_WIN * CI;                    // [WG_WIN][CO]
    int* in_rows = reinterpret_cast<int*>(Bs + WG_WIN * CO);
    int* out_rows = in_rows + WG_WIN;
    __shared__ int warp_cnt[NTHREADS / 32];

    const int k = blockIdx.x, chunk = blockIdx.y;
    const int begin = chunk * rows_per_chunk;
    const int end = min(n_out, begin + rows_per_chunk);
    const int rep = threadIdx.x / W::ACTIVE, tl = threadIdx.x % W::ACTIVE;
    const int tx = tl % W::NCG, ti = tl / W::NCG;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float acc[W::RI][4];
#pragma unroll
    for (int r = 0; r < W::RI; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;

    for (int win = begin; win < end; win += WG_WIN) {
        int o = win + threadIdx.x;
        int i = (o < end) ? __ldg(nbr + (size_t)k * n_out + o) : -1;
        unsigned m = __ballot_sync(0xffffffffu, i >= 0);
        if (lane == 0) warp_cnt[warp] = __popc(m);
        __syncthreads();   // also: previous window's compute is finished
        int off = 0, total = 0;
#pragma unroll
        for (int w = 0; w < NTHREADS / 32; ++w) {
            if (w < warp) off += warp_cnt[w];
            total += warp_cnt[w];
        }
        if (i >= 0) {
            int p = off + __popc(m & ((1u << lane) - 1u));
            in_rows[p] = i;
            out_rows[p] = o;
        }
        __syncthreads();
        if (total == 0) continue;
        for (int q = threadIdx.x; q < total * (CI / 4); q += NTHREADS) {
            int p = q / (CI / 4), c = q % (CI / 4);
            cp_async16(As + p * CI + c * 4, in + (size_t)in_rows[p] * CI + c * 4, true);
        }
        for (int q = threadIdx.x; q < total * (CO / 4); q += NTHREADS) {
            int p = q / (CO / 4), c = q % (CO / 4);
            cp_async16(Bs + p * CO + c * 4, dout + (size_t)out_rows[p] * CO + c * 4, true);
        }
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
#pragma unroll 4
        for (int p = rep; p < total; p += W::REP) {
            float4 b = *reinterpret_cast<const float4*>(Bs + p * CO + tx * 4);
#pragma unroll
            for (int r = 0; r < W::RI; ++r) {
                float a = As[p * CI + ti * W::RI + r];
                acc[r][0] = fmaf(a, b.x, acc[r][0]);
                acc[r][1] = fmaf(a, b.y, acc[r][1]);
                acc[r][2] = fmaf(a, b.z, acc[r][2]);
                acc[r][3] = fmaf(a, b.w, acc[r][3]);
            }
        }
    }
    float* dst = partial + ((size_t)chunk * K + k) * CI * CO;
    if constexpr (W::REP == 1) {
#pragma unroll
        for (int r = 0; r < W::RI; ++r)
            *reinterpret_cast<float4*>(dst + (ti * W::RI + r) * CO + tx * 4) = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
    } else {
        // fold the replicas through shared memory in replica order (deterministic)
        __syncthreads();
        float* red = As;   // REP * CI * CO floats <= WG_WIN * CI
#pragma unroll
        for (int r = 0; r < W::RI; ++r)
            *reinterpret_cast<float4*>(red + ((size_t)rep * CI + ti * W::RI + r) * CO + tx * 4) =
                make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
        __syncthreads();
        for (int e = threadIdx.x; e < CI * CO; e += NTHREADS) {
            float v = 0.f;
            for (int q = 0; q < W::REP; ++q) v += red[(size_t)q * CI * CO + e];
            dst[e] = v;
        }
    }
}

__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw, int R, int K, int cin,
                                    int cout) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;  // index into dw [co][k][ci]
    int total = K * cin * cout;
    if (i >= total) return;
    int ci = i % cin, k = (i / cin) % K, co = i / (cin * K);
    float v = 0.f;
    for (int r = 0; r < R; ++r) v += partial[(((size_t)r * K + k) * cin + ci) * cout + co];
    dw[i] = v;
}

// ------------------------------------------------------------------------------------------------
// host dispatch
// ------------------------------------------------------------------------------------------------
#define VC_FOR_CH(X) X(8) X(16) X(32) X(64)

template <int CI, int CO>
static int launch_gather(const float* in, const float* wt, const int32_t* nbr, float* out, int n_out, int K,
                         double* bn_sums, cudaStream_t stream, double* bn_part = nullptr) {
    size_t smem = Cfg<CI, CO>::smem_gather(K);
    auto kern = gather_gemm_kernel<CI, CO>;
    VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(cdiv(n_out, TM)), dim3(NTHREADS), smem, stream>>>(in, wt, nbr, out, n_out, K, bn_sums, bn_part);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
template <int CI, int CO>
static int launch_scatter(const float* in, const float* wt, const int32_t* nbr, float* out, int out_ld, int n_rows, int K,
                          cudaStream_t stream) {
    size_t smem = Cfg<CI, CO>::smem_scatter(K);
    auto kern = scatter_gemm_kernel<CI, CO>;
    VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(cdiv(n_rows, TM)), dim3(NTHREADS), smem, stream>>>(in, wt, nbr, out, out_ld, n_rows, K);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
template <int CI, int CO>
static int launch_wgrad(const float* in, const float* dout, const int32_t* nbr, float* partial, int n_out, int K,
                        int R, int rows_per_chunk, cudaStream_t stream) {
    size_t smem = WCfg<CI, CO>::smem;
    auto kern = wgrad_kernel<CI, CO>;
    VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(K, R), NTHREADS, smem, stream>>>(in, dout, nbr, partial, n_out, K, rows_per_chunk);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

static bool ch_ok(int c) { return c == 8 || c == 16 || c == 32 || c == 64; }

// dispatch on (ci, co): `ci` = channels of the tensor being gathered, `co` = channels produced
template <typename F>
static int dispatch(int ci, int co, F&& f) {
#define VC_CASE_CO(CIv, COv) \
    if (co == COv) return f(std::integral_constant<int, CIv>{}, std::integral_constant<int, COv>{});
#define VC_CASE_CI(CIv) \
    if (ci == CIv) { VC_CASE_CO(CIv, 8) VC_CASE_CO(CIv, 16) VC_CASE_CO(CIv, 32) VC_CASE_CO(CIv, 64) }
    VC_CASE_CI(8) VC_CASE_CI(16) VC_CASE_CI(32) VC_CASE_CI(64)
#undef VC_CASE_CI
#undef VC_CASE_CO
    set_error("unsupported channel pair (%d, %d): need 8/16/32/64", ci, co);
    return VC_ERR_UNSUPPORTED;
}

static int wgrad_chunks(int n_out, int K, int* rows_per_chunk) {
    int R = (2 * 132 + K - 1) / K;
    if (R > 64) R = 64;
    int max_r = (n_out + WG_WIN - 1) / WG_WIN;
    if (R > max_r) R = max_r;
    if (R < 1) R = 1;
    int rpc = ((n_out + R - 1) / R + WG_WIN - 1) / WG_WIN * WG_WIN;
    if (rpc < WG_WIN) rpc = WG_WIN;
    R = (n_out + rpc - 1) / rpc;
    if (R < 1) R = 1;
    *rows_per_chunk = rpc;
    return R;
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_conv_ws_bytes(int cin, int cout, int K) { return (size_t)K * cin * cout * sizeof(float); }

static int prep(const float* w, float* wt, int cin, int cout, int K, int mode, int mirror, cudaStream_t stream) {
    int total = K * cin * cout;
    prep_weights_kernel<<<dim3(cdiv(total, 256)), dim3(256), 0, stream>>>(w, wt, cin, cout, K, mode, mirror);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

static int check_conv_args(int n, int cin, int cout, int K, const void* a, const void* b, const void* c, const void* d,
                           void* ws, size_t ws_bytes) {
    VC_CHECK_ARG(n >= 0 && K >= 1 && K <= MAXK, "bad n=%d or K=%d", n, K);
    if (!ch_ok(cin) || !ch_ok(cout)) {
        set_error("unsupported channels cin=%d cout=%d (need 8/16/32/64)", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(a && b && c && d && ws, "null pointer");
    if (ws_bytes < vc_conv_ws_bytes(cin, cout, K)) {
        set_error("conv workspace %zu < %zu", ws_bytes, vc_conv_ws_bytes(cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    return VC_OK;
}

extern "C" int vc_conv_fwd_f32(const float* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                               int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = check_conv_args(n_out, cin, cout, K, in, w, nbr, out, ws, ws_bytes);
    if (rc || n_out == 0) return rc;
    float* wt = (float*)ws;
    if ((rc = prep(w, wt, cin, cout, K, 0, 0, stream))) return rc;
    return dispatch(cin, cout, [&](auto ci, auto co) {
        return launch_gather<decltype(ci)::value, decltype(co)::value>(in, wt, nbr, out, n_out, K, bn_sums, stream);
    });
}

int vc::conv_fwd_f32_part(const float* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin, int cout, int K,
                          double* bn_part, void* ws, size_t ws_bytes, cudaStream_t stream) {
    static_assert(TM == TCM_ROWS, "BN partials are per 128-row tile in both conv kernels");
    int rc = check_conv_args(n_out, cin, cout, K, in, w, nbr, out, ws, ws_bytes);
    if (rc || n_out == 0) return rc;
    VC_CHECK_ARG(bn_part, "null pointer");
    float* wt = (float*)ws;
    if ((rc = prep(w, wt, cin, cout, K, 0, 0, stream))) return rc;
    return dispatch(cin, cout, [&](auto ci, auto co) {
        return launch_gather<decltype(ci)::value, decltype(co)::value>(in, wt, nbr, out, n_out, K, nullptr, stream, bn_part);
    });
}

extern "C" int vc_conv_dgrad_f32(const float* dout, const float* w, const int32_t* nbr_t, float* din, int n_in, int cin,
                                 int cout, int K, int mirror, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = check_conv_args(n_in, cin, cout, K, dout, w, nbr_t, din, ws, ws_bytes);
    if (rc || n_in == 0) return rc;
    float* wt = (float*)ws;
    if ((rc = prep(w, wt, cin, cout, K, 1, mirror, stream))) return rc;
    return dispatch(cout, cin, [&](auto ci, auto co) {
        return launch_gather<decltype(ci)::value, decltype(co)::value>(dout, wt, nbr_t, din, n_in, K, nullptr, stream);
    });
}

int vc::conv_dgrad_scatter_f32_ld(const float* dout, const float* w, const int32_t* nbr, float* din, int din_ld, int n_out,
                                  int cin, int cout, int K, void* ws, size_t ws_bytes, cudaStream_t stream) {
    int rc = check_conv_args(n_out, cin, cout, K, dout, w, nbr, din, ws, ws_bytes);
    if (rc || n_out == 0) return rc;
    VC_CHECK_ARG(din_ld >= cin && din_ld % 4 == 0, "scatter dgrad: row pitch %d for %d channels", din_ld, cin);
    float* wt = (float*)ws;
    if ((rc = prep(w, wt, cin, cout, K, 1, 0, stream))) return rc;
    return dispatch(cout, cin, [&](auto ci, auto co) {
        return launch_scatter<decltype(ci)::value, decltype(co)::value>(dout, wt, nbr, din, din_ld, n_out, K, stream);
    });
}

extern "C" int vc_conv_dgrad_scatter_f32(const float* dout, const float* w, const int32_t* nbr, float* din, int n_out,
                                         int cin, int cout, int K, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    return vc::conv_dgrad_scatter_f32_ld(dout, w, nbr, din, cin, n_out, cin, cout, K, ws, ws_bytes, (cudaStream_t)stream_);
}

extern "C" size_t vc_conv_wgrad_ws_bytes(int n_out, int cin, int cout, int K) {
    int rpc;
    int R = wgrad_chunks(n_out, K, &rpc);
    return (size_t)R * K * cin * cout * sizeof(float);
}

extern "C" int vc_conv_wgrad_f32(const float* in, const float* dout, const int32_t* nbr, float* dw, int n_out, int cin,
                                 int cout, int K, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK && dw, "bad arguments");
    if (!ch_ok(cin) || !ch_ok(cout)) {
        set_error("unsupported channels cin=%d cout=%d (need 8/16/32/64)", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) {
        VC_CUDA(cudaMemsetAsync(dw, 0, (size_t)K * cin * cout * 4, stream));
        return VC_OK;
    }
    VC_CHECK_ARG(in && dout && nbr && ws, "null pointer");
    int rpc;
    int R = wgrad_chunks(n_out, K, &rpc);
    if (ws_bytes < (size_t)R * K * cin * cout * 4) {
        set_error("wgrad workspace %zu < %zu", ws_bytes, (size_t)R * K * cin * cout * 4);
        return VC_ERR_WORKSPACE;
    }
    float* partial = (float*)ws;
    int rc = dispatch(cin, cout, [&](auto ci, auto co) {
        return launch_wgrad<decltype(ci)::value, decltype(co)::value>(in, dout, nbr, partial, n_out, K, R, rpc, stream);
    });
    if (rc) return rc;
    int total = K * cin * cout;
    wgrad_reduce_kernel<<<cdiv(total, 256), 256, 0, stream>>>(partial, dw, R, K, cin, cout);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
