// Input gradient of the many-to-one 2-D image tables in gather form — deterministic, sm_90a.
//
// The image branch's submanifold tables map several rows to one pixel (rule 3 of DESIGN.md section 2: a neighbour look-up
// resolves to the LOWEST row at that pixel, the centre tap is the row itself).  The default backward scatters
// dout[o] @ W_k^T onto the looked-up rows with float atomics (tc_scatter_kernel, scatter_gemm_kernel), whose order varies.
// Here, used by the plan executor's deterministic mode: a non-centre tap of row o reads the representative (lowest) row at
// pixel p(o) + delta_k, so representative i receives W_k^T S[p(i) - delta_k], with S[p] the sum of dout over the rows at
// pixel p, and every row i receives its centre term W_c^T dout[i].  With U = [dout; S] (2 cap rows, S stored at its
// representative's row) this is ONE mirrored gather dgrad over the table nbr_g (see common.cuh), run by the existing gather
// kernels (gather_gemm_kernel, tc_conv_persist_kernel).  S is summed in ascending row order per pixel: rows are grouped
// with integer atomics (count, scan, place), each group is sorted, then summed.  Everything is integer work or a
// fixed-order fp32 sum: the same bits on every run.
#include <cuda_bf16.h>

#include "tc_common.cuh"

#define VC_TRY_RC(expr)           \
    do {                          \
        int rc__ = (expr);        \
        if (rc__) return rc__;    \
    } while (0)

namespace vc {
namespace {

constexpr int G2_SCAN = 1024;   // elements per block of the two-level scan (so cap <= 1024 * 1024)

__device__ __forceinline__ int rows_of(int cap, const int* n_dev) { return n_dev != nullptr ? min(cap, __ldg(n_dev)) : cap; }

// The grouping below is shared with the deterministic voxel-RoI pooling (voxel_pool.cu, roi_pool.cu): elements o in
// [0, E) (E capped by *n_dev when given) go to group key[o]; a negative key belongs to no group.
__global__ void g2_count_kernel(const int32_t* __restrict__ key, int E, const int* __restrict__ n_dev, int* cnt) {
    const int n = rows_of(E, n_dev), o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < n) {
        const int r = key[o];
        if (r >= 0) atomicAdd(&cnt[r], 1);
    }
}

__device__ __forceinline__ int block_incl_scan(int v, int* wsum) {   // inclusive scan over a 1024-thread block
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) wsum[w] = x;
    __syncthreads();
    if (w == 0) {
        int s = wsum[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += y;
        }
        wsum[lane] = s;
    }
    __syncthreads();
    return x + (w > 0 ? wsum[w - 1] : 0);
}

// off[i] = exclusive prefix of cnt inside its block of 1024, tot[b] = the block's total
__global__ void __launch_bounds__(G2_SCAN) g2_scan_local_kernel(const int* __restrict__ cnt, int cap, int* off, int* tot) {
    __shared__ int wsum[32];
    const int i = blockIdx.x * G2_SCAN + threadIdx.x;
    const int v = i < cap ? cnt[i] : 0;
    const int incl = block_incl_scan(v, wsum);
    if (i < cap) off[i] = incl - v;
    if (threadIdx.x == G2_SCAN - 1) tot[blockIdx.x] = incl;
}

// tot -> its exclusive prefix (one block)
__global__ void __launch_bounds__(G2_SCAN) g2_scan_tot_kernel(int* tot, int nb) {
    __shared__ int wsum[32];
    const int v = threadIdx.x < nb ? tot[threadIdx.x] : 0;
    const int incl = block_incl_scan(v, wsum);
    if (threadIdx.x < nb) tot[threadIdx.x] = incl - v;
}

// grid (cdiv(cap, 256), K): the gather table; the blocks of plane 0 also finish the group offsets
__global__ void g2_table_kernel(const int32_t* __restrict__ nbr, const int32_t* __restrict__ rep, int K, int cap,
                                const int* __restrict__ n_dev, int* off, const int* __restrict__ tot, int32_t* __restrict__ nbr_g) {
    const int n = rows_of(cap, n_dev), i = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
    if (i >= cap) return;
    if (k == 0) off[i] += tot[i / G2_SCAN];
    int v = -1;
    if (i < n) {
        if (k == K / 2) {
            v = i;                                   // centre tap: the row's own gradient (U rows [0, cap))
        } else if (rep[i] == i) {
            const int j = nbr[(size_t)k * cap + i];
            v = j >= 0 ? cap + j : -1;               // S of the pixel the tap reads (U rows [cap, 2 cap))
        }
    }
    nbr_g[(size_t)k * cap + i] = v;
}

__global__ void g2_place_kernel(const int32_t* __restrict__ key, int E, const int* __restrict__ n_dev, const int* __restrict__ off,
                                int* cur, int32_t* rows) {
    const int n = rows_of(E, n_dev), o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o < n) {
        const int r = key[o];
        if (r >= 0) rows[off[r] + atomicAdd(&cur[r], 1)] = o;
    }
}

// off[i] += tot[its block]: the second half of the two-level scan (gather2d does this inside g2_table_kernel)
__global__ void g2_scan_add_kernel(int* off, const int* __restrict__ tot, int G) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < G) off[i] += tot[i / G2_SCAN];
}

// the elements of each group in ascending order.  Without a `big` list every group is insertion-sorted by one thread (the
// rows of one pixel: short groups); with it, groups longer than G2_SHORT are queued there for g2_sort_big_kernel.
constexpr int G2_SHORT = 32;
__global__ void g2_sort_kernel(const int* __restrict__ cnt, const int* __restrict__ off, int cap, const int* __restrict__ n_dev,
                               int32_t* rows, int32_t* big, int* nbig) {
    const int n = rows_of(cap, n_dev), r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const int m = cnt[r];
    if (m < 2) return;
    if (big != nullptr && m > G2_SHORT) {
        big[atomicAdd(nbig, 1)] = r;      // queue order is irrelevant: each group is sorted on its own
        return;
    }
    int32_t* p = rows + off[r];
    for (int a = 1; a < m; ++a) {
        const int v = p[a];
        int b = a - 1;
        while (b >= 0 && p[b] > v) {
            p[b + 1] = p[b];
            --b;
        }
        p[b + 1] = v;
    }
}

// One block per long group (grid-stride over the queue): a merge sort of the group's distinct elements by rank — in pass
// w every element of a run of w goes to (its index in the run) + (the number of smaller elements of the partner run, by
// binary search).  log2(m) passes of O(m log m): never quadratic in the group size.  Groups up to G2_BIG_SMEM elements
// are sorted in shared memory, longer ones between `rows` and `scratch` (same offsets) in global memory.
constexpr int G2_BIG_THREADS = 256, G2_BIG_SMEM = 4096;

__device__ __forceinline__ void g2_merge_pass(const int32_t* src, int32_t* dst, int m, int w) {
    for (int i = threadIdx.x; i < m; i += G2_BIG_THREADS) {
        const int v = src[i], a = i / w, s0 = a * w, s1 = (a ^ 1) * w;
        int lo = s1 < m ? s1 : m, hi = s1 + w < m ? s1 + w : m;
        const int base = lo;
        while (lo < hi) {                          // first element of the partner run >= v
            const int mid = (lo + hi) >> 1;
            if (src[mid] < v) lo = mid + 1;
            else hi = mid;
        }
        dst[(a & ~1) * w + (i - s0) + (lo - base)] = v;
    }
}

__global__ void __launch_bounds__(G2_BIG_THREADS) g2_sort_big_kernel(const int* __restrict__ cnt, const int* __restrict__ off,
                                                                     const int32_t* __restrict__ big, const int* __restrict__ nbig,
                                                                     int32_t* rows, int32_t* scratch) {
    __shared__ int32_t buf[2][G2_BIG_SMEM];
    const int nq = *nbig;
    for (int q = blockIdx.x; q < nq; q += gridDim.x) {
        const int r = big[q], m = cnt[r];
        int32_t* p = rows + off[r];
        int32_t *src, *dst;
        if (m <= G2_BIG_SMEM) {
            for (int i = threadIdx.x; i < m; i += G2_BIG_THREADS) buf[0][i] = p[i];
            src = buf[0]; dst = buf[1];
        } else {
            src = p; dst = scratch + off[r];
        }
        __syncthreads();
        for (int w = 1; w < m; w <<= 1) {
            g2_merge_pass(src, dst, m, w);
            __syncthreads();
            int32_t* t = src; src = dst; dst = t;
        }
        if (src != p)
            for (int i = threadIdx.x; i < m; i += G2_BIG_THREADS) p[i] = src[i];
        __syncthreads();
    }
}

// thread per (group, 4 channels): U[cap + r] = sum over the group's rows in ascending order
__global__ void g2_sum_kernel(const float4* __restrict__ g, const uint2* __restrict__ gb, int c4, const int* __restrict__ cnt,
                              const int* __restrict__ off, const int32_t* __restrict__ rows, int cap, const int* __restrict__ n_dev,
                              float4* u, uint2* ub) {
    const int n = rows_of(cap, n_dev);
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int r = (int)(t / c4), q = (int)(t % c4);
    if (r >= n) return;
    const int m = cnt[r];
    if (m == 0) return;
    const int32_t* p = rows + off[r];
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < m; ++j) {
        const size_t e = (size_t)p[j] * c4 + q;
        float4 v;
        if (g != nullptr) {
            v = g[e];
        } else {
            const uint2 w = gb[e];
            const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w.x));
            const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w.y));
            v = make_float4(lo.x, lo.y, hi.x, hi.y);
        }
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    const size_t o = (size_t)(cap + r) * c4 + q;
    if (u != nullptr) u[o] = s;
    if (ub != nullptr) {
        __nv_bfloat162 a = __floats2bfloat162_rn(s.x, s.y), b = __floats2bfloat162_rn(s.z, s.w);
        ub[o] = make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&b));
    }
}

__global__ void add_rows_ld_kernel(float4* dst, int ld4, const float4* __restrict__ src, int cap, const int* __restrict__ n_dev, int c4) {
    const size_t total = (size_t)rows_of(cap, n_dev) * c4;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t r = i / c4, q = i % c4;
        float4 a = dst[r * ld4 + q];
        const float4 b = src[i];
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        dst[r * ld4 + q] = a;
    }
}

size_t al256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

size_t slot_groups_bytes(int E, int G) {
    return 3 * al256((size_t)E * 4) + 5 * al256((size_t)G * 4) + al256((size_t)G2_SCAN * 4) + 256;
}

SlotGroups slot_groups_carve(void* ws, int E, int G) {
    char* p = (char*)ws;
    SlotGroups P;
    P.key = (int32_t*)p; p += al256((size_t)E * 4);
    P.rows = (int32_t*)p; p += al256((size_t)E * 4);
    P.scratch = (int32_t*)p; p += al256((size_t)E * 4);
    P.cnt = (int32_t*)p; p += al256((size_t)G * 4);
    P.cur = (int32_t*)p; p += al256((size_t)G * 4);
    P.nbig = (int32_t*)p; p += 256;                         // (cnt, cur and nbig adjacent: one memset)
    P.off = (int32_t*)p; p += al256((size_t)G * 4);
    P.big = (int32_t*)p; p += al256((size_t)G * 4);
    P.tot = (int32_t*)p;
    return P;
}

int slot_groups_dev(int E, int G, const SlotGroups& P, int max_ctas, cudaStream_t st) {
    VC_CHECK_ARG(E >= 0 && G >= 0, "slot groups: %d elements, %d groups", E, G);
    if (G > G2_SCAN * G2_SCAN) {
        set_error("slot groups: %d groups > %d", G, G2_SCAN * G2_SCAN);
        return VC_ERR_UNSUPPORTED;
    }
    if (G == 0) return VC_OK;
    VC_CUDA(cudaMemsetAsync(P.cnt, 0, (size_t)((char*)P.off - (char*)P.cnt), st));
    if (E > 0) {
        g2_count_kernel<<<cdiv(E, 256), 256, 0, st>>>(P.key, E, nullptr, P.cnt);
        VC_LAUNCH_CHECK();
    }
    const int nb = cdiv(G, G2_SCAN);
    g2_scan_local_kernel<<<nb, G2_SCAN, 0, st>>>(P.cnt, G, P.off, P.tot);
    VC_LAUNCH_CHECK();
    g2_scan_tot_kernel<<<1, G2_SCAN, 0, st>>>(P.tot, nb);
    VC_LAUNCH_CHECK();
    g2_scan_add_kernel<<<cdiv(G, 256), 256, 0, st>>>(P.off, P.tot, G);
    VC_LAUNCH_CHECK();
    if (E == 0) return VC_OK;
    g2_place_kernel<<<cdiv(E, 256), 256, 0, st>>>(P.key, E, nullptr, P.off, P.cur, P.rows);
    VC_LAUNCH_CHECK();
    g2_sort_kernel<<<cdiv(G, 128), 128, 0, st>>>(P.cnt, P.off, G, nullptr, P.rows, P.big, P.nbig);
    VC_LAUNCH_CHECK();
    int blocks = num_sms() * 4;
    if (max_ctas > 0 && max_ctas < blocks) blocks = max_ctas;
    g2_sort_big_kernel<<<blocks, G2_BIG_THREADS, 0, st>>>(P.cnt, P.off, P.big, P.nbig, P.rows, P.scratch);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

size_t gather2d_prep_bytes(int cap, int K) {
    return al256((size_t)K * cap * 4) + 5 * al256((size_t)cap * 4) + al256((size_t)G2_SCAN * 4);
}

G2Prep gather2d_carve(void* ws, int cap, int K) {
    char* p = (char*)ws;
    G2Prep P;
    P.nbr_g = (int32_t*)p; p += al256((size_t)K * cap * 4);
    P.cnt = (int32_t*)p; p += al256((size_t)cap * 4);
    P.cur = (int32_t*)p; p += al256((size_t)cap * 4);      // (cnt and cur adjacent: one memset)
    P.off = (int32_t*)p; p += al256((size_t)cap * 4);
    P.rows = (int32_t*)p; p += al256((size_t)cap * 4);
    P.tot = (int32_t*)p;
    return P;
}

int gather2d_prep_dev(const int32_t* nbr, const int32_t* rep, int K, int cap, const int* n_dev, const G2Prep& P, cudaStream_t st) {
    VC_CHECK_ARG(cap >= 0 && cap <= G2_SCAN * G2_SCAN && K >= 1 && (K & 1), "gather-form 2-D dgrad: %d rows, K=%d", cap, K);
    if (cap == 0) return VC_OK;
    VC_CHECK_ARG(nbr && rep, "null pointer");
    VC_CUDA(cudaMemsetAsync(P.cnt, 0, (size_t)((char*)P.off - (char*)P.cnt), st));
    g2_count_kernel<<<cdiv(cap, 256), 256, 0, st>>>(rep, cap, n_dev, P.cnt);
    VC_LAUNCH_CHECK();
    const int nb = cdiv(cap, G2_SCAN);
    g2_scan_local_kernel<<<nb, G2_SCAN, 0, st>>>(P.cnt, cap, P.off, P.tot);
    VC_LAUNCH_CHECK();
    g2_scan_tot_kernel<<<1, G2_SCAN, 0, st>>>(P.tot, nb);
    VC_LAUNCH_CHECK();
    g2_table_kernel<<<dim3(cdiv(cap, 256), K), 256, 0, st>>>(nbr, rep, K, cap, n_dev, P.off, P.tot, P.nbr_g);
    VC_LAUNCH_CHECK();
    g2_place_kernel<<<cdiv(cap, 256), 256, 0, st>>>(rep, cap, n_dev, P.off, P.cur, P.rows);
    VC_LAUNCH_CHECK();
    g2_sort_kernel<<<cdiv(cap, 128), 128, 0, st>>>(P.cnt, P.off, cap, n_dev, P.rows, nullptr, nullptr);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int gather2d_sum_dev(const float* g, const void* g_bf16, int c, const G2Prep& P, int cap, const int* n_dev, float* u, void* u_bf16,
                     cudaStream_t st) {
    VC_CHECK_ARG(c > 0 && c % 4 == 0 && (g || g_bf16) && (u || u_bf16), "gather-form 2-D dgrad: bad sum arguments");
    if (cap == 0) return VC_OK;
    const int c4 = c / 4;
    g2_sum_kernel<<<dim3(cdiv((long long)cap * c4, 256)), dim3(256), 0, st>>>((const float4*)g, (const uint2*)g_bf16, c4,
        (const int*)P.cnt, (const int*)P.off, (const int32_t*)P.rows, cap, n_dev, (float4*)u, (uint2*)u_bf16);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int add_rows_ld_dev(float* dst, int ld, const float* src, int cap, const int* n_dev, int c, cudaStream_t st) {
    VC_CHECK_ARG(c % 4 == 0 && ld % 4 == 0 && ld >= c, "add_rows_ld: c=%d ld=%d", c, ld);
    if (cap == 0) return VC_OK;
    size_t b = ((size_t)cap * (c / 4) + 255) / 256;
    if (b > 132 * 8) b = 132 * 8;
    add_rows_ld_kernel<<<dim3((int)b), dim3(256), 0, st>>>((float4*)dst, ld / 4, (const float4*)src, cap, n_dev, c / 4);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_conv_dgrad_gather2d_ws_bytes(int n, int cin, int cout, int K) {
    if (n < 0 || K < 1) return 0;
    return gather2d_prep_bytes(n, K) + ((2 * (size_t)n * cout * 4 + 255) & ~(size_t)255) +
           (size_t)K * (cin > 16 ? cin : 16) * (cout > 16 ? cout : 16) * 4;
}

// precision 0: fp32 dout, fp32 gather kernel; 1: bf16 dout, tensor-core gather kernel
static int gather2d_call(int precision, const void* dout, const float* w, const int32_t* nbr, const int32_t* rep, float* din, int n,
                         const int32_t* n_dev, int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err, cudaStream_t st) {
    VC_CHECK_ARG(n >= 0 && K >= 1 && K <= MAXK_TC && (K & 1), "bad n=%d or K=%d", n, K);
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("gather-form 2-D dgrad: unsupported channels cin=%d cout=%d", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(dout && w && nbr && rep && din && ws, "null pointer");
    if (ws_bytes < vc_conv_dgrad_gather2d_ws_bytes(n, cin, cout, K)) {
        set_error("gather-form 2-D dgrad workspace %zu < %zu", ws_bytes, vc_conv_dgrad_gather2d_ws_bytes(n, cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    const G2Prep P = gather2d_carve(ws, n, K);
    char* u = (char*)ws + gather2d_prep_bytes(n, K);
    char* wimg = u + ((2 * (size_t)n * cout * 4 + 255) & ~(size_t)255);
    VC_TRY_RC(gather2d_prep_dev(nbr, rep, K, n, n_dev, P, st));
    const size_t esz = precision ? 2 : 4;
    VC_CUDA(cudaMemcpyAsync(u, dout, (size_t)n * cout * esz, cudaMemcpyDeviceToDevice, st));
    if (n_dev != nullptr) VC_CUDA(cudaMemsetAsync(din, 0, (size_t)n * cin * 4, st));
    if (precision == 0) {
        VC_TRY_RC(gather2d_sum_dev((const float*)dout, nullptr, cout, P, n, n_dev, (float*)u, nullptr, st));
        return vc_conv_dgrad_f32((const float*)u, w, P.nbr_g, din, n, cin, cout, K, 1, wimg, (size_t)K * cin * cout * 4, st);
    }
    VC_TRY_RC(gather2d_sum_dev(nullptr, dout, cout, P, n, n_dev, nullptr, u, st));
    TcPrepTable T;
    T.n = 1;
    TcPrepEntry& e = T.e[0];
    e.w = w; e.img = wimg; e.cin = cin; e.cout = cout; e.K = K; e.mode = 1; e.mirror = 1; e.layout = 1; e.first = 0;
    VC_TRY_RC(tc_prep_images(T, st));
    return tc2_conv(cout, cin, u, wimg, P.nbr_g, n, din, n, n_dev, K, nullptr, err, st, nullptr);
}

extern "C" int vc_conv_dgrad_gather2d_f32(const float* dout, const float* w, const int32_t* nbr, const int32_t* rep, float* din,
                                          int n, const int32_t* n_dev, int cin, int cout, int K, void* ws, size_t ws_bytes,
                                          vc_stream_t stream) {
    return gather2d_call(0, dout, w, nbr, rep, din, n, n_dev, cin, cout, K, ws, ws_bytes, nullptr, (cudaStream_t)stream);
}

extern "C" int vc_conv_dgrad_gather2d_tc(const void* dout_bf16, const float* w, const int32_t* nbr, const int32_t* rep, float* din,
                                         int n, const int32_t* n_dev, int cin, int cout, int K, void* ws, size_t ws_bytes,
                                         int32_t* err_flag, vc_stream_t stream) {
    return gather2d_call(1, dout_bf16, w, nbr, rep, din, n, n_dev, cin, cout, K, ws, ws_bytes, err_flag, (cudaStream_t)stream);
}
