// index2uv, dense(), row gather, error plumbing — sm_90a.
#include <cuda_bf16.h>
#include <stdarg.h>

#include "common.cuh"

namespace vc {

static thread_local char g_err[512] = "";
static long long g_launches = 0;
void count_launch() { ++g_launches; }

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

struct UVGrid {
    float vx, vy, vz, mx, my, mz;
};

// Voxel index -> pixel cell.  Every float op is an explicitly rounded fp32 multiply / add / divide in the
// order oracle/index2uv.py fixes (no FMA contraction), so the integer result is bit-identical to it.
// Reference arithmetic: spconv_backbone.py:8-24,54-83; X_transform.py:139-154; calibration_kitti.py:120-153.
__device__ __forceinline__ void index2uv_row(const int4* __restrict__ idx, int n, const int* __restrict__ n_dev,
                                             int batch_size, const float* __restrict__ params, const UVGrid& g, int stride,
                                             int u_max, int v_max, int32_t* __restrict__ uv, int i) {
    if (n_dev != nullptr) n = min(n, __ldg(n_dev));
    if (i >= n) return;
    int4 v = idx[i];  // (b, z, y, x)
    int b = v.x;
    float x = __fadd_rn(__fmul_rn((float)v.w, g.vx), g.mx);
    float y = __fadd_rn(__fmul_rn((float)v.z, g.vy), g.my);
    float z = __fadd_rn(__fmul_rn((float)v.y, g.vz), g.mz);
    int ui = 0, vi = 0;
    if (b >= 0 && b < batch_size) {
        const float* p = params + (size_t)b * 28;
        if (p[20] != 0.f) {
            float sc = p[21];
            x = __fdiv_rn(x, sc);
            y = __fdiv_rn(y, sc);
            z = __fdiv_rn(z, sc);
            if (p[22] != 0.f) y = -y;
            float c = p[23], s = p[24];
            float xr = __fadd_rn(__fmul_rn(x, c), __fmul_rn(y, -s));
            float yr = __fadd_rn(__fmul_rn(x, s), __fmul_rn(y, c));
            x = xr;
            y = yr;
        }
        float r[3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
            r[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, p[0 * 3 + j]), __fmul_rn(y, p[1 * 3 + j])),
                                       __fmul_rn(z, p[2 * 3 + j])),
                             p[3 * 3 + j]);
        float h[2];
#pragma unroll
        for (int j = 0; j < 2; ++j)
            h[j] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], p[12 + 0 * 2 + j]), __fmul_rn(r[1], p[12 + 1 * 2 + j])),
                                       __fmul_rn(r[2], p[12 + 2 * 2 + j])),
                             p[12 + 3 * 2 + j]);
        float uf = __fdiv_rn(h[0], r[2]);
        float vf = __fdiv_rn(h[1], r[2]);
        ui = __float2int_rz(uf);  // saturating, NaN -> 0: what `.int()` gives on the reference's CUDA path
        vi = __float2int_rz(vf);
    }
    ui = min(max(ui, 0), u_max - 1) / stride;
    vi = min(max(vi, 0), v_max - 1) / stride;
    int32_t* o = uv + (size_t)i * 3;
    o[0] = b;
    o[1] = ui;
    o[2] = vi;
}

__global__ void __launch_bounds__(256) index2uv_kernel(const int4* __restrict__ idx, int n, const int* __restrict__ n_dev,
                                                       int batch_size, const float* __restrict__ params, UVGrid g, int stride,
                                                       int u_max, int v_max, int32_t* __restrict__ uv) {
    index2uv_row(idx, n, n_dev, batch_size, params, g, stride, u_max, v_max, uv, blockIdx.x * blockDim.x + threadIdx.x);
}

// up to IDX_BATCH_MAX projections in one launch: stage e owns the blocks blk0[e] .. blk0[e + 1] - 1
struct UVEntry {
    const int4* idx;
    const int* n_dev;
    int32_t* uv;
    UVGrid g;
    int n, stride, u_max, v_max;
};
struct UVBatch {
    int E, batch_size;
    const float* params;
    int blk0[IDX_BATCH_MAX + 1];
    UVEntry e[IDX_BATCH_MAX];
};

__global__ void __launch_bounds__(256) index2uv_kernel(const __grid_constant__ UVBatch ub) {
    int i = 0;
    while (i + 1 < ub.E && (int)blockIdx.x >= ub.blk0[i + 1]) ++i;
    const UVEntry& e = ub.e[i];
    index2uv_row(e.idx, e.n, e.n_dev, ub.batch_size, ub.params, e.g, e.stride, e.u_max, e.v_max, e.uv,
                 (blockIdx.x - ub.blk0[i]) * blockDim.x + threadIdx.x);
}

// n_dev (may be NULL): device row count of a capacity-sized tensor (n = capacity); rows at or past it are not scattered, and
// their gradient is zero
__global__ void dense_kernel(const float* __restrict__ feat, const int32_t* __restrict__ idx, int n, int c, int ndim,
                             long long spatial, const int* __restrict__ n_dev, int s0, int s1, int s2,
                             float* __restrict__ out, int backward, float* __restrict__ dfeat) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * c) return;
    int row = (int)(t / c), ch = (int)(t % c);
    if (n_dev != nullptr && row >= __ldg(n_dev)) {
        if (backward) dfeat[t] = 0.f;
        return;
    }
    const int32_t* p = idx + (size_t)row * (1 + ndim);
    long long cell = p[1];
    if (ndim >= 2) cell = cell * s1 + p[2];
    if (ndim >= 3) cell = cell * s2 + p[3];
    long long o = ((long long)p[0] * c + ch) * spatial + cell;
    if (!backward)
        out[o] = feat[t];
    else
        dfeat[t] = out[o];
}

__global__ void gather_rows_kernel(const uint4* __restrict__ in, const int32_t* __restrict__ rows, uint4* __restrict__ out,
                                   int n_rows, int chunks) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n_rows * chunks) return;
    int r = (int)(t / chunks), c = (int)(t % chunks);
    out[t] = in[(size_t)rows[r] * chunks + c];
}
__global__ void gather_rows4_kernel(const uint32_t* __restrict__ in, const int32_t* __restrict__ rows,
                                    uint32_t* __restrict__ out, int n_rows, int words) {
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n_rows * words) return;
    int r = (int)(t / words), c = (int)(t % words);
    out[t] = in[(size_t)rows[r] * words + c];
}

// out[:, :ca] = a, out[:, ca:] = b (fp32) plus an optional bf16 shadow of the same matrix; float4 granularity
// (n_dev: device row count, n = capacity; rows [count, capacity) are written as zeros — the concat is a published tensor)
__global__ void cat2_kernel(const float4* __restrict__ a, const float4* __restrict__ b, float4* __restrict__ out,
                            uint2* __restrict__ out_bf16, int n, const int* __restrict__ n_dev, int ca4, int cb4) {
    const int cnt = n_dev != nullptr ? min(n, __ldg(n_dev)) : n;
    long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int w = ca4 + cb4;
    if (t >= (long long)n * w) return;
    int r = (int)(t / w), c = (int)(t % w);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < cnt) v = c < ca4 ? a[(size_t)r * ca4 + c] : b[(size_t)r * cb4 + (c - ca4)];
    out[t] = v;
    if (out_bf16 != nullptr) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<uint32_t*>(&lo);
        o.y = *reinterpret_cast<uint32_t*>(&hi);
        out_bf16[t] = o;
    }
}

// mean of the first n rows of a [cap, c] matrix: float64 per-thread sums over float4s in a fixed grid-stride order, a
// fixed-order block reduction, and the last CTA (atomic ticket) adds the CTA partials — all its threads, each over a fixed
// subset, then the same block reduction — so the result depends on the grid size only, never on timing.
constexpr int MM_THREADS = 256;

__device__ __forceinline__ double mm_block_sum(double s, double* warp_s) {   // valid in thread 0
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) warp_s[threadIdx.x >> 5] = s;
    __syncthreads();
    double b = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < MM_THREADS / 32; ++w) b += warp_s[w];
    return b;
}

__global__ void __launch_bounds__(MM_THREADS) masked_mean_kernel(const float4* __restrict__ x, long long cap_rows,
                                                                 const int* __restrict__ n_dev, int c4, double* part,
                                                                 unsigned* ticket, float* out) {
    const long long n = n_dev != nullptr ? min(cap_rows, (long long)max(__ldg(n_dev), 0)) : cap_rows;
    const long long total4 = n * c4;
    const long long stride = (long long)gridDim.x * MM_THREADS;
    long long i = (long long)blockIdx.x * MM_THREADS + threadIdx.x;
    double s = 0.0;
    for (; i + 3 * stride < total4; i += 4 * stride) {   // four loads in flight per thread
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = x[i + u * stride];
#pragma unroll
        for (int u = 0; u < 4; ++u) s += ((double)v[u].x + (double)v[u].y) + ((double)v[u].z + (double)v[u].w);
    }
    for (; i < total4; i += stride) {
        const float4 v = x[i];
        s += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
    }
    __shared__ double warp_s[MM_THREADS / 32];
    __shared__ bool last;
    const double b = mm_block_sum(s, warp_s);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = b;
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double t = 0.0;
    for (unsigned k = threadIdx.x; k < gridDim.x; k += MM_THREADS) t += __ldcg(part + k);
    t = mm_block_sum(t, warp_s);
    if (threadIdx.x == 0) *out = (float)(t / (double)(n * c4 * 4));   // (no rows: 0/0 = NaN, as torch's mean of an empty tensor)
}

// gradient of that mean: dx[r, :] = g / (n*c) for r < n, 0 for the rows [n, cap)
__global__ void __launch_bounds__(MM_THREADS) masked_mean_bwd_kernel(const float* __restrict__ g, long long cap_rows,
                                                                     const int* __restrict__ n_dev, int c4, float4* __restrict__ dx) {
    const long long n = n_dev != nullptr ? min(cap_rows, (long long)max(__ldg(n_dev), 0)) : cap_rows;
    const float v = __fdiv_rn(__ldg(g), (float)(n * c4 * 4));
    const float4 val = make_float4(v, v, v, v), zero = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long live4 = n * c4, total4 = cap_rows * c4;
    for (long long i = (long long)blockIdx.x * MM_THREADS + threadIdx.x; i < total4; i += (long long)gridDim.x * MM_THREADS)
        dx[i] = i < live4 ? val : zero;
}

int mm_grid(long long cap_rows, int c) {   // a function of the capacity only: the reduction order of a shape is fixed
    const long long b = cdiv(cap_rows * c / 4, (long long)MM_THREADS * 8);
    return (int)(b < 1 ? 1 : (b > 4 * 132 ? 4 * 132 : b));
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_masked_mean_ws_bytes(void) { return 256 + 4 * 132 * sizeof(double); }

extern "C" int vc_masked_mean_f32(const float* x, long long cap_rows, int c, const int32_t* n_dev, float* out, void* ws,
                                  size_t ws_bytes, vc_stream_t stream_) {
    VC_CHECK_ARG(cap_rows >= 0 && c > 0 && c % 4 == 0, "masked mean: bad shape [%lld, %d]", cap_rows, c);
    VC_CHECK_ARG(x && out && ws && ws_bytes >= vc_masked_mean_ws_bytes(), "masked mean: null pointer / workspace too small");
    VC_CUDA(cudaMemsetAsync(ws, 0, sizeof(unsigned), (cudaStream_t)stream_));   // the ticket
    masked_mean_kernel<<<mm_grid(cap_rows, c), MM_THREADS, 0, (cudaStream_t)stream_>>>(
        (const float4*)x, cap_rows, n_dev, c / 4, (double*)((char*)ws + 256), (unsigned*)ws, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_masked_mean_bwd_f32(const float* g, long long cap_rows, int c, const int32_t* n_dev, float* dx,
                                      vc_stream_t stream_) {
    VC_CHECK_ARG(cap_rows >= 0 && c > 0 && c % 4 == 0, "masked mean: bad shape [%lld, %d]", cap_rows, c);
    VC_CHECK_ARG(g && (dx || cap_rows == 0), "masked mean: null pointer");
    if (cap_rows == 0) return VC_OK;
    masked_mean_bwd_kernel<<<mm_grid(cap_rows, c), MM_THREADS, 0, (cudaStream_t)stream_>>>(g, cap_rows, n_dev, c / 4, (float4*)dx);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int vc::cat2_dev(const float* a, const float* b, float* out, void* out_bf16, int n, const int* n_dev, int ca, int cb,
                 cudaStream_t stream) {
    VC_CHECK_ARG(n >= 0 && ca > 0 && cb > 0 && ca % 4 == 0 && cb % 4 == 0, "bad cat2 arguments");
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(a && b && out, "null pointer");
    long long total = (long long)n * (ca + cb) / 4;
    cat2_kernel<<<dim3(cdiv(total, 256)), dim3(256), 0, stream>>>((const float4*)a, (const float4*)b, (float4*)out,
        (uint2*)out_bf16, n, n_dev, ca / 4, cb / 4);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_cat2_f32(const float* a, const float* b, float* out, void* out_bf16, int n, int ca, int cb,
                           vc_stream_t stream_) {
    return vc::cat2_dev(a, b, out, out_bf16, n, nullptr, ca, cb, (cudaStream_t)stream_);
}

extern "C" int vc_version(void) { return 100; }
extern "C" const char* vc_last_error(void) { return g_err; }
extern "C" long long vc_launch_count(void) { return g_launches; }

int vc::index2uv_dev(const int32_t* indices, int n, const int* n_dev, int batch_size, const float* params, const float* grid,
                     int stride, int u_max, int v_max, int32_t* uv_out, cudaStream_t stream) {
    VC_CHECK_ARG(n >= 0 && batch_size > 0 && stride > 0 && u_max > 0 && v_max > 0 && grid, "bad index2uv arguments");
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(indices && params && uv_out, "null pointer");
    UVGrid g{grid[0], grid[1], grid[2], grid[3], grid[4], grid[5]};
    index2uv_kernel<<<cdiv(n, 256), 256, 0, stream>>>((const int4*)indices, n, n_dev, batch_size, params, g, stride, u_max, v_max,
                                                      uv_out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int vc::index2uv_batch_dev(const UVStage* st, int n_st, int batch_size, const float* params, cudaStream_t stream) {
    VC_CHECK_ARG(n_st >= 1 && n_st <= IDX_BATCH_MAX && batch_size > 0, "bad index2uv batch");
    UVBatch ub;
    memset(&ub, 0, sizeof(ub));
    ub.batch_size = batch_size;
    ub.params = params;
    for (int i = 0; i < n_st; ++i) {
        const UVStage& s = st[i];
        VC_CHECK_ARG(s.n >= 0 && s.stride > 0 && s.u_max > 0 && s.v_max > 0 && s.grid, "bad index2uv arguments");
        if (s.n == 0) continue;
        VC_CHECK_ARG(s.idx && params && s.uv, "null pointer");
        UVEntry& e = ub.e[ub.E];
        e.idx = (const int4*)s.idx; e.n_dev = s.n_dev; e.uv = s.uv; e.n = s.n; e.stride = s.stride; e.u_max = s.u_max;
        e.v_max = s.v_max;
        e.g = UVGrid{s.grid[0], s.grid[1], s.grid[2], s.grid[3], s.grid[4], s.grid[5]};
        ub.blk0[ub.E + 1] = ub.blk0[ub.E] + cdiv(s.n, 256);
        ++ub.E;
    }
    if (ub.E == 0) return VC_OK;
    index2uv_kernel<<<ub.blk0[ub.E], 256, 0, stream>>>(ub);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_index2uv(const int32_t* indices, int n, int batch_size, const float* params, const float* grid,
                           int stride, int u_max, int v_max, int32_t* uv_out, vc_stream_t stream_) {
    return vc::index2uv_dev(indices, n, nullptr, batch_size, params, grid, stride, u_max, v_max, uv_out, (cudaStream_t)stream_);
}

static int dense_common(const float* features, const int32_t* indices, int n, int c, int ndim, int batch_size,
                        const int32_t* shape, float* dense, float* dfeat, int backward, cudaStream_t stream,
                        const int32_t* n_dev = nullptr) {
    VC_CHECK_ARG(n >= 0 && c > 0 && ndim >= 1 && ndim <= VC_MAX_NDIM && batch_size > 0 && shape, "bad dense arguments");
    if (n == 0) return VC_OK;
    long long spatial = 1;
    for (int d = 0; d < ndim; ++d) spatial *= shape[d];
    long long total = (long long)n * c;
    dense_kernel<<<cdiv(total, 256), 256, 0, stream>>>(features, indices, n, c, ndim, spatial, n_dev, shape[0],
                                                       ndim > 1 ? shape[1] : 1, ndim > 2 ? shape[2] : 1, dense, backward,
                                                       dfeat);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_dense_f32(const float* features, const int32_t* indices, int n, int c, int ndim, int batch_size,
                            const int32_t* spatial_shape, float* out, vc_stream_t stream_) {
    return dense_common(features, indices, n, c, ndim, batch_size, spatial_shape, out, nullptr, 0, (cudaStream_t)stream_);
}

extern "C" int vc_dense_bwd_f32(const float* dout, const int32_t* indices, int n, int c, int ndim, int batch_size,
                                const int32_t* spatial_shape, float* dfeatures, vc_stream_t stream_) {
    return dense_common(nullptr, indices, n, c, ndim, batch_size, spatial_shape, const_cast<float*>(dout), dfeatures, 1,
                        (cudaStream_t)stream_);
}

extern "C" int vc_dense_rows_f32(const float* features, const int32_t* indices, int cap, const int32_t* n_dev, int c, int ndim,
                                 int batch_size, const int32_t* spatial_shape, float* out, vc_stream_t stream_) {
    VC_CHECK_ARG(n_dev, "vc_dense_rows_f32: null row count");
    return dense_common(features, indices, cap, c, ndim, batch_size, spatial_shape, out, nullptr, 0, (cudaStream_t)stream_, n_dev);
}

extern "C" int vc_dense_rows_bwd_f32(const float* dout, const int32_t* indices, int cap, const int32_t* n_dev, int c, int ndim,
                                     int batch_size, const int32_t* spatial_shape, float* dfeatures, vc_stream_t stream_) {
    VC_CHECK_ARG(n_dev, "vc_dense_rows_bwd_f32: null row count");
    return dense_common(nullptr, indices, cap, c, ndim, batch_size, spatial_shape, const_cast<float*>(dout), dfeatures, 1,
                        (cudaStream_t)stream_, n_dev);
}

extern "C" int vc_gather_rows(const void* in, const int32_t* rows, void* out, int n_rows, int row_bytes,
                              vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_rows >= 0 && row_bytes > 0 && row_bytes % 4 == 0, "bad gather arguments");
    if (n_rows == 0) return VC_OK;
    VC_CHECK_ARG(in && rows && out, "null pointer");
    if (row_bytes % 16 == 0 && ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 16 == 0)) {
        int chunks = row_bytes / 16;
        gather_rows_kernel<<<cdiv((long long)n_rows * chunks, 256), 256, 0, stream>>>((const uint4*)in, rows, (uint4*)out,
                                                                                      n_rows, chunks);
    } else {
        int words = row_bytes / 4;
        gather_rows4_kernel<<<cdiv((long long)n_rows * words, 256), 256, 0, stream>>>((const uint32_t*)in, rows,
                                                                                      (uint32_t*)out, n_rows, words);
    }
    VC_LAUNCH_CHECK();
    return VC_OK;
}
