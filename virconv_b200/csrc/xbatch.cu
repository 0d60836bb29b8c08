// Test-time x-batching of the ROT_NUM transformed copies (spconv_backbone.py:339-471) without a host read — sm_90a.
//
// VirConv-T / -S evaluate R transformed copies of a scene in one LiDAR-stream pass: copy i's voxels are shifted by i*W
// along x into a [D, H, 4W] grid (:418-432; the factor 4 is hard-coded, :360), and the published tensors are split back
// into copies afterwards (`decompose_tensor`, :314-337).  Both steps here keep every row count in device memory, so the
// whole test-time forward can be captured into a CUDA graph.
//
//   vc_xbatch_pack : R <= 4 capacity-sized copies (features [cap_i, C] fp32, coordinates [cap_i, 4] int32 (b, z, y, x),
//                    valid row count *n_dev[i]) -> one capacity-sized input of cap_out >= sum(cap_i) rows: the valid rows of
//                    copy 0, then of copy 1, ... (the row order of torch.cat over the exact rows), x += i * W; zero feature
//                    tail, -1 coordinate tail, *n_out = sum of the counts.  One launch.
//   vc_xbatch_split: one capacity-sized published tensor (features [cap, C] fp32 with C in {16, 32, 64}, indices [cap, 4]
//                    int32, valid row count *n_dev, rows past it are never read) of a grid whose x extent is Wt -> R outputs,
//                    each with the parent's capacity (the split cannot overflow).  With q = Wt / 4, output i holds the rows
//                    with i*q < x < (i+1)*q in the parent's row order (strict on both sides: the x == i*q column belongs to no
//                    copy, the reference's rule at :325), x -= i*q; zero feature tail, -1 index tail, its own count
//                    *n_out[i].  An order-preserving compaction of all copies together in three launches: per-tile counts of
//                    every copy, one scan over the tiles, ranks from warp ballots.
// R outside [1, 4] -> VC_ERR_INVALID.  Both results are the same on every run.
#include "common.cuh"

namespace vc {
namespace {

constexpr int XB_MAX = 4;           // copies along x: the reference's fixed factor
constexpr int TILE = 256;           // rows per block of the split's count / emit passes
constexpr int SCAN_THREADS = 1024;

struct PackSrc {
    const float* f[XB_MAX];
    const int32_t* c[XB_MAX];
    const int* n[XB_MAX];
    int cap[XB_MAX];
};

struct SplitDst {
    float* f[XB_MAX];
    int32_t* c[XB_MAX];
    int* n[XB_MAX];
};

__device__ __forceinline__ int clamp_rows(const int* n_dev, int cap) {
    const int n = __ldg(n_dev);
    return n < 0 ? 0 : (n > cap ? cap : n);
}

// one thread per output row: which copy (if any) the row comes from, then its coordinates and features
__global__ void __launch_bounds__(256) xbatch_pack_kernel(PackSrc s, int R, int C, int W, int cap_out, float* __restrict__ out_f,
                                                          int32_t* __restrict__ out_c, int* __restrict__ n_out) {
    int base[XB_MAX + 1];
    base[0] = 0;
#pragma unroll
    for (int i = 0; i < XB_MAX; ++i) base[i + 1] = base[i] + (i < R ? clamp_rows(s.n[i], s.cap[i]) : 0);
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) *n_out = base[R];
    if (r >= cap_out) return;
    int cp = -1;
#pragma unroll
    for (int i = XB_MAX - 1; i >= 0; --i)
        if (i < R && r < base[i + 1]) cp = i;
    int32_t* oc = out_c + (size_t)r * 4;
    float* of = out_f + (size_t)r * C;
    if (cp < 0) {
        oc[0] = oc[1] = oc[2] = oc[3] = -1;
        for (int ch = 0; ch < C; ++ch) of[ch] = 0.f;
        return;
    }
    const size_t src = (size_t)(r - base[cp]);
    const int32_t* ic = s.c[cp] + src * 4;
    oc[0] = ic[0];
    oc[1] = ic[1];
    oc[2] = ic[2];
    oc[3] = ic[3] + cp * W;
    const float* inf = s.f[cp] + src * C;
    for (int ch = 0; ch < C; ++ch) of[ch] = inf[ch];
}

// the copy a live row belongs to: i*q < x < (i+1)*q for some i < R, else -1
__device__ __forceinline__ int copy_of(const int32_t* __restrict__ idx, long long p, int n, int q, int R) {
    if (p >= n) return -1;
    const int x = idx[p * 4 + 3];
    if (x <= 0) return -1;
    const int c = x / q;
    return (c < R && x != c * q) ? c : -1;
}

// exclusive rank of `f` among the TILE threads of the block (every thread takes part)
__device__ __forceinline__ int block_rank(bool f, int* s_w) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    __syncthreads();
    if (lane == 0) s_w[w] = __popc(m);
    __syncthreads();
    int off = 0;
#pragma unroll
    for (int j = 0; j < TILE / 32; ++j) off += j < w ? s_w[j] : 0;
    return off + __popc(m & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(TILE) xbatch_count_kernel(const int32_t* __restrict__ idx, int cap, const int* __restrict__ n_dev,
                                                           int q, int R, int nb, int* __restrict__ blk) {
    const int n = clamp_rows(n_dev, cap);
    const int cp = copy_of(idx, (long long)blockIdx.x * TILE + threadIdx.x, n, q, R);
    for (int i = 0; i < R; ++i) {
        const int k = __syncthreads_count(cp == i);
        if (threadIdx.x == 0) blk[(size_t)i * nb + blockIdx.x] = k;
    }
}

// one block: blk[i][b] := rows of copy i in the tiles before b; *n_out[i] := rows of copy i
__global__ void __launch_bounds__(SCAN_THREADS) xbatch_scan_kernel(int* __restrict__ blk, int nb, int R, SplitDst d) {
    __shared__ int s_w[SCAN_THREADS / 32];
    __shared__ int s_carry;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int i = 0; i < R; ++i) {
        int* row = blk + (size_t)i * nb;
        if (threadIdx.x == 0) s_carry = 0;
        __syncthreads();
        for (int base = 0; base < nb; base += SCAN_THREADS) {
            const int b = base + threadIdx.x;
            const int v = b < nb ? row[b] : 0;
            int x = v;
#pragma unroll
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
            const int excl = s_carry + woff + x - v;
            __syncthreads();
            if (b < nb) row[b] = excl;
            if (threadIdx.x == 0) s_carry += tot;
            __syncthreads();
        }
        if (threadIdx.x == 0) *d.n[i] = s_carry;
        __syncthreads();
    }
}

// every parent row p goes to position blk[copy][tile] + rank of its copy's output; position p of every output at or past
// that output's count gets the tail (zero features, -1 indices).  Features are moved by the whole block, float4 by float4.
__global__ void __launch_bounds__(TILE) xbatch_emit_kernel(const float4* __restrict__ f, const int32_t* __restrict__ idx, int cap,
                                                          const int* __restrict__ n_dev, int q, int R, int c4, const int* __restrict__ blk,
                                                          int nb, SplitDst d) {
    __shared__ int s_w[TILE / 32];
    __shared__ int s_cp[TILE], s_dst[TILE], s_tot[XB_MAX];
    const int n = clamp_rows(n_dev, cap);
    const long long p0 = (long long)blockIdx.x * TILE;
    const long long p = p0 + threadIdx.x;
    const int cp = copy_of(idx, p, n, q, R);
    if (threadIdx.x < R) s_tot[threadIdx.x] = *d.n[threadIdx.x];
    int dst = -1;
    for (int i = 0; i < R; ++i) {
        const int r = block_rank(cp == i, s_w);
        if (cp == i) dst = blk[(size_t)i * nb + blockIdx.x] + r;
    }
    s_cp[threadIdx.x] = cp;
    s_dst[threadIdx.x] = dst;
    __syncthreads();
    if (p < cap) {
        if (cp >= 0) {
            int4 v = *reinterpret_cast<const int4*>(idx + p * 4);
            v.w -= cp * q;
            *reinterpret_cast<int4*>(d.c[cp] + (size_t)dst * 4) = v;
        }
        for (int i = 0; i < R; ++i)
            if (p >= s_tot[i]) *reinterpret_cast<int4*>(d.c[i] + p * 4) = make_int4(-1, -1, -1, -1);
    }
    const long long rows = cap - p0 < TILE ? cap - p0 : TILE;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = threadIdx.x; e < rows * c4; e += TILE) {
        const int r = e / c4, ch = e % c4;
        const long long pp = p0 + r;
        const int c = s_cp[r];
        if (c >= 0) reinterpret_cast<float4*>(d.f[c])[(size_t)s_dst[r] * c4 + ch] = f[pp * c4 + ch];
        for (int i = 0; i < R; ++i)
            if (pp >= s_tot[i]) reinterpret_cast<float4*>(d.f[i])[pp * c4 + ch] = zero;
    }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_xbatch_pack(const float* const* feats, const int32_t* const* coords, const int32_t* const* n_dev,
                              const int32_t* caps, int R, int c, int W, int cap_out, float* out_features, int32_t* out_coords,
                              int32_t* n_out_dev, vc_stream_t stream) {
    VC_CHECK_ARG(R >= 1 && R <= XB_MAX, "vc_xbatch_pack: %d copies (1..%d: the x-batching factor is 4)", R, XB_MAX);
    VC_CHECK_ARG(feats && coords && n_dev && caps && c > 0 && W > 0 && cap_out >= 0 && n_out_dev,
                 "vc_xbatch_pack: bad arguments (c %d, W %d, cap_out %d)", c, W, cap_out);
    PackSrc s{};
    long long total = 0;
    for (int i = 0; i < R; ++i) {
        VC_CHECK_ARG(caps[i] >= 0 && n_dev[i] && (caps[i] == 0 || (feats[i] && coords[i])), "vc_xbatch_pack: copy %d", i);
        s.f[i] = feats[i];
        s.c[i] = coords[i];
        s.n[i] = n_dev[i];
        s.cap[i] = caps[i];
        total += caps[i];
    }
    VC_CHECK_ARG(total <= cap_out, "vc_xbatch_pack: output capacity %d < %lld input rows", cap_out, total);
    VC_CHECK_ARG(cap_out == 0 || (out_features && out_coords), "vc_xbatch_pack: null output");
    const int grid = cap_out > 0 ? cdiv(cap_out, 256) : 1;
    xbatch_pack_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(s, R, c, W, cap_out, out_features, out_coords, n_out_dev);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_xbatch_split_ws_bytes(int cap, int R) {
    const size_t nb = cap > 0 ? ((size_t)cap + TILE - 1) / TILE : 0;
    return align256((size_t)(R > 0 ? R : 0) * nb * 4);
}

extern "C" int vc_xbatch_split(const float* features, const int32_t* indices, int cap, const int32_t* n_dev, int c, int Wt, int R,
                               float* const* out_features, int32_t* const* out_indices, int32_t* const* n_out_dev, void* ws,
                               size_t ws_bytes, vc_stream_t stream) {
    VC_CHECK_ARG(R >= 1 && R <= XB_MAX, "vc_xbatch_split: %d copies (1..%d: the x-batching factor is 4)", R, XB_MAX);
    if (!(c == 16 || c == 32 || c == 64)) {
        set_error("vc_xbatch_split: %d channels (16, 32 or 64)", c);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(cap >= 0 && Wt >= 4 && n_dev && out_features && out_indices && n_out_dev,
                 "vc_xbatch_split: bad arguments (cap %d, Wt %d)", cap, Wt);
    SplitDst d{};
    for (int i = 0; i < R; ++i) {
        VC_CHECK_ARG(n_out_dev[i] && (cap == 0 || (out_features[i] && out_indices[i])), "vc_xbatch_split: output %d", i);
        d.f[i] = out_features[i];
        d.c[i] = out_indices[i];
        d.n[i] = n_out_dev[i];
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (cap == 0) {
        for (int i = 0; i < R; ++i) VC_CUDA(cudaMemsetAsync(d.n[i], 0, 4, st));
        return VC_OK;
    }
    VC_CHECK_ARG(features && indices && ws && ws_bytes >= vc_xbatch_split_ws_bytes(cap, R),
                 "vc_xbatch_split: inputs / workspace (%zu < %zu bytes)", ws_bytes, vc_xbatch_split_ws_bytes(cap, R));
    const int nb = cdiv(cap, TILE), q = Wt / 4;
    int* blk = (int*)ws;
    xbatch_count_kernel<<<nb, TILE, 0, st>>>(indices, cap, n_dev, q, R, nb, blk);
    VC_LAUNCH_CHECK();
    xbatch_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(blk, nb, R, d);
    VC_LAUNCH_CHECK();
    xbatch_emit_kernel<<<nb, TILE, 0, st>>>((const float4*)features, indices, cap, n_dev, q, R, c / 4, blk, nb, d);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
