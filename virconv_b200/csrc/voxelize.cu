// Hash-grid voxelisation + MeanVFE on the GPU — sm_90a.
//
// Replaces, with identical results, the CPU pair the reference runs in its dataloader / first model module:
//   * `VoxelGeneratorWrapper.generate` -> spconv `Point2VoxelCPU3d.point_to_voxel`
//     (pcdet/datasets/processor/data_processor.py:43-59, called at :156,:173): first-come voxel order per sample,
//     at most `max_voxels` voxels per sample, at most `max_points` points per voxel in point order, zyx coordinates;
//   * `MeanVFE.forward` (pcdet/models/backbones_3d/vfe/mean_vfe.py:39-58): per-voxel mean over the kept points,
//     last channel := max over the (zero-padded) slots when MODEL == 'max'.
// The sequential first-come semantics are recovered deterministically:
//   first point of a voxel  = atomicMin of the point index in a coordinate hash table   (-> voxel identity)
//   voxel order in a sample = rank of that first point among all first points           (bitmap + popcount scan)
//   first `max_points` points of a voxel in point order = lock-free atomicMin cascade over `max_points` slots
// Integer results (coords, counts, order) are bit exact against the numpy restatement; features are bit exact too
// because the per-voxel sum runs over the slots in slot order like the reference's sum over dim 1.
#include "common.cuh"

namespace vc {

static constexpr unsigned long long VH_EMPTY = ~0ULL;
static constexpr int VROW_BITS = 24;
static constexpr int VSCAN_WORDS = 2048;
static constexpr int VMAX_PTS = 8;
static constexpr int VSENT = 0x7f7f7f7f;   // memset-able sentinel, larger than any point index (< 2^24)

struct VoxGeom {
    float lo[3], vs[3];
    int grid[3];   // x, y, z
    int batch;
};

__device__ __forceinline__ bool point_voxel(const float* __restrict__ p, const VoxGeom& g, int& b, int* c) {
    b = (int)p[0];
    bool ok = b >= 0 && b < g.batch;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        // floor((p - lo) / vs) in fp32, the arithmetic of the reference voxeliser.  A NaN would convert to cell 0 and a point
        // with a NaN coordinate be kept: the reference's range tests are false for NaN, so it is dropped here too
        const float q = floorf(__fdiv_rn(__fsub_rn(p[1 + d], g.lo[d]), g.vs[d]));
        const int v = (int)q;
        ok &= isfinite(q) & (v >= 0) & (v < g.grid[d]);
        c[d] = v;
    }
    return ok;
}

__device__ __forceinline__ unsigned long long vkey(const VoxGeom& g, int b, const int* c) {
    return (((unsigned long long)b * g.grid[2] + c[2]) * g.grid[1] + c[1]) * g.grid[0] + c[0];
}

__global__ void vox_insert_kernel(const float* __restrict__ pts, int n, int stride, VoxGeom g, unsigned long long* table,
                                  uint32_t mask) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int b, c[3];
    if (!point_voxel(pts + (size_t)i * stride, g, b, c)) return;
    unsigned long long key = vkey(g, b, c);
    unsigned long long packed = (key << VROW_BITS) | (unsigned long long)i;
    uint32_t slot = mix64(key) & mask;
    while (true) {
        unsigned long long cur = table[slot];
        if (cur == VH_EMPTY) {
            cur = atomicCAS(&table[slot], VH_EMPTY, packed);
            if (cur == VH_EMPTY) return;
        }
        if ((cur >> VROW_BITS) == key) {
            atomicMin(&table[slot], packed);     // earliest point of the voxel
            return;
        }
        slot = (slot + 1) & mask;
    }
}

// per point: head = first point of its voxel; head bitmap; first-`max_points` slots of the voxel; sample starts
__global__ void __launch_bounds__(256) vox_assign_kernel(const float* __restrict__ pts, int n, int stride, VoxGeom g,
                                                         const unsigned long long* __restrict__ table, uint32_t mask,
                                                         int max_points, int32_t* __restrict__ head_of,
                                                         uint32_t* __restrict__ head_bits, int32_t* __restrict__ slots,
                                                         int32_t* __restrict__ sample_start) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    int head = -1;
    bool is_head = false;
    if (i < n) {
        const float* p = pts + (size_t)i * stride;
        int b, c[3];
        if (point_voxel(p, g, b, c)) {
            unsigned long long key = vkey(g, b, c);
            uint32_t slot = mix64(key) & mask;
            while (true) {
                unsigned long long cur = __ldg(table + slot);
                if ((cur >> VROW_BITS) == key) {
                    head = (int)(cur & ((1ULL << VROW_BITS) - 1));
                    break;
                }
                slot = (slot + 1) & mask;
            }
            is_head = head == i;
            int x = i;   // keep the max_points smallest point indices of the voxel, ascending
            int32_t* s = slots + (size_t)head * max_points;
            for (int r = 0; r < max_points && x != VSENT; ++r) {
                int old = atomicMin(&s[r], x);
                x = max(old, x);
            }
        }
        head_of[i] = head;
        int bi = (int)p[0];
        int bprev = i > 0 ? (int)pts[(size_t)(i - 1) * stride] : -1;
        if (bi != bprev && bi >= 0 && bi < g.batch) sample_start[bi] = i;   // samples are contiguous, ascending
    }
    unsigned m = __ballot_sync(0xffffffffu, is_head);
    if ((threadIdx.x & 31) == 0 && i < n + 31) head_bits[i >> 5] = m;
}

__global__ void __launch_bounds__(256) vscan_local_kernel(const uint32_t* __restrict__ bits, int n_words,
                                                          uint32_t* __restrict__ word_rank, uint32_t* __restrict__ block_sum) {
    __shared__ uint32_t warp_tot[8];
    int base = blockIdx.x * VSCAN_WORDS + threadIdx.x * 8;
    uint32_t cnt[8], tsum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int w = base + j;
        cnt[j] = (w < n_words) ? __popc(bits[w]) : 0;
        tsum += cnt[j];
    }
    uint32_t incl = tsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((threadIdx.x & 31) >= o) incl += v;
    }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
    __syncthreads();
    uint32_t woff = 0;
    for (int w = 0; w < (threadIdx.x >> 5); ++w) woff += warp_tot[w];
    uint32_t run = woff + incl - tsum;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int w = base + j;
        if (w < n_words) word_rank[w] = run;
        run += cnt[j];
    }
    if (threadIdx.x == 255) block_sum[blockIdx.x] = woff + incl;
}

__device__ __forceinline__ int head_rank(const uint32_t* bits, const uint32_t* word_rank, const uint32_t* block_off, int i) {
    int w = i >> 5;
    return (int)(block_off[w / VSCAN_WORDS] + word_rank[w] + __popc(bits[w] & ((1u << (i & 31)) - 1u)));
}

// one block: exclusive scan of the block sums, then per-sample voxel counts / output offsets
__global__ void __launch_bounds__(1024) vox_offsets_kernel(uint32_t* block_sum, int n_blocks, const uint32_t* __restrict__ bits,
                                                           const uint32_t* __restrict__ word_rank, int n, int batch,
                                                           int max_voxels, const int32_t* __restrict__ sample_start,
                                                           int32_t* __restrict__ sample_base_rank,
                                                           int32_t* __restrict__ sample_out_off, int32_t* __restrict__ n_out) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n_blocks; base += 1024) {
        int i = base + threadIdx.x;
        uint32_t v = (i < n_blocks) ? block_sum[i] : 0, incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
            if ((threadIdx.x & 31) >= o) incl += t;
        }
        if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
        __syncthreads();
        uint32_t woff = 0;
        for (int w = 0; w < (threadIdx.x >> 5); ++w) woff += warp_tot[w];
        uint32_t carry = carry_s;
        if (i < n_blocks) block_sum[i] = carry + woff + incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + woff + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int total_heads = (int)carry_s;
        int off = 0;
        for (int b = 0; b < batch; ++b) {
            int start = sample_start[b];            // n if the sample has no point
            int next = n;
            for (int b2 = b + 1; b2 < batch; ++b2)
                if (sample_start[b2] < n) { next = sample_start[b2]; break; }
            int r0 = start < n ? head_rank(bits, word_rank, block_sum, start) : total_heads;
            int r1 = next < n ? head_rank(bits, word_rank, block_sum, next) : total_heads;
            if (start >= n) r1 = r0;
            sample_base_rank[b] = r0;
            sample_out_off[b] = off;
            off += min(r1 - r0, max_voxels);
        }
        *n_out = off;
    }
}

// the reference's max over a voxel's slots (torch / numpy max): NaN if either is NaN, where fmaxf would drop it
__device__ __forceinline__ float max_nan(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }

// one thread per point: heads that survive the per-sample cap emit their voxel (coords, count, mean / max features)
__global__ void __launch_bounds__(256) vox_emit_kernel(const float* __restrict__ pts, int n, int stride, int c, VoxGeom g,
                                                       const int32_t* __restrict__ head_of, const uint32_t* __restrict__ bits,
                                                       const uint32_t* __restrict__ word_rank,
                                                       const uint32_t* __restrict__ block_off,
                                                       const int32_t* __restrict__ slots, int max_points, int max_voxels,
                                                       const int32_t* __restrict__ sample_base_rank,
                                                       const int32_t* __restrict__ sample_out_off, int vfe_max_last,
                                                       float* __restrict__ out_feat, int32_t* __restrict__ out_coords,
                                                       int32_t* __restrict__ out_num, float* __restrict__ out_voxels) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || head_of[i] != i) return;
    const float* p = pts + (size_t)i * stride;
    int b, cc[3];
    point_voxel(p, g, b, cc);
    int vid = head_rank(bits, word_rank, block_off, i) - sample_base_rank[b];
    if (vid >= max_voxels) return;
    int row = sample_out_off[b] + vid;
    const int32_t* s = slots + (size_t)i * max_points;
    int cnt = 0;
    float sum[16], mx = 0.f;   // zero padding takes part in the max, as in the reference's padded [M, P, C] tensor
    for (int ch = 0; ch < c; ++ch) sum[ch] = 0.f;
    bool first = true;
    for (int r = 0; r < max_points; ++r) {
        int pi = s[r];
        if (pi == VSENT) break;
        const float* q = pts + (size_t)pi * stride + 1;
        for (int ch = 0; ch < c; ++ch) {
            float v = q[ch];
            sum[ch] = __fadd_rn(sum[ch], v);
            if (out_voxels != nullptr) out_voxels[((size_t)row * max_points + r) * c + ch] = v;
        }
        mx = first ? q[c - 1] : max_nan(mx, q[c - 1]);
        first = false;
        ++cnt;
    }
    if (cnt < max_points) mx = max_nan(mx, 0.f);
    float denom = (float)max(cnt, 1);
    for (int ch = 0; ch < c; ++ch) out_feat[(size_t)row * c + ch] = __fdiv_rn(sum[ch], denom);
    if (vfe_max_last) out_feat[(size_t)row * c + c - 1] = mx;
    out_num[row] = cnt;
    int32_t* oc = out_coords + (size_t)row * 4;
    oc[0] = b; oc[1] = cc[2]; oc[2] = cc[1]; oc[3] = cc[0];
}

// dense voxel -> row map of `generate_voxel2pinds` (pcdet/utils/spconv_utils.py:13-21); out pre-filled with -1.  n_dev (may
// be NULL): device row count of a capacity-sized index tensor (n = capacity); rows at or past it are skipped
__global__ void voxel2pinds_kernel(const int32_t* __restrict__ idx, int n, const int* __restrict__ n_dev, int ndim, int s1, int s2,
                                   long long spatial, int32_t* __restrict__ out) {
    int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    if (n_dev != nullptr && row >= __ldg(n_dev)) return;
    const int32_t* p = idx + (size_t)row * (1 + ndim);
    long long cell = p[1];
    if (ndim >= 2) cell = cell * s1 + p[2];
    if (ndim >= 3) cell = cell * s2 + p[3];
    out[(long long)p[0] * spatial + cell] = row;
}

struct VoxWs {
    uint32_t slots_pow2;
    int n_words, n_blocks;
    unsigned long long* table;
    int32_t *head_of, *slots, *sample_start, *sample_base, *sample_off;
    uint32_t *bits, *word_rank, *block_sum;
    size_t bytes;
};

static VoxWs vox_layout(int n, int batch, int max_points, void* ws) {
    VoxWs w;
    uint32_t s = 1024;
    while (s < 2u * (uint32_t)(n > 0 ? n : 1)) s <<= 1;
    w.slots_pow2 = s;
    w.n_words = (n + 31) / 32 + 1;
    w.n_blocks = (w.n_words + VSCAN_WORDS - 1) / VSCAN_WORDS;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p + off; off += (bytes + 255) / 256 * 256; return r; };
    w.table = (unsigned long long*)take((size_t)s * 8);
    w.head_of = (int32_t*)take((size_t)n * 4);
    w.slots = (int32_t*)take((size_t)n * max_points * 4);
    w.bits = (uint32_t*)take((size_t)w.n_words * 4);
    w.word_rank = (uint32_t*)take((size_t)w.n_words * 4);
    w.block_sum = (uint32_t*)take((size_t)w.n_blocks * 4);
    w.sample_start = (int32_t*)take((size_t)batch * 4);
    w.sample_base = (int32_t*)take((size_t)batch * 4);
    w.sample_off = (int32_t*)take((size_t)batch * 4);
    w.bytes = off;
    return w;
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_voxelize_ws_bytes(int n_points, int batch_size, int max_points) {
    return vox_layout(n_points, batch_size, max_points, nullptr).bytes;
}

extern "C" int vc_voxelize_mean(const float* points, int n_points, int c, int batch_size, const float* pc_range,
                                const float* voxel_size, int max_points, int max_voxels, int vfe_max_last,
                                float* out_features, int32_t* out_coords, int32_t* out_num, float* out_voxels,
                                int32_t* n_out_dev, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_points >= 0 && n_points < (1 << VROW_BITS) && c >= 1 && c <= 16 && batch_size >= 1 && batch_size <= 1024,
                 "bad voxelize sizes");
    VC_CHECK_ARG(max_points >= 1 && max_points <= VMAX_PTS && max_voxels >= 1 && pc_range && voxel_size && n_out_dev && ws,
                 "bad voxelize arguments");
    VoxGeom g;
    g.batch = batch_size;
    double cells = batch_size;
    for (int d = 0; d < 3; ++d) {
        g.lo[d] = pc_range[d];
        g.vs[d] = voxel_size[d];
        g.grid[d] = (int)llround(((double)pc_range[3 + d] - (double)pc_range[d]) / (double)voxel_size[d]);
        VC_CHECK_ARG(g.grid[d] > 0, "empty grid");
        cells *= g.grid[d];
    }
    VC_CHECK_ARG(cells < 1099511627776.0, "grid too large for 40-bit keys");
    VoxWs w = vox_layout(n_points, batch_size, max_points, ws);
    if (ws_bytes < w.bytes) {
        set_error("voxelize workspace %zu < %zu", ws_bytes, w.bytes);
        return VC_ERR_WORKSPACE;
    }
    if (n_points == 0) {
        VC_CUDA(cudaMemsetAsync(n_out_dev, 0, 4, stream));
        return VC_OK;
    }
    VC_CHECK_ARG(points && out_features && out_coords && out_num, "null pointer");
    const int stride = 1 + c;
    VC_CUDA(cudaMemsetAsync(w.table, 0xFF, (size_t)w.slots_pow2 * 8, stream));
    VC_CUDA(cudaMemsetAsync(w.slots, 0x7F, (size_t)n_points * max_points * 4, stream));   // = VSENT everywhere
    VC_CUDA(cudaMemsetAsync(w.bits, 0, (size_t)w.n_words * 4, stream));
    VC_CUDA(cudaMemsetAsync(w.sample_start, 0x7F, (size_t)batch_size * 4, stream));
    vox_insert_kernel<<<cdiv(n_points, 256), 256, 0, stream>>>(points, n_points, stride, g, w.table, w.slots_pow2 - 1);
    VC_LAUNCH_CHECK();
    vox_assign_kernel<<<cdiv(n_points + 31, 256), 256, 0, stream>>>(points, n_points, stride, g, w.table, w.slots_pow2 - 1,
                                                                    max_points, w.head_of, w.bits, w.slots, w.sample_start);
    VC_LAUNCH_CHECK();
    vscan_local_kernel<<<w.n_blocks, 256, 0, stream>>>(w.bits, w.n_words, w.word_rank, w.block_sum);
    VC_LAUNCH_CHECK();
    vox_offsets_kernel<<<1, 1024, 0, stream>>>(w.block_sum, w.n_blocks, w.bits, w.word_rank, n_points, batch_size, max_voxels,
                                               w.sample_start, w.sample_base, w.sample_off, n_out_dev);
    VC_LAUNCH_CHECK();
    vox_emit_kernel<<<cdiv(n_points, 256), 256, 0, stream>>>(points, n_points, stride, c, g, w.head_of, w.bits, w.word_rank,
                                                             w.block_sum, w.slots, max_points, max_voxels, w.sample_base,
                                                             w.sample_off, vfe_max_last, out_features, out_coords, out_num,
                                                             out_voxels);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

static int voxel2pinds_common(const int32_t* indices, int n, const int32_t* n_dev, int ndim, int batch_size,
                              const int32_t* spatial_shape, int32_t* out, cudaStream_t stream) {
    VC_CHECK_ARG(n >= 0 && ndim >= 1 && ndim <= VC_MAX_NDIM && batch_size > 0 && spatial_shape && out, "bad arguments");
    long long spatial = 1;
    for (int d = 0; d < ndim; ++d) spatial *= spatial_shape[d];
    VC_CUDA(cudaMemsetAsync(out, 0xFF, (size_t)batch_size * spatial * 4, stream));
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(indices, "null pointer");
    voxel2pinds_kernel<<<cdiv(n, 256), 256, 0, stream>>>(indices, n, n_dev, ndim, ndim > 1 ? spatial_shape[1] : 1,
                                                         ndim > 2 ? spatial_shape[2] : 1, spatial, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_voxel2pinds(const int32_t* indices, int n, int ndim, int batch_size, const int32_t* spatial_shape,
                              int32_t* out, vc_stream_t stream_) {
    return voxel2pinds_common(indices, n, nullptr, ndim, batch_size, spatial_shape, out, (cudaStream_t)stream_);
}

extern "C" int vc_voxel2pinds_rows(const int32_t* indices, int cap, const int32_t* n_dev, int ndim, int batch_size,
                                   const int32_t* spatial_shape, int32_t* out, vc_stream_t stream_) {
    VC_CHECK_ARG(n_dev, "vc_voxel2pinds_rows: null row count");
    return voxel2pinds_common(indices, cap, n_dev, ndim, batch_size, spatial_shape, out, (cudaStream_t)stream_);
}
