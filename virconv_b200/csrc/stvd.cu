// StVD input point discard (bin-based, distance-aware) on the GPU — sm_90a.
//
// Replaces `DatasetTemplate.partition` + `DatasetTemplate.input_point_discard` (pcdet/datasets/dataset.py:120-189), which
// the reference runs per sample in numpy inside the dataloader (called at :275-290 for the virtual points of every
// frame): points are split into `bin_num` range bins along x (bin i = [i*w, (i+1)*w), w = 60/bin_num; the last bin is
// open-ended; x < 0 or NaN falls in no bin and is dropped), the bins are emitted far -> near, and the nearest `pos` bins
// are randomly subsampled to `per_bin` points with `np.random.permutation`.  The ORDER of the output rows matters
// downstream (first-come voxelisation), so it is reproduced exactly:
//   vc_stvd_partition : bin of every point, order-preserving rank inside its bin (block ballots + a scan over the block
//                       histograms), the per-bin point lists and the bin sizes;
//   (host)            : reads the <= 16 bin sizes, runs the reference's `position` / `per_bin` arithmetic and draws the
//                       permutations from the SAME numpy generator the reference would use (virconv_b200/preprocess.py);
//   vc_stvd_gather    : emits the kept rows, segment by segment (a segment = one bin; identity or a host-provided list
//                       of in-bin ranks).
// HBM-bound integer / copy work: N*(4 + C*4) bytes read, M*C*4 written.
#include "common.cuh"

namespace vc {
namespace {

constexpr int SB = 1024;        // points per block
constexpr int MAXB = 16;        // bins

struct StvdWs {
    int8_t* bin;        // [n]
    int32_t* rank;      // [n]      rank inside (block, bin)
    int32_t* blk_cnt;   // [nblk][MAXB]
    int32_t* blk_off;   // [nblk][MAXB]  exclusive scan over blocks
    int32_t* base;      // [MAXB]   start of each bin's list in `order`
    int32_t* order;     // [n]      point ids, bin-major, original order inside a bin
    size_t bytes;
};

StvdWs layout(int n, void* ws) {
    StvdWs w;
    const int nblk = (n + SB - 1) / SB;
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    char* p = (char*)ws;
    size_t o = 0;
    w.bin = (int8_t*)(p + o);      o += al((size_t)n);
    w.rank = (int32_t*)(p + o);    o += al((size_t)n * 4);
    w.blk_cnt = (int32_t*)(p + o); o += al((size_t)nblk * MAXB * 4);
    w.blk_off = (int32_t*)(p + o); o += al((size_t)nblk * MAXB * 4);
    w.base = (int32_t*)(p + o);    o += al(MAXB * 4);
    w.order = (int32_t*)(p + o);   o += al((size_t)n * 4);
    w.bytes = o;
    return w;
}

__global__ void __launch_bounds__(SB) stvd_bin_kernel(const float* __restrict__ pts, int n, int c, int num, double inter,
                                                      int8_t* __restrict__ bin, int32_t* __restrict__ rank,
                                                      int32_t* __restrict__ blk_cnt) {
    __shared__ int warp_cnt[SB / 32][MAXB];
    const int i = blockIdx.x * SB + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int b = -1;
    if (i < n) {
        // `points[:, 0] >= inter * i` / `< inter * (i + 1)`: a float32 array against a python float — numpy (1.x value-based
        // casting and 2.x weak scalars alike) compares in float32 with the edge `inter * i` (a float64 product) rounded
        // to float32 once
        const float x = pts[(size_t)i * c];
        if (x >= (float)(inter * (double)(num - 1))) {
            b = num - 1;
        } else {
            for (int k = num - 2; k >= 0; --k)
                if (x >= (float)(inter * (double)k) && x < (float)(inter * (double)(k + 1))) { b = k; break; }
        }
    }
    int my_rank = 0;
    for (int k = 0; k < num; ++k) {
        const unsigned m = __ballot_sync(0xffffffffu, b == k);
        if (lane == 0) warp_cnt[warp][k] = __popc(m);
        if (b == k) my_rank = __popc(m & ((1u << lane) - 1u));
    }
    __syncthreads();
    if (b >= 0)
        for (int w = 0; w < warp; ++w) my_rank += warp_cnt[w][b];
    if (i < n) {
        bin[i] = (int8_t)b;
        rank[i] = my_rank;
    }
    if (threadIdx.x < MAXB) {
        int t = 0;
        if (threadIdx.x < num)
            for (int w = 0; w < SB / 32; ++w) t += warp_cnt[w][threadIdx.x];
        blk_cnt[blockIdx.x * MAXB + threadIdx.x] = t;
    }
}

// one thread per bin: exclusive scan of the block histograms; totals; bin-major bases
__global__ void stvd_scan_kernel(const int32_t* __restrict__ blk_cnt, int nblk, int num, int32_t* __restrict__ blk_off,
                                 int32_t* __restrict__ totals, int32_t* __restrict__ base) {
    __shared__ int tot[MAXB];
    const int k = threadIdx.x;
    int run = 0;
    if (k < num)
        for (int b = 0; b < nblk; ++b) {
            blk_off[b * MAXB + k] = run;
            run += blk_cnt[b * MAXB + k];
        }
    if (k < MAXB) {
        tot[k] = k < num ? run : 0;
        totals[k] = tot[k];
    }
    __syncthreads();
    if (k == 0) {
        int acc = 0;
        for (int j = 0; j < MAXB; ++j) {
            base[j] = acc;
            acc += tot[j];
        }
    }
}

__global__ void __launch_bounds__(SB) stvd_order_kernel(const int8_t* __restrict__ bin, const int32_t* __restrict__ rank,
                                                        const int32_t* __restrict__ blk_off,
                                                        const int32_t* __restrict__ base, int n,
                                                        int32_t* __restrict__ order) {
    const int i = blockIdx.x * SB + threadIdx.x;
    if (i >= n) return;
    const int b = bin[i];
    if (b < 0) return;
    order[base[b] + blk_off[blockIdx.x * MAXB + b] + rank[i]] = i;
}

struct Segs {
    int n_seg;
    int bin[MAXB], out_base[MAXB], count[MAXB], sel_base[MAXB];   // sel_base < 0: identity
};

// thread per (output row, 16-byte chunk... rows are c <= 16 floats): one thread copies one row
__global__ void __launch_bounds__(256) stvd_gather_kernel(const float* __restrict__ pts, int c, Segs s,
                                                          const int32_t* __restrict__ base,
                                                          const int32_t* __restrict__ order,
                                                          const int32_t* __restrict__ sel, float* __restrict__ out,
                                                          int n_out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_out) return;
    int g = 0;
    while (g + 1 < s.n_seg && j >= s.out_base[g + 1]) ++g;
    const int r = j - s.out_base[g];
    const int src_rank = s.sel_base[g] >= 0 ? sel[s.sel_base[g] + r] : r;
    const int pid = order[base[s.bin[g]] + src_rank];
    const float* src = pts + (size_t)pid * c;
    float* dst = out + (size_t)j * c;
    for (int q = 0; q < c; ++q) dst[q] = src[q];
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" size_t vc_stvd_ws_bytes(int n_points) { return layout(n_points > 0 ? n_points : 1, nullptr).bytes; }

extern "C" int vc_stvd_partition(const float* points, int n, int c, int bin_num, double max_dis, int32_t* totals_dev,
                                 void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n >= 0 && c >= 1 && bin_num >= 1 && bin_num <= MAXB && max_dis > 0 && totals_dev && ws,
                 "bad stvd arguments (n=%d c=%d bins=%d)", n, c, bin_num);
    StvdWs w = layout(n > 0 ? n : 1, ws);
    if (ws_bytes < w.bytes) {
        set_error("stvd workspace %zu < %zu", ws_bytes, w.bytes);
        return VC_ERR_WORKSPACE;
    }
    if (n == 0) {
        VC_CUDA(cudaMemsetAsync(totals_dev, 0, MAXB * 4, stream));
        return VC_OK;
    }
    VC_CHECK_ARG(points, "null points");
    const int nblk = (n + SB - 1) / SB;
    stvd_bin_kernel<<<nblk, SB, 0, stream>>>(points, n, c, bin_num, max_dis / (double)bin_num, w.bin, w.rank, w.blk_cnt);
    VC_LAUNCH_CHECK();
    stvd_scan_kernel<<<1, 32, 0, stream>>>(w.blk_cnt, nblk, bin_num, w.blk_off, totals_dev, w.base);
    VC_LAUNCH_CHECK();
    stvd_order_kernel<<<nblk, SB, 0, stream>>>(w.bin, w.rank, w.blk_off, w.base, n, w.order);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_stvd_gather(const float* points, int n, int c, const int32_t* segs /*host [n_seg][4]*/, int n_seg,
                              const int32_t* sel_dev, float* out, int n_out, void* ws, size_t ws_bytes,
                              vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n >= 0 && c >= 1 && n_seg >= 0 && n_seg <= MAXB && n_out >= 0 && ws, "bad stvd gather arguments");
    if (n_out == 0) return VC_OK;
    VC_CHECK_ARG(points && segs && out && n_seg > 0, "null pointer");
    StvdWs w = layout(n > 0 ? n : 1, ws);
    if (ws_bytes < w.bytes) {
        set_error("stvd workspace %zu < %zu", ws_bytes, w.bytes);
        return VC_ERR_WORKSPACE;
    }
    Segs s;
    memset(&s, 0, sizeof(s));
    s.n_seg = n_seg;
    int expect = 0;
    for (int g = 0; g < n_seg; ++g) {
        s.bin[g] = segs[4 * g + 0];
        s.out_base[g] = segs[4 * g + 1];
        s.count[g] = segs[4 * g + 2];
        s.sel_base[g] = segs[4 * g + 3];
        VC_CHECK_ARG(s.bin[g] >= 0 && s.bin[g] < MAXB && s.out_base[g] == expect && s.count[g] >= 0, "segment %d malformed", g);
        VC_CHECK_ARG(s.sel_base[g] < 0 || sel_dev, "segment %d needs a selection list", g);
        expect += s.count[g];
    }
    VC_CHECK_ARG(expect == n_out, "segments cover %d rows, n_out = %d", expect, n_out);
    stvd_gather_kernel<<<cdiv(n_out, 256), 256, 0, stream>>>(points, c, s, w.base, w.order, sel_dev, out, n_out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// ------------------------------------------------------------------------------------------------------------------------
// The device-drawn front end (vc_stvd_input_front_end): split, StVD input discard, assembly, shuffle and range mask of the
// collated cloud, with no host read — what the dataloader hands the model (dataset.py:270-298, then data_processor.py's
// mask_points_and_boxes_outside_range and shuffle_points), for a CUDA graph to capture.
//   classify : scene, kind (LiDAR / virtual) and x bin of every row; per-scene virtual counts and per-(scene, bin) counts;
//              the virtual rows' discard keys u = word 0 of Philox4x32-10, counter (row, 0, 1, draw) (philox.cuh);
//   plan     : one thread per scene: the reference's position / per_bin / out_n arithmetic in float64 -> the rows each
//              (scene, bin) segment keeps (all of them, or `take`); a scene without virtual points gets status bit 1 (the
//              reference's ZeroDivisionError);
//   select   : the `take` smallest (u, row) of every subsampled segment: a radix select over the 64-bit key
//              (u << 32 | row) as in vc_stvd_layer_keep, segmented: per-segment histograms of one 8-bit digit, and one
//              block per segment resolving that digit, eight times;
//   mark     : category of every kept row inside its scene (0 LiDAR, 1 + j the j-th bin emitted far -> near), the range
//              mask applied; per-block and per-(scene, category) counts;
//   scan     : block offsets per category; per stream and scene the output base and size; row counts, overflow;
//   emit     : every kept row to its place — [LiDAR, bins far -> near] per scene, row order inside a category — or, when
//              shuffling, to its image under a per-(stream, scene) Feistel permutation (four Philox rounds, counter domain 2,
//              cycle-walking onto [0, rows of the scene)).
// ------------------------------------------------------------------------------------------------------------------------
#include "philox.cuh"

namespace vc {
namespace {

constexpr int FE_ROWS = 1024;       // rows per block of the row kernels (one per thread)
constexpr int FE_CATS = 17;         // LiDAR + 16 bins
constexpr int FE_PASSES = 8;        // 8-bit digits of the 64-bit selection key
constexpr int FE_SEG = 16;          // segments per scene (bins)

struct FeWs {
    int8_t* cat;        // [cap]  classify: -3 neither, -2 virtual without bin, -1 LiDAR, k bin; mark: category or -1
    int32_t* scene;     // [cap]  scene of the row or -1
    uint32_t* u;        // [cap]  discard key of a binned virtual row
    int32_t* blk;       // [nblk][FE_CATS]  kept rows per block and category, then the exclusive scan over blocks
    int32_t* take;      // [B][FE_SEG]  rows a segment keeps, -1: all
    int32_t* rem;       // [B][FE_SEG]  rank of the threshold key still to resolve
    uint64_t* prefix;   // [B][FE_SEG]  resolved digits of the threshold key
    int32_t* first;     // [B][FE_CATS] position of a category's first row in its scene's block of the stream
    int32_t* excl;      // [B][FE_CATS] kept rows of the category in earlier scenes
    int32_t* sbase;     // [2][B] first output row of a scene's block, per stream
    int32_t* scnt;      // [2][B] rows of a scene's block, per stream
    // zeroed by one memset: ---
    int32_t* vcount;    // [B]
    int32_t* rlast;     // [B]  1 + the last row of the scene (0: no row)
    int32_t* rfirst;    // [B]  cap - the first row of the scene (0: no row)
    int32_t* disorder;  // [1]  1: the scenes are not contiguous and ascending
    int32_t* segcnt;    // [B][FE_SEG]
    int32_t* cnt;       // [B][FE_CATS] kept rows per scene and category
    uint32_t* hist;     // [FE_PASSES][B][FE_SEG][256]
    char* zero_begin;
    size_t zero_bytes;
    size_t bytes;
};

FeWs fe_layout(int cap, int B, void* ws) {
    FeWs w;
    const size_t n = cap > 0 ? (size_t)cap : 1, nblk = (n + FE_ROWS - 1) / FE_ROWS, S = (size_t)B * FE_SEG;
    auto al = [](size_t v) { return (v + 255) / 256 * 256; };
    char* p = (char*)ws;
    size_t o = 0;
    w.prefix = (uint64_t*)(p + o);  o += al(S * 8);
    w.cat = (int8_t*)(p + o);       o += al(n);
    w.scene = (int32_t*)(p + o);    o += al(n * 4);
    w.u = (uint32_t*)(p + o);       o += al(n * 4);
    w.blk = (int32_t*)(p + o);      o += al(nblk * FE_CATS * 4);
    w.take = (int32_t*)(p + o);     o += al(S * 4);
    w.rem = (int32_t*)(p + o);      o += al(S * 4);
    w.first = (int32_t*)(p + o);    o += al((size_t)B * FE_CATS * 4);
    w.excl = (int32_t*)(p + o);     o += al((size_t)B * FE_CATS * 4);
    w.sbase = (int32_t*)(p + o);    o += al((size_t)2 * B * 4);
    w.scnt = (int32_t*)(p + o);     o += al((size_t)2 * B * 4);
    const size_t z0 = o;
    w.vcount = (int32_t*)(p + o);   o += al((size_t)B * 4);
    w.rlast = (int32_t*)(p + o);    o += al((size_t)B * 4);
    w.rfirst = (int32_t*)(p + o);   o += al((size_t)B * 4);
    w.disorder = (int32_t*)(p + o); o += al(4);
    w.segcnt = (int32_t*)(p + o);   o += al(S * 4);
    w.cnt = (int32_t*)(p + o);      o += al((size_t)B * FE_CATS * 4);
    w.hist = (uint32_t*)(p + o);    o += al((size_t)FE_PASSES * S * 256 * 4);
    w.zero_begin = p + z0;
    w.zero_bytes = o - z0;
    w.bytes = o;
    return w;
}

__device__ __forceinline__ int fe_live_rows(const int32_t* n_dev, int cap) {
    if (!n_dev) return cap;
    const int n = *n_dev;
    return n < 0 ? 0 : (n > cap ? cap : n);
}

// counts[key] += 1 for every lane with key >= 0, one atomic per distinct key of the warp (every lane takes part)
__device__ __forceinline__ void warp_count(int32_t* counts, int key) {
    const unsigned m = __match_any_sync(0xffffffffu, key);
    if (key >= 0 && __ffs(m) - 1 == (int)(threadIdx.x & 31)) atomicAdd(counts + key, __popc(m));
}

__device__ __forceinline__ uint64_t fe_key(const uint32_t* u, int i) { return ((uint64_t)u[i] << 32) | (uint32_t)i; }

// the x bin of a virtual point, as stvd_bin_kernel (and the reference's float32 comparisons) decide it; -1: none
__device__ __forceinline__ int fe_bin(float x, int num, double inter) {
    if (x >= (float)(inter * (double)(num - 1))) return num - 1;
    for (int k = num - 2; k >= 0; --k)
        if (x >= (float)(inter * (double)k) && x < (float)(inter * (double)(k + 1))) return k;
    return -1;
}

__global__ void __launch_bounds__(FE_ROWS) fe_classify_kernel(const float* __restrict__ pts, int cap, const int32_t* __restrict__ n_dev,
                                                             int w, int B, int num, double inter, const int64_t* __restrict__ seed,
                                                             uint32_t draw, int8_t* __restrict__ cat, int32_t* __restrict__ scene,
                                                             uint32_t* __restrict__ u, int32_t* __restrict__ vcount,
                                                             int32_t* __restrict__ segcnt, int32_t* __restrict__ rlast,
                                                             int32_t* __restrict__ rfirst) {
    const int n = fe_live_rows(n_dev, cap);
    const int i = blockIdx.x * FE_ROWS + threadIdx.x;
    int c = -3, s = -1;
    if (i < n) {
        const float* p = pts + (size_t)i * w;
        const float bf = p[0], ind = p[w - 1];
        if (bf >= 0.f && bf < (float)B) s = (int)bf;
        if (s >= 0 && ind == 2.f) {
            c = -1;
        } else if (s >= 0 && ind == 1.f) {
            c = fe_bin(p[1], num, inter);
            if (c < 0) c = -2;
            else {
                const uint64_t sd = (uint64_t)*seed;
                u[i] = philox_word0((uint32_t)i, 0u, 1u, draw, (uint32_t)sd, (uint32_t)(sd >> 32));
            }
        } else {
            s = -1;
        }
    }
    if (i < cap) {
        cat[i] = (int8_t)c;
        scene[i] = s;
    }
    warp_count(vcount, (c == -2 || c >= 0) ? s : -1);
    warp_count(segcnt, c >= 0 ? s * FE_SEG + c : -1);
    // extent of every scene's rows (one atomic per scene and warp), for the contiguity check of the plan kernel
    const unsigned m = __match_any_sync(0xffffffffu, s);
    const int hi = __reduce_max_sync(m, i + 1), lo = __reduce_max_sync(m, cap - i);
    if (s >= 0 && __ffs(m) - 1 == (int)(threadIdx.x & 31)) {
        atomicMax(rlast + s, hi);
        atomicMax(rfirst + s, lo);
    }
}

// one thread per scene: dataset.py:120-189 as preprocess._discard_plan restates it
__global__ void fe_plan_kernel(int B, int num, double rate, const int32_t* __restrict__ vcount, const int32_t* __restrict__ segcnt,
                               int32_t* __restrict__ take, int32_t* __restrict__ rem, uint64_t* __restrict__ prefix,
                               int32_t* __restrict__ status, int cap, const int32_t* __restrict__ rlast,
                               const int32_t* __restrict__ rfirst, int32_t* __restrict__ disorder) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= B) return;
    // the output layout takes every row of a scene after every row of the scenes before it: a scene whose rows reach past
    // the first row of the next scene that has rows voids the whole batch (the mark kernel keeps nothing)
    if (rlast[s] > 0)
        for (int t = s + 1; t < B; ++t)
            if (rlast[t] > 0) {
                if (cap - rfirst[t] < rlast[s]) atomicExch(disorder, 1);
                break;
            }
    const long long n_all = vcount[s];
    const int32_t* cnt = segcnt + s * FE_SEG;
    const double retain = 1.0 - rate;
    long long per_bin = 0;
    int position = num - 1;
    if (n_all > 0) {
        long long acc = 0, distant = 0;
        for (int it = 0; it < num; ++it) {
            const int i = num - it - 1;
            acc += cnt[i];
            if ((double)(acc + (long long)i * cnt[i]) / (double)n_all < retain) {
                position = i;
                distant = acc;
            }
        }
        position = position < 0 ? 0 : position;
        const long long out_n = (long long)((double)n_all * retain);
        per_bin = (long long)((double)(out_n - distant) / ((double)position + 0.0001));
    }
    status[s] = n_all > 0 ? 0 : 1;
    for (int i = 0; i < FE_SEG; ++i) {
        int t = -1;
        const int it = num - 1 - i;
        if (n_all > 0 && i < num && it >= num - position && cnt[i] > per_bin) {     // `permutation(cnt)[:per_bin]`
            const long long k = per_bin >= 0 ? per_bin : (long long)cnt[i] + per_bin;
            t = k < 0 ? 0 : (int)k;
        }
        take[s * FE_SEG + i] = t;
        rem[s * FE_SEG + i] = t;
        prefix[s * FE_SEG + i] = 0;
    }
}

__global__ void __launch_bounds__(FE_ROWS) fe_hist_kernel(int cap, const int32_t* __restrict__ n_dev, const int8_t* __restrict__ cat,
                                                         const int32_t* __restrict__ scene, const uint32_t* __restrict__ u,
                                                         const int32_t* __restrict__ take, const uint64_t* __restrict__ prefix,
                                                         uint32_t* __restrict__ hist, int pass) {
    const int n = fe_live_rows(n_dev, cap);
    const int i = blockIdx.x * FE_ROWS + threadIdx.x;
    if (i >= n || cat[i] < 0) return;
    const int seg = scene[i] * FE_SEG + cat[i];
    if (take[seg] <= 0) return;
    const uint64_t key = fe_key(u, i);
    if (pass > 0 && (key >> (64 - 8 * pass)) != prefix[seg]) return;
    atomicAdd(&hist[seg * 256 + (int)((key >> (56 - 8 * pass)) & 255u)], 1u);
}

// one block (256 threads) per segment: the digit of this pass that holds the rem-th smallest key
__global__ void __launch_bounds__(256) fe_resolve_kernel(const uint32_t* __restrict__ hist, const int32_t* __restrict__ take,
                                                         int32_t* __restrict__ rem, uint64_t* __restrict__ prefix) {
    __shared__ unsigned s_scan[256];
    const int seg = blockIdx.x, t = threadIdx.x;
    if (take[seg] <= 0) return;
    const unsigned r = (unsigned)rem[seg];    // (read before the one writer below updates it)
    s_scan[t] = hist[seg * 256 + t];
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {
        const unsigned v = t >= off ? s_scan[t - off] : 0u;
        __syncthreads();
        s_scan[t] += v;
        __syncthreads();
    }
    const unsigned incl = s_scan[t], excl = t ? s_scan[t - 1] : 0u;
    if (excl < r && r <= incl) {          // exactly one digit
        prefix[seg] = (prefix[seg] << 8) | (uint64_t)t;
        rem[seg] = (int)(r - excl);
    }
}

// rank of the thread's category among the block's rows of that category, and (optionally) the block's count per category
__device__ __forceinline__ int fe_block_rank(int c, int32_t* blk_row) {
    __shared__ int wc[FE_ROWS / 32][FE_CATS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int r = 0;
#pragma unroll
    for (int k = 0; k < FE_CATS; ++k) {
        const unsigned m = __ballot_sync(0xffffffffu, c == k);
        if (lane == 0) wc[warp][k] = __popc(m);
        if (c == k) r = __popc(m & ((1u << lane) - 1u));
    }
    __syncthreads();
    if (c >= 0)
        for (int j = 0; j < warp; ++j) r += wc[j][c];
    if (blk_row && threadIdx.x < FE_CATS) {
        int t = 0;
        for (int j = 0; j < FE_ROWS / 32; ++j) t += wc[j][threadIdx.x];
        blk_row[threadIdx.x] = t;
    }
    return r;
}

__global__ void __launch_bounds__(FE_ROWS) fe_mark_kernel(const float* __restrict__ pts, int cap, const int32_t* __restrict__ n_dev,
                                                         int w, int num, float x0, float y0, float x1, float y1,
                                                         int8_t* __restrict__ cat, const int32_t* __restrict__ scene,
                                                         const uint32_t* __restrict__ u, const int32_t* __restrict__ take,
                                                         const uint64_t* __restrict__ prefix, int32_t* __restrict__ blk,
                                                         int32_t* __restrict__ cnt, const int32_t* __restrict__ disorder) {
    const int n = fe_live_rows(n_dev, cap);
    const int i = blockIdx.x * FE_ROWS + threadIdx.x;
    int c = -1, s = -1;
    if (i < n && !*disorder) {
        const int k = cat[i];
        s = scene[i];
        if (k == -1) {
            c = 0;
        } else if (k >= 0) {
            const int seg = s * FE_SEG + k, t = take[seg];
            if (t < 0 || (t > 0 && fe_key(u, i) <= prefix[seg])) c = 1 + (num - 1 - k);
        }
        if (c >= 0) {      // mask_points_by_range (common_utils.py:59-62): x and y, bounds inclusive, float32
            const float x = pts[(size_t)i * w + 1], y = pts[(size_t)i * w + 2];
            if (!(x >= x0 && x <= x1 && y >= y0 && y <= y1)) c = -1;
        }
    }
    if (i < cap) cat[i] = (int8_t)c;
    fe_block_rank(c, blk + (size_t)blockIdx.x * FE_CATS);
    warp_count(cnt, c >= 0 ? s * FE_CATS + c : -1);
}

__device__ __forceinline__ int fe_stream(int c, int two) { return two && c > 0 ? 1 : 0; }

// one block: exclusive scan of the block counts per category; per stream and scene the output layout; counts and overflow
__global__ void __launch_bounds__(1024) fe_scan_kernel(int nblk, int32_t* __restrict__ blk, int B, int two,
                                                       const int32_t* __restrict__ cnt, int32_t* __restrict__ first,
                                                       int32_t* __restrict__ excl, int32_t* __restrict__ sbase,
                                                       int32_t* __restrict__ scnt, int cap0, int cap1,
                                                       int32_t* __restrict__ n_out, int32_t* __restrict__ overflow,
                                                       const int32_t* __restrict__ disorder, int32_t* __restrict__ status) {
    __shared__ int s_w[32];
    __shared__ int s_carry;
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    for (int k = 0; k < FE_CATS; ++k) {
        if (threadIdx.x == 0) s_carry = 0;
        __syncthreads();
        for (int base = 0; base < nblk; base += 1024) {
            const int b = base + threadIdx.x;
            const int v = b < nblk ? blk[(size_t)b * FE_CATS + k] : 0;
            int x = v;
            for (int off = 1; off < 32; off <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, off);
                if (lane >= off) x += y;
            }
            if (lane == 31) s_w[wp] = x;
            __syncthreads();
            int woff = 0, tot = 0;
            for (int j = 0; j < 32; ++j) {
                woff += j < wp ? s_w[j] : 0;
                tot += s_w[j];
            }
            if (b < nblk) blk[(size_t)b * FE_CATS + k] = s_carry + woff + x - v;
            __syncthreads();
            if (threadIdx.x == 0) s_carry += tot;
            __syncthreads();
        }
    }
    if (threadIdx.x != 0) return;
    long long excess = 0;
    for (int st = 0; st < (two ? 2 : 1); ++st) {
        long long run = 0;
        for (int s = 0; s < B; ++s) {
            int pos = 0;
            for (int k = 0; k < FE_CATS; ++k) {
                if (fe_stream(k, two) != st) continue;
                first[s * FE_CATS + k] = pos;
                pos += cnt[s * FE_CATS + k];
            }
            sbase[st * B + s] = (int)run;
            scnt[st * B + s] = pos;
            run += pos;
        }
        const int cp = st ? cap1 : cap0;
        n_out[st] = run < cp ? (int)run : cp;
        excess += run > cp ? run - cp : 0;
    }
    if (!two) n_out[1] = 0;
    for (int k = 0; k < FE_CATS; ++k) {
        int run = 0;
        for (int s = 0; s < B; ++s) {
            excl[s * FE_CATS + k] = run;
            run += cnt[s * FE_CATS + k];
        }
    }
    if (excess > 0 && overflow) atomicMax(overflow, excess > 0x7fffffff ? 0x7fffffff : (int)excess);
    if (*disorder)
        for (int s = 0; s < B; ++s) status[s] |= 2;
}

// a bijection of [0, n): balanced Feistel network of four Philox rounds on 2h >= log2(n) bits, cycle-walking back into range
__device__ uint32_t fe_permute(uint32_t x, uint32_t n, uint32_t tweak, uint32_t draw, uint32_t k0, uint32_t k1) {
    if (n <= 1) return x;
    const int bits = 32 - __clz(n - 1), h = (bits + 1) / 2;
    const uint32_t mask = (1u << h) - 1u;
    do {
        uint32_t l = x >> h, r = x & mask;
        for (uint32_t rd = 0; rd < 4; ++rd) {
            const uint32_t f = philox_word0(r, tweak, 2u, (draw << 8) | rd, k0, k1) & mask;
            const uint32_t nl = r;
            r = l ^ f;
            l = nl;
        }
        x = (l << h) | r;
    } while (x >= n);
    return x;
}

__global__ void __launch_bounds__(FE_ROWS) fe_emit_kernel(const float* __restrict__ pts, int cap, int w, const int8_t* __restrict__ cat,
                                                         const int32_t* __restrict__ scene, const int32_t* __restrict__ blk,
                                                         const int32_t* __restrict__ first, const int32_t* __restrict__ excl,
                                                         const int32_t* __restrict__ sbase, const int32_t* __restrict__ scnt, int B,
                                                         int two, int fuse, int shuffle, const int64_t* __restrict__ seed,
                                                         uint32_t draw, float* __restrict__ out0, int32_t* __restrict__ src0, int cap0,
                                                         float* __restrict__ out1, int32_t* __restrict__ src1, int cap1) {
    const int i = blockIdx.x * FE_ROWS + threadIdx.x;
    const int c = i < cap ? (int)cat[i] : -1;       // (rows past the live count were marked -1)
    const int r = fe_block_rank(c, nullptr);
    if (c < 0) return;
    const int s = scene[i], st = fe_stream(c, two);
    int pos = first[s * FE_CATS + c] + blk[(size_t)blockIdx.x * FE_CATS + c] + r - excl[s * FE_CATS + c];
    if (pos < 0 || pos >= scnt[st * B + s]) return;     // (cannot happen once the plan kernel found the scenes in order)
    if (shuffle) {
        const uint64_t sd = (uint64_t)*seed;
        pos = (int)fe_permute((uint32_t)pos, (uint32_t)scnt[st * B + s], ((uint32_t)st << 16) | (uint32_t)s, draw, (uint32_t)sd,
                              (uint32_t)(sd >> 32));
    }
    const int j = sbase[st * B + s] + pos;
    float* out = st ? out1 : out0;
    int32_t* src = st ? src1 : src0;
    if (j >= (st ? cap1 : cap0)) return;
    const float* p = pts + (size_t)i * w;
    float* d = out + (size_t)j * w;
    for (int q = 0; q < w; ++q) d[q] = p[q];
    // points[:, 3] /= 10 of the fused cloud (dataset.py:294), column 4 of a collated row: IEEE division like numpy's
    if (fuse) d[4] = __fdiv_rn(p[4], 10.f);
    if (src) src[j] = i;
}

// rows [n_out[st], cap) of each stream: batch column -1 (no voxel), zeros, source -1
__global__ void __launch_bounds__(256) fe_tail_kernel(int w, const int32_t* __restrict__ n_out, float* __restrict__ out0,
                                                      int32_t* __restrict__ src0, int cap0, float* __restrict__ out1,
                                                      int32_t* __restrict__ src1, int cap1) {
    const size_t total = (size_t)cap0 + (size_t)cap1, stride = (size_t)gridDim.x * blockDim.x;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
        const int st = e >= (size_t)cap0;
        const int j = (int)(st ? e - cap0 : e);
        if (j < n_out[st]) continue;
        float* d = (st ? out1 : out0) + (size_t)j * w;
        d[0] = -1.f;
        for (int q = 1; q < w; ++q) d[q] = 0.f;
        int32_t* src = st ? src1 : src0;
        if (src) src[j] = -1;
    }
}

}  // namespace
}  // namespace vc

extern "C" size_t vc_stvd_input_ws_bytes(int cap, int batch_size) {
    return fe_layout(cap, batch_size > 0 ? batch_size : 1, nullptr).bytes;
}

extern "C" int vc_stvd_input_front_end(const float* points, int cap, const int32_t* n_dev, int w, int batch_size, int bin_num,
                                       double max_dis, double rate, const float* pc_range, int later_fusion, int shuffle,
                                       const int64_t* seed_dev, int draw, float* out_points, int32_t* src_points, int cap_points,
                                       float* out_mm, int32_t* src_mm, int cap_mm, int32_t* n_out_dev, int32_t* status_dev,
                                       int32_t* overflow_dev, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    VC_CHECK_ARG(cap >= 0 && cap < (1 << 30) && w >= 4 && w <= 64 && batch_size >= 1 && batch_size <= 65535 && bin_num >= 1 &&
                     bin_num <= FE_SEG && max_dis > 0 && pc_range && seed_dev && n_out_dev && status_dev && ws && draw >= 0 &&
                     draw < (1 << 24),
                 "vc_stvd_input_front_end: bad arguments (cap=%d w=%d B=%d bins=%d draw=%d)", cap, w, batch_size, bin_num, draw);
    VC_CHECK_ARG(rate >= 0.0 && rate <= 1.0, "vc_stvd_input_front_end: rate %g outside [0, 1]", rate);
    VC_CHECK_ARG(later_fusion || w >= 5, "vc_stvd_input_front_end: the fused cloud needs an intensity column (w=%d)", w);
    VC_CHECK_ARG(cap_points >= 0 && (cap_points == 0 || out_points) && (!later_fusion || (cap_mm >= 0 && (cap_mm == 0 || out_mm))),
                 "vc_stvd_input_front_end: output buffers");
    FeWs W = fe_layout(cap, batch_size, ws);
    if (ws_bytes < W.bytes) {
        set_error("vc_stvd_input_front_end: workspace %zu < %zu bytes", ws_bytes, W.bytes);
        return VC_ERR_WORKSPACE;
    }
    VC_CHECK_ARG(cap == 0 || points, "vc_stvd_input_front_end: null points");
    const int two = later_fusion ? 1 : 0;
    const int c1 = two ? cap_mm : 0;
    const int nblk = cap > 0 ? cdiv(cap, FE_ROWS) : 1, S = batch_size * FE_SEG;
    VC_CUDA(cudaMemsetAsync(W.zero_begin, 0, W.zero_bytes, st));
    fe_classify_kernel<<<nblk, FE_ROWS, 0, st>>>(points, cap, n_dev, w, batch_size, bin_num, max_dis / (double)bin_num, seed_dev,
                                                 (uint32_t)draw, W.cat, W.scene, W.u, W.vcount, W.segcnt, W.rlast, W.rfirst);
    VC_LAUNCH_CHECK();
    fe_plan_kernel<<<cdiv(batch_size, 128), 128, 0, st>>>(batch_size, bin_num, rate, W.vcount, W.segcnt, W.take, W.rem, W.prefix,
                                                          status_dev, cap, W.rlast, W.rfirst, W.disorder);
    VC_LAUNCH_CHECK();
    for (int p = 0; p < FE_PASSES; ++p) {
        uint32_t* h = W.hist + (size_t)p * S * 256;
        fe_hist_kernel<<<nblk, FE_ROWS, 0, st>>>(cap, n_dev, W.cat, W.scene, W.u, W.take, W.prefix, h, p);
        VC_LAUNCH_CHECK();
        fe_resolve_kernel<<<S, 256, 0, st>>>(h, W.take, W.rem, W.prefix);
        VC_LAUNCH_CHECK();
    }
    fe_mark_kernel<<<nblk, FE_ROWS, 0, st>>>(points, cap, n_dev, w, bin_num, pc_range[0], pc_range[1], pc_range[3], pc_range[4], W.cat,
                                             W.scene, W.u, W.take, W.prefix, W.blk, W.cnt, W.disorder);
    VC_LAUNCH_CHECK();
    fe_scan_kernel<<<1, 1024, 0, st>>>(nblk, W.blk, batch_size, two, W.cnt, W.first, W.excl, W.sbase, W.scnt, cap_points, c1,
                                       n_out_dev, overflow_dev, W.disorder, status_dev);
    VC_LAUNCH_CHECK();
    if (cap_points + c1 > 0) {
        fe_tail_kernel<<<cdiv(cap_points + c1, 256) < 132 * 8 ? cdiv(cap_points + c1, 256) : 132 * 8, 256, 0, st>>>(
            w, n_out_dev, out_points, src_points, cap_points, out_mm, src_mm, c1);
        VC_LAUNCH_CHECK();
    }
    if (cap > 0) {
        fe_emit_kernel<<<nblk, FE_ROWS, 0, st>>>(points, cap, w, W.cat, W.scene, W.blk, W.first, W.excl, W.sbase, W.scnt, batch_size,
                                                 two, two ? 0 : 1, shuffle ? 1 : 0, seed_dev, (uint32_t)draw, out_points, src_points,
                                                 cap_points, out_mm, src_mm, c1);
        VC_LAUNCH_CHECK();
    }
    return VC_OK;
}
