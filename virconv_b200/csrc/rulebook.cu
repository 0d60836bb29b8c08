// Rulebook (neighbour table) construction for submanifold and regular sparse convolution — sm_90a.
//
// Replaces spconv `ops.get_indice_pairs` behind spconv_backbone.py:89,92-93,113,563-564.
// Canonical form: oracle/rulebook.py (SURVEY §8a-R).
//
// Data layout in HBM
//   indices   [N, 1+ndim] int32 (b, z, y, x) | (b, u, v)
//   hash      2^h x uint64, entry = (linear_key << 24) | row, EMPTY = ~0   (ws of vc_subm_rulebook)
//   nbr       [K, N_out] int32 — row o of offset-plane k is written by thread o: fully coalesced
//   bitmap    1 bit per OUTPUT cell (batch-major linear index), + per-word exclusive popcount rank
//             (ws of a chain of strided convs, vc_conv_rulebook_*) — gives the sorted, duplicate-free output set with
//             no sort, and a cell's row in it by one bit test and one rank (the neighbour tables over a chain level's
//             output set: no hash table).
// Roofline: all kernels here are HBM/L2-latency bound integer work (no FLOPs); algorithmic bytes per
// input voxel are stated in DESIGN.md §kernels.
//
// Every strided conv is built as a chain (conv_chain_*): 1 <= L <= 4 regular convs where each one's input set is the
// previous one's output set (no layer discard between them); a single strided conv is a chain of one.  Their output sets
// are built from the FIRST input set in one pass instead of L dependent count -> scan -> emit rounds.  Composition rule:
// with dilation 1, input coordinate c reaches output coordinate o
// of a level exactly when o * stride lies in [c + pad - (ksize - 1), c + pad] and 0 <= o < oshape, and the grid test and
// the window factor per dimension (the batch index passes through).  So the level-1 cells reached from one input voxel are
// a product of per-dimension integer intervals; the cells reached from an interval [lo, hi] are again one interval
// (c + pad - off covers [lo + pad - ksize + 1, hi + pad] without a hole, so every multiple of the stride in it is hit), and
// the union over a product of intervals is the product of the per-dimension unions.  Level l's output set is therefore the
// union over input voxels of one product of intervals, computed level by level from the voxel's own coordinates: exactly
// the set the level-by-level definition (oracle/rulebook.py) builds from the previous level's output indices, in the same
// ascending cell order (so every index set, count and table is bit-identical); with L = 1 the rule IS that definition.  A
// dilation leaves holes in a level's window, so the rule needs dilation 1 at every level of a chain of two or more; a
// dilated strided conv is a chain of one, its level 0 marked cell by cell per kernel offset (out_cell).  One exception,
// only when a capacity is too small: the level-by-level definition derives level l + 1 from the first `cap` rows of an
// overflowing level l, the composed pass from all of its cells, so the counts of the levels AFTER the first overflowing one
// may be larger (the overflow is reported either way and such a step is recomputed with larger capacities).
#include "common.cuh"

namespace vc {

static constexpr unsigned long long HASH_EMPTY = ~0ULL;
static constexpr int ROW_BITS = 24;
static constexpr int MAXK = 32;  // >= 27 kernel offsets

__device__ __forceinline__ void decode_k(const Geom& g, int k, int* off) {
    for (int d = g.ndim - 1; d >= 0; --d) {
        off[d] = k % g.ksize[d];
        k /= g.ksize[d];
    }
}

// a row takes part in a rulebook only if its batch index and coordinates lie inside the grid (a padding row with b = -1 or
// a wrong `batch_size` must not write outside the bitmap / alias hash keys — ADVICE r1)
__device__ __forceinline__ bool index_ok(const Geom& g, int b, const int* c) {
    bool ok = b >= 0 && b < g.batch;
    for (int d = 0; d < g.ndim; ++d) ok &= (c[d] >= 0) & (c[d] < g.shape[d]);
    return ok;
}

__device__ __forceinline__ void load_index(const int32_t* __restrict__ idx, int row, int ndim, int& b, int* c) {
    if (ndim == 3) {
        int4 v = __ldg(reinterpret_cast<const int4*>(idx) + row);
        b = v.x; c[0] = v.y; c[1] = v.z; c[2] = v.w;
    } else {
        const int32_t* p = idx + (size_t)row * (1 + ndim);
        b = __ldg(p);
        for (int d = 0; d < ndim; ++d) c[d] = __ldg(p + 1 + d);
    }
}

// ------------------------------------------------------------------------------------------------
// hash table
// ------------------------------------------------------------------------------------------------
// (every kernel below that takes a row count `n` also takes `n_dev`: when non-NULL the count is read from device memory
// and `n` is the capacity the grid / buffers were sized for — the plan executor's static mode, CUDA-graph capturable)

// Submanifold rulebooks of up to IDX_BATCH_MAX stages in one launch per kernel (subm_rulebook_batch_dev; a single rulebook is
// a batch of one).  The grid's x blocks are the stages' row blocks one after the other (stage e owns blocks blk0[e] ..
// blk0[e + 1] - 1), so a block belongs to one stage.  Passed by value as a __grid_constant__ parameter: the kernels read the
// geometry in place, with no per-thread copy on the stack.
struct SubmEntry {
    const int32_t* idx;
    const int* n_dev;
    unsigned long long* table;
    int32_t *nbr, *pair_num;
    int32_t* rep;   // optional [n]: the lowest row at each row's coordinate (the row itself when it is outside the grid)
    Geom g;
    int n, ky;   // ky: offsets probed (centre + 1 with the mirrored probe, else K)
    uint32_t mask;
};
struct SubmBatch {
    int E, sym;
    int blk0[IDX_BATCH_MAX + 1];
    SubmEntry e[IDX_BATCH_MAX];
};

__device__ __forceinline__ int batch_entry(const int* blk0, int E, int bx) {
    int e = 0;
    while (e + 1 < E && bx >= blk0[e + 1]) ++e;
    return e;
}

__global__ void hash_insert_kernel(const __grid_constant__ SubmBatch sb) {
    const int i = batch_entry(sb.blk0, sb.E, blockIdx.x);
    const SubmEntry& e = sb.e[i];
    const Geom& g = e.g;
    const int n = e.n_dev != nullptr ? min(e.n, __ldg(e.n_dev)) : e.n;
    const int row = (blockIdx.x - sb.blk0[i]) * blockDim.x + threadIdx.x;
    if (row >= n) return;
    int b, c[VC_MAX_NDIM];
    load_index(e.idx, row, g.ndim, b, c);
    if (!index_ok(g, b, c)) return;
    unsigned long long key = (unsigned long long)b;
    for (int d = 0; d < g.ndim; ++d) key = key * (unsigned long long)g.shape[d] + (unsigned long long)c[d];
    unsigned long long packed = (key << ROW_BITS) | (unsigned long long)row;
    uint32_t slot = mix64(key) & e.mask;
    while (true) {
        unsigned long long cur = e.table[slot];
        if (cur == HASH_EMPTY) {
            cur = atomicCAS(&e.table[slot], HASH_EMPTY, packed);
            if (cur == HASH_EMPTY) return;
        }
        if ((cur >> ROW_BITS) == key) {  // duplicate coordinate: lowest row index wins
            atomicMin(&e.table[slot], packed);
            return;
        }
        slot = (slot + 1) & e.mask;
    }
}

__device__ __forceinline__ int hash_lookup(const unsigned long long* __restrict__ table, uint32_t mask,
                                           unsigned long long key) {
    uint32_t slot = mix64(key) & mask;
    while (true) {
        unsigned long long cur = __ldg(table + slot);
        if (cur == HASH_EMPTY) return -1;
        if ((cur >> ROW_BITS) == key) return (int)(cur & ((1ULL << ROW_BITS) - 1));
        slot = (slot + 1) & mask;
    }
}

// One thread per (output row, kernel offset): grid (row blocks, max ky).  Every probe chain is independent, so the
// hash look-ups of all K offsets are in flight together (the per-row loop this replaced was latency bound);
// nbr[k, row] writes stay fully coalesced.  Pair counts: warp ballot -> shared counter -> one atomic per block.
// sym (every coordinate held by one row, odd kernel sizes): the table is its own transpose — nbr[k, i] = j exactly when
// nbr[K-1-k, j] = i, the relation the mirrored dgrad already relies on — so the grid covers the offsets k <= centre only
// and each neighbour found also writes its mirrored entry (the caller fills the rows k > centre with -1 first): half the
// hash look-ups, the same table.
__global__ void __launch_bounds__(256) subm_probe_kernel(const __grid_constant__ SubmBatch sb) {
    const int i = batch_entry(sb.blk0, sb.E, blockIdx.x);
    const SubmEntry& e = sb.e[i];
    const Geom& g = e.g;
    const int k = blockIdx.y, sym = sb.sym;
    if (k >= e.ky) return;
    __shared__ int cnt;
    const int pitch = e.n;                // table rows are [K][capacity]
    const int n = e.n_dev != nullptr ? min(e.n, __ldg(e.n_dev)) : e.n;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const int row = (blockIdx.x - sb.blk0[i]) * blockDim.x + threadIdx.x;
    int res = -1;
    if (row < n) {
        int centre = 0;
        for (int d = 0; d < g.ndim; ++d) centre = centre * g.ksize[d] + g.ksize[d] / 2;
        if (k == centre) {
            res = row;  // identity (spconv Native: out = features @ W[centre])
            if (e.rep != nullptr) {   // the lowest row at this row's own coordinate (the row itself when it is outside the grid)
                int b, c[VC_MAX_NDIM];
                load_index(e.idx, row, g.ndim, b, c);
                int r = row;
                if (index_ok(g, b, c)) {
                    unsigned long long key = (unsigned long long)b;
                    for (int d = 0; d < g.ndim; ++d) key = key * (unsigned long long)g.shape[d] + (unsigned long long)c[d];
                    r = hash_lookup(e.table, e.mask, key);
                }
                e.rep[row] = r;
            }
        } else {
            int b, c[VC_MAX_NDIM];
            load_index(e.idx, row, g.ndim, b, c);
            int off[VC_MAX_NDIM];
            decode_k(g, k, off);
            bool ok = index_ok(g, b, c);
            unsigned long long key = (unsigned long long)b;
            for (int d = 0; d < g.ndim; ++d) {
                int v = c[d] + (off[d] - g.ksize[d] / 2) * g.dil[d];
                ok &= (v >= 0) & (v < g.shape[d]);
                key = key * (unsigned long long)g.shape[d] + (unsigned long long)v;
            }
            if (ok) res = hash_lookup(e.table, e.mask, key);
            if (sym && res >= 0) e.nbr[(size_t)(g.K - 1 - k) * pitch + res] = row;
        }
        e.nbr[(size_t)k * pitch + row] = res;
    } else if (row < pitch) {
        e.nbr[(size_t)k * pitch + row] = -1;    // static mode: rows between the count and the capacity have no neighbours
        if (e.rep != nullptr && k == 0) e.rep[row] = -1;
    }
    unsigned m = __ballot_sync(0xffffffffu, res >= 0);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt, __popc(m));
    __syncthreads();
    if (e.pair_num != nullptr && threadIdx.x == 0 && cnt) {
        atomicAdd(&e.pair_num[k], cnt);
        if (sym && k != g.K - 1 - k) atomicAdd(&e.pair_num[g.K - 1 - k], cnt);
    }
}

// ------------------------------------------------------------------------------------------------
// regular conv: bitmap over output cells
// ------------------------------------------------------------------------------------------------
static constexpr int SCAN_WORDS = 2048;  // words per scan block (256 threads x 8)

// returns output linear cell (batch major) for (input coords c, offset k), or -1
__device__ __forceinline__ long long out_cell(const Geom& g, int b, const int* c, int k) {
    if (!index_ok(g, b, c)) return -1;
    int off[VC_MAX_NDIM];
    decode_k(g, k, off);
    long long lin = b;
    for (int d = 0; d < g.ndim; ++d) {
        int num = c[d] + g.pad[d] - off[d] * g.dil[d];
        if (num < 0) return -1;
        int o = num / g.stride[d];
        if (o * g.stride[d] != num || o >= g.oshape[d]) return -1;
        lin = lin * g.oshape[d] + o;
    }
    return lin;
}

__device__ __forceinline__ void mark_cell(uint32_t* bitmap, long long lin) {
    const uint32_t bit = 1u << (lin & 31);
    uint32_t* w = bitmap + (lin >> 5);
    if (!(*w & bit)) atomicOr(w, bit);
}

// local exclusive scan of popcounts inside blocks of SCAN_WORDS words; block totals to block_sum
__global__ void __launch_bounds__(256) scan_local_kernel(const uint32_t* __restrict__ bitmap, long long n_words,
                                                         uint32_t* __restrict__ word_rank,
                                                         uint32_t* __restrict__ block_sum) {
    __shared__ uint32_t warp_tot[8];
    long long base = (long long)blockIdx.x * SCAN_WORDS + threadIdx.x * 8;
    uint32_t cnt[8];
    uint32_t tsum = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        long long w = base + i;
        cnt[i] = (w < n_words) ? __popc(bitmap[w]) : 0;
        tsum += cnt[i];
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
    for (int i = 0; i < 8; ++i) {
        long long w = base + i;
        if (w < n_words) word_rank[w] = run;
        run += cnt[i];
    }
    if (threadIdx.x == 255) block_sum[blockIdx.x] = woff + incl;
}

// single block: exclusive scan of block sums in place; total -> n_out
// (cap > 0: the output buffers hold `cap` rows; a larger total is clamped and reported through *overflow)
__device__ __forceinline__ void scan_segment(uint32_t* block_sum, int n_blocks, int32_t* n_out, int cap, int* overflow) {
    __shared__ uint32_t warp_tot[32];
    __shared__ uint32_t carry_s;
    __syncthreads();   // (a previous segment's thread 0 has read carry_s)
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < n_blocks; base += 1024) {
        int i = base + threadIdx.x;
        uint32_t v = (i < n_blocks) ? block_sum[i] : 0;
        uint32_t incl = v;
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
        int total = (int)carry_s;
        if (cap > 0 && total > cap) {
            if (overflow != nullptr) atomicMax(overflow, total);
            total = cap;
        }
        *n_out = total;
    }
}

// Rows of the cells along one x run of a ranked set of which the first n rows are held: a cell's row is its rank, or -1
// when the cell is not in the set or ranks past the held rows (static mode: an overflowing level holds its first `cap`
// cells only).  Successive cells of a run mostly share a bitmap word: the word and its rank are loaded together, once per
// word.
struct RunRows {
    const ConvRank& r;
    int n;
    long long wc = -1;
    uint32_t word = 0, base = 0;
    __device__ __forceinline__ RunRows(const ConvRank& r_, int n_) : r(r_), n(n_) {}
    __device__ __forceinline__ int row(long long lin) {
        const long long w = lin >> 5;
        if (w != wc) {
            wc = w;
            word = __ldg(r.bitmap + w);
            base = __ldg(r.block_sum + (w / SCAN_WORDS)) + __ldg(r.word_rank + w);
        }
        const uint32_t bit = 1u << (lin & 31);
        if (!(word & bit)) return -1;
        const int row = (int)(base + __popc(word & (bit - 1u)));
        return row < n ? row : -1;
    }
};

// pair counts: per offset k, warp ballot -> shared counter cnt[k] -> (caller) one atomic per block
__device__ __forceinline__ void count_pairs(int* cnt, int k, bool hit) {
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt[k], __popc(m));
}

// chained strided convs (file header): per level the geometry, where its bitmap / ranks start in the concatenated
// workspace (w0 words, b0 scan blocks: every level starts on a SCAN_WORDS boundary, so a scan block never spans two
// levels), and for the emit its output buffer and capacity.  Passed by value.
struct ChainDesc {
    int L;
    int dilated;   // level 0 has a dilation (then L = 1)
    Geom g[CONV_CHAIN_MAX];
    long long w0[CONV_CHAIN_MAX + 1];
    int b0[CONV_CHAIN_MAX + 1];
    int32_t* out_idx[CONV_CHAIN_MAX];
    int cap[CONV_CHAIN_MAX];
};

// grid (rows, L): the cells of level blockIdx.y reached from one input row, the product of its per-dimension intervals.
// A dilated level 0: grid (rows, K), the cell of kernel offset blockIdx.y.
__global__ void conv_mark_kernel(const int32_t* __restrict__ idx, int n, const int* __restrict__ n_dev, ChainDesc cd,
                                  uint32_t* bitmap) {
    if (n_dev != nullptr) n = min(n, __ldg(n_dev));
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const int level = blockIdx.y;
    int b, lo[VC_MAX_NDIM], hi[VC_MAX_NDIM];
    load_index(idx, row, cd.g[0].ndim, b, lo);
    if (cd.dilated) {
        const long long lin = out_cell(cd.g[0], b, lo, blockIdx.y);
        if (lin >= 0) mark_cell(bitmap, lin);
        return;
    }
    if (!index_ok(cd.g[0], b, lo)) return;
    for (int d = 0; d < cd.g[0].ndim; ++d) hi[d] = lo[d];
    for (int l = 0; l <= level; ++l) {
        const Geom& g = cd.g[l];
        for (int d = 0; d < g.ndim; ++d) {
            const int first = lo[d] + g.pad[d] - (g.ksize[d] - 1), last = hi[d] + g.pad[d];   // o * stride in [first, last]
            const int olo = first <= 0 ? 0 : (first + g.stride[d] - 1) / g.stride[d];
            const int ohi = last < 0 ? -1 : min(last / g.stride[d], g.oshape[d] - 1);
            if (olo > ohi) return;   // no cell at this level, hence none further down
            lo[d] = olo;
            hi[d] = ohi;
        }
    }
    const Geom& g = cd.g[level];
    uint32_t* bm = bitmap + cd.w0[level];
    int c[VC_MAX_NDIM];
    for (int d = 0; d < g.ndim; ++d) c[d] = lo[d];
    while (true) {
        long long lin = b;
        for (int d = 0; d < g.ndim; ++d) lin = lin * g.oshape[d] + c[d];
        mark_cell(bm, lin);
        int d = g.ndim - 1;   // next cell of the product, last dimension fastest
        while (d >= 0 && c[d] == hi[d]) { c[d] = lo[d]; --d; }
        if (d < 0) break;
        ++c[d];
    }
}

// one block: the scan of each level's block sums as its own segment, each level's count clamped to its capacity
__global__ void __launch_bounds__(1024) scan_blocks_kernel(uint32_t* block_sum, ChainDesc cd, int32_t* n_out,
                                                                 int* overflow) {
    for (int l = 0; l < cd.L; ++l)
        scan_segment(block_sum + cd.b0[l], cd.b0[l + 1] - cd.b0[l], n_out + l, cd.cap[l], overflow);
}

// one thread per word of all levels: the output indices of the word's set bits, in rank order
__global__ void conv_emit_indices_kernel(const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ word_rank,
                                  const uint32_t* __restrict__ block_sum, ChainDesc cd) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= cd.w0[cd.L]) return;
    uint32_t word = bitmap[w];
    if (!word) return;
    int l = 0;
    while (w >= cd.w0[l + 1]) ++l;
    const Geom& g = cd.g[l];
    const long long wl = w - cd.w0[l];
    int row = (int)(block_sum[cd.b0[l] + wl / SCAN_WORDS] + word_rank[w]);
    const int cap = cd.cap[l];
    while (word) {
        int bit = __ffs(word) - 1;
        word &= word - 1;
        if (row >= cap) return;           // capacity overflow (flagged by scan_blocks_kernel)
        long long lin = (wl << 5) + bit;
        int c[VC_MAX_NDIM];
        for (int d = g.ndim - 1; d >= 0; --d) {
            c[d] = (int)(lin % g.oshape[d]);
            lin /= g.oshape[d];
        }
        int32_t* o = cd.out_idx[l] + (size_t)row * (1 + g.ndim);
        o[0] = (int32_t)lin;
        for (int d = 0; d < g.ndim; ++d) o[1 + d] = c[d];
        ++row;
    }
}

// The neighbour tables of up to IDX_BATCH_MAX strided convs in one launch (conv_tables_batch_dev; a single conv is a batch
// of one), laid out as the submanifold batch above.
struct TablesEntry {
    const int32_t* idx;
    const int* n_dev;
    ConvRank r;
    int32_t *nbr_fwd, *nbr_bwd, *pair_num;
    Geom g;
    int n, n_out;
};
struct TablesBatch {
    int E;
    int blk0[IDX_BATCH_MAX + 1];
    TablesEntry e[IDX_BATCH_MAX];
};

// One thread per input row, as the lookup kernels below: the output cells of the offsets along x lie on one x run of the
// output bitmap (RunRows).
__global__ void __launch_bounds__(256) conv_tables_kernel(const __grid_constant__ TablesBatch tb) {   // one thread per row
    const int i = batch_entry(tb.blk0, tb.E, blockIdx.x);
    const TablesEntry& e = tb.e[i];
    const Geom& g = e.g;
    const int xd = g.ndim - 1, kx = g.ksize[xd];
    __shared__ int cnt[MAXK];
    if (threadIdx.x < g.K) cnt[threadIdx.x] = 0;
    __syncthreads();
    const int pitch_in = e.n;             // nbr_bwd rows are [K][input capacity], nbr_fwd rows [K][n_out = output capacity]
    const int n = e.n_dev != nullptr ? min(e.n, __ldg(e.n_dev)) : e.n;
    const int row = (blockIdx.x - tb.blk0[i]) * blockDim.x + threadIdx.x;
    int b = 0, c[VC_MAX_NDIM] = {}, off[VC_MAX_NDIM];
    bool in = false;
    if (row < n) {
        load_index(e.idx, row, g.ndim, b, c);
        in = index_ok(g, b, c);
    }
    for (int k0 = 0; k0 < g.K; k0 += kx) {   // the offset groups
        bool ok = in;
        long long lin = b;
        decode_k(g, k0, off);
        for (int d = 0; d < xd; ++d) {
            const int num = c[d] + g.pad[d] - off[d] * g.dil[d], o = num / g.stride[d];
            ok &= (num >= 0) & (o * g.stride[d] == num) & (o < g.oshape[d]);
            lin = lin * g.oshape[d] + o;
        }
        lin *= g.oshape[xd];
        RunRows rr(e.r, e.n_out);   // (a rank at or past the output capacity: overflow, flagged by the count)
        for (int j = 0; j < kx; ++j) {
            const int num = c[xd] + g.pad[xd] - j * g.dil[xd], o = num / g.stride[xd];
            int orow = -1;
            if (row < n) {
                if (ok && num >= 0 && o * g.stride[xd] == num && o < g.oshape[xd]) {
                    orow = rr.row(lin + o);
                    if (orow >= 0 && e.nbr_fwd != nullptr)   // (else conv_fwd_lookup_kernel writes it)
                        e.nbr_fwd[(size_t)(k0 + j) * e.n_out + orow] = row;   // unique writer: (o,k) determines the input cell
                }
                e.nbr_bwd[(size_t)(k0 + j) * pitch_in + row] = orow;
            } else if (row < pitch_in) {
                e.nbr_bwd[(size_t)(k0 + j) * pitch_in + row] = -1;   // static mode: rows between the count and the capacity
            }
            count_pairs(cnt, k0 + j, orow >= 0);
        }
    }
    __syncthreads();
    if (e.pair_num != nullptr && threadIdx.x < g.K && cnt[threadIdx.x]) atomicAdd(&e.pair_num[threadIdx.x], cnt[threadIdx.x]);
}

// Lookups in a chain level's ranked output bitmap.  A chain level's rows are the set bits of its bitmap in rank order
// (conv_emit_indices_kernel), so the row of a cell of that set is one bit test and one rank: no hash table, and each
// table entry is written by the thread of its row, coalesced.  One thread per row, which loads the row's index once and
// walks its offset groups: a group is the offsets that differ along x only (the last dimension, fastest in both the
// offset and the cell order), whose cells lie along one x run of the bitmap (RunRows).  A neighbour cell is rejected per
// dimension against the grid, never by linear-index arithmetic (x = W is the next row's x = 0, and the last cell of one
// scene is the first of the next).

// nbr_fwd of the chained strided convs whose input set is the previous level's output set (conv_fwd_lookup_batch_dev):
// output row o and offset k look up the input cell o * stride - pad + k * dil in the input level's bitmap.  The pair
// counts come from conv_tables_kernel's nbr_bwd.
struct FwdLookupEntry {
    const int32_t* out_idx;
    const int *n_out_dev, *n_in_dev;
    ConvRank in_rank;
    int32_t* nbr_fwd;
    Geom g;
    int n_out, n_in;
};
struct FwdLookupBatch {
    int E;
    int blk0[IDX_BATCH_MAX + 1];
    FwdLookupEntry e[IDX_BATCH_MAX];
};

__global__ void __launch_bounds__(256) conv_fwd_lookup_kernel(const __grid_constant__ FwdLookupBatch fb) {   // one thread per row
    const int i = batch_entry(fb.blk0, fb.E, blockIdx.x);
    const FwdLookupEntry& e = fb.e[i];
    const Geom& g = e.g;
    const int xd = g.ndim - 1, kx = g.ksize[xd];
    const int n = e.n_out_dev != nullptr ? min(e.n_out, __ldg(e.n_out_dev)) : e.n_out;
    const int n_in = e.n_in_dev != nullptr ? min(e.n_in, __ldg(e.n_in_dev)) : e.n_in;
    const int row = (blockIdx.x - fb.blk0[i]) * blockDim.x + threadIdx.x;
    if (row >= e.n_out) return;
    int b = 0, c[VC_MAX_NDIM] = {}, off[VC_MAX_NDIM];
    bool in = row < n;   // (static mode: rows between the count and the capacity have no neighbours)
    if (in) {
        load_index(e.out_idx, row, g.ndim, b, c);
        in = b >= 0 && b < g.batch;
    }
    const int x0 = c[xd] * g.stride[xd] - g.pad[xd];
    for (int k0 = 0; k0 < g.K; k0 += kx) {   // the offset groups
        bool ok = in;
        long long lin = b;
        decode_k(g, k0, off);
        for (int d = 0; d < xd; ++d) {
            const int v = c[d] * g.stride[d] - g.pad[d] + off[d] * g.dil[d];
            ok &= (v >= 0) & (v < g.shape[d]);
            lin = lin * g.shape[d] + v;
        }
        lin *= g.shape[xd];
        RunRows rr(e.in_rank, n_in);
        for (int j = 0; j < kx; ++j) {
            const int x = x0 + j * g.dil[xd];
            e.nbr_fwd[(size_t)(k0 + j) * e.n_out + row] = ok && x >= 0 && x < g.shape[xd] ? rr.row(lin + x) : -1;
        }
    }
}

// Submanifold rulebooks over chain levels' output sets (subm_lookup_batch_dev), laid out as SubmBatch, every offset
// looked up; the centre identity and the static-mode -1 tail as in subm_probe_kernel.
struct LookupEntry {
    const int32_t* idx;
    const int* n_dev;
    ConvRank rank;
    int32_t *nbr, *pair_num;
    Geom g;
    int n;
};
struct LookupBatch {
    int E;
    int blk0[IDX_BATCH_MAX + 1];
    LookupEntry e[IDX_BATCH_MAX];
};

__global__ void __launch_bounds__(256) subm_lookup_kernel(const __grid_constant__ LookupBatch lb) {   // one thread per row
    const int i = batch_entry(lb.blk0, lb.E, blockIdx.x);
    const LookupEntry& e = lb.e[i];
    const Geom& g = e.g;
    const int xd = g.ndim - 1, kx = g.ksize[xd];
    __shared__ int cnt[MAXK];
    if (threadIdx.x < g.K) cnt[threadIdx.x] = 0;
    __syncthreads();
    const int pitch = e.n;                // table rows are [K][capacity]
    const int n = e.n_dev != nullptr ? min(e.n, __ldg(e.n_dev)) : e.n;
    const int row = (blockIdx.x - lb.blk0[i]) * blockDim.x + threadIdx.x;
    int b = 0, c[VC_MAX_NDIM] = {}, off[VC_MAX_NDIM], centre = 0;
    for (int d = 0; d < g.ndim; ++d) centre = centre * g.ksize[d] + g.ksize[d] / 2;
    bool in = false;
    if (row < n) {
        load_index(e.idx, row, g.ndim, b, c);
        in = index_ok(g, b, c);
    }
    const int x0 = c[xd] - kx / 2 * g.dil[xd];
    for (int k0 = 0; k0 < g.K; k0 += kx) {   // the offset groups
        bool ok = in;
        long long lin = b;
        decode_k(g, k0, off);
        for (int d = 0; d < xd; ++d) {
            const int v = c[d] + (off[d] - g.ksize[d] / 2) * g.dil[d];
            ok &= (v >= 0) & (v < g.shape[d]);
            lin = lin * g.shape[d] + v;
        }
        lin *= g.shape[xd];
        RunRows rr(e.rank, n);
        for (int j = 0; j < kx; ++j) {
            const int x = x0 + j * g.dil[xd];
            int res = -1;
            if (row < n) {
                if (k0 + j == centre) res = row;   // identity (spconv Native: out = features @ W[centre])
                else if (ok && x >= 0 && x < g.shape[xd]) res = rr.row(lin + x);
                e.nbr[(size_t)(k0 + j) * pitch + row] = res;
            } else if (row < pitch) {
                e.nbr[(size_t)(k0 + j) * pitch + row] = -1;    // static mode: rows between the count and the capacity have no neighbours
            }
            count_pairs(cnt, k0 + j, res >= 0);
        }
    }
    __syncthreads();
    if (e.pair_num != nullptr && threadIdx.x < g.K && cnt[threadIdx.x]) atomicAdd(&e.pair_num[threadIdx.x], cnt[threadIdx.x]);
}

// one block per offset: order-preserving compaction of nbr[k, :] into spconv-style pairs
__global__ void __launch_bounds__(1024) pairs_kernel(const int32_t* __restrict__ nbr, int K, int n,
                                                     int32_t* __restrict__ pairs, int32_t* __restrict__ pair_num) {
    __shared__ int warp_tot[32];
    __shared__ int carry_s;
    int k = blockIdx.x;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int32_t* src = nbr + (size_t)k * n;
    int32_t* pin = pairs + (size_t)k * n;
    int32_t* pout = pairs + (size_t)(K + k) * n;
    for (int base = 0; base < n; base += 1024) {
        int i = base + threadIdx.x;
        int v = (i < n) ? src[i] : -1;
        int f = v >= 0;
        unsigned m = __ballot_sync(0xffffffffu, f);
        int lane = threadIdx.x & 31;
        int wpre = __popc(m & ((1u << lane) - 1u));
        if (lane == 0) warp_tot[threadIdx.x >> 5] = __popc(m);
        __syncthreads();
        int woff = 0;
        for (int w = 0; w < (threadIdx.x >> 5); ++w) woff += warp_tot[w];
        int carry = carry_s;
        if (f) {
            pin[carry + woff + wpre] = v;
            pout[carry + woff + wpre] = i;
        }
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = carry + woff + wpre + f;
        __syncthreads();
    }
    int total = carry_s;
    for (int i = total + threadIdx.x; i < n; i += 1024) {
        pin[i] = -1;
        pout[i] = -1;
    }
    if (threadIdx.x == 0) pair_num[k] = total;
}

static int make_geom(Geom& g, int ndim, int batch_size, const int32_t* shape, const int32_t* ksize, const int32_t* stride,
                     const int32_t* pad, const int32_t* dil) {
    VC_CHECK_ARG(ndim >= 1 && ndim <= VC_MAX_NDIM, "ndim %d not in [1,%d]", ndim, VC_MAX_NDIM);
    VC_CHECK_ARG(batch_size > 0, "batch size %d", batch_size);
    memset(&g, 0, sizeof(g));
    g.ndim = ndim;
    g.batch = batch_size;
    g.K = 1;
    for (int d = 0; d < ndim; ++d) {
        g.shape[d] = shape[d];
        g.ksize[d] = ksize[d];
        g.stride[d] = stride ? stride[d] : 1;
        g.pad[d] = pad ? pad[d] : 0;
        g.dil[d] = dil ? dil[d] : 1;
        VC_CHECK_ARG(g.shape[d] > 0 && g.ksize[d] > 0 && g.stride[d] > 0 && g.dil[d] > 0 && g.pad[d] >= 0,
                     "bad geometry in dim %d", d);
        g.oshape[d] = (g.shape[d] + 2 * g.pad[d] - g.dil[d] * (g.ksize[d] - 1) - 1) / g.stride[d] + 1;
        VC_CHECK_ARG(g.oshape[d] > 0, "empty output shape in dim %d", d);
        g.K *= g.ksize[d];
    }
    VC_CHECK_ARG(g.K <= MAXK, "kernel volume %d > %d", g.K, MAXK);
    return VC_OK;
}

static uint32_t table_slots(int n) {
    uint32_t s = 1024;
    while (s < 2u * (uint32_t)(n > 0 ? n : 1)) s <<= 1;
    return s;
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_subm_rulebook_ws_bytes(int n) { return (size_t)table_slots(n) * sizeof(unsigned long long); }

// one submanifold stage's arguments -> its geometry and hash-table slots (0: no row, nothing to launch)
static int subm_stage_geom(const SubmStage& s, int batch_size, Geom& g, uint32_t& slots) {
    int rc = make_geom(g, s.ndim, batch_size, s.shape, s.ksize, nullptr, nullptr, s.dil);
    if (rc) return rc;
    VC_CHECK_ARG(s.n >= 0 && s.n < (1 << ROW_BITS), "row count %d out of range", s.n);
    double cells = (double)batch_size;
    for (int d = 0; d < s.ndim; ++d) cells *= g.shape[d];
    VC_CHECK_ARG(cells < 1099511627776.0, "grid too large for 40-bit keys");
    slots = 0;
    if (s.n == 0) return VC_OK;
    VC_CHECK_ARG(s.idx && s.nbr && s.table, "null pointer");
    slots = table_slots(s.n);
    if (s.table_bytes < (size_t)slots * 8) {
        set_error("subm rulebook workspace %zu < %zu", s.table_bytes, (size_t)slots * 8);
        return VC_ERR_WORKSPACE;
    }
    return VC_OK;
}

// one rulebook: its own clears, then a batch of one
int vc::subm_rulebook_dev(const int32_t* indices, int n, const int* n_dev, int ndim, int batch_size,
                          const int32_t* spatial_shape, const int32_t* ksize, const int32_t* dilation, int32_t* nbr,
                          int32_t* pair_num, void* ws, size_t ws_bytes, cudaStream_t stream, int32_t* rep, bool unique) {
    const SubmStage s{indices, n, n_dev, ndim, spatial_shape, ksize, dilation, nbr, pair_num, ws, ws_bytes, rep};
    Geom g;
    uint32_t slots;
    int rc = subm_stage_geom(s, batch_size, g, slots);
    if (rc) return rc;
    if (pair_num) VC_CUDA(cudaMemsetAsync(pair_num, 0, sizeof(int32_t) * g.K, stream));
    if (n == 0) return VC_OK;
    VC_CUDA(cudaMemsetAsync(ws, 0xFF, (size_t)slots * 8, stream));
    const int centre = g.K / 2;   // (odd kernel sizes: the centre offset is the middle one)
    if (rep == nullptr && subm_sym(ndim, ksize, unique))
        VC_CUDA(cudaMemsetAsync(nbr + (size_t)(centre + 1) * n, 0xFF, sizeof(int32_t) * (size_t)(g.K - 1 - centre) * n, stream));
    return subm_rulebook_batch_dev(&s, 1, batch_size, unique, stream);
}

extern "C" int vc_subm_rulebook(const int32_t* indices, int n, int ndim, int batch_size, const int32_t* spatial_shape,
                                const int32_t* ksize, const int32_t* dilation, int32_t* nbr, int32_t* pair_num,
                                void* ws, size_t ws_bytes, vc_stream_t stream_) {
    return vc::subm_rulebook_dev(indices, n, nullptr, ndim, batch_size, spatial_shape, ksize, dilation, nbr, pair_num, ws, ws_bytes,
                                 (cudaStream_t)stream_);
}

extern "C" int vc_subm_rulebook_rep(const int32_t* indices, int n, int ndim, int batch_size, const int32_t* spatial_shape,
                                    const int32_t* ksize, const int32_t* dilation, int32_t* nbr, int32_t* pair_num, int32_t* rep,
                                    void* ws, size_t ws_bytes, vc_stream_t stream_) {
    VC_CHECK_ARG(n == 0 || rep, "null pointer");
    return vc::subm_rulebook_dev(indices, n, nullptr, ndim, batch_size, spatial_shape, ksize, dilation, nbr, pair_num, ws, ws_bytes,
                                 (cudaStream_t)stream_, rep);
}

extern "C" int vc_conv_out_shape(int ndim, const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                                 const int32_t* padding, const int32_t* dilation, int32_t* out_shape) {
    Geom g;
    int rc = make_geom(g, ndim, 1, spatial_shape, ksize, stride, padding, dilation);
    if (rc) return rc;
    for (int d = 0; d < ndim; ++d) out_shape[d] = g.oshape[d];
    return VC_OK;
}

bool vc::subm_sym(int ndim, const int32_t* ksize, bool unique) {
    bool sym = unique;
    for (int d = 0; d < ndim; ++d) sym &= (ksize[d] & 1) == 1;
    return sym;
}

// The launches of up to IDX_BATCH_MAX submanifold rulebooks: one hash insert and one probe.  The caller has cleared every
// stage's table (0xFF), its mirrored rows k > centre (-1, when it probes mirrored) and its pair counts.
int vc::subm_rulebook_batch_dev(const SubmStage* st, int n_st, int batch_size, bool unique, cudaStream_t stream) {
    VC_CHECK_ARG(n_st >= 1 && n_st <= IDX_BATCH_MAX, "%d stages in one batch", n_st);
    SubmBatch sb;
    memset(&sb, 0, sizeof(sb));
    sb.sym = -1;
    int ky = 1;
    for (int i = 0; i < n_st; ++i) {
        const SubmStage& s = st[i];
        SubmEntry& e = sb.e[sb.E];
        uint32_t slots;
        int rc = subm_stage_geom(s, batch_size, e.g, slots);
        if (rc) return rc;
        const int sym = s.rep == nullptr && subm_sym(s.ndim, s.ksize, unique) ? 1 : 0;
        VC_CHECK_ARG(sb.sym < 0 || sb.sym == sym, "stages of one batch probe alike");
        sb.sym = sym;
        if (s.n == 0) continue;
        e.idx = s.idx; e.n = s.n; e.n_dev = s.n_dev; e.table = (unsigned long long*)s.table; e.mask = slots - 1;
        e.nbr = s.nbr; e.pair_num = s.pair_num; e.rep = s.rep;
        e.ky = sym ? e.g.K / 2 + 1 : e.g.K;
        ky = e.ky > ky ? e.ky : ky;
        sb.blk0[sb.E + 1] = sb.blk0[sb.E] + cdiv(s.n, 256);
        ++sb.E;
    }
    if (sb.E == 0) return VC_OK;
    hash_insert_kernel<<<sb.blk0[sb.E], 256, 0, stream>>>(sb);
    VC_LAUNCH_CHECK();
    subm_probe_kernel<<<dim3(sb.blk0[sb.E], ky), 256, 0, stream>>>(sb);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// The tables of up to IDX_BATCH_MAX strided convs in one launch.  The caller has filled every nbr_fwd with -1 and zeroed the
// pair counts; a stage without nbr_fwd (NULL) gets it from conv_fwd_lookup_batch_dev.
int vc::conv_tables_batch_dev(const TablesStage* st, int n_st, int batch_size, cudaStream_t stream) {
    VC_CHECK_ARG(n_st >= 1 && n_st <= IDX_BATCH_MAX, "%d stages in one batch", n_st);
    TablesBatch tb;
    memset(&tb, 0, sizeof(tb));
    for (int i = 0; i < n_st; ++i) {
        const TablesStage& s = st[i];
        TablesEntry& e = tb.e[tb.E];
        int rc = make_geom(e.g, s.ndim, batch_size, s.shape, s.ksize, s.stride, s.pad, s.dil);
        if (rc) return rc;
        if (s.n == 0) continue;
        VC_CHECK_ARG(s.idx && s.nbr_bwd, "null pointer");
        e.idx = s.idx; e.n = s.n; e.n_dev = s.n_dev; e.n_out = s.n_out; e.r = s.rank;
        e.nbr_fwd = s.nbr_fwd; e.nbr_bwd = s.nbr_bwd; e.pair_num = s.pair_num;
        tb.blk0[tb.E + 1] = tb.blk0[tb.E] + cdiv(s.n, 256);
        ++tb.E;
    }
    if (tb.E == 0) return VC_OK;
    conv_tables_kernel<<<tb.blk0[tb.E], 256, 0, stream>>>(tb);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// nbr_fwd of up to IDX_BATCH_MAX chained strided convs in one launch; every entry of each table is written (no fill).
int vc::conv_fwd_lookup_batch_dev(const FwdLookupStage* st, int n_st, int batch_size, cudaStream_t stream) {
    VC_CHECK_ARG(n_st >= 1 && n_st <= IDX_BATCH_MAX, "%d stages in one batch", n_st);
    FwdLookupBatch fb;
    memset(&fb, 0, sizeof(fb));
    for (int i = 0; i < n_st; ++i) {
        const FwdLookupStage& s = st[i];
        FwdLookupEntry& e = fb.e[fb.E];
        int rc = make_geom(e.g, s.ndim, batch_size, s.shape, s.ksize, s.stride, s.pad, s.dil);
        if (rc) return rc;
        if (s.n_out == 0) continue;
        VC_CHECK_ARG(s.out_idx && s.nbr_fwd && s.in_rank.bitmap && s.n_in >= 0, "bad arguments");
        e.out_idx = s.out_idx; e.n_out = s.n_out; e.n_out_dev = s.n_out_dev; e.n_in = s.n_in; e.n_in_dev = s.n_in_dev;
        e.in_rank = s.in_rank; e.nbr_fwd = s.nbr_fwd;
        fb.blk0[fb.E + 1] = fb.blk0[fb.E] + cdiv(s.n_out, 256);
        ++fb.E;
    }
    if (fb.E == 0) return VC_OK;
    conv_fwd_lookup_kernel<<<fb.blk0[fb.E], 256, 0, stream>>>(fb);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// Submanifold rulebooks of up to IDX_BATCH_MAX chain levels in one launch.  The caller has zeroed the pair counts.
int vc::subm_lookup_batch_dev(const SubmLookupStage* st, int n_st, int batch_size, cudaStream_t stream) {
    VC_CHECK_ARG(n_st >= 1 && n_st <= IDX_BATCH_MAX, "%d stages in one batch", n_st);
    LookupBatch lb;
    memset(&lb, 0, sizeof(lb));
    for (int i = 0; i < n_st; ++i) {
        const SubmLookupStage& s = st[i];
        LookupEntry& e = lb.e[lb.E];
        int rc = make_geom(e.g, s.ndim, batch_size, s.shape, s.ksize, nullptr, nullptr, s.dil);
        if (rc) return rc;
        VC_CHECK_ARG(s.n >= 0, "row count %d out of range", s.n);
        if (s.n == 0) continue;
        VC_CHECK_ARG(s.idx && s.nbr && s.rank.bitmap, "null pointer");
        e.idx = s.idx; e.n = s.n; e.n_dev = s.n_dev; e.rank = s.rank; e.nbr = s.nbr; e.pair_num = s.pair_num;
        lb.blk0[lb.E + 1] = lb.blk0[lb.E] + cdiv(s.n, 256);
        ++lb.E;
    }
    if (lb.E == 0) return VC_OK;
    subm_lookup_kernel<<<lb.blk0[lb.E], 256, 0, stream>>>(lb);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

namespace {
// scan blocks of one level's bitmap: every level starts on a SCAN_WORDS boundary, so a scan block never spans two levels
int level_blocks(int ndim, int batch, const int32_t* oshape) {
    long long cells = batch;
    for (int d = 0; d < ndim; ++d) cells *= oshape[d];
    return (int)(((cells + 31) / 32 + SCAN_WORDS - 1) / SCAN_WORDS);
}
// the chain's workspace: bitmap [W words], word ranks [W], block sums [B], W = B * SCAN_WORDS, B = cd.b0[L]
size_t chain_bytes(int blocks) { return (size_t)blocks * SCAN_WORDS * 8 + ((size_t)blocks * 4 + 255) / 256 * 256; }
struct ChainWs {
    uint32_t *bitmap, *word_rank, *block_sum;
    size_t bytes;
};
int chain_layout(const ConvChain& ch, ChainDesc& cd, ChainWs& w, const void* ws) {
    VC_CHECK_ARG(conv_chain_composable(ch), "chain of %d strided convs (2 or more need dilation 1)", ch.L);
    memset(&cd, 0, sizeof(cd));
    cd.L = ch.L;
    const int32_t* shape = ch.shape0;
    for (int l = 0; l < ch.L; ++l) {
        int rc = make_geom(cd.g[l], ch.ndim, ch.batch, shape, ch.ksize[l], ch.stride[l], ch.pad[l], ch.dil[l]);
        if (rc) return rc;
        shape = cd.g[l].oshape;
        cd.b0[l + 1] = cd.b0[l] + level_blocks(ch.ndim, ch.batch, cd.g[l].oshape);
        cd.w0[l + 1] = (long long)cd.b0[l + 1] * SCAN_WORDS;
    }
    for (int d = 0; d < ch.ndim; ++d) cd.dilated |= cd.g[0].dil[d] != 1;
    VC_CHECK_ARG(cd.w0[ch.L] < (1LL << 31), "output grids too large");
    w.bitmap = (uint32_t*)const_cast<void*>(ws);
    w.word_rank = w.bitmap + cd.w0[ch.L];
    w.block_sum = w.word_rank + cd.w0[ch.L];
    w.bytes = chain_bytes(cd.b0[ch.L]);
    return VC_OK;
}
}  // namespace

bool vc::conv_chain_composable(const ConvChain& ch) {
    if (ch.L < 1 || ch.L > CONV_CHAIN_MAX) return false;
    if (ch.L == 1) return true;   // level 0 alone: a dilation is marked per kernel offset
    for (int l = 0; l < ch.L; ++l)
        for (int d = 0; d < ch.ndim; ++d)
            if (ch.dil[l][d] != 1) return false;
    return true;
}

size_t vc::conv_chain_ws_bytes(const ConvChain& ch) {
    ChainDesc cd;
    ChainWs w;
    return chain_layout(ch, cd, w, nullptr) == VC_OK ? w.bytes : 0;
}

ConvRank vc::conv_chain_rank(const ConvChain& ch, const void* ws, int level) {
    ChainDesc cd;
    ChainWs w;
    if (chain_layout(ch, cd, w, ws) != VC_OK) return ConvRank{nullptr, nullptr, nullptr};
    return ConvRank{w.bitmap + cd.w0[level], w.word_rank + cd.w0[level], w.block_sum + cd.b0[level]};
}

int vc::conv_chain_count_dev(const ConvChain& ch, const int32_t* indices, int n, const int* n_dev, int32_t* n_out_dev, const int* caps,
                             int* overflow, void* ws, size_t ws_bytes, cudaStream_t stream) {
    ChainDesc cd;
    ChainWs w;
    int rc = chain_layout(ch, cd, w, ws);
    if (rc) return rc;
    VC_CHECK_ARG(n >= 0 && n_out_dev && ws, "bad arguments");
    if (ws_bytes < w.bytes) {
        set_error("conv chain workspace %zu < %zu", ws_bytes, w.bytes);
        return VC_ERR_WORKSPACE;
    }
    for (int l = 0; l < ch.L; ++l) cd.cap[l] = caps ? caps[l] : 0;
    VC_CUDA(cudaMemsetAsync(w.bitmap, 0, (size_t)cd.w0[ch.L] * 4, stream));
    if (n > 0) {
        conv_mark_kernel<<<dim3(cdiv(n, 256), cd.dilated ? cd.g[0].K : ch.L), 256, 0, stream>>>(indices, n, n_dev, cd, w.bitmap);
        VC_LAUNCH_CHECK();
    }
    scan_local_kernel<<<cd.b0[ch.L], 256, 0, stream>>>(w.bitmap, cd.w0[ch.L], w.word_rank, w.block_sum);
    VC_LAUNCH_CHECK();
    scan_blocks_kernel<<<1, 1024, 0, stream>>>(w.block_sum, cd, n_out_dev, overflow);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int vc::conv_chain_emit_dev(const ConvChain& ch, int32_t* const* out_idx, const int* caps, void* ws, size_t ws_bytes,
                            cudaStream_t stream) {
    ChainDesc cd;
    ChainWs w;
    int rc = chain_layout(ch, cd, w, ws);
    if (rc) return rc;
    VC_CHECK_ARG(ws && ws_bytes >= w.bytes, "conv chain workspace too small");
    for (int l = 0; l < ch.L; ++l) {
        VC_CHECK_ARG(caps[l] <= 0 || out_idx[l], "null output pointer");
        cd.out_idx[l] = out_idx[l];
        cd.cap[l] = caps[l];
    }
    conv_emit_indices_kernel<<<cdiv(cd.w0[ch.L], 256), 256, 0, stream>>>(w.bitmap, w.word_rank, w.block_sum, cd);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// The per-operator strided conv: a chain of one.  The count leaves its ranked output bitmap in `ws`; the fill emits the
// output indices and builds the tables from it.
extern "C" size_t vc_conv_rulebook_ws_bytes(int ndim, int batch_size, const int32_t* out_shape) {
    return chain_bytes(level_blocks(ndim, batch_size, out_shape));
}

extern "C" int vc_conv_rulebook_count(const int32_t* indices, int n, int ndim, int batch_size,
                                      const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                                      const int32_t* padding, const int32_t* dilation, int32_t* n_out_dev, void* ws,
                                      size_t ws_bytes, vc_stream_t stream_) {
    const ConvChain ch{1, ndim, batch_size, spatial_shape, {ksize}, {stride}, {padding}, {dilation}};
    return conv_chain_count_dev(ch, indices, n, nullptr, n_out_dev, nullptr, nullptr, ws, ws_bytes, (cudaStream_t)stream_);
}

extern "C" int vc_conv_rulebook_fill(const int32_t* indices, int n, int ndim, int batch_size,
                                     const int32_t* spatial_shape, const int32_t* ksize, const int32_t* stride,
                                     const int32_t* padding, const int32_t* dilation, int n_out, int32_t* out_indices,
                                     int32_t* nbr_fwd, int32_t* nbr_bwd, int32_t* pair_num, void* ws, size_t ws_bytes,
                                     vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    const ConvChain ch{1, ndim, batch_size, spatial_shape, {ksize}, {stride}, {padding}, {dilation}};
    Geom g;
    int rc = make_geom(g, ndim, batch_size, spatial_shape, ksize, stride, padding, dilation);
    if (rc) return rc;
    const size_t need = conv_chain_ws_bytes(ch);
    if (!ws || ws_bytes < need) {
        set_error("conv rulebook workspace %zu < %zu", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    if (n_out > 0) {
        VC_CHECK_ARG(nbr_fwd, "null output pointer");
        rc = conv_chain_emit_dev(ch, &out_indices, &n_out, ws, ws_bytes, stream);
        if (rc) return rc;
    }
    if (pair_num) VC_CUDA(cudaMemsetAsync(pair_num, 0, sizeof(int32_t) * g.K, stream));
    if (n_out > 0) VC_CUDA(cudaMemsetAsync(nbr_fwd, 0xFF, (size_t)g.K * n_out * 4, stream));
    const TablesStage s{indices, n, nullptr, ndim, spatial_shape, ksize, stride, padding, dilation, n_out,
                        conv_chain_rank(ch, ws, 0), nbr_fwd, nbr_bwd, pair_num};
    return conv_tables_batch_dev(&s, 1, batch_size, stream);
}

extern "C" int vc_pairs_from_nbr(const int32_t* nbr, int K, int n, int32_t* pairs, int32_t* pair_num,
                                 vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(K > 0 && n >= 0 && pairs && pair_num, "bad arguments");
    if (n == 0) {
        VC_CUDA(cudaMemsetAsync(pair_num, 0, sizeof(int32_t) * K, stream));
        return VC_OK;
    }
    pairs_kernel<<<K, 1024, 0, stream>>>(nbr, K, n, pairs, pair_num);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
