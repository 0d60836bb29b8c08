// Weight gradient of the sparse convolutions on tensor cores — persistent, wgmma, sm_90a.
//
//   dW[k] (C_in x C_out) = sum over output rows o of  in[nbr[k,o], :]^T (x) dout[o, :]
//
// Ring stages of 64 rows (16 KB), <= 111 KB shared memory and 448 threads per CTA, so that a wgrad CTA and a dgrad CTA of the
// main stream can share an SM: the plan executor runs this kernel on its own stream beside the dgrad chain.
// Same machinery as the persistent forward kernel (conv_tc2.cu): persistent CTAs walk 128-row output tiles (dynamic tile
// counter), a loader warp stages each tile's neighbour-table slice (bulk copies completing on an mbarrier) into a ring of
// 2-4 tile slots, a dout warp fills the slot's dout tile, 4 producer warps gather the rows with 16-byte cp.async into
// 32/64/128-byte-swizzled tiles, two consumer warpgroups (64 accumulator rows each) issue the MMAs.  What differs:
//   * the gathered tile is used MN-MAJOR (the reduction runs over the 128 rows): the row-major swizzled tile the forward
//     kernel builds is exactly the canonical Major-MN layout, and G = 128 / C_in kernel offsets are stacked along the MMA
//     M dimension through the descriptor's leading-byte offset (one ring stage = G half tiles);
//   * the second operand is the tile of dout itself (contiguous rows, loaded once per tile into the tile's slot);
//   * the accumulators of the pass's offset groups (<= 64 / C_out, 32 registers per thread: two CTAs fit an SM) stay
//     resident in registers across all tiles of the CTA (more groups: more passes, blockIdx.y); at the end each CTA adds
//     its [K, C_in, C_out] partial into ONE fp32 scratch image with 8-byte vector reductions.  Per-CTA partials re-read by a
//     second kernel (round 1) cost 218 MB + 218 MB per step for 1.7 MB of gradients; here the reduction traffic is
//     (#CTAs x gradient size) of L2 atomics and the only extra launch per STEP is the transposing finalize of all layers
//     (wgrad_finalize_kernel).  The order of those reductions depends on scheduling: results vary in the last bits.
//   * C = 8 layers run with channels padded to 16 (zero-filled by the gather).
// Replaces spconv `ops.indice_conv_backward` (filter gradient) behind spconv_backbone.py:89,92-93,113,563-564.
// Algorithmic bytes per launch: (N_in*C_in + N_out*C_out)*2 + P*8 + K*C_in*C_out*4;  FLOPs 2*P*C_in*C_out.
#include "tc_common.cuh"

namespace vc {

int g_wgrad3_ctas = 0;      // CTA cap of the plan executor's launches (vc_conv_wgrad_tc3_config); 0 = half the SMs per pass

namespace {

// Two CTAs per SM (like conv_tc2.cu: a CTA that leaves half the SM free can share it with the dgrad kernels of the main
// stream).  A ring stage is HALF a tile (64 rows) of the GW offsets of one accumulator group: 16 KB; the two producer groups
// (2 warps each) own the two halves.
constexpr int W_CONS_WARPS = 8;                                    // two consumer warpgroups
constexpr int W_WARP_LOADER = W_CONS_WARPS, W_WARP_DOUT = W_WARP_LOADER + 1, W_WARP_PROD0 = W_WARP_DOUT + 1;
constexpr int W_GROUPS = 2, W_GROUP_WARPS = 2;
constexpr int W_PROD_WARPS = W_GROUPS * W_GROUP_WARPS;             // 4
constexpr int W_THREADS = 32 * (W_WARP_PROD0 + W_PROD_WARPS);      // 448: still 72 registers per thread at two CTAs per SM
constexpr int W_MAX_STAGES = 8;
constexpr int W_MAX_NT = 4;                                       // tile slots (table slice + dout tile) a CTA loads ahead
constexpr int W_HROWS = TCM / 2;                                   // rows of a ring stage
constexpr int W_ROWS_PER_PROD = W_HROWS / W_GROUP_WARPS;           // 32
constexpr int W_ACC = 64;                                          // accumulator columns (x 64 rows) per consumer warpgroup
constexpr int W_SMEM_BUDGET = (227 * 1024) / 2 - 5 * 1024;

template <int CI, int CO>
struct WCfg2 {
    static constexpr int RA = CI * 2, RB = CO * 2;           // row bytes of a gathered tile / of the dout tile (= swizzle spans)
    static constexpr int CPA = CI / 8, CPB = CO / 8;         // 16-byte chunks per row
    static constexpr int GW = 128 / CI;                      // kernel offsets stacked along M (one accumulator group)
    static constexpr int A_BYTES = W_HROWS * RA;             // one offset's half tile
    static constexpr int STAGE = GW * A_BYTES;               // 16 KB for every C_in
    static constexpr int B_BYTES = TCM * RB;
};

struct WArgs {
    const __nv_bfloat16* in;    // [n_in, in_ld] gathered rows
    int in_c;                   // real channels (8 or CI)
    int in_ld;                  // row pitch (>= in_c: the rows may be a column slice of a wider matrix)
    const __nv_bfloat16* dout;  // [n_out, out_c]
    int out_c;                  // real channels (8 or CO)
    const int32_t* nbr;         // [K][pitch]
    long long pitch;
    float* scratch;             // [K][in_c][out_c] fp32, zero before the launch; every CTA adds its partial
    const int* n_dev;
    int n_host;
    int* tile_counter;          // [passes] or NULL
    int K, S, groups_per_pass;
    int NT;                     // tile slots in shared memory (see launch_wgrad3)
    int det_chunks;             // > 0: deterministic mode, scratch = [det_chunks][K][in_c][out_c] (see tc3_wgrad)
    int* err;
};

#define W_WAIT(bar, parity, code)                                     \
    do {                                                              \
        if (!mbar_wait_t((bar), (parity), a.err, (code))) goto done;  \
    } while (0)

__device__ __forceinline__ void w_sts_zero16(uint32_t saddr) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(saddr), "r"(0u) : "memory");
}

template <int CI, int CO>
__global__ void __launch_bounds__(W_THREADS, 2) tc_wgrad_half_kernel(const WArgs a) {
    using C = WCfg2<CI, CO>;
    constexpr int W_MAXG = W_ACC / CO, W_STAGES_PER_GROUP = 2, W_MMAS_PER_STAGE = W_HROWS / 16;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int S = a.S, K = a.K, NT = a.NT;
    unsigned char* ring = smem_raw;                                              // [S][GW x A half tile]
    unsigned char* dout_s = smem_raw + (size_t)S * C::STAGE;                     // [NT][B tile]
    int* nbr_s = reinterpret_cast<int*>(dout_s + (size_t)NT * C::B_BYTES);     // [NT][kcount][128]
    __shared__ __align__(8) uint64_t full_bar[W_MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[W_MAX_STAGES];
    __shared__ __align__(8) uint64_t tbl_full[W_MAX_NT], tbl_empty[W_MAX_NT];
    __shared__ __align__(8) uint64_t dout_full[W_MAX_NT], dout_empty[W_MAX_NT];
    __shared__ __align__(8) uint64_t claim_bar[W_MAX_NT];
    __shared__ int tile_s[W_MAX_NT];

    // the role index read through a shuffle: the compiler can then tell that the consumer branch is warp-uniform, and does not
    // serialize its wgmma instructions
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
    // this pass's slice of the kernel offsets (passes only when the accumulators of all groups exceed W_ACC columns)
    const int n_groups_total = (K + C::GW - 1) / C::GW;
    const int g_begin = blockIdx.y * a.groups_per_pass;
    const int g_count = min(a.groups_per_pass, n_groups_total - g_begin);
    const int k_begin = g_begin * C::GW;
    const int k_count = min(g_count * C::GW, K - k_begin);

    if (tid == W_WARP_LOADER * 32) {
        for (int s = 0; s < S; ++s) {
            // every producer thread of the stage's group (cp.async.mbarrier.arrive.noinc: fires when the thread's copies have
            // landed) + one release arrive per warp for its zero stores
            mbar_init(&full_bar[s], 32 * W_GROUP_WARPS + W_GROUP_WARPS);
            mbar_init(&empty_bar[s], 2);                       // one arrive per consumer warpgroup
        }
        for (int b = 0; b < NT; ++b) {
            mbar_init(&tbl_full[b], 1);                        // loader (arrive.expect_tx of the bulk copies, or a plain arrive)
            mbar_init(&tbl_empty[b], W_PROD_WARPS + W_CONS_WARPS + 1);   // producers + consumers + dout loader
            mbar_init(&dout_full[b], 32);                      // every dout-loader lane (cp.async arrive)
            mbar_init(&dout_empty[b], 2);                      // one arrive per consumer warpgroup
            mbar_init(&claim_bar[b], 1);                       // loader: tile_s holds the slot's tile
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const int n = a.n_dev != nullptr ? min(__ldg(a.n_dev), a.n_host) : a.n_host;
    // a pipeline wait that timed out in an EARLIER launch left the (sticky) error flag set: do nothing, so that whatever went
    // wrong costs one 2-second timeout, not one per launch
    const bool dead = a.err != nullptr && *reinterpret_cast<volatile int*>(a.err) != 0;
    const int n_tiles = dead ? 0 : (n + TCM - 1) / TCM;
    int* counter = a.tile_counter != nullptr ? a.tile_counter + blockIdx.y : nullptr;
    // deterministic mode: tiles [c * tpc, (c + 1) * tpc) form chunk c, claimed whole (from the row count alone: the same split
    // for every grid); each chunk's sum goes to its own partial image
    const int tpc = a.det_chunks > 0 ? max(1, (n_tiles + a.det_chunks - 1) / a.det_chunks) : 0;
    const int n_chunks = tpc > 0 ? (n_tiles + tpc - 1) / tpc : 0;
    const size_t part_floats = (size_t)K * a.in_c * a.out_c;
    __syncthreads();

    if (warp == W_WARP_LOADER) {
        // ------------------------------------------------------------ tile scheduler + neighbour-table loader
        // Tile slot it % NT holds the tile's table slice and its dout tile.  The slice (one 512-byte span per kernel offset) comes
        // in by bulk copies that complete on tbl_full, up to NT tiles ahead of the producers.  claim_bar publishes the slot's tile
        // before its table lands, so the dout warp starts on the dout tile at once; neither this warp nor the producers wait for
        // a dout buffer.
        const bool bulk_ok = (reinterpret_cast<uintptr_t>(a.nbr) & 15u) == 0 && (a.pitch & 3) == 0;
        bool stop = false;
        int claimed = 0;
        int c_next = 0, c_end = 0;          // deterministic mode: the rest of the claimed chunk
        for (int it = 0;; ++it) {
            const int tb = it % NT;
            int tile = -1;
            if (!stop && tpc > 0) {
                if (c_next >= c_end) {
                    int chunk;
                    if (counter != nullptr) {
                        chunk = lane == 0 ? atomicAdd(counter, 1) : 0;
                        chunk = __shfl_sync(0xffffffffu, chunk, 0);
                    } else {
                        chunk = blockIdx.x + claimed * gridDim.x;
                    }
                    ++claimed;
                    if (chunk >= n_chunks) {
                        stop = true;
                    } else {
                        c_next = chunk * tpc;
                        c_end = min(n_tiles, c_next + tpc);
                    }
                }
                if (!stop) tile = c_next++;
            } else if (!stop) {
                if (counter != nullptr) {
                    tile = lane == 0 ? atomicAdd(counter, 1) : 0;
                    tile = __shfl_sync(0xffffffffu, tile, 0);
                } else {
                    tile = blockIdx.x + claimed * gridDim.x;
                }
                ++claimed;
                if (tile >= n_tiles) {
                    tile = -1;
                    stop = true;
                }
            }
            if (it >= NT) W_WAIT(&tbl_empty[tb], (uint32_t)(((it / NT) - 1) & 1), 0x201);
            if (lane == 0) tile_s[tb] = tile;
            __syncwarp();
            if (lane == 0) mbar_arrive(&claim_bar[tb]);
            if (tile < 0) {
                if (lane == 0) mbar_arrive(&tbl_full[tb]);
                break;
            }
            int* dst = nbr_s + (size_t)tb * k_count * TCM;
            const int base = tile * TCM;
            if (bulk_ok && (long long)base + TCM <= a.pitch) {
                // the producers treat the rows at or past n as missing, whatever the table holds there
                if (lane == 0) mbar_expect_tx(&tbl_full[tb], (uint32_t)(k_count * TCM * 4));
                __syncwarp();
                for (int k = lane; k < k_count; k += 32)
                    bulk_g2s(smem_u32(dst + k * TCM), a.nbr + (size_t)(k_begin + k) * a.pitch + base, TCM * 4, &tbl_full[tb]);
            } else {
                for (int k = 0; k < k_count; ++k)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int row = base + q * 32 + lane;
                        dst[k * TCM + q * 32 + lane] = row < n ? __ldg(a.nbr + (size_t)(k_begin + k) * a.pitch + row) : -1;
                    }
                __syncwarp();
                if (lane == 0) mbar_arrive(&tbl_full[tb]);
            }
        }
    } else if (warp == W_WARP_DOUT) {
        // ------------------------------------------------------------ dout loader
        // the tile of dout (second operand of every group of the tile): contiguous rows, copied by the 32 lanes' cp.async into
        // its swizzled image (a bulk copy cannot swizzle) once the consumers have retired the slot's previous tile
        for (int it = 0;; ++it) {
            const int tb = it % NT;
            W_WAIT(&claim_bar[tb], (uint32_t)((it / NT) & 1), 0x202);
            const int tile = tile_s[tb];
            __syncwarp();
            if (lane == 0) mbar_arrive(&tbl_empty[tb]);
            if (tile < 0) break;
            const int base = tile * TCM;
            if (it >= NT) W_WAIT(&dout_empty[tb], (uint32_t)(((it / NT) - 1) & 1), 0x203);
            const uint32_t b_s = smem_u32(dout_s) + (uint32_t)tb * C::B_BYTES;
            for (int q = lane; q < TCM * C::CPB; q += 32) {
                const int r = q / C::CPB, c = q % C::CPB;
                const bool v = base + r < n && c * 8 < a.out_c;
                cp_async16_s(b_s + swz_off<C::RB>(r, c), v ? a.dout + (size_t)(base + r) * a.out_c + c * 8 : a.dout, v);
            }
            cp_async_arrive_noinc(&dout_full[tb]);
        }
    } else if (warp >= W_WARP_PROD0) {
        // ------------------------------------------------------------ gather producers
        const int grp = (warp - W_WARP_PROD0) / W_GROUP_WARPS, pw = (warp - W_WARP_PROD0) % W_GROUP_WARPS;   // grp = half of the tile
        constexpr int CW = C::CPA < 4 ? C::CPA : 4;
        constexpr int RPI = 32 / CW;
        constexpr int NIT = W_ROWS_PER_PROD / RPI;
        constexpr int NCG = C::CPA / CW;
        const int c_sub = lane % CW, r_sub = lane / CW;
        int rows[NIT];
        uint32_t dst_off[NIT][NCG];
        bool ch_ok[NCG];
#pragma unroll
        for (int i = 0; i < NIT; ++i) {
            rows[i] = grp * W_HROWS + pw * W_ROWS_PER_PROD + i * RPI + r_sub;
#pragma unroll
            for (int cg = 0; cg < NCG; ++cg) dst_off[i][cg] = swz_off<C::RA>(rows[i] - grp * W_HROWS, cg * CW + c_sub);
        }
#pragma unroll
        for (int cg = 0; cg < NCG; ++cg) ch_ok[cg] = (cg * CW + c_sub) * 8 < a.in_c;
        const uint32_t ring_s = smem_u32(ring);
        int s = 0, wr = 0, turn = 0;
        for (int it = 0;; ++it) {
            const int tb = it % NT;
            W_WAIT(&tbl_full[tb], (uint32_t)((it / NT) & 1), 0x211);
            const int tile = tile_s[tb];
            if (tile < 0) break;
            const int* tbl = nbr_s + (size_t)tb * k_count * TCM;
            const int rows_left = n - tile * TCM;       // rows at or past it are missing (the last tile's tail)
            for (int gs = 0; gs < 2 * g_count; ++gs) {         // stage (group g, half h) = 2 g + h; half h belongs to producer group h
                const int g = gs >> 1;
                if (turn == grp) {
                    int src[C::GW][NIT];
#pragma unroll
                    for (int j = 0; j < C::GW; ++j) {
                        const int kk = g * C::GW + j;
#pragma unroll
                        for (int i = 0; i < NIT; ++i) src[j][i] = kk < k_count && rows[i] < rows_left ? tbl[kk * TCM + rows[i]] : -1;
                    }
                    if (wr > 0) W_WAIT(&empty_bar[s], (uint32_t)((wr - 1) & 1), 0x213);
                    const uint32_t st_s = ring_s + (uint32_t)s * C::STAGE;
#pragma unroll
                    for (int j = 0; j < C::GW; ++j) {
                        const uint32_t a_s = st_s + (uint32_t)j * C::A_BYTES;
#pragma unroll
                        for (int i = 0; i < NIT; ++i) {
                            const bool v = src[j][i] >= 0;
                            const __nv_bfloat16* srow = a.in + (size_t)(v ? src[j][i] : 0) * a.in_ld + c_sub * 8;
#pragma unroll
                            for (int cg = 0; cg < NCG; ++cg) {
                                // a missing neighbour costs a shared-memory zero store, not a zero-fill cp.async
                                if (v && ch_ok[cg]) cp_async16_s(a_s + dst_off[i][cg], srow + cg * CW * 8, true);
                                else w_sts_zero16(a_s + dst_off[i][cg]);
                            }
                        }
                    }
                    cp_async_arrive_noinc(&full_bar[s]);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&full_bar[s]);     // release: publishes the warp's zero stores
                }
                if (++turn == W_GROUPS) turn = 0;
                if (++s == S) {
                    s = 0;
                    ++wr;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&tbl_empty[tb]);
        }
    } else {
        // ------------------------------------------------------------ consumers: MMAs into register accumulators, one flush per run
        const int wg = warp >> 2, t = tid & 127;
        float acc[W_MAXG][CO / 2];
#pragma unroll
        for (int gg = 0; gg < W_MAXG; ++gg)
#pragma unroll
            for (int j = 0; j < CO / 2; ++j) acc[gg][j] = 0.f;
        const uint32_t full0 = smem_u32(&full_bar[0]), doutf0 = smem_u32(&dout_full[0]);
        const uint32_t ring_a = smem_u32(ring) + (uint32_t)(wg * (64 / CI) * C::A_BYTES), dout_a = smem_u32(dout_s);
        int s = 0;
        uint32_t ph = 0;
        int it = 0;
        for (bool more = true; more;) {
            // one run of tiles summed into the accumulators, then one flush: the whole CTA, or in deterministic mode one chunk
            int chunk = -1, n_done = 0;
            for (;; ++it) {
                const int tb = it % NT;
                W_WAIT(&tbl_full[tb], (uint32_t)((it / NT) & 1), 0x221);
                const int tile = tile_s[tb];
                if (tile < 0) {
                    more = false;
                    break;
                }
                if (tpc > 0) {
                    if (n_done == 0) chunk = tile / tpc;
                    else if (tile / tpc != chunk) break;      // the chunk is complete; this tile starts the next run
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&tbl_empty[tb]);
                if (!mbar_spin(doutf0 + 8u * tb, (uint32_t)((it / NT) & 1), 4096u) &&
                    !mbar_wait_t_addr(doutf0 + 8u * tb, (uint32_t)((it / NT) & 1), a.err, 0x222))
                    goto done;
                const uint32_t b_s = dout_a + (uint32_t)tb * C::B_BYTES;
                int prev = -1;                       // ring slot whose MMAs may still be in flight
                for (int gs = 0; gs < W_STAGES_PER_GROUP * g_count; ++gs) {
                    if (!mbar_spin(full0 + 8u * s, ph, 4096u) && !mbar_wait_t_addr(full0 + 8u * s, ph, a.err, 0x223)) goto done;
                    fence_async_smem();     // generic-proxy (cp.async, st.shared) writes -> visible to the tensor core's async proxy
                    wg_fence();
                    wgrad_stage_mma<CI, CO, W_MMAS_PER_STAGE, W_MAXG, C::A_BYTES>(
                        acc, gs / W_STAGES_PER_GROUP, ring_a + (uint32_t)s * C::STAGE,
                        b_s + (uint32_t)((gs % W_STAGES_PER_GROUP) * W_MMAS_PER_STAGE * 16 * C::RB),
                        n_done > 0 || gs % W_STAGES_PER_GROUP != 0 ? 1u : 0u);
                    wg_commit();
                    wg_wait<1>();                    // the previous stage's MMAs have completed: release its ring slot
                    if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
                    prev = s;
                    if (++s == S) {
                        s = 0;
                        ph ^= 1u;
                    }
                }
                wg_wait<0>();
                if (t == 0) {
                    mbar_arrive(&empty_bar[prev]);
                    mbar_arrive(&dout_empty[tb]);
                }
                ++n_done;
            }
#pragma unroll
            for (int gg = 0; gg < W_MAXG; ++gg) wg_fence_acc(acc[gg]);
            // (the next run's first MMA of each group starts its sum afresh: no zeroing of the accumulators here)
            if (n_done > 0)
                wgrad_flush<CI, CO, W_MAXG>(acc, wg, t, g_count, k_begin, k_count, a.in_c, a.out_c,
                                            a.scratch + (tpc > 0 ? (size_t)chunk * part_floats : 0));
        }
    }
done:
    cp_async_wait<0>();
    __syncthreads();
}

// CTAs per pass of a launch over n_rows output rows: max_ctas is the budget of the whole launch, split over its passes, so
// grid.x * passes <= max_ctas whenever passes <= max_ctas.  Every pass keeps at least one CTA, so only a launch with more
// passes than max_ctas exceeds the cap (by taking one CTA per pass).
int wgrad3_grid_x(int n_rows, int passes, int max_ctas) {
    const int tiles = cdiv(n_rows, TCM), per_pass = max_ctas / passes;
    const int g = tiles < per_pass ? tiles : per_pass;
    return g < 1 ? 1 : g;
}

template <int CI, int CO>
int launch_wgrad3(const WArgs& a0, int n_cap, int max_ctas, cudaStream_t stream) {
    using C = WCfg2<CI, CO>;
    WArgs a = a0;
    const int n_groups = (a.K + C::GW - 1) / C::GW;
    const int max_groups = W_ACC / CO;
    int passes = (n_groups + max_groups - 1) / max_groups;
    int gpp = (n_groups + passes - 1) / passes;
    const int kcount = gpp * C::GW < a.K ? gpp * C::GW : a.K;
    a.groups_per_pass = gpp;
    const size_t slot = (size_t)C::B_BYTES + (size_t)kcount * TCM * 4;     // one tile slot: dout tile + table slice
    auto stages = [&](int nt) {
        const long long s = ((long long)W_SMEM_BUDGET - (long long)nt * (long long)slot) / C::STAGE;
        return (int)(s > W_MAX_STAGES ? W_MAX_STAGES : s);
    };
    // as many tile slots as fit without taking a stage from the gather ring (the stages hold most of the bytes in flight)
    int NT = 2;
    while (NT < W_MAX_NT && stages(NT + 1) >= stages(2)) ++NT;
    const int S = stages(NT);
    if (S < 2) {
        set_error("tensor-core wgrad: no room for the operand ring (K=%d, %d->%d)", a.K, CI, CO);
        return VC_ERR_UNSUPPORTED;
    }
    a.S = S;
    a.NT = NT;
    const size_t smem = (size_t)S * C::STAGE + (size_t)NT * slot;
    auto kern = tc_wgrad_half_kernel<CI, CO>;
    static bool attr_done = false;
    if (!attr_done) {
        VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, W_SMEM_BUDGET));
        attr_done = true;
    }
    kern<<<dim3(wgrad3_grid_x(n_cap, passes, max_ctas), passes), dim3(W_THREADS), smem, stream>>>(a);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

}  // namespace

// scratch: [K][cin][cout] fp32, ZERO on entry (the kernel accumulates); tile_counter: `wgrad3_passes(cin, cout, K)` ints, zero;
// at most max_ctas CTAs over all passes (wgrad3_grid_x)
int tc3_wgrad(int cin, int cout, const void* in_bf16, const void* dout_bf16, const int32_t* nbr, long long pitch, float* scratch,
              int n_rows, const int* n_dev, int K, int* err, cudaStream_t stream, int* tile_counter, int max_ctas, int in_ld,
              int det_chunks) {
    if (n_rows == 0) return VC_OK;
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout) || K < 1 || K > MAXK_TC) {
        set_error("tensor-core wgrad: unsupported shape (%d -> %d channels, K=%d)", cin, cout, K);
        return VC_ERR_UNSUPPORTED;
    }
    WArgs a;
    if (in_ld == 0) in_ld = cin;
    if (in_ld < cin || in_ld % 8 != 0) {
        set_error("tensor-core wgrad: row pitch %d for %d channels", in_ld, cin);
        return VC_ERR_INVALID;
    }
    a.in = (const __nv_bfloat16*)in_bf16; a.in_c = cin; a.in_ld = in_ld; a.dout = (const __nv_bfloat16*)dout_bf16; a.out_c = cout; a.nbr = nbr;
    a.pitch = pitch; a.scratch = scratch; a.n_dev = n_dev; a.n_host = n_rows; a.tile_counter = tile_counter; a.K = K; a.S = 0;
    a.groups_per_pass = 0; a.NT = 0; a.err = err; a.det_chunks = det_chunks;
    const int ci = tc_pad16(cin), co = tc_pad16(cout);
#define VC_W_CASE(A, B) \
    if (ci == A && co == B) return launch_wgrad3<A, B>(a, n_rows, max_ctas, stream);
    VC_W_CASE(16, 16) VC_W_CASE(16, 32) VC_W_CASE(16, 64)
    VC_W_CASE(32, 16) VC_W_CASE(32, 32) VC_W_CASE(32, 64)
    VC_W_CASE(64, 16) VC_W_CASE(64, 32) VC_W_CASE(64, 64)
#undef VC_W_CASE
    return VC_ERR_UNSUPPORTED;
}

int wgrad3_passes(int cin, int cout, int K) {
    const int ci = tc_pad16(cin), co = tc_pad16(cout);
    const int n_groups = (K + 128 / ci - 1) / (128 / ci);
    const int max_groups = W_ACC / co;
    return (n_groups + max_groups - 1) / max_groups;
}

// scratch [K][cin][cout] (one per layer) -> parameter layout dW [cout][K][cin], every layer of a step in ONE launch
__global__ void __launch_bounds__(256) wgrad_finalize_kernel(WgradFinTable t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.total) return;
    int lo = 0, hi = t.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t.e[mid].first <= i) lo = mid; else hi = mid - 1;
    }
    const WgradFinEntry& e = t.e[lo];
    const int j = i - e.first;                       // index in the parameter layout: coalesced writes
    const int ci = j % e.cin, k = (j / e.cin) % e.K, co = j / (e.cin * e.K);
    const size_t o = ((size_t)k * e.cin + ci) * e.cout + co, img = (size_t)e.K * e.cin * e.cout;
    if (e.n_part == 1) {
        e.dw[j] = __ldg(e.scratch + o);
    } else {                    // deterministic mode: the chunk images in chunk order, in float64, rounded once
        double v = 0.0;
        for (int p = 0; p < e.n_part; ++p) v += (double)__ldg(e.scratch + p * img + o);
        e.dw[j] = (float)v;
    }
}

int wgrad_finalize(WgradFinTable& t, cudaStream_t stream) {
    if (t.n == 0) return VC_OK;
    int total = 0;
    for (int i = 0; i < t.n; ++i) {
        t.e[i].first = total;
        total += t.e[i].K * t.e[i].cin * t.e[i].cout;
    }
    t.total = total;
    wgrad_finalize_kernel<<<cdiv(total, 256), 256, 0, stream>>>(t);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

}  // namespace vc

using namespace vc;

extern "C" int vc_conv_wgrad_tc3_config(int variant, int max_ctas) {
    VC_CHECK_ARG(variant == 1, "wgrad variant must be 1 (the half-tile-stage kernel is the only one)");
    VC_CHECK_ARG(max_ctas >= 0 && max_ctas <= 1024, "wgrad CTA cap out of range (%d)", max_ctas);
    g_wgrad3_ctas = max_ctas;
    return VC_OK;
}

extern "C" int vc_wgrad_launch_geometry(int cin, int cout, int K, int n_rows, int max_ctas, int32_t* out) {
    VC_CHECK_ARG(out && n_rows >= 0 && max_ctas >= 1 && K >= 1 && K <= MAXK_TC && tc2_ch_ok(cin) && tc2_ch_ok(cout),
                 "bad wgrad geometry query (%d -> %d channels, K=%d, %d rows, cap %d)", cin, cout, K, n_rows, max_ctas);
    out[1] = wgrad3_passes(cin, cout, K);
    out[0] = n_rows > 0 ? wgrad3_grid_x(n_rows, out[1], max_ctas) : 0;
    return VC_OK;
}

extern "C" size_t vc_conv_wgrad_tc_ws_bytes(int n_out, int cin, int cout, int K) {
    // the scratch image all CTAs accumulate into (whatever n_out), then one tile counter per pass
    const size_t passes = tc2_ch_ok(cin) && tc2_ch_ok(cout) && K >= 1 ? (size_t)wgrad3_passes(cin, cout, K) : 0;
    const size_t bytes = (size_t)K * cin * cout * sizeof(float) + passes * sizeof(int);
    return (bytes + 255) & ~(size_t)255;
}

extern "C" int vc_conv_wgrad_tc(const void* in_bf16, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out,
                                int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag,
                                vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK_TC && dw, "bad arguments");
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("tensor-core wgrad: unsupported channels cin=%d cout=%d", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) {
        VC_CUDA(cudaMemsetAsync(dw, 0, (size_t)K * cin * cout * 4, stream));
        return VC_OK;
    }
    VC_CHECK_ARG(in_bf16 && dout_bf16 && nbr && ws, "null pointer");
    const size_t need = vc_conv_wgrad_tc_ws_bytes(n_out, cin, cout, K);
    if (ws_bytes < need) {
        set_error("tensor-core wgrad workspace %zu < %zu", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    // accumulate into a zeroed scratch image, then one transposing pass
    const size_t wbytes = (size_t)K * cin * cout * sizeof(float);
    VC_CUDA(cudaMemsetAsync(ws, 0, need, stream));
    // alone on its stream the kernel measured fastest with one CTA per SM for each pass (DESIGN.md section 4)
    int rc = tc3_wgrad(cin, cout, in_bf16, dout_bf16, nbr, n_out, (float*)ws, n_out, nullptr, K, err_flag, stream,
                       reinterpret_cast<int*>((char*)ws + wbytes), num_sms() * wgrad3_passes(cin, cout, K));
    if (rc) return rc;
    WgradFinTable T;
    T.n = 1;
    T.e[0].scratch = (const float*)ws; T.e[0].dw = dw; T.e[0].cin = cin; T.e[0].cout = cout; T.e[0].K = K; T.e[0].first = 0;
    T.e[0].n_part = 1;
    return wgrad_finalize(T, stream);
}

extern "C" size_t vc_conv_wgrad_tc_det_ws_bytes(int n_out, int cin, int cout, int K) {
    (void)n_out;
    const size_t passes = tc2_ch_ok(cin) && tc2_ch_ok(cout) && K >= 1 ? (size_t)wgrad3_passes(cin, cout, K) : 0;
    const size_t bytes = (size_t)WGRAD_DET_CHUNKS * K * cin * cout * sizeof(float) + passes * sizeof(int);
    return (bytes + 255) & ~(size_t)255;
}

static int wgrad_tc_det(const void* in_bf16, int in_ld, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out, int cin,
                        int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag, cudaStream_t stream) {
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK_TC && dw, "bad arguments");
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("tensor-core wgrad: unsupported channels cin=%d cout=%d", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) {
        VC_CUDA(cudaMemsetAsync(dw, 0, (size_t)K * cin * cout * 4, stream));
        return VC_OK;
    }
    VC_CHECK_ARG(in_bf16 && dout_bf16 && nbr && ws, "null pointer");
    const size_t need = vc_conv_wgrad_tc_det_ws_bytes(n_out, cin, cout, K);
    if (ws_bytes < need) {
        set_error("deterministic tensor-core wgrad workspace %zu < %zu", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    const size_t pbytes = (size_t)WGRAD_DET_CHUNKS * K * cin * cout * sizeof(float);
    VC_CUDA(cudaMemsetAsync(ws, 0, need, stream));
    int rc = tc3_wgrad(cin, cout, in_bf16, dout_bf16, nbr, n_out, (float*)ws, n_out, nullptr, K, err_flag, stream,
                       reinterpret_cast<int*>((char*)ws + pbytes), g_wgrad3_ctas > 0 ? g_wgrad3_ctas : num_sms() * wgrad3_passes(cin, cout, K), in_ld,
                       WGRAD_DET_CHUNKS);
    if (rc) return rc;
    WgradFinTable T;
    T.n = 1;
    T.e[0].scratch = (const float*)ws; T.e[0].dw = dw; T.e[0].cin = cin; T.e[0].cout = cout; T.e[0].K = K; T.e[0].first = 0;
    T.e[0].n_part = WGRAD_DET_CHUNKS;
    return wgrad_finalize(T, stream);
}

extern "C" int vc_conv_wgrad_tc_det(const void* in_bf16, const void* dout_bf16, const int32_t* nbr, float* dw, int n_out,
                                    int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag,
                                    vc_stream_t stream_) {
    return wgrad_tc_det(in_bf16, 0, dout_bf16, nbr, dw, n_out, cin, cout, K, ws, ws_bytes, err_flag, (cudaStream_t)stream_);
}

extern "C" int vc_conv_wgrad_tc_det_ld(const void* in_bf16, int in_ld, const void* dout_bf16, const int32_t* nbr, float* dw,
                                       int n_out, int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag,
                                       vc_stream_t stream_) {
    return wgrad_tc_det(in_bf16, in_ld, dout_bf16, nbr, dw, n_out, cin, cout, K, ws, ws_bytes, err_flag, (cudaStream_t)stream_);
}
