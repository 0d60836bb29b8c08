// bf16 tensor-core sparse convolution, forward and gather dgrad — persistent gather-GEMM, wgmma, sm_90a.
//
// Output-stationary 128-row tiles, per kernel offset one [128 x C_in] x [C_in x C_out] product accumulating in fp32.
// A launch of one short-lived CTA per tile (round 1) was one wave of CTAs, each a chain of <= 27 dependent {table read ->
// gather round trip -> MMA} links on a 2-deep ring.  Here CTAs live for the whole launch, claim tiles from a counter and
// run a warp-specialised pipeline (DESIGN.md section 4 has the account).
// TWO CTAs per SM by default (<= 111 KB shared memory each; one CTA with the whole SM where a two-stage ring would not fit),
// 448 threads per CTA:
//   warps 0-7   two consumer warpgroups, one per 64-row half of the tile: wait for a ring stage, issue its wgmma.mma_async
//               (m64 x C_out x 16, accumulator in registers), release the stage once the MMAs reading it have completed
//               (wgmma.wait_group 1: the next stage's MMAs are already queued); after the tile's last stage each warpgroup
//               stores its 64 rows straight from the accumulator registers (fp32, + addend).  A launch that takes BatchNorm
//               channel sums instead sends the accumulator through a half-tile shared staging buffer to coalesced fp32
//               stores, with the sums per tile in fp32 over fixed row groups, accumulated per CTA in float64 (scheduling
//               independent), one set of atomics per CTA;
//   warp  8     tile scheduler + table loader: claims a tile, cp.async's its K x 128 slice of the neighbour table into one of
//               2-4 shared buffers one tile ahead, fixes rows beyond the (device) row count to -1 and — for the dgrad of a
//               strided conv — lists the kernel offsets that reach the tile at all (lane-parallel scan);
//   warp  9     weights: all K slices resident in shared memory for the launch (one bulk copy) when they fit beside >= 3 ring
//               stages, else one cp.async.bulk per stage with complete_tx on the stage's `full` barrier;
//   warps 10-13 gather producers: 32 rows each; a present neighbour is a 16-byte cp.async straight into the 32/64/128-byte-
//               swizzled K-major operand image, a missing one (and the padded channels of the C = 8 layers) a 16-byte zero
//               store; completion through cp.async.mbarrier.arrive.noinc per thread + one release arrive per warp.
// A ring stage holds 64 / C_in kernel offsets (16 KB of gathered rows); the ring runs ACROSS tile boundaries.
// The row count may come from device memory (n_dev): the grid is sized from a host-side capacity and every role derives
// its tile list from *n_dev, which is what makes the plan executor CUDA-graph capturable (no host read of a row count).
// Every mbarrier wait is time-bounded (2 s): a wedged pipeline stores a code in the error flag and the roles leave their loops.
// Replaces spconv `ops.indice_conv` / `indice_conv_backward` (input gradient) behind spconv_backbone.py:89,92-93,113,563-564.
// Algorithmic bytes per launch: N_in*C_in*2 + N_out*C_out*4 + P*8 + K*C_in*C_out*2;  FLOPs 2*P*C_in*C_out.
#include "bn_common.cuh"
#include "tc_common.cuh"

namespace vc {

int g_conv_bn_fused = 1;     // 1: BatchNorm + ReLU inside the forward conv (cooperative launch); 0: separate apply kernel

int num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    }
    return sms;
}

namespace {

#ifndef VC_P_GROUPS
#define VC_P_GROUPS 1            // producer groups of 8 warps; consecutive ring stages go to consecutive groups (1: two CTAs fit an SM)
#endif
constexpr int P_CONS_WARPS = 8;                                 // two consumer warpgroups
constexpr int P_CONS_THREADS = 32 * P_CONS_WARPS;
constexpr int P_WARP_LOADER = P_CONS_WARPS, P_WARP_W = P_WARP_LOADER + 1, P_WARP_PROD0 = P_WARP_W + 1;
constexpr int P_GROUPS = VC_P_GROUPS, P_PROD_WARPS = 4;
constexpr int P_THREADS = 32 * (P_WARP_PROD0 + P_GROUPS * P_PROD_WARPS);   // 448 with one group
constexpr int P_MAX_STAGES = 16;
constexpr int P_NTB = 4;                                        // neighbour-table buffers (<= 3 tiles loaded ahead)
constexpr int P_ROWS_PER_PROD = TCM / P_PROD_WARPS;             // 32
constexpr int P_W_CHUNK = 16384;                                // bytes per bulk copy of the resident weight image
constexpr int P_W_RESIDENT_MAX = 56 * 1024;
constexpr int SMEM_BUDGET = 227 * 1024 - 8192;                  // dynamic shared memory per CTA (static part: ~5.3 KB)

template <int KC, int NR>
struct PCfg {
    static constexpr int ROWB = KC * 2;                      // bytes per gathered operand row == swizzle span
    static constexpr int CPR = KC / 8;                       // 16-byte chunks per row
    static constexpr int G = 64 / KC;                        // kernel offsets per ring stage: 16 KB of gathered rows per stage
    static constexpr int A_BYTES = TCM * ROWB;               // one offset's gathered tile
    static constexpr int B_BYTES = NR * ROWB;                // one offset's weight slice
    static constexpr int STG_LD = NR + 1;                    // staging row pitch (floats)
    static constexpr int STG_BYTES = (TCM / 2) * STG_LD * 4;   // half a tile at a time (launches with BatchNorm sums only)
};

struct PArgs {
    const __nv_bfloat16* in;   // gathered operand rows, row pitch in_ld elements
    int in_c;                  // real channels of a row (8 or KC)
    int in_ld;                 // row pitch (>= in_c: the rows may be a column slice of a wider matrix)
    const unsigned char* wimg; // K swizzled [NR][KC] images
    const int32_t* nbr;        // [K][pitch]
    long long pitch;
    float* out;                // [n, out_c]
    int out_c;                 // real output channels (8 or NR)
    const float* addend;       // optional [n, out_c], may alias out
    double* bn_sums;           // optional [2, out_c]
    double* bn_part;           // optional [tiles, 2, out_c]: deterministic BN sums, one float64 partial per tile (bn_sums NULL)
    const int* n_dev;          // optional device row count (n_host is then the capacity of the buffers)
    int n_host;
    int* tile_counter;         // optional (zeroed by the caller): dynamic tile scheduling; NULL: tile = blockIdx.x + i * gridDim.x
    int K, S;
    int w_resident;            // all K weight slices stay in shared memory for the whole launch (else: streamed with the ring)
    int scan_k;                // the loader lists the kernel offsets that touch each tile (strided-conv dgrad: most do not)
    int ntb_alloc;             // neighbour-table buffers in shared memory (2 when two CTAs share an SM, else P_NTB)
    int zero_tail;             // store zeros into out's rows [count, n_host) (a static-mode input gradient)
    int* err;
    BnTail bn;                 // bn.bar != NULL: BatchNorm + ReLU after a grid-wide barrier (forward, cooperative launch)
};

#ifdef VC_TC_TRACE
// debug build only (profiles/trace_tc2.py): globaltimer stamps of CTA 0's pipeline events, 256 slots per role
// role 0 loader (table published), 1 producer leader (stage issued), 2 consumer (stage consumed), 4 consumer (tile start),
// 5 consumer (tile end), 6 misc (kernel start / roles start / end)
__device__ long long* g_trace2 = nullptr;
__device__ __forceinline__ void ptrace(long long* g_trace2, int role, int& idx) {
    if (g_trace2 != nullptr && idx < 256) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        g_trace2[role * 256 + idx] = (long long)t;
        ++idx;
    }
}
// roles 7 (producer leader) and 8 (consumer thread 0): SM-clock stamps of the phases inside one ring stage
__device__ __forceinline__ void pclock(long long* g_trace2, int role, int& idx) {
    if (g_trace2 != nullptr && idx < 256) {
        g_trace2[role * 256 + idx] = clock64();
        ++idx;
    }
}
#define P_TRACE(role, idx) ptrace(trc, role, idx)
#define P_CLOCK(role, idx) pclock(trc, role, idx)
#else
#define P_TRACE(role, idx) do { } while (0)
#define P_CLOCK(role, idx) do { } while (0)
#endif

#define P_WAIT(bar, parity, code)                                     \
    do {                                                              \
        if (!mbar_wait_t((bar), (parity), a.err, (code))) goto done;  \
    } while (0)

// Grid-wide barrier of a cooperative launch: the k-th barrier waits until the counter `bar` (zeroed before the launch) reaches
// target = k * gridDim.x.  Time-bounded like the pipeline waits: after 2 s it stores 0x160 in the error flag and the block
// gets false.
__device__ __forceinline__ bool grid_barrier(int* bar, int target, int* err, int* ok_s) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(bar, 1);
        int ok = 1;
        unsigned long long t0 = 0;
        for (unsigned spin = 0;; ++spin) {
            int v;
            asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
            if (v >= target) break;
            if ((spin & 63u) == 63u) {
                unsigned long long t;
                asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
                if (t0 == 0) {
                    t0 = t;
                } else if (t - t0 > 2000000000ULL) {
                    if (err) atomicCAS(err, 0, 0x160);
                    ok = 0;
                    break;
                }
            }
        }
        __threadfence();
        *ok_s = ok;
    }
    __syncthreads();
    return *ok_s != 0;
}

__device__ __forceinline__ void sts_zero16(uint32_t saddr) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(saddr), "r"(0u) : "memory");
}

template <int KC, int NR>
__global__ void __launch_bounds__(P_THREADS, P_GROUPS == 1 ? 2 : 1) tc_conv_persist_kernel(const PArgs a) {
    using C = PCfg<KC, NR>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int S = a.S, K = a.K;
    const bool wres = a.w_resident != 0;
    const uint32_t stage_bytes = (uint32_t)(C::G * C::A_BYTES + (wres ? 0 : C::G * C::B_BYTES));
    const uint32_t wres_bytes = wres ? (uint32_t)((K * C::B_BYTES + 1023) & ~1023) : 0u;
    unsigned char* ring = smem_raw;                                              // [S][G x A (| G x B)]
    unsigned char* wimg_s = smem_raw + (size_t)S * stage_bytes;                  // [K][B] when resident
    int* nbr_s = reinterpret_cast<int*>(wimg_s + wres_bytes);                    // [P_NTB][K][128]
    float* stg = reinterpret_cast<float*>(nbr_s + (size_t)a.ntb_alloc * K * TCM); // [64][STG_LD] (with BN sums)
    __shared__ __align__(8) uint64_t full_bar[P_MAX_STAGES];
    __shared__ __align__(8) uint64_t empty_bar[P_MAX_STAGES];
    __shared__ __align__(8) uint64_t tbl_full[P_NTB], tbl_empty[P_NTB];
    __shared__ __align__(8) uint64_t wres_bar;
    __shared__ int tile_s[P_NTB], nk_s[P_NTB];
    __shared__ int klist_s[P_NTB][MAXK_TC];
    __shared__ double red_s[2][P_CONS_THREADS];

    // the role index read through a shuffle: the compiler can then tell that the consumer branch is warp-uniform, and does not
    // serialize its wgmma instructions
    const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
#ifdef VC_TC_TRACE
    long long* const trc = blockIdx.x == 0 ? g_trace2 : nullptr;      // (read once: a stamp must not cost a global load)
#endif
    int tr = 0, tr2 = 0, tr3 = 0;      // trace cursors (debug build)
    (void)tr; (void)tr2; (void)tr3;
    if (tid == 0) P_TRACE(6, tr);

    if (tid == P_WARP_LOADER * 32) {
        for (int s = 0; s < S; ++s) {
            // every producer thread (cp.async.mbarrier.arrive.noinc: fires when its copies of the stage have landed) + one release
            // arrive per producer warp for its zero stores [+ the weight warp's expect_tx]
            mbar_init(&full_bar[s], 32 * P_PROD_WARPS + P_PROD_WARPS + (wres ? 0 : 1));
            mbar_init(&empty_bar[s], 2);                       // one arrive per consumer warpgroup
        }
        for (int b = 0; b < P_NTB; ++b) {
            mbar_init(&tbl_full[b], 1);                        // loader
            mbar_init(&tbl_empty[b], P_GROUPS * P_PROD_WARPS + P_CONS_WARPS + (wres ? 0 : 1));   // producers, consumers, weights
        }
        mbar_init(&wres_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    const int n = a.n_dev != nullptr ? min(__ldg(a.n_dev), a.n_host) : a.n_host;
    // a pipeline wait that timed out in an EARLIER launch left the (sticky) error flag set: do nothing, so that whatever went
    // wrong costs one 2-second timeout, not one per launch
    const bool dead = a.err != nullptr && *reinterpret_cast<volatile int*>(a.err) != 0;
    const int n_tiles = dead ? 0 : (n + TCM - 1) / TCM;
    // Table buffers in use == how many tiles a CTA holds claimed at once.  With dynamic scheduling a deep look-ahead
    // unbalances short launches (the first CTAs would grab every tile), so it grows with the tiles per CTA.
    int ntb = a.ntb_alloc;
    if (a.tile_counter != nullptr) {
        int d = n_tiles / (3 * (int)gridDim.x);
        d = d < 1 ? 1 : (d > a.ntb_alloc - 1 ? a.ntb_alloc - 1 : d);
        ntb = d + 1;
    }
    __syncthreads();
    if (tid == 0) P_TRACE(6, tr);
    // consumer threads: BatchNorm partial sums over all tiles of this CTA.  Every tile contributes fp32 partials over fixed
    // row groups, summed in float64 — the result does not depend on which CTA processed which tile (dynamic scheduling)
    double bs = 0.0, bq = 0.0;

    if (warp == P_WARP_LOADER) {
        // ------------------------------------------------------------ tile scheduler + neighbour-table loader
        // Table slices travel global -> shared with cp.async (no register staging), ntb - 1 tiles in flight: producers never
        // wait for global memory, and the loader's own latency (DRAM-cold table rows: 1-1.5 us under load) is pipelined
        // across tiles.
        const bool vec_ok = (reinterpret_cast<uintptr_t>(a.nbr) & 15u) == 0 && (a.pitch & 3) == 0;
        const int lag = ntb - 1;
        int tq0 = -1, tq1 = -1, tq2 = -1, tq3 = -1;      // tiles of the last four iterations (it & 3)
        bool stop = false;
        int claimed = 0;
        for (int it = 0;; ++it) {
            const int tb = it % ntb;
            int tile = -1;
            if (!stop) {
                if (a.tile_counter != nullptr) {
                    tile = lane == 0 ? atomicAdd(a.tile_counter, 1) : 0;
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
            switch (it & 3) {
                case 0: tq0 = tile; break;
                case 1: tq1 = tile; break;
                case 2: tq2 = tile; break;
                default: tq3 = tile; break;
            }
            if (it >= ntb) P_WAIT(&tbl_empty[tb], (uint32_t)(((it / ntb) - 1) & 1), 0x101);
            if (tile >= 0) {
                int* dst = nbr_s + (size_t)tb * K * TCM;
                const int base = tile * TCM;
                if (vec_ok && (long long)base + TCM <= a.pitch) {
                    uint32_t d = smem_u32(dst) + lane * 16;
                    const int32_t* sp = a.nbr + base + lane * 4;
                    for (int k = 0; k < K; ++k, d += TCM * 4, sp += a.pitch) cp_async16_s(d, sp, true);
                } else {
                    for (int k = 0; k < K; ++k) {
#pragma unroll
                        for (int q = 0; q < 4; ++q) {
                            const int row = base + q * 32 + lane;
                            if (row < n) {
                                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(dst + k * TCM + q * 32 + lane)),
                                             "l"(a.nbr + (size_t)k * a.pitch + row));
                            } else {
                                dst[k * TCM + q * 32 + lane] = -1;
                            }
                        }
                    }
                }
            }
            cp_async_commit();
            if (it >= lag) {
                const int pi = it - lag;             // publish the table issued `lag` iterations ago
                if (lag == 3) cp_async_wait<3>(); else if (lag == 2) cp_async_wait<2>(); else cp_async_wait<1>();
                __syncwarp();
                const int ptb = pi % ntb;
                const int ptile = (pi & 3) == 0 ? tq0 : (pi & 3) == 1 ? tq1 : (pi & 3) == 2 ? tq2 : tq3;
                if (ptile >= 0 && ptile * TCM + TCM > n) {
                    // rows beyond the count (static mode / last tile): no neighbour
                    int* dst = nbr_s + (size_t)ptb * K * TCM;
                    const int r0 = ptile * TCM + lane * 4;
                    for (int k = 0; k < K; ++k) {
                        int4 v = reinterpret_cast<const int4*>(dst + k * TCM)[lane];
                        if (r0 + 0 >= n) v.x = -1;
                        if (r0 + 1 >= n) v.y = -1;
                        if (r0 + 2 >= n) v.z = -1;
                        if (r0 + 3 >= n) v.w = -1;
                        reinterpret_cast<int4*>(dst + k * TCM)[lane] = v;
                    }
                }
                if (ptile >= 0) {
                    // the kernel offsets the tile's stages walk.  By default all of them (a slice without a single neighbour costs
                    // 128 zero stores and one MMA group, less than finding out); with scan_k — the dgrad of a strided conv,
                    // where a tile's rows share their (z, y) parity and 3 of 4 offsets cannot reach any output — lane k ORs
                    // table row k (rotated 16-byte chunks: conflict free) and the empty offsets are dropped
                    unsigned km = K >= 32 ? 0xffffffffu : ((1u << K) - 1u);
                    if (a.scan_k) {
                        __syncwarp();
                        bool any = false;
                        if (lane < K) {
                            const int4* row = reinterpret_cast<const int4*>(nbr_s + (size_t)ptb * K * TCM + (size_t)lane * TCM);
#pragma unroll 4
                            for (int j = 0; j < 32; ++j) {
                                const int4 v = row[(j + lane) & 31];
                                any |= (v.x & v.y & v.z & v.w) >= 0;      // some entry without the sign bit
                            }
                        }
                        km = __ballot_sync(0xffffffffu, any);
                    }
                    if (a.scan_k && (km >> lane & 1u)) klist_s[ptb][__popc(km & ((1u << lane) - 1u))] = lane;
                    if (lane == 0) nk_s[ptb] = __popc(km);
                }
                if (lane == 0) tile_s[ptb] = ptile;
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&tbl_full[ptb]);
                    P_TRACE(0, tr);
                }
                if (ptile < 0) break;
            }
        }
    } else if (warp >= P_WARP_PROD0) {
        // ------------------------------------------------------------ gather producers
        const int grp = (warp - P_WARP_PROD0) / P_PROD_WARPS, pw = (warp - P_WARP_PROD0) % P_PROD_WARPS;
        constexpr int CW = C::CPR < 4 ? C::CPR : 4;         // chunks of one row handled by adjacent lanes (full sectors)
        constexpr int RPI = 32 / CW;                        // rows per warp instruction
        constexpr int NIT = P_ROWS_PER_PROD / RPI;          // row groups per offset and warp
        constexpr int NCG = C::CPR / CW;                    // chunk groups per row
        static_assert(P_ROWS_PER_PROD % RPI == 0, "producer rows must be a multiple of the rows per instruction");
        const int c_sub = lane % CW, r_sub = lane / CW;
        int rows[NIT];
        uint32_t dst_off[NIT][NCG];
        bool ch_ok[NCG];
#pragma unroll
        for (int i = 0; i < NIT; ++i) {
            rows[i] = pw * P_ROWS_PER_PROD + i * RPI + r_sub;
#pragma unroll
            for (int cg = 0; cg < NCG; ++cg) dst_off[i][cg] = swz_off<C::ROWB>(rows[i], cg * CW + c_sub);
        }
#pragma unroll
        for (int cg = 0; cg < NCG; ++cg) ch_ok[cg] = (cg * CW + c_sub) * 8 < a.in_c;
        const uint32_t ring_s = smem_u32(ring);
        const bool leader = grp == 0 && pw == 0 && lane == 0;
        (void)leader;
        int s = 0, wr = 0;     // ring slot and wrap count of the NEXT stage in sequence (all groups count every stage)
        int turn = 0;          // whose stage it is: group `turn`
        // Completion: every stage is signalled on its own `full` barrier as soon as it is issued (hardware-tracked cp.async
        // arrivals), never later, so a producer that blocks on a barrier holds no unsignalled stage.
        for (int it = 0;; ++it) {
            const int tb = it % ntb;
            P_WAIT(&tbl_full[tb], (uint32_t)((it / ntb) & 1), 0x111);
            if (tile_s[tb] < 0) break;
            const int* tbl = nbr_s + (size_t)tb * K * TCM;
            const int nk = nk_s[tb];
            for (int t0 = 0; t0 < nk; t0 += C::G) {
                if (turn == grp) {
                    if (leader) P_CLOCK(7, tr3);                                  // phase 0: stage loop top
                    const int cnt = min(C::G, nk - t0);
                    int src[C::G][NIT];
#pragma unroll
                    for (int g = 0; g < C::G; ++g) {
#pragma unroll
                        const int kk = g < cnt ? (a.scan_k ? klist_s[tb][t0 + g] : t0 + g) : 0;
                        for (int i = 0; i < NIT; ++i) src[g][i] = g < cnt ? tbl[kk * TCM + rows[i]] : -1;
                    }
                    if (wr > 0) P_WAIT(&empty_bar[s], (uint32_t)((wr - 1) & 1), 0x112);
                    if (leader) P_CLOCK(7, tr3);                                  // phase 1: ring slot free
                    const uint32_t st_s = ring_s + (uint32_t)s * stage_bytes;
#pragma unroll
                    for (int g = 0; g < C::G; ++g) {
                        if (g < cnt) {
                            const uint32_t a_s = st_s + (uint32_t)g * C::A_BYTES;
#pragma unroll
                            for (int i = 0; i < NIT; ++i) {
                                const bool v = src[g][i] >= 0;
                                const __nv_bfloat16* srow = a.in + (size_t)(v ? src[g][i] : 0) * a.in_ld + c_sub * 8;
#pragma unroll
                                for (int cg = 0; cg < NCG; ++cg) {
                                    // a missing neighbour costs a shared-memory zero store, not a zero-fill cp.async
                                    if (v && ch_ok[cg]) cp_async16_s(a_s + dst_off[i][cg], srow + cg * CW * 8, true);
                                    else sts_zero16(a_s + dst_off[i][cg]);
                                }
                            }
                        }
                    }
                    if (leader) P_CLOCK(7, tr3);                                  // phase 2: copies issued
                    cp_async_arrive_noinc(&full_bar[s]);       // fires when this thread's copies of the stage have landed
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&full_bar[s]);  // release: publishes the warp's zero stores
                    if (leader) P_CLOCK(7, tr3);                                  // phase 3: stage signalled
                    if (leader) P_TRACE(1, tr);
                }
                if (++turn == P_GROUPS) turn = 0;
                if (++s == S) {
                    s = 0;
                    ++wr;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&tbl_empty[tb]);
        }
    } else if (warp == P_WARP_W) {
        // ------------------------------------------------------------ weight slices (TMA engine, linear bulk copies)
        if (wres) {
            if (lane == 0) {
                const uint32_t total = (uint32_t)(K * C::B_BYTES);
                mbar_expect_tx(&wres_bar, total);
                for (uint32_t off = 0; off < total; off += P_W_CHUNK)
                    bulk_g2s(smem_u32(wimg_s) + off, a.wimg + off, min((uint32_t)P_W_CHUNK, total - off), &wres_bar);
            }
        } else {
            int s = 0, wr = 0;
            for (int it = 0;; ++it) {
                const int tb = it % ntb;
                P_WAIT(&tbl_full[tb], (uint32_t)((it / ntb) & 1), 0x121);
                if (tile_s[tb] < 0) break;
                const int nk = nk_s[tb];
                int kl = lane < nk ? (a.scan_k ? klist_s[tb][lane] : lane) : 0;      // lane j: the j-th offset of the tile
                __syncwarp();
                if (lane == 0) mbar_arrive(&tbl_empty[tb]);
                for (int t0 = 0; t0 < nk; t0 += C::G) {
                    const int cnt = min(C::G, nk - t0);
                    if (wr > 0) P_WAIT(&empty_bar[s], (uint32_t)((wr - 1) & 1), 0x122);
                    if (lane == 0) mbar_expect_tx(&full_bar[s], (uint32_t)(cnt * C::B_BYTES));
                    __syncwarp();
                    if (lane >= t0 && lane < t0 + cnt)
                        bulk_g2s(smem_u32(ring) + (uint32_t)s * stage_bytes + C::G * C::A_BYTES + (uint32_t)(lane - t0) * C::B_BYTES,
                                 a.wimg + (size_t)kl * C::B_BYTES, (uint32_t)C::B_BYTES, &full_bar[s]);
                    __syncwarp();
                    if (++s == S) {
                        s = 0;
                        ++wr;
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------ consumers (warpgroup h: rows [64 h, 64 h + 64) of the tile)
        const int wg = warp >> 2, t = tid & 127;
        const int e = tid;                       // 0..255
        const int oc = a.out_c;
        const int ch = e % oc, rg = e / oc, n_rg = P_CONS_THREADS / oc;
        const uint32_t full0 = smem_u32(&full_bar[0]);
        const uint32_t ring_a = smem_u32(ring), wimg_a = smem_u32(wimg_s);
        const uint32_t a_half = (uint32_t)(wg * 64 * C::ROWB);
        float acc[NR / 2];
#pragma unroll
        for (int j = 0; j < NR / 2; ++j) acc[j] = 0.f;
        int s = 0;
        uint32_t ph = 0;
        bool w_ready = !wres;
        for (int it = 0;; ++it) {
            const int tb = it % ntb;
            P_WAIT(&tbl_full[tb], (uint32_t)((it / ntb) & 1), 0x141);
            const int tile = tile_s[tb];
            if (tile < 0) break;
            if (!w_ready) {
                P_WAIT(&wres_bar, 0u, 0x132);
                w_ready = true;
            }
            if (tid == 0) P_TRACE(4, tr);
            const int base = tile * TCM;
            const int nk = nk_s[tb];
            const int kl = lane < nk ? (a.scan_k ? klist_s[tb][lane] : lane) : 0;      // lane j: the j-th offset of the tile
            __syncwarp();
            if (lane == 0) mbar_arrive(&tbl_empty[tb]);
            int prev = -1;                       // ring slot whose MMAs may still be in flight
            for (int t0 = 0; t0 < nk; t0 += C::G) {
                const int cnt = min(C::G, nk - t0);
                if (tid == 0) P_CLOCK(8, tr3);                                        // phase 0: before the wait
                if (!mbar_spin(full0 + 8u * s, ph, 4096u) && !mbar_wait_t_addr(full0 + 8u * s, ph, a.err, 0x134)) goto done;
                if (tid == 0) P_CLOCK(8, tr3);                                        // phase 1: stage landed
                fence_async_smem();     // generic-proxy (cp.async, st.shared) writes -> visible to the tensor core's async proxy
                wg_fence();
                const uint32_t st_s = ring_a + (uint32_t)s * stage_bytes;
#pragma unroll
                for (int g = 0; g < C::G; ++g) {
                    if (g < cnt) {
                        const int kk = a.scan_k ? __shfl_sync(0xffffffffu, kl, t0 + g) : t0 + g;
                        const uint32_t a_s = st_s + (uint32_t)(g * C::A_BYTES) + a_half;
                        const uint32_t b_s = wres ? wimg_a + (uint32_t)(kk * C::B_BYTES)
                                                  : st_s + (uint32_t)(C::G * C::A_BYTES + g * C::B_BYTES);
#pragma unroll
                        for (int m = 0; m < KC / 16; ++m)
                            wgmma_bf16<NR, 0, 0>(acc, gmma_desc_sw<C::ROWB>(a_s + 32u * m), gmma_desc_sw<C::ROWB>(b_s + 32u * m),
                                                 (t0 > 0 || g > 0 || m > 0) ? 1u : 0u);
                    }
                }
                wg_commit();
                wg_wait<1>();                    // the previous stage's MMAs have completed: release its ring slot
                if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
                if (tid == 0) {
                    P_CLOCK(8, tr3);                                                  // phase 2: MMAs issued
                    P_TRACE(2, tr);
                }
                prev = s;
                if (++s == S) {
                    s = 0;
                    ph ^= 1u;
                }
            }
            wg_wait<0>();
            wg_fence_acc(acc);
            if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
            const bool empty_tile = nk == 0;
            if (a.bn_sums == nullptr && a.bn_part == nullptr) {
                // no BatchNorm sums: each warpgroup stores its own 64 rows straight from the accumulators, two adjacent columns
                // per float2 (wg_col); the four lanes of a row cover 32 contiguous bytes, one sector.  The addend is loaded
                // first (independent loads, all in flight together); the same element is read and written by this thread
                // only, so `addend` may alias `out`.  No shared memory, and the two warpgroups do not wait for each other
                const int r0 = base + wg * 64 + wg_row(0, t);       // this thread's rows: r0 and r0 + 8
                const bool ok0 = r0 < n, ok1 = r0 + 8 < n;
                if (empty_tile) {        // (the registers still hold the last tile)
#pragma unroll
                    for (int j = 0; j < NR / 2; ++j) acc[j] = 0.f;
                }
                if (a.addend != nullptr) {
#pragma unroll
                    for (int j = 0; j < NR / 2; j += 2) {
                        const int c = wg_col(j, t);
                        if (((j & 2) ? ok1 : ok0) && c < oc) {
                            const float2 w = *reinterpret_cast<const float2*>(a.addend + (size_t)(r0 + (j & 2) * 4) * oc + c);
                            acc[j] += w.x;
                            acc[j + 1] += w.y;
                        }
                    }
                }
#pragma unroll
                for (int j = 0; j < NR / 2; j += 2) {
                    const int c = wg_col(j, t);
                    if (((j & 2) ? ok1 : ok0) && c < oc)
                        *reinterpret_cast<float2*>(a.out + (size_t)(r0 + (j & 2) * 4) * oc + c) = make_float2(acc[j], acc[j + 1]);
                }
                if (tid == 0) P_TRACE(5, tr2);
                continue;
            }
            // two halves of 64 rows through a [64][NR + 1] staging buffer (half the shared memory of a full-tile buffer: what
            // lets two CTAs share an SM): the warpgroup owning the half unloads its accumulator, then all 8 warps store it
            const int oc4 = oc >> 2;
#pragma unroll 1
            for (int half = 0; half < 2; ++half) {
                if (wg == half) {
#pragma unroll
                    for (int j = 0; j < NR / 2; ++j) {
                        const int c = wg_col(j, t);
                        if (c < oc) stg[wg_row(j, t) * C::STG_LD + c] = empty_tile ? 0.f : acc[j];
                    }
                }
                named_bar_sync(1, P_CONS_THREADS);
                const int hbase = base + half * 64;
                // coalesced fp32 stores: consecutive threads -> consecutive float4 of the [64, out_c] half tile
                for (int q = e; q < 64 * oc4; q += P_CONS_THREADS) {
                    const int rr = q / oc4, c4 = q % oc4;
                    if (hbase + rr < n) {
                        const float* sp = stg + rr * C::STG_LD + c4 * 4;
                        float4 v = make_float4(sp[0], sp[1], sp[2], sp[3]);
                        const size_t o = (size_t)(hbase + rr) * oc + c4 * 4;
                        if (a.addend != nullptr) {      // same element read and written by this thread only: aliasing `out` is safe
                            const float4 w = *reinterpret_cast<const float4*>(a.addend + o);
                            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
                        }
                        *reinterpret_cast<float4*>(a.out + o) = v;
                    }
                }
                if (a.bn_sums != nullptr || a.bn_part != nullptr) {
                    const int rows_valid = max(0, min(64, n - hbase));
                    float ts = 0.f, tq = 0.f;
                    for (int rr = rg; rr < rows_valid; rr += n_rg) {
                        const float x = stg[rr * C::STG_LD + ch];
                        ts += x;
                        tq = fmaf(x, x, tq);
                    }
                    bs += (double)ts;
                    bq += (double)tq;
                }
                named_bar_sync(1, P_CONS_THREADS);
            }
            if (a.bn_part != nullptr) {
                // deterministic mode: this tile's sums (row groups added in order) to its own slot; the caller adds the
                // tiles in tile order (bn_sums_reduce_dev)
                red_s[0][e] = bs;
                red_s[1][e] = bq;
                bs = bq = 0.0;
                named_bar_sync(1, P_CONS_THREADS);
                if (e < 2 * oc) {
                    const int which = e / oc, c = e % oc;
                    double v = 0.0;
                    for (int g = 0; g < n_rg; ++g) v += red_s[which][g * oc + c];
                    a.bn_part[((size_t)tile * 2 + which) * oc + c] = v;
                }
                named_bar_sync(1, P_CONS_THREADS);
            }
            if (tid == 0) P_TRACE(5, tr2);
        }
    }
done:
    cp_async_wait<0>();
    if (warp < P_CONS_WARPS && a.bn_sums != nullptr) {
        // (after a pipeline timeout the sums are garbage like everything else; the error flag says so)
        const int e = tid, oc = a.out_c, n_rg = P_CONS_THREADS / oc;
        red_s[0][e] = bs;
        red_s[1][e] = bq;
        named_bar_sync(2, P_CONS_THREADS);
        if (e < 2 * oc) {
            const int which = e / oc, c = e % oc;
            double v = 0.0;
            for (int g = 0; g < n_rg; ++g) v += red_s[which][g * oc + c];
            atomicAdd(a.bn_sums + which * oc + c, v);
        }
    }
    if (wres && warp == P_WARP_W && lane == 0) {
        // a CTA that was handed no tile must still see its weight copy land before it exits (the copy targets its smem)
        mbar_wait_t(&wres_bar, 0u, a.err, 0x150);
    }
    if (a.zero_tail) {   // (the tiles store rows below the count only)
        float4* o4 = reinterpret_cast<float4*>(a.out);
        const size_t c4 = a.out_c / 4;
        for (size_t i = (size_t)n * c4 + (size_t)blockIdx.x * blockDim.x + tid; i < (size_t)a.n_host * c4; i += (size_t)gridDim.x * blockDim.x)
            o4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    if (a.bn.bar == nullptr) return;

    // ---------------------------------------------------------------- fused BatchNorm + ReLU (bn_apply_relu_kernel's work)
    // Once every CTA has stored its tiles and added its channel sums, the whole output is read back and normalised,
    // grid-stride over float4 like the apply kernel: the layer's fp32 output (<= 20 MB) is still in L2 whichever SM wrote it.
    __shared__ int ok_s;
    const BnTail& b = a.bn;
    const int oc = a.out_c;
    bool ok = grid_barrier(b.bar, gridDim.x, a.err, &ok_s);
    if (ok && b.training && a.bn_part != nullptr) {
        // deterministic mode: the tile partials in tile order (bn_sums_reduce_kernel's arithmetic), one column per CTA
        const int n_parts = (n + TCM - 1) / TCM;
        for (int j = blockIdx.x; j < 2 * oc; j += gridDim.x) {
            const double v = bn_sums_column(a.bn_part, n_parts, oc, j, red_s[0]);
            if (tid == 0) b.sums[j] = v;
        }
        ok = grid_barrier(b.bar, 2 * gridDim.x, a.err, &ok_s);
    }
    if (!ok) return;
    // scale / shift in the dead operand ring (>= 2 x 16 KB; a launch without BN sums, e.g. an eval-mode BN, has no staging
    // buffer), whose last accesses were the async proxy's (bulk copies, wgmma reads)
    float* sc_s = reinterpret_cast<float*>(ring);
    float* sh_s = sc_s + oc;
    fence_async_smem();
    if (tid < oc)
        bn_channel(b.training ? __ldcg(b.sums + tid) : 0.0, b.training ? __ldcg(b.sums + oc + tid) : 0.0, tid, oc, n, b.gamma, b.beta,
                   b.running_mean, b.running_var, b.momentum, b.eps, b.training, sc_s, sh_s, blockIdx.x == 0, b.stats);
    if (b.training && blockIdx.x == 0 && tid == 0 && b.nbt != nullptr) *b.nbt += 1;
    __syncthreads();
    static_assert(P_THREADS % 16 == 0, "the fused apply keeps each thread on one channel group (c / 4 <= 16)");
    const int c4 = oc >> 2;
    const size_t n4 = (size_t)n * c4, stride = (size_t)gridDim.x * P_THREADS;
    const size_t i0 = (size_t)blockIdx.x * P_THREADS + tid;
    const int cg = (int)(i0 % c4);
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        sc[j] = sc_s[cg * 4 + j];
        sh[j] = sh_s[cg * 4 + j];
    }
    const float4* x4 = reinterpret_cast<const float4*>(a.out);
    float4* y4 = reinterpret_cast<float4*>(b.y);
    uint2* yb = reinterpret_cast<uint2*>(b.yb);
    const int y_ld4 = b.y_ld >> 2, yb_ld4 = b.yb_ld >> 2;
    for (size_t i = i0; i < n4; i += stride) {
        const float4 v = bn_relu4(__ldcg(x4 + i), sc, sh, 1);     // (written by other CTAs of this grid: not through L1)
        const size_t r = i / c4;
        if (y4 != nullptr) y4[r * y_ld4 + cg] = v;
        if (yb != nullptr) yb[r * yb_ld4 + cg] = pack_bf16x4(v);
    }
    if (b.tail_zero) {
        const size_t t4 = (size_t)a.n_host * c4;
        for (size_t i = n4 + i0; i < t4; i += stride) {
            const size_t r = i / c4;
            if (y4 != nullptr) y4[r * y_ld4 + cg] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (yb != nullptr) yb[r * yb_ld4 + cg] = make_uint2(0u, 0u);
        }
    }
}

// weight images for the kernel above: per offset k a [NRp rows][KCp] bf16 matrix, K-major, rows = one swizzle span,
// zero padded to NRp / KCp = max(16, .)
//   mode 0 (forward): B[n=co][kk=ci] = w[co][k][ci]
//   mode 1 (dgrad)  : B[n=ci][kk=co] = w[co][k'][ci],  k' = mirror ? K-1-k : k
template <int ROWB>
__device__ __forceinline__ size_t img_off(int k, int n, int kk, int NRp) {
    return (size_t)k * NRp * ROWB + swz_off<ROWB>(n, kk >> 3) + (size_t)(kk & 7) * 2;
}

#ifndef VC_P_MIN_STAGES2
#define VC_P_MIN_STAGES2 2       // two CTAs per SM are used when each still gets a ring of at least this many stages
#endif
int g_p_ctas = 0;                // 0: automatic; 1 / 2: forced CTAs per SM (vc_conv_tc2_config, A/B runs)

struct PPlan {
    int S, resident, ntb;
    size_t smem;
};

// shared-memory plan of one CTA under a budget: weights resident if they fit beside a ring of >= min_stages, else streamed
// (staged: the launch takes BatchNorm sums, whose epilogue needs the staging buffer)
template <int KC, int NR>
bool plan_smem(int K, size_t budget, int ntb, size_t resident_max, int min_stages, bool staged, PPlan& p) {
    using C = PCfg<KC, NR>;
    const size_t fixed = (size_t)ntb * K * TCM * 4 + (staged ? C::STG_BYTES : 0);
    const size_t wbytes = ((size_t)K * C::B_BYTES + 1023) & ~(size_t)1023;
    if (fixed + (size_t)min_stages * C::G * C::A_BYTES > budget) return false;
    int s_res = 0;
    if (wbytes <= resident_max && fixed + wbytes < budget) s_res = (int)((budget - fixed - wbytes) / ((size_t)C::G * C::A_BYTES));
    const size_t stage_str = (size_t)C::G * (C::A_BYTES + C::B_BYTES);
    int s_str = (int)((budget - fixed) / stage_str);
    const bool resident = s_res >= min_stages && s_res >= s_str - 1;
    int S = resident ? s_res : s_str;
    if (S < min_stages) return false;
    if (S > P_MAX_STAGES) S = P_MAX_STAGES;
    p.S = S;
    p.resident = resident ? 1 : 0;
    p.ntb = ntb;
    p.smem = (size_t)S * (resident ? (size_t)C::G * C::A_BYTES : stage_str) + (resident ? wbytes : 0) + fixed;
    return true;
}

// Two CTAs per SM (half the shared memory each, 2 table buffers) when the ring still has VC_P_MIN_STAGES2 stages: two
// independent pipelines per SM (each a serial chain of barrier wait -> MMA issue -> release per stage) and room for CTAs
// of another stream's kernel.  Otherwise one CTA with the whole SM.
template <int KC, int NR>
int choose_plan(int K, bool staged, PPlan& p, int& ctas) {
    ctas = 1;
    const size_t budget2 = (size_t)(227 * 1024) / 2 - 7 * 1024;      // static shared memory + 1 KB/CTA reserved by the driver
    if (P_GROUPS == 1 && g_p_ctas != 1 && plan_smem<KC, NR>(K, budget2, 2, 28 * 1024, VC_P_MIN_STAGES2, staged, p)) {
        ctas = 2;
    } else if (!plan_smem<KC, NR>(K, SMEM_BUDGET, P_NTB, P_W_RESIDENT_MAX, 2, staged, p)) {
        set_error("tensor-core conv: no room for the operand ring (K=%d, %d->%d)", K, KC, NR);
        return VC_ERR_UNSUPPORTED;
    }
    return VC_OK;
}

template <int KC, int NR>
int launch_persist(const PArgs& a0, int n_cap, cudaStream_t stream, bool* bn_done, bool coop2) {
    PArgs a = a0;
    PPlan p;
    int ctas = 1;
    if (const int rc = choose_plan<KC, NR>(a.K, a.bn_sums != nullptr || a.bn_part != nullptr, p, ctas)) return rc;
    a.S = p.S;
    a.w_resident = p.resident;
    a.ntb_alloc = p.ntb;
    auto kern = tc_conv_persist_kernel<KC, NR>;
    static bool attr_done = false;            // per instantiation
    if (!attr_done) {
        VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
        attr_done = true;
    }
    const int tiles = cdiv(n_cap, TCM);
    const int slots = ctas * num_sms();
    const int grid = tiles < slots ? (tiles < 1 ? 1 : tiles) : slots;
    if (a.bn.bar != nullptr) {
        // The grid-wide barrier needs every CTA resident at once: a cooperative launch, which starts only when ALL its CTAs fit.
        // At two CTAs per SM that means waiting until the index stream's rulebook kernels have left the SMs (measured: 0.14 ms
        // per step SLOWER than the separate apply kernel); at one CTA per SM the grid fits beside them and the step gets
        // 0.15 ms faster (DESIGN.md section 8).  Same shared-memory plan, half the CTAs.  Running the whole index phase
        // before the forward instead, so that the grid could take both CTAs of each SM, was slower still (DESIGN.md
        // section 8, item 3) until the index work was batched: with no index kernel beside it (coop2, the executor's static
        // mode, index phase first) the grid takes both.  vc_conv_tc2_config(2) forces the two-CTA grid (tests, A/B runs).
        const int cgrid = (g_p_ctas == 2 || coop2 || grid < num_sms()) ? grid : num_sms();
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(cgrid);
        cfg.blockDim = dim3(P_THREADS);
        cfg.dynamicSmemBytes = p.smem;
        cfg.stream = stream;
        cudaLaunchAttribute at{};
        at.id = cudaLaunchAttributeCooperative;
        at.val.cooperative = 1;
        cfg.attrs = &at;
        cfg.numAttrs = 1;
        if (cudaLaunchKernelEx(&cfg, kern, a) == cudaSuccess) {
            count_launch();
            *bn_done = true;
            return VC_OK;
        }
        // (a device / driver configuration that refuses it: the conv alone, the caller applies BN, for good)
        cudaGetLastError();
        g_conv_bn_fused = 0;
        a.bn = BnTail{};
    }
    kern<<<dim3(grid), dim3(P_THREADS), p.smem, stream>>>(a);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

}  // namespace

__global__ void __launch_bounds__(256) prep_weights_tc_batch_kernel(TcPrepTable t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.total) return;
    int lo = 0, hi = t.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t.e[mid].first <= i) lo = mid; else hi = mid - 1;
    }
    const TcPrepEntry& e = t.e[lo];
    const int j = i - e.first;
    const int cin = e.cin, cout = e.cout, K = e.K;
    const int NRr = e.mode == 0 ? cout : cin, KCc = e.mode == 0 ? cin : cout;     // real dims
    const int NRp = e.layout ? tc_pad16(NRr) : NRr, KCp = e.layout ? tc_pad16(KCc) : KCc;
    const int kk = j % KCp, n = (j / KCp) % NRp, k = j / (KCp * NRp);
    float v = 0.f;
    if (n < NRr && kk < KCc) {
        if (e.mode == 0) {
            v = e.w[((size_t)n * K + k) * cin + kk];
        } else {
            const int ks = e.mirror ? (K - 1 - k) : k;
            v = e.w[((size_t)kk * K + ks) * cin + n];
        }
    }
    const __nv_bfloat16 b = __float2bfloat16_rn(v);
    if (e.layout == 0) {      // 8-row x 16-byte core matrices, no swizzle (tc_scatter_kernel)
        const size_t off = (size_t)k * NRr * KCc + ((size_t)((n >> 3) * (KCc >> 3) + (kk >> 3)) * 64) + (n & 7) * 8 + (kk & 7);
        reinterpret_cast<__nv_bfloat16*>(e.img)[off] = b;
    } else {
        unsigned char* p = reinterpret_cast<unsigned char*>(e.img);
        const size_t off = KCp == 64 ? img_off<128>(k, n, kk, NRp) : KCp == 32 ? img_off<64>(k, n, kk, NRp) : img_off<32>(k, n, kk, NRp);
        *reinterpret_cast<__nv_bfloat16*>(p + off) = b;
    }
}

size_t tc_image_bytes(int cin, int cout, int K, int layout) {
    return layout ? (size_t)K * tc_pad16(cin) * tc_pad16(cout) * 2 : (size_t)K * cin * cout * 2;
}

int tc_prep_images(TcPrepTable& t, cudaStream_t stream) {
    if (t.n == 0) return VC_OK;
    int total = 0;
    for (int i = 0; i < t.n; ++i) {
        t.e[i].first = total;
        total += (int)(tc_image_bytes(t.e[i].cin, t.e[i].cout, t.e[i].K, t.e[i].layout) / 2);
    }
    t.total = total;
    prep_weights_tc_batch_kernel<<<cdiv(total, 256), 256, 0, stream>>>(t);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

bool tc2_ch_ok(int c) { return c == 8 || c == 16 || c == 32 || c == 64; }

// kc = channels of the gathered operand rows (reduction), nr = channels of the result; wimg = K swizzled images
// (layout 1).  n_dev (optional) overrides n_rows on the device; n_rows is then the capacity the grid is sized for.
int tc2_conv(int kc, int nr, const void* in_bf16, const void* wimg, const int32_t* nbr, long long pitch, float* out,
             int n_rows, const int* n_dev, int K, double* bn_sums, int* err, cudaStream_t stream, const float* addend,
             int* tile_counter, int flags, int in_ld, double* bn_part, const BnTail* bn, bool* bn_done) {
    if (bn_done != nullptr) *bn_done = false;
    if (n_rows == 0) return VC_OK;
    if (!tc2_ch_ok(kc) || !tc2_ch_ok(nr) || K < 1 || K > MAXK_TC) {
        set_error("tensor-core conv: unsupported shape (%d -> %d channels, K=%d)", kc, nr, K);
        return VC_ERR_UNSUPPORTED;
    }
    PArgs a;
    if (in_ld == 0) in_ld = kc;
    if (in_ld < kc || in_ld % 8 != 0) {
        set_error("tensor-core conv: row pitch %d for %d channels", in_ld, kc);
        return VC_ERR_INVALID;
    }
    a.in = (const __nv_bfloat16*)in_bf16; a.in_c = kc; a.in_ld = in_ld; a.wimg = (const unsigned char*)wimg; a.nbr = nbr; a.pitch = pitch;
    a.out = out; a.out_c = nr; a.addend = addend; a.bn_sums = bn_part ? nullptr : bn_sums; a.bn_part = bn_part; a.n_dev = n_dev; a.n_host = n_rows; a.tile_counter = tile_counter;
    a.K = K; a.S = 0; a.w_resident = 0; a.ntb_alloc = P_NTB; a.scan_k = flags & 1; a.zero_tail = n_dev != nullptr && (flags & 4);
    a.err = err;
    a.bn = BnTail{};
    bool done_dummy = false;
    if (bn != nullptr && g_conv_bn_fused) {
        if (!bn->bar || !bn->stats || !bn->gamma || !bn->beta || !bn->running_mean || !bn->running_var || (!bn->y && !bn->yb) ||
            (bn->training && !bn->sums) || bn->y_ld % 4 || bn->yb_ld % 4 || bn->y_ld < nr || bn->yb_ld < nr || addend) {
            set_error("tensor-core conv: bad fused BatchNorm arguments");
            return VC_ERR_INVALID;
        }
        a.bn = *bn;
    }
    if (bn_done == nullptr) bn_done = &done_dummy;
    const int kcp = tc_pad16(kc), nrp = tc_pad16(nr);
#define VC_P_CASE(A, B) \
    if (kcp == A && nrp == B) return launch_persist<A, B>(a, n_rows, stream, bn_done, (flags >> 1) & 1);
    VC_P_CASE(16, 16) VC_P_CASE(16, 32) VC_P_CASE(16, 64)
    VC_P_CASE(32, 16) VC_P_CASE(32, 32) VC_P_CASE(32, 64)
    VC_P_CASE(64, 16) VC_P_CASE(64, 32) VC_P_CASE(64, 64)
#undef VC_P_CASE
    return VC_ERR_UNSUPPORTED;
}

}  // namespace vc

#ifdef VC_TC_TRACE
extern "C" int vc_debug_set_trace2(long long* buf) {
    return cudaMemcpyToSymbol(vc::g_trace2, &buf, sizeof(buf)) == cudaSuccess ? 0 : -2;
}
#endif

extern "C" int vc_conv_tc2_config(int ctas_per_sm) {
    VC_CHECK_ARG(ctas_per_sm >= 0 && ctas_per_sm <= 2, "CTAs per SM must be 0 (automatic), 1 or 2");
    vc::g_p_ctas = ctas_per_sm;
    return VC_OK;
}

extern "C" int vc_conv_tc2_plan(int cin, int cout, int K, int bn_sums, int32_t* out) {
    VC_CHECK_ARG(out != nullptr, "null pointer");
    if (!vc::tc2_ch_ok(cin) || !vc::tc2_ch_ok(cout) || K < 1 || K > vc::MAXK_TC) {
        vc::set_error("tensor-core conv: unsupported shape (%d -> %d channels, K=%d)", cin, cout, K);
        return VC_ERR_UNSUPPORTED;
    }
    vc::PPlan p{};
    int ctas = 1, rc = VC_ERR_UNSUPPORTED;
    const int kcp = vc::tc_pad16(cin), nrp = vc::tc_pad16(cout);
#define VC_P_CASE(A, B) \
    if (kcp == A && nrp == B) rc = vc::choose_plan<A, B>(K, bn_sums != 0, p, ctas);
    VC_P_CASE(16, 16) VC_P_CASE(16, 32) VC_P_CASE(16, 64)
    VC_P_CASE(32, 16) VC_P_CASE(32, 32) VC_P_CASE(32, 64)
    VC_P_CASE(64, 16) VC_P_CASE(64, 32) VC_P_CASE(64, 64)
#undef VC_P_CASE
    if (rc) return rc;
    out[0] = p.S;
    out[1] = p.resident;
    out[2] = ctas;
    out[3] = (int32_t)p.smem;
    return VC_OK;
}

extern "C" int vc_set_conv_bn_fused(int enable) {
    vc::g_conv_bn_fused = enable ? 1 : 0;
    return VC_OK;
}

extern "C" int vc_set_tc_variant(int variant) {
    VC_CHECK_ARG(variant == 1, "tensor-core conv variant must be 1 (the persistent kernel is the only one)");
    return VC_OK;
}
