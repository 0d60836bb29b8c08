// wgmma / mbarrier helpers shared by the tensor-core kernels (conv_tc.cu, conv_tc2.cu, wgrad_tc3.cu) — sm_90a.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace vc {

static constexpr int TCM = 128;        // rows per tile (two m64 wgmma row blocks)
static constexpr int MAXK_TC = 32;
static constexpr unsigned SPIN_LIMIT = 1u << 24;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// bounded spin: a wedged pipeline must not hang the GPU (sets *err and returns false instead)
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* err) {
    uint32_t addr = smem_u32(bar), done = 0;
    for (unsigned spin = 0; spin < SPIN_LIMIT; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return true;
    }
    if (err) atomicCAS(err, 0, 0x300);
    return false;
}
// time-bounded wait (2 s of %globaltimer): used by the persistent kernels, whose roles abandon their loops on a timeout
// `code` says which wait of which kernel gave up (0x1xx persistent conv, 0x2xx persistent wgrad; the first one sticks)
__device__ __forceinline__ bool mbar_wait_t(uint64_t* bar, uint32_t parity, int* err, int code = 1) {
    uint32_t addr = smem_u32(bar), done = 0;
    unsigned long long t0 = 0;
    for (unsigned spin = 0;; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return true;
        if ((spin & 255u) == 255u) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ULL) break;
        }
    }
    if (err) atomicCAS(err, 0, code);
    return false;
}
// one non-blocking probe of a phase
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// the arrival is triggered when all cp.async operations issued so far by this thread have landed; it is one of the
// arrivals the barrier was initialised with (no increment of the pending count)
__device__ __forceinline__ void cp_async_arrive_noinc(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// linear bulk copy global -> shared through the TMA engine, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- Hopper warpgroup MMA (wgmma) ------------------------------------------------------------------------------------------
// A warpgroup (4 consecutive warps, the first a multiple of 4) issues wgmma.mma_async m64nNk16 with both operands in shared
// memory and the fp32 accumulator in registers: thread t of the warpgroup (warp w = t / 32, lane l) holds, for j < N / 2,
//   row 16 w + l / 4 + 8 ((j >> 1) & 1),  column 8 (j >> 2) + 2 (l & 3) + (j & 1)     (wg_row / wg_col)
__device__ __forceinline__ int wg_row(int j, int t) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((j >> 1) & 1); }
__device__ __forceinline__ int wg_col(int j, int t) { return 8 * (j >> 2) + 2 * (t & 3) + (j & 1); }

// GMMA shared-memory descriptor: [0,14) start >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4, [62,64) layout type
// (0 = no swizzle, 1 = 128-byte, 2 = 64-byte, 3 = 32-byte swizzle).  No swizzle, K-major: 8-row x 16-byte core matrices,
// LBO = distance between core matrices along K, SBO = along M/N.  Swizzled K-major rows of exactly one swizzle span
// (ROWB = 32 / 64 / 128 bytes): SBO = 8 ROWB between 8-row atoms, LBO unused (1), the K step of 16 elements advances the
// start address by 32 bytes.  Swizzled MN-major: LBO = distance between swizzle atoms along M/N, SBO = 8 ROWB between
// 8-row groups along K.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}
template <int ROWB>
__host__ __device__ constexpr uint32_t gmma_swz() { return ROWB == 128 ? 1u : ROWB == 64 ? 2u : 3u; }
template <int ROWB>
__device__ __forceinline__ uint64_t gmma_desc_sw(uint32_t saddr) { return gmma_desc(saddr, 16, 8 * ROWB, gmma_swz<ROWB>()); }
template <int ROWB>
__device__ __forceinline__ uint64_t gmma_desc_mn(uint32_t saddr, uint32_t lbo_bytes) {
    return gmma_desc(saddr, lbo_bytes, 8 * ROWB, gmma_swz<ROWB>());
}
// byte offset of 16-byte chunk c of row r inside such a tile (the GMMA swizzle: address bits [4,4+b) ^= bits [7,7+b))
template <int ROWB>
__host__ __device__ __forceinline__ uint32_t swz_off(int r, int c) {
    constexpr uint32_t MASK = ROWB == 128 ? 7u : ROWB == 64 ? 3u : ROWB == 32 ? 1u : 0u;
    const uint32_t off = (uint32_t)r * ROWB + (uint32_t)c * 16;
    return off ^ (((off >> 7) & MASK) << 4);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void wg_fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] B[16 x N], bf16 operands, fp32 accumulate; TA / TB = 1: operand MN-major (transposed)
template <int N, int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 16 || N == 32 || N == 64, "wgmma N");
    if constexpr (N == 16) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
            : "memory");
    } else if constexpr (N == 32) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "
            "%16, %17, p, 1, 1, %19, %20;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
              "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
            : "memory");
    } else {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
            "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
              "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
              "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
              "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB)
            : "memory");
    }
}

// up to `tries` probes inside one asm block; 1 when the phase completed
__device__ __forceinline__ uint32_t mbar_spin(uint32_t bar_addr, uint32_t parity, uint32_t tries) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p, q;\n\t.reg .u32 c;\n\t"
        "mov.u32 c, 0;\n"
        "VC_SPIN:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "@p bra VC_SPIN_DONE;\n\t"
        "add.u32 c, c, 1;\n\t"
        "setp.lt.u32 q, c, %3;\n\t"
        "@q bra VC_SPIN;\n"
        "VC_SPIN_DONE:\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar_addr), "r"(parity), "r"(tries)
        : "memory");
    return ok;
}
// time-bounded wait on a precomputed shared-window address (cold path behind mbar_spin)
__device__ __forceinline__ bool mbar_wait_t_addr(uint32_t addr, uint32_t parity, int* err, int code) {
    uint32_t done = 0;
    unsigned long long t0 = 0;
    for (unsigned spin = 0;; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return true;
        if ((spin & 255u) == 255u) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
            if (t0 == 0) t0 = t;
            else if (t - t0 > 2000000000ULL) break;
        }
    }
    if (err) atomicCAS(err, 0, code);
    return false;
}

__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// ---- weight-gradient consumers (wgrad_tc3.cu) ---------------------------------------------------------------------------
// D[(offset j, channel ci), co] += sum over rows of in[nbr[k, row], ci] * dout[row, co]: the gathered tiles and the dout tile are
// both used MN-major (the reduction runs over the rows).  A group = 128 / CI kernel offsets stacked along M; warpgroup wg
// owns M rows [64 wg, 64 wg + 64), i.e. starts 64 / CI gathered tiles into the stage.  acc[g] is group g of the pass; a group
// index only known at run time selects its accumulator through an unrolled compare (registers cannot be indexed).
// acc_in = 0: the stage's first MMA overwrites the group's accumulators instead of adding to them (a fresh sum).
template <int CI, int CO, int NKS, int MAXG, int A_BYTES>
__device__ __forceinline__ void wgrad_stage_mma(float (&acc)[MAXG][CO / 2], int g, uint32_t a_s, uint32_t b_s, uint32_t acc_in) {
#pragma unroll
    for (int gg = 0; gg < MAXG; ++gg) {
        if (gg == g) {
#pragma unroll
            for (int m = 0; m < NKS; ++m)      // 16 rows per MMA
                wgmma_bf16<CO, 1, 1>(acc[gg], gmma_desc_mn<2 * CI>(a_s + (uint32_t)(m * 32 * CI), (uint32_t)A_BYTES),
                                     gmma_desc_mn<2 * CO>(b_s + (uint32_t)(m * 32 * CO), 16u), m == 0 ? acc_in : 1u);
        }
    }
}
// adds groups [0, g_count) of this warpgroup's accumulators into scratch [K][ic][oc] (fp32 vector reductions)
template <int CI, int CO, int MAXG>
__device__ __forceinline__ void wgrad_flush(float (&acc)[MAXG][CO / 2], int wg, int t, int g_count, int k_begin, int k_count,
                                            int ic, int oc, float* scratch) {
    constexpr int GW = 128 / CI;
#pragma unroll
    for (int gg = 0; gg < MAXG; ++gg) {
        if (gg >= g_count) break;
#pragma unroll
        for (int j = 0; j < CO / 2; j += 2) {
            const int m = 64 * wg + wg_row(j, t), co = wg_col(j, t);
            const int kk = gg * GW + m / CI, ci = m % CI;
            if (kk < k_count && ci < ic && co < oc)
                red_add_v2(scratch + ((size_t)(k_begin + kk) * ic + ci) * oc + co, acc[gg][j], acc[gg][j + 1]);
        }
    }
}

__host__ __device__ constexpr int tc_pad16(int c) { return c < 16 ? 16 : c; }

}  // namespace vc
