// Parameter update of the adam_onecycle / adam_cosin training step (the reference's train_utils.py:50-52 over
// fastai_optim.py:132-149 and torch.optim.Adam): gradient-norm clipping, true weight decay and Adam over every parameter
// tensor in two launches, whatever the number of tensors.
//
//   norm pass    one 4096-element chunk at a time: sum of g^2 in float64 into the chunk's own slot.  The last CTA to finish
//                (ticket) adds the slots in an order fixed by the chunk count alone, evaluates the guard, and writes the status
//                block: total norm, clip factor, `apply`, and the step's fp32 scalars (formed in float64, rounded once).
//                It advances the applied-step counter t, or the skipped counter.
//   update pass  elementwise over the same chunks, from the status block alone.
//
// A chunk's sum does not depend on which CTA took it, nor on the pointers' alignment (the vector and the scalar path give a
// thread the same elements), so the norm and everything after it are bit-identical run to run and for every grid size.
#include <math.h>

#include "common.cuh"

namespace vc {

static constexpr int OPT_THREADS = 256;
static constexpr int OPT_SLOTS_OFF = 256;   // byte offset of the chunk slots in the workspace (the ticket sits at 0)

struct OptGuards {
    const int32_t* w[VC_OPTIM_MAX_GUARDS];
    int n;
};

__device__ __forceinline__ bool opt_aligned16(const void* a) { return ((uintptr_t)a & 15) == 0; }

// elements [i, i + 4) of x, of which the first `left` exist
__device__ __forceinline__ float4 opt_load4(const float* __restrict__ x, long long i, int left, bool vec) {
    if (vec && left >= 4) return *reinterpret_cast<const float4*>(x + i);
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (left > 0) r.x = x[i];
    if (left > 1) r.y = x[i + 1];
    if (left > 2) r.z = x[i + 2];
    if (left > 3) r.w = x[i + 3];
    return r;
}
__device__ __forceinline__ void opt_store4(float* __restrict__ x, long long i, int left, bool vec, float4 r) {
    if (vec && left >= 4) {
        *reinterpret_cast<float4*>(x + i) = r;
        return;
    }
    if (left > 0) x[i] = r.x;
    if (left > 1) x[i + 1] = r.y;
    if (left > 2) x[i + 2] = r.z;
    if (left > 3) x[i + 3] = r.w;
}

__device__ __forceinline__ double opt_block_sum(double s, double* warp_s) {   // fixed tree: lanes, then warps in order
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) warp_s[threadIdx.x >> 5] = s;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < OPT_THREADS / 32; ++w) t += warp_s[w];
    __syncthreads();
    return t;   // valid in thread 0
}

__global__ void __launch_bounds__(OPT_THREADS) optim_norm_kernel(const vc_optim_seg* __restrict__ segs,
                                                                 const vc_optim_chunk* __restrict__ chunks, int n_chunks,
                                                                 double max_norm, OptGuards guards,
                                                                 const double* __restrict__ hyper, long long* counters,
                                                                 vc_optim_status* status, unsigned* ticket, double* slots) {
    __shared__ double warp_s[OPT_THREADS / 32];
    __shared__ bool last;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const vc_optim_chunk ch = chunks[c];
        const float* g = segs[ch.seg].g;
        double s = 0.0;
        if (g != nullptr) {
            const bool vec = opt_aligned16(g);
            for (int e = threadIdx.x * 4; e < ch.len; e += OPT_THREADS * 4) {
                const float4 v = opt_load4(g, ch.off + e, ch.len - e, vec);
                s += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
            }
        }
        s = opt_block_sum(s, warp_s);
        if (threadIdx.x == 0) slots[c] = s;
    }
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double s = 0.0;
    for (int c = threadIdx.x; c < n_chunks; c += OPT_THREADS) s += __ldcg(slots + c);
    s = opt_block_sum(s, warp_s);
    if (threadIdx.x != 0) return;
    *ticket = 0u;   // ready for the next step
    const double total = sqrt(s);
    bool apply = isfinite(total);
#pragma unroll
    for (int i = 0; i < VC_OPTIM_MAX_GUARDS; ++i)
        if (i < guards.n) apply = apply && *guards.w[i] == 0;
    double coef = 1.0;
    if (max_norm >= 0.0 && apply) coef = fmin(1.0, max_norm / (total + 1e-6));
    const double lr = hyper[0], beta1 = hyper[1], beta2 = hyper[2], eps = hyper[3], wd = hyper[4];
    const double t = (double)(counters[0] + 1);
    status->total_norm = total;
    status->clip_coef = coef;
    status->apply = apply ? 1 : 0;
    status->clip = (float)coef;
    status->decay = (float)(1.0 - wd * lr);
    status->step_size = (float)(lr / (1.0 - pow(beta1, t)));
    status->bc2_sqrt = (float)sqrt(1.0 - pow(beta2, t));
    status->eps = (float)eps;
    status->w1 = (float)(1.0 - beta1);
    status->beta2 = (float)beta2;
    status->w2 = (float)(1.0 - beta2);
    counters[apply ? 0 : 1] += 1;
}

__global__ void __launch_bounds__(OPT_THREADS) optim_update_kernel(const vc_optim_seg* __restrict__ segs,
                                                                   const vc_optim_chunk* __restrict__ chunks, int n_chunks,
                                                                   const vc_optim_status* __restrict__ status) {
    if (status->apply == 0) return;
    const float clip = status->clip, decay = status->decay, step_size = status->step_size, bc2_sqrt = status->bc2_sqrt,
                eps = status->eps, w1 = status->w1, beta2 = status->beta2, w2 = status->w2;
    for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
        const vc_optim_chunk ch = chunks[c];
        const vc_optim_seg sg = segs[ch.seg];
        if (sg.p == nullptr) continue;   // a tensor that only counts in the norm
        if (sg.g == nullptr) {   // a trainable parameter without a gradient: decayed only
            const bool vec = opt_aligned16(sg.p);
            for (int e = threadIdx.x * 4; e < ch.len; e += OPT_THREADS * 4) {
                float4 p = opt_load4(sg.p, ch.off + e, ch.len - e, vec);
                p.x *= decay, p.y *= decay, p.z *= decay, p.w *= decay;
                opt_store4(sg.p, ch.off + e, ch.len - e, vec, p);
            }
            continue;
        }
        const bool vec = opt_aligned16(sg.p) && opt_aligned16(sg.g) && opt_aligned16(sg.m) && opt_aligned16(sg.v);
        for (int e = threadIdx.x * 4; e < ch.len; e += OPT_THREADS * 4) {
            const long long i = ch.off + e;
            const int left = ch.len - e;
            float4 p4 = opt_load4(sg.p, i, left, vec), m4 = opt_load4(sg.m, i, left, vec), v4 = opt_load4(sg.v, i, left, vec);
            const float4 g4 = opt_load4(sg.g, i, left, vec);
            float* p = &p4.x;
            float* m = &m4.x;
            float* v = &v4.x;
            const float* g = &g4.x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float gh = clip * g[k];
                p[k] = p[k] * decay;
                m[k] = m[k] + w1 * (gh - m[k]);
                v[k] = v[k] * beta2 + (w2 * gh) * gh;
                p[k] = p[k] - step_size * (m[k] / (sqrtf(v[k]) / bc2_sqrt + eps));
            }
            opt_store4(sg.p, i, left, vec, p4);
            opt_store4(sg.m, i, left, vec, m4);
            opt_store4(sg.v, i, left, vec, v4);
        }
    }
}

}  // namespace vc

using namespace vc;

extern "C" size_t vc_optim_ws_bytes(int n_chunks) { return OPT_SLOTS_OFF + (size_t)(n_chunks > 0 ? n_chunks : 0) * sizeof(double); }

extern "C" int vc_optim_step(const vc_optim_seg* segs, int n_segs, const vc_optim_chunk* chunks, int n_chunks, double max_norm,
                             const int32_t* const* guards, int n_guards, const double* hyper, long long* counters,
                             vc_optim_status* status, int max_ctas, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    VC_CHECK_ARG(n_segs >= 0 && n_chunks >= 0 && max_ctas >= 0, "optim: negative count");
    VC_CHECK_ARG(n_chunks == 0 || (segs && chunks), "optim: null segment table / chunk list");
    VC_CHECK_ARG(hyper && counters && status && ws, "optim: null hyper / counter / status block or workspace");
    VC_CHECK_ARG(ws_bytes >= vc_optim_ws_bytes(n_chunks), "optim: workspace of %zu bytes, %zu needed", ws_bytes,
                 vc_optim_ws_bytes(n_chunks));
    VC_CHECK_ARG(n_guards >= 0 && n_guards <= VC_OPTIM_MAX_GUARDS && (n_guards == 0 || guards), "optim: 0..%d guard words",
                 VC_OPTIM_MAX_GUARDS);
    VC_CHECK_ARG(!isnan(max_norm), "optim: max_norm is NaN");
    OptGuards gw{};
    gw.n = n_guards;
    for (int i = 0; i < n_guards; ++i) {
        VC_CHECK_ARG(guards[i] != nullptr, "optim: guard word %d is null", i);
        gw.w[i] = guards[i];
    }
    int grid = n_chunks > 0 ? n_chunks : 1;
    if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
    cudaStream_t stream = (cudaStream_t)stream_;
    optim_norm_kernel<<<grid, OPT_THREADS, 0, stream>>>(segs, chunks, n_chunks, max_norm, gw, hyper, counters, status,
                                                        (unsigned*)ws, (double*)((char*)ws + OPT_SLOTS_OFF));
    VC_LAUNCH_CHECK();
    optim_update_kernel<<<grid, OPT_THREADS, 0, stream>>>(segs, chunks, n_chunks, status);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
