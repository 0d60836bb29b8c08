// bf16 tensor-core sparse convolution, per-operator C ABI — wgmma, sm_90a.
//
//   * vc_cast_f32_bf16: the f32 -> bf16 cast of the gathered operand;
//   * vc_conv_fwd_tc / vc_conv_dgrad_tc: build the weight image of the call and run the persistent gather-GEMM kernel of
//     conv_tc2.cu (the plan executor calls that kernel directly with images it prepares once per step);
//   * vc_conv_dgrad_scatter_tc: the input gradient of a many-to-one table (tc_scatter_kernel below), which has no gather form.
// Replaces spconv `ops.indice_conv` / `indice_conv_backward` behind spconv_backbone.py:89,92-93,113,563-564 in the bf16
// (benchmark) precision mode; the fp32 kernels in conv_f32.cu stay the 1e-4 parity path.
#include <cuda_bf16.h>

#include "tc_common.cuh"

namespace vc {

// f32 -> bf16 cast of a feature matrix (the gathered operand)
__global__ void cast_bf16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, size_t n4) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n4; i += stride) {
        float4 v = in[i];
        __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
        uint2 o;
        o.x = *reinterpret_cast<uint32_t*>(&a);
        o.y = *reinterpret_cast<uint32_t*>(&b);
        out[i] = o;
    }
}

// operands of the scatter kernel in the GMMA canonical K-major, no-swizzle layout: 8-row x 16-byte core matrices, chunk
// (r, c) of a [rows x KC] matrix at ((r/8)*KC/8 + c)*128 + (r%8)*16 (weight-image layout 0 of tc_prep_images)
template <int KC, int NR>
struct TcCfg {
    static constexpr int CPR = KC / 8;                       // 16-byte chunks per row
    static constexpr int A_BYTES = TCM * KC * 2;             // the dout tile
    static constexpr int B_BYTES = NR * KC * 2;              // one offset's weight image
};

// ------------------------------------------------------------------------------------------------
// dgrad of a MANY-TO-ONE table (the image branch: several rows share a pixel, so the transposed relation is not a
// table and the gradient has to be scattered):  din[nbr[k,o], :] += dout[o, :] @ W_k.
// The fp32 kernel this replaces (conv_f32.cu scatter_gemm_kernel) spent its time in the CUDA-core tile GEMM.  Here the
// GEMM is free: the dout tile [128 x C_out] is CONTIGUOUS (no gather) and is loaded once, all K weight images arrive
// through one bulk copy, and for each offset that reaches the tile the warpgroup computes dout_tile @ W_k with wgmma into
// registers and adds every row of it to its destination row with 8-byte vector reductions (red.global.add.v2.f32).
// What is left is the atomic traffic itself: P * C_in * 4 bytes.
// ------------------------------------------------------------------------------------------------
template <int KC, int NR>
__global__ void __launch_bounds__(128)
tc_scatter_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ wimg,
                  const int32_t* __restrict__ nbr, float* __restrict__ din, int din_ld, int n_out, int K, int* __restrict__ err) {
    using C = TcCfg<KC, NR>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* A = smem_raw;                               // [128 x KC] bf16, GMMA K-major core-matrix image
    unsigned char* B = smem_raw + C::A_BYTES;                  // [K] weight images, as laid out by the prep kernel
    int* nbr_s = reinterpret_cast<int*>(B + (size_t)K * C::B_BYTES);   // [K][128]
    __shared__ __align__(8) uint64_t load_bar;

    const int tid = threadIdx.x;
    const int base = blockIdx.x * TCM;
    if (tid == 0) {
        mbar_init(&load_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    stage_nbr_tile<128, 8>(nbr, n_out, 0, K, base, nbr_s);
    __syncthreads();
    if (tid == 0) {
        const uint32_t bar = smem_u32(&load_bar);
        const uint32_t bytes = (uint32_t)K * C::B_BYTES;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(B)),
                     "l"(wimg), "r"(bytes), "r"(bar)
                     : "memory");
    }
    // the dout tile: consecutive threads -> consecutive 16-byte chunks of consecutive rows (fully coalesced)
    for (int q = tid; q < TCM * C::CPR; q += 128) {
        const int r = q / C::CPR, c = q % C::CPR;
        const bool v = base + r < n_out;
        cp_async16(A + ((r >> 3) * C::CPR + c) * 128 + (r & 7) * 16, dout + (size_t)(v ? base + r : 0) * KC + c * 8, v);
    }
    cp_async_commit();
    cp_async_wait<0>();
    fence_async_smem();
    __syncthreads();
    bool ok = mbar_wait(&load_bar, 0u, err);
    const uint32_t a0 = smem_u32(A), b0 = smem_u32(B);
    float acc[2][NR / 2];                                      // rows [0, 64) and [64, 128)
    for (int k = 0; k < K; ++k) {
        if (!__syncthreads_or(nbr_s[k * TCM + tid] >= 0)) continue;     // no row of the tile reaches offset k
        wg_fence();
#pragma unroll
        for (int m = 0; m < KC / 16; ++m) {
            const uint64_t bd = gmma_desc(b0 + (uint32_t)k * C::B_BYTES + m * 256, 128, C::CPR * 128, 0);
#pragma unroll
            for (int h = 0; h < 2; ++h)
                wgmma_bf16<NR, 0, 0>(acc[h], gmma_desc(a0 + h * 8 * C::CPR * 128 + m * 256, 128, C::CPR * 128, 0), bd, m > 0 ? 1u : 0u);
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_acc(acc[0]);
        wg_fence_acc(acc[1]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int j = 0; j < NR / 2; j += 2) {
                const int dst = nbr_s[k * TCM + 64 * h + wg_row(j, tid)];
                if (dst >= 0) red_add_v2(din + (size_t)dst * din_ld + wg_col(j, tid), acc[h][j], acc[h][j + 1]);
            }
        }
    }
    (void)ok;
}

template <int KC, int NR>
static int launch_tc_scatter(const __nv_bfloat16* dout, const __nv_bfloat16* wimg, const int32_t* nbr, float* din, int din_ld,
                             int n_out, int K, int* err, cudaStream_t stream) {
    size_t smem = (size_t)TcCfg<KC, NR>::A_BYTES + (size_t)K * TcCfg<KC, NR>::B_BYTES + (size_t)K * TCM * 4;
    auto kern = tc_scatter_kernel<KC, NR>;
    VC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<cdiv(n_out, TCM), 128, smem, stream>>>(dout, wimg, nbr, din, din_ld, n_out, K, err);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

// kc = C_out (reduction), nr = C_in (gradient channels); wimg = the K dgrad images (prep mode 1, layout 0, no mirror)
int tc_scatter_with_image(int kc, int nr, const void* dout_bf16, const void* wimg, const int32_t* nbr, float* din, int n_out,
                          int K, int* err, cudaStream_t stream, int din_ld) {
    if (n_out == 0) return VC_OK;
    if (din_ld == 0) din_ld = nr;
    if (din_ld < nr || din_ld % 2 != 0) {
        set_error("tensor-core scatter dgrad: row pitch %d for %d channels", din_ld, nr);
        return VC_ERR_INVALID;
    }
    const __nv_bfloat16* a = (const __nv_bfloat16*)dout_bf16;
    const __nv_bfloat16* b = (const __nv_bfloat16*)wimg;
#define VC_TS_CASE(A, B) \
    if (kc == A && nr == B) return launch_tc_scatter<A, B>(a, b, nbr, din, din_ld, n_out, K, err, stream);
    VC_TS_CASE(16, 16) VC_TS_CASE(16, 32) VC_TS_CASE(16, 64)
    VC_TS_CASE(32, 16) VC_TS_CASE(32, 32) VC_TS_CASE(32, 64)
    VC_TS_CASE(64, 16) VC_TS_CASE(64, 32) VC_TS_CASE(64, 64)
#undef VC_TS_CASE
    set_error("tensor-core scatter dgrad: unsupported channel pair (%d, %d), need 16/32/64", kc, nr);
    return VC_ERR_UNSUPPORTED;
}

}  // namespace vc

using namespace vc;

extern "C" int vc_cast_f32_bf16(const float* in, void* out, long long n, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n >= 0 && n % 4 == 0, "cast: element count %lld must be a multiple of 4", n);
    if (n == 0) return VC_OK;
    VC_CHECK_ARG(in && out, "null pointer");
    size_t n4 = (size_t)n / 4;
    int blocks = (int)((n4 + 255) / 256);
    if (blocks > 132 * 8) blocks = 132 * 8;
    cast_bf16_kernel<<<blocks, 256, 0, stream>>>((const float4*)in, (uint2*)out, n4);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_conv_tc_ws_bytes(int cin, int cout, int K) { return vc::tc_image_bytes(cin, cout, K, 1); }   // >= either layout

static int tc_one_image(const float* w, void* img, int cin, int cout, int K, int mode, int mirror, int layout, cudaStream_t stream) {
    TcPrepTable T;
    T.n = 1;
    TcPrepEntry& e = T.e[0];
    e.w = w; e.img = img; e.cin = cin; e.cout = cout; e.K = K; e.mode = mode; e.mirror = mirror; e.layout = layout; e.first = 0;
    return tc_prep_images(T, stream);
}

static int tc_common(const void* feats_bf16, const float* w, const int32_t* nbr, float* out, int n_rows, int cin, int cout,
                     int K, int mode, int mirror, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err, cudaStream_t stream,
                     int in_ld = 0) {
    VC_CHECK_ARG(n_rows >= 0 && K >= 1 && K <= MAXK_TC, "bad n=%d or K=%d", n_rows, K);
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("tensor-core conv: unsupported channels cin=%d cout=%d", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_rows == 0) return VC_OK;
    VC_CHECK_ARG(feats_bf16 && w && nbr && out && ws, "null pointer");
    if (ws_bytes < vc_conv_tc_ws_bytes(cin, cout, K)) {
        set_error("tensor-core conv workspace %zu < %zu", ws_bytes, vc_conv_tc_ws_bytes(cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    int rc = tc_one_image(w, ws, cin, cout, K, mode, mirror, 1, stream);
    if (rc) return rc;
    int kc = mode == 0 ? cin : cout, nr = mode == 0 ? cout : cin;
    return tc2_conv(kc, nr, feats_bf16, ws, nbr, n_rows, out, n_rows, nullptr, K, bn_sums, err, stream, nullptr, nullptr,
                    (mode == 1 && !mirror) ? 1 : 0, in_ld);
}

extern "C" int vc_conv_fwd_tc(const void* in_bf16, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                              int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag,
                              vc_stream_t stream_) {
    return tc_common(in_bf16, w, nbr, out, n_out, cin, cout, K, 0, 0, bn_sums, ws, ws_bytes, err_flag, (cudaStream_t)stream_);
}

extern "C" int vc_conv_fwd_tc_ld(const void* in_bf16, int in_ld, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                                 int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag,
                                 vc_stream_t stream_) {
    return tc_common(in_bf16, w, nbr, out, n_out, cin, cout, K, 0, 0, bn_sums, ws, ws_bytes, err_flag, (cudaStream_t)stream_,
                     in_ld);
}

static size_t det_w_bytes(int cin, int cout, int K) {
    const size_t a = vc_conv_ws_bytes(cin, cout, K), b = vc_conv_tc_ws_bytes(cin, cout, K);
    return ((a > b ? a : b) + 255) & ~(size_t)255;
}

extern "C" size_t vc_conv_fwd_det_ws_bytes(int n_out, int cin, int cout, int K) {
    if (n_out < 0 || cin <= 0 || cout <= 0 || K < 1) return 0;
    return det_w_bytes(cin, cout, K) + (size_t)cdiv(n_out > 0 ? n_out : 1, TCM) * 2 * cout * sizeof(double);
}

extern "C" int vc_conv_fwd_det(int precision, const void* in, const float* w, const int32_t* nbr, float* out, int n_out, int cin,
                               int cout, int K, double* bn_sums, void* ws, size_t ws_bytes, int32_t* err_flag, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK_TC, "bad n=%d or K=%d", n_out, K);
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("unsupported channels cin=%d cout=%d (need 8/16/32/64)", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) return VC_OK;
    VC_CHECK_ARG(in && w && nbr && out && bn_sums && ws, "null pointer");
    if (ws_bytes < vc_conv_fwd_det_ws_bytes(n_out, cin, cout, K)) {
        set_error("deterministic conv workspace %zu < %zu", ws_bytes, vc_conv_fwd_det_ws_bytes(n_out, cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    const size_t wb = det_w_bytes(cin, cout, K);
    double* part = reinterpret_cast<double*>((char*)ws + wb);
    int rc;
    if (precision == 0) {
        rc = conv_fwd_f32_part((const float*)in, w, nbr, out, n_out, cin, cout, K, part, ws, wb, stream);
    } else {
        rc = tc_one_image(w, ws, cin, cout, K, 0, 0, 1, stream);
        if (!rc)
            rc = tc2_conv(cin, cout, in, ws, nbr, n_out, out, n_out, nullptr, K, nullptr, err_flag, stream, nullptr, nullptr, 0, 0,
                          part);
    }
    if (rc) return rc;
    return bn_sums_reduce_dev(part, n_out, nullptr, TCM, cout, bn_sums, stream);
}

extern "C" size_t vc_conv_bn_relu_tc_ws_bytes(int n_out, int cin, int cout, int K) {
    if (n_out < 0 || cin <= 0 || cout <= 0 || K < 1) return 0;
    return det_w_bytes(cin, cout, K) + ((size_t)cdiv(n_out > 0 ? n_out : 1, TCM) + 1) * 2 * cout * sizeof(double) + 256;
}

extern "C" int vc_conv_bn_relu_tc(const void* in_bf16, const float* w, const int32_t* nbr, float* x, int n_out, const int32_t* n_dev,
                                  int cin, int cout, int K, int deterministic, const float* gamma, const float* beta,
                                  float* running_mean, float* running_var, long long* num_batches_tracked, float momentum, float eps,
                                  int training, float* y, int y_ld, void* y_bf16, int yb_ld, float* stats_out, void* ws,
                                  size_t ws_bytes, int32_t* err_flag, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK_TC, "bad n=%d or K=%d", n_out, K);
    if (!tc2_ch_ok(cin) || !tc2_ch_ok(cout)) {
        set_error("unsupported channels cin=%d cout=%d (need 8/16/32/64)", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) return VC_OK;
    VC_CHECK_ARG(in_bf16 && w && nbr && x && ws && (y || y_bf16), "null pointer");
    VC_CHECK_ARG(y_ld % 4 == 0 && yb_ld % 4 == 0 && y_ld >= cout && yb_ld >= cout, "bad output pitch");
    if (ws_bytes < vc_conv_bn_relu_tc_ws_bytes(n_out, cin, cout, K)) {
        set_error("conv + BN workspace %zu < %zu", ws_bytes, vc_conv_bn_relu_tc_ws_bytes(n_out, cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    const size_t wb = det_w_bytes(cin, cout, K);
    double* sums = reinterpret_cast<double*>((char*)ws + wb);
    int* bar = reinterpret_cast<int*>(sums + 2 * cout);
    double* part = deterministic && training ? reinterpret_cast<double*>((char*)bar + 256) : nullptr;
    VC_CUDA(cudaMemsetAsync(sums, 0, 2 * cout * sizeof(double) + 256, stream));
    int rc = tc_one_image(w, ws, cin, cout, K, 0, 0, 1, stream);
    if (rc) return rc;
    const BnTail bt{gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps, training, sums, y, y_ld, y_bf16, yb_ld,
                    stats_out, n_dev != nullptr, bar};
    bool done = false;
    rc = tc2_conv(cin, cout, in_bf16, ws, nbr, n_out, x, n_out, n_dev, K, training ? sums : nullptr, err_flag, stream, nullptr, nullptr,
                  0, 0, part, &bt, &done);
    if (rc || done) return rc;
    if (part && (rc = bn_sums_reduce_dev(part, n_out, n_dev, TCM, cout, sums, stream)) != VC_OK) return rc;
    return bn_apply_relu_dev(x, sums, n_out, n_dev, cout, gamma, beta, running_mean, running_var, num_batches_tracked, momentum, eps,
                             training, y, y_ld, y_bf16, yb_ld, stats_out, 1, n_dev != nullptr, stream);
}

/* din[nbr[k,o], :] += dout[o, :] @ w[:, k, :] on tensor cores (many-to-one tables; din zeroed by the caller) */
extern "C" int vc_conv_dgrad_scatter_tc(const void* dout_bf16, const float* w, const int32_t* nbr, float* din, int n_out,
                                        int cin, int cout, int K, void* ws, size_t ws_bytes, int32_t* err_flag,
                                        vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_out >= 0 && K >= 1 && K <= MAXK_TC, "bad n=%d or K=%d", n_out, K);
    if (!tc_scatter_ch_ok(cin) || !tc_scatter_ch_ok(cout)) {
        set_error("tensor-core scatter dgrad: unsupported channels cin=%d cout=%d (need 16/32/64)", cin, cout);
        return VC_ERR_UNSUPPORTED;
    }
    if (n_out == 0) return VC_OK;
    VC_CHECK_ARG(dout_bf16 && w && nbr && din && ws, "null pointer");
    if (ws_bytes < vc_conv_tc_ws_bytes(cin, cout, K)) {
        set_error("tensor-core conv workspace %zu < %zu", ws_bytes, vc_conv_tc_ws_bytes(cin, cout, K));
        return VC_ERR_WORKSPACE;
    }
    int rc = tc_one_image(w, ws, cin, cout, K, 1, 0, 0, stream);
    if (rc) return rc;
    return tc_scatter_with_image(cout, cin, dout_bf16, ws, nbr, din, n_out, K, err_flag, stream);
}

extern "C" int vc_conv_dgrad_tc(const void* dout_bf16, const float* w, const int32_t* nbr_t, float* din, int n_in, int cin,
                                int cout, int K, int mirror, void* ws, size_t ws_bytes, int32_t* err_flag,
                                vc_stream_t stream_) {
    return tc_common(dout_bf16, w, nbr_t, din, n_in, cin, cout, K, 1, mirror, nullptr, ws, ws_bytes, err_flag,
                     (cudaStream_t)stream_);
}
