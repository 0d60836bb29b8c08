// BatchNorm arithmetic shared by bn.cu's apply / reduce kernels and the fused tail of the persistent tensor-core conv
// (conv_tc2.cu): both paths call the same functions, so a fused and an unfused forward give the same bits.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace vc {

__device__ __forceinline__ uint2 pack_bf16x4(float4 v) {
    __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&a);
    o.y = *reinterpret_cast<uint32_t*>(&b);
    return o;
}

// Channel ch of y = relu(x*scale + shift): derives scale / shift from the float64 sums (S = sum x, Q = sum x^2 over n_rows;
// training) or from the running buffers (eval) into sc_s / sh_s; publish (one block): stats_out [4, c] = scale, shift,
// mean, invstd and the running-statistics update.
__device__ __forceinline__ void bn_channel(double S, double Q, int ch, int c, int n_rows, const float* gamma, const float* beta,
                                           float* running_mean, float* running_var, float momentum, float eps, int training,
                                           float* sc_s, float* sh_s, bool publish, float* stats_out) {
    float mean, invstd;
    double var = 0.0;
    if (training) {
        const double n = (double)(n_rows > 0 ? n_rows : 1);
        const double m = S / n;
        var = Q / n - m * m;
        if (var < 0.0) var = 0.0;
        mean = (float)m;
        invstd = (float)(1.0 / sqrt(var + (double)eps));
    } else {
        mean = running_mean[ch];
        invstd = 1.f / sqrtf(running_var[ch] + eps);
    }
    const float scv = gamma[ch] * invstd;
    const float shv = beta[ch] - mean * scv;
    sc_s[ch] = scv;
    sh_s[ch] = shv;
    if (publish) {
        stats_out[ch] = scv;
        stats_out[c + ch] = shv;
        stats_out[2 * c + ch] = mean;
        stats_out[3 * c + ch] = invstd;
        if (training) {
            const double n = (double)n_rows;
            const double unbiased = n_rows > 1 ? var * n / (n - 1.0) : var;
            running_mean[ch] = (1.f - momentum) * running_mean[ch] + momentum * mean;
            running_var[ch] = (1.f - momentum) * running_var[ch] + momentum * (float)unbiased;
        }
    }
}

__device__ __forceinline__ float4 bn_relu4(float4 v, const float (&sc)[4], const float (&sh)[4], int relu) {
    v.x = fmaf(v.x, sc[0], sh[0]); v.y = fmaf(v.y, sc[1], sh[1]);
    v.z = fmaf(v.z, sc[2], sh[2]); v.w = fmaf(v.w, sc[3], sh[3]);
    if (relu) {
        v.x = relu_nan(v.x); v.y = relu_nan(v.y); v.z = relu_nan(v.z); v.w = relu_nan(v.w);
    }
    return v;
}

// Deterministic BN sums: column j of part [n_parts][2c] added in part order — thread t < 256 takes parts t, t + 256, ...,
// then a fixed tree over red [256] (shared).  Every thread of the block calls it (it holds __syncthreads); the sum is
// returned to thread 0.
__device__ __forceinline__ double bn_sums_column(const double* part, int n_parts, int c, int j, double* red) {
    const int t = threadIdx.x;
    if (t < 256) {
        double v = 0.0;
        for (int p = t; p < n_parts; p += 256) v += __ldcg(part + (size_t)p * 2 * c + j);
        red[t] = v;
    }
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (t < s) red[t] += red[t + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

}  // namespace vc
