// ResidualCoder.encode_torch / decode_torch (box_coder_utils.py:13-79, 7 codes, encode_angle_by_sincos False) as
// __host__ __device__ code shared by the anchor target assignment (fp32, anchor_targets.cu) and the detection losses
// (float64, head_losses.cu).  T is float or double; the overloaded math calls resolve to the fp32 / fp64 functions.
#pragma once
#include <math.h>

#include "common.cuh"

namespace vc {

#ifndef VC_HD
#define VC_HD __host__ __device__ __forceinline__
#endif

// encode_torch: sizes of both boxes clamped below at 1e-5, then diag = sqrt(dxa^2 + dya^2); (xg-xa)/diag, (yg-ya)/diag,
// (zg-za)/dza, log(dxg/dxa), log(dyg/dya), log(dzg/dza), rg - ra
template <typename T>
VC_HD void residual_encode(const T* g, const T* a, T* t) {
    const T lo = (T)1e-5f;
    const T dxa = fmax(a[3], lo), dya = fmax(a[4], lo), dza = fmax(a[5], lo);
    const T dxg = fmax(g[3], lo), dyg = fmax(g[4], lo), dzg = fmax(g[5], lo);
    const T diag = sqrt(dxa * dxa + dya * dya);
    t[0] = (g[0] - a[0]) / diag;
    t[1] = (g[1] - a[1]) / diag;
    t[2] = (g[2] - a[2]) / dza;
    t[3] = log(dxg / dxa);
    t[4] = log(dyg / dya);
    t[5] = log(dzg / dza);
    t[6] = g[6] - a[6];
}

// decode_torch (no clamp): diag = sqrt(dxa^2 + dya^2); xt*diag + xa, yt*diag + ya, zt*dza + za, exp(dxt)*dxa,
// exp(dyt)*dya, exp(dzt)*dza, rt + ra
template <typename T>
VC_HD void residual_decode(const T* t, const T* a, T* g) {
    const T diag = sqrt(a[3] * a[3] + a[4] * a[4]);
    g[0] = t[0] * diag + a[0];
    g[1] = t[1] * diag + a[1];
    g[2] = t[2] * a[5] + a[2];
    g[3] = exp(t[3]) * a[3];
    g[4] = exp(t[4]) * a[4];
    g[5] = exp(t[5]) * a[5];
    g[6] = t[6] + a[6];
}

}  // namespace vc
