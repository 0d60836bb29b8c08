// RoI grid points and their voxel coordinates of TEDMHead.roi_grid_pool / roi_grid_pool_mm (VirConv-L / -T / -S) —
// sm_90a, fp32, SIMT.
//
// vc_roi_grid_points = get_global_grid_points_of_roi (ted_head.py:652-673) and the coordinate lines (:481-485, :528-532)
// for all scenes, all RoIs and up to VC_ROI_GRID_MAX_SOURCES feature sources in one launch.  rois [B, N, ld] (ld >= 7:
// x, y, z, dx, dy, dz, heading) fp32 -> new_xyz [B*N*G^3, 3] fp32 and new_coords [S, B*N*G^3, 4] int32 (b, x, y, z).
// The rules, each operation rounding once in fp32 (this file is compiled without contraction):
//
//   G1. Grid point order.  Row m = (b * N + n) * G^3 + (i * G + j) * G + k: the order of ones(G, G, G).nonzero(), x index
//       i slowest, z index k fastest.
//   G2. Local point.  l = ((idx + 0.5) / G) * size - size / 2 per axis, size = roi[3], roi[4], roi[5].
//   G3. Rotation.  rotate_points_along_z (common_utils.py:34-56) is the row vector [lx, ly, lz] times
//       [[c, s, 0], [-s, c, 0], [0, 0, 1]], c, s = cosf, sinf(roi[6]) (torch's CUDA cos / sin):
//       x' = lx * c + ly * (-s) + lz * 0, y' = lx * s + ly * c + lz * 0, z' = lx * 0 + ly * 0 + lz * 1, added left to
//       right.  Then the centre roi[0:3] is added: new_xyz.
//   G4. Voxel coordinate.  v = (new_xyz - range) // voxel_size, then v // stride for each source, with torch's float
//       floor division (c10/util/generic_math.h div_floor_floating: fmod, the sign fix-up, the 0.5 correction; not
//       floorf(a / b), which differs on a few inputs), then truncated to int32 as .int() does.  range and voxel_size are
//       the float32 values torch's wrapped-scalar rule gives (the caller rounds them); the stride is an exact float.
#include <math.h>

#include "common.cuh"

namespace vc {
namespace {

constexpr int THREADS = 256;

struct RgParams {
    const float* rois;
    int N, ld, G;
    long long M;                      // B * N * G^3
    float range[3], voxel[3];
    float stride[VC_ROI_GRID_MAX_SOURCES];
    int S;
};

// torch's div_floor_floating for float (G4)
__device__ __forceinline__ float div_floor_f(float a, float b) {
    if (b == 0.0f) return __fdiv_rn(a, b);
    const float mod = fmodf(a, b);
    float div = __fdiv_rn(__fsub_rn(a, mod), b);
    if (mod != 0.0f && ((b < 0.0f) != (mod < 0.0f))) div = __fsub_rn(div, 1.0f);
    float fl;
    if (div != 0.0f) {
        fl = floorf(div);
        if (__fsub_rn(div, fl) > 0.5f) fl = __fadd_rn(fl, 1.0f);
    } else {
        fl = copysignf(0.0f, __fdiv_rn(a, b));
    }
    return fl;
}

__global__ void __launch_bounds__(THREADS) rg_points_kernel(RgParams p, float* __restrict__ new_xyz,
                                                             int* __restrict__ new_coords) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= p.M) return;
    const int G = p.G, G3 = G * G * G;
    const long long r = m / G3;
    const int q = (int)(m - r * G3);
    const int idx[3] = {q / (G * G), (q / G) % G, q % G};                                   // G1
    const int b = (int)(r / p.N);
    const float* roi = p.rois + r * p.ld;
    const float Gf = (float)G;
    float l[3];
    for (int a = 0; a < 3; ++a) {                                                           // G2
        const float size = roi[3 + a];
        l[a] = __fsub_rn(__fmul_rn(__fdiv_rn(__fadd_rn((float)idx[a], 0.5f), Gf), size), __fdiv_rn(size, 2.0f));
    }
    const float c = cosf(roi[6]), s = sinf(roi[6]);                                         // G3
    float g[3];
    g[0] = __fadd_rn(__fadd_rn(__fmul_rn(l[0], c), __fmul_rn(l[1], -s)), __fmul_rn(l[2], 0.0f));
    g[1] = __fadd_rn(__fadd_rn(__fmul_rn(l[0], s), __fmul_rn(l[1], c)), __fmul_rn(l[2], 0.0f));
    g[2] = __fadd_rn(__fadd_rn(__fmul_rn(l[0], 0.0f), __fmul_rn(l[1], 0.0f)), __fmul_rn(l[2], 1.0f));
    float v[3];
    for (int a = 0; a < 3; ++a) {
        g[a] = __fadd_rn(g[a], roi[a]);
        new_xyz[m * 3 + a] = g[a];
        v[a] = div_floor_f(__fsub_rn(g[a], p.range[a]), p.voxel[a]);                       // G4
    }
    for (int k = 0; k < p.S; ++k) {
        int4 o;
        o.x = b;
        o.y = (int)div_floor_f(v[0], p.stride[k]);
        o.z = (int)div_floor_f(v[1], p.stride[k]);
        o.w = (int)div_floor_f(v[2], p.stride[k]);
        reinterpret_cast<int4*>(new_coords)[(long long)k * p.M + m] = o;
    }
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_roi_grid_points(const float* rois, int B, int N, int ld, int G, const float* range3,
                                  const float* voxel3, const int32_t* strides, int S, float* new_xyz, int* new_coords,
                                  vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && N >= 0 && ld >= 7 && G >= 1 && G <= 64, "roi grid: bad arguments (B=%d, N=%d, ld=%d, G=%d)",
                 B, N, ld, G);
    VC_CHECK_ARG(range3 && voxel3 && (strides || S == 0), "null pointer");
    if (S < 0 || S > VC_ROI_GRID_MAX_SOURCES) {
        set_error("roi grid: %d feature sources (limit %d)", S, VC_ROI_GRID_MAX_SOURCES);
        return VC_ERR_UNSUPPORTED;
    }
    RgParams p;
    p.rois = rois;
    p.N = N;
    p.ld = ld;
    p.G = G;
    p.M = (long long)B * N * G * G * G;
    p.S = S;
    for (int a = 0; a < 3; ++a) {
        p.range[a] = range3[a];
        p.voxel[a] = voxel3[a];
    }
    for (int k = 0; k < VC_ROI_GRID_MAX_SOURCES; ++k) {
        if (k < S) VC_CHECK_ARG(strides[k] >= 1, "roi grid: stride %d of source %d", strides[k], k);
        p.stride[k] = k < S ? (float)strides[k] : 1.0f;
    }
    if (p.M == 0) return VC_OK;
    VC_CHECK_ARG(rois && new_xyz && (new_coords || S == 0), "null pointer");
    VC_CHECK_ARG(p.M <= (long long)THREADS * 0x7fffffff, "roi grid: %lld grid points exceed the launch grid", p.M);
    rg_points_kernel<<<cdiv(p.M, THREADS), THREADS, 0, stream>>>(p, new_xyz, new_coords);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
