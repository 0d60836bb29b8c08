// Part-score RoI pooling of TEDMHead's PART branch (VirConv-T / -S) — sm_90a, fp32, SIMT.
//
// vc_part_pool_fwd = TEDMHead.obtain_conf_preds (ted_head.py:425-442) with the sample grid of gen_sample_grid
// (:110-135) and the position-sensitive bilinear_interpolate_torch_gridsample (:137-156), for all scenes in one call;
// vc_part_pool_bwd = its gradient with respect to the part map.  parts [B, S*S, H, W] and rois [B, N, ld] (ld >= 7:
// x, y, z, dx, dy, dz, heading) are fp32; out [B * N] is torch.cat(confi) in scene-major order.  The rules:
//
//   R1. Sample position.  Part p = i * S + j with i, j in [0, S) (the row-major order of nonzero() over an S x S
//       tensor).  lx = (i / (S - 1)) * dx - dx / 2, ly = (j / (S - 1)) * dy - dy / 2 with dx, dy = roi[3], roi[4].
//       The rotation is rotate_points_along_z's (common_utils.py:34-56): the row vector [lx, ly, 1] times
//       [[c, s, 0], [-s, c, 0], [0, 0, 1]], c, s = cos, sin(roi[6]), so gx = lx * c + ly * (-s) + 1 * 0 and
//       gy = lx * s + ly * c + 1 * 0, added left to right.  Then gx += roi[0], gy += roi[1], X = (gx + ox) * scale,
//       Y = (gy + oy) * scale.  Every operation rounds once in fp32: this file is compiled without contraction.
//   R2. grid_sample, align_corners=False, padding_mode='zeros'.  The reference's normalisation gx' = (X / W) * 2 - 1 and
//       torch's unnormalisation ix = ((gx' + 1) * W - 1) / 2 (likewise iy with Y and H).  Taps nw, ne, sw, se at
//       (floor(ix), floor(iy)), (+1, 0), (0, +1), (+1, +1) with torch's weights nw = (x1 - ix) * (y1 - iy),
//       ne = (ix - x0) * (y1 - iy), sw = (x1 - ix) * (iy - y0), se = (ix - x0) * (iy - y0), added in that order from 0.
//       A tap outside [0, W-1] x [0, H-1] contributes nothing.  Part p of every RoI samples channel p only.
//   R3. Mean.  out[b * N + n] = (v_0 + v_1 + ... + v_{S*S-1}) / (S * S), summed left to right whatever the launch shape.
//   R4. Backward.  The only gradient is dparts: each in-bounds tap adds (g[b * N + n] / (S * S)) * w to
//       dparts[b, p, y, x].  Every element of dparts is written (0 where no tap lands), and each element's
//       contributions are added in ascending (n, tap) order starting from 0, with no float atomics: the result is
//       bit-identical run to run whatever the grid and whatever torch's deterministic flag says.
//
// The forward and the backward compute the sample positions with the same device function (pp_sample); nothing is
// saved between them.
//
// Layout: the forward is one warp per RoI; the lanes compute the S*S part values into shared memory and lane 0 adds
// them in order.  The backward is one CTA per (scene, part) channel, because only part p's taps reach channel p: the CTA
// zeroes the channel, builds the 4N tap records (key = pixel << 32 | n * 4 + tap, value) in shared memory, sorts the keys
// (bitonic; the keys are unique, so the order within a pixel is (n, tap)) and lets the first record of each pixel add its
// run.  The grouping of gather2d.cu / voxel_pool.cu (slot_groups_dev) works over a global per-group table of several
// launches; with at most 4N records per channel one in-CTA sort is simpler and needs no workspace.
// Limits: N <= VC_PART_POOL_MAX_ROIS (the keys and values of 4N records fill the 48 KB of shared memory a launch gets
// without opting in) and 2 <= S <= VC_PART_POOL_MAX_GRID (the forward's per-warp part buffer); beyond them
// VC_ERR_UNSUPPORTED.
#include <math.h>

#include "common.cuh"

namespace vc {
namespace {

constexpr int FWD_WARPS = 8;
constexpr int BWD_THREADS = 512;
constexpr int MAX_PARTS = VC_PART_POOL_MAX_GRID * VC_PART_POOL_MAX_GRID;
constexpr unsigned long long NO_TAP = ~0ull;

struct PpParams {
    const float* parts;   // [B, S*S, H, W]
    const float* rois;    // [B, N, ld]
    int B, N, ld, S, H, W;
    float ox, oy, scale;
};

struct Taps {
    int pix[4];      // y * W + x of nw, ne, sw, se
    float w[4];
    bool in[4];
};

// R1 + R2: the four taps of part q of one RoI
__device__ __forceinline__ Taps pp_sample(const PpParams& p, const float* roi, int q) {
    const int i = q / p.S, j = q - i * p.S;
    const float dx = roi[3], dy = roi[4];
    const float den = (float)(p.S - 1);
    const float lx = ((float)i / den) * dx - dx / 2.f;
    const float ly = ((float)j / den) * dy - dy / 2.f;
    const float c = cosf(roi[6]), s = sinf(roi[6]);
    float gx = lx * c + ly * (-s) + 1.f * 0.f;
    float gy = lx * s + ly * c + 1.f * 0.f;
    gx = gx + roi[0];
    gy = gy + roi[1];
    const float X = (gx + p.ox) * p.scale, Y = (gy + p.oy) * p.scale;
    const float fW = (float)p.W, fH = (float)p.H;
    const float ix = (((X / fW) * 2.f - 1.f + 1.f) * fW - 1.f) / 2.f;
    const float iy = (((Y / fH) * 2.f - 1.f + 1.f) * fH - 1.f) / 2.f;
    const float x0 = floorf(ix), y0 = floorf(iy);
    const float x1 = x0 + 1.f, y1 = y0 + 1.f;
    Taps t;
    t.w[0] = (x1 - ix) * (y1 - iy);
    t.w[1] = (ix - x0) * (y1 - iy);
    t.w[2] = (x1 - ix) * (iy - y0);
    t.w[3] = (ix - x0) * (iy - y0);
    const float xs[4] = {x0, x1, x0, x1}, ys[4] = {y0, y0, y1, y1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        // bounds tested on the floats: no int conversion of an out-of-range or NaN coordinate
        t.in[k] = xs[k] >= 0.f && xs[k] <= fW - 1.f && ys[k] >= 0.f && ys[k] <= fH - 1.f;
        t.pix[k] = t.in[k] ? (int)ys[k] * p.W + (int)xs[k] : 0;
    }
    return t;
}

// ---- forward: one warp per RoI (R1-R3) ----
__global__ void __launch_bounds__(FWD_WARPS * 32) pp_fwd_kernel(PpParams p, float* __restrict__ out) {
    __shared__ float v[FWD_WARPS][MAX_PARTS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * FWD_WARPS + warp;   // b * N + n
    if (r >= p.B * p.N) return;
    const int b = r / p.N;
    const int S2 = p.S * p.S;
    const size_t hw = (size_t)p.H * p.W;
    const float* roi = p.rois + (size_t)r * p.ld;
    for (int q = lane; q < S2; q += 32) {
        const Taps t = pp_sample(p, roi, q);
        const float* ch = p.parts + ((size_t)b * S2 + q) * hw;
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (t.in[k]) acc += __ldg(ch + t.pix[k]) * t.w[k];
        v[warp][q] = acc;
    }
    __syncwarp();
    if (lane == 0) {
        float s = 0.f;
        for (int q = 0; q < S2; ++q) s += v[warp][q];
        out[r] = s / (float)S2;
    }
}

// ---- backward: one CTA per (part, scene) channel (R4) ----
__global__ void __launch_bounds__(BWD_THREADS) pp_bwd_kernel(PpParams p, const float* __restrict__ g,
                                                             float* __restrict__ dparts, int P) {
    extern __shared__ __align__(16) unsigned char smem[];
    unsigned long long* key = reinterpret_cast<unsigned long long*>(smem);   // [P], P = 4N rounded up to a power of 2
    float* val = reinterpret_cast<float*>(key + P);                         // [4N], indexed by n * 4 + tap
    const int q = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int S2 = p.S * p.S;
    const int hw = p.H * p.W;
    float* ch = dparts + ((size_t)b * S2 + q) * hw;
    for (int i = tid; i < hw; i += BWD_THREADS) ch[i] = 0.f;
    for (int n = tid; n < p.N; n += BWD_THREADS) {
        const Taps t = pp_sample(p, p.rois + ((size_t)b * p.N + n) * p.ld, q);
        const float gs = g[(size_t)b * p.N + n] / (float)S2;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int rec = n * 4 + k;
            key[rec] = t.in[k] ? ((unsigned long long)(unsigned)t.pix[k] << 32) | (unsigned)rec : NO_TAP;
            val[rec] = gs * t.w[k];
        }
    }
    for (int i = 4 * p.N + tid; i < P; i += BWD_THREADS) key[i] = NO_TAP;
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += BWD_THREADS) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = key[i], c = key[l];
                    if ((a > c) == ((i & k) == 0)) {
                        key[i] = c;
                        key[l] = a;
                    }
                }
            }
            __syncthreads();
        }
    }
    // the zeroing above is ordered before these stores by the barriers of the sort
    for (int i = tid; i < P; i += BWD_THREADS) {
        const unsigned long long k0 = key[i];
        if (k0 == NO_TAP) continue;
        const unsigned pix = (unsigned)(k0 >> 32);
        if (i > 0 && (unsigned)(key[i - 1] >> 32) == pix) continue;
        float s = 0.f;
        for (int t = i; t < P && key[t] != NO_TAP && (unsigned)(key[t] >> 32) == pix; ++t) s += val[(unsigned)key[t]];
        ch[pix] = s;
    }
}

int pp_check(const float* rois, int B, int N, int ld, int S, int H, int W, float scale) {
    VC_CHECK_ARG(B >= 0 && N >= 0 && ld >= 7 && H >= 1 && W >= 1 && (long long)H * W < (1ll << 31),
                 "part pool: bad arguments (B=%d, N=%d, ld=%d, H=%d, W=%d)", B, N, ld, H, W);
    VC_CHECK_ARG(B <= 65535, "part pool: %d scenes exceed the grid", B);
    VC_CHECK_ARG(isfinite(scale), "part pool: spatial scale %g is not finite", (double)scale);
    if (N > VC_PART_POOL_MAX_ROIS || S < 2 || S > VC_PART_POOL_MAX_GRID) {
        set_error("part pool: %d RoIs per scene (limit %d), grid size %d (2..%d)", N, VC_PART_POOL_MAX_ROIS, S,
                  VC_PART_POOL_MAX_GRID);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(rois || B == 0 || N == 0, "null pointer");
    return VC_OK;
}

PpParams pp_params(const float* parts, const float* rois, int B, int N, int ld, int S, int H, int W, float ox, float oy,
                   float scale) {
    PpParams p{};
    p.parts = parts;
    p.rois = rois;
    p.B = B;
    p.N = N;
    p.ld = ld;
    p.S = S;
    p.H = H;
    p.W = W;
    p.ox = ox;
    p.oy = oy;
    p.scale = scale;
    return p;
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_part_pool_fwd(const float* parts, const float* rois, int B, int N, int ld, int S, int H, int W,
                                float ox, float oy, float scale, float* out, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rc = pp_check(rois, B, N, ld, S, H, W, scale);
    if (rc != VC_OK) return rc;
    if (B == 0 || N == 0) return VC_OK;
    VC_CHECK_ARG(parts && out, "null pointer");
    const PpParams p = pp_params(parts, rois, B, N, ld, S, H, W, ox, oy, scale);
    pp_fwd_kernel<<<cdiv((long long)B * N, FWD_WARPS), FWD_WARPS * 32, 0, stream>>>(p, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_part_pool_bwd_ws_bytes(int B, int N, int S) {
    (void)B;
    (void)N;
    (void)S;
    return 0;   // the tap records live in shared memory
}

extern "C" int vc_part_pool_bwd(const float* rois, const float* g, int B, int N, int ld, int S, int H, int W, float ox,
                                float oy, float scale, float* dparts, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    (void)ws;
    (void)ws_bytes;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rc = pp_check(rois, B, N, ld, S, H, W, scale);
    if (rc != VC_OK) return rc;
    if (B == 0) return VC_OK;
    VC_CHECK_ARG(dparts && (g || N == 0), "null pointer");
    const PpParams p = pp_params(nullptr, rois, B, N, ld, S, H, W, ox, oy, scale);
    int P = 2;
    while (P < 4 * N) P <<= 1;
    const size_t smem = (size_t)P * sizeof(unsigned long long) + (size_t)4 * N * sizeof(float);
    pp_bwd_kernel<<<dim3(S * S, B), BWD_THREADS, smem, stream>>>(p, g, dparts, P);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
