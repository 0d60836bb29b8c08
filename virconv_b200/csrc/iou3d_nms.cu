// Rotated-box IoU and NMS of the detector heads (the reference's compiled `iou3d_nms_cuda`, pcdet/ops/iou3d_nms) — sm_90a,
// fp32, SIMT.
//
// Callers on the VirConv path: the proposal NMS of RoIHeadTemplate.proposal_layer (roi_head_template.py:89-111), the final
// class-agnostic NMS (model_nms_utils.py:125-144), the RoI target assignment (proposal_target_layer.py, boxes_iou3d_gpu) and
// the CPU IoU of GT sampling / WBF (boxes_bev_iou_cpu).  The semantics are the reference's
// (iou3d_nms_kernel.cu:15-372, iou3d_nms.cpp:90-186, iou3d_nms_utils.py:67-100), rule by rule:
//
//   1. Box = (x, y, z, dx, dy, dz, heading).  Its BEV rectangle is centred at (x, y), sides dx, dy, rotated by `heading`
//      about the centre; corners k = 0..3 are (-dx/2,-dy/2), (dx/2,-dy/2), (dx/2,dy/2), (-dx/2,dy/2) rotated, edge k runs
//      from corner k to corner k+1 (mod 4).
//   2. Intersection polygon vertex set, in this insertion order:
//        a. for edge i of a (i-major), edge j of b: their crossing point, when the two segments' bounding boxes overlap
//           (<=) and both cross-product sign products are strictly positive; the point is the cross-product ratio
//           (s5*q0 - s1*q1) / (s5 - s1), or the solve of the two line equations when |s5 - s1| <= 1e-8;
//        b. for k = 0..3: corner k of b if it lies inside a, then corner k of a if it lies inside b, where "inside" has
//           the reference's 1 cm margin: |local x| < dx/2 + 0.01 and |local y| < dy/2 + 0.01.  (Corners up to 1 cm
//           outside count, which moves the area by ~1e-2 m^2 near touching boxes: exact clipping is NOT equivalent.)
//   3. Area: vertices ordered by angle around their mean (ascending, stable: equal keys keep insertion order), fan sum
//      from vertex 0, |sum| / 2; fewer than 3 vertices -> 0.  The key is a pseudo-angle, monotone in atan2's angle
//      with the same branch cut, instead of atan2 itself.
//   4. IoU.  BEV: overlap / max(area_a + area_b - overlap, 1e-8).  3-D: overlap * max(min(top) - max(bottom), 0) /
//      max(vol_a + vol_b - overlap_3d, 1e-6), top/bottom = z +- dz/2, vol = dx*dy*dz (iou3d_nms_utils.py:67-100, fused).
//      Axis-aligned ("normal") IoU ignores the heading (iou3d_nms_kernel.cu:314-325).
//   5. NMS over boxes sorted by descending score: box j is suppressed by an earlier KEPT box i if iou(i, j) > thresh
//      (strict), greedy in sorted order.  iou(i, j) is evaluated with the earlier box as `a`.
//
// Differences in cost, not in result: every box's record (sin/cos, corners, area, padded bounds) is computed once per
// tile instead of per pair; pairs whose bounds (padded by 2 cm, more than the margin can reach) are disjoint are rejected
// before any polygon work, which is exact (their vertex set is empty); the vertex sort is an insertion sort on
// pseudo-angles.  The NMS mask covers only the upper triangle of 64 x 64 tiles, and the greedy pass runs on the device
// (one CTA per segment, removed-bitset in shared memory), so a batched NMS is two launches with no host read.
//
// The geometry is __host__ __device__ and this file is compiled without floating-point contraction (build.py), and
// sin/cos come from a polynomial evaluated with explicit fma, so vc_boxes_iou_bev_host computes bit for bit what the GPU
// computes.
#include <math.h>

#include <vector>

#include "common.cuh"

namespace vc {
namespace {

#define VC_HD __host__ __device__ __forceinline__

constexpr float IOU_MARGIN = 1e-2f;   // rule 2b
constexpr float IOU_EPS = 1e-8f;      // rule 2a, 4
constexpr float AABB_PAD = 2e-2f;     // > 0.01 * sqrt(2): a corner inside the margin band lies within the padded bounds
constexpr int MAXV = 24;              // 16 edge pairs + 8 corners

struct BoxRec {
    float cx, cy, hx, hy;      // centre, half sides
    float c, s;                // cos / sin of the heading
    float px[4], py[4];        // corners
    float lox, loy, hix, hiy;  // bounds of the corners, padded by AABB_PAD
    float area, zlo, zhi, vol;
};

// sin / cos of a float angle, identical on host and device: Cody-Waite reduction by pi/2 and Taylor polynomials on
// [-pi/4, pi/4] in double (error ~1e-16 before the final rounding to float).
VC_HD void sincos_box(float h, float* s_out, float* c_out) {
    const double x = (double)h;
    if (!(fabs(x) < 1e15)) {
        *s_out = *c_out = (float)(x - x);   // NaN for inf / NaN
        return;
    }
    const double k = rint(x * 0.63661977236758134308);
    double r = fma(-k, 1.5707963267948966192e+00, x);
    r = fma(-k, 6.1232339957367660359e-17, r);
    const double r2 = r * r;
    double ps = 1.0 / 355687428096000.0;
    ps = fma(ps, r2, -1.0 / 1307674368000.0);
    ps = fma(ps, r2, 1.0 / 6227020800.0);
    ps = fma(ps, r2, -1.0 / 39916800.0);
    ps = fma(ps, r2, 1.0 / 362880.0);
    ps = fma(ps, r2, -1.0 / 5040.0);
    ps = fma(ps, r2, 1.0 / 120.0);
    ps = fma(ps, r2, -1.0 / 6.0);
    const double sn = fma(r * r2, ps, r);
    double pc = -1.0 / 6402373705728000.0;
    pc = fma(pc, r2, 1.0 / 20922789888000.0);
    pc = fma(pc, r2, -1.0 / 87178291200.0);
    pc = fma(pc, r2, 1.0 / 479001600.0);
    pc = fma(pc, r2, -1.0 / 3628800.0);
    pc = fma(pc, r2, 1.0 / 40320.0);
    pc = fma(pc, r2, -1.0 / 720.0);
    pc = fma(pc, r2, 1.0 / 24.0);
    pc = fma(pc, r2, -0.5);
    const double cs = fma(r2, pc, 1.0);
    switch ((int)((long long)k & 3)) {
        case 0: *s_out = (float)sn; *c_out = (float)cs; break;
        case 1: *s_out = (float)cs; *c_out = (float)-sn; break;
        case 2: *s_out = (float)-sn; *c_out = (float)-cs; break;
        default: *s_out = (float)-cs; *c_out = (float)sn; break;
    }
}

VC_HD BoxRec make_rec(const float* b) {
    BoxRec r;
    r.cx = b[0];
    r.cy = b[1];
    r.hx = b[3] / 2;
    r.hy = b[4] / 2;
    sincos_box(b[6], &r.s, &r.c);
    // the axis-aligned corner first, then its offset from the centre rotated (the reference's rounding order)
    const float x1 = r.cx - r.hx, x2 = r.cx + r.hx, y1 = r.cy - r.hy, y2 = r.cy + r.hy;
    const float lx[4] = {x1 - r.cx, x2 - r.cx, x2 - r.cx, x1 - r.cx}, ly[4] = {y1 - r.cy, y1 - r.cy, y2 - r.cy, y2 - r.cy};
    r.lox = r.loy = INFINITY;
    r.hix = r.hiy = -INFINITY;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        r.px[k] = (lx[k] * r.c + ly[k] * (-r.s)) + r.cx;
        r.py[k] = (lx[k] * r.s + ly[k] * r.c) + r.cy;
        r.lox = fminf(r.lox, r.px[k]);
        r.hix = fmaxf(r.hix, r.px[k]);
        r.loy = fminf(r.loy, r.py[k]);
        r.hiy = fmaxf(r.hiy, r.py[k]);
    }
    r.lox -= AABB_PAD;
    r.loy -= AABB_PAD;
    r.hix += AABB_PAD;
    r.hiy += AABB_PAD;
    r.area = b[3] * b[4];
    r.zlo = b[2] - b[5] / 2;
    r.zhi = b[2] + b[5] / 2;
    r.vol = b[3] * b[4] * b[5];
    return r;
}

// (p1 - p0) x (p2 - p0)
VC_HD float cross3(float p1x, float p1y, float p2x, float p2y, float p0x, float p0y) {
    return (p1x - p0x) * (p2y - p0y) - (p2x - p0x) * (p1y - p0y);
}

// rule 2a: segment p0 -> p1 (edge of a) against q0 -> q1 (edge of b)
VC_HD bool seg_cross(float p0x, float p0y, float p1x, float p1y, float q0x, float q0y, float q1x, float q1y, float* ox,
                     float* oy) {
    if (!(fminf(p0x, p1x) <= fmaxf(q0x, q1x) && fminf(q0x, q1x) <= fmaxf(p0x, p1x) && fminf(p0y, p1y) <= fmaxf(q0y, q1y) &&
          fminf(q0y, q1y) <= fmaxf(p0y, p1y)))
        return false;
    const float s1 = cross3(q0x, q0y, p1x, p1y, p0x, p0y);
    const float s2 = cross3(p1x, p1y, q1x, q1y, p0x, p0y);
    const float s3 = cross3(p0x, p0y, q1x, q1y, q0x, q0y);
    const float s4 = cross3(q1x, q1y, p1x, p1y, q0x, q0y);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return false;
    const float s5 = cross3(q1x, q1y, p1x, p1y, p0x, p0y);
    if (fabsf(s5 - s1) > IOU_EPS) {
        *ox = (s5 * q0x - s1 * q1x) / (s5 - s1);
        *oy = (s5 * q0y - s1 * q1y) / (s5 - s1);
    } else {
        const float a0 = p0y - p1y, b0 = p1x - p0x, c0 = p0x * p1y - p1x * p0y;
        const float a1 = q0y - q1y, b1 = q1x - q0x, c1 = q0x * q1y - q1x * q0y;
        const float d = a0 * b1 - a1 * b0;
        *ox = (b0 * c1 - b1 * c0) / d;
        *oy = (a1 * c0 - a0 * c1) / d;
    }
    return true;
}

// rule 2b: point inside box r with the 1 cm margin (the point rotated by -heading about the centre)
VC_HD bool inside_margin(const BoxRec& r, float x, float y) {
    const float dx = x - r.cx, dy = y - r.cy;
    const float lx = dx * r.c + dy * r.s;
    const float ly = dx * (-r.s) + dy * r.c;
    return fabsf(lx) < r.hx + IOU_MARGIN && fabsf(ly) < r.hy + IOU_MARGIN;
}

// pseudo-angle of (dx, dy): monotone in atan2(dy, dx) on (-pi, pi], same branch cut (negative x axis -> maximum)
VC_HD float angle_key(float dx, float dy) {
    const float l1 = fabsf(dx) + fabsf(dy);
    if (l1 == 0.f) return 0.f;
    const float p = dy / l1;
    if (dx >= 0.f) return p;
    return signbit(dy) ? -2.f - p : 2.f - p;
}

VC_HD float box_overlap(const BoxRec& a, const BoxRec& b) {
    if (a.hix < b.lox || b.hix < a.lox || a.hiy < b.loy || b.hiy < a.loy) return 0.f;   // empty vertex set
    float vx[MAXV], vy[MAXV], key[MAXV];
    int n = 0;
    float sx = 0.f, sy = 0.f;
    for (int i = 0; i < 4; ++i) {
        const int i1 = (i + 1) & 3;
        for (int j = 0; j < 4; ++j) {
            const int j1 = (j + 1) & 3;
            float ox, oy;
            if (seg_cross(a.px[i], a.py[i], a.px[i1], a.py[i1], b.px[j], b.py[j], b.px[j1], b.py[j1], &ox, &oy)) {
                vx[n] = ox;
                vy[n] = oy;
                sx += ox;
                sy += oy;
                ++n;
            }
        }
    }
    for (int k = 0; k < 4; ++k) {
        if (inside_margin(a, b.px[k], b.py[k])) {
            vx[n] = b.px[k];
            vy[n] = b.py[k];
            sx += b.px[k];
            sy += b.py[k];
            ++n;
        }
        if (inside_margin(b, a.px[k], a.py[k])) {
            vx[n] = a.px[k];
            vy[n] = a.py[k];
            sx += a.px[k];
            sy += a.py[k];
            ++n;
        }
    }
    if (n < 3) return 0.f;
    const float mx = sx / n, my = sy / n;
    for (int i = 0; i < n; ++i) key[i] = angle_key(vx[i] - mx, vy[i] - my);
    for (int i = 1; i < n; ++i) {   // stable insertion sort by key
        const float kx = vx[i], ky = vy[i], kk = key[i];
        int j = i - 1;
        while (j >= 0 && key[j] > kk) {
            vx[j + 1] = vx[j];
            vy[j + 1] = vy[j];
            key[j + 1] = key[j];
            --j;
        }
        vx[j + 1] = kx;
        vy[j + 1] = ky;
        key[j + 1] = kk;
    }
    float area = 0.f;
    for (int k = 0; k < n - 1; ++k) {
        const float ax = vx[k] - vx[0], ay = vy[k] - vy[0], bx = vx[k + 1] - vx[0], by = vy[k + 1] - vy[0];
        area += ax * by - ay * bx;
    }
    return fabsf(area) / 2.0f;
}

VC_HD float iou_bev(const BoxRec& a, const BoxRec& b) {
    const float ov = box_overlap(a, b);
    return ov / fmaxf(a.area + b.area - ov, IOU_EPS);
}

VC_HD float iou_3d(const BoxRec& a, const BoxRec& b) {
    const float ov = box_overlap(a, b);
    const float h = fmaxf(fminf(a.zhi, b.zhi) - fmaxf(a.zlo, b.zlo), 0.f);
    const float o3 = ov * h;
    return o3 / fmaxf(a.vol + b.vol - o3, 1e-6f);
}

VC_HD float iou_normal(const BoxRec& a, const BoxRec& b) {
    const float left = fmaxf(a.cx - a.hx, b.cx - b.hx), right = fminf(a.cx + a.hx, b.cx + b.hx);
    const float top = fmaxf(a.cy - a.hy, b.cy - b.hy), bottom = fminf(a.cy + a.hy, b.cy + b.hy);
    const float inter = fmaxf(right - left, 0.f) * fmaxf(bottom - top, 0.f);
    return inter / fmaxf(a.area + b.area - inter, IOU_EPS);
}

// ---- pairwise [na, nb]: a warp spans 32 consecutive b boxes (record in registers, coalesced stores), the CTA's 32 a
// boxes are staged as records in shared memory and read as broadcasts; each of the 4 warps takes every 4th a row ----
constexpr int PAIR_B = 32, PAIR_A = 32, PAIR_WARPS = 4;

template <int MODE>   // 0 BEV overlap, 1 BEV IoU, 2 3-D IoU
__global__ void __launch_bounds__(PAIR_WARPS * 32, 4) pair_kernel(int na, int nb, const float* __restrict__ A,
                                                               const float* __restrict__ B, float* __restrict__ out) {
    __shared__ BoxRec sa[PAIR_A];
    const int a0 = blockIdx.y * PAIR_A;
    const int rows = min(PAIR_A, na - a0);
    if (threadIdx.x < rows) sa[threadIdx.x] = make_rec(A + (size_t)(a0 + threadIdx.x) * 7);
    __syncthreads();
    const int bi = blockIdx.x * PAIR_B + (threadIdx.x & 31);
    if (bi >= nb) return;
    const BoxRec rb = make_rec(B + (size_t)bi * 7);
    for (int i = threadIdx.x >> 5; i < rows; i += PAIR_WARPS) {
        const BoxRec& ra = sa[i];
        const float v = MODE == 0 ? box_overlap(ra, rb) : MODE == 1 ? iou_bev(ra, rb) : iou_3d(ra, rb);
        out[(size_t)(a0 + i) * nb + bi] = v;
    }
}

// ---- batched NMS ----
constexpr int NMS_TILE = 64;
constexpr int NMS_MAX_WORDS = VC_NMS_MAX_BOXES / NMS_TILE;

__device__ __forceinline__ int seg_count(const int32_t* counts, int seg, int n_max) { return min(max(counts[seg], 0), n_max); }

// (a) suppression mask, upper triangle: blockIdx.x enumerates the tiles (row r, col c >= r) row by row, blockIdx.z is the
// segment.  mask[seg][row][c] bit j = iou(row, 64c + j) > thresh, for 64c + j > row only.
__global__ void __launch_bounds__(NMS_TILE, 8) nms_mask_kernel(const float* __restrict__ boxes, int ld, long long seg_stride,
                                                            const int32_t* __restrict__ counts, int n_max, int words,
                                                            float thresh, int normal, unsigned long long* __restrict__ mask) {
    const int seg = blockIdx.z;
    const int n = seg_count(counts, seg, n_max);
    const long long t = blockIdx.x;
    // row r starts at tile r*words - r(r-1)/2
    int r = (int)(((2.0 * words + 1.0) - sqrt((2.0 * words + 1.0) * (2.0 * words + 1.0) - 8.0 * (double)t)) / 2.0);
    r = max(0, min(r, words - 1));
    while (r > 0 && (long long)r * words - (long long)r * (r - 1) / 2 > t) --r;
    while (r + 1 < words && (long long)(r + 1) * words - (long long)(r + 1) * r / 2 <= t) ++r;
    const int c = r + (int)(t - ((long long)r * words - (long long)r * (r - 1) / 2));
    if (c * NMS_TILE >= n) return;   // c >= r: the row tile is past the end as well, or only the columns are
    const float* sb = boxes + (size_t)seg * seg_stride;
    __shared__ BoxRec cs[NMS_TILE];
    const int col_size = min(NMS_TILE, n - c * NMS_TILE), row_size = min(NMS_TILE, n - r * NMS_TILE);
    if ((int)threadIdx.x < col_size) cs[threadIdx.x] = make_rec(sb + (size_t)(c * NMS_TILE + threadIdx.x) * ld);
    __syncthreads();
    if ((int)threadIdx.x >= row_size) return;
    const int row = r * NMS_TILE + threadIdx.x;
    const BoxRec me = make_rec(sb + (size_t)row * ld);
    unsigned long long bits = 0;
    for (int j = (r == c) ? threadIdx.x + 1 : 0; j < col_size; ++j) {
        const float v = normal ? iou_normal(me, cs[j]) : iou_bev(me, cs[j]);
        if (v > thresh) bits |= 1ULL << j;
    }
    mask[((size_t)seg * n_max + row) * words + c] = bits;
}

// (b) greedy pass, one CTA per segment.  Per 64-box word: the in-word decisions come from the diagonal tile (only kept
// boxes are visited: the lowest box not yet removed is kept, its diagonal word is ORed in), then the kept rows' mask
// words right of the diagonal are ORed into the removed-bitset in parallel.
constexpr int GREEDY_THREADS = 256;

__global__ void __launch_bounds__(GREEDY_THREADS) nms_greedy_kernel(const unsigned long long* __restrict__ mask,
                                                                    const int32_t* __restrict__ counts, int n_max, int words,
                                                                    int post_max, int32_t* __restrict__ keep,
                                                                    int32_t* __restrict__ num_keep) {
    __shared__ unsigned long long remv[NMS_MAX_WORDS];
    __shared__ unsigned long long diag[NMS_TILE];
    __shared__ int klist[NMS_TILE];
    const int seg = blockIdx.x;
    const int n = seg_count(counts, seg, n_max);
    const int nw = (n + NMS_TILE - 1) / NMS_TILE;
    int32_t* kp = keep + (size_t)seg * post_max;
    for (int i = threadIdx.x; i < nw; i += GREEDY_THREADS) remv[i] = 0;
    for (int i = threadIdx.x; i < post_max; i += GREEDY_THREADS) kp[i] = -1;
    __syncthreads();
    const unsigned long long* mseg = mask + (size_t)seg * n_max * words;
    int cnt = 0;   // uniform across the CTA
    for (int w = 0; w < nw && cnt < post_max; ++w) {
        const unsigned long long* mrow = mseg + (size_t)w * NMS_TILE * words;
        const int valid = min(NMS_TILE, n - w * NMS_TILE);
        if ((int)threadIdx.x < valid) diag[threadIdx.x] = mrow[(size_t)threadIdx.x * words + w];
        __syncthreads();
        const unsigned long long vmask = valid == NMS_TILE ? ~0ULL : ((1ULL << valid) - 1);
        unsigned long long rm = remv[w];
        unsigned long long cand = ~rm & vmask;
        int nk = 0;
        while (cand && cnt < post_max) {
            const int i = __ffsll((long long)cand) - 1;
            if (threadIdx.x == 0) {
                kp[cnt] = w * NMS_TILE + i;
                klist[nk] = i;
            }
            ++cnt;
            ++nk;
            rm |= diag[i];
            cand = ~rm & vmask & ~((2ULL << i) - 1);   // i = 63: 2 << 63 == 0, mask of nothing left
        }
        __syncthreads();
        const int ncol = nw - w - 1;
        if (cnt < post_max && ncol > 0) {
            for (int q = threadIdx.x; q < nk * ncol; q += GREEDY_THREADS) {
                const int col = w + 1 + q % ncol;
                atomicOr(&remv[col], mrow[(size_t)klist[q / ncol] * words + col]);
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) num_keep[seg] = cnt;
}

int pair_launch(int mode, const float* a, int na, const float* b, int nb, float* out, cudaStream_t stream) {
    VC_CHECK_ARG(na >= 0 && nb >= 0, "bad box counts %d, %d", na, nb);
    if (na == 0 || nb == 0) return VC_OK;
    VC_CHECK_ARG(a && b && out, "null pointer");
    const dim3 grid(cdiv(nb, PAIR_B), cdiv(na, PAIR_A));
    VC_CHECK_ARG(grid.y <= 65535, "boxes_a: %d boxes exceed the grid", na);
    if (mode == 0) pair_kernel<0><<<grid, PAIR_WARPS * 32, 0, stream>>>(na, nb, a, b, out);
    else if (mode == 1) pair_kernel<1><<<grid, PAIR_WARPS * 32, 0, stream>>>(na, nb, a, b, out);
    else pair_kernel<2><<<grid, PAIR_WARPS * 32, 0, stream>>>(na, nb, a, b, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

int nms_words(int n_max) { return (n_max + NMS_TILE - 1) / NMS_TILE; }

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_boxes_overlap_bev(const float* a, int na, const float* b, int nb, float* out, vc_stream_t stream) {
    return pair_launch(0, a, na, b, nb, out, (cudaStream_t)stream);
}

extern "C" int vc_boxes_iou_bev(const float* a, int na, const float* b, int nb, float* out, vc_stream_t stream) {
    return pair_launch(1, a, na, b, nb, out, (cudaStream_t)stream);
}

extern "C" int vc_boxes_iou3d(const float* a, int na, const float* b, int nb, float* out, vc_stream_t stream) {
    return pair_launch(2, a, na, b, nb, out, (cudaStream_t)stream);
}

extern "C" int vc_boxes_iou_bev_host(const float* a, int na, const float* b, int nb, float* out) {
    VC_CHECK_ARG(na >= 0 && nb >= 0, "bad box counts %d, %d", na, nb);
    if (na == 0 || nb == 0) return VC_OK;
    VC_CHECK_ARG(a && b && out, "null pointer");
    std::vector<BoxRec> rb(nb);
    for (int j = 0; j < nb; ++j) rb[j] = make_rec(b + (size_t)j * 7);
    for (int i = 0; i < na; ++i) {
        const BoxRec ra = make_rec(a + (size_t)i * 7);
        for (int j = 0; j < nb; ++j) out[(size_t)i * nb + j] = iou_bev(ra, rb[j]);
    }
    return VC_OK;
}

extern "C" size_t vc_nms_ws_bytes(int batch, int n_max) {
    if (batch <= 0 || n_max <= 0) return 0;
    return (size_t)batch * n_max * nms_words(n_max) * sizeof(unsigned long long);
}

extern "C" int vc_nms_boxes(const float* boxes, int batch, int n_max, int ld, const int32_t* counts, float thresh, int normal,
                            int post_max, int32_t* keep, int32_t* num_keep, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(batch >= 0 && n_max >= 0 && ld >= 7 && post_max >= 0, "bad nms arguments (B=%d, n_max=%d, ld=%d, post_max=%d)",
                 batch, n_max, ld, post_max);
    if (n_max > VC_NMS_MAX_BOXES) {
        set_error("nms: %d boxes per segment exceed the limit of %d", n_max, VC_NMS_MAX_BOXES);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(batch <= 65535, "nms: %d segments exceed the grid", batch);
    if (batch == 0) return VC_OK;
    VC_CHECK_ARG(counts && num_keep && (keep || post_max == 0), "null pointer");
    const int words = nms_words(n_max);
    if (n_max > 0) {
        VC_CHECK_ARG(boxes && ws, "null pointer");
        if (ws_bytes < vc_nms_ws_bytes(batch, n_max)) {
            set_error("nms: workspace of %zu bytes, %zu needed", ws_bytes, vc_nms_ws_bytes(batch, n_max));
            return VC_ERR_WORKSPACE;
        }
        const dim3 grid(words * (words + 1) / 2, 1, batch);
        nms_mask_kernel<<<grid, NMS_TILE, 0, stream>>>(boxes, ld, (long long)n_max * ld, counts, n_max, words, thresh, normal,
                                                       (unsigned long long*)ws);
        VC_LAUNCH_CHECK();
    }
    nms_greedy_kernel<<<batch, GREEDY_THREADS, 0, stream>>>((const unsigned long long*)ws, counts, n_max, words, post_max, keep,
                                                            num_keep);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
