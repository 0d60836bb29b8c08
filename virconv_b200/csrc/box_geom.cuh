// Rotated-box geometry of the reference's iou3d_nms kernels (rules 1-4 of iou3d_nms.cu, which states them), shared by
// iou3d_nms.cu and roi_targets.cu so that the RoI target assignment matches with exactly the IoU vc_boxes_iou3d computes.
// __host__ __device__; every includer is compiled without floating-point contraction (build.py), so the values round
// identically on the host and in every kernel.
#pragma once
#include <math.h>

#include "common.cuh"

namespace vc {

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

}  // namespace vc
