// Overlap geometry of the KITTI evaluation (kitti_object_eval_python: rotate_iou.py's numba CUDA kernel, eval.py's
// image_box_overlap and d3_box_overlap_kernel).  Its includers are compiled without contraction, so that every
// operation below rounds once, in the type stated.
//
// The rotated-box rules follow the types numba gives rotate_iou.py's device functions (float32 arrays, float64 Python
// literals), not iou3d_nms's (box_geom.cuh): no 1 cm margin on the edge tests, vertices sorted by a pseudo-angle
// instead of atan2, and the triangle areas summed in float64.
//
//   E1. Corners of a box (x, y, dx, dy, a), float32: c, s = cos(a), sin(a) in float64 rounded to float32 (as numba's
//       simulator computes math.cos; an ulp of cosf moves a corner at 50 m by an ulp and the IoU by up to 1e-5, the
//       float32 geometry being that ill-conditioned); the local corners (-dx/2, -dy/2),
//       (-dx/2, dy/2), (dx/2, dy/2), (dx/2, -dy/2); corner = ((c*lx + s*ly) + x, ((-s)*lx + c*ly) + y).
//   E2. Intersection polygon of boxes p (the query box) and q, in this order: for each corner i = 0..3, p's corner i if
//       inside q, then q's corner i if inside p (inside: 0 <= ab.ap <= ab.ab and 0 <= ad.ap <= ad.ad with corners
//       a, b, d = 0, 1, 3 of the other box); then for each edge i of p and edge j of q, their crossing if the
//       orientation tests differ on both sides (strict >), at (Dx / DH, Dy / DH) as rotate_iou.py's
//       line_segment_intersection forms them.  At most 16 vertices (8 corners + 16 crossings cannot all occur).
//   E3. Vertex order: the centre is the float32 mean (sum in order, then / n); each vertex's v = (p - centre) /
//       sqrtf(|p - centre|^2), key = v.x, or -2 - v.x where v.y < 0; a stable insertion sort by key ascending.
//   E4. Area: for i = 0..n-3 the triangle (v0, v_{i+1}, v_{i+2}): t = (a.x-c.x)*(b.y-c.y) - (a.y-c.y)*(b.x-c.x) in
//       float32, summed as |t / 2| in float64.  IoU with criterion -1: inter / ((area_p + area_q) - inter) with the
//       box areas dx*dy in float32 and their sum in float32, the rest in float64; 0: inter / area_p; 1: inter / area_q;
//       2: inter.  The result is stored as float32.
//   E5. Image-box overlap (float64): iw = min(x1) - max(x0); if iw > 0, ih likewise; if ih > 0, iw*ih / ua, ua =
//       (area_b + area_q) - iw*ih (criterion -1) or area_b (criterion 0).  Otherwise 0.
//   E6. 3-D overlap: r = E4's intersection with criterion 2 (float32); if r > 0: iw = min(y_b, y_q) - max(y_b - h_b,
//       y_q - h_q) in float64 (camera y points down, y is the bottom face); if iw > 0, inc = iw * r, IoU = inc /
//       ((vol_b + vol_q) - inc), vol = (l*h)*w, stored as float32; else 0.
#pragma once
#include <math.h>

namespace vc {
namespace ke {

struct RBox {
    float x, y, dx, dy, a;
};

__device__ __forceinline__ void corners(const RBox& b, float* c) {
    const float ca = (float)cos((double)b.a), sa = (float)sin((double)b.a);
    const float hx = b.dx * 0.5f, hy = b.dy * 0.5f;
    const float lx[4] = {-hx, -hx, hx, hx}, ly[4] = {-hy, hy, hy, -hy};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        c[2 * i] = (ca * lx[i] + sa * ly[i]) + b.x;
        c[2 * i + 1] = ((-sa) * lx[i] + ca * ly[i]) + b.y;
    }
}

__device__ __forceinline__ bool in_quad(float px, float py, const float* q) {
    const float ab0 = q[2] - q[0], ab1 = q[3] - q[1];
    const float ad0 = q[6] - q[0], ad1 = q[7] - q[1];
    const float ap0 = px - q[0], ap1 = py - q[1];
    const float abab = ab0 * ab0 + ab1 * ab1, abap = ab0 * ap0 + ab1 * ap1;
    const float adad = ad0 * ad0 + ad1 * ad1, adap = ad0 * ap0 + ad1 * ap1;
    return abab >= abap && abap >= 0.0f && adad >= adap && adap >= 0.0f;
}

__device__ __forceinline__ bool seg_cross(const float* p1, const float* p2, int i, int j, float* out) {
    const float a0 = p1[2 * i], a1 = p1[2 * i + 1];
    const float b0 = p1[2 * ((i + 1) & 3)], b1 = p1[2 * ((i + 1) & 3) + 1];
    const float c0 = p2[2 * j], c1 = p2[2 * j + 1];
    const float d0 = p2[2 * ((j + 1) & 3)], d1 = p2[2 * ((j + 1) & 3) + 1];
    const float ba0 = b0 - a0, ba1 = b1 - a1, da0 = d0 - a0, ca0 = c0 - a0, da1 = d1 - a1, ca1 = c1 - a1;
    const bool acd = da1 * ca0 > ca1 * da0;
    const bool bcd = (d1 - b1) * (c0 - b0) > (c1 - b1) * (d0 - b0);
    if (acd != bcd) {
        const bool abc = ca1 * ba0 > ba1 * ca0;
        const bool abd = da1 * ba0 > ba1 * da0;
        if (abc != abd) {
            const float dc0 = d0 - c0, dc1 = d1 - c1;
            const float abba = a0 * b1 - b0 * a1;
            const float cddc = c0 * d1 - d0 * c1;
            const float dh = ba1 * dc0 - ba0 * dc1;
            out[0] = (abba * dc0 - ba0 * cddc) / dh;
            out[1] = (abba * dc1 - ba1 * cddc) / dh;
            return true;
        }
    }
    return false;
}

// E2-E4: intersection area of p (query) and q
__device__ inline double rinter(const RBox& p, const RBox& q) {
    float c1[8], c2[8], pts[2 * 24];
    corners(p, c1);
    corners(q, c2);
    int n = 0;
    for (int i = 0; i < 4; ++i) {
        if (in_quad(c1[2 * i], c1[2 * i + 1], c2)) {
            pts[2 * n] = c1[2 * i];
            pts[2 * n + 1] = c1[2 * i + 1];
            ++n;
        }
        if (in_quad(c2[2 * i], c2[2 * i + 1], c1)) {
            pts[2 * n] = c2[2 * i];
            pts[2 * n + 1] = c2[2 * i + 1];
            ++n;
        }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            if (n < 24 && seg_cross(c1, c2, i, j, pts + 2 * n)) ++n;
    if (n > 0) {
        float cx = 0.0f, cy = 0.0f;
        for (int i = 0; i < n; ++i) {
            cx += pts[2 * i];
            cy += pts[2 * i + 1];
        }
        cx /= (float)n;
        cy /= (float)n;
        float vs[24];
        for (int i = 0; i < n; ++i) {
            float v0 = pts[2 * i] - cx, v1 = pts[2 * i + 1] - cy;
            const float d = sqrtf(v0 * v0 + v1 * v1);
            v0 = v0 / d;
            v1 = v1 / d;
            if (v1 < 0.0f) v0 = -2.0f - v0;
            vs[i] = v0;
        }
        for (int i = 1; i < n; ++i) {
            if (vs[i - 1] > vs[i]) {
                const float t = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
                int j = i;
                while (j > 0 && vs[j - 1] > t) {
                    vs[j] = vs[j - 1];
                    pts[2 * j] = pts[2 * j - 2];
                    pts[2 * j + 1] = pts[2 * j - 1];
                    --j;
                }
                vs[j] = t;
                pts[2 * j] = tx;
                pts[2 * j + 1] = ty;
            }
        }
    }
    double area = 0.0;
    for (int i = 0; i + 2 < n; ++i) {
        const float* a = pts;
        const float* b = pts + 2 * i + 2;
        const float* c = pts + 2 * i + 4;
        const float t = (a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0]);
        area += fabs((double)t / 2.0);
    }
    return area;
}

// E4: rotate_iou_gpu_eval's entry for query box p and box q
__device__ inline float rotate_iou(const RBox& p, const RBox& q, int criterion) {
    const float a1 = p.dx * p.dy, a2 = q.dx * q.dy;
    const double inter = rinter(p, q);
    if (criterion == -1) return (float)(inter / ((double)(a1 + a2) - inter));
    if (criterion == 0) return (float)(inter / (double)a1);
    if (criterion == 1) return (float)(inter / (double)a2);
    return (float)inter;
}

// E5: image_box_overlap's entry for box b and query box q
__device__ inline double image_iou(const double* b, const double* q, int criterion) {
    const double iw = fmin(b[2], q[2]) - fmax(b[0], q[0]);
    if (!(iw > 0.0)) return 0.0;
    const double ih = fmin(b[3], q[3]) - fmax(b[1], q[1]);
    if (!(ih > 0.0)) return 0.0;
    const double ba = (b[2] - b[0]) * (b[3] - b[1]);
    const double ua = criterion == -1 ? (ba + (q[2] - q[0]) * (q[3] - q[1])) - iw * ih : criterion == 0 ? ba : 1.0;
    return iw * ih / ua;
}

}  // namespace ke
}  // namespace vc
