// Box decoding of the detector heads and the cascade stage transforms of TEDMHead (VirConv-T / -S) — sm_90a, fp32,
// SIMT, one thread per box, all scenes in one launch, no atomics, no host read.
//
//   vc_anchor_decode      = AnchorHeadTemplate.generate_predicted_boxes (anchor_head_template.py:335-382) for one
//                           anchor set and ResidualCoder (7 codes): box_preds [B, A, 7], dir_cls [B, A, NB] (or none),
//                           anchors [A, 7] broadcast over the scenes -> boxes [B, A, 7].
//   vc_anchor_decode_bwd  = its gradient with respect to box_preds.
//   vc_roi_decode         = RoIHeadTemplate.generate_predicted_boxes (roi_head_template.py:294-324): box_preds [B*N, 7],
//                           rois [B, N, ld] (ld >= 7) -> boxes [B, N, 7].
//   vc_roi_decode_bwd     = its gradient with respect to box_preds.
//   vc_box_xtrans         = X_TRANS.backward_with_param then forward_with_param on boxes (X_transform.py:49-154), the
//                           per-scene parameters read on the device: TEDMHead.roi_x_trans / roi_score_trans / pred_x_trans
//                           (ted_head.py:675-746).
//
// The rules, each fp32 operation rounding once (this file is compiled without contraction), as torch's CUDA elementwise
// kernels round them:
//
//   R1. RPN decode.  residual_decode (box_coder.cuh): diag = sqrt(dxa*dxa + dya*dya); t0*diag + xa, t1*diag + ya,
//       t2*dza + za, exp(t3)*dxa, exp(t4)*dya, exp(t5)*dza, h = t6 + ra.  With a direction classifier:
//         label = the first maximal bin (torch.max(dim=-1)); a NaN bin is maximal, the first NaN wins;
//         val   = h - dir_offset;
//         q     = val * inv_period + dir_limit_offset, inv_period = 1.0f / period (float): torch's CUDA division by a
//                 CPU scalar multiplies by the float reciprocal (BinaryDivTrueKernel.cu); torch's CPU division divides.
//                 The two can differ in the last bit, so floor(q) can differ where q lies within an ulp of an integer:
//                 there the bin is the one val * inv_period gives;
//         rot   = val - floor(q) * period;
//         h     = (rot + dir_offset) + period * (float)label.
//       period = 2 pi / NUM_DIR_BINS and the offsets are the Python floats rounded to float32 (torch's wrapped-scalar
//       rule).
//   R2. RCNN decode.  residual_decode against the RoI with x = y = z = 0 (so t0*diag + 0, ...), heading kept; then
//       rotate_points_along_z's row vector [x y z] times [[c, s, 0], [-s, c, 0], [0, 0, 1]], c, s = cosf, sinf(roi[6]):
//       x' = (x*c + y*(-s)) + z*0, y' = (x*s + y*c) + z*0, z' = (x*0 + y*0) + z*1; then the RoI centre is added.  RoI
//       columns beyond 7 are not read.
//   R2b. Gradients with respect to box_preds, as torch's autograd forms them:
//       RPN:  d0 = g0*diag, d1 = g1*diag, d2 = g2*dza, d3 = (g3*dxa)*exp(t3), d4 = (g4*dya)*exp(t4),
//             d5 = (g5*dza)*exp(t5), d6 = g6 (+ 0 from floor's zero gradient where a direction classifier is used).
//       RCNN: the rotation's transpose first, gx' = (g0*c + g1*s) + g2*0, gy' = (g0*(-s) + g1*c) + g2*0,
//             gz' = (g0*0 + g1*0) + g2*1, then as the RPN with the RoI's sizes; d6 = g6.
//       The anchors, RoIs and direction logits get none (the reference gives the RoIs one through rotate_points_along_z;
//       the Python layer sends RoIs that require a gradient to the reference method).
//   R3. X_TRANS on boxes, parameters p = transform_param[b, stage] = (theta, flip, scale):
//       backward (from stage): columns 0..5 divided by scale; if flip != 0 (NaN counts as set, as `if tensor` does),
//       y = -(y + 0) and h = -(h + 0); then rotated by a = -theta (c, s = cosf, sinf(a), R2's formula) and h = h + a.
//       forward (to stage): rotated by theta and h = h + theta; then the flip; then columns 0..5 times scale.
//       Columns beyond 7 are copied.  A stage < 0 is skipped.
#include <math.h>

#include "box_coder.cuh"
#include "common.cuh"

namespace vc {
namespace {

constexpr int THREADS = 256;

// [x y z] * [[c, s, 0], [-s, c, 0], [0, 0, 1]] (R2)
__device__ __forceinline__ void rotate_z(float* v, float c, float s) {
    const float x = v[0], y = v[1], z = v[2];
    v[0] = (x * c + y * (-s)) + z * 0.0f;
    v[1] = (x * s + y * c) + z * 0.0f;
    v[2] = (x * 0.0f + y * 0.0f) + z * 1.0f;
}

struct AnchorParams {
    const float* box;
    const float* dir;
    const float* anchors;
    long long M;       // B * A
    int A, NB;
    float dir_offset, dir_limit_offset, period, inv_period;
};

__global__ void __launch_bounds__(THREADS) anchor_decode_kernel(AnchorParams p, float* __restrict__ out) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= p.M) return;
    const float* anc = p.anchors + (m % p.A) * 7;
    float t[7], a[7], g[7];
    for (int k = 0; k < 7; ++k) {
        t[k] = p.box[m * 7 + k];
        a[k] = anc[k];
    }
    residual_decode<float>(t, a, g);
    if (p.dir) {
        const float* d = p.dir + m * p.NB;
        int label = 0;
        float best = d[0];
        for (int k = 1; k < p.NB && !isnan(best); ++k) {
            const float v = d[k];
            if (isnan(v) || v > best) {
                best = v;
                label = k;
            }
        }
        const float val = g[6] - p.dir_offset;
        const float q = val * p.inv_period + p.dir_limit_offset;
        const float rot = val - floorf(q) * p.period;
        g[6] = (rot + p.dir_offset) + p.period * (float)label;
    }
    for (int k = 0; k < 7; ++k) out[m * 7 + k] = g[k];
}

__global__ void __launch_bounds__(THREADS) anchor_decode_bwd_kernel(const float* __restrict__ grad,
                                                                    const float* __restrict__ box,
                                                                    const float* __restrict__ anchors, long long M,
                                                                    int A, int with_dir, float* __restrict__ dbox) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= M) return;
    const float* a = anchors + (m % A) * 7;
    const float* t = box + m * 7;
    const float* g = grad + m * 7;
    float* d = dbox + m * 7;
    const float diag = sqrtf(a[3] * a[3] + a[4] * a[4]);
    d[0] = g[0] * diag;
    d[1] = g[1] * diag;
    d[2] = g[2] * a[5];
    d[3] = (g[3] * a[3]) * expf(t[3]);
    d[4] = (g[4] * a[4]) * expf(t[4]);
    d[5] = (g[5] * a[5]) * expf(t[5]);
    d[6] = with_dir ? g[6] + 0.0f : g[6];
}

__global__ void __launch_bounds__(THREADS) roi_decode_kernel(const float* __restrict__ box,
                                                             const float* __restrict__ rois, long long M, int ld,
                                                             float* __restrict__ out) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= M) return;
    const float* r = rois + m * ld;
    float t[7], a[7], g[7];
    for (int k = 0; k < 7; ++k) {
        t[k] = box[m * 7 + k];
        a[k] = k < 3 ? 0.0f : r[k];
    }
    residual_decode<float>(t, a, g);
    rotate_z(g, cosf(r[6]), sinf(r[6]));
    for (int k = 0; k < 3; ++k) g[k] = g[k] + r[k];
    for (int k = 0; k < 7; ++k) out[m * 7 + k] = g[k];
}

__global__ void __launch_bounds__(THREADS) roi_decode_bwd_kernel(const float* __restrict__ grad,
                                                                 const float* __restrict__ box,
                                                                 const float* __restrict__ rois, long long M, int ld,
                                                                 float* __restrict__ dbox) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= M) return;
    const float* r = rois + m * ld;
    const float* t = box + m * 7;
    const float* g = grad + m * 7;
    float* d = dbox + m * 7;
    const float c = cosf(r[6]), s = sinf(r[6]);
    const float gx = (g[0] * c + g[1] * s) + g[2] * 0.0f;
    const float gy = (g[0] * (-s) + g[1] * c) + g[2] * 0.0f;
    const float gz = (g[0] * 0.0f + g[1] * 0.0f) + g[2] * 1.0f;
    const float diag = sqrtf(r[3] * r[3] + r[4] * r[4]);
    d[0] = gx * diag;
    d[1] = gy * diag;
    d[2] = gz * r[5];
    d[3] = (g[3] * r[3]) * expf(t[3]);
    d[4] = (g[4] * r[4]) * expf(t[4]);
    d[5] = (g[5] * r[5]) * expf(t[5]);
    d[6] = g[6];
}

__device__ __forceinline__ void xt_flip(float* v, float f) {
    if (!(f == 0.0f)) {
        v[1] = -(v[1] + 0.0f);
        v[6] = -(v[6] + 0.0f);
    }
}

__global__ void __launch_bounds__(THREADS) box_xtrans_kernel(const float* __restrict__ boxes,
                                                             const float* __restrict__ tparam, long long M, int N,
                                                             int ld, int R, int from, int to,
                                                             float* __restrict__ out) {
    const long long m = (long long)blockIdx.x * THREADS + threadIdx.x;
    if (m >= M) return;
    const long long b = m / N;
    const float* src = boxes + m * ld;
    float* dst = out + m * ld;
    float v[7];
    for (int k = 0; k < 7; ++k) v[k] = src[k];
    if (from >= 0) {                                            // backward_with_param: scaling, flip, rotation
        const float* p = tparam + (b * R + from) * 3;
        const float th = p[0], f = p[1], sc = p[2];
        for (int k = 0; k < 6; ++k) v[k] = v[k] / sc;
        xt_flip(v, f);
        const float a = -th;
        rotate_z(v, cosf(a), sinf(a));
        v[6] = v[6] + a;
    }
    if (to >= 0) {                                              // forward_with_param: rotation, flip, scaling
        const float* p = tparam + (b * R + to) * 3;
        const float th = p[0], f = p[1], sc = p[2];
        rotate_z(v, cosf(th), sinf(th));
        v[6] = v[6] + th;
        xt_flip(v, f);
        for (int k = 0; k < 6; ++k) v[k] = v[k] * sc;
    }
    for (int k = 0; k < 7; ++k) dst[k] = v[k];
    for (int k = 7; k < ld; ++k) dst[k] = src[k];
}

}  // namespace
}  // namespace vc

using namespace vc;

#define VC_BD_LAUNCH(M, kernel, ...)                                                                        \
    do {                                                                                                    \
        VC_CHECK_ARG((M) <= (long long)THREADS * 0x7fffffff, "box decode: %lld boxes exceed the launch grid", \
                     (long long)(M));                                                                       \
        kernel<<<cdiv((M), THREADS), THREADS, 0, stream>>>(__VA_ARGS__);                                    \
        VC_LAUNCH_CHECK();                                                                                  \
    } while (0)

extern "C" int vc_anchor_decode(const float* box_preds, const float* dir_cls, const float* anchors, int B, int A,
                                int NB, float dir_offset, float dir_limit_offset, float period, float* out,
                                vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && A >= 0, "anchor decode: bad arguments (B=%d, A=%d)", B, A);
    VC_CHECK_ARG(!dir_cls || NB >= 1, "anchor decode: %d direction bins", NB);
    AnchorParams p;
    p.box = box_preds;
    p.dir = dir_cls;
    p.anchors = anchors;
    p.M = (long long)B * A;
    p.A = A;
    p.NB = NB;
    p.dir_offset = dir_offset;
    p.dir_limit_offset = dir_limit_offset;
    p.period = period;
    p.inv_period = 1.0f / period;
    if (p.M == 0) return VC_OK;
    VC_CHECK_ARG(box_preds && anchors && out, "null pointer");
    VC_BD_LAUNCH(p.M, anchor_decode_kernel, p, out);
    return VC_OK;
}

extern "C" int vc_anchor_decode_bwd(const float* grad, const float* box_preds, const float* anchors, int B, int A,
                                    int with_dir, float* dbox, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && A >= 0, "anchor decode backward: bad arguments (B=%d, A=%d)", B, A);
    const long long M = (long long)B * A;
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(grad && box_preds && anchors && dbox, "null pointer");
    VC_BD_LAUNCH(M, anchor_decode_bwd_kernel, grad, box_preds, anchors, M, A, with_dir ? 1 : 0, dbox);
    return VC_OK;
}

extern "C" int vc_roi_decode(const float* box_preds, const float* rois, int B, int N, int ld, float* out,
                             vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && N >= 0 && ld >= 7, "roi decode: bad arguments (B=%d, N=%d, ld=%d)", B, N, ld);
    const long long M = (long long)B * N;
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(box_preds && rois && out, "null pointer");
    VC_BD_LAUNCH(M, roi_decode_kernel, box_preds, rois, M, ld, out);
    return VC_OK;
}

extern "C" int vc_roi_decode_bwd(const float* grad, const float* box_preds, const float* rois, int B, int N, int ld,
                                 float* dbox, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && N >= 0 && ld >= 7, "roi decode backward: bad arguments (B=%d, N=%d, ld=%d)", B, N, ld);
    const long long M = (long long)B * N;
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(grad && box_preds && rois && dbox, "null pointer");
    VC_BD_LAUNCH(M, roi_decode_bwd_kernel, grad, box_preds, rois, M, ld, dbox);
    return VC_OK;
}

extern "C" int vc_box_xtrans(const float* boxes, const float* transform_param, int B, int N, int ld, int R,
                             int from_stage, int to_stage, float* out, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && N >= 0 && ld >= 7 && R >= 1, "box x_trans: bad arguments (B=%d, N=%d, ld=%d, R=%d)", B, N,
                 ld, R);
    VC_CHECK_ARG(from_stage < R && to_stage < R, "box x_trans: stage %d -> %d of %d", from_stage, to_stage, R);
    const long long M = (long long)B * N;
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(boxes && transform_param && out, "null pointer");
    VC_BD_LAUNCH(M, box_xtrans_kernel, boxes, transform_param, M, N, ld, R, from_stage, to_stage, out);
    return VC_OK;
}
