// Training losses of the detector heads (VirConv-L / -T / -S) with their gradients — sm_90a, float64 arithmetic on fp32
// tensors, SIMT.
//
// Two entry points replace the reference's loss code, which runs every training step (VoxelRCNN.get_training_loss,
// detectors/voxel_rcnn.py:24-30) and reads the device on the host ~35 times a step for VirConv-L (~95 for -T / -S):
//   * vc_rpn_loss  = AnchorHeadTemplate.get_loss (anchor_head_template.py:178-333) with OD_LOSS off, the reference's
//                    WeightedSmoothL1Loss, one head, a 7-value ResidualCoder without sin/cos angle encoding;
//   * vc_rcnn_loss = RoIHeadTemplate.get_loss (roi_head_template.py:161-291) with CLS_LOSS BinaryCrossEntropy and
//                    REG_LOSS smooth-l1, all K <= 18 branches (targets_dict{i} / _pi{i} / _p{i}, i < 6) in one launch.
// Each writes the loss values and d total / d prediction for every prediction tensor; the caller's autograd backward only
// scales them by the incoming gradient.  Nothing is read back on the host, so both are graph-capturable.  Every term is
// formed in float64 from the fp32 inputs; losses are fp32, gradients fp32.
//
// RPN rules (per scene b, anchor i, label y = box_cls_labels[b, i]):
//   R1. Normalisers are per scene: n_b = clamp(#(y > 0 in scene b), 1) (:193-195, :250-252).  Classification and box
//       weights are fp32(1 / n_b), as positives.float() / clamp(...) rounds them (:187-195, :250-252); the direction
//       weight is 1 / n_b in the logits' dtype (:286-287; float64 here).
//   R2. Classification weight (:183-188): 1 for y >= 0 (negatives and positives), 0 for y = -1 ("cared").
//   R3. n_cls == 1 folds positive labels to 1 (:189-191); the caller's labels are not written.  The target is the one-hot
//       of y * (y >= 0) without the background column (:198-207): class y > 0 sets column y - 1, y <= 0 sets none.
//   R4. Sigmoid focal loss (loss_utils.py:44-72), alpha 0.25, gamma 2: p = sigmoid(x), alpha_w = t a + (1-t)(1-a),
//       pt = t (1-p) + (1-t) p, loss = alpha_w pt^gamma (max(x, 0) - x t + log1p(exp(-|x|))).  Gradient as autograd
//       gives it: clamp(x, min=0) passes at x = 0, and abs has sign(0) = 0.
//   R5. Box term (:264-270; WeightedSmoothL1Loss, loss_utils.py:100-136): on code 6 the sin-difference (:218-224)
//       x' = sin(x6) cos(t6), t' = cos(x6) sin(t6); then t := x where t is NaN (a NaN target gives a zero term and a zero
//       gradient on codes 0-5; on code 6 cos(NaN) also makes x' NaN, and the term is NaN as in the reference);
//       d = (x - t) * code_weight, n = |d|, loss = where(n < beta, 0.5 n^2 / beta, n - 0.5 beta), the branch picked as
//       written; beta = 1/9.  Weight fp32(1 / n_b) on positives, 0 elsewhere.
//   R6. Direction (:227-240, :278-292): rot = t6 + a6 (anchor i's heading), off = limit_period(rot - DIR_OFFSET, 0, 2 pi)
//       = v - floor(v / 2pi) 2pi, bin = floor(off / (2 pi / NUM_DIR_BINS)) clamped to [0, bins - 1];
//       loss = logsumexp(z) - z[bin] (F.cross_entropy), weight positives / clamp(#positives of the scene, 1).
//   R7. Values: cls = sum / B * cls_weight, loc = sum / B * loc_weight, dir = sum / B * dir_weight, total = their sum
//       (the reference's tb values rpn_loss_cls / _loc / _dir / rpn_loss).  Gradients are those of the total.
//
// RCNN rules (per branch k with weight w_k: 1 for targets_dict{i}, 0.5 for _pi{i} and _p{i}; n rows):
//   C1. Normalisers over the whole branch, not per scene: fg = #(reg_valid_mask > 0) (:171-172), nv = #(label >= 0)
//       (:253-254).
//   C2. BCE exactly as F.binary_cross_entropy(sigmoid(x), y) (:252): both logs clamped at -100; loss =
//       (y - 1) max(log(1-p), -100) - y max(log p, -100); d/dp = (p - y) / max(p (1-p), 1e-12), then the sigmoid's
//       p (1-p): a saturated logit (p = 0 or 1 in float64) gets zero gradient.  cls = sum(loss * (y >= 0)) /
//       max(nv, 1) * rcnn_cls_weight.
//   C3. Reg (:176-190): targets = encode(gt_of_rois[:, :7], rois with x = y = z = heading = 0) (box_coder.cuh), the
//       smooth-L1 of R5 without the sin-difference, summed over the foreground rows, / max(fg, 1) * rcnn_reg_weight.
//   C4. Corner (:192-219, loss_utils.py:209-232), only when CORNER_LOSS_REGULARIZATION and fg > 0, on foreground rows:
//       pred = decode(reg, rois with x = y = z = 0, heading kept) (no clamp), its centre rotated by the RoI's heading
//       (common_utils.rotate_points_along_z: x cos - y sin, x sin + y cos) plus the RoI's centre; the 8 corners of pred
//       (box_utils.boxes_to_corners_3d) against those of gt_of_rois_src and of it with heading + pi:
//       dist = min(|pc - gc|, |pc - gc_flip|), smooth-L1 with beta 1, mean over the corners, mean over the foreground
//       rows, * rcnn_corner_weight.  A tie of the min splits the gradient in half (torch's minimum backward); a zero
//       norm gives zero gradient (torch's norm backward).
//   C5. bb_loss (utils/bbloss.py:4-48; :223-241) on foreground rows: pred = decode(reg, rois with x = y = z = heading
//       = 0), target = gt_of_rois[:, :7].  Per axis a: compute_iou(p_a, p_{a+3}, g_a, g_{a+3}) = clamp_min(min(hi) -
//       max(lo), 0) / clamp_min(max(hi) - min(lo), 0); ioua = 1 - |sin(limit(p6) - limit(g6))| with limit = torch's
//       % 2 pi then the two masked shifts by 2 pi (gradient: identity); angle = 1.25 (1 - |cos(p6 - g6)|); centre =
//       sum of (g - p)^2 over x, y, z; loss = 1.5 (1 - iou_x iou_y iou_z ioua + angle + centre), summed / (fg + 1);
//       0 when fg = 0.  clamp_min passes at 0; min / max ties split the gradient in half.
//   C6. losses[k, 0..3] = (cls, reg, corner, bb) of branch k; losses[K * 4] = sum over k in order of w_k (cls + reg +
//       corner + bb) = the reference's rcnn_loss.  Gradients are those of that total.
//
// Structure and determinism: vc_rpn_loss is a count pass (per-scene positives, integer atomics) and one thread per
// (scene, anchor) that forms the terms and writes its gradient rows; vc_rcnn_loss is one CTA per branch that counts,
// then forms the terms and gradient rows in a strided row loop.  Both sum their terms in float64 per CTA in a fixed tree,
// and the last CTA to finish (an atomic ticket) adds the CTA partials in CTA order.  No float atomics: losses and
// gradients are bit-identical run to run.  Counters live in the workspace and are cleared inside the call.
//
// This file is compiled without floating-point contraction, so every operation rounds once, as torch's kernels do.
#include <math.h>

#include "box_coder.cuh"
#include "common.cuh"

namespace vc {
namespace {

constexpr int HL_THREADS = 256;
constexpr double TWO_PI = 6.283185307179586;   // 2 * np.pi
constexpr double PI_D = 3.141592653589793;     // np.pi

// torch's sign (sign(0) = 0)
__device__ __forceinline__ double sgn(double v) { return (double)((v > 0.0) - (v < 0.0)); }

// sum of NV doubles over the CTA in a fixed order (warp shuffles, then warp 0); the result is valid in thread 0.
// Every thread of the CTA must call it; blockDim.x is a multiple of 32.
template <int NV>
__device__ void block_sum(double (&v)[NV], double (*sh)[NV]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int k = 0; k < NV; ++k)
        for (int o = 16; o; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < NV; ++k) sh[warp][k] = v[k];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            v[k] = lane < nw ? sh[lane][k] : 0.0;
            for (int o = 16; o; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
        }
    }
    __syncthreads();
}

__device__ int block_count(int v, int* sh) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    v = __reduce_add_sync(0xffffffffu, v);
    if (lane == 0) sh[warp] = v;
    __syncthreads();
    int s = 0;
    for (int w = 0; w < nw; ++w) s += sh[w];
    __syncthreads();
    return s;
}

// smooth-L1 of R5 on d: value and d loss / d d (abs has sign(0) = 0; the where's branch as written)
__device__ __forceinline__ double smooth_l1(double d, double beta, double* grad) {
    const double n = fabs(d);
    if (n < beta) {
        *grad = n / beta * sgn(d);
        return 0.5 * (n * n) / beta;
    }
    *grad = sgn(d);
    return n - 0.5 * beta;
}

// ---- RPN --------------------------------------------------------------------------------------------------------
struct RpnParams {
    const float* cls;        // [B, N, C]
    const float* box;        // [B, N, 7]
    const float* dir;        // [B, N, nb] or null
    const int32_t* labels;   // [B, N]
    const float* tgt;        // [B, N, 7]
    const float* anchors;    // [N, 7]
    float* g_cls;
    float* g_box;
    float* g_dir;
    float* losses;           // [4]
    int* npos;               // [B]
    unsigned* ticket;
    double* part;            // [gridDim.x][3]
    int B, N, C, nb;
    double alpha, gamma, beta, w_cls, w_loc, w_dir, dir_offset;
    double cw[7];
};

__global__ void __launch_bounds__(HL_THREADS) rpn_count_kernel(const int32_t* __restrict__ labels, int N, int* npos) {
    __shared__ int sh[HL_THREADS / 32];
    const int b = blockIdx.y;
    const int i = blockIdx.x * HL_THREADS + threadIdx.x;
    const int v = (i < N && labels[(size_t)b * N + i] > 0) ? 1 : 0;
    const int s = block_count(v, sh);
    if (threadIdx.x == 0 && s) atomicAdd(npos + b, s);
}

__global__ void __launch_bounds__(HL_THREADS) rpn_loss_kernel(RpnParams p) {
    __shared__ double sh[HL_THREADS / 32][3];
    __shared__ bool last;
    const long long total = (long long)p.B * p.N;
    const long long e = (long long)blockIdx.x * HL_THREADS + threadIdx.x;
    double acc[3] = {0.0, 0.0, 0.0};
    if (e < total) {
        const int b = (int)(e / p.N), i = (int)(e % p.N);
        const int y = p.labels[e];
        const int np = max(__ldg(p.npos + b), 1);
        const double wpos = (double)(1.0f / (float)np);                     // R1: fp32
        const double sc = p.w_cls / p.B, sl = p.w_loc / p.B, sd = p.w_dir / p.B;
        // R2-R4: focal loss over the classes
        const double wc = y >= 0 ? wpos : 0.0;
        const int tcls = y > 0 ? (p.C == 1 ? 1 : y) : 0;
        for (int c = 0; c < p.C; ++c) {
            const double x = (double)p.cls[e * p.C + c];
            const double t = (tcls == c + 1) ? 1.0 : 0.0;
            const double pr = 1.0 / (1.0 + exp(-x));
            const double aw = t * p.alpha + (1.0 - t) * (1.0 - p.alpha);
            const double pt = t * (1.0 - pr) + (1.0 - t) * pr;
            const double fw = aw * pow(pt, p.gamma);
            const double ex = exp(-fabs(x));
            const double bce = fmax(x, 0.0) - x * t + log1p(ex);
            acc[0] += fw * bce * wc;
            const double dfw = p.gamma == 0.0 ? 0.0 : aw * (p.gamma * pow(pt, p.gamma - 1.0));
            const double dpt = (1.0 - 2.0 * t) * ((1.0 - pr) * pr);
            const double dbce = (x >= 0.0 ? 1.0 : 0.0) - t - sgn(x) * (ex / (1.0 + ex));
            p.g_cls[e * p.C + c] = (float)((dfw * dpt * bce + fw * dbce) * wc * sc);
        }
        // R5: box regression with the sin-difference on code 6
        const double wr = y > 0 ? wpos : 0.0;
        const float* xb = p.box + e * 7;
        const float* tb = p.tgt + e * 7;
#pragma unroll
        for (int k = 0; k < 7; ++k) {
            const double x = (double)xb[k], t = (double)tb[k];
            double xi = x, ti = t, dxi = 1.0, dti = 0.0;
            if (k == 6) {
                xi = sin(x) * cos(t);
                ti = cos(x) * sin(t);
                dxi = cos(x) * cos(t);
                dti = -(sin(x) * sin(t));
            }
            if (isnan(ti)) {
                ti = xi;
                dti = dxi;
            }
            double dl;
            const double l = smooth_l1((xi - ti) * p.cw[k], p.beta, &dl);
            acc[1] += l * wr;
            p.g_box[e * 7 + k] = (float)(dl * p.cw[k] * (dxi - dti) * wr * sl);
        }
        // R6: direction bins
        if (p.dir) {
            const double wd = y > 0 ? 1.0 / (double)np : 0.0;
            const double v = ((double)tb[6] + (double)p.anchors[(size_t)i * 7 + 6]) - p.dir_offset;
            const double off = v - floor(v / TWO_PI) * TWO_PI;
            int bin = (int)floor(off / (TWO_PI / p.nb));
            bin = min(max(bin, 0), p.nb - 1);
            const float* z = p.dir + e * p.nb;
            double m = -INFINITY;
            for (int j = 0; j < p.nb; ++j) m = fmax(m, (double)z[j]);
            double se = 0.0;
            for (int j = 0; j < p.nb; ++j) se += exp((double)z[j] - m);
            const double lse = m + log(se);
            acc[2] += (lse - (double)z[bin]) * wd;
            for (int j = 0; j < p.nb; ++j)
                p.g_dir[e * p.nb + j] = (float)((exp((double)z[j] - m) / se - (j == bin ? 1.0 : 0.0)) * wd * sd);
        }
    }
    block_sum<3>(acc, sh);
    if (threadIdx.x == 0) {
        double* o = p.part + (size_t)blockIdx.x * 3;
        o[0] = acc[0];
        o[1] = acc[1];
        o[2] = acc[2];
        __threadfence();
        last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double s[3] = {0.0, 0.0, 0.0};
    for (unsigned c = threadIdx.x; c < gridDim.x; c += HL_THREADS)   // fixed CTA order per thread, fixed tree after
        for (int k = 0; k < 3; ++k) s[k] += __ldcg(p.part + (size_t)c * 3 + k);
    block_sum<3>(s, sh);
    if (threadIdx.x == 0) {   // R7
        const double cls = s[0] / p.B * p.w_cls, loc = s[1] / p.B * p.w_loc, dir = p.dir ? s[2] / p.B * p.w_dir : 0.0;
        p.losses[0] = (float)cls;
        p.losses[1] = (float)loc;
        p.losses[2] = (float)dir;
        p.losses[3] = (float)(cls + loc + dir);
    }
}

// ---- RCNN -------------------------------------------------------------------------------------------------------
struct RcnnParams {
    vc_rcnn_branch br[VC_RCNN_MAX_BRANCHES];
    int K, corner;
    double beta, w_cls, w_reg, w_corner;
    double cw[7];
    double* part;        // [K][4]: the branch's final (cls, reg, corner, bb)
    unsigned* ticket;
    float* losses;       // [K * 4 + 1]
};

// box_utils.boxes_to_corners_3d's template, already / 2
__constant__ double kCorner[8][3] = {{0.5, 0.5, -0.5},  {0.5, -0.5, -0.5},  {-0.5, -0.5, -0.5}, {-0.5, 0.5, -0.5},
                                     {0.5, 0.5, 0.5},   {0.5, -0.5, 0.5},   {-0.5, -0.5, 0.5},  {-0.5, 0.5, 0.5}};

// corner j of box b: the template scaled by the size, rotated by the heading (x c - y s, x s + y c), plus the centre
__device__ __forceinline__ void corner_of(const double* b, double c, double s, int j, double* o) {
    const double lx = b[3] * kCorner[j][0], ly = b[4] * kCorner[j][1], lz = b[5] * kCorner[j][2];
    o[0] = (lx * c - ly * s) + b[0];
    o[1] = (lx * s + ly * c) + b[1];
    o[2] = lz + b[2];
}

// weights of torch.min(a, b) / torch.max(a, b)'s backward for the first argument (ties split in half)
__device__ __forceinline__ double pick_min(double a, double b) { return a < b ? 1.0 : (a == b ? 0.5 : 0.0); }
__device__ __forceinline__ double pick_max(double a, double b) { return a > b ? 1.0 : (a == b ? 0.5 : 0.0); }

// torch's `ang % (2 pi)` then the two masked shifts of bbloss.limit
__device__ __forceinline__ double limit_ang(double a) {
    a = a - floor(a / TWO_PI) * TWO_PI;
    if (a > PI_D) a = a - TWO_PI;
    if (a < -PI_D) a = a + TWO_PI;
    return a;
}

// compute_iou of one axis (C5): value and d iou / d (x, w)
__device__ double iou_1d(double x, double w, double y, double l, double* gx, double* gw) {
    const double hi1 = x + w * 0.5, lo1 = x - w * 0.5, hi2 = y + l * 0.5, lo2 = y - l * 0.5;
    const double ov_raw = fmin(hi1, hi2) - fmax(lo1, lo2);
    const double al_raw = fmax(hi1, hi2) - fmin(lo1, lo2);
    const double ov = ov_raw < 0.0 ? 0.0 : ov_raw, al = al_raw < 0.0 ? 0.0 : al_raw;
    const double iou = ov / al;
    const double d_ov = 1.0 / al, d_al = -(ov / (al * al));
    const double p_ov = ov_raw >= 0.0 ? 1.0 : 0.0, p_al = al_raw >= 0.0 ? 1.0 : 0.0;
    const double d_hi1 = d_ov * p_ov * pick_min(hi1, hi2) + d_al * p_al * pick_max(hi1, hi2);
    const double d_lo1 = -(d_ov * p_ov * pick_max(lo1, lo2)) - d_al * p_al * pick_min(lo1, lo2);
    *gx = d_hi1 + d_lo1;
    *gw = (d_hi1 - d_lo1) * 0.5;
    return iou;
}

__global__ void __launch_bounds__(HL_THREADS) rcnn_loss_kernel(RcnnParams p) {
    __shared__ double sh[HL_THREADS / 32][4];
    __shared__ int shi[HL_THREADS / 32];
    __shared__ bool last;
    const vc_rcnn_branch& br = p.br[blockIdx.x];
    const int n = br.n;
    // C1
    int c_fg = 0, c_nv = 0;
    for (int i = threadIdx.x; i < n; i += HL_THREADS) {
        c_fg += br.reg_valid_mask[i] > 0;
        c_nv += br.rcnn_cls_labels[i] >= 0.f;
    }
    const int fg = block_count(c_fg, shi), nv = block_count(c_nv, shi);
    const double bw = (double)br.weight;
    const double g_cls_s = p.w_cls / (double)max(nv, 1) * bw;
    const double g_reg_s = p.w_reg / (double)max(fg, 1) * bw;
    const bool do_corner = p.corner && fg > 0;
    const double g_cor_s = do_corner ? p.w_corner / (double)fg / 8.0 * bw : 0.0;
    const double g_bb_s = 1.5 / (double)(fg + 1) * bw;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += HL_THREADS) {
        // C2
        const double x = (double)br.rcnn_cls[i], y = (double)br.rcnn_cls_labels[i];
        const double pr = 1.0 / (1.0 + exp(-x));
        const double lp = fmax(log(pr), -100.0), l1p = fmax(log(1.0 - pr), -100.0);
        const double vm = y >= 0.0 ? 1.0 : 0.0;
        acc[0] += ((y - 1.0) * l1p - y * lp) * vm;
        const double q = (1.0 - pr) * pr;
        br.g_cls[i] = (float)((pr - y) / fmax(q, 1e-12) * q * vm * g_cls_s);
        // C3
        const bool is_fg = br.reg_valid_mask[i] > 0;
        double r[7], roi[7], gt[7];
        for (int k = 0; k < 7; ++k) {
            r[k] = (double)br.rcnn_reg[(size_t)i * 7 + k];
            roi[k] = (double)br.rois[(size_t)i * br.ldr + k];
            gt[k] = (double)br.gt_of_rois[(size_t)i * br.ldg + k];
        }
        double g_r[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        {
            const double anc[7] = {0.0, 0.0, 0.0, roi[3], roi[4], roi[5], 0.0};
            double t[7];
            residual_encode(gt, anc, t);
            for (int k = 0; k < 7; ++k) {
                const double ti = isnan(t[k]) ? r[k] : t[k];
                double dl;
                const double l = smooth_l1((r[k] - ti) * p.cw[k], p.beta, &dl);
                if (is_fg) {
                    acc[1] += l;
                    g_r[k] = isnan(t[k]) ? 0.0 : dl * p.cw[k] * g_reg_s;
                }
            }
        }
        if (!is_fg) {
            for (int k = 0; k < 7; ++k) br.g_reg[(size_t)i * 7 + k] = 0.f;
            continue;
        }
        // C4
        if (do_corner) {
            const double anc[7] = {0.0, 0.0, 0.0, roi[3], roi[4], roi[5], roi[6]};
            double pb[7];
            residual_decode(r, anc, pb);
            const double c0 = cos(roi[6]), s0 = sin(roi[6]);
            const double cx = pb[0], cy = pb[1];
            pb[0] = (cx * c0 - cy * s0) + roi[0];
            pb[1] = (cx * s0 + cy * c0) + roi[1];
            pb[2] = pb[2] + roi[2];
            double gs[7], gf[7];
            for (int k = 0; k < 7; ++k) gs[k] = gf[k] = (double)br.gt_of_rois_src[(size_t)i * br.ldg + k];
            gf[6] = gs[6] + PI_D;
            const double ch = cos(pb[6]), shd = sin(pb[6]);
            const double cg = cos(gs[6]), sg = sin(gs[6]), cf = cos(gf[6]), sf = sin(gf[6]);
            double gC[3] = {0.0, 0.0, 0.0}, gD[3] = {0.0, 0.0, 0.0}, gH = 0.0, lsum = 0.0;
            for (int j = 0; j < 8; ++j) {
                double pc[3], gc[3], fc[3];
                corner_of(pb, ch, shd, j, pc);
                corner_of(gs, cg, sg, j, gc);
                corner_of(gf, cf, sf, j, fc);
                const double d1[3] = {pc[0] - gc[0], pc[1] - gc[1], pc[2] - gc[2]};
                const double d2[3] = {pc[0] - fc[0], pc[1] - fc[1], pc[2] - fc[2]};
                const double n1 = sqrt(d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2]);
                const double n2 = sqrt(d2[0] * d2[0] + d2[1] * d2[1] + d2[2] * d2[2]);
                const double dist = fmin(n1, n2);
                double dl;
                lsum += smooth_l1(dist, 1.0, &dl);
                const double a1 = pick_min(n1, n2) * dl, a2 = pick_min(n2, n1) * dl;
                double gp[3];
                for (int k = 0; k < 3; ++k)
                    gp[k] = (n1 == 0.0 ? 0.0 : a1 * (d1[k] / n1)) + (n2 == 0.0 ? 0.0 : a2 * (d2[k] / n2));
                const double lx = pb[3] * kCorner[j][0], ly = pb[4] * kCorner[j][1];
                for (int k = 0; k < 3; ++k) gC[k] += gp[k];
                gD[0] += (gp[0] * ch + gp[1] * shd) * kCorner[j][0];
                gD[1] += (-gp[0] * shd + gp[1] * ch) * kCorner[j][1];
                gD[2] += gp[2] * kCorner[j][2];
                gH += gp[0] * -(lx * shd + ly * ch) + gp[1] * (lx * ch - ly * shd);
            }
            acc[2] += lsum / 8.0;
            const double gxl = gC[0] * c0 + gC[1] * s0, gyl = -gC[0] * s0 + gC[1] * c0;   // back through the rotation
            const double diag = sqrt(roi[3] * roi[3] + roi[4] * roi[4]);
            g_r[0] += gxl * diag * g_cor_s;
            g_r[1] += gyl * diag * g_cor_s;
            g_r[2] += gC[2] * roi[5] * g_cor_s;
            g_r[3] += gD[0] * pb[3] * g_cor_s;
            g_r[4] += gD[1] * pb[4] * g_cor_s;
            g_r[5] += gD[2] * pb[5] * g_cor_s;
            g_r[6] += gH * g_cor_s;
        }
        // C5
        {
            const double anc[7] = {0.0, 0.0, 0.0, roi[3], roi[4], roi[5], 0.0};
            double pb[7];
            residual_decode(r, anc, pb);
            double gx[3], gw[3], iu[3];
            for (int a = 0; a < 3; ++a) iu[a] = iou_1d(pb[a], pb[a + 3], gt[a], gt[a + 3], gx + a, gw + a);
            const double dlt = limit_ang(pb[6]) - limit_ang(gt[6]);
            const double ia = 1.0 - fabs(sin(dlt));
            const double dia = -(sgn(sin(dlt)) * cos(dlt));
            const double iou = iu[0] * iu[1] * iu[2] * ia;
            const double da = pb[6] - gt[6];
            const double af = 1.25 * (1.0 - fabs(cos(da)));
            const double daf = 1.25 * (sgn(cos(da)) * sin(da));
            double cd = 0.0;
            for (int a = 0; a < 3; ++a) cd += (gt[a] - pb[a]) * (gt[a] - pb[a]);
            acc[3] += (1.0 - iou + af + cd) * 1.5;
            const double pi_[4] = {iu[1] * iu[2] * ia, iu[0] * iu[2] * ia, iu[0] * iu[1] * ia, iu[0] * iu[1] * iu[2]};
            const double diag = sqrt(roi[3] * roi[3] + roi[4] * roi[4]);
            const double sc[3] = {diag, diag, roi[5]};
            for (int a = 0; a < 3; ++a) {
                const double gpa = -(pi_[a] * gx[a]) + 2.0 * (pb[a] - gt[a]);
                g_r[a] += gpa * sc[a] * g_bb_s;
                g_r[a + 3] += -(pi_[a] * gw[a]) * pb[a + 3] * g_bb_s;
            }
            g_r[6] += (-(pi_[3] * dia) + daf) * g_bb_s;
        }
        for (int k = 0; k < 7; ++k) br.g_reg[(size_t)i * 7 + k] = (float)g_r[k];
    }
    block_sum<4>(acc, sh);
    if (threadIdx.x == 0) {
        double* o = p.part + (size_t)blockIdx.x * 4;
        o[0] = acc[0] / (double)max(nv, 1) * p.w_cls;
        o[1] = acc[1] / (double)max(fg, 1) * p.w_reg;
        o[2] = do_corner ? acc[2] / (double)fg * p.w_corner : 0.0;
        o[3] = fg > 0 ? acc[3] / (double)(fg + 1) : 0.0;
        __threadfence();
        last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last || threadIdx.x != 0) return;
    __threadfence();
    double tot = 0.0;
    for (int k = 0; k < p.K; ++k) {   // C6, in branch order
        double s = 0.0;
        for (int m = 0; m < 4; ++m) {
            const double v = __ldcg(p.part + (size_t)k * 4 + m);
            p.losses[k * 4 + m] = (float)v;
            s += v;
        }
        tot += (double)p.br[k].weight * s;
    }
    p.losses[p.K * 4] = (float)tot;
}

constexpr size_t kCounterBytes = 256;

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" size_t vc_rpn_loss_ws_bytes(int B, int N) {
    if (B <= 0 || N <= 0) return 0;
    const long long ctas = cdiv((long long)B * N, HL_THREADS);
    return kCounterBytes + (size_t)B * sizeof(int) + 256 + (size_t)ctas * 3 * sizeof(double);
}

extern "C" int vc_rpn_loss(const float* cls_preds, const float* box_preds, const float* dir_cls_preds,
                           const int32_t* labels, const float* reg_targets, const float* anchors, int B, int N, int n_cls,
                           int n_bins, double alpha, double gamma, double beta, const double* code_weights,
                           double cls_weight, double loc_weight, double dir_weight, double dir_offset, float* losses,
                           float* g_cls, float* g_box, float* g_dir, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 1 && N >= 1 && n_cls >= 1, "rpn loss: bad arguments (B=%d, N=%d, n_cls=%d)", B, N, n_cls);
    VC_CHECK_ARG(!dir_cls_preds || n_bins >= 1, "rpn loss: %d direction bins", n_bins);
    VC_CHECK_ARG(B <= 65535 && (long long)B * N < (1ll << 31), "rpn loss: %d x %d anchors exceed the grid", B, N);
    VC_CHECK_ARG(cls_preds && box_preds && labels && reg_targets && code_weights && losses && g_cls && g_box && ws &&
                     (!dir_cls_preds || (anchors && g_dir)),
                 "null pointer");
    const size_t need = vc_rpn_loss_ws_bytes(B, N);
    if (ws_bytes < need) {
        set_error("rpn loss: workspace of %zu bytes, %zu needed", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    RpnParams p{};
    p.cls = cls_preds;
    p.box = box_preds;
    p.dir = dir_cls_preds;
    p.labels = labels;
    p.tgt = reg_targets;
    p.anchors = anchors;
    p.g_cls = g_cls;
    p.g_box = g_box;
    p.g_dir = g_dir;
    p.losses = losses;
    p.ticket = (unsigned*)ws;
    p.npos = (int*)((char*)ws + kCounterBytes);
    p.part = (double*)((char*)ws + kCounterBytes + (((size_t)B * sizeof(int) + 255) / 256) * 256);
    p.B = B;
    p.N = N;
    p.C = n_cls;
    p.nb = n_bins;
    p.alpha = alpha;
    p.gamma = gamma;
    p.beta = beta;
    p.w_cls = cls_weight;
    p.w_loc = loc_weight;
    p.w_dir = dir_weight;
    p.dir_offset = dir_offset;
    for (int k = 0; k < 7; ++k) p.cw[k] = code_weights[k];
    VC_CUDA(cudaMemsetAsync(ws, 0, kCounterBytes + (size_t)B * sizeof(int), stream));
    rpn_count_kernel<<<dim3(cdiv(N, HL_THREADS), B), HL_THREADS, 0, stream>>>(labels, N, p.npos);
    VC_LAUNCH_CHECK();
    const long long ctas = cdiv((long long)B * N, HL_THREADS);
    rpn_loss_kernel<<<(unsigned)ctas, HL_THREADS, 0, stream>>>(p);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_rcnn_loss_ws_bytes(int K) {
    if (K <= 0) return 0;
    return kCounterBytes + (size_t)K * 4 * sizeof(double);
}

extern "C" int vc_rcnn_loss(const vc_rcnn_branch* branches, int K, double beta, const double* code_weights,
                            double cls_weight, double reg_weight, double corner_weight, int corner, float* losses,
                            void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(K >= 1 && K <= VC_RCNN_MAX_BRANCHES, "rcnn loss: %d branches (1..%d)", K, VC_RCNN_MAX_BRANCHES);
    VC_CHECK_ARG(branches && code_weights && losses && ws, "null pointer");
    const size_t need = vc_rcnn_loss_ws_bytes(K);
    if (ws_bytes < need) {
        set_error("rcnn loss: workspace of %zu bytes, %zu needed", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    RcnnParams p{};
    for (int k = 0; k < K; ++k) {
        const vc_rcnn_branch& b = branches[k];
        VC_CHECK_ARG(b.n >= 0 && b.ldr >= 7 && b.ldg >= 7, "rcnn loss: branch %d: bad arguments (n=%d, ldr=%d, ldg=%d)", k,
                     b.n, b.ldr, b.ldg);
        VC_CHECK_ARG(b.n == 0 || (b.rcnn_cls && b.rcnn_reg && b.rois && b.gt_of_rois && b.gt_of_rois_src &&
                                  b.reg_valid_mask && b.rcnn_cls_labels && b.g_cls && b.g_reg),
                     "rcnn loss: branch %d: null pointer", k);
        p.br[k] = b;
    }
    p.K = K;
    p.corner = corner != 0;
    p.beta = beta;
    p.w_cls = cls_weight;
    p.w_reg = reg_weight;
    p.w_corner = corner_weight;
    for (int k = 0; k < 7; ++k) p.cw[k] = code_weights[k];
    p.ticket = (unsigned*)ws;
    p.part = (double*)((char*)ws + kCounterBytes);
    p.losses = losses;
    VC_CUDA(cudaMemsetAsync(ws, 0, kCounterBytes, stream));
    rcnn_loss_kernel<<<K, HL_THREADS, 0, stream>>>(p);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
