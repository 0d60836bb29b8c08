// RoI target sampling of the two-stage head (`ProposalTargetLayer` + `RoIHeadTemplate.assign_targets` of TEDMHead,
// VirConv-L / -T / -S) — sm_90a, fp32, SIMT.
//
// vc_roi_targets = ProposalTargetLayer.forward (roi_heads/target_assigner/proposal_target_layer.py:32-353) followed by
// the canonical transform of RoIHeadTemplate.assign_targets (roi_head_template.py:133-158), for all scenes in one call,
// for the configuration every VirConv YAML uses (TARGET_CONFIG.STAGE*: SAMPLE_ROI_BY_EACH_CLASS True, CLS_SCORE_TYPE
// roi_iou_x, ENABLE_HARD_SAMPLING True or False).  The reference's host randomness (np.random.permutation / rand /
// randint, torch.randint) is replaced by caller-supplied device uniforms in [0, 1); nothing reads the device on the host,
// so the call can be captured in a CUDA graph.  The rules are the reference's:
//
//   1. GT trimming.  Per scene, rows of gt [G, C] are dropped from the end while their sum over ALL C columns (class
//      included) is 0; row 0 always stays, so a scene whose rows are all zero keeps one zero row (G = 0 acts as one
//      zero row as well).  Interior zero rows stay.  Rows whose nonzero entries cancel to exactly 0 are not pinned.
//   2. Matching (get_max_iou_with_same_class, :356-389).  RoI i with label k (int64) is compared only with the kept GTs
//      whose class long(gt[:, -1]) (truncation) equals k, by the 3-D IoU of box_geom.cuh (rule 4 of iou3d_nms.cu, the
//      RoI as box a, exactly what vc_boxes_iou3d computes).  ov = the max, asg = the FIRST argmax in GT row order
//      (torch.max's tie rule over the class-filtered list, which keeps row order).  No GT of its class: ov = 0, asg = 0.
//   3. Categories (subsample_rois, :254-323), with c = gt[asg, -1] compared as a float with i + 1 and every threshold
//      rounded to fp32 (torch compares a float tensor with a Python scalar in fp32):
//        foreground: ov >= min(REG_FG[i], CLS_FG[i]) and c == i + 1 for some class i;
//        easy background: ov < CLS_BG_THRESH_LO (no class test);
//        hard background: CLS_BG_THRESH_LO <= ov < REG_FG[i] and c == i + 1 for some i.
//      Each list is in ascending RoI order.  A RoI in none of them (e.g. its GT's class has no threshold entry) is never
//      sampled; the lists are computed independently, as the reference does.
//   4. Sampling.  R = ROI_PER_IMAGE, F = int(np.round(FG_RATIO * R)), nf / nh / ne the list lengths, nb = nh + ne, and
//      draw(u, n) = min(int(double(u) * n), n - 1) (the product in float64, as numpy's floor(rand * n) takes it):
//        nf > 0, nb > 0: the kf = min(F, nf) foreground RoIs with the smallest keys u_fg[b, p] (p = position in the
//                        foreground list), in ascending key order, ties by p (np.random.permutation's prefix); then
//                        bg(R - kf);
//        nf > 0 only:    R draws with replacement, fg[draw(u_fg[b, r], nf)] (the reference's branch draws these and then
//                        fails in torch.cat((fg_inds, [])) with a TypeError; this is the sample it evidently means);
//        nb > 0 only:    bg(R);
//        neither:        the reference prints and raises NotImplementedError.  Here the scene's outputs are all zero
//                        and the call's status word is incremented (vc_roi_targets zeroes it first).
//      bg(n) (sample_bg_inds, :325-353, draws with replacement): with both lists non-empty, h = min(int(n *
//      HARD_BG_RATIO), nh) (float64) hard draws hard[draw(u_bg[b, j], nh)], j < h, then n - h easy draws
//      easy[draw(u_bg[b, j], ne)], h <= j < n; with one list, all n draws from it with u_bg[b, 0:n].  Output rows:
//      foreground, then hard, then easy (torch.cat's order).
//   5. Labels (forward, :57-184).  gt_iou_of_rois = ov.  reg_valid_mask (int64) = the sum over classes i of
//      [ov > REG_FG[i] and c == i + 1], plus, with hard sampling, [REG_FG[i] > ov > HS_THRESH[i] and c == i + 1] on the
//      selected scenes b = s, s + t, s + 2t, ... with t = int(1 / HARD_SAMPLING_RATIO[i]) and s = draw(u_hs[i], t)
//      (np.random.randint(0, t); the reference's mask indexes dimension 0 of the [B, R] tensor, so it selects scenes).
//      rcnn_cls_labels (fp32) on rows with c == i + 1: 1 if ov > CLS_FG[i], else 0 if ov < CLS_BG[i], else
//      (ov - BG) * inv with inv = 1.0f / float(FG - BG) (torch on CUDA divides by a Python scalar as a multiply by the
//      fp32 reciprocal of the scalar); 0 on every other row.
//   6. Canonical transform (assign_targets, :133-158).  gt_of_rois_src = the gathered GT rows.  gt_of_rois = the same rows
//      with x, y, z minus the RoI centre, ry = remainder(roi[6], float(2 pi)) (torch's floating remainder: fmod, plus
//      the divisor when the signs differ), heading - ry, then x, y rotated by -ry with rotate_points_along_z's matrix
//      (x' = x cos - y sin, y' = x sin + y cos, cos / sin of -ry), and the heading folded: h = remainder(h, 2 pi); h in
//      (pi/2, 3 pi/2) -> remainder(h + pi, 2 pi); h > pi -> h - 2 pi; clamp to [-pi/2, pi/2] (all constants fp32).  The
//      reference rotates with a cuBLAS batched matmul, so this part is specified to a few ulp, not bit for bit.
//
// Layout: pass 1 (rt_match_kernel) is one warp per RoI with the scene's GT box records staged in shared memory (each CTA
// trims the rows itself); the lanes stride over the GTs and a warp reduction keeps (max, first argmax).  Pass 2
// (rt_sample_kernel) is one CTA per scene: block-scan compaction of the three lists, the key ranks of the foreground
// list in shared memory, then one thread per output row gathers, labels and transforms.  This file is compiled without
// contraction (build.py), as iou3d_nms.cu is, so the IoU is bit for bit vc_boxes_iou3d's.
#include <math.h>

#include "box_geom.cuh"
#include "common.cuh"

namespace vc {
namespace {

constexpr int MATCH_WARPS = 8;
constexpr int SAMPLE_THREADS = 512;
constexpr float TWO_PI_F = (float)(2.0 * 3.14159265358979323846);    // float(2 * np.pi)
constexpr float PI_F = (float)3.14159265358979323846;                  // float(np.pi)
constexpr float HALF_PI_F = (float)(3.14159265358979323846 * 0.5);    // float(np.pi * 0.5), float(np.pi / 2)
constexpr float THREE_HALF_PI_F = (float)(3.14159265358979323846 * 1.5);

struct RtParams {
    const float* rois;          // [B, M, ldr]
    const float* scores;        // [B, M]
    const int64_t* labels;      // [B, M]
    const float* gt;            // [B, G, ldg]
    const float* u_fg;          // [B, ld_ufg]
    const float* u_bg;          // [B, R]
    const float* u_hs;          // [n_cls]
    float* o_rois;              // [B, R, ldr]
    float* o_gt_src;            // [B, R, ldg]
    float* o_gt;                // [B, R, ldg]
    float* o_iou;               // [B, R]
    float* o_scores;            // [B, R]
    int64_t* o_labels;          // [B, R]
    int64_t* o_reg;             // [B, R]
    float* o_cls;               // [B, R]
    int32_t* status;            // [1]
    float* ov;                  // ws [B, M]
    int32_t* asg;               // ws [B, M]
    int32_t* lists;             // ws [3, B, M]: foreground, hard, easy
    int32_t* perm;              // ws [B, M]: perm[rank] = position in the foreground list
    int B, M, G, ldr, ldg, R, F, n_cls, hard_sampling, ld_ufg;
    double hard_bg_ratio;
    float lo;
    float fg_thr[VC_ROI_TARGETS_MAX_CLASSES], reg_fg[VC_ROI_TARGETS_MAX_CLASSES], cls_fg[VC_ROI_TARGETS_MAX_CLASSES],
        cls_bg[VC_ROI_TARGETS_MAX_CLASSES], cls_inv[VC_ROI_TARGETS_MAX_CLASSES], hs_thr[VC_ROI_TARGETS_MAX_CLASSES];
    int hs_period[VC_ROI_TARGETS_MAX_CLASSES];
};

__device__ __forceinline__ int draw(float u, int n) { return min((int)((double)u * (double)n), n - 1); }

// torch.remainder for floating types (fmod, plus the divisor when the signs differ)
__device__ __forceinline__ float remainder_f(float a, float b) {
    float m = fmodf(a, b);
    if (m != 0.f && ((b < 0.f) != (m < 0.f))) m += b;
    return m;
}

// ---- pass 1: per-class IoU maximum, one warp per RoI (rules 1, 2) ----
__global__ void __launch_bounds__(MATCH_WARPS * 32) rt_match_kernel(RtParams p) {
    extern __shared__ __align__(16) unsigned char smem[];
    BoxRec* recs = reinterpret_cast<BoxRec*>(smem);
    long long* cls = reinterpret_cast<long long*>(recs + p.G);
    __shared__ int last;
    const int b = blockIdx.y;
    if (threadIdx.x == 0) last = 0;
    __syncthreads();
    const float* g = p.gt + (size_t)b * p.G * p.ldg;
    for (int j = threadIdx.x; j < p.G; j += blockDim.x) {
        const float* r = g + (size_t)j * p.ldg;
        float sum = 0.f;
        for (int k = 0; k < p.ldg; ++k) sum += r[k];
        if (sum != 0.f) atomicMax(&last, j);
        recs[j] = make_rec(r);
        cls[j] = (long long)r[p.ldg - 1];
    }
    __syncthreads();
    const int ng = p.G == 0 ? 0 : last + 1;
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * MATCH_WARPS + (threadIdx.x >> 5);
    if (i >= p.M) return;
    const size_t o = (size_t)b * p.M + i;
    const long long label = p.labels[o];
    const BoxRec a = make_rec(p.rois + o * p.ldr);
    float best = -1.f;   // IoU >= 0: -1 marks "no GT of the class seen"
    int arg = INT_MAX;
    for (int j = lane; j < ng; j += 32) {
        if (cls[j] != label) continue;
        const float v = iou_3d(a, recs[j]);
        if (v > best) {   // lanes visit their GTs in ascending order: the first maximum stays
            best = v;
            arg = j;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, off);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, off);
        if (ob > best || (ob == best && oa < arg)) {
            best = ob;
            arg = oa;
        }
    }
    if (lane == 0) {
        const bool found = arg != INT_MAX;
        p.ov[o] = found ? best : 0.f;
        p.asg[o] = found ? arg : 0;
    }
}

// Appends the indices i (ascending) with flag set to list[count...]; all threads of the CTA call it with the same count.
__device__ __forceinline__ int block_append(bool flag, int i, int32_t* list, int count, int* warp_sums) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, flag);
    if (lane == 0) warp_sums[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < nwarps; ++w) {
        const int s = warp_sums[w];
        before += w < warp ? s : 0;
        total += s;
    }
    if (flag) list[count + before + __popc(m & ((1u << lane) - 1u))] = i;
    __syncthreads();   // warp_sums is reused by the next call
    return count + total;
}

// ---- pass 2: one CTA per scene (rules 3-6) ----
__global__ void __launch_bounds__(SAMPLE_THREADS) rt_sample_kernel(RtParams p) {
    __shared__ int warp_sums[SAMPLE_THREADS / 32];
    __shared__ float keys[VC_ROI_TARGETS_MAX_ROIS];
    const int b = blockIdx.x;
    const float* ov = p.ov + (size_t)b * p.M;
    const int32_t* asg = p.asg + (size_t)b * p.M;
    const float* g = p.gt + (size_t)b * p.G * p.ldg;
    int32_t* fg = p.lists + (size_t)b * p.M;
    int32_t* hard = p.lists + ((size_t)p.B + b) * p.M;
    int32_t* easy = p.lists + ((size_t)2 * p.B + b) * p.M;
    int32_t* perm = p.perm + (size_t)b * p.M;
    // rule 3: the three lists, ascending
    int nf = 0, nh = 0, ne = 0;
    for (int base = 0; base < p.M; base += SAMPLE_THREADS) {
        const int i = base + threadIdx.x;
        bool is_fg = false, is_hard = false, is_easy = false;
        if (i < p.M) {
            const float o = ov[i];
            const float c = p.G > 0 ? g[(size_t)asg[i] * p.ldg + p.ldg - 1] : 0.f;
            for (int k = 0; k < p.n_cls; ++k) {
                if (c != (float)(k + 1)) continue;
                is_fg |= o >= p.fg_thr[k];
                is_hard |= o < p.reg_fg[k] && o >= p.lo;
            }
            is_easy = o < p.lo;
        }
        nf = block_append(is_fg, i, fg, nf, warp_sums);
        nh = block_append(is_hard, i, hard, nh, warp_sums);
        ne = block_append(is_easy, i, easy, ne, warp_sums);
    }
    const int nb = nh + ne;
    const bool both = nf > 0 && nb > 0;
    // rule 4, first branch: ranks of the foreground keys (ascending, ties by position)
    const int kf = both ? min(p.F, nf) : 0;
    if (both) {
        const float* u = p.u_fg + (size_t)b * p.ld_ufg;
        for (int q = threadIdx.x; q < nf; q += SAMPLE_THREADS) keys[q] = u[q];
        __syncthreads();
        for (int q = threadIdx.x; q < nf; q += SAMPLE_THREADS) {
            const float k = keys[q];
            int rank = 0;
            for (int t = 0; t < nf; ++t) {
                const float kt = keys[t];
                rank += (kt < k) || (kt == k && t < q);
            }
            if (rank < kf) perm[rank] = q;
        }
        __syncthreads();
    }
    if (nf == 0 && nb == 0 && threadIdx.x == 0) atomicAdd(p.status, 1);
    const int n_bg = nf > 0 ? (both ? p.R - kf : 0) : p.R;
    const int h = (nh > 0 && ne > 0) ? min((int)((double)n_bg * p.hard_bg_ratio), nh) : (nh > 0 ? n_bg : 0);
    const float* ubg = p.u_bg + (size_t)b * p.R;
    for (int r = threadIdx.x; r < p.R; r += SAMPLE_THREADS) {
        const size_t orow = (size_t)b * p.R + r;
        float* o_roi = p.o_rois + orow * p.ldr;
        float* o_src = p.o_gt_src + orow * p.ldg;
        float* o_gt = p.o_gt + orow * p.ldg;
        if (nf == 0 && nb == 0) {   // the reference raises here; the outputs are zero and the status word is set
            for (int k = 0; k < p.ldr; ++k) o_roi[k] = 0.f;
            for (int k = 0; k < p.ldg; ++k) o_src[k] = o_gt[k] = 0.f;
            p.o_iou[orow] = p.o_scores[orow] = p.o_cls[orow] = 0.f;
            p.o_labels[orow] = p.o_reg[orow] = 0;
            continue;
        }
        int i;
        if (both && r < kf) {
            i = fg[perm[r]];
        } else if (nf > 0 && !both) {
            i = fg[draw(p.u_fg[(size_t)b * p.ld_ufg + r], nf)];
        } else {
            const int j = r - kf;
            i = j < h ? hard[draw(ubg[j], nh)] : easy[draw(ubg[j], ne)];
        }
        const size_t src = (size_t)b * p.M + i;
        const float o = ov[i];
        const float* roi = p.rois + src * p.ldr;
        for (int k = 0; k < p.ldr; ++k) o_roi[k] = roi[k];
        p.o_iou[orow] = o;
        p.o_scores[orow] = p.scores[src];
        p.o_labels[orow] = p.labels[src];
        // rule 6: the gathered GT row and its canonical form
        float row[VC_ROI_TARGETS_MAX_LDG];
        for (int k = 0; k < p.ldg; ++k) row[k] = p.G > 0 ? g[(size_t)asg[i] * p.ldg + k] : 0.f;
        for (int k = 0; k < p.ldg; ++k) o_src[k] = row[k];
        const float c = row[p.ldg - 1];
        // rule 5
        long long reg = 0;
        float cl = 0.f;
        for (int k = 0; k < p.n_cls; ++k) {
            if (c != (float)(k + 1)) continue;
            reg += o > p.reg_fg[k];
            if (p.hard_sampling) {
                const int t = p.hs_period[k], s = draw(p.u_hs[k], t);
                reg += o < p.reg_fg[k] && o > p.hs_thr[k] && b >= s && (b - s) % t == 0;
            }
            cl = o > p.cls_fg[k] ? 1.f : o < p.cls_bg[k] ? 0.f : (o - p.cls_bg[k]) * p.cls_inv[k];
        }
        p.o_reg[orow] = reg;
        p.o_cls[orow] = cl;
        const float x = row[0] - roi[0], y = row[1] - roi[1], z = row[2] - roi[2];
        const float ry = remainder_f(roi[6], TWO_PI_F);
        const float cs = cosf(-ry), sn = sinf(-ry);
        row[0] = x * cs + y * (-sn);
        row[1] = x * sn + y * cs;
        row[2] = z;
        float hd = remainder_f(row[6] - ry, TWO_PI_F);
        if (hd > HALF_PI_F && hd < THREE_HALF_PI_F) hd = remainder_f(hd + PI_F, TWO_PI_F);
        if (hd > PI_F) hd = hd - TWO_PI_F;
        row[6] = fminf(fmaxf(hd, -HALF_PI_F), HALF_PI_F);
        for (int k = 0; k < p.ldg; ++k) o_gt[k] = row[k];
    }
}

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" size_t vc_roi_targets_ws_bytes(int B, int M, int G) {
    if (B <= 0 || M <= 0 || G < 0) return 0;
    const size_t per = align256((size_t)B * M * sizeof(int32_t));
    return 6 * per;   // ov, asg, three lists, perm
}

extern "C" int vc_roi_targets(const float* rois, const float* roi_scores, const int64_t* roi_labels, int B, int M, int ldr,
                              const float* gt, int G, int ldg, int n_cls, const double* reg_fg, const double* cls_fg,
                              const double* cls_bg, double cls_bg_lo, const double* hs_thresh, const double* hs_ratio,
                              int hard_sampling, int R, int F, double hard_bg_ratio, const float* u_fg, int ld_ufg,
                              const float* u_bg, const float* u_hs, float* o_rois, float* o_gt_src, float* o_gt,
                              float* o_iou, float* o_scores, int64_t* o_labels, int64_t* o_reg, float* o_cls,
                              int32_t* status, void* ws, size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(B >= 0 && M >= 0 && G >= 0 && ldr >= 7 && ldg >= 8 && R >= 0 && F >= 0 && F <= R,
                 "roi targets: bad arguments (B=%d, M=%d, G=%d, ldr=%d, ldg=%d, R=%d, F=%d)", B, M, G, ldr, ldg, R, F);
    VC_CHECK_ARG(n_cls >= 1 && n_cls <= VC_ROI_TARGETS_MAX_CLASSES, "roi targets: %d classes (1..%d)", n_cls,
                 VC_ROI_TARGETS_MAX_CLASSES);
    if (M > VC_ROI_TARGETS_MAX_ROIS || G > VC_ROI_TARGETS_MAX_GT || ldg > VC_ROI_TARGETS_MAX_LDG) {
        set_error("roi targets: %d RoIs (limit %d), %d GT rows (limit %d), %d GT columns (limit %d) per scene", M,
                  VC_ROI_TARGETS_MAX_ROIS, G, VC_ROI_TARGETS_MAX_GT, ldg, VC_ROI_TARGETS_MAX_LDG);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(B <= 65535, "roi targets: %d scenes exceed the grid", B);
    VC_CHECK_ARG(reg_fg && cls_fg && cls_bg && status, "null pointer");
    VC_CHECK_ARG(M > 0 || R == 0 || B == 0, "roi targets: %d rows to sample from no RoIs", R);
    VC_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), stream));
    if (B == 0 || R == 0) return VC_OK;
    VC_CHECK_ARG(rois && roi_scores && roi_labels && (gt || G == 0) && u_fg && ld_ufg >= (M > R ? M : R) && u_bg &&
                 o_rois && o_gt_src && o_gt && o_iou && o_scores && o_labels && o_reg && o_cls && ws, "null pointer");
    VC_CHECK_ARG(!hard_sampling || (hs_thresh && hs_ratio && u_hs), "null pointer");
    const size_t need = vc_roi_targets_ws_bytes(B, M, G);
    if (ws_bytes < need) {
        set_error("roi targets: workspace of %zu bytes, %zu needed", ws_bytes, need);
        return VC_ERR_WORKSPACE;
    }
    RtParams p{};
    p.rois = rois;
    p.scores = roi_scores;
    p.labels = roi_labels;
    p.gt = gt;
    p.u_fg = u_fg;
    p.u_bg = u_bg;
    p.u_hs = u_hs;
    p.o_rois = o_rois;
    p.o_gt_src = o_gt_src;
    p.o_gt = o_gt;
    p.o_iou = o_iou;
    p.o_scores = o_scores;
    p.o_labels = o_labels;
    p.o_reg = o_reg;
    p.o_cls = o_cls;
    p.status = status;
    const size_t per = align256((size_t)B * M * sizeof(int32_t));
    unsigned char* w = (unsigned char*)ws;
    p.ov = (float*)w;
    p.asg = (int32_t*)(w + per);
    p.lists = (int32_t*)(w + 2 * per);   // three [B, M] lists, contiguous
    p.perm = (int32_t*)(w + 5 * per);
    p.B = B;
    p.M = M;
    p.G = G;
    p.ldr = ldr;
    p.ldg = ldg;
    p.R = R;
    p.F = F;
    p.n_cls = n_cls;
    p.hard_sampling = hard_sampling ? 1 : 0;
    p.ld_ufg = ld_ufg;
    p.hard_bg_ratio = hard_bg_ratio;
    p.lo = (float)cls_bg_lo;
    for (int k = 0; k < n_cls; ++k) {
        p.fg_thr[k] = (float)(reg_fg[k] < cls_fg[k] ? reg_fg[k] : cls_fg[k]);
        p.reg_fg[k] = (float)reg_fg[k];
        p.cls_fg[k] = (float)cls_fg[k];
        p.cls_bg[k] = (float)cls_bg[k];
        p.cls_inv[k] = 1.0f / (float)(cls_fg[k] - cls_bg[k]);
        if (hard_sampling) {
            p.hs_thr[k] = (float)hs_thresh[k];
            const double t = 1.0 / hs_ratio[k];
            VC_CHECK_ARG(t >= 1.0 && t < 2147483647.0, "roi targets: HARD_SAMPLING_RATIO %g outside (0, 1]", hs_ratio[k]);
            p.hs_period[k] = (int)t;
        }
    }
    if (M > 0) {
        const size_t smem = (size_t)G * (sizeof(BoxRec) + sizeof(long long));
        if (smem > 40 * 1024) VC_CUDA(cudaFuncSetAttribute(rt_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rt_match_kernel<<<dim3(cdiv(M, MATCH_WARPS), B), MATCH_WARPS * 32, smem, stream>>>(p);
        VC_LAUNCH_CHECK();
    }
    rt_sample_kernel<<<B, SAMPLE_THREADS, 0, stream>>>(p);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
