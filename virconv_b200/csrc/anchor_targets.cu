// Anchor-head target assignment of the RPN (`AnchorHeadSingle` of VirConv-L / -T / -S) — sm_90a, fp32, SIMT.
//
// Two entry points replace host-driven torch code that runs on every training step:
//   * vc_anchor_mask    = AnchorHeadSingle.get_anchor_mask (anchor_head_single.py:75-115): which BEV cells keep anchors;
//   * vc_anchor_targets = AxisAlignedTargetAssigner.assign_targets (axis_aligned_target_assigner.py:46-243) with
//                         POS_FRACTION < 0, MATCH_HEIGHT False, USE_MULTIHEAD False, for all scenes and anchor sets at once.
// Neither reads the device on the host, so both can be captured in a CUDA graph.  The rules are the reference's:
//
//   0. Anchor mask.  stride = round(voxel_size * 8 * 10) (the caller passes 1/stride rounded to fp32, see rule 2);
//      c = long((p - min) * (1/stride)) for p = points[:, 1] (x) and points[:, 2] (y) of every point of the batch
//      (truncation toward zero), clamped from above only, to W/10 - 1 (x) and H/10 - 1 (y).  A negative c wraps like a
//      torch index (c + W/10); one below -W/10 would raise IndexError in the reference and is ignored here.  Every
//      occupied coarse cell (cy, cx) sets the fine cells (10 cy + i, 10 cx + j), i, j in [-10, 10), and negative fine
//      indices wrap again: y in -10..-1 sets rows H-10..H-1 and x in -10..-1 columns W-10..W-1 (for W = 176 the columns
//      170-175 can only be set this way).
//   1. GT trimming.  Per scene, rows of gt [M, C] (C >= 8; class in the last column, box in the first seven) are dropped
//      from the end while their sum over the first C-1 columns is 0, but row 0 always stays (`cnt > 0`); interior zero
//      rows stay.  M = 0 means no GT.  A GT's class is c = int(last column) (truncation); it belongs to anchor set s when
//      class_names[c - 1] == anchor_class_names[s], with numpy's wrap of negative indices (c = 0 -> the last name).
//      Classes whose name index falls outside the list (an IndexError in the reference) match no set.  The sum is taken
//      in column order; rows whose nonzero entries cancel to exactly 0 are not pinned.
//   2. IoU = box_utils.boxes3d_nearest_bev_iou (box_utils.py:238-287), anchor first: r = |limit_period(heading, 0.5, pi)|
//      picks (dx, dy) when r < float(pi/4), else (dy, dx); the box is [x - d/2, y - d/2, x + d/2, y + d/2]; then
//      inter = max(min(x2) - max(x1), 0) * max(min(y2) - max(y1), 0) and iou = inter / max((area_a + area_b) - inter,
//      1e-6), area = (x2 - x1) * (y2 - y1).  limit_period is val - floor(val / pi + 0.5) * pi, and torch on CUDA divides a
//      float tensor by a Python scalar as a multiply by the fp32 reciprocal: val * (1.0f / float(pi)).  That is what the
//      reference computes on the GPU, and what this file does (torch on the CPU divides; the two differ by an ulp in
//      about 15 % of headings, which moves the swap only within an ulp of r = pi/4 or of the wrap).  Every operation is
//      one fp32 rounding, as torch's elementwise kernels round them: this file is compiled without contraction.
//   3. Matching, per (scene, anchor set) over that set's GTs in row order: an anchor's max and FIRST argmax over the GTs;
//      a GT's column maximum over the set's anchors, replaced by -1 when it is 0; an anchor is forced when its IoU with
//      some GT equals that GT's column maximum, and then takes the class of its own argmax GT.  Label: forced -> class;
//      else max < unmatched_threshold -> 0; else max >= matched_threshold -> class; else -1 (the reference's assignment
//      order: positives, then background, then forced).  gt_ious = the anchor's max.  A set without GT: labels 0,
//      gt_ious -0.0 (the reference's zeros * -1), targets and reg_weights 0.
//   4. Targets (ResidualCoder.encode_torch, box_coder_utils.py:13-44) where label > 0, with g = the argmax GT, a = the
//      anchor, sizes clamped below at 1e-5: diag = sqrt(dxa*dxa + dya*dya); (xg-xa)/diag, (yg-ya)/diag, (zg-za)/dza,
//      log(dxg/dxa), log(dyg/dya), log(dzg/dza), rg - ra.  0 elsewhere.  reg_weights = 1 where label > 0, else 0
//      (NORM_BY_NUM_EXAMPLES False).
//   5. Output order: anchor i's outputs go to row i of every scene.  The caller passes the anchors in the reference's
//      output order (each set viewed as (shape[0], shape[1], -1) and concatenated along the last axis, :121-135, so the
//      sets interleave per location) with each anchor's set index.
//
// Cost: pass 1 (at_colmax_kernel) is one thread per anchor with the scene's GT boxes in shared memory; each GT's column
// maximum is a warp max over the fp32 bits (IoU >= +0, so the bits order like the values) and one atomicMax per warp that
// saw a positive IoU.  Pass 2 (at_assign_kernel) recomputes the IoUs with the same device function, so they are bit for
// bit those of pass 1, and writes every output.  Both passes trim and classify the GT rows themselves (rule 1).
#include <math.h>

#include "box_coder.cuh"
#include "common.cuh"

namespace vc {
namespace {

constexpr float PI_F = 3.14159265358979323846f;          // float(np.pi)
constexpr float INV_PI_F = 0x1.45f306p-2f;                // 1.0f / float(np.pi), rounded to fp32 (torch's scalar divide)
constexpr float PI4_F = (float)(3.14159265358979323846 / 4.0);   // np.pi / 4 compared in fp32
constexpr int AT_THREADS = 256;
constexpr int MASK_THREADS = 256;

struct Bev {
    float x1, y1, x2, y2, area;
};

// boxes3d_lidar_to_aligned_bev_boxes + the area of boxes_iou_normal (rule 2)
__device__ __forceinline__ Bev nearest_bev(const float* __restrict__ b) {
    const float h = b[6];
    const float r = fabsf(h - floorf(h * INV_PI_F + 0.5f) * PI_F);
    const bool keep = r < PI4_F;
    const float hx = (keep ? b[3] : b[4]) * 0.5f, hy = (keep ? b[4] : b[3]) * 0.5f;
    Bev o;
    o.x1 = b[0] - hx;
    o.y1 = b[1] - hy;
    o.x2 = b[0] + hx;
    o.y2 = b[1] + hy;
    o.area = (o.x2 - o.x1) * (o.y2 - o.y1);
    return o;
}

__device__ __forceinline__ float iou_nearest(const Bev& a, float4 b, float b_area) {
    const float xl = fmaxf(fminf(a.x2, b.z) - fmaxf(a.x1, b.x), 0.f);
    const float yl = fmaxf(fminf(a.y2, b.w) - fmaxf(a.y1, b.y), 0.f);
    const float inter = xl * yl;
    return inter / fmaxf(a.area + b_area - inter, 1e-6f);
}

struct AtParams {
    const float* anchors;     // [N, 7]
    const int32_t* aset;      // [N]
    const float* gt;          // [B, M, ld]
    uint32_t* colmax;         // [B, S, M] fp32 bits, zeroed
    int32_t* labels;          // [B, N]
    float* targets;           // [B, N, 7]
    float* reg_weights;       // [B, N]
    float* gt_ious;           // [B, N]
    int N, M, ld, S, n_names;
    uint32_t name_sets[VC_ANCHOR_MAX_NAMES];
    float matched[VC_ANCHOR_MAX_SETS], unmatched[VC_ANCHOR_MAX_SETS];
};

struct SceneGt {
    float4 bev[VC_ANCHOR_MAX_GT];
    float area[VC_ANCHOR_MAX_GT];
    uint32_t sets[VC_ANCHOR_MAX_GT];   // bit s: the GT belongs to anchor set s
    int cls[VC_ANCHOR_MAX_GT];
    int last;                          // last row with a nonzero sum (rule 1)
};

// stage scene b's GT rows; returns the trimmed count (rule 1).  Every thread of the CTA must call it.
__device__ int load_scene(const AtParams& p, int b, SceneGt& s) {
    if (threadIdx.x == 0) s.last = 0;
    __syncthreads();
    const float* g = p.gt + (size_t)b * p.M * p.ld;
    for (int j = threadIdx.x; j < p.M; j += blockDim.x) {
        const float* r = g + (size_t)j * p.ld;
        float sum = 0.f;
        for (int k = 0; k < p.ld - 1; ++k) sum += r[k];
        if (sum != 0.f) atomicMax(&s.last, j);
        const Bev e = nearest_bev(r);
        s.bev[j] = make_float4(e.x1, e.y1, e.x2, e.y2);
        s.area[j] = e.area;
        const int c = (int)r[p.ld - 1];
        int n = c - 1;
        if (n < 0) n += p.n_names;
        s.sets[j] = (n >= 0 && n < p.n_names) ? p.name_sets[n] : 0u;
        s.cls[j] = c;
    }
    __syncthreads();
    return p.M == 0 ? 0 : s.last + 1;
}

__global__ void __launch_bounds__(AT_THREADS) at_colmax_kernel(AtParams p) {
    __shared__ SceneGt s;
    const int b = blockIdx.y;
    const int ng = load_scene(p, b, s);
    const int i = blockIdx.x * AT_THREADS + threadIdx.x;
    const bool valid = i < p.N;
    Bev a{};
    int set = -1;
    if (valid) {
        a = nearest_bev(p.anchors + (size_t)i * 7);
        set = p.aset[i];
    }
    uint32_t* cm = p.colmax + (size_t)b * p.S * p.M;
    const int lane = threadIdx.x & 31;
    for (int j = 0; j < ng; ++j) {
        const uint32_t sets = s.sets[j];               // uniform across the CTA
        if (!sets) continue;
        const float v = (set >= 0 && (sets >> set & 1u)) ? iou_nearest(a, s.bev[j], s.area[j]) : 0.f;
        const uint32_t bits = v > 0.f ? __float_as_uint(v) : 0u;
        for (uint32_t q = sets; q; q &= q - 1) {       // one set per GT unless two anchor sets share a class name
            const int t = __ffs(q) - 1;
            const uint32_t m = __reduce_max_sync(0xffffffffu, set == t ? bits : 0u);
            if (lane == 0 && m) atomicMax(cm + (size_t)t * p.M + j, m);
        }
    }
}

__global__ void __launch_bounds__(AT_THREADS) at_assign_kernel(AtParams p) {
    __shared__ SceneGt s;
    const int b = blockIdx.y;
    const int ng = load_scene(p, b, s);
    const int i = blockIdx.x * AT_THREADS + threadIdx.x;
    if (i >= p.N) return;
    const float* anc = p.anchors + (size_t)i * 7;
    const Bev a = nearest_bev(anc);
    const int set = p.aset[i];
    const uint32_t* cm = p.colmax + ((size_t)b * p.S + set) * p.M;
    float best = -1.f;
    int arg = -1;
    bool forced = false;
    for (int j = 0; j < ng; ++j) {
        if (!(s.sets[j] >> set & 1u)) continue;
        const float v = iou_nearest(a, s.bev[j], s.area[j]);
        if (v > best) {
            best = v;
            arg = j;
        }
        const uint32_t c = __ldg(cm + j);
        forced |= v == (c ? __uint_as_float(c) : -1.f);
    }
    const size_t o = (size_t)b * p.N + i;
    float t[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int label = 0;
    float gi = -0.f;
    if (arg >= 0) {
        const int cls = s.cls[arg];
        label = forced ? cls : best < p.unmatched[set] ? 0 : best >= p.matched[set] ? cls : -1;
        gi = best;
        if (label > 0) residual_encode(p.gt + ((size_t)b * p.M + arg) * p.ld, anc, t);   // rule 4
    }
    p.labels[o] = label;
    p.gt_ious[o] = gi;
    p.reg_weights[o] = label > 0 ? 1.f : 0.f;
    float* to = p.targets + o * 7;
#pragma unroll
    for (int k = 0; k < 7; ++k) to[k] = t[k];
}

// rule 0, step 1: coarse occupancy [H/10, W/10] from the points
__global__ void __launch_bounds__(MASK_THREADS) mask_coarse_kernel(const float* __restrict__ pts, int n, int ld, float min_x,
                                                                  float min_y, float inv_stride, int h10, int w10,
                                                                  unsigned char* coarse) {
    const int i = blockIdx.x * MASK_THREADS + threadIdx.x;
    if (i >= n) return;
    const float* r = pts + (size_t)i * ld;
    long long cx = (long long)((r[1] - min_x) * inv_stride);
    long long cy = (long long)((r[2] - min_y) * inv_stride);
    cx = cx < w10 - 1 ? cx : w10 - 1;
    cy = cy < h10 - 1 ? cy : h10 - 1;
    if (cx < -w10 || cy < -h10) return;
    if (cx < 0) cx += w10;
    if (cy < 0) cy += h10;
    coarse[cy * w10 + cx] = 1;
}

// rule 0, step 2: fine cell (r, c) is set when an occupied coarse cell's window covers it.  Row r is covered by coarse
// row cy through i = r - 10 cy in [-10, 10), i.e. cy = r / 10 or r / 10 + 1, and, through the wrap, by cy = 0 when
// r >= H - 10; the same for columns.
__global__ void __launch_bounds__(MASK_THREADS) mask_expand_kernel(const unsigned char* __restrict__ coarse, int H, int W,
                                                                  unsigned char* mask) {
    const int e = blockIdx.x * MASK_THREADS + threadIdx.x;
    if (e >= H * W) return;
    const int r = e / W, c = e % W, h10 = H / 10, w10 = W / 10;
    int cys[3], cxs[3], ny = 0, nx = 0;
    if (r / 10 < h10) cys[ny++] = r / 10;
    if (r / 10 + 1 < h10) cys[ny++] = r / 10 + 1;
    if (r >= H - 10) cys[ny++] = 0;
    if (c / 10 < w10) cxs[nx++] = c / 10;
    if (c / 10 + 1 < w10) cxs[nx++] = c / 10 + 1;
    if (c >= W - 10) cxs[nx++] = 0;
    unsigned char v = 0;
    for (int y = 0; y < ny; ++y)
        for (int x = 0; x < nx; ++x) v |= coarse[cys[y] * w10 + cxs[x]];
    mask[e] = v;
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_anchor_mask(const float* points, int n_points, int ld, float min_x, float min_y, float inv_stride, int H,
                              int W, unsigned char* coarse, unsigned char* mask, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(n_points >= 0 && ld >= 3 && H >= 10 && W >= 10, "anchor mask: bad arguments (n=%d, ld=%d, H=%d, W=%d)",
                 n_points, ld, H, W);
    VC_CHECK_ARG(coarse && mask && (points || n_points == 0), "null pointer");
    if (n_points > 0) {
        mask_coarse_kernel<<<cdiv(n_points, MASK_THREADS), MASK_THREADS, 0, stream>>>(points, n_points, ld, min_x, min_y,
                                                                                   inv_stride, H / 10, W / 10, coarse);
        VC_LAUNCH_CHECK();
    }
    mask_expand_kernel<<<cdiv((long long)H * W, MASK_THREADS), MASK_THREADS, 0, stream>>>(coarse, H, W, mask);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_anchor_targets_ws_bytes(int B, int n_sets, int M) {
    if (B <= 0 || n_sets <= 0 || M <= 0) return 0;
    return (size_t)B * n_sets * M * sizeof(uint32_t);
}

extern "C" int vc_anchor_targets(const float* anchors, const int32_t* anchor_set, int N, int n_sets, const float* matched,
                                 const float* unmatched, const float* gt, int B, int M, int ld, const int32_t* name_sets,
                                 int n_names, int32_t* labels, float* targets, float* reg_weights, float* gt_ious, void* ws,
                                 size_t ws_bytes, vc_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    VC_CHECK_ARG(N >= 0 && B >= 0 && M >= 0 && ld >= 8, "anchor targets: bad arguments (N=%d, B=%d, M=%d, ld=%d)", N, B, M,
                 ld);
    VC_CHECK_ARG(n_sets >= 1 && n_sets <= VC_ANCHOR_MAX_SETS && n_names >= 1 && n_names <= VC_ANCHOR_MAX_NAMES,
                 "anchor targets: %d anchor sets (1..%d), %d class names (1..%d)", n_sets, VC_ANCHOR_MAX_SETS, n_names,
                 VC_ANCHOR_MAX_NAMES);
    if (M > VC_ANCHOR_MAX_GT) {
        set_error("anchor targets: %d GT rows per scene exceed the limit of %d", M, VC_ANCHOR_MAX_GT);
        return VC_ERR_UNSUPPORTED;
    }
    VC_CHECK_ARG(B <= 65535, "anchor targets: %d scenes exceed the grid", B);
    if (N == 0 || B == 0) return VC_OK;
    VC_CHECK_ARG(anchors && anchor_set && matched && unmatched && name_sets && labels && targets && reg_weights && gt_ious &&
                 (gt || M == 0), "null pointer");
    AtParams p{};
    p.anchors = anchors;
    p.aset = anchor_set;
    p.gt = gt;
    p.labels = labels;
    p.targets = targets;
    p.reg_weights = reg_weights;
    p.gt_ious = gt_ious;
    p.N = N;
    p.M = M;
    p.ld = ld;
    p.S = n_sets;
    p.n_names = n_names;
    for (int k = 0; k < n_names; ++k) p.name_sets[k] = (uint32_t)name_sets[k] & ((1u << n_sets) - 1u);
    for (int k = 0; k < n_sets; ++k) {
        p.matched[k] = matched[k];
        p.unmatched[k] = unmatched[k];
    }
    const dim3 grid(cdiv(N, AT_THREADS), B);
    if (M > 0) {
        VC_CHECK_ARG(ws, "null pointer");
        const size_t need = vc_anchor_targets_ws_bytes(B, n_sets, M);
        if (ws_bytes < need) {
            set_error("anchor targets: workspace of %zu bytes, %zu needed", ws_bytes, need);
            return VC_ERR_WORKSPACE;
        }
        p.colmax = (uint32_t*)ws;
        VC_CUDA(cudaMemsetAsync(ws, 0, need, stream));
        at_colmax_kernel<<<grid, AT_THREADS, 0, stream>>>(p);
        VC_LAUNCH_CHECK();
    }
    at_assign_kernel<<<grid, AT_THREADS, 0, stream>>>(p);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
