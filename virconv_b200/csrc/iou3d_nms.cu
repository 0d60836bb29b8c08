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
// The geometry (box_geom.cuh, shared with roi_targets.cu) is __host__ __device__ and this file is compiled without
// floating-point contraction (build.py), and sin/cos come from a polynomial evaluated with explicit fma, so
// vc_boxes_iou_bev_host computes bit for bit what the GPU computes.
#include <math.h>

#include <vector>

#include "box_geom.cuh"
#include "common.cuh"

namespace vc {
namespace {

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
