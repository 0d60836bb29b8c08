// KITTI evaluation (kitti_object_eval_python/eval.py: eval_class for the three metrics of get_official_eval_result)
// over a whole evaluation set in a fixed number of launches — sm_90a, SIMT, no atomics on values, no host read.
//
//   vc_kitti_overlaps   the per-frame [n_dt, n_gt] overlap blocks of one metric, pair p of frame f at pair_off[f] +
//                       j * n_gt + i (detection j, GT i), one thread per pair (kitti_eval_geom.cuh, E1-E6):
//                       metric 0 image_box_overlap (float64), 1 rotate_iou_gpu_eval on (x, z, l, w, ry) with criterion -1
//                       (float32, widened), 2 d3_box_overlap (float32, widened).
//   vc_kitti_rotate_iou rotate_iou_gpu_eval itself: boxes [N, 5], query boxes [K, 5] -> float32 [N, K].
//   vc_kitti_eval       the overlaps of the three metrics, then for every lane (metric, class, difficulty, overlap
//                       setting — eval_class's loop order):
//     1. ignore flags   clean_data per object, class and difficulty (one thread per object and (class, difficulty));
//     2. score order    the detections sorted by score, high to low (one CTA, LSD radix sort on the float64 bits);
//     3. pass 1         compute_statistics_jit(thresh=0, compute_fp=False) per (lane, frame): marks the detections
//                       counted as true positives;
//     4. thresholds     per lane: the number of valid GT and of marked detections, get_thresholds' selection as ranks
//                       (it depends on the ranks only), then the marked scores at those ranks, read along the score
//                       order with a CTA scan;
//     5. pass 2         compute_statistics_jit(compute_fp=True) per (lane, frame) at every threshold, with the
//                       DontCare step for metric 0 and the AOS similarity; CTA partial sums over 128 frames in a fixed
//                       tree;
//     6. tables         per lane: the partial sums in segment order, recall, precision and AOS, and the running max of
//                       precision and AOS over the higher thresholds (NaN propagates, as np.max does).
//   Nine launches whatever the frame count; tp / fp / fn are integer sums and the similarity sums run in a fixed order,
//   so two runs are bit-identical.
#include <math.h>

#include "common.cuh"
#include "kitti_eval_geom.cuh"

namespace vc {
namespace {

constexpr int GW = VC_KE_ROW;      // doubles per packed object row
constexpr int NS = VC_KE_SAMPLES;  // 41
constexpr int LW = VC_KE_LANE_W;
constexpr int MATCH_T = 128;       // pass-2 CTA: frames per segment
constexpr int SORT_T = 1024;
constexpr double NO_DET = -10000000.0;
__constant__ int MIN_HEIGHT[3] = {40, 25, 25};
__constant__ int MAX_OCCLUSION[3] = {0, 1, 2};
__constant__ double MAX_TRUNCATION[3] = {0.15, 0.3, 0.5};

struct Frames {
    const double* gt;
    const double* dt;
    const long long* gt_off;
    const long long* dt_off;
    const long long* pair_off;
    int F;
};

__device__ __forceinline__ int frame_of(const long long* off, int F, long long p) {  // last f with off[f] <= p
    int lo = 0, hi = F - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= p) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(256) overlap_kernel(Frames fr, long long P, int metric, double* __restrict__ ov) {
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int f = frame_of(fr.pair_off, fr.F, p);
    const int ng = (int)(fr.gt_off[f + 1] - fr.gt_off[f]);
    const long long q = p - fr.pair_off[f];
    const int j = (int)(q / ng), i = (int)(q % ng);
    const double* g = fr.gt + (fr.gt_off[f] + i) * GW;
    const double* d = fr.dt + (fr.dt_off[f] + j) * GW;
    double r;
    if (metric == 0) {
        r = ke::image_iou(d, g, -1);
    } else {
        const ke::RBox gb{(float)g[5], (float)g[7], (float)g[8], (float)g[10], (float)g[11]};
        const ke::RBox db{(float)d[5], (float)d[7], (float)d[8], (float)d[10], (float)d[11]};
        if (metric == 1) {
            r = (double)ke::rotate_iou(gb, db, -1);
        } else {
            const float rinc = ke::rotate_iou(gb, db, 2);
            r = 0.0;
            if (rinc > 0.0f) {
                const double iw = fmin(d[6], g[6]) - fmax(d[6] - d[9], g[6] - g[9]);
                if (iw > 0.0) {
                    const double inc = iw * (double)rinc;
                    r = (double)(float)(inc / ((d[8] * d[9] * d[10] + g[8] * g[9] * g[10]) - inc));
                }
            }
        }
    }
    ov[p] = r;
}

__global__ void __launch_bounds__(256) rotate_iou_kernel(const float* __restrict__ b, const float* __restrict__ q, int N,
                                                         int K, int criterion, float* __restrict__ out) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)N * K) return;
    const int n = (int)(e / K), k = (int)(e % K);
    const ke::RBox bb{b[5 * n], b[5 * n + 1], b[5 * n + 2], b[5 * n + 3], b[5 * n + 4]};
    const ke::RBox qb{q[5 * k], q[5 * k + 1], q[5 * k + 2], q[5 * k + 3], q[5 * k + 4]};
    out[e] = ke::rotate_iou(qb, bb, criterion);
}

struct Classes {
    int c[VC_KE_MAX_CLASSES];
};

// clean_data.  Class ids: car 0, pedestrian 1, cyclist 2, van 3, person_sitting 4, truck 5, other -1.
__global__ void __launch_bounds__(256) flags_kernel(Frames fr, int NG, int ND, int C, Classes cls,
                                                    signed char* __restrict__ ig, signed char* __restrict__ idt) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per = (long long)NG + ND;
    if (e >= per * C * 3) return;
    const int cd = (int)(e / per), o = (int)(e % per);
    const int c = cls.c[cd / 3], d = cd % 3;
    if (o < NG) {
        const double* g = fr.gt + (long long)o * GW;
        const int gc = (int)g[14];
        const int valid = gc == c ? 1 : ((c == 1 && gc == 4) || (c == 0 && gc == 3)) ? 0 : -1;
        const double h = g[3] - g[1];
        const bool ignore = g[13] > MAX_OCCLUSION[d] || g[12] > MAX_TRUNCATION[d] || h <= MIN_HEIGHT[d];
        ig[(long long)cd * NG + o] = (valid == 1 && !ignore) ? 0 : (valid == 0 || (ignore && valid == 1)) ? 1 : -1;
    } else {
        const int j = o - NG;
        const double* t = fr.dt + (long long)j * GW;
        const double h = fabs(t[3] - t[1]);
        idt[(long long)cd * ND + j] = h < MIN_HEIGHT[d] ? 1 : ((int)t[13] == c ? 0 : -1);
    }
}

__device__ __forceinline__ unsigned long long desc_key(double s) {
    unsigned long long u = (unsigned long long)__double_as_longlong(s);
    u = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
    return ~u;
}

// one CTA: order[] = detection indices by score, high to low (8-bit LSD passes; a pass whose digit is the same for
// every key is skipped)
__global__ void __launch_bounds__(SORT_T) sort_kernel(const double* __restrict__ dt, int ND,
                                                      unsigned long long* k0, unsigned long long* k1,
                                                      int* i0, int* i1, int* __restrict__ order) {
    __shared__ int hist[256];
    __shared__ int wcnt[SORT_T / 32][256];
    __shared__ int skip;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    for (int e = tid; e < ND; e += SORT_T) {
        k0[e] = desc_key(dt[(long long)e * GW + 12]);
        i0[e] = e;
    }
    __syncthreads();
    for (int pass = 0; pass < 8; ++pass) {
        const int sh = pass * 8;
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        for (int e = tid; e < ND; e += SORT_T) atomicAdd(&hist[(int)((k0[e] >> sh) & 255)], 1);
        __syncthreads();
        if (tid == 0) {
            int acc = 0;
            skip = 0;
            for (int b = 0; b < 256; ++b) {
                const int h = hist[b];
                if (h == ND) skip = 1;
                hist[b] = acc;
                acc += h;
            }
        }
        __syncthreads();
        if (skip) continue;
        for (int base = 0; base < ND; base += SORT_T) {
            for (int x = tid; x < (SORT_T / 32) * 256; x += SORT_T) (&wcnt[0][0])[x] = 0;
            __syncthreads();
            const int e = base + tid;
            const bool valid = e < ND;
            unsigned long long key = valid ? k0[e] : 0ull;
            const int dig = valid ? (int)((key >> sh) & 255) : 256;
            const unsigned peers = __match_any_sync(0xffffffffu, dig);
            const int rank = __popc(peers & ((1u << lane) - 1u));
            if (valid && rank == 0) wcnt[w][dig] = __popc(peers);
            __syncthreads();
            if (tid < 256) {
                int acc = hist[tid];
                for (int ww = 0; ww < SORT_T / 32; ++ww) {
                    const int t = wcnt[ww][tid];
                    wcnt[ww][tid] = acc;
                    acc += t;
                }
                hist[tid] = acc;
            }
            __syncthreads();
            if (valid) {
                const int pos = wcnt[w][dig] + rank;
                k1[pos] = key;
                i1[pos] = i0[e];
            }
            __syncthreads();
        }
        unsigned long long* tk = k0; k0 = k1; k1 = tk;
        int* ti = i0; i0 = i1; i1 = ti;
    }
    for (int e = tid; e < ND; e += SORT_T) order[e] = i0[e];   // i0: the buffer the last executed pass wrote
}

struct Lanes {
    const double* mo;       // [L] min overlap
    int C, K, L;
};

__device__ __forceinline__ void lane_of(const Lanes& ln, int lane, int& m, int& cd) {
    const int per_m = ln.C * 3 * ln.K;
    m = lane / per_m;
    cd = (lane % per_m) / ln.K;
}

struct Stats {
    int tp, fp, fn;
    double sim;
};

// compute_statistics_jit for one frame.  as[j]: bit 0 assigned, bit 1 counted as a true positive.
__device__ Stats match(const double* __restrict__ o, int ng, int nd, const signed char* __restrict__ ig,
                       const signed char* __restrict__ idt, const double* __restrict__ g, const double* __restrict__ d,
                       unsigned char* __restrict__ as, double mo, double thresh, bool fp_mode, int metric, bool aos) {
    Stats s{0, 0, 0, 0.0};
    for (int j = 0; j < nd; ++j) as[j] = 0;
    for (int i = 0; i < ng; ++i) {
        const int igi = ig[i];
        if (igi == -1) continue;
        int det = -1;
        double valid = NO_DET, maxov = 0.0;
        bool ass_ign = false;
        for (int j = 0; j < nd; ++j) {
            const int idj = idt[j];
            if (idj == -1 || (as[j] & 1)) continue;
            const double sc = d[(long long)j * GW + 12];
            if (fp_mode && sc < thresh) continue;
            const double ov = o[(long long)j * ng + i];
            if (!fp_mode) {
                if (ov > mo && sc > valid) {
                    det = j;
                    valid = sc;
                }
            } else if (ov > mo && (ov > maxov || ass_ign) && idj == 0) {
                maxov = ov;
                det = j;
                valid = 1.0;
                ass_ign = false;
            } else if (ov > mo && valid == NO_DET && idj == 1) {
                det = j;
                valid = 1.0;
                ass_ign = true;
            }
        }
        if (valid == NO_DET) {
            if (igi == 0) ++s.fn;
        } else if (igi == 1 || idt[det] == 1) {
            as[det] |= 1;
        } else {
            ++s.tp;
            as[det] |= 3;
            if (aos) s.sim += (1.0 + cos(g[(long long)i * GW + 4] - d[(long long)det * GW + 4])) / 2.0;
        }
    }
    if (fp_mode) {
        for (int j = 0; j < nd; ++j)
            if (!((as[j] & 1) || idt[j] != 0 || d[(long long)j * GW + 12] < thresh)) ++s.fp;
        if (metric == 0) {
            int nstuff = 0;
            for (int i = 0; i < ng; ++i) {
                if (g[(long long)i * GW + 15] == 0.0) continue;  // DontCare boxes, in GT order
                for (int j = 0; j < nd; ++j) {
                    if ((as[j] & 1) || idt[j] != 0 || d[(long long)j * GW + 12] < thresh) continue;
                    if (ke::image_iou(d + (long long)j * GW, g + (long long)i * GW, 0) > mo) {
                        as[j] |= 1;
                        ++nstuff;
                    }
                }
            }
            s.fp -= nstuff;
        }
        if (aos && !(s.tp > 0 || s.fp > 0)) s.sim = -1.0;
    }
    return s;
}

struct EvalArgs {
    Frames fr;
    Lanes ln;
    int NG, ND, S, compute_aos;
    long long P;
    const double* ov;            // [3][P]
    const signed char* ig;       // [C*3][NG]
    const signed char* idt;      // [C*3][ND]
    unsigned char* as;           // [L][ND]
    const int* order;            // [ND]
    int* part_i;                 // [L][S][NS][3]
    double* part_d;              // [L][S][NS]
    double* out;                 // [L][LW]
};

__global__ void __launch_bounds__(256) pass1_kernel(EvalArgs a) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (long long)a.ln.L * a.fr.F) return;
    const int lane = (int)(e / a.fr.F), f = (int)(e % a.fr.F);
    int m, cd;
    lane_of(a.ln, lane, m, cd);
    const long long g0 = a.fr.gt_off[f], j0 = a.fr.dt_off[f];
    const int ng = (int)(a.fr.gt_off[f + 1] - g0), nd = (int)(a.fr.dt_off[f + 1] - j0);
    match(a.ov + m * a.P + a.fr.pair_off[f], ng, nd, a.ig + (long long)cd * a.NG + g0, a.idt + (long long)cd * a.ND + j0,
          a.fr.gt + g0 * GW, a.fr.dt + j0 * GW, a.as + (long long)lane * a.ND + j0, a.ln.mo[lane], 0.0, false, m, false);
}

template <typename T>
__device__ T block_sum(T v, T* sh) {  // fixed-order tree over blockDim.x (a power of two); result in every thread
    const int tid = threadIdx.x;
    sh[tid] = v;
    __syncthreads();
    for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
        if (tid < s) sh[tid] = sh[tid] + sh[tid + s];
        __syncthreads();
    }
    const T r = sh[0];
    __syncthreads();
    return r;
}

// one CTA per lane (256 threads)
__global__ void __launch_bounds__(256) thresholds_kernel(EvalArgs a) {
    __shared__ long long shl[256];
    __shared__ int ranks[NS];
    __shared__ int n_sel;
    const int lane = blockIdx.x, tid = threadIdx.x;
    int m, cd;
    lane_of(a.ln, lane, m, cd);
    const unsigned char* as = a.as + (long long)lane * a.ND;
    long long nv = 0, nh = 0;
    for (int i = tid; i < a.NG; i += 256) nv += a.ig[(long long)cd * a.NG + i] == 0;
    for (int j = tid; j < a.ND; j += 256) nh += (as[j] >> 1) & 1;
    nv = block_sum(nv, shl);
    nh = block_sum(nh, shl);
    if (tid == 0) {
        // get_thresholds over ranks: rank i is skipped while (r - cur) < (cur - l), l = (i+1)/num_gt, r = (i+2)/num_gt,
        // except the last; the test is monotone in i, so the walk starts a few ranks below where it turns.
        int cnt = 0;
        double cur = 0.0;
        long long i = 0;
        const double ng = (double)nv;
        while (i < nh && cnt < NS) {
            const long long guess = (long long)floor(ng * cur - 1.5) - 3;
            if (guess > i) i = guess < nh - 1 ? guess : nh - 1;   // the last rank is always taken
            for (; i < nh; ++i) {
                const double l = (double)(i + 1) / ng;
                const double r = i < nh - 1 ? (double)(i + 2) / ng : l;
                if (!((r - cur) < (cur - l) && i < nh - 1)) break;
            }
            if (i >= nh) break;
            ranks[cnt++] = (int)i;
            cur += 1.0 / (NS - 1.0);
            ++i;
        }
        n_sel = cnt;
    }
    __syncthreads();
    double* out = a.out + (long long)lane * LW;
    const int T = n_sel;
    if (tid == 0) out[0] = (double)T;
    long long base = 0;
    for (int e0 = 0; e0 < a.ND && T > 0; e0 += 256) {
        const int e = e0 + tid;
        const int j = e < a.ND ? a.order[e] : 0;
        const long long hit = e < a.ND ? (as[j] >> 1) & 1 : 0;
        // inclusive scan in shared memory (Hillis-Steele)
        shl[tid] = hit;
        __syncthreads();
        for (int s = 1; s < 256; s <<= 1) {
            const long long v = tid >= s ? shl[tid - s] : 0;
            __syncthreads();
            shl[tid] += v;
            __syncthreads();
        }
        const long long rank = base + shl[tid] - hit;
        if (hit) {
            int lo = 0, hi = T - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (ranks[mid] < rank) lo = mid + 1; else hi = mid;
            }
            if (ranks[lo] == rank) out[1 + lo] = a.fr.dt[(long long)j * GW + 12];
        }
        base += shl[255];
        __syncthreads();
    }
}

// grid (L, S), MATCH_T threads: frame seg * MATCH_T + tid at every threshold of the lane
__global__ void __launch_bounds__(MATCH_T) pass2_kernel(EvalArgs a) {
    __shared__ int shi[MATCH_T];
    __shared__ double shd[MATCH_T];
    const int lane = blockIdx.x, seg = blockIdx.y, tid = threadIdx.x;
    const int f = seg * MATCH_T + tid;
    int m, cd;
    lane_of(a.ln, lane, m, cd);
    const double* out = a.out + (long long)lane * LW;
    const int T = (int)out[0];
    const bool aos = a.compute_aos && m == 0;
    long long g0 = 0, j0 = 0;
    int ng = 0, nd = 0;
    if (f < a.fr.F) {
        g0 = a.fr.gt_off[f];
        j0 = a.fr.dt_off[f];
        ng = (int)(a.fr.gt_off[f + 1] - g0);
        nd = (int)(a.fr.dt_off[f + 1] - j0);
    }
    for (int t = 0; t < T; ++t) {
        Stats s{0, 0, 0, 0.0};
        if (f < a.fr.F)
            s = match(a.ov + m * a.P + a.fr.pair_off[f], ng, nd, a.ig + (long long)cd * a.NG + g0,
                      a.idt + (long long)cd * a.ND + j0, a.fr.gt + g0 * GW, a.fr.dt + j0 * GW,
                      a.as + (long long)lane * a.ND + j0, a.ln.mo[lane], out[1 + t], true, m, aos);
        const int tp = block_sum(s.tp, shi), fp = block_sum(s.fp, shi), fn = block_sum(s.fn, shi);
        const double sim = block_sum(s.sim != -1.0 ? s.sim : 0.0, shd);
        if (tid == 0) {
            int* pi = a.part_i + (((long long)lane * a.S + seg) * NS + t) * 3;
            pi[0] = tp;
            pi[1] = fp;
            pi[2] = fn;
            a.part_d[((long long)lane * a.S + seg) * NS + t] = sim;
        }
    }
}

__device__ __forceinline__ double max_nan(double x, double y) { return (isnan(x) || isnan(y)) ? NAN : fmax(x, y); }

__global__ void __launch_bounds__(128) tables_kernel(EvalArgs a) {
    const int lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= a.ln.L) return;
    int m, cd;
    lane_of(a.ln, lane, m, cd);
    const bool aos = a.compute_aos && m == 0;
    double* out = a.out + (long long)lane * LW;
    const int T = (int)out[0];
    double* pr = out + 1 + NS;
    double* prec = pr + 4 * NS;
    double* rec = prec + NS;
    double* ao = rec + NS;
    for (int t = 0; t < T; ++t) {
        long long tp = 0, fp = 0, fn = 0;
        double sim = 0.0;
        for (int s = 0; s < a.S; ++s) {
            const int* pi = a.part_i + (((long long)lane * a.S + s) * NS + t) * 3;
            tp += pi[0];
            fp += pi[1];
            fn += pi[2];
            sim += a.part_d[((long long)lane * a.S + s) * NS + t];
        }
        pr[4 * t] = (double)tp;
        pr[4 * t + 1] = (double)fp;
        pr[4 * t + 2] = (double)fn;
        pr[4 * t + 3] = sim;
        rec[t] = (double)tp / (double)(tp + fn);
        prec[t] = (double)tp / (double)(tp + fp);
        if (aos) ao[t] = sim / (double)(tp + fp);
    }
    double run_p = prec[NS - 1], run_a = ao[NS - 1];
    for (int t = NS - 1; t >= 0; --t) {
        run_p = t == NS - 1 ? prec[t] : max_nan(prec[t], run_p);
        run_a = t == NS - 1 ? ao[t] : max_nan(ao[t], run_a);
        if (t < T) {
            prec[t] = run_p;
            if (aos) ao[t] = run_a;
        }
    }
}

struct Ws {
    signed char *ig, *idt;
    unsigned char* as;
    unsigned long long *k0, *k1;
    int *i0, *i1, *order, *part_i;
    double* part_d;
    size_t bytes;
};

Ws carve(void* base, int F, int NG, int ND, int C, int K) {
    const long long L = 3ll * C * 3 * K, S = cdiv(F > 0 ? F : 1, MATCH_T);
    Ws w{};
    char* p = (char*)base;
    size_t off = 0;
    auto take = [&](size_t n) {
        char* r = p ? p + off : nullptr;
        off += (n + 255) & ~(size_t)255;
        return r;
    };
    w.k0 = (unsigned long long*)take(sizeof(unsigned long long) * ND);
    w.k1 = (unsigned long long*)take(sizeof(unsigned long long) * ND);
    w.part_d = (double*)take(sizeof(double) * L * S * NS);
    w.i0 = (int*)take(sizeof(int) * ND);
    w.i1 = (int*)take(sizeof(int) * ND);
    w.order = (int*)take(sizeof(int) * ND);
    w.part_i = (int*)take(sizeof(int) * 3 * L * S * NS);
    w.ig = (signed char*)take((size_t)C * 3 * NG);
    w.idt = (signed char*)take((size_t)C * 3 * ND);
    w.as = (unsigned char*)take((size_t)L * ND);
    w.bytes = off;
    return w;
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" int vc_kitti_overlaps(const double* gt, const double* dt, const long long* offs, int F, long long n_pair,
                                 int metric, double* ov, vc_stream_t stream) {
    VC_CHECK_ARG(F >= 0 && n_pair >= 0 && metric >= 0 && metric <= 2, "kitti overlaps: bad arguments (F=%d, P=%lld, metric=%d)",
                 F, n_pair, metric);
    if (n_pair == 0) return VC_OK;
    VC_CHECK_ARG(gt && dt && offs && ov, "null pointer");
    VC_CHECK_ARG(n_pair <= 256ll * 0x7fffffff, "kitti overlaps: %lld pairs exceed the launch grid", n_pair);
    const Frames fr{gt, dt, offs, offs + (F + 1), offs + 2 * (F + 1), F};
    overlap_kernel<<<cdiv(n_pair, 256), 256, 0, (cudaStream_t)stream>>>(fr, n_pair, metric, ov);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" int vc_kitti_rotate_iou(const float* boxes, const float* qboxes, int N, int K, int criterion, float* out,
                                   vc_stream_t stream) {
    VC_CHECK_ARG(N >= 0 && K >= 0, "kitti rotate iou: bad arguments (N=%d, K=%d)", N, K);
    const long long M = (long long)N * K;
    if (M == 0) return VC_OK;
    VC_CHECK_ARG(boxes && qboxes && out, "null pointer");
    VC_CHECK_ARG(M <= 256ll * 0x7fffffff, "kitti rotate iou: %lld pairs exceed the launch grid", M);
    rotate_iou_kernel<<<cdiv(M, 256), 256, 0, (cudaStream_t)stream>>>(boxes, qboxes, N, K, criterion, out);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

extern "C" size_t vc_kitti_eval_ws_bytes(int F, int NG, int ND, int C, int K) {
    if (F < 0 || NG < 0 || ND < 0 || C < 1 || K < 1) return 0;
    return carve(nullptr, F, NG, ND, C, K).bytes;
}

extern "C" int vc_kitti_eval(const double* gt, const double* dt, const long long* offs, const double* lane_mo, int F,
                             int NG, int ND, long long n_pair, int C, const int* classes, int K, int compute_aos,
                             double* ov, double* out, void* ws, size_t ws_bytes, vc_stream_t stream) {
    VC_CHECK_ARG(F >= 0 && NG >= 0 && ND >= 0 && n_pair >= 0, "kitti eval: bad sizes (F=%d, NG=%d, ND=%d)", F, NG, ND);
    VC_CHECK_ARG(C >= 1 && C <= VC_KE_MAX_CLASSES && K >= 1 && K <= VC_KE_MAX_OVERLAPS,
                 "kitti eval: %d classes (1..%d), %d overlap settings (1..%d)", C, VC_KE_MAX_CLASSES, K,
                 VC_KE_MAX_OVERLAPS);
    VC_CHECK_ARG(classes, "null pointer");
    Classes cls{};
    for (int c = 0; c < C; ++c) {
        VC_CHECK_ARG(classes[c] >= 0 && classes[c] < 6, "kitti eval: class id %d (0..5)", classes[c]);
        cls.c[c] = classes[c];
    }
    const Ws w = carve(ws, F, NG, ND, C, K);
    VC_CHECK_ARG(ws_bytes >= w.bytes, "kitti eval: workspace of %zu bytes, %zu needed", ws_bytes, w.bytes);
    VC_CHECK_ARG(offs && lane_mo && out && (n_pair == 0 || ov) && (NG == 0 || gt) && (ND == 0 || dt), "null pointer");
    const int L = 3 * C * 3 * K;
    const int S = cdiv(F > 0 ? F : 1, MATCH_T);
    cudaStream_t st = (cudaStream_t)stream;
    VC_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * L * LW, st));
    if (F == 0) return VC_OK;
    for (int m = 0; m < 3; ++m) {
        const int rc = vc_kitti_overlaps(gt, dt, offs, F, n_pair, m, ov + m * n_pair, stream);
        if (rc != VC_OK) return rc;
    }
    const Frames fr{gt, dt, offs, offs + (F + 1), offs + 2 * (F + 1), F};
    const long long nf = (long long)(NG + ND) * C * 3;
    if (nf > 0) {
        flags_kernel<<<cdiv(nf, 256), 256, 0, st>>>(fr, NG, ND, C, cls, w.ig, w.idt);
        VC_LAUNCH_CHECK();
    }
    if (ND > 0) {
        sort_kernel<<<1, SORT_T, 0, st>>>(dt, ND, w.k0, w.k1, w.i0, w.i1, w.order);
        VC_LAUNCH_CHECK();
    }
    EvalArgs a{fr, Lanes{lane_mo, C, K, L}, NG, ND, S, compute_aos ? 1 : 0, n_pair, ov, w.ig, w.idt, w.as, w.order,
               w.part_i, w.part_d, out};
    pass1_kernel<<<cdiv((long long)L * F, 256), 256, 0, st>>>(a);
    VC_LAUNCH_CHECK();
    thresholds_kernel<<<L, 256, 0, st>>>(a);
    VC_LAUNCH_CHECK();
    pass2_kernel<<<dim3(L, S), MATCH_T, 0, st>>>(a);
    VC_LAUNCH_CHECK();
    tables_kernel<<<cdiv(L, 128), 128, 0, st>>>(a);
    VC_LAUNCH_CHECK();
    return VC_OK;
}
