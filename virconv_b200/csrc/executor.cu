// Plan executor: one C-ABI call runs a whole backbone forward (or backward) — sm_90a.
//
// The reference drives its backbone layer by layer from Python (spconv_backbone.py:609-699 VirConvL8x.forward, :207-229
// NRConvBlock.forward, :339-535 VirConv8x.forward): ~100 operator calls and ~220 kernel launches per training step,
// whose host time can exceed the time the kernels take to run.
// Here the host side of that loop is native: Python describes the layer graph ONCE as a small op list (the "plan"),
// and vc_exec_forward / vc_exec_backward walk it, carving every activation, rulebook and scratch buffer out of one
// caller-owned arena and enqueueing the same kernels the per-operator entry points launch.
//
//   * two streams: index ops (rulebooks, voxel->pixel projection; they depend on coordinates only) run on the SIDE
//     stream and run ahead of the feature ops (conv+BN+ReLU, concat) on the MAIN stream; the four data-dependent row
//     counts of the strided convs are read back on the side stream, so the host never waits for feature kernels;
//   * cross-stream dependencies are CUDA events from a small library-owned pool; the arena is bump-allocated and never
//     reused inside a step, so there are no memory hazards between the streams;
//   * all tensor-core weight images of the step are produced by one launch (tc_prep_images);
//   * backward walks the list in reverse with gradient accumulation rules (first contribution writes, later ones add).
// The state a forward leaves behind for its backward (buffer addresses, row counts) is a plain host struct in a
// caller-owned blob; the library keeps nothing between calls except the event pool.
#include <cuda_bf16.h>

#include <new>

#include "common.cuh"

namespace vc {
namespace {

constexpr int MAX_OPS = 256, MAX_F = 160, MAX_I = 64, MAX_RB = 64, MAX_L = 96, OPI = 24, OPF = 8;
constexpr uint64_t STATE_MAGIC = 0x5643455845433031ULL;  // "VCEXEC01"
enum { OP_SUBM_RB = 1, OP_CONV_RB = 2, OP_INDEX2UV = 3, OP_CBR = 4, OP_CAT = 5, OP_DISCARD = 6 };
enum { G_EMPTY = 0, G_EXT = 1, G_OWN = 2 };
// op int fields
enum { F_KIND = 0, F_STREAM = 1, F_A = 2, F_B = 3, F_C = 4, F_NDIM = 5, F_KS = 6, F_ST = 9, F_PD = 12, F_DL = 15, F_CIN = 18,
       F_COUT = 19, F_LAYER = 20, F_X0 = 21, F_X1 = 22, F_X2 = 23 };
// layer pointer table columns
enum { P_W = 0, P_GAMMA, P_BETA, P_RM, P_RV, P_NBT, P_DW, P_DGAMMA, P_DBETA, P_COLS };

struct ISet {
    int32_t* idx;
    const int* n_dev;      // static mode: the row count lives on the device and `n` is the capacity of the buffers
    int n, ndim, shape[3];
    int ev;  // event to wait on when consumed from the other stream (-1: none), stream that produced it
    int prod;
};
struct FSlot {
    float* f32;            // NULL where no reader needs fp32 (the bf16 kernels read the shadow)
    void* bf16;
    float* grad;           // [rows, c], row pitch gld
    const int* n_dev;      // static mode (see ISet)
    int rows, c, ld;       // ld: row pitch of f32 / bf16 (> c: a column slice of an in-place concat)
    int gld;               // row pitch of grad (> c: a column slice of the concat's gradient; only scatter dgrads and BN read it)
    int grad_state, ev, prod;
};
struct RBk {
    int32_t *nbr, *nbr_bwd, *pair_num;
    const int *n_in_dev, *n_out_dev;   // static mode (see ISet); table pitches are n_out (nbr) and n_in (nbr_bwd)
    int K, n_in, n_out, subm, unique, ev, prod;
    G2Prep g2;             // deterministic mode, many-to-one table: the gather-form dgrad's groups and table (gather2d.cu)
};
constexpr int CTR_PER_LAYER = 20;  // forward, dgrad, up to 14 wgrad passes (C_in = C_out = 64, K = 27: 14 groups, one per pass in wgrad_tc3),
                                   // the forward's grid barrier (BN inside the conv); a multiple of 4: the wgrad accumulators
                                   // that follow the counters are accessed as float4
constexpr int CTR_BN_BAR = 16;

// conv launches of a layer; the values are the timing records' kinds (vc_exec_timing_read, executor.KIND_NAMES)
enum ConvKind : int { K_NONE = -1 /* no input gradient */, K_FWD_F32 = 0, K_FWD_TC = 1, K_DGRAD_F32 = 2, K_DGRAD_TC = 3,
                      K_DGRAD_SCATTER_F32 = 4, K_WGRAD_F32 = 5, K_WGRAD_TC = 6, K_DGRAD_SCATTER_TC = 7,
                      K_DGRAD_GATHER2D_F32 = 8, K_DGRAD_GATHER2D_TC = 9 };

struct Layer {
    float *x, *y, *stats;
    double* sums;          // [4*cout]: forward sums, backward sums
    int* tile_ctr;         // [CTR_PER_LAYER] tile-scheduler counters of the persistent kernels (forward, dgrad, wgrad passes), zeroed with the sums
    float* wscratch;       // [K][cin][cout] fp32 accumulator of the persistent wgrad kernel (zeroed with the sums), or NULL
    void *wimg_fwd, *wimg_dgrad;
    int in_slot, out_slot, rb, cin, cout;
    ConvKind fwd, dgrad, wgrad;   // chosen by choose_kernels
    // what vc_exec_backward used for this layer (vc_exec_query 6): the upstream gradient (row pitch dy_ld) and the BN
    // backward's outputs, dx (NULL where no fp32 reader exists) and its bf16 shadow dxb (bf16 mode)
    const float* dy;
    float* dx;
    void* dxb;
    int dy_ld;
};
struct Disc {              // a DISCARD op (StVD layer discard): what its selection left behind
    int32_t *keep, *pos;   // keep [n_in]: kept rows ascending, tail -1; pos [n_in]: position in keep or -1
    int32_t* kept_dev;     // device int32[1]: number of kept rows
    int n_in, k, site;     // k: kept rows (exact mode) or the capacity n_in (static mode)
};
struct State {
    uint64_t magic;
    size_t used;           // arena bytes in use after the last call
    int n_ops, n_layers, training, precision, batch_size, is_static;
    int deterministic;     // flags bit 2 of the forward: fixed-order reductions, no float atomics (the backward follows it)
    size_t det_bytes;      // arena bytes of the deterministic mode's partials, tables and operands (vc_exec_query 0)
    ISet iset[MAX_I];
    FSlot f[MAX_F];
    RBk rb[MAX_RB];
    Layer layer[MAX_L];
    Disc disc[MAX_OPS];    // by op index
};

struct Arena {
    char* base;
    size_t cap, used;
    bool failed;
    void* alloc(size_t bytes) {
        size_t a = (used + 255) & ~(size_t)255;
        if (a + bytes > cap) {
            failed = true;
            used = a + bytes;   // keep counting: the error message reports what would have been needed so far
            return nullptr;
        }
        used = a + bytes;
        return base + a;
    }
};

// library-owned event pool (cross-stream ordering only; timing disabled).  An event may be re-recorded as soon as the
// wait on its previous recording has been ENQUEUED, so a small round-robin pool is enough.
constexpr int EV_POOL = 512;   // > the events of one forward / backward call: the cursor restarts at every call
// (process-wide, not per thread: autograd runs backward on its own thread; one process drives one device)
cudaEvent_t g_ev[EV_POOL];
int g_ev_dev = -1, g_ev_next = 0;

int ev_init() {
    int dev = 0;
    VC_CUDA(cudaGetDevice(&dev));
    if (g_ev_dev == dev) return VC_OK;
    if (g_ev_dev >= 0)
        for (int i = 0; i < EV_POOL; ++i) cudaEventDestroy(g_ev[i]);
    for (int i = 0; i < EV_POOL; ++i) VC_CUDA(cudaEventCreateWithFlags(&g_ev[i], cudaEventDisableTiming));
    g_ev_dev = dev;
    g_ev_next = 0;
    return VC_OK;
}

// optional per-kernel timing (bench.py's roofline pass): event pairs around the conv launches
struct TimeRec {
    cudaEvent_t a, b;
    int kind, layer;   // kind: a ConvKind
};
constexpr int T_MAX = 4096;
TimeRec g_t[T_MAX];
int g_t_n = 0, g_t_created = 0;
bool g_timing = false;

struct Timed {
    int idx;
    cudaStream_t st;
    Timed(int kind, int layer, cudaStream_t s, bool launches = true) : idx(-1), st(s) {   // launches: the kernel is enqueued
        if (!launches || !g_timing || g_t_n >= T_MAX) return;
        if (g_t_n >= g_t_created) {
            if (cudaEventCreate(&g_t[g_t_n].a) != cudaSuccess || cudaEventCreate(&g_t[g_t_n].b) != cudaSuccess) return;
            g_t_created = g_t_n + 1;
        }
        idx = g_t_n++;
        g_t[idx].kind = kind;
        g_t[idx].layer = layer;
        cudaEventRecord(g_t[idx].a, st);
    }
    ~Timed() {
        if (idx >= 0) cudaEventRecord(g_t[idx].b, st);
    }
};

__global__ void __launch_bounds__(256) add_kernel(const float4* a, const float4* b, float4* c, size_t n4) {   // c may alias a or b
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n4; i += stride) {
        float4 x = a[i], y = b[i];
        c[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
    }
}

// backward of the channel concat: da = dcat[:, :ca] (+ a_add), db = dcat[:, ca:] (+ b_add); add pointers may alias
// the outputs (in-place accumulation) or be NULL
__global__ void __launch_bounds__(256) cat2_bwd_kernel(const float4* __restrict__ dcat, int n, int ca4, int cb4,
                                                       float4* da, const float4* a_add, float4* db, const float4* b_add) {
    const int c4 = ca4 + cb4;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)n * c4, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < total; i += stride) {
        const size_t r = i / c4;
        const int c = (int)(i % c4);
        float4 v = dcat[i];
        if (c < ca4) {
            const size_t o = r * ca4 + c;
            if (a_add) { float4 w = a_add[o]; v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
            da[o] = v;
        } else {
            const size_t o = r * cb4 + (c - ca4);
            if (b_add) { float4 w = b_add[o]; v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w; }
            db[o] = v;
        }
    }
}

int ew_grid(size_t n4) {
    size_t b = (n4 + 255) / 256;
    if (b > 132 * 8) b = 132 * 8;
    return (int)(b < 1 ? 1 : b);
}

int launch_add(const float* a, const float* b, float* c, size_t n, cudaStream_t st) {
    if (n == 0) return VC_OK;
    add_kernel<<<dim3(ew_grid(n / 4)), dim3(256), 0, st>>>((const float4*)a, (const float4*)b, (float4*)c, n / 4);
    VC_LAUNCH_CHECK();
    return VC_OK;
}

struct Ctx {
    const int32_t* oi;
    const float* of;
    int n_ops;
    const uint64_t* lp;
    const float* lf;
    int n_layers;
    State* S;
    Arena A;
    cudaStream_t st[3];   // forward: main, index stream, second index stream (image branch); backward: main, wgrad
    int32_t* err;
    // SyncBatchNorm (vc_exec_forward_sync / vc_exec_backward_sync; xfn NULL: plain BatchNorm): the caller's float64 exchange
    // buffer, its slot offsets [n_layers, 2] (forward, backward) and the callback that all-reduces a slot
    double* xchg;
    const int64_t* xoff;
    vc_bn_exchange_fn xfn;
    void* xuser;
    const int* op(int i) const { return oi + (size_t)i * OPI; }
    double* xslot(int layer, int dir) const { return xchg + xoff[2 * layer + dir]; }
    template <class T>
    T* P(int layer, int col) const { return reinterpret_cast<T*>(lp[(size_t)layer * P_COLS + col]); }
};

#define VC_TRY(expr)              \
    do {                          \
        int rc__ = (expr);        \
        if (rc__) return rc__;    \
    } while (0)

#define VC_ALLOC(var, type, bytes)                                                                     \
    type var = (type)C.A.alloc(bytes);                                                                 \
    if (!var && (bytes) > 0) {                                                                         \
        set_error("plan executor: arena too small (%zu bytes given, > %zu needed)", C.A.cap, C.A.used); \
        return VC_ERR_WORKSPACE;                                                                       \
    }

// SyncBatchNorm: the caller all-reduces slot `dir` (0 forward, 1 backward) of layer `li` over the ranks, enqueued on the main
// stream (under capture: captured there, once)
int exchange(Ctx& C, int li, int dir, int n) {
    if (C.xfn(C.xuser, li, dir, C.xslot(li, dir), n) != 0) {
        set_error("SyncBatchNorm exchange of layer %d (%s) failed", li, dir ? "backward" : "forward");
        return VC_ERR_INVALID;
    }
    return VC_OK;
}

// make `consumer` stream wait for a resource produced on the other stream
int wait_for(Ctx& C, int& ev, int prod, int consumer) {
    if (ev >= 0 && C.st[prod] != C.st[consumer]) VC_CUDA(cudaStreamWaitEvent(C.st[consumer], g_ev[ev], 0));
    return VC_OK;
}
int record_on(Ctx& C, int s) {   // -> event id recorded at the current tail of stream s
    if (C.st[0] == C.st[1] && C.st[0] == C.st[2]) return -1;
    int e = g_ev_next;
    g_ev_next = (g_ev_next + 1) % EV_POOL;
    if (cudaEventRecord(g_ev[e], C.st[s]) != cudaSuccess) return -1;
    return e;
}

int check_plan(const int32_t* oi, int n_ops, int n_layers) {
    VC_CHECK_ARG(oi && n_ops > 0 && n_ops <= MAX_OPS && n_layers >= 0 && n_layers <= MAX_L, "bad plan size");
    for (int i = 0; i < n_ops; ++i) {
        const int* o = oi + (size_t)i * OPI;
        VC_CHECK_ARG(o[F_KIND] >= OP_SUBM_RB && o[F_KIND] <= OP_DISCARD, "op %d: unknown kind %d", i, o[F_KIND]);
        VC_CHECK_ARG(o[F_STREAM] >= 0 && o[F_STREAM] <= 2, "op %d: bad stream", i);
        const int lim_a = (o[F_KIND] == OP_CBR || o[F_KIND] == OP_CAT) ? MAX_F : MAX_I;
        VC_CHECK_ARG(o[F_A] >= 0 && o[F_A] < lim_a, "op %d: slot a out of range", i);
        if (o[F_KIND] == OP_CBR) {
            VC_CHECK_ARG(o[F_B] >= 0 && o[F_B] < MAX_F && o[F_C] >= 0 && o[F_C] < MAX_RB, "op %d: bad slots", i);
            VC_CHECK_ARG(o[F_LAYER] >= 0 && o[F_LAYER] < n_layers, "op %d: bad layer", i);
        } else if (o[F_KIND] == OP_CAT) {
            VC_CHECK_ARG(o[F_B] >= 0 && o[F_B] < MAX_F && o[F_C] >= 0 && o[F_C] < MAX_F, "op %d: bad slots", i);
        } else if (o[F_KIND] == OP_SUBM_RB) {
            VC_CHECK_ARG(o[F_C] >= 0 && o[F_C] < MAX_RB, "op %d: bad rulebook id", i);
        } else if (o[F_KIND] == OP_CONV_RB) {
            VC_CHECK_ARG(o[F_B] >= 0 && o[F_B] < MAX_I && o[F_C] >= 0 && o[F_C] < MAX_RB, "op %d: bad ids", i);
        } else if (o[F_KIND] == OP_DISCARD) {
            VC_CHECK_ARG(o[F_B] >= 0 && o[F_B] < MAX_I && o[F_C] >= 0 && o[F_CIN] >= 0 && o[F_CIN] < MAX_F && o[F_COUT] > 0 &&
                             o[F_COUT] < MAX_F && o[F_CIN] != o[F_COUT],
                         "op %d: bad discard ids", i);
        } else {
            VC_CHECK_ARG(o[F_B] >= 0 && o[F_B] < MAX_I, "op %d: bad index-set id", i);
        }
    }
    return VC_OK;
}

// the one place that decides which conv kernels a layer runs (the tensor-core backward only in a BN-training step; in the
// deterministic mode the many-to-one tables take the gather-form dgrad instead of the atomic scatter)
void choose_kernels(Layer& L, int precision, int training, int need_dgrad, const RBk& R, int det) {
    const bool tc = precision == 1 && tc2_ch_ok(L.cin) && tc2_ch_ok(L.cout);
    const bool tc_bwd = tc && training;
    L.fwd = tc ? K_FWD_TC : K_FWD_F32;
    L.wgrad = tc_bwd ? K_WGRAD_TC : K_WGRAD_F32;
    if (!need_dgrad || L.in_slot == 0)
        L.dgrad = K_NONE;
    else if (R.subm && !R.unique && det)
        L.dgrad = tc_bwd ? K_DGRAD_GATHER2D_TC : K_DGRAD_GATHER2D_F32;
    else if (R.subm && !R.unique)   // many-to-one table (the image branch's projected pixels collide): atomic scatter
        L.dgrad = tc_bwd && tc_scatter_ch_ok(L.cin) && tc_scatter_ch_ok(L.cout) ? K_DGRAD_SCATTER_TC : K_DGRAD_SCATTER_F32;
    else
        L.dgrad = tc_bwd ? K_DGRAD_TC : K_DGRAD_F32;
}

// fp32 accumulator of the tensor-core wgrad (deterministic mode: one image per row chunk), padded to 64 floats
size_t wgrad_acc_floats(const Layer& L, int K, int det) {
    return L.wgrad == K_WGRAD_TC ? ((size_t)(det ? WGRAD_DET_CHUNKS : 1) * K * L.cin * L.cout + 63) / 64 * 64 : 0;
}

// what the forward shares between its planning pass and its per-op enqueue functions (value-initialised)
struct FwdCtx : Ctx {
    // derived from the plan alone by plan_step, before any CUDA call: both phases of a phased step derive the same, so they
    // agree on every arena address (rulebook meta and layer kinds go straight into the State)
    int slot_c[MAX_F], cat_out[MAX_F], cat_col[MAX_F];   // cat_out: the in-place concat a slot is a column slice of, or -1
    bool need_f32[MAX_F], cat_inplace[MAX_OPS];
    size_t sums_doubles, n_cbr, wg_floats;               // the zeroed region: BN sums, tile counters, wgrad accumulators
    const float* proj;
    const int64_t* seed;   // of the DISCARD ops
    const int32_t* caps;
    int32_t *overflow, *pinned;
    int n_syncs, last_ev[3] = {-1, -1, -1};   // last_ev: latest event of each side stream (joined into main at the end)
    bool do_idx, do_feat, two;   // do_idx / do_feat: enqueue the index / feature operators (both unless phased)
    bool idx_first;              // the whole index phase is enqueued before this walk: no index kernel runs beside a conv
    bool batched[MAX_OPS];       // op enqueued by a batched call of its chain (fwd_chain_tables, fwd_chain_stages)
    ConvRank rank[MAX_I];        // per index set a strided conv wrote: where its ranked output bitmap lies (for the tables)
    template <class T>
    void produced(T& r, int s) {   // r was written on stream s: consumers on the other streams wait for r.ev
        r.prod = s;
        r.ev = s == 0 ? -1 : (last_ev[s] = record_on(*this, s));
    }
};

// Which feature slots need an fp32 copy: published ones (x1 of the producing op), the input of a layer without the
// tensor-core forward + wgrad pair (fp32 conv or fp32 wgrad), and the fp32 precision mode.  Everything else is read as
// bf16 only, so its fp32 copy is not written.  A concat whose inputs need no fp32 copy of their own is built in place:
// the BN-apply of each input layer writes its column slice of the concat (fp32 if the concat needs it, and bf16), and
// the concat op launches nothing.
void plan_step(FwdCtx& C, int c0, int precision, int training) {
    for (int i = 0; i < MAX_F; ++i) C.cat_out[i] = -1;
    C.slot_c[0] = c0;
    C.need_f32[0] = true;
    for (int i = 0; i < C.n_ops; ++i) {
        const int* o = C.op(i);
        if (o[F_KIND] == OP_SUBM_RB || o[F_KIND] == OP_CONV_RB) {
            RBk& R = C.S->rb[o[F_C]];
            R.K = 1;
            for (int d = 0; d < o[F_NDIM]; ++d) R.K *= o[F_KS + d];
            R.subm = o[F_KIND] == OP_SUBM_RB;
            R.unique = R.subm ? o[F_X0] : 1;
        } else if (o[F_KIND] == OP_CBR) {
            Layer& L = C.S->layer[o[F_LAYER]];
            L.cin = o[F_CIN]; L.cout = o[F_COUT]; L.in_slot = o[F_A]; L.out_slot = o[F_B]; L.rb = o[F_C];
            choose_kernels(L, precision, training, o[F_X0], C.S->rb[L.rb], C.S->deterministic);
            C.slot_c[L.out_slot] = L.cout;
            if (precision == 0 || o[F_X1]) C.need_f32[L.out_slot] = true;
            if (L.fwd == K_FWD_F32 || L.wgrad == K_WGRAD_F32) C.need_f32[L.in_slot] = true;
            C.sums_doubles += 4 * (size_t)L.cout;
            ++C.n_cbr;
            C.wg_floats += wgrad_acc_floats(L, C.S->rb[L.rb].K, C.S->deterministic);
        } else if (o[F_KIND] == OP_CAT) {
            C.slot_c[o[F_C]] = C.slot_c[o[F_A]] + C.slot_c[o[F_B]];
            if (precision == 0 || o[F_X1]) C.need_f32[o[F_C]] = true;
        } else if (o[F_KIND] == OP_DISCARD) {   // the discard gathers fp32 rows (and rounds its own bf16 shadow)
            C.slot_c[o[F_COUT]] = C.slot_c[o[F_CIN]];
            C.need_f32[o[F_CIN]] = true;
            if (precision == 0 || o[F_X1]) C.need_f32[o[F_COUT]] = true;
        }
    }
    for (int i = 0; i < C.n_ops; ++i) {
        const int* o = C.op(i);
        if (o[F_KIND] != OP_CAT) continue;
        const int a = o[F_A], b = o[F_B];
        C.cat_inplace[i] = precision == 1 && a != 0 && b != 0 && a != b && !C.need_f32[a] && !C.need_f32[b] && C.cat_out[a] < 0 &&
                           C.cat_out[b] < 0;
        if (C.cat_inplace[i]) {
            C.cat_out[a] = C.cat_out[b] = o[F_C];
            C.cat_col[b] = C.slot_c[a];
        } else {
            C.need_f32[a] = C.need_f32[b] = true;
        }
    }
}

// one function per op kind: op i (plan row o), enqueued on stream s
int fwd_subm_rb(FwdCtx& C, int i, const int* o, int s) {
    ISet& I = C.S->iset[o[F_A]];
    RBk& R = C.S->rb[o[F_C]];
    VC_CHECK_ARG(I.idx && I.ndim == o[F_NDIM], "op %d: index set %d not built / wrong ndim", i, o[F_A]);
    VC_TRY(wait_for(C, I.ev, I.prod, s));
    R.n_in = R.n_out = I.n;
    R.n_in_dev = R.n_out_dev = I.n_dev;
    VC_ALLOC(nbr, int32_t*, (size_t)R.K * I.n * 4);
    VC_ALLOC(pn, int32_t*, (size_t)R.K * 4);
    R.nbr = nbr; R.pair_num = pn;
    const size_t wsb = vc_subm_rulebook_ws_bytes(I.n);
    VC_ALLOC(ws, void*, wsb);
    int32_t* rep = nullptr;
    if (C.S->deterministic && !R.unique && I.n > 0) {   // the gather-form dgrad's row groups and table (gather2d.cu)
        const size_t gb = ((size_t)I.n + 63) / 64 * 256 + gather2d_prep_bytes(I.n, R.K);
        VC_ALLOC(g2ws, int32_t*, gb);
        rep = g2ws;
        R.g2 = gather2d_carve(g2ws + ((size_t)I.n + 63) / 64 * 64, I.n, R.K);
        C.S->det_bytes += gb;
    }
    if (C.do_idx) {
        VC_TRY(subm_rulebook_dev(I.idx, I.n, I.n_dev, I.ndim, C.S->batch_size, I.shape, o + F_KS, o + F_DL, R.nbr, R.pair_num, ws, wsb,
                                 C.st[s], rep, R.unique != 0));
        if (rep) VC_TRY(gather2d_prep_dev(R.nbr, rep, R.K, I.n, I.n_dev, R.g2, C.st[s]));
    }
    C.produced(R, s);
    return VC_OK;
}

double op_rate(const int* o) {   // the float64 rate of a DISCARD op, stored as two int32 halves
    const uint64_t bits = (uint64_t)(uint32_t)o[F_KS] | ((uint64_t)(uint32_t)o[F_KS + 1] << 32);
    double r;
    memcpy(&r, &bits, 8);
    return r;
}

// index part of DISCARD op j on the index stream: row selection (vc_stvd_layer_keep) and the kept rows' indices
int fwd_discard_keep(FwdCtx& C, int j) {
    const int* o = C.op(j);
    const int s = C.two ? o[F_STREAM] : 0;
    cudaStream_t st = C.st[s];
    ISet& I = C.S->iset[o[F_A]];
    ISet& O = C.S->iset[o[F_B]];
    Disc& D = C.S->disc[j];
    const double rate = op_rate(o);
    VC_CHECK_ARG(I.idx, "op %d: index set %d not built", j, o[F_A]);
    VC_CHECK_ARG(rate >= 0.0 && rate <= 1.0, "op %d: discard rate %g outside [0, 1]", j, rate);
    VC_TRY(wait_for(C, I.ev, I.prod, s));
    int k = I.n;   // static mode: the capacity; the kept count stays on the device
    if (!C.S->is_static) {
        k = (int)((double)I.n * (1.0 - rate));
        VC_CHECK_ARG(k > 0, "StVD layer discard at site %d: %d rows at rate %g keep no row", o[F_C], I.n, rate);
    }
    const int cap = I.n > 0 ? I.n : 1;
    VC_ALLOC(keep, int32_t*, (size_t)cap * 4);
    VC_ALLOC(pos, int32_t*, (size_t)cap * 4);
    VC_ALLOC(kept_dev, int32_t*, 4);
    const size_t wsb = vc_stvd_layer_keep_ws_bytes(I.n);
    VC_ALLOC(ws, void*, wsb);
    VC_ALLOC(oidx, int32_t*, (size_t)(k > 0 ? k : 1) * (1 + I.ndim) * 4);
    if (C.do_idx) {
        VC_TRY(vc_stvd_layer_keep(nullptr, C.seed, o[F_C], I.n, I.n_dev, rate, keep, kept_dev, pos, ws, wsb, st));
        VC_TRY(stvd_gather_idx_dev(I.idx, 1 + I.ndim, keep, k, oidx, st));
    }
    D.keep = keep; D.pos = pos; D.kept_dev = kept_dev; D.n_in = I.n; D.k = k; D.site = o[F_C];
    O.idx = oidx; O.n = k; O.ndim = I.ndim; O.n_dev = C.S->is_static ? kept_dev : nullptr;
    for (int d = 0; d < 3; ++d) O.shape[d] = I.shape[d];
    C.produced(O, s);
    return VC_OK;
}

// DISCARD op i: its index part (unless the first strided conv's read-backs ran it), then the feature gather on the main
// stream — the kept fp32 rows (the published x_conv*) and their bf16 rounding (the next down conv's operand), zero tail in
// static mode
int fwd_discard(FwdCtx& C, int i, const int* o) {
    if (!C.S->iset[o[F_B]].idx) VC_TRY(fwd_discard_keep(C, i));
    const Disc& D = C.S->disc[i];
    ISet& O = C.S->iset[o[F_B]];
    FSlot& X = C.S->f[o[F_CIN]];
    FSlot& Y = C.S->f[o[F_COUT]];
    VC_CHECK_ARG(X.f32 && X.ld == X.c && X.rows == D.n_in, "op %d: discard input slot %d not built / rows %d vs %d", i, o[F_CIN],
                 X.rows, D.n_in);
    VC_TRY(wait_for(C, O.ev, O.prod, 0));
    VC_TRY(wait_for(C, X.ev, X.prod, 0));
    const size_t elems = (size_t)O.n * X.c;
    float* y = nullptr;
    void* yb = nullptr;
    if (C.need_f32[o[F_COUT]]) {
        VC_ALLOC(y_, float*, elems * 4);
        y = y_;
    }
    if (C.S->precision == 1) {
        VC_ALLOC(yb_, void*, elems * 2);
        yb = yb_;
    }
    if (C.do_feat) VC_TRY(stvd_gather_feats_dev(X.f32, X.c, D.keep, O.n, y, yb, C.st[0]));
    Y.f32 = y; Y.bf16 = yb; Y.rows = O.n; Y.c = Y.ld = X.c; Y.n_dev = O.n_dev;
    C.produced(Y, 0);
    return VC_OK;
}

// The tables of all the chain's strided convs on the chain's stream: nbr_bwd, pair counts and level 0's nbr_fwd in one
// launch (conv_tables_batch_dev), and the nbr_fwd of the levels whose input set is the previous level's output by lookup
// in that level's bitmap (conv_fwd_lookup_batch_dev), which writes every entry.  Level 0's input set (the voxels) has no
// bitmap: its nbr_fwd is scattered from the input rows into a -1 filled table.  The nbr_fwd tables lie back to back and
// the pair counts too: one fill and one zeroing.
int fwd_chain_tables(FwdCtx& C, const int* ops, int L, int s) {
    size_t fwd_ints = 0, pn_ints = 0;
    for (int l = 0; l < L; ++l) {
        const RBk& R = C.S->rb[C.op(ops[l])[F_C]];
        fwd_ints += (size_t)R.K * (R.n_out > 0 ? R.n_out : 1);
        pn_ints += R.K;
    }
    VC_ALLOC(fwd_all, int32_t*, fwd_ints * 4);
    VC_ALLOC(pn_all, int32_t*, pn_ints * 4);
    TablesStage ts[CONV_CHAIN_MAX];
    FwdLookupStage fs[CONV_CHAIN_MAX];
    for (int l = 0, fo = 0, po = 0; l < L; ++l) {
        const int* o = C.op(ops[l]);
        const ISet& I = C.S->iset[o[F_A]];
        RBk& R = C.S->rb[o[F_C]];
        VC_ALLOC(nbr_bwd, int32_t*, (size_t)R.K * I.n * 4);
        R.nbr = fwd_all + fo; R.nbr_bwd = nbr_bwd; R.pair_num = pn_all + po;
        fo += R.K * (R.n_out > 0 ? R.n_out : 1);
        po += R.K;
        ts[l] = TablesStage{I.idx, I.n, I.n_dev, I.ndim, I.shape, o + F_KS, o + F_ST, o + F_PD, o + F_DL, R.n_out, C.rank[o[F_B]],
                            l == 0 ? R.nbr : nullptr, R.nbr_bwd, R.pair_num};
        if (l > 0)
            fs[l - 1] = FwdLookupStage{C.S->iset[o[F_B]].idx, R.n_out, R.n_out_dev, I.n, I.n_dev, C.rank[o[F_A]], I.ndim,
                                       I.shape, o + F_KS, o + F_ST, o + F_PD, o + F_DL, R.nbr};
        C.batched[ops[l]] = true;
    }
    if (C.do_idx) {
        const RBk& R0 = C.S->rb[C.op(ops[0])[F_C]];
        VC_CUDA(cudaMemsetAsync(pn_all, 0, pn_ints * 4, C.st[s]));
        VC_CUDA(cudaMemsetAsync(fwd_all, 0xFF, (size_t)R0.K * R0.n_out * 4, C.st[s]));
        VC_TRY(conv_tables_batch_dev(ts, L, C.S->batch_size, C.st[s]));
        if (L > 1) VC_TRY(conv_fwd_lookup_batch_dev(fs, L - 1, C.S->batch_size, C.st[s]));
    }
    RBk& R0 = C.S->rb[C.op(ops[0])[F_C]];
    C.produced(R0, s);   // one event for the batch
    for (int l = 1; l < L; ++l) {
        RBk& R = C.S->rb[C.op(ops[l])[F_C]];
        R.ev = R0.ev; R.prod = R0.prod;
    }
    return VC_OK;
}

// The submanifold rulebooks and projections over the chain's output sets (the stage 2-4 work of the plan's
// image-branch stream), one launch per kind: bitmap lookup of the 3-D sets (each is a chain level), index2uv, hash insert +
// probe of the projected sets (their pixels collide: many-to-one tables).  Applies when all of them run on one stream and
// the 2-D ones probe alike; else each op keeps its own launches.  The deterministic mode's 2-D rulebooks (the gather-form
// dgrad's `rep` rows) stay per op.
int fwd_chain_stages(FwdCtx& C, int i0, const int* ops, int L) {
    int sub3[IDX_BATCH_MAX], uvop[IDX_BATCH_MAX], sub2[IDX_BATCH_MAX], n3 = 0, nuv = 0, n2 = 0, s = -1;
    bool ok = true;
    auto take = [&](int j, int* list, int& n) {
        const int sj = C.two ? C.op(j)[F_STREAM] : 0;
        if (n == IDX_BATCH_MAX || (s >= 0 && sj != s)) ok = false;
        else { list[n++] = j; s = sj; }
    };
    for (int j = i0 + 1; j < C.n_ops && ok; ++j) {
        const int* o = C.op(j);
        bool from_chain = false;
        for (int l = 0; l < L; ++l) from_chain |= o[F_A] == C.op(ops[l])[F_B];
        if (o[F_KIND] == OP_SUBM_RB && from_chain && !(C.S->deterministic && !o[F_X0])) take(j, sub3, n3);
        else if (o[F_KIND] == OP_INDEX2UV && from_chain) take(j, uvop, nuv);
    }
    for (int j = i0 + 1; j < C.n_ops && ok; ++j) {
        const int* o = C.op(j);
        bool from_uv = false;
        for (int u = 0; u < nuv; ++u) from_uv |= o[F_A] == C.op(uvop[u])[F_B];
        if (o[F_KIND] == OP_SUBM_RB && from_uv && !(C.S->deterministic && !o[F_X0])) take(j, sub2, n2);
    }
    for (int a = 1; a < n2; ++a) ok &= C.op(sub2[a])[F_X0] == C.op(sub2[0])[F_X0];
    if (!ok || s < 0) return VC_OK;
    for (int a = 0; a < n3; ++a) {
        const int* o = C.op(sub3[a]);
        ISet& I = C.S->iset[o[F_A]];
        VC_CHECK_ARG(I.ndim == o[F_NDIM], "op %d: index set %d has the wrong ndim", sub3[a], o[F_A]);
        VC_TRY(wait_for(C, I.ev, I.prod, s));
    }
    for (int a = 0; a < nuv; ++a) {
        ISet& I = C.S->iset[C.op(uvop[a])[F_A]];
        VC_CHECK_ARG(I.ndim == 3 && C.proj, "op %d: index2uv needs a built 3-D index set and projection params", uvop[a]);
        VC_TRY(wait_for(C, I.ev, I.prod, s));
    }
    // pair counts of every rulebook: one region, one zeroing
    size_t pn_ints = 0;
    for (int a = 0; a < n3; ++a) pn_ints += C.S->rb[C.op(sub3[a])[F_C]].K;
    for (int a = 0; a < n2; ++a) pn_ints += C.S->rb[C.op(sub2[a])[F_C]].K;
    VC_ALLOC(pn_all, int32_t*, pn_ints * 4);
    if (C.do_idx && pn_ints) VC_CUDA(cudaMemsetAsync(pn_all, 0, pn_ints * 4, C.st[s]));
    int32_t* pn = pn_all;
    // 3-D: by lookup in the bitmap of the chain level each index set is (every table entry written, nothing to clear)
    SubmLookupStage st3[IDX_BATCH_MAX];
    for (int a = 0; a < n3; ++a) {
        const int* o = C.op(sub3[a]);
        ISet& I = C.S->iset[o[F_A]];
        RBk& R = C.S->rb[o[F_C]];
        R.n_in = R.n_out = I.n;
        R.n_in_dev = R.n_out_dev = I.n_dev;
        VC_ALLOC(nbr, int32_t*, (size_t)R.K * I.n * 4);
        R.nbr = nbr; R.pair_num = pn;
        pn += R.K;
        st3[a] = SubmLookupStage{I.idx, I.n, I.n_dev, I.ndim, I.shape, o + F_KS, o + F_DL, C.rank[o[F_A]], R.nbr, R.pair_num};
        C.batched[sub3[a]] = true;
    }
    if (n3) {
        if (C.do_idx) VC_TRY(subm_lookup_batch_dev(st3, n3, C.S->batch_size, C.st[s]));
        RBk& R0 = C.S->rb[C.op(sub3[0])[F_C]];
        C.produced(R0, s);
        for (int a = 1; a < n3; ++a) {
            RBk& R = C.S->rb[C.op(sub3[a])[F_C]];
            R.ev = R0.ev; R.prod = R0.prod;
        }
    }
    UVStage uvs[IDX_BATCH_MAX];
    for (int a = 0; a < nuv; ++a) {
        const int* o = C.op(uvop[a]);
        ISet& I = C.S->iset[o[F_A]];
        ISet& O = C.S->iset[o[F_B]];
        VC_ALLOC(uv, int32_t*, (size_t)I.n * 3 * 4);
        O.idx = uv; O.n = I.n; O.ndim = 2; O.shape[0] = o[F_KS]; O.shape[1] = o[F_KS + 1]; O.shape[2] = 0; O.n_dev = I.n_dev;
        uvs[a] = UVStage{I.idx, I.n, I.n_dev, C.of + (size_t)uvop[a] * OPF, o[F_X0], o[F_X1], o[F_X2], uv};
        C.batched[uvop[a]] = true;
    }
    if (nuv) {
        if (C.do_idx) VC_TRY(index2uv_batch_dev(uvs, nuv, C.S->batch_size, C.proj, C.st[s]));
        ISet& O0 = C.S->iset[C.op(uvop[0])[F_B]];
        C.produced(O0, s);
        for (int a = 1; a < nuv; ++a) {
            ISet& O = C.S->iset[C.op(uvop[a])[F_B]];
            O.ev = O0.ev; O.prod = O0.prod;
        }
    }
    // 2-D: the hash tables of all stages back to back, one 0xFF fill (the full probe writes every table row)
    SubmStage st2[IDX_BATCH_MAX];
    char *t0 = nullptr, *t1 = nullptr;
    for (int a = 0; a < n2; ++a) {
        const int* o = C.op(sub2[a]);
        ISet& I = C.S->iset[o[F_A]];
        VC_CHECK_ARG(I.idx && I.ndim == o[F_NDIM], "op %d: index set %d not built / wrong ndim", sub2[a], o[F_A]);
        const size_t wsb = vc_subm_rulebook_ws_bytes(I.n);
        VC_ALLOC(ws, void*, wsb);
        if (!t0) t0 = (char*)ws;
        t1 = (char*)ws + wsb;
        st2[a] = SubmStage{I.idx, I.n, I.n_dev, I.ndim, I.shape, o + F_KS, o + F_DL, nullptr, nullptr, ws, wsb};
    }
    for (int a = 0; a < n2; ++a) {
        const int* o = C.op(sub2[a]);
        ISet& I = C.S->iset[o[F_A]];
        RBk& R = C.S->rb[o[F_C]];
        R.n_in = R.n_out = I.n;
        R.n_in_dev = R.n_out_dev = I.n_dev;
        VC_ALLOC(nbr, int32_t*, (size_t)R.K * I.n * 4);
        R.nbr = st2[a].nbr = nbr; R.pair_num = st2[a].pair_num = pn;
        pn += R.K;
        C.batched[sub2[a]] = true;
    }
    if (n2) {
        if (C.do_idx) {
            VC_CUDA(cudaMemsetAsync(t0, 0xFF, t1 - t0, C.st[s]));
            VC_TRY(subm_rulebook_batch_dev(st2, n2, C.S->batch_size, C.op(sub2[0])[F_X0] != 0, C.st[s]));
        }
        RBk& R0 = C.S->rb[C.op(sub2[0])[F_C]];
        C.produced(R0, s);
        for (int a = 1; a < n2; ++a) {
            RBk& R = C.S->rb[C.op(sub2[a])[F_C]];
            R.ev = R0.ev; R.prod = R0.prod;
        }
    }
    return VC_OK;
}

// The chain of strided convs from op i (rulebook.cu header): op i and the strided convs after it that each read the
// previous one's output set, up to CONV_CHAIN_MAX and no further than a layer discard; a dilated conv is a chain of its own.
// A function of the plan alone.  -> L, the chain's ops and geometry
int chain_from(const FwdCtx& C, int i, int* ops, ConvChain& ch) {
    const int* o0 = C.op(i);
    ch = ConvChain{};
    ch.ndim = o0[F_NDIM]; ch.batch = C.S->batch_size; ch.shape0 = C.S->iset[o0[F_A]].shape;
    for (int j = i, cur = o0[F_A]; j < C.n_ops && ch.L < CONV_CHAIN_MAX; ++j) {
        const int* o = C.op(j);
        if (o[F_KIND] == OP_DISCARD) break;
        if (o[F_KIND] != OP_CONV_RB) continue;
        if (o[F_A] != cur || o[F_NDIM] != o0[F_NDIM]) break;
        const int l = ch.L++;
        ch.ksize[l] = o + F_KS; ch.stride[l] = o + F_ST; ch.pad[l] = o + F_PD; ch.dil[l] = o + F_DL;
        if (!conv_chain_composable(ch)) {   // a dilated level, or one after a dilated level 0
            --ch.L;
            break;
        }
        ops[l] = j;
        cur = o[F_B];
    }
    return ch.L;
}

// count + row-count read-back + output indices of the chain from op i: every level's count and output indices in one
// composed pass (rulebook.cu), one host read of all of them in exact mode
int fwd_chain_count(FwdCtx& C, int i) {
    const int* o0 = C.op(i);
    ISet& I = C.S->iset[o0[F_A]];
    VC_CHECK_ARG(I.idx && I.ndim == o0[F_NDIM], "op %d: index set %d not built / wrong ndim", i, o0[F_A]);
    int ops[CONV_CHAIN_MAX];
    ConvChain ch;
    chain_from(C, i, ops, ch);
    const int s = C.two ? o0[F_STREAM] : 0;
    cudaStream_t st = C.st[s];
    VC_TRY(wait_for(C, I.ev, I.prod, s));
    const size_t wsb = conv_chain_ws_bytes(ch);
    VC_CHECK_ARG(wsb > 0, "op %d: bad chain of strided convs", i);
    VC_ALLOC(ws, void*, wsb);
    VC_ALLOC(n_dev, int32_t*, 4 * CONV_CHAIN_MAX);
    int n_out[CONV_CHAIN_MAX];
    int32_t* oidx[CONV_CHAIN_MAX];
    if (C.S->is_static) {
        for (int l = 0; l < ch.L; ++l) {
            n_out[l] = C.caps[C.op(ops[l])[F_B]];
            VC_CHECK_ARG(n_out[l] > 0, "op %d: static mode needs a capacity for index set %d", ops[l], C.op(ops[l])[F_B]);
        }
        if (C.do_idx) VC_TRY(conv_chain_count_dev(ch, I.idx, I.n, I.n_dev, n_dev, n_out, C.overflow, ws, wsb, st));
    } else {
        VC_TRY(conv_chain_count_dev(ch, I.idx, I.n, nullptr, n_dev, nullptr, nullptr, ws, wsb, st));
        VC_CUDA(cudaMemcpyAsync(C.pinned + 8, n_dev, 4 * ch.L, cudaMemcpyDeviceToHost, st));
        // the tensor-core kernels' pipeline-timeout flag rides along with the first read-back of a step (it reports on the
        // kernels of EARLIER steps: a wedged mbarrier wait must not go unnoticed in production — ADVICE r1)
        if (C.n_syncs == 0 && C.err != nullptr) VC_CUDA(cudaMemcpyAsync(C.pinned + 15, C.err, 4, cudaMemcpyDeviceToHost, st));
        VC_CUDA(cudaStreamSynchronize(st));        // the data-dependent sizes of all the chain's convs at once
        for (int l = 0; l < ch.L; ++l) n_out[l] = C.pinned[8 + l];
        if (C.n_syncs == 0 && C.err != nullptr && C.pinned[15] != 0) {
            set_error("a tensor-core kernel's pipeline wait timed out in an earlier step (error flag %d): its results are invalid",
                      C.pinned[15]);
            return VC_ERR_PIPELINE;
        }
        ++C.n_syncs;
    }
    for (int l = 0; l < ch.L; ++l) {
        const int* o = C.op(ops[l]);
        ISet& In = C.S->iset[o[F_A]];
        ISet& O = C.S->iset[o[F_B]];
        RBk& R = C.S->rb[o[F_C]];
        int32_t oshape[3] = {0, 0, 0};
        VC_TRY(vc_conv_out_shape(In.ndim, In.shape, o + F_KS, o + F_ST, o + F_PD, o + F_DL, oshape));
        R.n_in = In.n; R.n_out = n_out[l];
        R.n_in_dev = In.n_dev; R.n_out_dev = C.S->is_static ? n_dev + l : nullptr;
        O.n = n_out[l]; O.ndim = In.ndim; O.n_dev = R.n_out_dev;
        for (int d = 0; d < 3; ++d) O.shape[d] = oshape[d];
        VC_ALLOC(oi, int32_t*, (size_t)(n_out[l] > 0 ? n_out[l] : 1) * (1 + In.ndim) * 4);
        O.idx = oidx[l] = oi;
        if (C.S->is_static && C.do_idx) VC_CUDA(cudaMemsetAsync(oi, 0xFF, (size_t)n_out[l] * (1 + In.ndim) * 4, st));
        C.rank[o[F_B]] = conv_chain_rank(ch, ws, l);
    }
    if (C.do_idx) VC_TRY(conv_chain_emit_dev(ch, oidx, n_out, ws, wsb, st));
    for (int l = 0; l < ch.L; ++l) C.produced(C.S->iset[C.op(ops[l])[F_B]], s);
    return VC_OK;
}

int fwd_conv_rb(FwdCtx& C, int i, const int* o, int s) {
    // First strided conv reached.  In exact mode the host reads here the row counts of EVERY chain of strided convs in the
    // plan, back to back: each chain's count -> (host read) -> emit, and the row selection of each layer discard between
    // chains (the next count reads its rows), in plan order.  That is the only part of the forward the host has to wait
    // for, and each read waits for counting work only; the neighbour tables, submanifold rulebooks and projections queue up
    // behind it without further synchronisation.  Static mode reads nothing on the host, so it keeps the natural order
    // (count -> indices -> tables per chain): the tables of an early chain do not queue behind the counting of later ones.
    if (!C.S->iset[o[F_B]].idx) {
        if (C.S->is_static) {
            VC_TRY(fwd_chain_count(C, i));
        } else {
            for (int j = i; j < C.n_ops; ++j) {
                const int* oj = C.op(j);
                if ((oj[F_KIND] != OP_CONV_RB && oj[F_KIND] != OP_DISCARD) || C.S->iset[oj[F_B]].idx || !C.S->iset[oj[F_A]].idx)
                    continue;
                VC_TRY(oj[F_KIND] == OP_CONV_RB ? fwd_chain_count(C, j) : fwd_discard_keep(C, j));
            }
        }
    }
    VC_CHECK_ARG(C.S->iset[o[F_B]].idx, "op %d: index set %d not built", i, o[F_A]);
    int ops[CONV_CHAIN_MAX];
    ConvChain ch;
    const int L = chain_from(C, i, ops, ch);
    VC_TRY(fwd_chain_tables(C, ops, L, s));
    return fwd_chain_stages(C, i, ops, L);
}

int fwd_index2uv(FwdCtx& C, int i, const int* o, int s) {
    ISet& I = C.S->iset[o[F_A]];
    ISet& O = C.S->iset[o[F_B]];
    VC_CHECK_ARG(I.idx && I.ndim == 3 && C.proj, "op %d: index2uv needs a built 3-D index set and projection params", i);
    VC_TRY(wait_for(C, I.ev, I.prod, s));
    VC_ALLOC(uv, int32_t*, (size_t)I.n * 3 * 4);
    O.idx = uv; O.n = I.n; O.ndim = 2; O.shape[0] = o[F_KS]; O.shape[1] = o[F_KS + 1]; O.shape[2] = 0; O.n_dev = I.n_dev;
    if (C.do_idx)
        VC_TRY(index2uv_dev(I.idx, I.n, I.n_dev, C.S->batch_size, C.proj, C.of + (size_t)i * OPF, o[F_X0], o[F_X1], o[F_X2], uv, C.st[s]));
    C.produced(O, s);
    return VC_OK;
}

int fwd_cbr(FwdCtx& C, int i, const int* o, int s) {
    State* S = C.S;
    cudaStream_t st = C.st[s];
    const int li = o[F_LAYER];
    Layer& L = S->layer[li];
    FSlot& X = S->f[L.in_slot];
    FSlot& Y = S->f[L.out_slot];
    RBk& R = S->rb[L.rb];
    VC_CHECK_ARG((X.f32 || X.bf16) && R.nbr && X.c == L.cin && X.rows == R.n_in,
                 "op %d: input slot / rulebook mismatch (rows %d vs %d, c %d vs %d)", i, X.rows, R.n_in, X.c, L.cin);
    VC_TRY(wait_for(C, R.ev, R.prod, s));
    VC_TRY(wait_for(C, X.ev, X.prod, s));
    const size_t elems = (size_t)R.n_out * L.cout;
    VC_ALLOC(x, float*, elems * 4);
    VC_ALLOC(stats, float*, (size_t)4 * L.cout * 4);
    float* y = nullptr;
    void* yb = nullptr;
    int y_ld = L.cout;
    const int cat = C.cat_out[L.out_slot];
    if (cat >= 0) {   // a column slice of an in-place concat (allocated by its first input)
        FSlot& O = S->f[cat];
        if (O.bf16 == nullptr) {
            O.rows = R.n_out; O.c = O.ld = C.slot_c[cat];
            if (C.need_f32[cat]) {
                VC_ALLOC(of_, float*, (size_t)O.rows * O.c * 4);
                O.f32 = of_;
            }
            VC_ALLOC(ob_, void*, (size_t)O.rows * O.c * 2);
            O.bf16 = ob_;
        }
        VC_CHECK_ARG(O.rows == R.n_out, "op %d: concat inputs with different row counts", i);
        y_ld = O.ld;
        if (O.f32) y = O.f32 + C.cat_col[L.out_slot];
        yb = (__nv_bfloat16*)O.bf16 + C.cat_col[L.out_slot];
    } else {
        if (C.need_f32[L.out_slot]) {
            VC_ALLOC(y_, float*, elems * 4);
            y = y_;
        }
        if (S->precision == 1) {
            VC_ALLOC(yb_, void*, elems * 2);
            yb = yb_;
        }
    }
    L.x = x; L.y = y; L.stats = stats;
    double* sums = S->training ? L.sums : nullptr;
    double* part = nullptr;   // deterministic mode: the conv's BN sums per 128-row tile, added in tile order below
    if (sums && S->deterministic) {
        const size_t pb = (size_t)cdiv(R.n_out > 0 ? R.n_out : 1, VC_TILE_ROWS) * 2 * L.cout * 8;
        VC_ALLOC(p_, double*, pb);
        part = p_;
        S->det_bytes += pb;
    }
    bool bn_done = false;
    // SyncBatchNorm over more than one rank: conv with epilogue sums -> exchange -> apply (the fused conv + BN cannot wait
    // for the other ranks' sums)
    const bool sync = C.xfn != nullptr && S->training;
    if (L.fwd == K_FWD_TC && R.n_out > 0) {
        if (!X.bf16) {   // no producer wrote a shadow (network input): cast once
            VC_CHECK_ARG(X.ld == X.c, "op %d: no bf16 copy of a strided input", i);
            VC_ALLOC(xb, void*, (size_t)X.rows * X.c * 2);
            if (C.do_feat) VC_TRY(vc_cast_f32_bf16(X.f32, xb, (long long)X.rows * X.c, st));
            X.bf16 = xb;
        }
        Timed t(K_FWD_TC, li, st, C.do_feat);
        // BatchNorm + ReLU in the same launch (conv_tc2.cu): one kernel and one pass over x fewer per layer
        const BnTail bt{C.P<const float>(li, P_GAMMA), C.P<const float>(li, P_BETA), C.P<float>(li, P_RM), C.P<float>(li, P_RV),
                        C.P<long long>(li, P_NBT), C.lf[2 * li + 1], C.lf[2 * li], S->training, L.sums, y, y_ld, yb, y_ld, stats,
                        C.S->is_static, L.tile_ctr + CTR_BN_BAR};
        if (C.do_feat)
            VC_TRY(tc2_conv(L.cin, L.cout, X.bf16, L.wimg_fwd, R.nbr, R.n_out, x, R.n_out, R.n_out_dev, R.K, sums, C.err, st, nullptr,
                            L.tile_ctr, C.idx_first ? 2 : 0, X.ld, part, sync ? nullptr : &bt, &bn_done));
    } else {   // (also a tensor-core layer without output rows)
        const size_t wsb = vc_conv_ws_bytes(L.cin, L.cout, R.K);
        VC_ALLOC(ws, void*, wsb);
        VC_CHECK_ARG(X.f32 && X.ld == X.c, "op %d: the fp32 conv needs a dense fp32 input", i);
        Timed t(K_FWD_F32, li, st, C.do_feat);
        if (C.do_feat && part)
            VC_TRY(conv_fwd_f32_part(X.f32, C.P<const float>(li, P_W), R.nbr, x, R.n_out, L.cin, L.cout, R.K, part, ws, wsb, st));
        else if (C.do_feat)
            VC_TRY(vc_conv_fwd_f32(X.f32, C.P<const float>(li, P_W), R.nbr, x, R.n_out, L.cin, L.cout, R.K, sums, ws, wsb, st));
    }
    if (C.do_feat && !bn_done && part && R.n_out > 0)
        VC_TRY(bn_sums_reduce_dev(part, R.n_out, R.n_out_dev, VC_TILE_ROWS, L.cout, L.sums, st));
    const double* sums_in = L.sums;
    const double* n_glob = nullptr;
    if (C.do_feat && sync) {   // slot = [sum x, sum x^2, rows], all-reduced in place
        VC_TRY(bn_sync_pack_dev(L.sums, L.cout, R.n_out, R.n_out_dev, C.xslot(li, 0), nullptr, nullptr, st));
        VC_TRY(exchange(C, li, 0, 2 * L.cout + 1));
        sums_in = C.xslot(li, 0);
        n_glob = sums_in + 2 * L.cout;
    }
    if (C.do_feat && !bn_done)
        VC_TRY(bn_apply_relu_dev(x, sums_in, R.n_out, R.n_out_dev, L.cout, C.P<const float>(li, P_GAMMA), C.P<const float>(li, P_BETA),
                                 C.P<float>(li, P_RM), C.P<float>(li, P_RV), C.P<long long>(li, P_NBT), C.lf[2 * li + 1], C.lf[2 * li],
                                 S->training, y, y_ld, yb, y_ld, stats, 1, C.S->is_static, st, n_glob));
    Y.f32 = y; Y.bf16 = yb; Y.rows = R.n_out; Y.c = L.cout; Y.ld = y_ld; Y.n_dev = R.n_out_dev;
    C.produced(Y, s);
    return VC_OK;
}

int fwd_cat(FwdCtx& C, int i, const int* o, int s) {
    FSlot& Aa = C.S->f[o[F_A]];
    FSlot& Bb = C.S->f[o[F_B]];
    FSlot& O = C.S->f[o[F_C]];
    VC_TRY(wait_for(C, Aa.ev, Aa.prod, s));
    VC_TRY(wait_for(C, Bb.ev, Bb.prod, s));
    if (C.cat_inplace[i]) {   // both halves are already written (fwd_cbr): nothing to launch
        VC_CHECK_ARG(Aa.bf16 && Bb.bf16 && Aa.rows == Bb.rows && O.bf16, "op %d: concat inputs not built / row mismatch", i);
    } else {
        VC_CHECK_ARG(Aa.f32 && Bb.f32 && Aa.ld == Aa.c && Bb.ld == Bb.c && Aa.rows == Bb.rows,
                     "op %d: concat inputs not built / row mismatch", i);
        const size_t elems = (size_t)Aa.rows * (Aa.c + Bb.c);
        VC_ALLOC(out, float*, elems * 4);
        void* ob = nullptr;
        if (C.S->precision == 1) {
            VC_ALLOC(ob_, void*, elems * 2);
            ob = ob_;
        }
        if (C.do_feat) VC_TRY(cat2_dev(Aa.f32, Bb.f32, out, ob, Aa.rows, Aa.n_dev, Aa.c, Bb.c, C.st[s]));
        O.f32 = out; O.bf16 = ob; O.rows = Aa.rows; O.c = O.ld = Aa.c + Bb.c;
    }
    O.n_dev = Aa.n_dev;
    C.produced(O, s);
    return VC_OK;
}

}  // namespace
}  // namespace vc

using namespace vc;

extern "C" size_t vc_exec_state_bytes(void) { return sizeof(State); }

extern "C" int vc_exec_timing(int enable) {
    g_timing = enable != 0;
    g_t_n = 0;
    return VC_OK;
}

// ms_out[i], kind_layer_out[2*i..] for the records since vc_exec_timing(1); synchronises the device.  Returns the count.
extern "C" int vc_exec_timing_read(float* ms_out, int32_t* kind_layer_out, int max_records) {
    if (cudaDeviceSynchronize() != cudaSuccess) return VC_ERR_CUDA;
    int n = g_t_n < max_records ? g_t_n : max_records;
    for (int i = 0; i < n; ++i) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, g_t[i].a, g_t[i].b);
        ms_out[i] = ms;
        kind_layer_out[2 * i] = g_t[i].kind;
        kind_layer_out[2 * i + 1] = g_t[i].layer;
    }
    return n;
}

extern "C" int vc_exec_query(const void* state, int what, int id, long long* out) {
    const State* S = (const State*)state;
    VC_CHECK_ARG(S && S->magic == STATE_MAGIC && out, "not an executor state");
    switch (what) {
        case 0:
            out[0] = (long long)S->used;
            out[1] = (long long)S->det_bytes;
            out[2] = S->deterministic;
            return VC_OK;
        case 1: {
            VC_CHECK_ARG(id >= 0 && id < MAX_F, "slot id");
            const FSlot& f = S->f[id];
            out[0] = (long long)(uintptr_t)f.f32; out[1] = (long long)(uintptr_t)f.bf16; out[2] = f.rows; out[3] = f.c;
            out[4] = f.ld; out[5] = (long long)(uintptr_t)f.grad; out[6] = f.gld;
            return VC_OK;
        }
        case 2: {
            VC_CHECK_ARG(id >= 0 && id < MAX_I, "index-set id");
            const ISet& s = S->iset[id];
            out[0] = (long long)(uintptr_t)s.idx; out[1] = s.n; out[2] = s.ndim; out[3] = s.shape[0]; out[4] = s.shape[1];
            out[5] = s.shape[2]; out[6] = (long long)(uintptr_t)s.n_dev;
            return VC_OK;
        }
        case 3: {
            VC_CHECK_ARG(id >= 0 && id < MAX_RB, "rulebook id");
            const RBk& r = S->rb[id];
            out[0] = (long long)(uintptr_t)r.nbr; out[1] = (long long)(uintptr_t)r.nbr_bwd;
            out[2] = (long long)(uintptr_t)r.pair_num; out[3] = r.K; out[4] = r.n_in; out[5] = r.n_out; out[6] = r.subm;
            out[7] = r.unique;
            return VC_OK;
        }
        case 4: {
            VC_CHECK_ARG(id >= 0 && id < MAX_L, "layer id");
            const Layer& l = S->layer[id];
            out[0] = (long long)(uintptr_t)l.x; out[1] = (long long)(uintptr_t)l.y; out[2] = (long long)(uintptr_t)l.stats;
            out[3] = l.fwd == K_FWD_TC; out[4] = l.rb; out[5] = l.in_slot; out[6] = l.out_slot;
            return VC_OK;
        }
        case 5: {
            VC_CHECK_ARG(id >= 0 && id < MAX_OPS && S->disc[id].keep, "op %d is not a layer discard of this run", id);
            const Disc& d = S->disc[id];
            out[0] = (long long)(uintptr_t)d.keep; out[1] = d.k; out[2] = (long long)(uintptr_t)d.kept_dev; out[3] = d.n_in;
            out[4] = d.site;
            return VC_OK;
        }
        case 6: {
            VC_CHECK_ARG(id >= 0 && id < MAX_L, "layer id");
            const Layer& l = S->layer[id];
            out[0] = (long long)(uintptr_t)l.dy; out[1] = l.dy_ld; out[2] = (long long)(uintptr_t)l.dx;
            out[3] = (long long)(uintptr_t)l.dxb; out[4] = l.fwd; out[5] = l.wgrad; out[6] = l.dgrad;
            return VC_OK;
        }
    }
    set_error("vc_exec_query: unknown selector %d", what);
    return VC_ERR_INVALID;
}

extern "C" int vc_exec_forward(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs,
                               const float* layer_f, int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0,
                               const int32_t* shape0, int batch_size, const float* proj_params, int training, int precision,
                               int flags, void* arena, size_t arena_bytes, int32_t* pinned_host, int32_t* err_flag,
                               void* state, size_t state_bytes, vc_stream_t main_stream, vc_stream_t side_stream,
                               int side_waits_main, const int32_t* caps, const int32_t* n0_dev, int32_t* overflow_flag,
                               vc_stream_t side2_stream) {
    return vc_exec_forward_seeded(ops_i, ops_f, n_ops, layer_ptrs, layer_f, n_layers, feats0, c0, idx0, n0, shape0, batch_size,
                                  proj_params, training, precision, flags, arena, arena_bytes, pinned_host, err_flag, state,
                                  state_bytes, main_stream, side_stream, side_waits_main, caps, n0_dev, overflow_flag, side2_stream,
                                  nullptr);
}

namespace {
// one walk of the plan (both phases, or the one `flags` selects); idx_first: the index phase was enqueued by a walk before
int exec_forward(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs, const float* layer_f,
                 int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0, const int32_t* shape0, int batch_size,
                 const float* proj_params, int training, int precision, int flags, void* arena, size_t arena_bytes,
                 int32_t* pinned_host, int32_t* err_flag, void* state, size_t state_bytes, vc_stream_t main_stream,
                 vc_stream_t side_stream, int side_waits_main, const int32_t* caps, const int32_t* n0_dev, int32_t* overflow_flag,
                 vc_stream_t side2_stream, const int64_t* rng_seed_dev, bool idx_first, double* xchg, const int64_t* xchg_off,
                 vc_bn_exchange_fn exchange_fn, void* exchange_user) {
    // static mode and phased execution: include/virconv_b200.h.  Both phases walk the whole plan with the same
    // deterministic bump allocation, so they agree on every address and leave the same state blob.
    const bool is_static = n0_dev != nullptr;
    VC_CHECK_ARG(!is_static || (caps && overflow_flag), "static mode needs capacities and an overflow flag");
    const int phase = (flags >> 8) & 3;
    VC_CHECK_ARG(phase == 0 || (is_static && phase <= 2), "phased execution needs static mode");
    VC_TRY(check_plan(ops_i, n_ops, n_layers));
    for (int i = 0; i < n_ops; ++i)
        VC_CHECK_ARG(ops_i[(size_t)i * OPI + F_KIND] != OP_DISCARD || rng_seed_dev,
                     "op %d: a StVD layer discard needs a seed (vc_exec_forward_seeded with rng_seed_dev)", i);
    VC_CHECK_ARG(state && state_bytes >= sizeof(State), "state blob too small (%zu < %zu)", state_bytes, sizeof(State));
    VC_CHECK_ARG(feats0 && idx0 && n0 > 0 && shape0 && batch_size > 0 && arena && pinned_host && ops_f && layer_ptrs && layer_f,
                 "null / empty argument");
    VC_CHECK_ARG(precision == 0 || precision == 1, "precision must be 0 (fp32) or 1 (bf16)");
    State* S = new (state) State();
    memset(S, 0, sizeof(State));
    S->n_ops = n_ops; S->n_layers = n_layers; S->training = training; S->precision = precision; S->batch_size = batch_size;
    S->is_static = is_static;
    S->deterministic = (flags >> 2) & 1;
    for (int i = 0; i < MAX_I; ++i) S->iset[i].ev = -1;
    for (int i = 0; i < MAX_F; ++i) S->f[i].ev = -1;
    for (int i = 0; i < MAX_RB; ++i) S->rb[i].ev = -1;
    S->iset[0].idx = const_cast<int32_t*>(idx0); S->iset[0].n = n0; S->iset[0].ndim = 3; S->iset[0].n_dev = n0_dev;
    for (int d = 0; d < 3; ++d) S->iset[0].shape[d] = shape0[d];
    S->f[0].f32 = const_cast<float*>(feats0); S->f[0].rows = n0; S->f[0].c = c0; S->f[0].ld = c0; S->f[0].n_dev = n0_dev;

    FwdCtx C = {};
    C.oi = ops_i; C.of = ops_f; C.n_ops = n_ops; C.lp = layer_ptrs; C.lf = layer_f; C.n_layers = n_layers; C.S = S;
    C.A = Arena{(char*)arena, arena_bytes, 0, false};
    C.st[0] = (cudaStream_t)main_stream;
    C.st[1] = side_stream ? (cudaStream_t)side_stream : (cudaStream_t)main_stream;
    C.st[2] = (side_stream && side2_stream) ? (cudaStream_t)side2_stream : C.st[1];   // image-branch index ops (index2uv + 2-D rulebooks)
    C.err = err_flag;
    C.proj = proj_params; C.seed = rng_seed_dev; C.caps = caps; C.overflow = overflow_flag; C.pinned = pinned_host;
    C.do_idx = phase != 2; C.do_feat = phase != 1; C.two = C.st[0] != C.st[1];
    C.idx_first = idx_first;
    C.xchg = xchg; C.xoff = xchg_off; C.xfn = exchange_fn; C.xuser = exchange_user;
    plan_step(C, c0, precision, training);

    VC_TRY(ev_init());
    g_ev_next = 0;
    // BatchNorm accumulators + tile-scheduler counters (+ the wgrad accumulators of a training step) of every layer: one
    // region, one memset
    const size_t zero_bytes = C.sums_doubles * 8 + C.n_cbr * CTR_PER_LAYER * sizeof(int) + C.wg_floats * 4;
    VC_ALLOC(sums_all, double*, zero_bytes);
    int* ctr_all = reinterpret_cast<int*>(sums_all + C.sums_doubles);
    float* wg_all = reinterpret_cast<float*>(ctr_all + C.n_cbr * CTR_PER_LAYER);
    if (zero_bytes && C.do_feat) VC_CUDA(cudaMemsetAsync(sums_all, 0, zero_bytes, C.st[0]));

    // tensor-core weight images of every layer, one launch
    TcPrepTable T;
    T.n = 0;
    for (int i = 0; i < n_ops; ++i) {
        const int* o = C.op(i);
        if (o[F_KIND] != OP_CBR) continue;
        Layer& L = S->layer[o[F_LAYER]];
        const RBk& R = S->rb[L.rb];
        L.sums = sums_all;
        sums_all += 4 * (size_t)L.cout;
        L.tile_ctr = ctr_all;
        ctr_all += CTR_PER_LAYER;
        L.wscratch = L.wgrad == K_WGRAD_TC ? wg_all : nullptr;
        wg_all += wgrad_acc_floats(L, R.K, S->deterministic);
        if (L.wscratch && S->deterministic) S->det_bytes += (wgrad_acc_floats(L, R.K, 1) - wgrad_acc_floats(L, R.K, 0)) * 4;
        // dgrad image: mirrored for a submanifold table used as its own transpose, plain for a strided conv's nbr_bwd table
        // (gather dgrad), layout 0 for the many-to-one image-branch table (tensor-core scatter)
        const int n_img = L.fwd != K_FWD_TC                                                                   ? 0
                          : (L.dgrad == K_DGRAD_TC || L.dgrad == K_DGRAD_SCATTER_TC || L.dgrad == K_DGRAD_GATHER2D_TC) ? 2
                                                                                                                      : 1;
        for (int mode = 0; mode < n_img; ++mode) {
            const int layout = (mode == 1 && L.dgrad == K_DGRAD_SCATTER_TC) ? 0 : 1;
            VC_ALLOC(img, void*, tc_image_bytes(L.cin, L.cout, R.K, layout));
            (mode == 0 ? L.wimg_fwd : L.wimg_dgrad) = img;
            if (T.n == TC_PREP_MAX) {
                if (C.do_feat) VC_TRY(tc_prep_images(T, C.st[0]));
                T.n = 0;
            }
            TcPrepEntry& e = T.e[T.n++];
            e.w = C.P<const float>(o[F_LAYER], P_W); e.img = img; e.cin = L.cin; e.cout = L.cout; e.K = R.K; e.mode = mode;
            e.mirror = mode == 1 && ((L.dgrad == K_DGRAD_TC && R.subm) || L.dgrad == K_DGRAD_GATHER2D_TC);
            e.layout = layout;
        }
    }
    if (C.do_feat) VC_TRY(tc_prep_images(T, C.st[0]));

    // the side stream starts after everything already queued on main (the caller's inputs) — unless the caller vouches
    // that idx0 / proj_params are already valid for the side stream and the arena is safe to write from it
    // (side_waits_main = 0): the index pipeline of this step then overlaps whatever main is still running (the
    // previous step's backward)
    if (C.two && side_waits_main) {
        int e = record_on(C, 0);
        if (e >= 0) {
            VC_CUDA(cudaStreamWaitEvent(C.st[1], g_ev[e], 0));
            if (C.st[2] != C.st[1]) VC_CUDA(cudaStreamWaitEvent(C.st[2], g_ev[e], 0));
        }
    }
    for (int i = 0; i < n_ops; ++i) {
        const int* o = C.op(i);
        const int s = C.two ? o[F_STREAM] : 0;
        if (C.batched[i]) continue;
        switch (o[F_KIND]) {
            case OP_SUBM_RB: VC_TRY(fwd_subm_rb(C, i, o, s)); break;
            case OP_CONV_RB: VC_TRY(fwd_conv_rb(C, i, o, s)); break;
            case OP_INDEX2UV: VC_TRY(fwd_index2uv(C, i, o, s)); break;
            case OP_CBR: VC_TRY(fwd_cbr(C, i, o, s)); break;
            case OP_CAT: VC_TRY(fwd_cat(C, i, o, s)); break;
            case OP_DISCARD: VC_TRY(fwd_discard(C, i, o)); break;
        }
    }
    for (int s = 1; s <= 2; ++s)
        if (C.two && C.last_ev[s] >= 0) VC_CUDA(cudaStreamWaitEvent(C.st[0], g_ev[C.last_ev[s]], 0));   // join
    S->used = C.A.used;
    S->magic = STATE_MAGIC;
    return VC_OK;
}
}  // namespace

extern "C" int vc_exec_forward_seeded(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs,
                                      const float* layer_f, int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0,
                                      const int32_t* shape0, int batch_size, const float* proj_params, int training, int precision,
                                      int flags, void* arena, size_t arena_bytes, int32_t* pinned_host, int32_t* err_flag,
                                      void* state, size_t state_bytes, vc_stream_t main_stream, vc_stream_t side_stream,
                                      int side_waits_main, const int32_t* caps, const int32_t* n0_dev, int32_t* overflow_flag,
                                      vc_stream_t side2_stream, const int64_t* rng_seed_dev) {
    return vc_exec_forward_sync(ops_i, ops_f, n_ops, layer_ptrs, layer_f, n_layers, feats0, c0, idx0, n0, shape0, batch_size,
                                proj_params, training, precision, flags, arena, arena_bytes, pinned_host, err_flag, state,
                                state_bytes, main_stream, side_stream, side_waits_main, caps, n0_dev, overflow_flag, side2_stream,
                                rng_seed_dev, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int vc_exec_forward_sync(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs,
                                    const float* layer_f, int n_layers, const float* feats0, int c0, const int32_t* idx0, int n0,
                                    const int32_t* shape0, int batch_size, const float* proj_params, int training, int precision,
                                    int flags, void* arena, size_t arena_bytes, int32_t* pinned_host, int32_t* err_flag,
                                    void* state, size_t state_bytes, vc_stream_t main_stream, vc_stream_t side_stream,
                                    int side_waits_main, const int32_t* caps, const int32_t* n0_dev, int32_t* overflow_flag,
                                    vc_stream_t side2_stream, const int64_t* rng_seed_dev, double* xchg, const int64_t* xchg_off,
                                    vc_bn_exchange_fn exchange_fn, void* exchange_user) {
    VC_CHECK_ARG(!exchange_fn || (xchg && xchg_off), "a SyncBatchNorm exchange needs its buffer and slot offsets");
    // Static mode (no host read splits the index phase): the index walk first, then the feature walk, so that no index
    // kernel is resident while the convs run and the fused conv + BN grids take two CTAs per SM (conv_tc2.cu launch_persist).
    const bool idx_first = n0_dev != nullptr && ((flags >> 8) & 3) == 0 && side_stream != nullptr && side_stream != main_stream;
    const int f = idx_first ? (flags & ~(3 << 8)) : flags;
    if (idx_first)
        VC_TRY(exec_forward(ops_i, ops_f, n_ops, layer_ptrs, layer_f, n_layers, feats0, c0, idx0, n0, shape0, batch_size, proj_params,
                            training, precision, f | (1 << 8), arena, arena_bytes, pinned_host, err_flag, state, state_bytes,
                            main_stream, side_stream, side_waits_main, caps, n0_dev, overflow_flag, side2_stream, rng_seed_dev, false,
                            xchg, xchg_off, exchange_fn, exchange_user));
    return exec_forward(ops_i, ops_f, n_ops, layer_ptrs, layer_f, n_layers, feats0, c0, idx0, n0, shape0, batch_size, proj_params,
                        training, precision, idx_first ? f | (2 << 8) : flags, arena, arena_bytes, pinned_host, err_flag, state,
                        state_bytes, main_stream, side_stream, side_waits_main, caps, n0_dev, overflow_flag, side2_stream, rng_seed_dev,
                        idx_first, xchg, xchg_off, exchange_fn, exchange_user);
}

namespace vc {
namespace {

// hand a gradient contribution of shape [rows, c] to slot F: `write(dst)` must enqueue kernels that OVERWRITE dst
template <class W>
int contribute(Ctx& C, FSlot& F, cudaStream_t st, W&& write) {
    const size_t n = (size_t)F.rows * F.c;
    VC_CHECK_ARG(F.gld == F.c, "a column slice of a gradient cannot take this contribution");
    if (F.grad_state == G_EMPTY) {
        VC_ALLOC(buf, float*, n * 4);
        VC_TRY(write(buf));
        F.grad = buf;
    } else if (F.grad_state == G_EXT) {
        VC_ALLOC(buf, float*, n * 4);
        VC_TRY(write(buf));
        VC_TRY(launch_add(buf, F.grad, buf, n, st));
        F.grad = buf;
    } else {
        VC_ALLOC(tmp, float*, n * 4);
        VC_TRY(write(tmp));
        VC_TRY(launch_add(F.grad, tmp, F.grad, n, st));
    }
    F.grad_state = G_OWN;
    return VC_OK;
}

// contribution by a kernel that can ADD an existing [rows, c] matrix in its epilogue (the tensor-core gather dgrad):
// `write(dst, addend)` overwrites dst with result + addend (addend may be NULL or alias dst) — no add kernel, no temporary
template <class W>
int contribute_fused(Ctx& C, FSlot& F, W&& write) {
    const size_t n = (size_t)F.rows * F.c;
    VC_CHECK_ARG(F.gld == F.c, "a column slice of a gradient cannot take this contribution");
    if (F.grad_state == G_OWN) {
        VC_TRY(write(F.grad, (const float*)F.grad));
    } else {
        VC_ALLOC(buf, float*, n * 4);
        VC_TRY(write(buf, F.grad_state == G_EXT ? (const float*)F.grad : nullptr));
        F.grad = buf;
    }
    F.grad_state = G_OWN;
    return VC_OK;
}

// contribution by a kernel that ACCUMULATES with atomics (the scatter dgrads): `scatter(dst, ld)` adds into dst (row pitch
// ld), which must hold the sum so far — zeros, a copy of the outside gradient, or the slot's own buffer (then nothing is
// staged at all; it may be a column slice of the concat's gradient)
template <class W>
int contribute_scatter(Ctx& C, FSlot& F, cudaStream_t st, W&& scatter) {
    const size_t n = (size_t)F.rows * F.c;
    if (F.grad_state != G_OWN) {
        VC_ALLOC(buf, float*, n * 4);
        if (F.grad_state == G_EXT)
            VC_CUDA(cudaMemcpyAsync(buf, F.grad, n * 4, cudaMemcpyDeviceToDevice, st));
        else
            VC_CUDA(cudaMemsetAsync(buf, 0, n * 4, st));
        F.grad = buf;
        F.gld = F.c;
        F.grad_state = G_OWN;
    }
    return scatter(F.grad, F.gld);
}

}  // namespace
}  // namespace vc

extern "C" int vc_exec_backward(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs,
                                const float* layer_f, int n_layers, const int32_t* pub_slots, const uint64_t* ext_grads,
                                int n_pub, void* arena, size_t arena_bytes, int32_t* err_flag, void* state,
                                vc_stream_t stream_, vc_stream_t wgrad_stream_) {
    return vc_exec_backward_sync(ops_i, ops_f, n_ops, layer_ptrs, layer_f, n_layers, pub_slots, ext_grads, n_pub, arena, arena_bytes,
                                 err_flag, state, stream_, wgrad_stream_, nullptr, nullptr, nullptr, nullptr);
}

extern "C" int vc_exec_backward_sync(const int32_t* ops_i, const float* ops_f, int n_ops, const uint64_t* layer_ptrs,
                                     const float* layer_f, int n_layers, const int32_t* pub_slots, const uint64_t* ext_grads,
                                     int n_pub, void* arena, size_t arena_bytes, int32_t* err_flag, void* state,
                                     vc_stream_t stream_, vc_stream_t wgrad_stream_, double* xchg, const int64_t* xchg_off,
                                     vc_bn_exchange_fn exchange_fn, void* exchange_user) {
    VC_TRY(check_plan(ops_i, n_ops, n_layers));
    VC_CHECK_ARG(!exchange_fn || (xchg && xchg_off), "a SyncBatchNorm exchange needs its buffer and slot offsets");
    State* S = (State*)state;
    VC_CHECK_ARG(S && S->magic == STATE_MAGIC && S->n_ops == n_ops && S->n_layers == n_layers, "state does not belong to this plan");
    VC_CHECK_ARG(arena && layer_ptrs && (n_pub == 0 || (pub_slots && ext_grads)), "null argument");
    Ctx C;
    C.oi = ops_i; C.of = ops_f; C.n_ops = n_ops; C.lp = layer_ptrs; C.lf = layer_f; C.n_layers = n_layers; C.S = S;
    C.A = Arena{(char*)arena, arena_bytes, S->used, false};
    C.st[0] = (cudaStream_t)stream_;
    C.st[1] = wgrad_stream_ ? (cudaStream_t)wgrad_stream_ : (cudaStream_t)stream_;
    C.st[2] = C.st[1];
    C.err = err_flag;
    C.xchg = xchg; C.xoff = xchg_off; C.xfn = exchange_fn; C.xuser = exchange_user;
    g_ev_next = 0;
    cudaStream_t st = C.st[0];
    cudaStream_t wst = C.st[1];      // weight gradients: off the dgrad chain's critical path
    const bool two = st != wst;
    if (two) VC_TRY(ev_init());
    int last_w_ev = -1;
    const int training = S->training;
    WgradFinTable fin;          // persistent wgrad kernels accumulate into scratch images; ONE transposing launch at the end
    fin.n = 0;
    // CTAs of a wgrad launch: a cap set with vc_conv_wgrad_tc3_config is a budget over all its passes; by default half the
    // SMs for each pass, so that a CTA of the dgrad chain fits beside each.  (A budget of three quarters of the SMs per
    // launch ran faster, but fewer CTAs per pass lengthen each CTA's fp32 accumulation: DESIGN.md section 8, item 6)
    const int half_sms = (num_sms() + 1) / 2;

    for (int i = 0; i < MAX_F; ++i) { S->f[i].grad = nullptr; S->f[i].gld = S->f[i].c; S->f[i].grad_state = G_EMPTY; }
    for (int i = 0; i < n_pub; ++i) {
        VC_CHECK_ARG(pub_slots[i] > 0 && pub_slots[i] < MAX_F, "published slot id");
        if (ext_grads[i]) {
            FSlot& F = S->f[pub_slots[i]];
            VC_CHECK_ARG(F.grad_state == G_EMPTY, "slot %d published twice", pub_slots[i]);
            F.grad = reinterpret_cast<float*>(ext_grads[i]);
            F.grad_state = G_EXT;
        }
    }

    for (int i = n_ops - 1; i >= 0; --i) {
        const int* o = C.op(i);
        if (o[F_KIND] == OP_CAT) {
            FSlot& Aa = S->f[o[F_A]];
            FSlot& Bb = S->f[o[F_B]];
            FSlot& O = S->f[o[F_C]];
            if (O.grad_state == G_EMPTY) continue;
            VC_CHECK_ARG(O.gld == O.c, "op %d: the gradient of a concat is a slice itself", i);
            if (S->precision == 1 && O.grad_state == G_OWN && Aa.grad_state == G_EMPTY && Bb.grad_state == G_EMPTY) {
                // the inputs' gradients are the two column slices of the concat's own buffer: nothing is split or copied.
                // Their readers take a row pitch: BN backward, and the scatter dgrad of the image branch, which adds into
                // the first input's slice in place (nothing reads the concat's gradient after this op)
                Aa.grad = O.grad; Aa.gld = O.c; Aa.grad_state = G_OWN;
                Bb.grad = O.grad + Aa.c; Bb.gld = O.c; Bb.grad_state = G_OWN;
                continue;
            }
            float *da, *db;
            const float *a_add = nullptr, *b_add = nullptr;
            if (Aa.grad_state == G_OWN) { da = Aa.grad; a_add = Aa.grad; }
            else { VC_ALLOC(t, float*, (size_t)Aa.rows * Aa.c * 4); da = t; a_add = Aa.grad_state == G_EXT ? Aa.grad : nullptr; }
            if (Bb.grad_state == G_OWN) { db = Bb.grad; b_add = Bb.grad; }
            else { VC_ALLOC(t, float*, (size_t)Bb.rows * Bb.c * 4); db = t; b_add = Bb.grad_state == G_EXT ? Bb.grad : nullptr; }
            if (O.rows > 0) {
                cat2_bwd_kernel<<<dim3(ew_grid((size_t)O.rows * O.c / 4)), dim3(256), 0, st>>>((const float4*)O.grad, O.rows,
                    Aa.c / 4, Bb.c / 4, (float4*)da, (const float4*)a_add, (float4*)db, (const float4*)b_add);
                VC_LAUNCH_CHECK();
            }
            Aa.grad = da; Aa.gld = Aa.c; Aa.grad_state = G_OWN;
            Bb.grad = db; Bb.gld = Bb.c; Bb.grad_state = G_OWN;
            continue;
        }
        if (o[F_KIND] == OP_DISCARD) {
            // dense gather through pos: every input row gets its kept row's gradient or zero.  The buffer becomes the gradient
            // of the concat that fed the discard, which the concat's backward then hands on in column slices
            FSlot& X = S->f[o[F_CIN]];
            FSlot& Y = S->f[o[F_COUT]];
            if (Y.grad_state == G_EMPTY || o[F_CIN] == 0) continue;
            VC_CHECK_ARG(X.grad_state == G_EMPTY, "op %d: the input of a layer discard has a second gradient source", i);
            VC_ALLOC(dx, float*, (size_t)X.rows * X.c * 4);
            VC_TRY(stvd_grad_dev(Y.grad, Y.gld, X.c, S->disc[i].pos, X.rows, dx, X.c, st));
            X.grad = dx; X.gld = X.c; X.grad_state = G_OWN;
            continue;
        }
        if (o[F_KIND] != OP_CBR) continue;
        const int li = o[F_LAYER];
        Layer& L = S->layer[li];
        FSlot& X = S->f[L.in_slot];
        FSlot& Y = S->f[L.out_slot];
        RBk& R = S->rb[L.rb];
        float* dw = C.P<float>(li, P_DW);
        float* dgamma = C.P<float>(li, P_DGAMMA);
        float* dbeta = C.P<float>(li, P_DBETA);
        const size_t wn = (size_t)R.K * L.cin * L.cout;
        L.dy = nullptr; L.dy_ld = 0; L.dx = nullptr; L.dxb = nullptr;
        if (Y.grad_state == G_EMPTY || R.n_out == 0) {   // nothing flowed back into this layer
            VC_CUDA(cudaMemsetAsync(dw, 0, wn * 4, st));
            VC_CUDA(cudaMemsetAsync(dgamma, 0, (size_t)L.cout * 4, st));
            VC_CUDA(cudaMemsetAsync(dbeta, 0, (size_t)L.cout * 4, st));
            if (C.xfn != nullptr && training && Y.grad_state != G_EMPTY) {   // (no rows here, but the other ranks' exchange waits)
                VC_CUDA(cudaMemsetAsync(C.xslot(li, 1), 0, (size_t)2 * L.cout * 8, st));
                VC_TRY(exchange(C, li, 1, 2 * L.cout));
            }
            continue;
        }
        const size_t elems = (size_t)R.n_out * L.cout;
        // the fp32 input gradient is read by the fp32 wgrad and the fp32 dgrads only (the tensor-core ones read dxb)
        // (gather-form dgrad: dx / dxb are the first half of its operand U = [dout; S], 2 n_out rows)
        const bool g2 = L.dgrad == K_DGRAD_GATHER2D_F32 || L.dgrad == K_DGRAD_GATHER2D_TC;
        float* dx = nullptr;
        if (L.wgrad == K_WGRAD_F32 || L.dgrad == K_DGRAD_F32 || L.dgrad == K_DGRAD_SCATTER_F32 || L.dgrad == K_DGRAD_GATHER2D_F32) {
            VC_ALLOC(t, float*, elems * 4 * (L.dgrad == K_DGRAD_GATHER2D_F32 ? 2 : 1));
            dx = t;
        }
        void* dxb = nullptr;
        if (S->precision == 1) {
            VC_ALLOC(t, void*, elems * 2 * (L.dgrad == K_DGRAD_GATHER2D_TC ? 2 : 1));
            dxb = t;
        }
        L.dy = Y.grad; L.dy_ld = Y.gld; L.dx = dx; L.dxb = dxb;
        double* bpart = nullptr;   // deterministic mode: BN backward partials per BN_DET_ROWS chunk, added in chunk order
        if (S->deterministic) {
            const size_t pb = (size_t)cdiv(R.n_out, BN_DET_ROWS) * 2 * L.cout * 8;
            VC_ALLOC(t, double*, pb);
            bpart = t;
            S->det_bytes += pb + (g2 ? elems * (L.dgrad == K_DGRAD_GATHER2D_TC ? 2 : 4) : 0);
        }
        if (C.xfn != nullptr && training) {
            // SyncBatchNorm: local sums (and the local dgamma / dbeta) -> exchange -> dx from the all-reduced sums and the
            // forward slot's global row count
            VC_TRY(bn_relu_bwd_local_dev(Y.grad, Y.gld, L.x, L.stats, R.n_out, R.n_out_dev, L.cout, L.sums + 2 * L.cout, bpart, dgamma,
                                         dbeta, C.xslot(li, 1), st));
            VC_TRY(exchange(C, li, 1, 2 * L.cout));
            VC_TRY(bn_relu_bwd_apply_dev(Y.grad, Y.gld, L.x, C.P<const float>(li, P_GAMMA), L.stats, C.xslot(li, 1),
                                         C.xslot(li, 0) + 2 * L.cout, dx, dxb, R.n_out, R.n_out_dev, L.cout, S->is_static, st));
        } else {
            VC_TRY(bn_relu_bwd_dev(Y.grad, Y.gld, L.x, C.P<const float>(li, P_GAMMA), L.stats, dx, dxb, dgamma, dbeta, R.n_out,
                                   R.n_out_dev, L.cout, training, L.sums + 2 * L.cout, S->is_static, st, bpart));
        }
        // the wgrad needs dx / its bf16 shadow: on its own stream it waits for this event, and it is enqueued after the
        // dgrad, which is on the critical path (the dgrad's CTAs reach the SMs first)
        const int bn_ev = two ? record_on(C, 0) : -1;
        // dgrad
        const int32_t* table = R.subm ? R.nbr : R.nbr_bwd;
        const size_t wsb = vc_conv_ws_bytes(L.cin, L.cout, R.K);
        void* ws = nullptr;   // the fp32 dgrads' workspace
        if (L.dgrad == K_DGRAD_F32 || L.dgrad == K_DGRAD_SCATTER_F32 || L.dgrad == K_DGRAD_GATHER2D_F32) {
            VC_ALLOC(t, void*, wsb);
            ws = t;
        }
        switch (L.dgrad) {
            case K_DGRAD_SCATTER_TC:
                VC_TRY(contribute_scatter(C, X, st, [&](float* dst, int ld) -> int {
                    Timed t(L.dgrad, li, st);
                    return tc_scatter_with_image(L.cout, L.cin, dxb, L.wimg_dgrad, R.nbr, dst, R.n_out, R.K, C.err, st, ld);
                }));
                break;
            case K_DGRAD_SCATTER_F32:
                VC_TRY(contribute_scatter(C, X, st, [&](float* dst, int ld) -> int {
                    Timed t(L.dgrad, li, st);
                    return conv_dgrad_scatter_f32_ld(dx, C.P<const float>(li, P_W), R.nbr, dst, ld, R.n_out, L.cin, L.cout, R.K, ws, wsb, st);
                }));
                break;
            case K_DGRAD_GATHER2D_TC:
            case K_DGRAD_GATHER2D_F32:
                // S into U's second half, one mirrored gather dgrad over the group table, then added into the slot's gradient
                // (which may be a column slice of the concat's gradient: row pitch ld)
                VC_TRY(contribute_scatter(C, X, st, [&](float* dst, int ld) -> int {
                    const bool tc = L.dgrad == K_DGRAD_GATHER2D_TC;
                    VC_ALLOC(tmp, float*, (size_t)R.n_in * L.cin * 4);
                    S->det_bytes += (size_t)R.n_in * L.cin * 4;
                    Timed t(L.dgrad, li, st);
                    VC_TRY(gather2d_sum_dev(tc ? nullptr : dx, tc ? dxb : nullptr, L.cout, R.g2, R.n_in, R.n_in_dev, tc ? nullptr : dx,
                                            tc ? dxb : nullptr, st));
                    if (tc)
                        VC_TRY(tc2_conv(L.cout, L.cin, dxb, L.wimg_dgrad, R.g2.nbr_g, R.n_in, tmp, R.n_in, R.n_in_dev, R.K, nullptr, C.err,
                                        st, nullptr, L.tile_ctr + 1));
                    else
                        VC_TRY(vc_conv_dgrad_f32(dx, C.P<const float>(li, P_W), R.g2.nbr_g, tmp, R.n_in, L.cin, L.cout, R.K, 1, ws, wsb,
                                                 st));
                    return add_rows_ld_dev(dst, ld, tmp, R.n_in, R.n_in_dev, L.cin, st);
                }));
                break;
            case K_DGRAD_TC:
                VC_TRY(contribute_fused(C, X, [&](float* dst, const float* addend) -> int {
                    Timed t(L.dgrad, li, st);
                    // (static mode: the slot's gradient has zero rows past its count, as every BN output has)
                    return tc2_conv(L.cout, L.cin, dxb, L.wimg_dgrad, table, R.n_in, dst, R.n_in, R.n_in_dev, R.K, nullptr, C.err, st,
                                    addend, L.tile_ctr + 1, (R.subm ? 0 : 1) | 4);
                }));
                break;
            case K_DGRAD_F32:
                VC_TRY(contribute(C, X, st, [&](float* dst) -> int {
                    Timed t(L.dgrad, li, st);
                    return vc_conv_dgrad_f32(dx, C.P<const float>(li, P_W), table, dst, R.n_in, L.cin, L.cout, R.K, R.subm ? 1 : 0, ws,
                                             wsb, st);
                }));
                break;
            default: break;   // K_NONE
        }
        // wgrad
        if (bn_ev >= 0) VC_CUDA(cudaStreamWaitEvent(wst, g_ev[bn_ev], 0));
        if (L.wgrad == K_WGRAD_TC) {
            Timed t(L.wgrad, li, wst);
            VC_TRY(tc3_wgrad(L.cin, L.cout, X.bf16, dxb, R.nbr, R.n_out, L.wscratch, R.n_out, R.n_out_dev, R.K, C.err, wst,
                             L.tile_ctr + 2, g_wgrad3_ctas > 0 ? g_wgrad3_ctas : half_sms * wgrad3_passes(L.cin, L.cout, R.K), X.ld,
                             S->deterministic ? WGRAD_DET_CHUNKS : 0));
            if (fin.n == WGRAD_FIN_MAX) {
                VC_TRY(wgrad_finalize(fin, wst));
                fin.n = 0;
            }
            WgradFinEntry& fe = fin.e[fin.n++];
            fe.scratch = L.wscratch; fe.dw = dw; fe.cin = L.cin; fe.cout = L.cout; fe.K = R.K; fe.first = 0;
            fe.n_part = S->deterministic ? WGRAD_DET_CHUNKS : 1;
        } else {
            const size_t wsb = vc_conv_wgrad_ws_bytes(R.n_out, L.cin, L.cout, R.K);
            VC_ALLOC(ws, void*, wsb);
            VC_CHECK_ARG(X.f32 && X.ld == X.c, "layer %d: the fp32 wgrad needs a dense fp32 input", li);
            Timed t(L.wgrad, li, wst);
            VC_TRY(vc_conv_wgrad_f32(X.f32, dx, R.nbr, dw, R.n_out, L.cin, L.cout, R.K, ws, wsb, wst));
        }
        if (two) last_w_ev = record_on(C, 1);
    }
    if (fin.n > 0) {
        VC_TRY(wgrad_finalize(fin, wst));
        if (two) last_w_ev = record_on(C, 1);
    }
    if (two && last_w_ev >= 0) VC_CUDA(cudaStreamWaitEvent(st, g_ev[last_w_ev], 0));   // join: gradients complete on `stream`
    S->used = C.A.used;
    return VC_OK;
}
