// api.cu -- the extern "C" boundary of liblfd_b200.so (declared in include/lfd_b200.h).
#include <stdarg.h>
#include <cmath>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../include/lfd_b200.h"
#include "conv_common.cuh"
#include "kernels.cuh"
#include "train.cuh"

using namespace lfd;

static thread_local char g_err[512] = "";
static long long* g_trace = nullptr;   // debugging: see lfd_debug_set_trace
static unsigned long long* g_timeline = nullptr;   // debugging: see lfd_debug_set_timeline

static int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) return fail(LFD_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

static inline cudaStream_t st_of(lfd_stream s) { return reinterpret_cast<cudaStream_t>(s); }

static int sm_count() {   // of the CURRENT device (cached per device ordinal)
    static int cached[kMaxDevices] = {};
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return 0;
    if (cached[dev] > 0) return cached[dev];
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    cached[dev] = n;
    return n;
}

struct PlannedOp {
    lfd_op op;
    UmmaConvParams cp;  // CONV via wgmma
    size_t smem;
    int grid;
    InputTransform xf;  // STEM0 / STEM4 (and a training plan's WGRAD_STEM): the op's input transform with the all-zero default resolved
};

// Stream the CUDA graphs are captured on: the main chain (the backbone: the critical path of the step) runs two priority levels above
// the side streams of the per-level chains (created at the default = lowest level) -- captured kernel nodes inherit the level, so when
// SMs free up the pending CTAs of the critical path are placed first.  The levels above are left to the caller's latency-critical
// streams (lfd/pipeline.py runs the post-process of the previous batch there).  A device that reports no priority range gets a
// stream at the default level.
static cudaError_t create_capture_stream(cudaStream_t* cap) {
    int least = 0, greatest = 0;
    if (cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess && greatest < least) {
        const int level = least - 2 < greatest ? greatest : least - 2;     // numerically lower = higher priority
        return cudaStreamCreateWithPriority(cap, cudaStreamNonBlocking, level);
    }
    return cudaStreamCreateWithFlags(cap, cudaStreamNonBlocking);
}

// Runs the op list of either plan kind (lfd_plan, lfd_train_plan).  Op i runs on the caller's stream (branch 0) or on side stream b,
// forked after the main-stream op that precedes the branch's first op; wait_mask bit w makes it wait for everything enqueued so far on
// branch w; every started branch is joined back into the caller's stream at the end.  With use_graph the sequence is captured into a
// CUDA graph on the first use of a pointer tuple and replayed afterwards.  launch(i, stream) enqueues op i and returns a status.
struct BranchExecutor {
    std::vector<int> branch, wait_mask;    // per op
    int n_branches = 1;                    // side[b], fork_ev[b] and join_ev[b] exist for 1 <= b < n_branches
    cudaStream_t side[LFD_MAX_BRANCHES];
    cudaEvent_t fork_ev[LFD_MAX_BRANCHES], join_ev[LFD_MAX_BRANCHES];
    std::vector<cudaEvent_t> dep_ev;       // one per (op, wait_mask bit): mid-graph cross-branch dependencies
    int64_t clear_off = 0, clear_bytes = 0;   // workspace region zeroed on the caller's stream before the first op
    size_t max_graphs = 0;
    struct Graph {
        cudaGraphExec_t exec;
        const void* input;
        void* ws;
        float* cls;
        float* reg;
        int fmt;
        const void* ext;
    };
    std::vector<Graph> graphs;             // one instantiated graph per (input, workspace, cls, reg, format, geometry table) tuple, oldest first

    BranchExecutor() = default;
    BranchExecutor(const BranchExecutor&) = delete;
    BranchExecutor& operator=(const BranchExecutor&) = delete;
    ~BranchExecutor() {
        for (auto& g : graphs) cudaGraphExecDestroy(g.exec);
        for (int b = 1; b < n_branches; ++b) {
            cudaStreamDestroy(side[b]);
            cudaEventDestroy(fork_ev[b]);
            cudaEventDestroy(join_ev[b]);
        }
        for (auto ev : dep_ev) cudaEventDestroy(ev);
    }

    // Validates the schedule (branch_of(i), wait_of(i)) and creates the side streams and events.  On failure it keeps only what it
    // created completely, which the destructor releases.
    template <typename BranchOf, typename WaitOf>
    int init(const char* who, int n_ops, BranchOf branch_of, WaitOf wait_of, size_t graph_cap) {
        max_graphs = graph_cap;
        int nb = 1;
        size_t n_dep = 0;
        for (int i = 0; i < n_ops; ++i) {
            const int b = branch_of(i), w = wait_of(i);
            if (b < 0 || b >= LFD_MAX_BRANCHES || w < 0 || w >= (1 << LFD_MAX_BRANCHES))
                return fail(LFD_ERR_INVALID, "%s: op %d: branch %d / wait_mask 0x%x out of range", who, i, b, w);
            branch.push_back(b);
            wait_mask.push_back(w);
            if (b + 1 > nb) nb = b + 1;
            n_dep += (size_t)__builtin_popcount((unsigned)w);
        }
        for (int b = 1; b < nb; ++b) {
            if (cudaStreamCreateWithFlags(&side[b], cudaStreamNonBlocking) != cudaSuccess) return fail(LFD_ERR_CUDA, "%s: cannot create side streams", who);
            if (cudaEventCreateWithFlags(&fork_ev[b], cudaEventDisableTiming) != cudaSuccess) {
                cudaStreamDestroy(side[b]);
                return fail(LFD_ERR_CUDA, "%s: cannot create events", who);
            }
            if (cudaEventCreateWithFlags(&join_ev[b], cudaEventDisableTiming) != cudaSuccess) {
                cudaStreamDestroy(side[b]);
                cudaEventDestroy(fork_ev[b]);
                return fail(LFD_ERR_CUDA, "%s: cannot create events", who);
            }
            n_branches = b + 1;
        }
        for (size_t i = 0; i < n_dep; ++i) {
            cudaEvent_t ev;
            if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) return fail(LFD_ERR_CUDA, "%s: cannot create dependency events", who);
            dep_ev.push_back(ev);
        }
        return LFD_OK;
    }

    // Fork / wait / launch / join.  Every started branch is joined also on error paths, so that a stream capture can be closed.
    template <typename Launch>
    int enqueue(uint8_t* ws, cudaStream_t st, const Launch& launch) {
        if (clear_bytes > 0) CUDA_TRY(cudaMemsetAsync(ws + clear_off, 0, (size_t)clear_bytes, st));
        bool started[LFD_MAX_BRANCHES] = {false};
        int rc = LFD_OK;
        size_t dep = 0;
        cudaError_t ce = cudaSuccess;
        for (size_t i = 0; i < branch.size() && !rc && ce == cudaSuccess; ++i) {
            const int b = branch[i];
            cudaStream_t s = b > 0 ? side[b] : st;
            if (b > 0 && !started[b]) {   // fork: everything enqueued on the main stream so far precedes this branch
                if ((ce = cudaEventRecord(fork_ev[b], st)) != cudaSuccess || (ce = cudaStreamWaitEvent(s, fork_ev[b], 0)) != cudaSuccess) break;
                started[b] = true;
            }
            for (int w = 0; w < LFD_MAX_BRANCHES && ce == cudaSuccess; ++w) {   // explicit cross-branch dependencies
                if (!((wait_mask[i] >> w) & 1)) continue;
                cudaEvent_t ev = dep_ev[dep++];
                if (w == b || (w > 0 && (w >= n_branches || !started[w]))) continue;   // nothing to wait for
                if ((ce = cudaEventRecord(ev, w == 0 ? st : side[w])) == cudaSuccess) ce = cudaStreamWaitEvent(s, ev, 0);
            }
            if (ce == cudaSuccess) rc = launch(i, s);
        }
        for (int b = 1; b < n_branches; ++b)
            if (started[b]) {
                cudaEventRecord(join_ev[b], side[b]);
                cudaStreamWaitEvent(st, join_ev[b], 0);
            }
        if (!rc && ce != cudaSuccess) rc = fail(LFD_ERR_CUDA, "plan stream dependencies: %s", cudaGetErrorString(ce));
        return rc;
    }

    template <typename Launch>
    int run(const void* input, int fmt, void* workspace, float* cls, float* reg, const void* ext, int use_graph, cudaStream_t st, Launch launch) {
        uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
        if (!use_graph) return enqueue(ws, st, launch);
        for (auto& g : graphs)
            if (g.input == input && g.ws == workspace && g.cls == cls && g.reg == reg && g.fmt == fmt && g.ext == ext) {
                CUDA_TRY(cudaGraphLaunch(g.exec, st));
                return LFD_OK;
            }
        // first use of this pointer tuple: one eager pass (sets function attributes outside of capture, surfaces launch errors directly
        // and produces this call's results), then capture + instantiate for the following calls.  Capture executes nothing, so the
        // state (statistics, staging) is untouched.
        int rc = enqueue(ws, st, launch);
        if (rc) return rc;
        if (graphs.size() >= max_graphs) {
            cudaGraphExecDestroy(graphs.front().exec);
            graphs.erase(graphs.begin());
        }
        cudaStream_t cap;
        CUDA_TRY(create_capture_stream(&cap));
        cudaGraph_t graph = nullptr;
        cudaError_t ce = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
        if (ce != cudaSuccess) { cudaStreamDestroy(cap); return fail(LFD_ERR_CUDA, "cudaStreamBeginCapture: %s", cudaGetErrorString(ce)); }
        rc = enqueue(ws, cap, launch);
        ce = cudaStreamEndCapture(cap, &graph);
        if (rc || ce != cudaSuccess) {
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cap);
            return rc ? rc : fail(LFD_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
        }
        Graph e = {nullptr, input, workspace, cls, reg, fmt, ext};
        ce = cudaGraphInstantiate(&e.exec, graph, 0);
        cudaGraphDestroy(graph);
        cudaStreamDestroy(cap);
        if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ce));
        graphs.push_back(e);
        return LFD_OK;
    }

    // One eager pass with every op on the caller's stream and an event pair around each -> ms_per_op[i].
    template <typename Launch>
    int profile(const char* who, uint8_t* ws, float* ms_per_op, cudaStream_t st, Launch launch) {
        const size_t n = branch.size();
        std::vector<cudaEvent_t> ev(n + 1);
        for (auto& e : ev) CUDA_TRY(cudaEventCreate(&e));
        if (clear_bytes > 0) CUDA_TRY(cudaMemsetAsync(ws + clear_off, 0, (size_t)clear_bytes, st));
        int rc = LFD_OK;
        CUDA_TRY(cudaEventRecord(ev[0], st));
        for (size_t i = 0; i < n && !rc; ++i) {
            rc = launch(i, st);
            cudaEventRecord(ev[i + 1], st);
        }
        cudaError_t ce = cudaStreamSynchronize(st);
        if (!rc && ce == cudaSuccess)
            for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
        for (auto& e : ev) cudaEventDestroy(e);
        if (rc) return rc;
        if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "%s: %s", who, cudaGetErrorString(ce));
        return LFD_OK;
    }
};


extern "C" int lfd_debug_set_trace(void* device_buffer) {
    g_trace = reinterpret_cast<long long*>(device_buffer);
    return LFD_OK;
}
extern "C" int lfd_debug_set_timeline(void* device_buffer) {
    g_timeline = reinterpret_cast<unsigned long long*>(device_buffer);
    return LFD_OK;
}
extern "C" int lfd_abi_version(void) { return LFD_B200_ABI_VERSION; }
extern "C" int lfd_struct_bytes(int which) {
    switch (which) {
        case 0: return (int)sizeof(lfd_op);
        case 1: return (int)sizeof(lfd_top);
        case 2: return (int)sizeof(lfd_pack_desc);
        case 3: return (int)sizeof(lfd_unpack_desc);
        case 4: return (int)sizeof(lfd_post_cfg);
        case 5: return (int)sizeof(lfd_loss_cfg);
        case 6: return (int)sizeof(lfd_levels);
        case 7: return (int)sizeof(lfd_input_desc);
        case 8: return (int)sizeof(lfd_extent);
        case 9: return (int)sizeof(lfd_engine_desc);
    }
    return -1;
}
extern "C" const char* lfd_last_error(void) { return g_err; }
extern "C" int lfd_device_sm_count(void) {
    int n = sm_count();
    if (n <= 0) fail(LFD_ERR_CUDA, "no usable CUDA device");
    return n;
}

static ConvGeom geom_of(const lfd_op& o) {
    ConvGeom g;
    g.N = o.N; g.H = o.H; g.W = o.W; g.Cin = o.Cin; g.Ho = o.Ho; g.Wo = o.Wo; g.Cout = o.Cout; g.ksize = o.ksize; g.stride = o.stride;
    g.stem = o.kind == LFD_OP_STEM0 ? 1 : 0;
    g.stem4 = o.kind == LFD_OP_STEM4 ? 1 : 0;
    g.tail_cout = o.tail_cout;
    g.ds_cout = o.ds_cout;
    if (g.stem) g.Cin = 16;   // K of one filter row: 4 pixels x 4 (padded) channels
    return g;
}

extern "C" int lfd_conv_query(int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int ksize, int stride, int tail_cout, int ds_cout, int* cc,
                              int* stages, int* weights_resident, int* num_tiles, int64_t* smem_bytes) {
    ConvGeom g = {N, H, W, Cin, Ho, Wo, Cout, ksize, stride, tail_cout, ds_cout, 0};
    UmmaConvParams p;
    size_t smem = 0;
    int grid = 0;
    int rc = umma_conv_configure(g, 132, &p, &smem, &grid);
    if (rc) return fail(LFD_ERR_UNSUPPORTED, "conv %dx%d s%d Cin=%d Cout=%d not supported by the wgmma kernel (rc=%d)", ksize, ksize, stride, Cin, Cout, rc);
    if (cc) *cc = p.Cc;
    if (stages) *stages = p.stages;
    if (weights_resident) *weights_resident = p.b_resident;
    if (num_tiles) *num_tiles = p.num_tiles;
    if (smem_bytes) *smem_bytes = (int64_t)smem;
    return LFD_OK;
}

extern "C" int lfd_conv_schedule(int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int ksize, int stride, int tail_cout, int ds_cout,
                                 int* solo) {
    ConvGeom g = {N, H, W, Cin, Ho, Wo, Cout, ksize, stride, tail_cout, ds_cout, 0};
    UmmaConvParams p;
    size_t smem = 0;
    int grid = 0;
    int rc = umma_conv_configure(g, sm_count() > 0 ? sm_count() : 132, &p, &smem, &grid);
    if (rc) return fail(LFD_ERR_UNSUPPORTED, "conv %dx%d s%d Cin=%d Cout=%d not supported by the wgmma kernel (rc=%d)", ksize, ksize, stride, Cin, Cout, rc);
    if (solo) *solo = p.solo;
    return LFD_OK;
}

extern "C" int lfd_stem4_query(int N, int H, int W, int* num_tiles, int64_t* smem_bytes, int* Ho, int* Wo) {
    const int h1 = (H - 1) / 2 + 1, w1 = (W - 1) / 2 + 1;
    ConvGeom g = {N, H, W, 3, (h1 - 1) / 2 + 1, (w1 - 1) / 2 + 1, 64, 3, 2, 64, 0, 0, 1};
    UmmaConvParams p;
    size_t smem = 0;
    int grid = 0;
    if (N < 1 || H < 1 || W < 1 || umma_conv_configure(g, 132, &p, &smem, &grid)) return fail(LFD_ERR_UNSUPPORTED, "stem4: unsupported size N=%d H=%d W=%d", N, H, W);
    if (num_tiles) *num_tiles = p.num_tiles;
    if (smem_bytes) *smem_bytes = (int64_t)smem;
    if (Ho) *Ho = p.Ho;
    if (Wo) *Wo = p.Wo;
    return LFD_OK;
}

// The input transform of an op as the kernels take it (constants by byte position, kernels.cuh) from the C-ABI's fields (by network
// channel, see lfd_op): all seven fields zero = simple_normalize; anything else has to be a complete transform.  One place for lfd_op
// and lfd_top, and for both image kinds: BGR (cin 3) and gray (cin 1), whose one channel is (byte - mean[0]) * scale[0] -- it has no
// channel swap and takes three equal constants, so every byte position of the resolved transform holds channel 0's.
static int input_transform_of(int cin, int32_t swap, const float* mean, const float* scale, InputTransform* out) {
    bool zero = swap == 0;
    for (int c = 0; c < 3; ++c) zero = zero && mean[c] == 0.f && scale[c] == 0.f;
    if (zero) {
        out->swap = 0;
        for (int c = 0; c < 3; ++c) { out->mean[c] = 127.5f; out->scale[c] = 1.0f / 127.5f; }
        return LFD_OK;
    }
    if (swap != 0 && swap != 1) return fail(LFD_ERR_INVALID, "input transform: in_swap_rb = %d (0 or 1)", swap);
    if (cin == 1 && (swap || mean[1] != mean[0] || mean[2] != mean[0] || scale[1] != scale[0] || scale[2] != scale[0]))
        return fail(LFD_ERR_INVALID, "input transform of a gray (1-channel) image: in_swap_rb must be 0 and the three in_mean / in_scale equal "
                    "(got swap %d, mean %g %g %g, scale %g %g %g)", swap, (double)mean[0], (double)mean[1], (double)mean[2], (double)scale[0],
                    (double)scale[1], (double)scale[2]);
    for (int c = 0; c < 3; ++c)
        if (!std::isfinite(mean[c]) || !std::isfinite(scale[c]) || scale[c] == 0.f)
            return fail(LFD_ERR_INVALID, "input transform: channel %d has mean %g, scale %g (set all of in_swap_rb / in_mean / in_scale with finite means and "
                        "finite non-zero scales, or none of them)", c, (double)mean[c], (double)scale[c]);
    out->swap = swap;
    for (int m = 0; m < 3; ++m) { out->mean[m] = mean[swap ? 2 - m : m]; out->scale[m] = scale[swap ? 2 - m : m]; }   // by byte position
    return LFD_OK;
}

static int check_op(const lfd_op& o) {
    const int eh = (o.H + 2 * (o.ksize / 2) - o.ksize) / (o.stride > 0 ? o.stride : 1) + 1;
    const int ew = (o.W + 2 * (o.ksize / 2) - o.ksize) / (o.stride > 0 ? o.stride : 1) + 1;
    if (o.dtype != LFD_DTYPE_BF16 && o.dtype != LFD_DTYPE_FP16) return fail(LFD_ERR_INVALID, "op dtype %d: expected LFD_DTYPE_BF16 or LFD_DTYPE_FP16", o.dtype);
    switch (o.kind) {
        case LFD_OP_STEM0:
            if (o.scale || o.tail_scale) return fail(LFD_ERR_INVALID, "conv scale must be folded into the packed weights (pass scale = NULL)");
            if ((o.Cin != 3 && o.Cin != 1) || o.ksize != 3 || o.stride != 2)
                return fail(LFD_ERR_UNSUPPORTED, "stem0 supports 3x3/s2 on 3 (BGR) or 1 (gray) input channels only (got Cin=%d k=%d s=%d)", o.Cin, o.ksize, o.stride);
            if (o.Cout != 16 && o.Cout != 32 && o.Cout != 48 && o.Cout != 64) return fail(LFD_ERR_UNSUPPORTED, "stem0 Cout must be 16/32/48/64 (got %d)", o.Cout);
            if (o.Ho != eh || o.Wo != ew) return fail(LFD_ERR_INVALID, "stem0 output size mismatch");
            break;
        case LFD_OP_STEM4:
            if (o.scale || o.tail_scale) return fail(LFD_ERR_INVALID, "conv scale must be folded into the packed weights (pass scale = NULL)");
            if ((o.Cin != 3 && o.Cin != 1) || o.ksize != 3 || o.stride != 2 || o.Cout != 64 || o.tail_cout != 64 || o.ds_cout || o.res_off >= 0 || o.gn_groups)
                return fail(LFD_ERR_UNSUPPORTED, "stem4 is 3x3/s2 3->64 or 1->64 (got Cin=%d), 1x1 64->64, 3x3/s2 64->64, 1x1 64->64 without residual / statistics", o.Cin);
            if (!o.weight || !o.tail_weight || !o.s2_weight || !o.s3_weight) return fail(LFD_ERR_INVALID, "stem4 needs the weights of all four convs");
            if (o.Ho != (eh - 1) / 2 + 1 || o.Wo != (ew - 1) / 2 + 1) return fail(LFD_ERR_INVALID, "stem4 output size mismatch (expected the stem3 map)");
            break;
        case LFD_OP_CONV:
            if (o.scale || o.tail_scale) return fail(LFD_ERR_INVALID, "conv scale must be folded into the packed weights (pass scale = NULL)");
            if (o.Ho != eh || o.Wo != ew) return fail(LFD_ERR_INVALID, "conv output size mismatch (%dx%d vs %dx%d)", o.Ho, o.Wo, eh, ew);
            if (o.gn_groups && ((o.tail_cout ? o.tail_cout : o.Cout) != o.gn_groups * 8 || o.gn_groups != 16)) return fail(LFD_ERR_UNSUPPORTED, "fused GroupNorm statistics need 16 groups of 8 channels (Cout=%d groups=%d)", o.Cout, o.gn_groups);
            if (o.cc <= 0 || o.Cin % o.cc) return fail(LFD_ERR_INVALID, "conv cc=%d does not divide Cin=%d", o.cc, o.Cin);
            if (o.ds_cout && (o.ksize != 3 || o.stride != 2 || o.tail_cout || o.res_off >= 0 || o.gn_groups || o.ds_cout != o.Cout || !o.ds_weight || o.ds_out_off < 0))
                return fail(LFD_ERR_INVALID, "a fused shortcut conv needs a 3x3/s2 conv without tail / residual / GroupNorm, ds_cout == Cout, weights and an output offset");
            break;
        case LFD_OP_GN_APPLY:
        case LFD_OP_HEAD_FINAL:
            if (o.kind == LFD_OP_HEAD_FINAL && o.gn_groups == 0) break;   // head without norm layers: the input is already activated
            if (o.Cin != o.gn_groups * 8) return fail(LFD_ERR_UNSUPPORTED, "GroupNorm needs groups of 8 channels (C=%d groups=%d)", o.Cin, o.gn_groups);
            break;
        default:
            return fail(LFD_ERR_INVALID, "unknown op kind %d", o.kind);
    }
    return LFD_OK;
}

// GN_APPLY / HEAD_FINAL and the SIMT training ops size their grids from the SM count: a max_ctas bound (side-branch layers, see lfd_op;
// forced small grids in the tests) scales them the same way
static int bounded_sms(int max_ctas) {
    const int sms = sm_count() > 0 ? sm_count() : 132;
    return max_ctas > 0 && max_ctas < sms ? max_ctas : sms;
}

static int plan_op(const lfd_op& o, PlannedOp* out) {
    int rc = check_op(o);
    if (rc) return rc;
    out->op = o;
    out->smem = 0;
    out->grid = 0;
    if (o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4) {
        rc = input_transform_of(o.Cin, o.in_swap_rb, o.in_mean, o.in_scale, &out->xf);
        if (rc) return rc;
    }
    if (o.kind == LFD_OP_CONV || o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4) {
        rc = umma_conv_configure(geom_of(o), sm_count() > 0 ? sm_count() : 132, &out->cp, &out->smem, &out->grid);
        if (rc) return fail(LFD_ERR_UNSUPPORTED, "conv %dx%d s%d Cin=%d Cout=%d unsupported (rc=%d)", o.ksize, o.ksize, o.stride, o.Cin, o.Cout, rc);
        if (o.kind == LFD_OP_CONV && out->cp.Cc != o.cc) return fail(LFD_ERR_INVALID, "weights packed with cc=%d but the kernel needs cc=%d", o.cc, out->cp.Cc);
        if (o.max_ctas < 0) return fail(LFD_ERR_INVALID, "max_ctas = %d", o.max_ctas);
        if (o.max_ctas > 0 && out->grid > o.max_ctas) out->grid = o.max_ctas;   // tiles are strided by gridDim (fused stem: contiguous runs): any grid size is valid
    }
    return LFD_OK;
}

// The image a stem op reads: its format, its op's channel count and resolved transform.  fp32 planes are taken as they are, in the
// order they lie: the transform and its channel swap apply to uint8 input only.
static ImageIn image_in(const void* input, int format, int cin, int H, int W, const InputTransform& xf) {
    ImageIn img = {input, format, cin, H, W, xf};
    if (format == LFD_INPUT_F32_NCHW) img.xf.swap = 0;
    return img;
}

// ext: null, or this op's row of a plan's device geometry table (lfd_plan_forward_extent), which the kernel reads when it starts
static int launch_op(const PlannedOp& po, size_t index, const void* input, int input_format, uint8_t* ws, float* cls, float* reg, int P,
                     int cls_channels, int conv_impl, cudaStream_t st, const lfd_extent* ext = nullptr) {
    const lfd_op& o = po.op;
    unsigned long long* tl = g_timeline ? g_timeline + 2 * index : nullptr;
    const int* ext_row = ext ? &ext->H : nullptr;
    if (ext && conv_impl == LFD_CONV_SIMT) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels run full-size frames only");
    switch (o.kind) {
        case LFD_OP_STEM0: {
            if (!input) return fail(LFD_ERR_INVALID, "stem0 needs the external input pointer");
            if (conv_impl == LFD_CONV_SIMT) {
                if (o.tail_cout) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels do not implement fused tails");
                Stem0Params p;
                p.img = image_in(input, input_format, o.Cin, o.H, o.W, po.xf);
                p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off);
                p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift;
                p.N = o.N; p.Ho = o.Ho; p.Wo = o.Wo; p.Cout = o.Cout; p.relu = o.relu; p.f16 = o.dtype;
                CUDA_TRY(stem0_launch(p, st));
            } else {
                UmmaConvParams p = po.cp;
                p.img = image_in(input, input_format, o.Cin, o.H, o.W, po.xf); p.in = nullptr;
                p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off); p.res = nullptr;
                p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift; p.stats = nullptr;
                p.relu = o.relu; p.gn_groups = 0; p.trace = g_trace; p.tl = tl; p.f16 = o.dtype;
                p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.tail_weight); p.shift2 = o.tail_shift; p.relu2 = o.tail_relu;
                p.ext = ext_row;
                if (umma_conv_encode_maps(&p)) return fail(LFD_ERR_CUDA, "cuTensorMapEncodeTiled failed for the stem conv");
                CUDA_TRY(umma_conv_launch(p, po.smem, po.grid, st));
            }
            break;
        }
        case LFD_OP_STEM4: {
            if (!input) return fail(LFD_ERR_INVALID, "stem4 needs the external input pointer");
            if (conv_impl == LFD_CONV_SIMT) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels do not implement the fused stem (plan its four convs)");
            UmmaConvParams p = po.cp;
            p.img = image_in(input, input_format, o.Cin, o.H, o.W, po.xf); p.in = nullptr;
            // the word loader: rows of whole aligned words (BGR: 3 words per 4 pixels; gray: 1 word per 4 pixels; NV12: a Y word and a UV
            // word, its image pitch H * W * 3 / 2 then being a multiple of 4 as well, since H is even)
            p.in_words = input_format != LFD_INPUT_F32_NCHW && o.W % 4 == 0 && (reinterpret_cast<uintptr_t>(input) & 3) == 0;
            p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off); p.res = nullptr; p.stats = nullptr;
            p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift; p.relu = o.relu;
            p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.tail_weight); p.shift2 = o.tail_shift; p.relu2 = o.tail_relu;
            p.w_s2 = reinterpret_cast<const __nv_bfloat16*>(o.s2_weight); p.shift_s2 = o.s2_shift; p.relu_s2 = o.s2_relu;
            p.w_s3 = reinterpret_cast<const __nv_bfloat16*>(o.s3_weight); p.shift_s3 = o.s3_shift; p.relu_s3 = o.s3_relu;
            p.gn_groups = 0; p.trace = g_trace; p.tl = tl; p.f16 = o.dtype; p.ext = ext_row;
            if (umma_conv_encode_maps(&p)) return fail(LFD_ERR_CUDA, "cuTensorMapEncodeTiled failed for the fused stem");
            CUDA_TRY(umma_conv_launch(p, po.smem, po.grid, st));
            break;
        }
        case LFD_OP_CONV: {
            const __nv_bfloat16* in =reinterpret_cast<const __nv_bfloat16*>(ws + o.in_off);
            __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off);
            const __nv_bfloat16* res = o.res_off >= 0 ? reinterpret_cast<const __nv_bfloat16*>(ws + o.res_off) : nullptr;
            double* stats = o.gn_groups ? reinterpret_cast<double*>(ws + o.stats_off) : nullptr;
            if (conv_impl == LFD_CONV_SIMT) {
                if (o.tail_cout || o.ds_cout) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels do not implement fused tails / shortcuts");
                CUDA_TRY(simt_conv_launch(geom_of(o), o.cc, in, out, res, reinterpret_cast<const __nv_bfloat16*>(o.weight),
                                          o.shift, stats, o.gn_groups, o.relu, o.dtype, st));
            } else {
                UmmaConvParams p = po.cp;
                p.in = in; p.out = out; p.res = res; p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight);
                p.shift = o.shift; p.stats = stats; p.relu = o.relu; p.gn_groups = o.gn_groups; p.f16 = o.dtype;
                p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.tail_weight); p.shift2 = o.tail_shift; p.relu2 = o.tail_relu;
                if (o.ds_cout) {
                    p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.ds_weight); p.shift2 = o.ds_shift; p.relu2 = 0;
                    p.out3 = reinterpret_cast<__nv_bfloat16*>(ws + o.ds_out_off);
                }
                p.trace = g_trace; p.tl = tl; p.ext = ext_row;
                if (umma_conv_encode_maps(&p)) return fail(LFD_ERR_CUDA, "cuTensorMapEncodeTiled failed for conv %dx%d Cf=%d", o.ksize, o.ksize, p.Cf);
                CUDA_TRY(umma_conv_launch(p, po.smem, po.grid, st));
            }
            break;
        }
        case LFD_OP_GN_APPLY: {
            GnApplyParams p;
            p.in = reinterpret_cast<const __nv_bfloat16*>(ws + o.in_off); p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off);
            p.stats = reinterpret_cast<const double*>(ws + o.stats_off); p.gamma = o.gamma; p.beta = o.beta;
            p.N = o.N; p.HW = o.H * o.W; p.C = o.Cin; p.groups = o.gn_groups; p.eps = 1e-5f; p.tl = tl; p.f16 = o.dtype;
            p.ext = ext_row; p.W = o.W;
            CUDA_TRY(gn_apply_launch(p, bounded_sms(o.max_ctas), st));
            break;
        }
        case LFD_OP_HEAD_FINAL: {
            HeadFinalParams p;
            p.in = reinterpret_cast<const __nv_bfloat16*>(ws + o.in_off);
            p.stats = o.gn_groups ? reinterpret_cast<const double*>(ws + o.stats_off) : nullptr; p.gamma = o.gamma; p.beta = o.beta;
            p.w = reinterpret_cast<const float*>(o.weight); p.scale = o.scale; p.shift = o.shift;
            p.cls = o.n_cls ? cls : nullptr; p.reg = o.n_reg ? reg : nullptr;
            p.N = o.N; p.HW = o.H * o.W; p.C = o.Cin; p.groups = o.gn_groups; p.n_out = o.n_cls + o.n_reg; p.n_cls = o.n_cls;
            p.P = P; p.point_off = o.point_off; p.cls_stride = cls_channels; p.eps = 1e-5f; p.tl = tl; p.f16 = o.dtype;
            p.ext = ext_row; p.W = o.W;
            if ((o.n_cls && !cls) || (o.n_reg && !reg)) return fail(LFD_ERR_INVALID, "head_final needs cls/reg output pointers");
            if (o.n_reg && o.n_reg != 4) return fail(LFD_ERR_INVALID, "head_final n_reg must be 0 or 4");
            CUDA_TRY(head_final_launch(p, bounded_sms(o.max_ctas), st));
            break;
        }
    }
    return LFD_OK;
}

// graph-cache bounds: how many pointer tuples a plan keeps an instantiated graph for (callers rotate input buffers and output slots)
static constexpr size_t kMaxInferenceGraphs = 32;
static constexpr size_t kMaxTrainingGraphs = 8;

// Host staging of the geometry table: a frame's table is written into the next slot of a ring of pinned buffers and copied to the device
// table on the caller's stream; a slot is rewritten only after the event recorded behind its last copy has completed.
static constexpr int kExtentRing = 4;

struct lfd_plan {
    std::vector<PlannedOp> ops;
    int P, cls_channels, conv_impl;
    BranchExecutor ex;   // the GroupNorm statistics region is its clear region
    // lfd_plan_forward_extent, allocated on its first call: the device geometry table (one lfd_extent per op), its pinned staging ring
    lfd_extent* ext_dev = nullptr;
    lfd_extent* ext_host = nullptr;      // [kExtentRing][ops]
    cudaEvent_t ext_ev[kExtentRing] = {};
    int ext_slot = 0;
    ~lfd_plan() {
        for (auto ev : ext_ev)
            if (ev) cudaEventDestroy(ev);
        if (ext_dev) cudaFree(ext_dev);
        if (ext_host) cudaFreeHost(ext_host);
    }
};

extern "C" int lfd_plan_create(const lfd_op* ops, int n_ops, int N, int P, int cls_channels, int64_t stats_off, int64_t stats_bytes,
                               int64_t workspace_bytes, int conv_impl, lfd_plan** out) {
    if (!ops || n_ops <= 0 || !out) return fail(LFD_ERR_INVALID, "lfd_plan_create: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_plan_create: no CUDA device (there is no CPU fallback)");
    lfd_plan* pl = new lfd_plan();
    pl->P = P; pl->cls_channels = cls_channels; pl->conv_impl = conv_impl;
    pl->ex.clear_off = stats_off; pl->ex.clear_bytes = stats_bytes;
    pl->ops.resize(n_ops);
    int rc = LFD_OK;
    for (int i = 0; i < n_ops && !rc; ++i) rc = plan_op(ops[i], &pl->ops[i]);
    if (!rc) rc = pl->ex.init("lfd_plan_create", n_ops, [&](int i) { return ops[i].branch; }, [&](int i) { return ops[i].wait_mask; }, kMaxInferenceGraphs);
    if (rc) { delete pl; return rc; }
    *out = pl;
    return LFD_OK;
}

extern "C" int lfd_plan_destroy(lfd_plan* plan) {
    delete plan;
    return LFD_OK;
}

extern "C" int lfd_plan_num_launches(const lfd_plan* plan) { return plan ? (int)plan->ops.size() : 0; }

// The input format of an inference entry point, before anything is enqueued: 0, 1 or 2.  An NV12 frame (h x w) has an even height and
// width, on an image op whose capacity (H x W: the UV plane's pitch and twice its rows) is even too.
static int check_input_format(const char* fn, int fmt, const lfd_op* img, int h, int w) {
    if (fmt != LFD_INPUT_F32_NCHW && fmt != LFD_INPUT_U8_NHWC && fmt != LFD_INPUT_U8_NV12)
        return fail(LFD_ERR_INVALID, "%s: input format %d (0 = float32 NCHW, 1 = uint8 NHWC, 2 = uint8 NV12)", fn, fmt);
    if (fmt == LFD_INPUT_U8_NV12 && img) {
        if ((img->H | img->W) & 1) return fail(LFD_ERR_UNSUPPORTED, "%s: NV12 frames need an even capacity, the plan's is %dx%d", fn, img->H, img->W);
        if ((h | w) & 1) return fail(LFD_ERR_INVALID, "%s: an NV12 frame has an even height and width, got %dx%d", fn, h, w);
    }
    return LFD_OK;
}

// the op that reads the image (a plan's first op), or null
static const lfd_op* image_op(const lfd_plan* pl) {
    const lfd_op& o = pl->ops[0].op;
    return o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4 ? &o : nullptr;
}

// Training reads float32 NCHW or uint8 NHWC only
static int check_train_format(const char* fn, int fmt) {
    if (fmt == LFD_INPUT_U8_NV12) return fail(LFD_ERR_UNSUPPORTED, "%s: NV12 input is for inference plans only", fn);
    if (fmt != LFD_INPUT_F32_NCHW && fmt != LFD_INPUT_U8_NHWC)
        return fail(LFD_ERR_INVALID, "%s: input format %d (0 = float32 NCHW, 1 = uint8 NHWC)", fn, fmt);
    return LFD_OK;
}

extern "C" int lfd_plan_forward(lfd_plan* pl, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                                int use_graph, lfd_stream stream) {
    if (!pl || !input || !workspace || !cls_out || !reg_out) return fail(LFD_ERR_INVALID, "lfd_plan_forward: null argument");
    const lfd_op* img = image_op(pl);
    int rc = check_input_format("lfd_plan_forward", input_format, img, img ? img->H : 0, img ? img->W : 0);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    return pl->ex.run(input, input_format, workspace, cls_out, reg_out, nullptr, use_graph, st_of(stream), [&](size_t i, cudaStream_t s) {
        return launch_op(pl->ops[i], i, input, input_format, ws, cls_out, reg_out, pl->P, pl->cls_channels, pl->conv_impl, s);
    });
}

// A frame's table must describe the plan's own op list at no more than its capacity: every extent within the op's, the image op at h x w, and
// the head outputs inside the frame's P <= the plan's P
static int check_extent(const lfd_plan* pl, int h, int w, const lfd_extent* ext) {
    const int n = (int)pl->ops.size();
    int P = -1;
    for (int i = 0; i < n; ++i) {
        const lfd_op& o = pl->ops[i].op;
        const lfd_extent& e = ext[i];
        if (e.H < 1 || e.W < 1 || e.Ho < 1 || e.Wo < 1 || e.H > o.H || e.W > o.W || e.Ho > o.Ho || e.Wo > o.Wo)
            return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: op %d: extent %dx%d -> %dx%d outside the plan's %dx%d -> %dx%d", i, e.H, e.W, e.Ho,
                        e.Wo, o.H, o.W, o.Ho, o.Wo);
        if ((o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4) && (e.H != h || e.W != w))
            return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: the image op's extent %dx%d is not the frame's %dx%d", e.H, e.W, h, w);
        if (o.kind == LFD_OP_HEAD_FINAL) {
            if (P < 0) P = e.P;
            if (e.P != P || P > pl->P || e.point_off < 0 || (int64_t)e.point_off + (int64_t)e.H * e.W > P)
                return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: op %d: points [%d, %d + %d x %d) outside the frame's %d (plan: %d)", i, e.point_off,
                            e.point_off, e.H, e.W, e.P, pl->P);
        }
    }
    return LFD_OK;
}

extern "C" int lfd_plan_forward_extent(lfd_plan* pl, const void* input, int input_format, int h, int w, const lfd_extent* ext, void* workspace,
                                       float* cls_out, float* reg_out, int use_graph, lfd_stream stream) {
    if (!pl || !input || !workspace || !cls_out || !reg_out) return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: null argument");
    const lfd_op& img = pl->ops[0].op;
    if (img.kind != LFD_OP_STEM0 && img.kind != LFD_OP_STEM4) return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: the plan does not start on the image");
    if (h < 1 || w < 1 || h > img.H || w > img.W)
        return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: frame %dx%d outside the plan's capacity %dx%d", h, w, img.H, img.W);
    int rc = check_input_format("lfd_plan_forward_extent", input_format, &img, h, w);
    if (rc) return rc;
    if (h == img.H && w == img.W) return lfd_plan_forward(pl, input, input_format, workspace, cls_out, reg_out, use_graph, stream);
    if (pl->conv_impl == LFD_CONV_SIMT) return fail(LFD_ERR_UNSUPPORTED, "lfd_plan_forward_extent: the SIMT cross-check kernels run full-size frames only");
    if (!ext) return fail(LFD_ERR_INVALID, "lfd_plan_forward_extent: a frame below the capacity needs its geometry table");
    rc = check_extent(pl, h, w, ext);
    if (rc) return rc;
    const size_t n = pl->ops.size(), bytes = n * sizeof(lfd_extent);
    if (!pl->ext_ev[kExtentRing - 1]) {
        if (!pl->ext_dev) CUDA_TRY(cudaMalloc(&pl->ext_dev, bytes));
        if (!pl->ext_host) CUDA_TRY(cudaHostAlloc(&pl->ext_host, kExtentRing * bytes, cudaHostAllocDefault));
        for (auto& ev : pl->ext_ev)
            if (!ev) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    }
    cudaStream_t st = st_of(stream);
    const int slot = pl->ext_slot;
    pl->ext_slot = (slot + 1) % kExtentRing;
    CUDA_TRY(cudaEventSynchronize(pl->ext_ev[slot]));   // the copy that last read this slot has been performed
    lfd_extent* host = pl->ext_host + slot * n;
    memcpy(host, ext, bytes);
    CUDA_TRY(cudaMemcpyAsync(pl->ext_dev, host, bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaEventRecord(pl->ext_ev[slot], st));
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    return pl->ex.run(input, input_format, workspace, cls_out, reg_out, pl->ext_dev, use_graph, st, [&](size_t i, cudaStream_t s) {
        return launch_op(pl->ops[i], i, input, input_format, ws, cls_out, reg_out, pl->P, pl->cls_channels, pl->conv_impl, s, pl->ext_dev + i);
    });
}

extern "C" int lfd_plan_num_graphs(const lfd_plan* plan) { return plan ? (int)plan->ex.graphs.size() : 0; }

extern "C" int lfd_plan_profile(lfd_plan* pl, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                                float* ms_per_op, lfd_stream stream) {
    if (!pl || !input || !workspace || !cls_out || !reg_out || !ms_per_op) return fail(LFD_ERR_INVALID, "lfd_plan_profile: null argument");
    const lfd_op* img = image_op(pl);
    int rc = check_input_format("lfd_plan_profile", input_format, img, img ? img->H : 0, img ? img->W : 0);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    return pl->ex.profile("lfd_plan_profile", ws, ms_per_op, st_of(stream), [&](size_t i, cudaStream_t s) {
        return launch_op(pl->ops[i], i, input, input_format, ws, cls_out, reg_out, pl->P, pl->cls_channels, pl->conv_impl, s);
    });
}


extern "C" int lfd_run_op(const lfd_op* op, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                          int P, int cls_channels, int conv_impl, lfd_stream stream) {
    if (!op || !workspace) return fail(LFD_ERR_INVALID, "lfd_run_op: null argument");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_run_op: no CUDA device (there is no CPU fallback)");
    PlannedOp po;
    int rc = plan_op(*op, &po);
    if (rc) return rc;
    const bool reads_image = op->kind == LFD_OP_STEM0 || op->kind == LFD_OP_STEM4;
    rc = check_input_format("lfd_run_op", input_format, reads_image ? op : nullptr, op->H, op->W);
    if (rc) return rc;
    return launch_op(po, 0, input, input_format, reinterpret_cast<uint8_t*>(workspace), cls_out, reg_out, P, cls_channels, conv_impl,
                     reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------------ post-process
static int pow2_at_least(int v) {
    int p = 1;
    while (p < v) p <<= 1;
    return p;
}
static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

struct PostLayout {
    size_t box, score, src, count, scratch, scratch_stride, total;
    int cap_pow2;
};
static PostLayout post_layout(int N, int cap) {
    PostLayout L;
    L.cap_pow2 = pow2_at_least(cap);
    size_t o = 0;
    L.box = o; o = align256(o + (size_t)N * cap * 16);
    L.score = o; o = align256(o + (size_t)N * cap * 4);
    L.src = o; o = align256(o + (size_t)N * cap * 4);
    L.count = o; o = align256(o + (size_t)N * 4);
    L.scratch_stride = nms_scratch_stride(cap, L.cap_pow2);
    L.scratch = o; o = align256(o + (size_t)N * L.scratch_stride);
    L.total = o;
    return L;
}

extern "C" size_t lfd_postprocess_workspace_bytes(const lfd_post_cfg* cfg) {
    if (!cfg || cfg->N <= 0 || cfg->cap <= 0) return 0;
    return post_layout(cfg->N, cfg->cap).total;
}

// soft == nullptr: greedy NMS (lfd_postprocess); else Soft-NMS with soft->method / sigma / min_score (lfd_postprocess_soft_nms)
static int postprocess_impl(const char* fn, const lfd_post_cfg* c, const float* cls, const float* reg, const float* img_w, const float* img_h,
                            const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                            int32_t* overflow, const SoftNmsParams* soft, lfd_stream stream) {
    if (!c || !cls || !reg || !img_w || !img_h || !resize_scale || !workspace || !dets || !labels || !src || !count || !overflow)
        return fail(LFD_ERR_INVALID, "%s: null argument", fn);
    if (c->num_levels < 1 || c->num_levels > LFD_MAX_LEVELS || c->C < 1 || c->cap < 1) return fail(LFD_ERR_INVALID, "%s: bad config", fn);
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "%s: no CUDA device (there is no CPU fallback)", fn);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const PostLayout L = post_layout(c->N, c->cap);
    PostParams p;
    p.cls = cls; p.reg = reg; p.img_w = img_w; p.img_h = img_h; p.resize_scale = resize_scale;
    p.N = c->N; p.P = c->P; p.C = c->C; p.cls_stride = c->cls_channels; p.cls_mode = c->cls_mode; p.bbox_mode = c->bbox_mode;
    p.num_levels = c->num_levels; p.cap = c->cap;
    for (int l = 0; l < LFD_MAX_LEVELS; ++l) {
        p.level_off[l] = c->level_off[l]; p.level_w[l] = c->level_w[l]; p.level_stride[l] = c->level_stride[l]; p.level_hi[l] = c->level_hi[l];
    }
    p.score_thr = c->score_thr;
    p.cand_box = reinterpret_cast<float*>(ws + L.box); p.cand_score = reinterpret_cast<float*>(ws + L.score);
    p.cand_src = reinterpret_cast<int*>(ws + L.src); p.cand_count = reinterpret_cast<int*>(ws + L.count);
    CUDA_TRY(cudaMemsetAsync(p.cand_count, 0, (size_t)c->N * 4, st));
    CUDA_TRY(cudaMemsetAsync(overflow, 0, 4, st));
    CUDA_TRY(candidates_launch(p, c->max_ctas > 0 ? c->max_ctas : sm_count(), st));
    NmsParams q;
    q.cand_box = p.cand_box; q.cand_score = p.cand_score; q.cand_src = p.cand_src; q.cand_count = p.cand_count;
    q.scratch = ws + L.scratch; q.scratch_stride = L.scratch_stride; q.cap = c->cap; q.cap_pow2 = L.cap_pow2; q.C = c->C;
    q.class_agnostic = c->class_agnostic; q.iou_thr = c->iou_thr;
    q.out_dets = dets; q.out_label = labels; q.out_src = src; q.out_count = count; q.overflow = overflow;
    if (soft) {
        SoftNmsParams sq = *soft;
        sq.nms = q;
        CUDA_TRY(soft_nms_launch(sq, c->N, st));
    } else {
        CUDA_TRY(nms_launch(q, c->N, st));
    }
    return LFD_OK;
}

extern "C" int lfd_postprocess(const lfd_post_cfg* c, const float* cls, const float* reg, const float* img_w, const float* img_h,
                               const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                               int32_t* overflow, lfd_stream stream) {
    return postprocess_impl("lfd_postprocess", c, cls, reg, img_w, img_h, resize_scale, workspace, dets, labels, src, count, overflow, nullptr, stream);
}

// the reference's soft_nms method codes (nms.py:101); method 0 of soft_nms_cpu (hard suppression) is not reachable from its Python
static int soft_params(const char* fn, int method, float sigma, float min_score, SoftNmsParams* out) {
    if (method != 1 && method != 2) return fail(LFD_ERR_INVALID, "%s: method must be 1 (linear) or 2 (gaussian)", fn);
    out->method = method; out->sigma = sigma; out->min_score = min_score;
    return LFD_OK;
}

extern "C" size_t lfd_postprocess_soft_nms_workspace_bytes(const lfd_post_cfg* cfg) { return lfd_postprocess_workspace_bytes(cfg); }

extern "C" int lfd_postprocess_soft_nms(const lfd_post_cfg* c, const float* cls, const float* reg, const float* img_w, const float* img_h,
                                        const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                                        int32_t* overflow, int method, float sigma, float min_score, lfd_stream stream) {
    SoftNmsParams sq;
    const int rc = soft_params("lfd_postprocess_soft_nms", method, sigma, min_score, &sq);
    if (rc) return rc;
    return postprocess_impl("lfd_postprocess_soft_nms", c, cls, reg, img_w, img_h, resize_scale, workspace, dets, labels, src, count, overflow, &sq,
                            stream);
}

// multiclass_nms / batched_nms on explicit boxes (lfd/model/utils/nms.py:119-220): threshold + class-offset NMS, all on the device
extern "C" size_t lfd_multiclass_nms_workspace_bytes(int cap) { return cap > 0 ? post_layout(1, cap).total : 256; }

static int multiclass_impl(const char* fn, const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in,
                           int n, int C, float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels,
                           int32_t* src, int32_t* count, int32_t* overflow, const SoftNmsParams* soft, lfd_stream stream) {
    if (n < 0 || C < 1 || cap < 1 || !workspace || !dets || !labels || !src || !count || !overflow || (n > 0 && (!boxes || !scores)))
        return fail(LFD_ERR_INVALID, "%s: bad arguments", fn);
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "%s: no CUDA device (there is no CPU fallback)", fn);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const PostLayout L = post_layout(1, cap);
    float* cbox = reinterpret_cast<float*>(ws + L.box);
    float* cscore = reinterpret_cast<float*>(ws + L.score);
    int* csrc = reinterpret_cast<int*>(ws + L.src);
    int* ccount = reinterpret_cast<int*>(ws + L.count);
    CUDA_TRY(cudaMemsetAsync(ccount, 0, 4, st));
    CUDA_TRY(cudaMemsetAsync(overflow, 0, 4, st));
    CUDA_TRY(box_candidates_launch(boxes, box_per_class, scores, score_stride, labels_in, n, C, score_thr, cap, cbox, cscore, csrc, ccount, st));
    NmsParams q;
    q.cand_box = cbox; q.cand_score = cscore; q.cand_src = csrc; q.cand_count = ccount;
    q.scratch = ws + L.scratch; q.scratch_stride = L.scratch_stride; q.cap = cap; q.cap_pow2 = L.cap_pow2; q.C = C;
    q.class_agnostic = class_agnostic; q.iou_thr = iou_thr;
    q.out_dets = dets; q.out_label = labels; q.out_src = src; q.out_count = count; q.overflow = overflow;
    if (soft) {
        SoftNmsParams sq = *soft;
        sq.nms = q;
        CUDA_TRY(soft_nms_launch(sq, 1, st));
    } else {
        CUDA_TRY(nms_launch(q, 1, st));
    }
    return LFD_OK;
}

extern "C" int lfd_multiclass_nms(const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in, int n, int C,
                                  float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels, int32_t* src,
                                  int32_t* count, int32_t* overflow, lfd_stream stream) {
    return multiclass_impl("lfd_multiclass_nms", boxes, box_per_class, scores, score_stride, labels_in, n, C, score_thr, iou_thr, class_agnostic, cap,
                           workspace, dets, labels, src, count, overflow, nullptr, stream);
}

extern "C" size_t lfd_multiclass_soft_nms_workspace_bytes(int cap) { return lfd_multiclass_nms_workspace_bytes(cap); }

extern "C" int lfd_multiclass_soft_nms(const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in, int n,
                                       int C, float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels,
                                       int32_t* src, int32_t* count, int32_t* overflow, int method, float sigma, float min_score, lfd_stream stream) {
    SoftNmsParams sq;
    const int rc = soft_params("lfd_multiclass_soft_nms", method, sigma, min_score, &sq);
    if (rc) return rc;
    return multiclass_impl("lfd_multiclass_soft_nms", boxes, box_per_class, scores, score_stride, labels_in, n, C, score_thr, iou_thr, class_agnostic,
                           cap, workspace, dets, labels, src, count, overflow, &sq, stream);
}

// standalone NMS on raw dets (mirror of nms_ext.nms)
__global__ void nms_split_kernel(const float* dets, int n, float* box, float* score, int* src, int* count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *count = n;
    if (i >= n) return;
    reinterpret_cast<float4*>(box)[i] = make_float4(dets[i * 5], dets[i * 5 + 1], dets[i * 5 + 2], dets[i * 5 + 3]);
    score[i] = dets[i * 5 + 4];
    src[i] = i;
}
__global__ void nms_keep_kernel(const int* src, const int* count, long long* keep, int* n_keep) {
    const int k = *count;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < k; i += gridDim.x * blockDim.x) keep[i] = src[i];
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_keep = k;
}

struct RawNmsLayout {
    PostLayout base;
    size_t dets, label, src, count, overflow, total;
};
static RawNmsLayout raw_layout(int n) {
    RawNmsLayout R;
    R.base = post_layout(1, n);
    size_t o = R.base.total;
    R.dets = o; o = align256(o + (size_t)n * 20);
    R.label = o; o = align256(o + (size_t)n * 4);
    R.src = o; o = align256(o + (size_t)n * 4);
    R.count = o; o = align256(o + 4);
    R.overflow = o; o = align256(o + 4);
    R.total = o;
    return R;
}
extern "C" size_t lfd_nms_workspace_bytes(int n) { return n > 0 ? raw_layout(n).total : 256; }

extern "C" int lfd_nms(const float* dets, int n, float iou_thr, void* workspace, int64_t* keep, int32_t* n_keep, lfd_stream stream) {
    if (!n_keep || n < 0) return fail(LFD_ERR_INVALID, "lfd_nms: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_nms: no CUDA device (there is no CPU fallback)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (n == 0) {
        CUDA_TRY(cudaMemsetAsync(n_keep, 0, 4, st));
        return LFD_OK;
    }
    if (!dets || !workspace || !keep) return fail(LFD_ERR_INVALID, "lfd_nms: null argument");
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const RawNmsLayout R = raw_layout(n);
    NmsParams q;
    q.cand_box = reinterpret_cast<float*>(ws + R.base.box); q.cand_score = reinterpret_cast<float*>(ws + R.base.score);
    q.cand_src = reinterpret_cast<int*>(ws + R.base.src); q.cand_count = reinterpret_cast<int*>(ws + R.base.count);
    q.scratch = ws + R.base.scratch; q.scratch_stride = R.base.scratch_stride; q.cap = n; q.cap_pow2 = R.base.cap_pow2; q.C = 1;
    q.class_agnostic = 1; q.iou_thr = iou_thr;
    q.out_dets = reinterpret_cast<float*>(ws + R.dets); q.out_label = reinterpret_cast<int*>(ws + R.label);
    q.out_src = reinterpret_cast<int*>(ws + R.src); q.out_count = reinterpret_cast<int*>(ws + R.count);
    q.overflow = reinterpret_cast<int*>(ws + R.overflow);
    nms_split_kernel<<<(n + 255) / 256, 256, 0, st>>>(dets, n, const_cast<float*>(q.cand_box), const_cast<float*>(q.cand_score),
                                                      const_cast<int*>(q.cand_src), const_cast<int*>(q.cand_count));
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(nms_launch(q, 1, st));
    nms_keep_kernel<<<(n + 255) / 256, 256, 0, st>>>(q.out_src, q.out_count, reinterpret_cast<long long*>(keep), n_keep);
    CUDA_TRY(cudaGetLastError());
    return LFD_OK;
}

// ------------------------------------------------------------------------------------------------ losses
static void fill_levels(const lfd_levels* lv, LevelTable* t) {
    t->num_levels = lv->num_levels;
    for (int l = 0; l < kMaxLevels; ++l) {
        t->off[l] = lv->off[l]; t->w[l] = lv->w[l]; t->stride[l] = lv->stride[l];
        t->lo[l] = lv->lo[l]; t->hi[l] = lv->hi[l]; t->glo[l] = lv->glo[l]; t->ghi[l] = lv->ghi[l];
    }
}

extern "C" int lfd_assign_targets(const lfd_levels* lv, int N, int P, int C, int gmax, int assign_mode, int independent,
                                  const float* gt_boxes, const int32_t* gt_labels, const int32_t* gt_count, float* cls_target,
                                  float* reg_target, int32_t* label, int32_t* counters, lfd_stream stream) {
    if (!lv || !gt_count || !cls_target || !reg_target || !label || !counters || (gmax > 0 && (!gt_boxes || !gt_labels)))
        return fail(LFD_ERR_INVALID, "lfd_assign_targets: null argument");
    if (lv->num_levels < 1 || lv->num_levels > LFD_MAX_LEVELS || N < 1 || P < 1 || C < 1) return fail(LFD_ERR_INVALID, "lfd_assign_targets: bad shape");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_assign_targets: no CUDA device (there is no CPU fallback)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    AssignParams p;
    fill_levels(lv, &p.lv);
    p.gt_boxes = gt_boxes; p.gt_labels = gt_labels; p.gt_count = gt_count;
    p.N = N; p.P = P; p.C = C; p.gmax = gmax; p.assign_mode = assign_mode; p.independent = independent;
    p.cls_target = cls_target; p.reg_target = reg_target; p.label = label; p.counters = counters;
    CUDA_TRY(cudaMemsetAsync(counters, 0, 8, st));
    CUDA_TRY(assign_targets_launch(p, st));
    return LFD_OK;
}

static int detection_loss(const char* fn, const lfd_levels* lv, const lfd_loss_cfg* c, const float* cls_logits, const float* reg,
                          const float* cls_target, const float* reg_target, const int32_t* label, const int32_t* counters, float* grad_cls,
                          float* grad_reg, double* loss_sums, int cls_weighted, int reg_weighted, const double* weight_sum, lfd_stream stream) {
    if (!lv || !c || !cls_logits || !reg || !reg_target || !label || !counters || !loss_sums) return fail(LFD_ERR_INVALID, "%s: null argument", fn);
    if (c->cls_mode < LFD_CLS_SIGMOID || c->cls_mode > LFD_CLS_QFL) return fail(LFD_ERR_INVALID, "%s: unknown classification loss %d", fn, c->cls_mode);
    if ((c->cls_mode == LFD_CLS_BCE || c->cls_mode == LFD_CLS_QFL) && !cls_target) return fail(LFD_ERR_INVALID, "%s: BCE / QFL need the soft classification targets", fn);
    if (c->reg_loss < LFD_REG_IOU || c->reg_loss > LFD_REG_MSE) return fail(LFD_ERR_INVALID, "%s: unknown regression loss %d", fn, c->reg_loss);
    const bool indep = c->reg_loss == LFD_REG_SMOOTH_L1 || c->reg_loss == LFD_REG_MSE;
    if (indep != (c->bbox_mode == LFD_BBOX_INDEPENDENT)) return fail(LFD_ERR_INVALID, "%s: SmoothL1 / MSE go with the 'independent' targets, the IoU family with sigmoid / exp", fn);
    if (c->reg_loss == LFD_REG_SMOOTH_L1 && !(c->smooth_l1_beta > 0.f)) return fail(LFD_ERR_INVALID, "%s: SmoothL1 beta must be > 0", fn);
    if ((cls_weighted != 0 && cls_weighted != 1) || (reg_weighted != 0 && reg_weighted != 1))
        return fail(LFD_ERR_INVALID, "%s: cls_weighted / reg_weighted must be 0 or 1 (got %d, %d)", fn, cls_weighted, reg_weighted);
    if ((cls_weighted || reg_weighted) && !weight_sum) return fail(LFD_ERR_INVALID, "%s: weighting needs weight_sum (lfd_loss_weight_sum)", fn);
    if (reg_weighted && !cls_target) return fail(LFD_ERR_INVALID, "%s: regression weighting reads the weights from cls_target", fn);
    if (reg_weighted && indep)
        return fail(LFD_ERR_INVALID, "%s: regression weighting with SmoothL1 / MSE: the reference multiplies the (n, 4) element loss by the (n,) "
                                     "weight, which does not broadcast", fn);
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "%s: no CUDA device (there is no CPU fallback)", fn);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int sms = c->max_ctas > 0 ? c->max_ctas : sm_count();
    CUDA_TRY(cudaMemsetAsync(loss_sums, 0, 16, st));
    ClsLossParams k;
    k.logits = cls_logits; k.cls_target = cls_target; k.label = label; k.counters = counters; k.grad = grad_cls; k.loss_sum = loss_sums;
    k.N = c->N; k.P = c->P; k.C = c->C; k.cls_mode = c->cls_mode; k.gamma = c->gamma; k.alpha = c->alpha; k.loss_weight = c->cls_weight;
    k.weighted = cls_weighted; k.weight_sum = weight_sum;
    CUDA_TRY(cls_loss_launch(k, sms, st));
    RegLossParams r;
    fill_levels(lv, &r.lv);
    r.reg = reg; r.reg_target = reg_target; r.label = label; r.counters = counters; r.grad = grad_reg; r.loss_sum = loss_sums + 1;
    r.N = c->N; r.P = c->P; r.C = c->C; r.bbox_mode = c->bbox_mode; r.loss_kind = c->reg_loss; r.eps = c->reg_eps; r.loss_weight = c->reg_weight;
    r.beta = c->smooth_l1_beta;
    r.weighted = reg_weighted; r.weight_sum = weight_sum; r.cls_target = cls_target;
    CUDA_TRY(iou_loss_launch(r, sms, st));
    return LFD_OK;
}

extern "C" int lfd_detection_loss(const lfd_levels* lv, const lfd_loss_cfg* c, const float* cls_logits, const float* reg, const float* cls_target,
                                  const float* reg_target, const int32_t* label, const int32_t* counters, float* grad_cls, float* grad_reg,
                                  double* loss_sums, lfd_stream stream) {
    return detection_loss("lfd_detection_loss", lv, c, cls_logits, reg, cls_target, reg_target, label, counters, grad_cls, grad_reg, loss_sums,
                          0, 0, nullptr, stream);
}

extern "C" int lfd_detection_loss_weighted(const lfd_levels* lv, const lfd_loss_cfg* c, const float* cls_logits, const float* reg,
                                           const float* cls_target, const float* reg_target, const int32_t* label, const int32_t* counters,
                                           float* grad_cls, float* grad_reg, double* loss_sums, int cls_weighted, int reg_weighted,
                                           const double* weight_sum, lfd_stream stream) {
    return detection_loss("lfd_detection_loss_weighted", lv, c, cls_logits, reg, cls_target, reg_target, label, counters, grad_cls, grad_reg,
                          loss_sums, cls_weighted, reg_weighted, weight_sum, stream);
}

extern "C" size_t lfd_loss_weight_sum_workspace_bytes(const lfd_loss_cfg* c) {
    if (!c) { fail(LFD_ERR_INVALID, "lfd_loss_weight_sum_workspace_bytes: null argument"); return 0; }
    const int sms = c->max_ctas > 0 ? c->max_ctas : sm_count();
    if (sms <= 0) { fail(LFD_ERR_CUDA, "lfd_loss_weight_sum_workspace_bytes: no CUDA device"); return 0; }
    return (size_t)loss_weight_blocks(sms) * sizeof(double);
}

extern "C" int lfd_loss_weight_sum(const lfd_loss_cfg* c, const float* cls_target, const int32_t* label, void* workspace, double* weight_sum,
                                   lfd_stream stream) {
    if (!c || !cls_target || !label || !workspace || !weight_sum) return fail(LFD_ERR_INVALID, "lfd_loss_weight_sum: null argument");
    if (c->N < 1 || c->P < 1 || c->C < 1) return fail(LFD_ERR_INVALID, "lfd_loss_weight_sum: bad shape");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_loss_weight_sum: no CUDA device (there is no CPU fallback)");
    const int sms = c->max_ctas > 0 ? c->max_ctas : sm_count();
    CUDA_TRY(loss_weight_sum_launch(cls_target, label, (size_t)c->N * c->P, c->C, sms, reinterpret_cast<double*>(workspace), weight_sum,
                                    reinterpret_cast<cudaStream_t>(stream)));
    return LFD_OK;
}

extern "C" int lfd_box_loss(int kind, const float* pred, const float* target, int n, float eps, float* loss, float* grad_pred, lfd_stream stream) {
    if (kind < LFD_REG_IOU || kind > LFD_REG_CIOU || n < 0 || (n > 0 && (!pred || !target || !loss))) return fail(LFD_ERR_INVALID, "lfd_box_loss: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_box_loss: no CUDA device (there is no CPU fallback)");
    CUDA_TRY(box_loss_launch(kind, pred, target, n, eps, loss, grad_pred, reinterpret_cast<cudaStream_t>(stream)));
    return LFD_OK;
}

extern "C" int lfd_sigmoid_focal_loss_forward(const float* logits, const int64_t* targets, int M, int C, float gamma, float alpha,
                                              float* losses, lfd_stream stream) {
    if (M < 0 || C < 1 || (M > 0 && (!logits || !targets || !losses))) return fail(LFD_ERR_INVALID, "lfd_sigmoid_focal_loss_forward: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "sigmoid focal loss: no CUDA device (the reference has no CPU path either, sigmoid_focal_loss_ext.cpp:32)");
    CUDA_TRY(focal_forward_launch(logits, reinterpret_cast<const long long*>(targets), M, C, gamma, alpha, losses, reinterpret_cast<cudaStream_t>(stream)));
    return LFD_OK;
}
extern "C" int lfd_sigmoid_focal_loss_backward(const float* logits, const int64_t* targets, const float* d_losses, int M, int C,
                                               float gamma, float alpha, float* d_logits, lfd_stream stream) {
    if (M < 0 || C < 1 || (M > 0 && (!logits || !targets || !d_losses || !d_logits))) return fail(LFD_ERR_INVALID, "lfd_sigmoid_focal_loss_backward: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "sigmoid focal loss: no CUDA device");
    CUDA_TRY(focal_backward_launch(logits, reinterpret_cast<const long long*>(targets), d_losses, M, C, gamma, alpha, d_logits, reinterpret_cast<cudaStream_t>(stream)));
    return LFD_OK;
}

// ------------------------------------------------------------------------------------------------ training plan
struct PlannedTop {
    lfd_top op;
    PlannedOp conv;   // STEM0 / CONV: the wgmma configuration (same kernels as the inference plan)
};

struct lfd_train_plan {
    std::vector<PlannedTop> ops;
    BranchExecutor ex;
};

static lfd_op conv_op_of(const lfd_top& t) {
    lfd_op o;
    memset(&o, 0, sizeof(o));
    o.kind = t.kind == LFD_TOP_STEM0 ? LFD_OP_STEM0 : LFD_OP_CONV;
    o.N = t.N; o.H = t.H; o.W = t.W; o.Cin = t.Cin; o.Ho = t.Ho; o.Wo = t.Wo; o.Cout = t.Cout;
    o.ksize = t.ksize; o.stride = t.stride; o.relu = t.relu; o.gn_groups = t.groups; o.cc = t.cc;
    o.in_off = t.off[0]; o.out_off = t.off[1]; o.res_off = t.off[2]; o.stats_off = t.off[3];
    o.ds_out_off = -1;
    o.dtype = LFD_DTYPE_BF16;
    o.max_ctas = t.max_ctas;
    o.in_swap_rb = t.in_swap_rb;
    memcpy(o.in_mean, t.in_mean, sizeof(o.in_mean));
    memcpy(o.in_scale, t.in_scale, sizeof(o.in_scale));
    return o;
}

static int plan_top(const lfd_top& t, int64_t ws_bytes, PlannedTop* out) {
    out->op = t;
    for (int i = 0; i < 8; ++i)
        if (t.off[i] >= ws_bytes && !(t.kind == LFD_TOP_ZERO && i == 1)) return fail(LFD_ERR_INVALID, "training op kind %d: off[%d] = %lld outside the workspace", t.kind, i, (long long)t.off[i]);
    switch (t.kind) {
        case LFD_TOP_STEM0:
        case LFD_TOP_CONV: {
            if (t.off[1] < 0 || t.off[4] < 0 || (t.kind == LFD_TOP_CONV && t.off[0] < 0)) return fail(LFD_ERR_INVALID, "training conv: missing in / out / packed-weight offset");
            lfd_op o = conv_op_of(t);
            o.weight = reinterpret_cast<const void*>(1);   // placeholder: resolved against the workspace at launch
            return plan_op(o, &out->conv);
        }
        case LFD_TOP_INFER: {
            if (!t.ptr[0]) return fail(LFD_ERR_INVALID, "infer: missing op descriptor");
            lfd_op o = *reinterpret_cast<const lfd_op*>(t.ptr[0]);
            if (o.kind != LFD_OP_STEM0 && o.kind != LFD_OP_CONV && o.kind != LFD_OP_STEM4)
                return fail(LFD_ERR_UNSUPPORTED, "infer: op kind %d (STEM0 / CONV / STEM4 only)", o.kind);
            if (o.dtype != LFD_DTYPE_BF16 || o.gn_groups) return fail(LFD_ERR_UNSUPPORTED, "infer: bf16 ops without GroupNorm statistics only");
            if (t.off[1] < 0 || (o.kind == LFD_OP_CONV && t.off[0] < 0)) return fail(LFD_ERR_INVALID, "infer: missing in / out offset");
            o.in_off = t.off[0]; o.out_off = t.off[1]; o.res_off = t.off[2]; o.ds_out_off = t.off[3]; o.stats_off = -1;
            o.branch = 0; o.wait_mask = 0; o.max_ctas = t.max_ctas;
            return plan_op(o, &out->conv);
        }
        case LFD_TOP_WGRAD: {
            WgradGeom g = {t.N, t.H, t.W, t.Cin, t.Ho, t.Wo, t.Cout, t.ksize, t.stride};
            if (t.impl == LFD_WGRAD_UMMA && !wgrad_umma_supported(g))
                return fail(LFD_ERR_UNSUPPORTED, "wgrad %dx%d s%d Cin=%d Cout=%d unsupported by the wgmma kernel", t.ksize, t.ksize, t.stride, t.Cin, t.Cout);
            break;
        }
        case LFD_TOP_PACK: case LFD_TOP_UNPACK:
            if (!t.ptr[0] || t.n_desc < 0 || t.max_n < 0) return fail(LFD_ERR_INVALID, "pack / unpack: missing table");
            break;
        case LFD_TOP_BN_STATS: case LFD_TOP_BN_APPLY: case LFD_TOP_GN_APPLY: case LFD_TOP_HEAD_FINAL: case LFD_TOP_HEAD_FINAL_BWD:
        case LFD_TOP_NORM_BWD_REDUCE: case LFD_TOP_NORM_BWD_APPLY: case LFD_TOP_ZERO:
            break;
        case LFD_TOP_WGRAD_STEM:
            if (t.Cin != 3 && t.Cin != 1) return fail(LFD_ERR_UNSUPPORTED, "wgrad_stem: 3 (BGR) or 1 (gray) input channels (got Cin=%d)", t.Cin);
            return input_transform_of(t.Cin, t.in_swap_rb, t.in_mean, t.in_scale, &out->conv.xf);
        default:
            return fail(LFD_ERR_INVALID, "unknown training op kind %d", t.kind);
    }
    return LFD_OK;
}

template <typename T>
static T* at(uint8_t* ws, int64_t off) { return off >= 0 ? reinterpret_cast<T*>(ws + off) : nullptr; }

static int launch_top(const PlannedTop& pt, const void* input, int fmt, uint8_t* ws, cudaStream_t st) {
    const lfd_top& t = pt.op;
    const int sms = bounded_sms(t.max_ctas);   // the SIMT ops size their grids from it; CONV reads max_ctas itself (conv_op_of)
    switch (t.kind) {
        case LFD_TOP_PACK:
            CUDA_TRY(pack_launch(reinterpret_cast<const PackDesc*>(t.ptr[0]), t.n_desc, t.max_n, st));
            break;
        case LFD_TOP_UNPACK:
            CUDA_TRY(unpack_launch(reinterpret_cast<const UnpackDesc*>(t.ptr[0]), t.n_desc, t.max_n, st));
            break;
        case LFD_TOP_ZERO:
            CUDA_TRY(cudaMemsetAsync(ws + t.off[0], 0, (size_t)t.off[1], st));
            break;
        case LFD_TOP_STEM0:
        case LFD_TOP_CONV: {
            PlannedOp po = pt.conv;
            po.op.weight = ws + t.off[4];
            return launch_op(po, 0, input, fmt, ws, nullptr, nullptr, 0, 0, t.impl, st);
        }
        case LFD_TOP_INFER:
            return launch_op(pt.conv, 0, input, fmt, ws, nullptr, nullptr, 0, 0, LFD_CONV_UMMA, st);
        case LFD_TOP_BN_STATS: {
            BnStatsParams p;
            p.z = at<const __nv_bfloat16>(ws, t.off[0]); p.sums = at<double>(ws, t.off[3]);
            p.M = (long long)t.N * t.H * t.W; p.C = t.Cout;
            CUDA_TRY(bn_stats_launch(p, sms, st));
            break;
        }
        case LFD_TOP_BN_APPLY: {
            BnApplyParams p;
            p.z = at<const __nv_bfloat16>(ws, t.off[0]); p.y = at<__nv_bfloat16>(ws, t.off[1]); p.res = at<const __nv_bfloat16>(ws, t.off[2]);
            p.sums = at<const double>(ws, t.off[3]);
            p.gamma = reinterpret_cast<const float*>(t.ptr[0]); p.beta = reinterpret_cast<const float*>(t.ptr[1]);
            p.running_mean = reinterpret_cast<float*>(const_cast<void*>(t.ptr[2])); p.running_var = reinterpret_cast<float*>(const_cast<void*>(t.ptr[3]));
            p.M = (long long)t.N * t.H * t.W; p.C = t.Cout; p.relu = t.relu; p.eps = t.eps; p.momentum = t.momentum; p.frozen = t.frozen;
            if (!p.gamma || !p.beta || (t.frozen && (!p.running_mean || !p.running_var))) return fail(LFD_ERR_INVALID, "bn_apply: gamma / beta / running statistics missing");
            CUDA_TRY(bn_apply_launch(p, sms, st));
            break;
        }
        case LFD_TOP_GN_APPLY: {
            GnApplyParams p;
            p.in = at<const __nv_bfloat16>(ws, t.off[0]); p.out = at<__nv_bfloat16>(ws, t.off[1]); p.stats = at<const double>(ws, t.off[3]);
            p.gamma = reinterpret_cast<const float*>(t.ptr[0]); p.beta = reinterpret_cast<const float*>(t.ptr[1]);
            p.N = t.N; p.HW = t.H * t.W; p.C = t.Cout; p.groups = t.groups; p.eps = t.eps; p.f16 = 0; p.tl = nullptr;
            CUDA_TRY(gn_apply_launch(p, sms, st));
            break;
        }
        case LFD_TOP_HEAD_FINAL: {
            HeadFinalParams p;
            const int no = t.n_cls + t.n_reg;
            const float* stg = at<const float>(ws, t.off[4]);
            p.in = at<const __nv_bfloat16>(ws, t.off[0]); p.stats = at<const double>(ws, t.off[3]);
            p.gamma = reinterpret_cast<const float*>(t.ptr[0]); p.beta = reinterpret_cast<const float*>(t.ptr[1]);
            p.w = stg; p.scale = stg + (size_t)no * t.Cout; p.shift = p.scale + no;
            p.cls = t.n_cls ? reinterpret_cast<float*>(const_cast<void*>(t.ptr[2])) : nullptr;
            p.reg = t.n_reg ? reinterpret_cast<float*>(const_cast<void*>(t.ptr[3])) : nullptr;
            p.N = t.N; p.HW = t.H * t.W; p.C = t.Cout; p.groups = t.groups; p.n_out = no; p.n_cls = t.n_cls;
            p.P = t.P; p.point_off = t.point_off; p.cls_stride = t.cls_stride; p.eps = t.eps; p.f16 = 0; p.tl = nullptr;
            if ((t.n_cls && !p.cls) || (t.n_reg && !p.reg)) return fail(LFD_ERR_INVALID, "head_final: output pointers missing");
            CUDA_TRY(head_final_launch(p, sms, st));
            break;
        }
        case LFD_TOP_HEAD_FINAL_BWD: {
            HeadFinalBwdParams p;
            p.raw = at<const __nv_bfloat16>(ws, t.off[0]); p.dact = at<__nv_bfloat16>(ws, t.off[1]); p.stats = at<const double>(ws, t.off[3]);
            p.w = at<const float>(ws, t.off[4]); p.dstage = at<float>(ws, t.off[5]); p.dscale = at<float>(ws, t.off[6]);
            p.gamma = reinterpret_cast<const float*>(t.ptr[0]); p.beta = reinterpret_cast<const float*>(t.ptr[1]);
            p.gcls = reinterpret_cast<const float*>(t.ptr[2]); p.greg = reinterpret_cast<const float*>(t.ptr[3]);
            p.N = t.N; p.HW = t.H * t.W; p.C = t.Cout; p.groups = t.groups; p.n_out = t.n_cls + t.n_reg; p.n_cls = t.n_cls;
            p.P = t.P; p.point_off = t.point_off; p.cls_stride = t.cls_stride; p.eps = t.eps;
            if ((t.n_cls && !p.gcls) || (t.n_reg && !p.greg) || !p.dact || !p.dstage) return fail(LFD_ERR_INVALID, "head_final_bwd: missing pointer");
            CUDA_TRY(head_final_bwd_launch(p, sms, st));
            break;
        }
        case LFD_TOP_NORM_BWD_REDUCE:
        case LFD_TOP_NORM_BWD_APPLY: {
            NormBwdParams p;
            p.dy = at<const __nv_bfloat16>(ws, t.off[0]); p.y = at<const __nv_bfloat16>(ws, t.off[1]); p.z = at<const __nv_bfloat16>(ws, t.off[2]);
            p.fsums = at<const double>(ws, t.off[3]); p.bsums = at<double>(ws, t.off[4]);
            p.dz = at<__nv_bfloat16>(ws, t.off[5]); p.dz_up = at<__nv_bfloat16>(ws, t.off[6]); p.dres = at<__nv_bfloat16>(ws, t.off[7]);
            p.gamma = reinterpret_cast<const float*>(t.ptr[0]); p.beta = reinterpret_cast<const float*>(t.ptr[1]);
            p.dgamma = reinterpret_cast<float*>(const_cast<void*>(t.ptr[2])); p.dbeta = reinterpret_cast<float*>(const_cast<void*>(t.ptr[3]));
            p.N = t.N; p.H = t.H; p.W = t.W; p.C = t.Cout; p.groups = t.groups; p.relu = t.relu; p.upH = t.upH; p.upW = t.upW;
            p.dres_accumulate = t.accumulate; p.eps = t.eps; p.frozen = t.frozen;
            p.running_mean = reinterpret_cast<const float*>(t.ptr[4]); p.running_var = reinterpret_cast<const float*>(t.ptr[5]);
            if (t.frozen && (t.groups || !p.running_mean || !p.running_var)) return fail(LFD_ERR_INVALID, "norm backward: frozen BatchNorm needs its running statistics");
            if (!p.dy || !p.z || (!p.fsums && !t.frozen) || !p.bsums || !p.gamma || (t.groups && !p.beta) || (!t.groups && t.relu && !p.y))
                return fail(LFD_ERR_INVALID, "norm backward: missing tensor");
            if (t.kind == LFD_TOP_NORM_BWD_REDUCE) CUDA_TRY(norm_bwd_reduce_launch(p, sms, st));
            else {
                if (!p.dz) return fail(LFD_ERR_INVALID, "norm backward apply: dz missing");
                CUDA_TRY(norm_bwd_apply_launch(p, sms, st));
            }
            break;
        }
        case LFD_TOP_WGRAD: {
            WgradGeom g = {t.N, t.H, t.W, t.Cin, t.Ho, t.Wo, t.Cout, t.ksize, t.stride};
            const __nv_bfloat16* x = at<const __nv_bfloat16>(ws, t.off[0]);
            const __nv_bfloat16* dz = at<const __nv_bfloat16>(ws, t.off[1]);
            float* ds = at<float>(ws, t.off[5]);
            if (!x || !dz || !ds) return fail(LFD_ERR_INVALID, "wgrad: missing tensor");
            if (t.impl == LFD_WGRAD_SIMT) CUDA_TRY(wgrad_simt_launch(g, x, dz, ds, st));
            else CUDA_TRY(wgrad_umma_launch(g, x, dz, ds, sms, st));
            break;
        }
        case LFD_TOP_WGRAD_STEM: {
            WgradGeom g = {t.N, t.H, t.W, t.Cin, t.Ho, t.Wo, t.Cout, t.ksize, t.stride};
            if (!input || t.off[1] < 0 || t.off[5] < 0) return fail(LFD_ERR_INVALID, "wgrad_stem: missing tensor");
            const ImageIn img = image_in(input, fmt, t.Cin, t.H, t.W, pt.conv.xf);
            if (t.off[0] >= 0 && t.impl == LFD_WGRAD_UMMA) {
                // tensor-core path: im2col into the scratch tensor X27 [N][Ho][Wo][32] at off[0], then the 1x1 wgrad (32 -> Cout) over it;
                // the staging at off[5] must hold 32 rows of Cout floats (rows 27..31 stay zero)
                __nv_bfloat16* x27 = at<__nv_bfloat16>(ws, t.off[0]);
                CUDA_TRY(stem_im2col_launch(g, img, x27, sms, st));
                WgradGeom g1 = {t.N, t.Ho, t.Wo, 32, t.Ho, t.Wo, t.Cout, 1, 1};
                CUDA_TRY(wgrad_umma_launch(g1, x27, at<const __nv_bfloat16>(ws, t.off[1]), at<float>(ws, t.off[5]), sms, st));
            } else {
                CUDA_TRY(wgrad_stem_launch(g, img, at<const __nv_bfloat16>(ws, t.off[1]), at<float>(ws, t.off[5]), sms, st));
            }
            break;
        }
        default:
            return fail(LFD_ERR_INVALID, "unknown training op kind %d", t.kind);
    }
    return LFD_OK;
}

extern "C" int lfd_train_plan_create(const lfd_top* ops, int n_ops, int64_t workspace_bytes, lfd_train_plan** out) {
    if (!ops || n_ops <= 0 || !out || workspace_bytes <= 0) return fail(LFD_ERR_INVALID, "lfd_train_plan_create: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_train_plan_create: no CUDA device (there is no CPU fallback)");
    lfd_train_plan* pl = new lfd_train_plan();
    pl->ops.resize(n_ops);
    int rc = LFD_OK;
    for (int i = 0; i < n_ops && !rc; ++i) rc = plan_top(ops[i], workspace_bytes, &pl->ops[i]);
    if (!rc) rc = pl->ex.init("lfd_train_plan_create", n_ops, [&](int i) { return ops[i].branch; }, [&](int i) { return ops[i].wait_mask; }, kMaxTrainingGraphs);
    if (rc) { delete pl; return rc; }
    *out = pl;
    return LFD_OK;
}

extern "C" int lfd_train_plan_destroy(lfd_train_plan* plan) {
    delete plan;
    return LFD_OK;
}

extern "C" int lfd_train_plan_num_ops(const lfd_train_plan* plan) { return plan ? (int)plan->ops.size() : 0; }

extern "C" int lfd_train_plan_run(lfd_train_plan* pl, const void* input, int input_format, void* workspace, int use_graph, lfd_stream stream) {
    if (!pl || !workspace) return fail(LFD_ERR_INVALID, "lfd_train_plan_run: null argument");
    int rc = check_train_format("lfd_train_plan_run", input_format);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    return pl->ex.run(input, input_format, workspace, nullptr, nullptr, nullptr, use_graph, st_of(stream), [&](size_t i, cudaStream_t s) {
        return launch_top(pl->ops[i], input, input_format, ws, s);
    });
}

extern "C" int lfd_train_plan_profile(lfd_train_plan* pl, const void* input, int input_format, void* workspace, float* ms_per_op, lfd_stream stream) {
    if (!pl || !workspace || !ms_per_op) return fail(LFD_ERR_INVALID, "lfd_train_plan_profile: null argument");
    int rc = check_train_format("lfd_train_plan_profile", input_format);
    if (rc) return rc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    return pl->ex.profile("lfd_train_plan_profile", ws, ms_per_op, st_of(stream), [&](size_t i, cudaStream_t s) {
        return launch_top(pl->ops[i], input, input_format, ws, s);
    });
}

extern "C" int lfd_run_top(const lfd_top* op, const void* input, int input_format, void* workspace, lfd_stream stream) {
    if (!op || !workspace) return fail(LFD_ERR_INVALID, "lfd_run_top: null argument");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_run_top: no CUDA device (there is no CPU fallback)");
    PlannedTop pt;
    int rc = plan_top(*op, INT64_MAX, &pt);
    if (rc) return rc;
    rc = check_train_format("lfd_run_top", input_format);
    if (rc) return rc;
    return launch_top(pt, input, input_format, reinterpret_cast<uint8_t*>(workspace), reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int lfd_grad_sqnorm(const float* grads, int64_t n, double* sqnorm, lfd_stream stream) {
    if (!grads || !sqnorm || n <= 0) return fail(LFD_ERR_INVALID, "lfd_grad_sqnorm: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_grad_sqnorm: no CUDA device (there is no CPU fallback)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaMemsetAsync(sqnorm, 0, 8, st));
    CUDA_TRY(sqnorm_launch(grads, n, sqnorm, sm_count(), st));
    return LFD_OK;
}

extern "C" int lfd_sgd_step(float* params, float* grads, float* momentum_buf, int64_t n, float lr, float momentum, float dampening,
                            float weight_decay, int nesterov, float max_norm, float grad_scale, const double* sqnorm, lfd_stream stream) {
    if (!params || !grads || n <= 0 || (max_norm > 0.f && !sqnorm)) return fail(LFD_ERR_INVALID, "lfd_sgd_step: bad arguments");
    if (nesterov && (momentum <= 0.f || dampening != 0.f || !momentum_buf)) return fail(LFD_ERR_INVALID, "lfd_sgd_step: nesterov needs momentum > 0 and zero dampening");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_sgd_step: no CUDA device (there is no CPU fallback)");
    SgdParams p;
    p.p = params; p.g = grads; p.m = (momentum != 0.f) ? momentum_buf : nullptr; p.n = n;
    p.lr = lr; p.momentum = momentum; p.dampening = dampening; p.weight_decay = weight_decay; p.nesterov = nesterov;
    p.max_norm = max_norm; p.sqnorm = sqnorm; p.grad_scale = grad_scale;
    if (momentum != 0.f && !momentum_buf) return fail(LFD_ERR_INVALID, "lfd_sgd_step: momentum buffer missing");
    CUDA_TRY(sgd_launch(p, sm_count(), st_of(stream)));
    return LFD_OK;
}

extern "C" int lfd_input_batch(const lfd_input_desc* descs, int n, const uint8_t* src, void* out, int out_mode, int swap_rb, int H, int W,
                               const float* mean, const float* scale, lfd_stream stream) {
    if (n < 0 || H < 1 || W < 1 || (n > 0 && (!descs || !src || !out))) return fail(LFD_ERR_INVALID, "lfd_input_batch: bad arguments (n=%d H=%d W=%d)", n, H, W);
    if (out_mode < LFD_INPUT_OUT_U8_NHWC || out_mode > LFD_INPUT_OUT_F32_GRAY) return fail(LFD_ERR_INVALID, "lfd_input_batch: out_mode %d", out_mode);
    const bool gray = out_mode == LFD_INPUT_OUT_U8_GRAY || out_mode == LFD_INPUT_OUT_F32_GRAY;
    if ((out_mode == LFD_INPUT_OUT_F32_NCHW || out_mode == LFD_INPUT_OUT_F32_GRAY) && (!mean || !scale))
        return fail(LFD_ERR_INVALID, "lfd_input_batch: the fp32 modes need mean and scale");
    if (gray && swap_rb) return fail(LFD_ERR_INVALID, "lfd_input_batch: swap_rb=%d with the gray out_mode %d (one channel has no channel order)", swap_rb, out_mode);
    if (W > 6144) return fail(LFD_ERR_UNSUPPORTED, "lfd_input_batch: W=%d > 6144 (the column table lives in 48 KB of shared memory)", W);
    if (n > 65535) return fail(LFD_ERR_UNSUPPORTED, "lfd_input_batch: n=%d > 65535", n);
    if (n == 0) return LFD_OK;
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_input_batch: no CUDA device (there is no CPU fallback)");
    CUDA_TRY(input_batch_launch(descs, n, src, out, out_mode, swap_rb, H, W, mean, scale, st_of(stream)));
    return LFD_OK;
}

// ------------------------------------------------------------------------------------------------ model files (lfd_engine_*)
// The layout is documented in include/lfd_b200.h and DESIGN.md "Model files"; lfd/_engine.py InferencePlan.export is the writer.
static constexpr size_t kModelHeaderBytes = 48, kModelPlanBytes = 120;
static constexpr int kModelMaxOps = 4096, kModelMaxN = 1024, kModelMaxSide = 16384, kModelMaxChannels = 4096, kModelMaxCap = 1 << 20;
static constexpr int64_t kModelMaxWorkspace = (int64_t)1 << 40, kModelMaxBlob = (int64_t)1 << 34;
static constexpr uint64_t kBlobOffsetMask = ((uint64_t)1 << 56) - 1;

struct lfd_engine {
    int32_t N = 0, H = 0, W = 0, P = 0, cls_channels = 0, dtype = 0, conv_impl = 0;
    int64_t stats_off = 0, stats_bytes = 0, ws_bytes = 0;
    int32_t soft = 0, soft_method = 0;
    float soft_sigma = 0.f, soft_min_score = 0.f;
    int32_t in_swap_rb = 0;                   // the plan's input transform, which op 0 carries
    float in_mean[3] = {0.f, 0.f, 0.f}, in_scale[3] = {0.f, 0.f, 0.f};
    lfd_post_cfg post{};
    std::vector<lfd_op> ops;                  // as stored: pointer fields in the (blob, offset) encoding
    std::vector<int32_t> src, level;
    std::vector<uint8_t> blob[2];
    // lfd_engine_bind
    lfd_plan* plan = nullptr;
    uint8_t *weights = nullptr, *ws = nullptr, *post_ws = nullptr;
    std::vector<lfd_extent> ext;              // the geometry table of the last frame below the capacity
    int meta_h = 0, meta_w = 0;               // the frame size the post-process workspace holds (0: none yet), written on meta_stream
    cudaStream_t meta_stream = nullptr;
    ~lfd_engine() { lfd_plan_destroy(plan); }
};

static size_t blob1_base(const lfd_engine* e) { return align256(e->blob[0].size()); }
static size_t engine_weights_bytes(const lfd_engine* e) { return blob1_base(e) + align256(e->blob[1].size()); }
// forward workspace: the plan's, then the engine's own cls and reg outputs
static size_t engine_cls_off(const lfd_engine* e) { return align256((size_t)e->ws_bytes); }
static size_t engine_reg_off(const lfd_engine* e) { return engine_cls_off(e) + align256((size_t)e->N * e->P * e->cls_channels * 4); }
static size_t engine_ws_bytes(const lfd_engine* e) { return engine_reg_off(e) + align256((size_t)e->N * e->P * 16); }
// post-process workspace: lfd_postprocess's, then img_w / img_h / resize_scale float[N] each, then src int32[N][cap]
static size_t engine_meta_off(const lfd_engine* e) { return align256(post_layout(e->N, e->post.cap).total); }
static size_t engine_src_off(const lfd_engine* e) { return engine_meta_off(e) + align256((size_t)e->N * 12); }
static size_t engine_post_bytes(const lfd_engine* e) { return engine_src_off(e) + align256((size_t)e->N * e->post.cap * 4); }

// CRC-32 (IEEE 802.3, reflected 0xEDB88320: zlib.crc32)
struct Crc32Table {
    uint32_t t[256];
    Crc32Table() {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            t[i] = c;
        }
    }
};
static uint32_t crc32_of(const uint8_t* p, size_t n) {
    static const Crc32Table tab;   // initialised once, thread-safe (a function-local static)
    const uint32_t* table = tab.t;
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

template <typename T> static T rd(const uint8_t* p) {
    T v;
    memcpy(&v, p, sizeof(T));
    return v;
}

static int bad_file(const char* fmt, ...) {
    char msg[400];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, sizeof(msg), fmt, ap);
    va_end(ap);
    return fail(LFD_ERR_INVALID, "lfd_engine_open: %s", msg);
}

static bool in_range(int64_t v, int64_t lo, int64_t hi) { return v >= lo && v <= hi; }

// a workspace range [off, off + bytes): off = -1 only where the op does not use it
static int check_ws(int i, const char* field, int64_t off, int64_t bytes, bool used, int64_t ws_bytes) {
    if (!used) return off == -1 ? LFD_OK : bad_file("op %d: %s = %lld on an op that does not use it (expected -1)", i, field, (long long)off);
    if (off < 0 || off % 16 || bytes > ws_bytes || off > ws_bytes - bytes)
        return bad_file("op %d: %s = %lld (+ %lld bytes) outside the workspace of workspace_bytes = %lld", i, field, (long long)off, (long long)bytes,
                        (long long)ws_bytes);
    return LFD_OK;
}

// a pointer field: 0 = NULL, else ((blob + 1) << 56) | offset, in the blob of its type, aligned to its element, with `bytes` inside the blob
static int check_ptr(const lfd_engine* e, int i, const char* field, const void* p, int blob, int64_t bytes, bool used, bool required) {
    const uint64_t v = (uint64_t)(uintptr_t)p;
    if (v == 0) return used && required ? bad_file("op %d: %s is missing", i, field) : LFD_OK;
    if (!used) return bad_file("op %d: %s is set on an op that does not read it", i, field);
    const uint64_t tag = v >> 56, off = v & kBlobOffsetMask;
    if (tag != (uint64_t)blob + 1) return bad_file("op %d: %s refers to blob %lld, expected blob %d", i, field, (long long)tag - 1, blob);
    const uint64_t size = e->blob[blob].size(), align = blob == 0 ? 4 : 16;
    if (off % align || (uint64_t)bytes > size || off > size - (uint64_t)bytes)
        return bad_file("op %d: %s = blob %d offset %llu (+ %lld bytes) outside the blob of %llu bytes", i, field, blob, (unsigned long long)off,
                        (long long)bytes, (unsigned long long)size);
    return LFD_OK;
}

static int check_model_op(const lfd_engine* e, int i) {
    const lfd_op& o = e->ops[i];
    if (o.kind < LFD_OP_STEM0 || o.kind > LFD_OP_STEM4) return bad_file("op %d: unknown op kind %d", i, o.kind);
    const bool image = o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4;
    if (image != (i == 0)) return bad_file("op %d: kind %d, but the image op (STEM0 / STEM4) is op 0 and only op 0", i, o.kind);
    if (o.N != e->N) return bad_file("op %d: N = %d, the plan's is %d", i, o.N, e->N);
    if (o.dtype != e->dtype) return bad_file("op %d: dtype %d, the plan's is %d", i, o.dtype, e->dtype);
    // the image op reads the caller's frames: its geometry is the capacity lfd_engine_info reports and lfd_engine_detect checks against
    if (image && (o.H != e->H || o.W != e->W))
        return bad_file("op 0: the image op reads %dx%d frames, the plan's capacity H x W is %dx%d", o.H, o.W, e->H, e->W);
    // the input transform that runs is op 0's: it is the plan's, and no other op carries one
    const bool same_xf = image ? o.in_swap_rb == e->in_swap_rb && !memcmp(o.in_mean, e->in_mean, sizeof(o.in_mean)) &&
                                     !memcmp(o.in_scale, e->in_scale, sizeof(o.in_scale))
                               : o.in_swap_rb == 0 && !memcmp(o.in_mean, "\0\0\0\0\0\0\0\0\0\0\0\0", 12) &&
                                     !memcmp(o.in_scale, "\0\0\0\0\0\0\0\0\0\0\0\0", 12);
    if (!same_xf) return bad_file("op %d: input transform (in_swap_rb / in_mean / in_scale) %s", i, image ? "differs from the plan's" : "set on an op that does not read the image");
    if (image) {
        InputTransform xf;
        if (o.Cin != 3 && o.Cin != 1) return bad_file("op 0: an image of %d channels (3: BGR, 1: gray)", o.Cin);
        if (input_transform_of(o.Cin, o.in_swap_rb, o.in_mean, o.in_scale, &xf)) return bad_file("op 0: %s", g_err);
    }
    const int32_t dims[] = {o.H, o.W, o.Ho, o.Wo};
    for (int32_t d : dims)
        if (!in_range(d, 1, kModelMaxSide)) return bad_file("op %d: H / W / Ho / Wo = %d / %d / %d / %d outside [1, %d]", i, o.H, o.W, o.Ho, o.Wo, kModelMaxSide);
    const int32_t chans[] = {o.Cin, o.Cout, o.tail_cout, o.ds_cout, o.gn_groups, o.n_cls, o.n_reg, o.cc, o.ksize, o.stride};
    for (int32_t c : chans)
        if (!in_range(c, 0, kModelMaxChannels))
            return bad_file("op %d: a channel count, group count, ksize or stride is outside [0, %d] (Cin %d Cout %d)", i, kModelMaxChannels, o.Cin, o.Cout);
    if (o.branch < 0 || o.branch >= LFD_MAX_BRANCHES || o.wait_mask < 0 || o.wait_mask >= (1 << LFD_MAX_BRANCHES))
        return bad_file("op %d: branch %d / wait_mask 0x%x out of range", i, o.branch, o.wait_mask);
    if (o.max_ctas < 0) return bad_file("op %d: max_ctas = %d", i, o.max_ctas);
    if (o.point_off < 0) return bad_file("op %d: point_off = %d", i, o.point_off);
    const int64_t N = o.N, in_px = N * o.H * o.W, out_px = N * o.Ho * o.Wo;
    const int64_t cf = o.tail_cout ? o.tail_cout : o.Cout, stats = N * o.gn_groups * 16, wsb = e->ws_bytes;
    const bool conv = o.kind == LFD_OP_CONV, gn = o.kind == LFD_OP_GN_APPLY, head = o.kind == LFD_OP_HEAD_FINAL;
    int rc = LFD_OK;
    if (!rc) rc = check_ws(i, "in_off", o.in_off, in_px * o.Cin * 2, conv || gn || head, wsb);
    if (!rc) rc = check_ws(i, "out_off", o.out_off, (gn ? in_px * o.Cin : out_px * cf) * 2, !head, wsb);
    if (!rc) rc = check_ws(i, "res_off", o.res_off, out_px * cf * 2, conv && o.res_off != -1, wsb);
    if (!rc) rc = check_ws(i, "stats_off", o.stats_off, stats, o.gn_groups > 0, wsb);
    if (!rc) rc = check_ws(i, "ds_out_off", o.ds_out_off, out_px * o.ds_cout * 2, o.ds_cout > 0, wsb);
    const bool stem4 = o.kind == LFD_OP_STEM4, conv_like = conv || o.kind == LFD_OP_STEM0 || stem4;
    const int64_t k2 = (int64_t)o.ksize * o.ksize, n_out = o.n_cls + o.n_reg;
    const int64_t w_bytes = conv ? o.Cin * k2 * o.Cout * 2 : conv_like ? 96 * (int64_t)o.Cout : head ? n_out * o.Cin * 4 : 0;
    if (!rc) rc = check_ptr(e, i, "weight", o.weight, head ? 0 : 1, w_bytes, conv_like || head, true);
    if (!rc) rc = check_ptr(e, i, "scale", o.scale, 0, n_out * 4, head, true);
    if (!rc) rc = check_ptr(e, i, "shift", o.shift, 0, (head ? n_out : o.Cout) * 4, conv_like || head, head);
    if (!rc) rc = check_ptr(e, i, "gamma", o.gamma, 0, o.Cin * 4, gn || (head && o.gn_groups), true);
    if (!rc) rc = check_ptr(e, i, "beta", o.beta, 0, o.Cin * 4, gn || (head && o.gn_groups), true);
    if (!rc) rc = check_ptr(e, i, "tail_weight", o.tail_weight, 1, (int64_t)o.Cout * o.tail_cout * 2, conv_like && o.tail_cout, true);
    if (!rc) rc = check_ptr(e, i, "tail_scale", o.tail_scale, 0, 0, false, false);
    if (!rc) rc = check_ptr(e, i, "tail_shift", o.tail_shift, 0, (int64_t)o.tail_cout * 4, conv_like && o.tail_cout, false);
    if (!rc) rc = check_ptr(e, i, "ds_weight", o.ds_weight, 1, (int64_t)o.Cin * o.ds_cout * 2, conv && o.ds_cout, true);
    if (!rc) rc = check_ptr(e, i, "ds_shift", o.ds_shift, 0, (int64_t)o.ds_cout * 4, conv && o.ds_cout, false);
    if (!rc) rc = check_ptr(e, i, "s2_weight", o.s2_weight, 1, 9 * 64 * 64 * 2, stem4, true);
    if (!rc) rc = check_ptr(e, i, "s2_shift", o.s2_shift, 0, 64 * 4, stem4, false);
    if (!rc) rc = check_ptr(e, i, "s3_weight", o.s3_weight, 1, 64 * 64 * 2, stem4, true);
    if (!rc) rc = check_ptr(e, i, "s3_shift", o.s3_shift, 0, 64 * 4, stem4, false);
    if (rc) return rc;
    if (conv && ((o.ksize != 1 && o.ksize != 3) || (o.stride != 1 && o.stride != 2)))
        return bad_file("op %d: conv ksize %d / stride %d (1 or 3 / 1 or 2)", i, o.ksize, o.stride);
    if (check_op(o)) {   // the same geometry rules lfd_plan_create applies
        char msg[sizeof(g_err)];
        snprintf(msg, sizeof(msg), "%s", g_err);
        return bad_file("op %d: %s", i, msg);
    }
    if (conv_like) {   // the wgmma kernel's configuration, as lfd_plan_create derives it (host only)
        UmmaConvParams cp;
        size_t smem = 0;
        int grid = 0;
        if (umma_conv_configure(geom_of(o), 132, &cp, &smem, &grid))
            return bad_file("op %d: conv %dx%d s%d Cin=%d Cout=%d tail_cout=%d ds_cout=%d is not supported by the wgmma kernel", i, o.ksize, o.ksize,
                            o.stride, o.Cin, o.Cout, o.tail_cout, o.ds_cout);
        if (conv && cp.Cc != o.cc) return bad_file("op %d: cc = %d, the wgmma kernel packs this conv with cc = %d", i, o.cc, cp.Cc);
    }
    if (head && o.n_reg != 0 && o.n_reg != 4) return bad_file("op %d: n_reg = %d (0 or 4)", i, o.n_reg);
    if (head && o.n_cls + o.n_reg == 0) return bad_file("op %d: a head op without outputs (n_cls = n_reg = 0)", i);
    // the producer / level table: what lfd_engine_detect derives a smaller frame's geometry from
    const int32_t s = e->src[i], l = e->level[i];
    if (image ? s != -1 : (s < 0 || s >= i)) return bad_file("op %d: src_op = %d (the image op has -1, every other op an earlier op)", i, s);
    if (!image) {   // the op reads one of its producer's outputs, of its size and channel count
        const lfd_op& p = e->ops[s];
        if (p.Ho != o.H || p.Wo != o.W) return bad_file("op %d: src_op = %d makes %dx%d, this op reads %dx%d", i, s, p.Ho, p.Wo, o.H, o.W);
        const int32_t main_c = p.kind == LFD_OP_GN_APPLY ? p.Cin : (p.tail_cout ? p.tail_cout : p.Cout);
        const int32_t c = o.in_off == p.out_off ? main_c : (p.ds_cout && o.in_off == p.ds_out_off) ? p.ds_cout : -1;
        if (p.kind == LFD_OP_HEAD_FINAL || c < 0)
            return bad_file("op %d: in_off = %lld is not an output of src_op = %d", i, (long long)o.in_off, s);
        if (c != o.Cin) return bad_file("op %d: Cin = %d, but src_op = %d stores %d channels", i, o.Cin, s, c);
    }
    if (head ? !in_range(l, 0, e->post.num_levels - 1) : l != -1) return bad_file("op %d: level = %d (head ops: 0 .. num_levels - 1, others -1)", i, l);
    if (head && (o.point_off != e->post.level_off[l] || o.W != e->post.level_w[l]))
        return bad_file("op %d: head of level %d at point_off %d, width %d; the post-process has level_off %d, level_w %d", i, l, o.point_off, o.W,
                        e->post.level_off[l], e->post.level_w[l]);
    if (head && (int64_t)o.point_off + (int64_t)o.H * o.W > e->P) return bad_file("op %d: points [%d, %d + %dx%d) beyond P = %d", i, o.point_off, o.point_off, o.H, o.W, e->P);
    if (head && (o.n_cls > e->cls_channels || (o.n_cls && o.n_cls != e->cls_channels))) return bad_file("op %d: n_cls = %d, cls_channels = %d", i, o.n_cls, e->cls_channels);
    return LFD_OK;
}

static int parse_model(const uint8_t* b, size_t n, lfd_engine* e) {
    if (n < kModelHeaderBytes) return bad_file("the file has %zu bytes, less than the %zu-byte header", n, kModelHeaderBytes);
    if (memcmp(b, "LFDMODEL", 8)) return bad_file("magic: not an LFD model file");
    const uint32_t version = rd<uint32_t>(b + 8), abi = rd<uint32_t>(b + 12);
    if (version != LFD_MODEL_FORMAT_VERSION)
        return fail(LFD_ERR_UNSUPPORTED, "lfd_engine_open: format version %u, this library reads version %d", version, LFD_MODEL_FORMAT_VERSION);
    if (abi != LFD_B200_ABI_VERSION) return fail(LFD_ERR_UNSUPPORTED, "lfd_engine_open: abi version %u, this library is version %d", abi, LFD_B200_ABI_VERSION);
    if (memcmp(b + 16, "sm_90a\0\0", 8)) return fail(LFD_ERR_UNSUPPORTED, "lfd_engine_open: target \"%.8s\", this library runs sm_90a", (const char*)(b + 16));
    const uint32_t op_bytes = rd<uint32_t>(b + 24), post_bytes = rd<uint32_t>(b + 28);
    if (op_bytes != sizeof(lfd_op)) return bad_file("lfd_op struct bytes %u, this library's lfd_op has %zu", op_bytes, sizeof(lfd_op));
    if (post_bytes != sizeof(lfd_post_cfg)) return bad_file("lfd_post_cfg struct bytes %u, this library's lfd_post_cfg has %zu", post_bytes, sizeof(lfd_post_cfg));
    const uint64_t payload = rd<uint64_t>(b + 32);
    const uint32_t checksum = rd<uint32_t>(b + 40), reserved = rd<uint32_t>(b + 44);
    if (reserved) return bad_file("reserved header word = %u (expected 0)", reserved);
    if (payload != n - kModelHeaderBytes)
        return bad_file("payload_bytes = %llu, but the file holds %zu bytes after the header (truncated or trailing bytes)", (unsigned long long)payload,
                        n - kModelHeaderBytes);
    const uint8_t* p = b + kModelHeaderBytes;
    if (crc32_of(p, payload) != checksum) return bad_file("checksum: the payload's CRC-32 is 0x%08x, the header says 0x%08x", crc32_of(p, payload), checksum);
    if (payload < kModelPlanBytes + sizeof(lfd_post_cfg)) return bad_file("payload_bytes = %llu, too short for the plan section", (unsigned long long)payload);
    e->N = rd<int32_t>(p + 0); e->H = rd<int32_t>(p + 4); e->W = rd<int32_t>(p + 8); e->P = rd<int32_t>(p + 12);
    e->cls_channels = rd<int32_t>(p + 16); e->dtype = rd<int32_t>(p + 20); e->conv_impl = rd<int32_t>(p + 24);
    const int32_t n_ops = rd<int32_t>(p + 28);
    e->stats_off = rd<int64_t>(p + 32); e->stats_bytes = rd<int64_t>(p + 40); e->ws_bytes = rd<int64_t>(p + 48);
    const int32_t swap = rd<int32_t>(p + 56);
    float* mean = e->in_mean;
    float* scale = e->in_scale;
    e->in_swap_rb = swap;
    for (int c = 0; c < 3; ++c) { mean[c] = rd<float>(p + 60 + 4 * c); scale[c] = rd<float>(p + 72 + 4 * c); }
    if (rd<int32_t>(p + 100) != 0) return bad_file("reserved plan word at byte 100 = %d (expected 0)", rd<int32_t>(p + 100));
    e->soft = rd<int32_t>(p + 84); e->soft_method = rd<int32_t>(p + 88);
    e->soft_sigma = rd<float>(p + 92); e->soft_min_score = rd<float>(p + 96);
    const int64_t blob_bytes[2] = {rd<int64_t>(p + 104), rd<int64_t>(p + 112)};
    memcpy(&e->post, p + kModelPlanBytes, sizeof(lfd_post_cfg));
    if (n_ops < 1 || n_ops > kModelMaxOps) return bad_file("n_ops = %d outside [1, %d]", n_ops, kModelMaxOps);
    if (!in_range(e->N, 1, kModelMaxN) || !in_range(e->H, 1, kModelMaxSide) || !in_range(e->W, 1, kModelMaxSide))
        return bad_file("capacity N x H x W = %d x %d x %d outside [1, %d] x [1, %d] x [1, %d]", e->N, e->H, e->W, kModelMaxN, kModelMaxSide, kModelMaxSide);
    if (!in_range(e->P, 1, (int64_t)e->H * e->W) || !in_range(e->cls_channels, 1, kModelMaxChannels))
        return bad_file("P = %d / cls_channels = %d out of range", e->P, e->cls_channels);
    if (e->dtype != LFD_DTYPE_BF16 && e->dtype != LFD_DTYPE_FP16) return bad_file("dtype = %d", e->dtype);
    if (e->conv_impl != LFD_CONV_UMMA) return fail(LFD_ERR_UNSUPPORTED, "lfd_engine_open: conv_impl = %d, model files hold wgmma (LFD_CONV_UMMA) plans", e->conv_impl);
    if (!in_range(e->ws_bytes, 256, kModelMaxWorkspace)) return bad_file("workspace_bytes = %lld outside [256, 2^40]", (long long)e->ws_bytes);
    if (e->stats_off < 0 || e->stats_bytes < 0 || e->stats_bytes > e->ws_bytes || e->stats_off > e->ws_bytes - e->stats_bytes)
        return bad_file("stats_off / stats_bytes = %lld / %lld outside the workspace", (long long)e->stats_off, (long long)e->stats_bytes);
    InputTransform xf;
    if (input_transform_of(3, swap, mean, scale, &xf)) return bad_file("input transform: %s", g_err);   // op 0 checks it for its own image kind
    if (e->soft != 0 && e->soft != 1) return bad_file("nms_type = %d (0 greedy, 1 soft_nms)", e->soft);
    if (e->soft && ((e->soft_method != LFD_SOFT_NMS_LINEAR && e->soft_method != LFD_SOFT_NMS_GAUSSIAN) || !std::isfinite(e->soft_sigma) ||
                    !std::isfinite(e->soft_min_score)))
        return bad_file("soft_nms method %d / sigma %g / min_score %g", e->soft_method, (double)e->soft_sigma, (double)e->soft_min_score);
    for (int b = 0; b < 2; ++b)
        if (!in_range(blob_bytes[b], 0, kModelMaxBlob) || blob_bytes[b] % 16) return bad_file("blob %d bytes = %lld", b, (long long)blob_bytes[b]);
    const lfd_post_cfg& c = e->post;
    if (c.N != e->N || c.P != e->P || c.cls_channels != e->cls_channels)
        return bad_file("post-process N / P / cls_channels = %d / %d / %d, the plan's are %d / %d / %d", c.N, c.P, c.cls_channels, e->N, e->P, e->cls_channels);
    if (!in_range(c.C, 1, c.cls_channels) || (c.cls_mode == LFD_CLS_SIGMOID ? c.C != c.cls_channels : c.cls_mode == LFD_CLS_SOFTMAX ? c.C + 1 != c.cls_channels : true))
        return bad_file("post-process C = %d / cls_mode = %d do not fit cls_channels = %d", c.C, c.cls_mode, c.cls_channels);
    if (!in_range(c.bbox_mode, LFD_BBOX_SIGMOID, LFD_BBOX_INDEPENDENT) || (c.class_agnostic != 0 && c.class_agnostic != 1) || c.max_ctas != 0)
        return bad_file("post-process bbox_mode %d / class_agnostic %d / max_ctas %d", c.bbox_mode, c.class_agnostic, c.max_ctas);
    if (!in_range(c.num_levels, 1, LFD_MAX_LEVELS) || !in_range(c.cap, 1, kModelMaxCap)) return bad_file("post-process num_levels %d / cap %d", c.num_levels, c.cap);
    if (!std::isfinite(c.score_thr) || !std::isfinite(c.iou_thr)) return bad_file("post-process score_thr %g / iou_thr %g", (double)c.score_thr, (double)c.iou_thr);
    for (int l = 0; l < c.num_levels; ++l)
        if (!in_range(c.level_stride[l], 1, 1 << 16) || !std::isfinite(c.level_hi[l])) return bad_file("post-process level %d: stride %d", l, c.level_stride[l]);
    const size_t ops_at = kModelPlanBytes + sizeof(lfd_post_cfg), aux_at = ops_at + (size_t)n_ops * sizeof(lfd_op), blob_at = aux_at + (size_t)n_ops * 8;
    if (payload != blob_at + (uint64_t)blob_bytes[0] + (uint64_t)blob_bytes[1])
        return bad_file("payload_bytes = %llu, the sections need %llu (n_ops = %d, blob bytes %lld + %lld)", (unsigned long long)payload,
                        (unsigned long long)(blob_at + blob_bytes[0] + blob_bytes[1]), n_ops, (long long)blob_bytes[0], (long long)blob_bytes[1]);
    e->ops.resize(n_ops);
    memcpy(e->ops.data(), p + ops_at, (size_t)n_ops * sizeof(lfd_op));
    e->src.resize(n_ops);
    e->level.resize(n_ops);
    for (int i = 0; i < n_ops; ++i) { e->src[i] = rd<int32_t>(p + aux_at + 8 * i); e->level[i] = rd<int32_t>(p + aux_at + 8 * i + 4); }
    e->blob[0].assign(p + blob_at, p + blob_at + blob_bytes[0]);
    e->blob[1].assign(p + blob_at + blob_bytes[0], p + blob_at + blob_bytes[0] + blob_bytes[1]);
    int64_t points = 0;
    int heads = 0;
    for (int i = 0; i < n_ops; ++i) {
        const int rc = check_model_op(e, i);
        if (rc) return rc;
        if (e->ops[i].kind == LFD_OP_HEAD_FINAL && e->ops[i].n_reg) { points += (int64_t)e->ops[i].H * e->ops[i].W; ++heads; }
    }
    if (heads != c.num_levels || points != e->P) return bad_file("the head ops cover %d levels and %lld points, the plan has %d levels and P = %d", heads, (long long)points, c.num_levels, e->P);
    return LFD_OK;
}

extern "C" int lfd_engine_open(const void* bytes, size_t n, lfd_engine** out) {
    if (!bytes || !out) return fail(LFD_ERR_INVALID, "lfd_engine_open: null argument");
    lfd_engine* e = new lfd_engine();
    const int rc = parse_model(reinterpret_cast<const uint8_t*>(bytes), n, e);
    if (rc) { delete e; return rc; }
    *out = e;
    return LFD_OK;
}

extern "C" int lfd_engine_close(lfd_engine* engine) {
    delete engine;
    return LFD_OK;
}

extern "C" int lfd_engine_info(const lfd_engine* e, lfd_engine_desc* out) {
    if (!e || !out) return fail(LFD_ERR_INVALID, "lfd_engine_info: null argument");
    lfd_engine_desc d{};
    d.N = e->N; d.H = e->H; d.W = e->W; d.P = e->P; d.cls_channels = e->cls_channels; d.num_classes = e->post.C; d.dtype = e->dtype;
    d.n_ops = (int32_t)e->ops.size(); d.cap = e->post.cap; d.soft_nms = e->soft;
    d.weights_bytes = (int64_t)engine_weights_bytes(e);
    d.workspace_bytes = (int64_t)engine_ws_bytes(e);
    d.post_workspace_bytes = (int64_t)engine_post_bytes(e);
    *out = d;
    return LFD_OK;
}

extern "C" int lfd_engine_op(const lfd_engine* e, int i, lfd_op* op, int32_t* src_op, int32_t* level) {
    if (!e || !op || i < 0 || i >= (int)e->ops.size()) return fail(LFD_ERR_INVALID, "lfd_engine_op: bad arguments (op %d)", i);
    *op = e->ops[i];
    if (src_op) *src_op = e->src[i];
    if (level) *level = e->level[i];
    return LFD_OK;
}

extern "C" int lfd_engine_num_launches(const lfd_engine* e) { return e ? lfd_plan_num_launches(e->plan) : 0; }

extern "C" int lfd_engine_bind(lfd_engine* e, void* weights, size_t weights_bytes, void* workspace, size_t workspace_bytes, void* post_workspace,
                               size_t post_workspace_bytes, lfd_stream stream) {
    if (!e || !weights || !workspace || !post_workspace) return fail(LFD_ERR_INVALID, "lfd_engine_bind: null argument");
    if (weights_bytes < engine_weights_bytes(e) || workspace_bytes < engine_ws_bytes(e) || post_workspace_bytes < engine_post_bytes(e))
        return fail(LFD_ERR_CAPACITY, "lfd_engine_bind: buffers of %zu / %zu / %zu bytes, the model needs weights %zu, workspace %zu, post workspace %zu",
                    weights_bytes, workspace_bytes, post_workspace_bytes, engine_weights_bytes(e), engine_ws_bytes(e), engine_post_bytes(e));
    if (((uintptr_t)weights | (uintptr_t)workspace | (uintptr_t)post_workspace) & 255)
        return fail(LFD_ERR_INVALID, "lfd_engine_bind: weights %p / workspace %p / post workspace %p must be 256-byte aligned (as cudaMalloc returns)",
                    weights, workspace, post_workspace);
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_engine_bind: no CUDA device (there is no CPU fallback)");
    uint8_t* wb = reinterpret_cast<uint8_t*>(weights);
    const uint8_t* base[2] = {wb, wb + blob1_base(e)};
    std::vector<lfd_op> ops = e->ops;
    for (auto& o : ops) {
        const void** fields[] = {&o.weight, (const void**)&o.scale, (const void**)&o.shift, (const void**)&o.gamma, (const void**)&o.beta,
                                 &o.tail_weight, (const void**)&o.tail_scale, (const void**)&o.tail_shift, &o.ds_weight, (const void**)&o.ds_shift,
                                 &o.s2_weight, (const void**)&o.s2_shift, &o.s3_weight, (const void**)&o.s3_shift};
        for (const void** f : fields) {
            const uint64_t v = (uint64_t)(uintptr_t)*f;
            if (v) *f = base[(v >> 56) - 1] + (v & kBlobOffsetMask);
        }
    }
    lfd_plan* plan = nullptr;
    int rc = lfd_plan_create(ops.data(), (int)ops.size(), e->N, e->P, e->cls_channels, e->stats_off, e->stats_bytes, e->ws_bytes, e->conv_impl, &plan);
    if (rc) return rc;
    cudaStream_t st = st_of(stream);
    for (int b = 0; b < 2; ++b) {
        cudaError_t ce = e->blob[b].empty() ? cudaSuccess : cudaMemcpyAsync(const_cast<uint8_t*>(base[b]), e->blob[b].data(), e->blob[b].size(),
                                                                            cudaMemcpyHostToDevice, st);
        if (ce != cudaSuccess) { lfd_plan_destroy(plan); return fail(LFD_ERR_CUDA, "lfd_engine_bind: weight copy: %s", cudaGetErrorString(ce)); }
    }
    lfd_plan_destroy(e->plan);
    e->plan = plan;
    e->weights = wb;
    e->ws = reinterpret_cast<uint8_t*>(workspace);
    e->post_ws = reinterpret_cast<uint8_t*>(post_workspace);
    e->meta_h = e->meta_w = 0;
    return LFD_OK;
}

// cuMemsetD32Async: the post-process's per-image width / height / scale, as 32-bit patterns, without a host buffer
typedef int (*MemsetD32Fn)(unsigned long long, unsigned int, size_t, cudaStream_t);
static MemsetD32Fn memset_d32_fn() {
    static const MemsetD32Fn fn = []() -> MemsetD32Fn {   // looked up once, thread-safe (a function-local static)
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuMemsetD32Async", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            return reinterpret_cast<MemsetD32Fn>(ptr);
        return nullptr;
    }();
    return fn;
}

static int fill_f32(float* dst, float v, size_t n, cudaStream_t st) {
    MemsetD32Fn fn = memset_d32_fn();
    if (!fn) return fail(LFD_ERR_CUDA, "lfd_engine_detect: cuMemsetD32Async is not available");
    unsigned int bits;
    memcpy(&bits, &v, 4);
    if (fn((unsigned long long)(uintptr_t)dst, bits, n, st) != 0) return fail(LFD_ERR_CUDA, "lfd_engine_detect: cuMemsetD32Async failed");
    return LFD_OK;
}

extern "C" int lfd_engine_detect(lfd_engine* e, const void* input, int input_format, int h, int w, float* dets, int32_t* labels, int32_t* count,
                                 float* cls_out, float* reg_out, int use_graph, lfd_stream stream) {
    if (!e || !input || !dets || !labels || !count) return fail(LFD_ERR_INVALID, "lfd_engine_detect: null argument");
    if (!e->plan) return fail(LFD_ERR_INVALID, "lfd_engine_detect: the engine is not bound (lfd_engine_bind)");
    if (h < 1 || w < 1 || h > e->H || w > e->W) return fail(LFD_ERR_INVALID, "lfd_engine_detect: frame %dx%d outside the capacity %dx%d", h, w, e->H, e->W);
    int rc = check_input_format("lfd_engine_detect", input_format, &e->ops[0], h, w);
    if (rc) return rc;
    const int n_ops = (int)e->ops.size();
    // the frame's geometry: every op's extent follows from its producer's, as a plan built for h x w has it (lfd/_engine.py extent_table)
    e->ext.assign(n_ops, lfd_extent{});
    int level_h[LFD_MAX_LEVELS] = {0}, level_w[LFD_MAX_LEVELS] = {0};
    for (int i = 0; i < n_ops; ++i) {
        const lfd_op& o = e->ops[i];
        lfd_extent& x = e->ext[i];
        x.H = i == 0 ? h : e->ext[e->src[i]].Ho;
        x.W = i == 0 ? w : e->ext[e->src[i]].Wo;
        x.Ho = x.H; x.Wo = x.W;
        if (o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_CONV) {
            x.Ho = (x.H + 2 * (o.ksize / 2) - o.ksize) / o.stride + 1;
            x.Wo = (x.W + 2 * (o.ksize / 2) - o.ksize) / o.stride + 1;
        } else if (o.kind == LFD_OP_STEM4) {
            x.Ho = ((x.H - 1) / 2) / 2 + 1;
            x.Wo = ((x.W - 1) / 2) / 2 + 1;
        }
        if (o.kind == LFD_OP_HEAD_FINAL) { level_h[e->level[i]] = x.H; level_w[e->level[i]] = x.W; }
    }
    lfd_post_cfg cfg = e->post;
    int P = 0;
    for (int l = 0; l < cfg.num_levels; ++l) {
        cfg.level_off[l] = P;
        cfg.level_w[l] = level_w[l];
        P += level_h[l] * level_w[l];
    }
    cfg.P = P;
    for (int i = 0; i < n_ops; ++i)
        if (e->ops[i].kind == LFD_OP_HEAD_FINAL) { e->ext[i].point_off = cfg.level_off[e->level[i]]; e->ext[i].P = P; }
    float* cls = cls_out ? cls_out : reinterpret_cast<float*>(e->ws + engine_cls_off(e));
    float* reg = reg_out ? reg_out : reinterpret_cast<float*>(e->ws + engine_reg_off(e));
    cudaStream_t st = st_of(stream);
    rc = lfd_plan_forward_extent(e->plan, input, input_format, h, w, e->ext.data(), e->ws, cls, reg, use_graph, stream);
    if (rc) return rc;
    float* meta = reinterpret_cast<float*>(e->post_ws + engine_meta_off(e));
    const size_t N = (size_t)e->N;
    // written once per frame size and stream: the post-process workspace is the engine's alone, and a call on another stream writes it
    // again so that its post-process is ordered after the values it reads
    if (h != e->meta_h || w != e->meta_w || st != e->meta_stream) {
        e->meta_h = e->meta_w = 0;
        if ((rc = fill_f32(meta, (float)w, N, st)) || (rc = fill_f32(meta + N, (float)h, N, st)) || (rc = fill_f32(meta + 2 * N, 1.0f, N, st))) return rc;
        e->meta_h = h;
        e->meta_w = w;
        e->meta_stream = st;
    }
    int32_t* src = reinterpret_cast<int32_t*>(e->post_ws + engine_src_off(e));
    if (e->soft)
        return lfd_postprocess_soft_nms(&cfg, cls, reg, meta, meta + N, meta + 2 * N, e->post_ws, dets, labels, src, count, count + N, e->soft_method,
                                        e->soft_sigma, e->soft_min_score, stream);
    return lfd_postprocess(&cfg, cls, reg, meta, meta + N, meta + 2 * N, e->post_ws, dets, labels, src, count, count + N, stream);
}
