// api.cu -- the extern "C" boundary of liblfd_b200.so (declared in include/lfd_b200.h).
#include <stdarg.h>
#include <stdio.h>

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
};

struct lfd_plan {
    std::vector<PlannedOp> ops;
    int N, P, cls_channels, conv_impl;
    int64_t stats_off, stats_bytes, workspace_bytes;
    // CUDA graph cache: one instantiated graph per (input, workspace, cls, reg, format) pointer tuple
    struct GraphEntry {
        cudaGraphExec_t exec;
        const void* input;
        void* ws;
        float* cls;
        float* reg;
        int fmt;
    };
    std::vector<GraphEntry> graphs;
    // side streams for independent branches (the per-level neck + head chains)
    cudaStream_t side[LFD_MAX_BRANCHES];
    cudaEvent_t fork_ev[LFD_MAX_BRANCHES], join_ev[LFD_MAX_BRANCHES];
    std::vector<cudaEvent_t> dep_ev;   // one per (op, wait_mask bit): mid-graph cross-branch dependencies
    int n_branches;
};
static constexpr size_t kMaxGraphs = 32;

// Stream the CUDA graphs are captured on: the main chain (the backbone: the critical path of the step) runs two priority levels above
// the side streams of the per-level chains (created at the default = lowest level) -- captured kernel nodes inherit the level, so when
// SMs free up the pending CTAs of the critical path are placed first.  The levels above are left to the caller's latency-critical
// streams (lfd/pipeline.py runs the post-process of the previous batch there).  LFD_B200_GRAPH_PRIO=0 disables it (A/B runs).
static cudaError_t create_capture_stream(cudaStream_t* cap) {
    static const bool prio = !(getenv("LFD_B200_GRAPH_PRIO") && atoi(getenv("LFD_B200_GRAPH_PRIO")) == 0);
    int least = 0, greatest = 0;
    if (prio && cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess && greatest < least) {
        const int level = least - 2 < greatest ? greatest : least - 2;     // numerically lower = higher priority
        return cudaStreamCreateWithPriority(cap, cudaStreamNonBlocking, level);
    }
    return cudaStreamCreateWithFlags(cap, cudaStreamNonBlocking);
}


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

static int check_op(const lfd_op& o) {
    const int eh = (o.H + 2 * (o.ksize / 2) - o.ksize) / (o.stride > 0 ? o.stride : 1) + 1;
    const int ew = (o.W + 2 * (o.ksize / 2) - o.ksize) / (o.stride > 0 ? o.stride : 1) + 1;
    if (o.dtype != LFD_DTYPE_BF16 && o.dtype != LFD_DTYPE_FP16) return fail(LFD_ERR_INVALID, "op dtype %d: expected LFD_DTYPE_BF16 or LFD_DTYPE_FP16", o.dtype);
    switch (o.kind) {
        case LFD_OP_STEM0:
            if (o.scale || o.tail_scale) return fail(LFD_ERR_INVALID, "conv scale must be folded into the packed weights (pass scale = NULL)");
            if (o.Cin != 3 || o.ksize != 3 || o.stride != 2) return fail(LFD_ERR_UNSUPPORTED, "stem0 supports 3x3/s2 on 3 input channels only (got Cin=%d k=%d s=%d)", o.Cin, o.ksize, o.stride);
            if (o.Cout != 16 && o.Cout != 32 && o.Cout != 64) return fail(LFD_ERR_UNSUPPORTED, "stem0 Cout must be 16/32/64 (got %d)", o.Cout);
            if (o.Ho != eh || o.Wo != ew) return fail(LFD_ERR_INVALID, "stem0 output size mismatch");
            break;
        case LFD_OP_STEM4:
            if (o.scale || o.tail_scale) return fail(LFD_ERR_INVALID, "conv scale must be folded into the packed weights (pass scale = NULL)");
            if (o.Cin != 3 || o.ksize != 3 || o.stride != 2 || o.Cout != 64 || o.tail_cout != 64 || o.ds_cout || o.res_off >= 0 || o.gn_groups)
                return fail(LFD_ERR_UNSUPPORTED, "stem4 is 3x3/s2 3->64, 1x1 64->64, 3x3/s2 64->64, 1x1 64->64 without residual / statistics");
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

static int plan_op(const lfd_op& o, int conv_impl, PlannedOp* out) {
    int rc = check_op(o);
    if (rc) return rc;
    out->op = o;
    out->smem = 0;
    out->grid = 0;
    if (o.kind == LFD_OP_CONV || o.kind == LFD_OP_STEM0 || o.kind == LFD_OP_STEM4) {
        rc = umma_conv_configure(geom_of(o), sm_count() > 0 ? sm_count() : 132, &out->cp, &out->smem, &out->grid);
        if (rc) return fail(LFD_ERR_UNSUPPORTED, "conv %dx%d s%d Cin=%d Cout=%d unsupported (rc=%d)", o.ksize, o.ksize, o.stride, o.Cin, o.Cout, rc);
        if (o.kind == LFD_OP_CONV && out->cp.Cc != o.cc) return fail(LFD_ERR_INVALID, "weights packed with cc=%d but the kernel needs cc=%d", o.cc, out->cp.Cc);
        if (o.max_ctas < 0) return fail(LFD_ERR_INVALID, "max_ctas = %d", o.max_ctas);
        if (o.max_ctas > 0 && out->grid > o.max_ctas) out->grid = o.max_ctas;   // tiles are strided by gridDim (fused stem: contiguous runs): any grid size is valid
    }
    (void)conv_impl;
    return LFD_OK;
}

static int launch_op(const PlannedOp& po, size_t index, const void* input, int input_format, uint8_t* ws, float* cls, float* reg, int P,
                     int cls_channels, int conv_impl, cudaStream_t st) {
    const lfd_op& o = po.op;
    unsigned long long* tl = g_timeline ? g_timeline + 2 * index : nullptr;
    switch (o.kind) {
        case LFD_OP_STEM0: {
            if (!input) return fail(LFD_ERR_INVALID, "stem0 needs the external input pointer");
            if (conv_impl == LFD_CONV_SIMT) {
                if (o.tail_cout) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels do not implement fused tails");
                Stem0Params p;
                p.in = input; p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off);
                p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift;
                p.input_format = input_format; p.N = o.N; p.H = o.H; p.W = o.W; p.Ho = o.Ho; p.Wo = o.Wo; p.Cout = o.Cout; p.relu = o.relu; p.f16 = o.dtype;
                CUDA_TRY(stem0_launch(p, st));
            } else {
                UmmaConvParams p = po.cp;
                p.in_raw = input; p.input_format = input_format; p.in = nullptr;
                p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off); p.res = nullptr;
                p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift; p.stats = nullptr;
                p.relu = o.relu; p.gn_groups = 0; p.trace = g_trace; p.tl = tl; p.f16 = o.dtype;
                p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.tail_weight); p.shift2 = o.tail_shift; p.relu2 = o.tail_relu;
                if (umma_conv_encode_maps(&p)) return fail(LFD_ERR_CUDA, "cuTensorMapEncodeTiled failed for the stem conv");
                CUDA_TRY(umma_conv_launch(p, po.smem, po.grid, st));
            }
            break;
        }
        case LFD_OP_STEM4: {
            if (!input) return fail(LFD_ERR_INVALID, "stem4 needs the external input pointer");
            if (conv_impl == LFD_CONV_SIMT) return fail(LFD_ERR_UNSUPPORTED, "the SIMT cross-check kernels do not implement the fused stem (plan its four convs)");
            UmmaConvParams p = po.cp;
            p.in_raw = input; p.input_format = input_format; p.in = nullptr;
            p.in_words = input_format == LFD_INPUT_U8_NHWC && o.W % 4 == 0 && (reinterpret_cast<uintptr_t>(input) & 3) == 0;
            p.out = reinterpret_cast<__nv_bfloat16*>(ws + o.out_off); p.res = nullptr; p.stats = nullptr;
            p.w = reinterpret_cast<const __nv_bfloat16*>(o.weight); p.shift = o.shift; p.relu = o.relu;
            p.w2 = reinterpret_cast<const __nv_bfloat16*>(o.tail_weight); p.shift2 = o.tail_shift; p.relu2 = o.tail_relu;
            p.w_s2 = reinterpret_cast<const __nv_bfloat16*>(o.s2_weight); p.shift_s2 = o.s2_shift; p.relu_s2 = o.s2_relu;
            p.w_s3 = reinterpret_cast<const __nv_bfloat16*>(o.s3_weight); p.shift_s3 = o.s3_shift; p.relu_s3 = o.s3_relu;
            p.gn_groups = 0; p.trace = g_trace; p.tl = tl; p.f16 = o.dtype;
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
                p.trace = g_trace; p.tl = tl;
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
            if ((o.n_cls && !cls) || (o.n_reg && !reg)) return fail(LFD_ERR_INVALID, "head_final needs cls/reg output pointers");
            if (o.n_reg && o.n_reg != 4) return fail(LFD_ERR_INVALID, "head_final n_reg must be 0 or 4");
            CUDA_TRY(head_final_launch(p, bounded_sms(o.max_ctas), st));
            break;
        }
    }
    return LFD_OK;
}

extern "C" int lfd_plan_create(const lfd_op* ops, int n_ops, int N, int P, int cls_channels, int64_t stats_off, int64_t stats_bytes,
                               int64_t workspace_bytes, int conv_impl, lfd_plan** out) {
    if (!ops || n_ops <= 0 || !out) return fail(LFD_ERR_INVALID, "lfd_plan_create: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_plan_create: no CUDA device (there is no CPU fallback)");
    lfd_plan* pl = new lfd_plan();
    pl->N = N; pl->P = P; pl->cls_channels = cls_channels; pl->conv_impl = conv_impl;
    pl->stats_off = stats_off; pl->stats_bytes = stats_bytes; pl->workspace_bytes = workspace_bytes;
    pl->n_branches = 1;
    for (int i = 0; i < n_ops; ++i) {
        PlannedOp po;
        int rc = plan_op(ops[i], conv_impl, &po);
        if (rc) { delete pl; return rc; }
        if (ops[i].branch < 0 || ops[i].branch >= LFD_MAX_BRANCHES) { delete pl; return fail(LFD_ERR_INVALID, "op %d: branch %d out of range", i, ops[i].branch); }
        if (ops[i].branch + 1 > pl->n_branches) pl->n_branches = ops[i].branch + 1;
        if (ops[i].wait_mask < 0 || ops[i].wait_mask >= (1 << LFD_MAX_BRANCHES)) { delete pl; return fail(LFD_ERR_INVALID, "op %d: wait_mask 0x%x out of range", i, ops[i].wait_mask); }
        pl->ops.push_back(po);
    }
    size_t n_dep = 0;
    for (auto& po : pl->ops) n_dep += (size_t)__builtin_popcount((unsigned)po.op.wait_mask);
    for (int b = 1; b < pl->n_branches; ++b) {
        if (cudaStreamCreateWithFlags(&pl->side[b], cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&pl->fork_ev[b], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&pl->join_ev[b], cudaEventDisableTiming) != cudaSuccess) {
            pl->n_branches = b;  // destroy what exists
            lfd_plan_destroy(pl);
            return fail(LFD_ERR_CUDA, "lfd_plan_create: cannot create side streams");
        }
    }
    for (size_t i = 0; i < n_dep; ++i) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) {
            lfd_plan_destroy(pl);
            return fail(LFD_ERR_CUDA, "lfd_plan_create: cannot create dependency events");
        }
        pl->dep_ev.push_back(ev);
    }
    *out = pl;
    return LFD_OK;
}

extern "C" int lfd_plan_destroy(lfd_plan* plan) {
    if (!plan) return LFD_OK;
    for (auto& g : plan->graphs) cudaGraphExecDestroy(g.exec);
    for (int b = 1; b < plan->n_branches; ++b) {
        cudaStreamDestroy(plan->side[b]);
        cudaEventDestroy(plan->fork_ev[b]);
        cudaEventDestroy(plan->join_ev[b]);
    }
    for (auto ev : plan->dep_ev) cudaEventDestroy(ev);
    delete plan;
    return LFD_OK;
}

extern "C" int lfd_plan_num_launches(const lfd_plan* plan) { return plan ? (int)plan->ops.size() : 0; }

static int enqueue_all(lfd_plan* pl, const void* input, int fmt, uint8_t* ws, float* cls, float* reg, cudaStream_t st) {
    if (pl->stats_bytes > 0) CUDA_TRY(cudaMemsetAsync(ws + pl->stats_off, 0, (size_t)pl->stats_bytes, st));
    bool started[LFD_MAX_BRANCHES] = {false};
    int rc = LFD_OK;
    size_t dep = 0;
    for (size_t i = 0; i < pl->ops.size() && !rc; ++i) {
        const int b = pl->ops[i].op.branch;
        cudaStream_t s = st;
        if (b > 0) {
            s = pl->side[b];
            if (!started[b]) {  // fork: everything enqueued on the main stream so far precedes this branch
                CUDA_TRY(cudaEventRecord(pl->fork_ev[b], st));
                CUDA_TRY(cudaStreamWaitEvent(s, pl->fork_ev[b], 0));
                started[b] = true;
            }
        }
        for (int w = 0; w < LFD_MAX_BRANCHES; ++w) {   // explicit cross-branch dependencies
            if (!((pl->ops[i].op.wait_mask >> w) & 1)) continue;
            cudaEvent_t ev = pl->dep_ev[dep++];
            if (w == b || (w > 0 && (w >= pl->n_branches || !started[w]))) continue;   // nothing to wait for
            CUDA_TRY(cudaEventRecord(ev, w == 0 ? st : pl->side[w]));
            CUDA_TRY(cudaStreamWaitEvent(s, ev, 0));
        }
        rc = launch_op(pl->ops[i], i, input, fmt, ws, cls, reg, pl->P, pl->cls_channels, pl->conv_impl, s);
    }
    for (int b = 1; b < pl->n_branches; ++b)   // join (also on error paths, so that a stream capture can be closed)
        if (started[b]) {
            cudaEventRecord(pl->join_ev[b], pl->side[b]);
            cudaStreamWaitEvent(st, pl->join_ev[b], 0);
        }
    return rc;
}

extern "C" int lfd_plan_forward(lfd_plan* pl, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                                int use_graph, lfd_stream stream) {
    if (!pl || !input || !workspace || !cls_out || !reg_out) return fail(LFD_ERR_INVALID, "lfd_plan_forward: null argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    if (!use_graph) return enqueue_all(pl, input, input_format, ws, cls_out, reg_out, st);
    for (auto& g : pl->graphs)
        if (g.input == input && g.ws == workspace && g.cls == cls_out && g.reg == reg_out && g.fmt == input_format) {
            CUDA_TRY(cudaGraphLaunch(g.exec, st));
            return LFD_OK;
        }
    // first use of this pointer tuple: one eager pass (sets function attributes outside of capture, surfaces launch
    // errors directly and produces this call's outputs), then capture + instantiate for the following calls
    int rc = enqueue_all(pl, input, input_format, ws, cls_out, reg_out, st);
    if (rc) return rc;
    if (pl->graphs.size() >= kMaxGraphs) {
        cudaGraphExecDestroy(pl->graphs.front().exec);
        pl->graphs.erase(pl->graphs.begin());
    }
    cudaStream_t cap;
    CUDA_TRY(create_capture_stream(&cap));
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) { cudaStreamDestroy(cap); return fail(LFD_ERR_CUDA, "cudaStreamBeginCapture: %s", cudaGetErrorString(ce)); }
    rc = enqueue_all(pl, input, input_format, ws, cls_out, reg_out, cap);
    ce = cudaStreamEndCapture(cap, &graph);
    if (rc || ce != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        cudaStreamDestroy(cap);
        return rc ? rc : fail(LFD_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
    }
    lfd_plan::GraphEntry e;
    e.exec = nullptr; e.input = input; e.ws = workspace; e.cls = cls_out; e.reg = reg_out; e.fmt = input_format;
    ce = cudaGraphInstantiate(&e.exec, graph, 0);
    cudaGraphDestroy(graph);
    cudaStreamDestroy(cap);
    if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ce));
    pl->graphs.push_back(e);
    return LFD_OK;
}

extern "C" int lfd_plan_profile(lfd_plan* pl, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                                float* ms_per_op, lfd_stream stream) {
    if (!pl || !input || !workspace || !cls_out || !reg_out || !ms_per_op) return fail(LFD_ERR_INVALID, "lfd_plan_profile: null argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const size_t n = pl->ops.size();
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) CUDA_TRY(cudaEventCreate(&e));
    if (pl->stats_bytes > 0) CUDA_TRY(cudaMemsetAsync(ws + pl->stats_off, 0, (size_t)pl->stats_bytes, st));
    int rc = LFD_OK;
    CUDA_TRY(cudaEventRecord(ev[0], st));
    for (size_t i = 0; i < n && !rc; ++i) {
        rc = launch_op(pl->ops[i], i, input, input_format, ws, cls_out, reg_out, pl->P, pl->cls_channels, pl->conv_impl, st);
        cudaEventRecord(ev[i + 1], st);
    }
    cudaError_t ce = cudaStreamSynchronize(st);
    if (!rc && ce == cudaSuccess)
        for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
    for (auto& e : ev) cudaEventDestroy(e);
    if (rc) return rc;
    if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "lfd_plan_profile: %s", cudaGetErrorString(ce));
    return LFD_OK;
}


extern "C" int lfd_run_op(const lfd_op* op, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                          int P, int cls_channels, int conv_impl, lfd_stream stream) {
    if (!op || !workspace) return fail(LFD_ERR_INVALID, "lfd_run_op: null argument");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_run_op: no CUDA device (there is no CPU fallback)");
    PlannedOp po;
    int rc = plan_op(*op, conv_impl, &po);
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

extern "C" int lfd_postprocess(const lfd_post_cfg* c, const float* cls, const float* reg, const float* img_w, const float* img_h,
                               const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                               int32_t* overflow, lfd_stream stream) {
    if (!c || !cls || !reg || !img_w || !img_h || !resize_scale || !workspace || !dets || !labels || !src || !count || !overflow)
        return fail(LFD_ERR_INVALID, "lfd_postprocess: null argument");
    if (c->num_levels < 1 || c->num_levels > LFD_MAX_LEVELS || c->C < 1 || c->cap < 1) return fail(LFD_ERR_INVALID, "lfd_postprocess: bad config");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_postprocess: no CUDA device (there is no CPU fallback)");
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
    CUDA_TRY(nms_launch(q, c->N, st));
    return LFD_OK;
}

// multiclass_nms / batched_nms on explicit boxes (lfd/model/utils/nms.py:119-220): threshold + class-offset NMS, all on the device
extern "C" size_t lfd_multiclass_nms_workspace_bytes(int cap) { return cap > 0 ? post_layout(1, cap).total : 256; }

extern "C" int lfd_multiclass_nms(const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in, int n, int C,
                                  float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels, int32_t* src,
                                  int32_t* count, int32_t* overflow, lfd_stream stream) {
    if (n < 0 || C < 1 || cap < 1 || !workspace || !dets || !labels || !src || !count || !overflow || (n > 0 && (!boxes || !scores)))
        return fail(LFD_ERR_INVALID, "lfd_multiclass_nms: bad arguments");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_multiclass_nms: no CUDA device (there is no CPU fallback)");
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
    CUDA_TRY(nms_launch(q, 1, st));
    return LFD_OK;
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

extern "C" int lfd_detection_loss(const lfd_levels* lv, const lfd_loss_cfg* c, const float* cls_logits, const float* reg, const float* cls_target,
                                  const float* reg_target, const int32_t* label, const int32_t* counters, float* grad_cls, float* grad_reg,
                                  double* loss_sums, lfd_stream stream) {
    if (!lv || !c || !cls_logits || !reg || !reg_target || !label || !counters || !loss_sums) return fail(LFD_ERR_INVALID, "lfd_detection_loss: null argument");
    if (c->cls_mode < LFD_CLS_SIGMOID || c->cls_mode > LFD_CLS_QFL) return fail(LFD_ERR_INVALID, "lfd_detection_loss: unknown classification loss %d", c->cls_mode);
    if ((c->cls_mode == LFD_CLS_BCE || c->cls_mode == LFD_CLS_QFL) && !cls_target) return fail(LFD_ERR_INVALID, "lfd_detection_loss: BCE / QFL need the soft classification targets");
    if (c->reg_loss < LFD_REG_IOU || c->reg_loss > LFD_REG_MSE) return fail(LFD_ERR_INVALID, "lfd_detection_loss: unknown regression loss %d", c->reg_loss);
    const bool indep = c->reg_loss == LFD_REG_SMOOTH_L1 || c->reg_loss == LFD_REG_MSE;
    if (indep != (c->bbox_mode == LFD_BBOX_INDEPENDENT)) return fail(LFD_ERR_INVALID, "lfd_detection_loss: SmoothL1 / MSE go with the 'independent' targets, the IoU family with sigmoid / exp");
    if (c->reg_loss == LFD_REG_SMOOTH_L1 && !(c->smooth_l1_beta > 0.f)) return fail(LFD_ERR_INVALID, "lfd_detection_loss: SmoothL1 beta must be > 0");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_detection_loss: no CUDA device (there is no CPU fallback)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int sms = c->max_ctas > 0 ? c->max_ctas : sm_count();
    CUDA_TRY(cudaMemsetAsync(loss_sums, 0, 16, st));
    ClsLossParams k;
    k.logits = cls_logits; k.cls_target = cls_target; k.label = label; k.counters = counters; k.grad = grad_cls; k.loss_sum = loss_sums;
    k.N = c->N; k.P = c->P; k.C = c->C; k.cls_mode = c->cls_mode; k.gamma = c->gamma; k.alpha = c->alpha; k.loss_weight = c->cls_weight;
    CUDA_TRY(cls_loss_launch(k, sms, st));
    RegLossParams r;
    fill_levels(lv, &r.lv);
    r.reg = reg; r.reg_target = reg_target; r.label = label; r.counters = counters; r.grad = grad_reg; r.loss_sum = loss_sums + 1;
    r.N = c->N; r.P = c->P; r.C = c->C; r.bbox_mode = c->bbox_mode; r.loss_kind = c->reg_loss; r.eps = c->reg_eps; r.loss_weight = c->reg_weight;
    r.beta = c->smooth_l1_beta;
    CUDA_TRY(iou_loss_launch(r, sms, st));
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
    int64_t workspace_bytes;
    struct GraphEntry { cudaGraphExec_t exec; const void* input; void* ws; int fmt; };
    std::vector<GraphEntry> graphs;
    // side streams of the independent per-level chains (same fork / wait / join protocol as lfd_plan)
    cudaStream_t side[LFD_MAX_BRANCHES];
    cudaEvent_t fork_ev[LFD_MAX_BRANCHES], join_ev[LFD_MAX_BRANCHES];
    std::vector<cudaEvent_t> dep_ev;
    int n_branches = 1;
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
            return plan_op(o, t.impl, &out->conv);
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
            return plan_op(o, LFD_CONV_UMMA, &out->conv);
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
        case LFD_TOP_NORM_BWD_REDUCE: case LFD_TOP_NORM_BWD_APPLY: case LFD_TOP_WGRAD_STEM: case LFD_TOP_ZERO:
            break;
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
            if (t.off[0] >= 0 && t.impl == LFD_WGRAD_UMMA) {
                // tensor-core path: im2col into the scratch tensor X27 [N][Ho][Wo][32] at off[0], then the 1x1 wgrad (32 -> Cout) over it;
                // the staging at off[5] must hold 32 rows of Cout floats (rows 27..31 stay zero)
                __nv_bfloat16* x27 = at<__nv_bfloat16>(ws, t.off[0]);
                CUDA_TRY(stem_im2col_launch(g, input, fmt, x27, sms, st));
                WgradGeom g1 = {t.N, t.Ho, t.Wo, 32, t.Ho, t.Wo, t.Cout, 1, 1};
                CUDA_TRY(wgrad_umma_launch(g1, x27, at<const __nv_bfloat16>(ws, t.off[1]), at<float>(ws, t.off[5]), sms, st));
            } else {
                CUDA_TRY(wgrad_stem_launch(g, input, fmt, at<const __nv_bfloat16>(ws, t.off[1]), at<float>(ws, t.off[5]), sms, st));
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
    pl->workspace_bytes = workspace_bytes;
    size_t n_dep = 0;
    for (int i = 0; i < n_ops; ++i) {
        PlannedTop pt;
        int rc = plan_top(ops[i], workspace_bytes, &pt);
        if (rc) { delete pl; return rc; }
        if (ops[i].branch < 0 || ops[i].branch >= LFD_MAX_BRANCHES || ops[i].wait_mask < 0 || ops[i].wait_mask >= (1 << LFD_MAX_BRANCHES)) {
            delete pl;
            return fail(LFD_ERR_INVALID, "training op %d: branch %d / wait_mask 0x%x out of range", i, ops[i].branch, ops[i].wait_mask);
        }
        if (ops[i].branch + 1 > pl->n_branches) pl->n_branches = ops[i].branch + 1;
        n_dep += (size_t)__builtin_popcount((unsigned)ops[i].wait_mask);
        pl->ops.push_back(pt);
    }
    const int nb = pl->n_branches;
    pl->n_branches = 1;
    for (int b = 1; b < nb; ++b) {
        if (cudaStreamCreateWithFlags(&pl->side[b], cudaStreamNonBlocking) != cudaSuccess) { lfd_train_plan_destroy(pl); return fail(LFD_ERR_CUDA, "lfd_train_plan_create: cannot create side streams"); }
        if (cudaEventCreateWithFlags(&pl->fork_ev[b], cudaEventDisableTiming) != cudaSuccess) { cudaStreamDestroy(pl->side[b]); lfd_train_plan_destroy(pl); return fail(LFD_ERR_CUDA, "lfd_train_plan_create: cannot create events"); }
        if (cudaEventCreateWithFlags(&pl->join_ev[b], cudaEventDisableTiming) != cudaSuccess) { cudaStreamDestroy(pl->side[b]); cudaEventDestroy(pl->fork_ev[b]); lfd_train_plan_destroy(pl); return fail(LFD_ERR_CUDA, "lfd_train_plan_create: cannot create events"); }
        pl->n_branches = b + 1;
    }
    for (size_t i = 0; i < n_dep; ++i) {
        cudaEvent_t ev;
        if (cudaEventCreateWithFlags(&ev, cudaEventDisableTiming) != cudaSuccess) { lfd_train_plan_destroy(pl); return fail(LFD_ERR_CUDA, "lfd_train_plan_create: cannot create dependency events"); }
        pl->dep_ev.push_back(ev);
    }
    *out = pl;
    return LFD_OK;
}

extern "C" int lfd_train_plan_destroy(lfd_train_plan* plan) {
    if (!plan) return LFD_OK;
    for (auto& g : plan->graphs) cudaGraphExecDestroy(g.exec);
    for (int b = 1; b < plan->n_branches; ++b) {
        cudaStreamDestroy(plan->side[b]);
        cudaEventDestroy(plan->fork_ev[b]);
        cudaEventDestroy(plan->join_ev[b]);
    }
    for (auto ev : plan->dep_ev) cudaEventDestroy(ev);
    delete plan;
    return LFD_OK;
}

extern "C" int lfd_train_plan_num_ops(const lfd_train_plan* plan) { return plan ? (int)plan->ops.size() : 0; }

static int train_enqueue(lfd_train_plan* pl, const void* input, int fmt, uint8_t* ws, cudaStream_t st) {
    bool started[LFD_MAX_BRANCHES] = {false};
    int rc = LFD_OK;
    size_t dep = 0;
    cudaError_t ce = cudaSuccess;
    for (size_t i = 0; i < pl->ops.size() && !rc && ce == cudaSuccess; ++i) {
        const lfd_top& t = pl->ops[i].op;
        const int b = t.branch;
        cudaStream_t s = st;
        if (b > 0) {
            s = pl->side[b];
            if (!started[b]) {   // fork: everything enqueued on the main stream so far precedes this branch
                if ((ce = cudaEventRecord(pl->fork_ev[b], st)) != cudaSuccess || (ce = cudaStreamWaitEvent(s, pl->fork_ev[b], 0)) != cudaSuccess) break;
                started[b] = true;
            }
        }
        for (int w = 0; w < LFD_MAX_BRANCHES && ce == cudaSuccess; ++w) {
            if (!((t.wait_mask >> w) & 1)) continue;
            cudaEvent_t ev = pl->dep_ev[dep++];
            if (w == b || (w > 0 && (w >= pl->n_branches || !started[w]))) continue;
            if ((ce = cudaEventRecord(ev, w == 0 ? st : pl->side[w])) == cudaSuccess) ce = cudaStreamWaitEvent(s, ev, 0);
        }
        if (ce == cudaSuccess) rc = launch_top(pl->ops[i], input, fmt, ws, s);
    }
    for (int b = 1; b < pl->n_branches; ++b)   // join (also on error paths, so that a stream capture can be closed)
        if (started[b]) {
            cudaEventRecord(pl->join_ev[b], pl->side[b]);
            cudaStreamWaitEvent(st, pl->join_ev[b], 0);
        }
    if (!rc && ce != cudaSuccess) rc = fail(LFD_ERR_CUDA, "training plan stream dependencies: %s", cudaGetErrorString(ce));
    return rc;
}

extern "C" int lfd_train_plan_run(lfd_train_plan* pl, const void* input, int input_format, void* workspace, int use_graph, lfd_stream stream) {
    if (!pl || !workspace) return fail(LFD_ERR_INVALID, "lfd_train_plan_run: null argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    if (!use_graph) return train_enqueue(pl, input, input_format, ws, st);
    for (auto& g : pl->graphs)
        if (g.input == input && g.ws == workspace && g.fmt == input_format) {
            CUDA_TRY(cudaGraphLaunch(g.exec, st));
            return LFD_OK;
        }
    int rc = train_enqueue(pl, input, input_format, ws, st);   // eager first pass (function attributes, launch errors)
    if (rc) return rc;
    if (pl->graphs.size() >= 8) {
        cudaGraphExecDestroy(pl->graphs.front().exec);
        pl->graphs.erase(pl->graphs.begin());
    }
    // The first eager pass already produced this call's results; the graph is captured for the FOLLOWING calls.  Capture does
    // not execute anything, so the state (statistics, staging) is untouched.
    cudaStream_t cap;
    CUDA_TRY(create_capture_stream(&cap));
    cudaGraph_t graph = nullptr;
    cudaError_t ce = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (ce != cudaSuccess) { cudaStreamDestroy(cap); return fail(LFD_ERR_CUDA, "cudaStreamBeginCapture: %s", cudaGetErrorString(ce)); }
    rc = train_enqueue(pl, input, input_format, ws, cap);
    ce = cudaStreamEndCapture(cap, &graph);
    if (rc || ce != cudaSuccess) {
        if (graph) cudaGraphDestroy(graph);
        cudaStreamDestroy(cap);
        return rc ? rc : fail(LFD_ERR_CUDA, "cudaStreamEndCapture: %s", cudaGetErrorString(ce));
    }
    lfd_train_plan::GraphEntry e;
    e.exec = nullptr; e.input = input; e.ws = workspace; e.fmt = input_format;
    ce = cudaGraphInstantiate(&e.exec, graph, 0);
    cudaGraphDestroy(graph);
    cudaStreamDestroy(cap);
    if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(ce));
    pl->graphs.push_back(e);
    return LFD_OK;
}

extern "C" int lfd_train_plan_profile(lfd_train_plan* pl, const void* input, int input_format, void* workspace, float* ms_per_op, lfd_stream stream) {
    if (!pl || !workspace || !ms_per_op) return fail(LFD_ERR_INVALID, "lfd_train_plan_profile: null argument");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    const size_t n = pl->ops.size();
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) CUDA_TRY(cudaEventCreate(&e));
    int rc = LFD_OK;
    CUDA_TRY(cudaEventRecord(ev[0], st));
    for (size_t i = 0; i < n && !rc; ++i) {
        rc = launch_top(pl->ops[i], input, input_format, ws, st);
        cudaEventRecord(ev[i + 1], st);
    }
    cudaError_t ce = cudaStreamSynchronize(st);
    if (!rc && ce == cudaSuccess)
        for (size_t i = 0; i < n; ++i) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
    for (auto& e : ev) cudaEventDestroy(e);
    if (rc) return rc;
    if (ce != cudaSuccess) return fail(LFD_ERR_CUDA, "lfd_train_plan_profile: %s", cudaGetErrorString(ce));
    return LFD_OK;
}

extern "C" int lfd_run_top(const lfd_top* op, const void* input, int input_format, void* workspace, lfd_stream stream) {
    if (!op || !workspace) return fail(LFD_ERR_INVALID, "lfd_run_top: null argument");
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_run_top: no CUDA device (there is no CPU fallback)");
    PlannedTop pt;
    int rc = plan_top(*op, INT64_MAX, &pt);
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
    if (out_mode != LFD_INPUT_OUT_U8_NHWC && out_mode != LFD_INPUT_OUT_F32_NCHW) return fail(LFD_ERR_INVALID, "lfd_input_batch: out_mode %d", out_mode);
    if (out_mode == LFD_INPUT_OUT_F32_NCHW && (!mean || !scale)) return fail(LFD_ERR_INVALID, "lfd_input_batch: the fp32 mode needs mean and scale");
    if (W > 6144) return fail(LFD_ERR_UNSUPPORTED, "lfd_input_batch: W=%d > 6144 (the column table lives in 48 KB of shared memory)", W);
    if (n > 65535) return fail(LFD_ERR_UNSUPPORTED, "lfd_input_batch: n=%d > 65535", n);
    if (n == 0) return LFD_OK;
    if (sm_count() <= 0) return fail(LFD_ERR_CUDA, "lfd_input_batch: no CUDA device (there is no CPU fallback)");
    CUDA_TRY(input_batch_launch(descs, n, src, out, out_mode, swap_rb, H, W, mean, scale, st_of(stream)));
    return LFD_OK;
}
