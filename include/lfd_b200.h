/* lfd_b200.h -- C-ABI of liblfd_b200.so: the H100 (sm_90a) implementation of the LFD dense-conv hot path.
 *
 * Conventions
 *   - plain C: raw device pointers, explicit shapes, a cudaStream_t passed as void*; no torch / C++ types.
 *   - nothing is allocated inside: the caller supplies outputs and workspaces (sizes via the *_bytes queries).
 *   - every function returns 0 (LFD_OK) or an lfd_status; lfd_last_error() gives a thread-local message.
 *     No exceptions cross the boundary.  Calls are asynchronous on the given stream unless stated otherwise.
 *   - there is no CPU fallback: every entry point launches CUDA kernels and fails if no sm_90 device is present.
 *
 * Reference interfaces replaced (paths relative to the reference repository root):
 *   lfd_plan_*                     LFD.forward                         lfd/model/lfd.py:511-542
 *                                  (LFDResNet.forward lfd/model/backbone/lfd_resnet.py:488-501,
 *                                   SimpleNeck.forward lfd/model/neck/simple_neck.py:67-74,
 *                                   LFDHead.forward    lfd/model/head/lfd_head.py:164-185)
 *   lfd_postprocess                LFD._get_results_for_single_image   lfd/model/lfd.py:434-509, predict path :577-641,
 *                                  multiclass_nms / batched_nms        lfd/model/utils/nms.py:119-220
 *   lfd_multiclass_nms             multiclass_nms / batched_nms        lfd/model/utils/nms.py:119-220 (on explicit boxes)
 *   lfd_postprocess_soft_nms,      soft_nms, nms_cfg type 'soft_nms'   lfd/model/utils/nms.py:62-158,
 *   lfd_multiclass_soft_nms                                            build/nms/src/cpu/nms_cpu.cpp:76-217
 *   lfd_nms                        nms_ext.nms                         lfd/model/utils/build/nms/src/nms_ext.cpp:18-29,
 *                                                                      cpu/nms_cpu.cpp:8-75, cuda/nms_kernel.cu:71-138
 *   lfd_sigmoid_focal_loss_forward sigmoid_focal_loss_ext.forward      lfd/model/losses/build/sigmoid_focal_loss/src/sigmoid_focal_loss_ext.cpp:19-34
 *   lfd_sigmoid_focal_loss_backward sigmoid_focal_loss_ext.backward    same file :36-50
 *   lfd_assign_targets             LFD.annotation_to_target            lfd/model/lfd.py:109-259
 *   lfd_detection_loss             LFD.get_loss (loss + d loss/d outputs) lfd/model/lfd.py:284-395 with
 *                                  FocalLoss / CrossEntropyLoss / IoULoss lfd/model/losses/{focal_loss,cross_entropy_loss,iou_loss}.py
 *   lfd_loss_weight_sum,           the same with enable_classification_weight / enable_regression_weight (lfd/model/lfd.py:322-384,
 *   lfd_detection_loss_weighted    weight_reduce_loss lfd/model/losses/utils.py:28-53)
 */
#ifndef LFD_B200_H_
#define LFD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LFD_B200_ABI_VERSION 5
#define LFD_MAX_LEVELS 8
#define LFD_MAX_BRANCHES 8

typedef enum lfd_status {
    LFD_OK = 0,
    LFD_ERR_INVALID = 1,      /* bad argument / unsupported shape */
    LFD_ERR_CUDA = 2,         /* a CUDA runtime call failed (message has the CUDA error string) */
    LFD_ERR_UNSUPPORTED = 3,  /* configuration outside the implemented hot path */
    LFD_ERR_CAPACITY = 4      /* caller-provided capacity too small */
} lfd_status;

typedef void* lfd_stream; /* cudaStream_t */
typedef struct lfd_plan lfd_plan;

int lfd_abi_version(void);
/* sizeof of the structs of this header as the library was compiled, for bindings that mirror them field by field (ctypes, cffi):
 * which = 0 lfd_op, 1 lfd_top, 2 lfd_pack_desc, 3 lfd_unpack_desc, 4 lfd_post_cfg, 5 lfd_loss_cfg, 6 lfd_levels, 7 lfd_input_desc,
 * 8 lfd_extent, 9 lfd_engine_desc;
 * -1 for anything else. */
int lfd_struct_bytes(int which);
const char* lfd_last_error(void);
/* number of SMs of the current device (0 + error when there is no usable device) */
int lfd_device_sm_count(void);

/* ------------------------------------------------------------------------------------------ forward plan */
enum { LFD_OP_STEM0 = 0, LFD_OP_CONV = 1, LFD_OP_GN_APPLY = 2, LFD_OP_HEAD_FINAL = 3, LFD_OP_STEM4 = 4 };
enum { LFD_INPUT_F32_NCHW = 0, LFD_INPUT_U8_NHWC = 1, LFD_INPUT_U8_NV12 = 2 };
/* LFD_INPUT_U8_NV12 (inference only): YUV 4:2:0 video frames, one contiguous uint8 buffer without row padding.  Image n starts at byte
 * n * H * W * 3 / 2 and holds a Y plane of H rows x W bytes, then an interleaved UV plane of H / 2 rows x W bytes (U at even bytes, V at
 * odd bytes): the bytes of a uint8 [N][3H/2][W] tensor.  H and W are even.  A pixel (y, x) is turned into the three bytes (B, G, R) from
 * its Y byte and the (U, V) pair at UV row y / 2, UV column x & ~1, by BT.601 limited range in 20-bit fixed point:
 *     y' = max(0, Y - 16) * 1220542,  u = U - 128,  v = V - 128,  h = 1 << 19
 *     B = sat8((y' + h + 2116026 * u) >> 20)
 *     G = sat8((y' + h - 852492 * v - 409993 * u) >> 20)
 *     R = sat8((y' + h + 1673527 * v) >> 20)          (arithmetic shifts; sat8 clamps to 0..255)
 * which is, bit for bit, cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12).  From there the frame is a uint8 BGR frame: the input transform
 * below applies to the three bytes by their position (B = 0, G = 1, R = 2), and every op and plan gives on an NV12 frame exactly what it
 * gives on the converted BGR frame.  A frame below a plan's capacity (lfd_plan_forward_extent) lies in the capacity layout: its h x w
 * Y rows in the top-left corner of the H x W Y plane, its h / 2 UV rows in the top-left corner of the H / 2 x W UV plane.
 * lfd_plan_forward, lfd_plan_forward_extent, lfd_plan_profile and lfd_run_op check before anything is enqueued: an odd frame height or
 * width is LFD_ERR_INVALID, an NV12 frame on a plan (an image op) of odd capacity H or W is LFD_ERR_UNSUPPORTED.  lfd_train_plan_run,
 * lfd_train_plan_profile and lfd_run_top refuse NV12 with LFD_ERR_UNSUPPORTED.  Every entry point refuses a format other than these three
 * with LFD_ERR_INVALID.
 * GRAY (1-channel) PLANS: an image op (STEM0 / STEM4; lfd_top STEM0 / WGRAD_STEM) with Cin = 1 reads one value per pixel, and the same
 * format numbers then mean: LFD_INPUT_F32_NCHW float[N][1][H][W]; LFD_INPUT_U8_NHWC uint8[N][H][W] (1 byte per pixel); LFD_INPUT_U8_NV12
 * the usual NV12 buffer above, of which only the Y plane is read (the UV bytes are never touched): Y is the gray byte, as
 * cv2.cvtColor(frame, cv2.COLOR_YUV2GRAY_NV12) defines it.  A gray model with stem weights W1 gives, bit for bit, what the 3-channel model
 * with stem weights [W1, 0, 0] gives on a frame whose channel 0 is the gray frame. */
enum { LFD_CONV_UMMA = 0, LFD_CONV_SIMT = 1 }; /* SIMT = cross-check kernel, validation only */
/* 16-bit storage type of activations and packed weights (fp32 accumulation either way; same bytes, same tensor-core rate):
 * bf16 = the north-star dtype; fp16 = 3 more mantissa bits, the variant that meets 1e-3 END TO END (DESIGN.md "Parity") and the
 * dtype of BASELINE config 5 (WIDERFACE-XS fp16 4K sweep).  "bf16" in the op descriptions below reads "the plan's 16-bit type". */
enum { LFD_DTYPE_BF16 = 0, LFD_DTYPE_FP16 = 1 };

/* The input transform of the ops that read the uint8 image (lfd_op: STEM0, STEM4; lfd_top: STEM0, WGRAD_STEM; an INFER op carries its
 * lfd_op's): in_swap_rb (0 / 1), in_mean[3], in_scale[3] in float32, indexed by NETWORK input channel:
 *     input channel c of a pixel = ((float) byte[in_swap_rb ? 2 - c : c] - in_mean[c]) * in_scale[c]     (fp32: a subtract, then a multiply)
 * which is albumentations' Normalize (mean[c] = mean * max_pixel_value, scale[c] = float32(1 / (std * max_pixel_value))) after an optional
 * BGR -> RGB, so the 16-bit value a stem kernel builds for a pixel is the rounding of the fp32 number the host pipeline would have uploaded.
 * Pixels outside the image (conv padding, beyond a smaller frame's extent) are 0 after the transform.  ALL SEVEN FIELDS ZERO selects
 * simple_normalize on BGR, mean 127.5 and scale float32(1 / 127.5): a zero-filled struct behaves as the library always did.  Anything else
 * must be complete: in_swap_rb 0 or 1, every mean finite, every scale finite and non-zero; otherwise the op fails with LFD_ERR_INVALID when
 * it is planned, before anything is enqueued.  On a gray op (Cin = 1) the one channel is ((float) byte - in_mean[0]) * in_scale[0]: a
 * nonzero in_swap_rb, or unequal in_mean / in_scale values, is LFD_ERR_INVALID there.  The LFD_INPUT_F32_NCHW input is taken as it is and
 * ignores these fields. */

/* One fused layer.  Activations are bf16 NHWC at byte offsets into the caller's workspace.
 *   STEM0      3x3/s2 conv on the image + shift (+ReLU), Cin = 3 (BGR) or 1 (gray), scale folded into the weights like CONV; in_off ignored
 *              (reads the external input);
 *              weight = bf16 packed [kh][2][Cout][8]: element (kh, kc, n, j) = weight of output n, input channel j % 4, filter
 *              column kw = 2*kc + j/4 (zero for kw = 3 and for the padded 4th channel): the kernel keeps the image patch as
 *              4-channel bf16 pixels and lets the wgmma address generator do the im2col (K = 16 per filter row).  A gray op's weight is
 *              packed the same way with its one channel in the channel-0 lanes and zeros in the others.
 *   STEM4      the four convolutions of a 'faster' stem in one kernel: stem0 3x3/s2 3->64 (weight / shift / relu, packed as STEM0),
 *              stem1 1x1 64->64 (tail_weight / tail_shift / tail_relu, tail_cout = 64), stem2 3x3/s2 64->64 (s2_weight = bf16 packed
 *              [9][8][64][8], i.e. the CONV packing with cc = 64; s2_shift / s2_relu) and stem3 1x1 64->64 (s3_weight = bf16 packed
 *              [8][64][8]; s3_shift / s3_relu).  Cin = 3 or 1, Cout = 64, ksize = 3, stride = 2; H x W = the image, Ho x Wo = the stem3
 *              output (two stride-2 steps); in_off ignored.  Every intermediate is rounded to bf16 exactly as the STEM0 + CONV pair
 *              path rounds it, so the output is bit-identical to it; the stem1 map never reaches HBM.  Sizes: lfd_stem4_query.
 *   CONV       ksize in {1,3}, stride in {1,2}, pad = ksize/2; y = conv(x) + shift (+res) (ReLU) -> bf16; Cout in {16, 32, 48, 64, 128}
 *              (3x3: from 32), Cin a multiple of 16; STEM0 Cout in {16, 32, 48, 64};
 *              weight = bf16 packed [Cin/cc][ksize^2][cc/8][Cout][8] with cc from lfd_conv_query, ALREADY MULTIPLIED by the
 *              per-output-channel scale (folded BatchNorm); `scale` must be NULL; `shift` (fp32 [Cout], may be NULL) is rounded
 *              to bf16 and added on the tensor core;
 *              gn_groups > 0: also accumulates sum / sum-of-squares of the stored output (after residual and ReLU, as rounded
 *              to bf16) per (image, group) into double[N][gn_groups][2] at stats_off (group size must be 8).
 *   GN_APPLY   y = relu(gamma * (x - mean) * rstd + beta) from the statistics at stats_off, bf16 -> bf16.
 *   HEAD_FINAL GN_APPLY (as above, rounded to bf16; gn_groups = 0: no normalisation, the input is an already activated tensor --
 *              heads built with norm_cfg=None) followed by the final 1x1 convs of one level: outputs
 *              [0, n_cls) -> cls[n][point_off + pixel][.] and [n_cls, n_cls + n_reg) -> reg[n][point_off + pixel][.];
 *              weight = float[n_cls + n_reg][Cin]; scale/shift = per-output scale and (scale * bias).
 */
typedef struct lfd_op {
    int32_t kind;
    int32_t N, H, W, Cin, Ho, Wo, Cout;
    int32_t ksize, stride, relu, gn_groups;
    int32_t n_cls, n_reg, point_off, cc;
    int32_t branch, wait_mask; /* branch 0 = main stream; ops of branch b > 0 run on side stream b, forked after the
                                 main-stream op that precedes the branch's first op and joined at the end.  wait_mask:
                                 bit w set = this op additionally waits for everything enqueued so far on branch w
                                 (mid-graph joins, e.g. a residual block's last conv waiting for its side-branch
                                 downsample conv, or a side-branch op waiting for a later main-stream tensor) */
    int64_t in_off, out_off, res_off, stats_off; /* bytes; -1 = unused */
    const void* weight;
    const float* scale; /* HEAD_FINAL: per-output scale; STEM0 / CONV: must be NULL (fold it into the weights) */
    const float* shift;
    const float* gamma;
    const float* beta;
    /* STEM0 / CONV only: a 1x1/s1 conv (Cout -> tail_cout) + scale/shift (+ReLU) fused behind this layer inside the same
     * kernel; tail_weight = bf16 packed [Cout/8][tail_cout][8] (scale folded in, tail_scale must be NULL); tail_cout = 48 goes with Cout = 48
     * only, and the other tail widths (16 / 32 / 64 / 128) with the other Cout.  The stored tensor then has tail_cout channels and
     * res_off / gn_groups / stats_off refer to it; the Cout-channel intermediate never reaches HBM.  0 = no tail. */
    int32_t tail_cout, tail_relu;
    const void* tail_weight;
    const float* tail_scale;
    const float* tail_shift;
    /* CONV 3x3/s2 only (no tail, no residual): the residual block's 1x1/s2 shortcut conv on the SAME input (Cin -> ds_cout,
     * ds_cout == Cout) is computed by the same kernel -- its input pixel is this conv's centre tap -- and stored (no ReLU) at
     * ds_out_off.  ds_weight = bf16 packed [Cin/8][ds_cout][8] with the BatchNorm scale folded in.  0 = none. */
    int32_t ds_cout;
    int32_t dtype; /* LFD_DTYPE_*: 16-bit type of this op's activations AND packed weights (every op of one plan uses the same) */
    int32_t max_ctas; /* STEM0 / CONV: upper bound on the persistent CTAs of this layer, 0 = one per SM slot.  The CTAs of a large side-branch
                         layer hold their SMs for the whole layer; bounding them leaves SMs to the small, latency-bound layers of the
                         critical path that run concurrently (lfd/_engine.py::InferencePlan.autotune picks the bounds by timing). */
    int32_t pad_;
    int64_t ds_out_off;
    const void* ds_weight;
    const float* ds_shift;
    /* STEM4 only: the third and fourth convolution of the fused stem (see STEM4 above) */
    int32_t s2_relu, s3_relu;
    const void* s2_weight;
    const float* s2_shift;
    const void* s3_weight;
    const float* s3_shift;
    /* STEM0 / STEM4 on a LFD_INPUT_U8_NHWC or LFD_INPUT_U8_NV12 image: the input transform (see below).  All zero = simple_normalize on BGR. */
    int32_t in_swap_rb;
    float in_mean[3];
    float in_scale[3];
    int32_t pad2_;
} lfd_op;

/* Tile / pipeline configuration the wgmma kernel will use for a conv (host only, no launch).  Output widths: 16 / 32 / 48 / 64 / 128
 * (3x3 from 32; tail_cout as for lfd_op); fails with LFD_ERR_UNSUPPORTED otherwise.
 * cc = input-channel chunk the weights must be packed with. */
int lfd_conv_query(int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int ksize, int stride, int tail_cout, int ds_cout, int* cc,
                   int* stages, int* weights_resident, int* num_tiles, int64_t* smem_bytes);
/* The consumer schedule the wgmma kernel runs for that conv on this device (host only): *solo = 1 when each of its two consumer
 * warpgroups computes whole tiles and the two alternate on the tensor cores (64 -> 64 channel 3x3/s1 convs without tail with at least
 * two tiles per CTA), 0 when both work on every tile. */
int lfd_conv_schedule(int N, int H, int W, int Cin, int Ho, int Wo, int Cout, int ksize, int stride, int tail_cout, int ds_cout, int* solo);
/* The same for a STEM4 op on N images of H x W (host only): its tiles (16 x 8 stem3 pixels each), dynamic shared memory per CTA
 * and stem3 output size. */
int lfd_stem4_query(int N, int H, int W, int* num_tiles, int64_t* smem_bytes, int* Ho, int* Wo);

/* The plan copies the op list.  stats_off/stats_bytes: region of the workspace zeroed at the start of each forward. */
int lfd_plan_create(const lfd_op* ops, int n_ops, int N, int P, int cls_channels, int64_t stats_off, int64_t stats_bytes,
                    int64_t workspace_bytes, int conv_impl, lfd_plan** out);
int lfd_plan_destroy(lfd_plan* plan);
int lfd_plan_num_launches(const lfd_plan* plan); /* kernels launched per forward */
/* cls_out float[N][P][cls_channels], reg_out float[N][P][4].  use_graph != 0: the launch sequence is captured into a
 * CUDA graph on first use for this (input, workspace, cls_out, reg_out) tuple and replayed afterwards. */
int lfd_plan_forward(lfd_plan* plan, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                     int use_graph, lfd_stream stream);
/* Frames smaller than the plan: the plan's (N, H, W) is its capacity, and a frame of h <= H rows and w <= W columns runs on the same
 * kernels, workspace and CUDA graph.  Every tensor keeps the plan's layout (row pitch = the plan's width of that tensor) with the valid
 * h x w region, and its successors, in the top-left corner; nothing outside it is read.  ext[n_ops] (host) gives per op the valid
 * input H x W and output Ho x Wo, and for HEAD_FINAL the level's first point and the frame's point count P (0 for the other ops), exactly
 * the fields of a plan built for the frame.  The table is copied, stream-ordered, into a device table that the kernels read when they
 * start.  `input` holds the frame in the capacity layout: uint8 [N][H][W][3], float32 [N][3][H][W] or NV12 uint8 [N][3H/2][W] (see
 * LFD_INPUT_U8_NV12) with the frame in the top-left corner.  cls_out / reg_out receive the frame's outputs as a plan built for it lays them out: float[N][P][cls_channels] and
 * float[N][P][4] at the start of the buffers.  h == H and w == W is lfd_plan_forward (ext is not read).  A frame outside the capacity
 * or an inconsistent table fails with LFD_ERR_INVALID before anything is enqueued; the SIMT cross-check path runs full-size frames only
 * (LFD_ERR_UNSUPPORTED).  use_graph: one graph per pointer tuple as in lfd_plan_forward, shared by every frame size. */
typedef struct lfd_extent {
    int32_t H, W, Ho, Wo;
    int32_t point_off, P;
    int32_t pad_[2];
} lfd_extent;
int lfd_plan_forward_extent(lfd_plan* plan, const void* input, int input_format, int h, int w, const lfd_extent* ext, void* workspace,
                            float* cls_out, float* reg_out, int use_graph, lfd_stream stream);
/* CUDA graphs the plan holds instantiated (tests) */
int lfd_plan_num_graphs(const lfd_plan* plan);
/* One eager forward with a CUDA event pair around every op: ms_per_op float[lfd_plan_num_launches()] (host).
 * Synchronises the stream.  Used by bench.py for the live per-kernel roofline. */
int lfd_plan_profile(lfd_plan* plan, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out,
                     float* ms_per_op, lfd_stream stream);
/* Debugging aid: device buffer long long[4][32][4] that CTA 0 of every following wgmma conv launch fills with a
 * clock64() timeline (role 0 producer / 1 MMA issuer / 2 epilogue, per tile); NULL switches it off. */
int lfd_debug_set_trace(void* device_buffer);
/* Debugging aid (LFD_B200_TIMELINE builds): device buffer unsigned long long[2 * lfd_plan_num_launches()], pre-set by the caller
 * to {UINT64_MAX, 0} pairs; op i of every following plan launch (CUDA-graph replays included, when set before the capture)
 * records its earliest CTA start and latest CTA end in %globaltimer nanoseconds.  NULL switches it off. */
int lfd_debug_set_timeline(void* device_buffer);
/* run a single op (tests / debugging) */
int lfd_run_op(const lfd_op* op, const void* input, int input_format, void* workspace, float* cls_out, float* reg_out, int P,
               int cls_channels, int conv_impl, lfd_stream stream);

/* ------------------------------------------------------------------------------------------ post-process */
enum { LFD_CLS_SIGMOID = 0, LFD_CLS_SOFTMAX = 1 };
enum { LFD_BBOX_SIGMOID = 0, LFD_BBOX_EXP = 1, LFD_BBOX_INDEPENDENT = 2 };

typedef struct lfd_post_cfg {
    int32_t N, P, C;            /* C = number of foreground classes */
    int32_t cls_channels;       /* C (sigmoid) or C + 1 (softmax, background last) */
    int32_t cls_mode, bbox_mode, class_agnostic;
    int32_t num_levels;
    int32_t level_off[LFD_MAX_LEVELS], level_w[LFD_MAX_LEVELS], level_stride[LFD_MAX_LEVELS];
    float level_hi[LFD_MAX_LEVELS]; /* upper end of the level's regression range */
    float score_thr, iou_thr;
    int32_t cap;                /* per-image capacity for candidates and outputs */
    int32_t max_ctas;           /* 0 = default.  > 0: stands in for the SM count the sigmoid multi-class candidate launch is sized from
                                   (at most 8 * max_ctas blocks per image), so its grid-stride loop runs more rounds (tests) */
} lfd_post_cfg;

size_t lfd_postprocess_workspace_bytes(const lfd_post_cfg* cfg);
/* img_w / img_h / resize_scale: device float[N].  Outputs (device): dets float[N][cap][5] = x1,y1,x2,y2,score in
 * score-descending kept order; labels int[N][cap]; src int[N][cap] = point * C + class; count int[N];
 * overflow int[1] set to 1 if an image produced more than cap candidates. */
int lfd_postprocess(const lfd_post_cfg* cfg, const float* cls, const float* reg, const float* img_w, const float* img_h,
                    const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                    int32_t* overflow, lfd_stream stream);

/* multiclass_nms / batched_nms of lfd/model/utils/nms.py:119-220 on explicit (already decoded) boxes.
 * labels_in == NULL: boxes float[n][4] (box_per_class = 0) or float[n][C][4] (1), scores float[n][score_stride]: candidate (row i, class c < C)
 *   when scores[i][c] > score_thr (strict); labels_in != NULL (the batched_nms form): one candidate per row (boxes[i], scores[i], labels_in[i]),
 *   C = number of label values.  Class-aware suppression reproduces the reference's label * (max coordinate + 1) offsets in fp32.
 * Outputs (device): dets float[cap][5] = x1,y1,x2,y2,score in kept (score-descending) order, labels int32[cap], src int32[cap] = row * C +
 * class, count int32[1], overflow int32[1] (1: more than cap candidates). */
size_t lfd_multiclass_nms_workspace_bytes(int cap);
int lfd_multiclass_nms(const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in, int n, int C,
                       float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels, int32_t* src,
                       int32_t* count, int32_t* overflow, lfd_stream stream);

/* Soft-NMS (soft_nms of lfd/model/utils/nms.py:62-116, nms_cfg type 'soft_nms' in batched_nms / multiclass_nms :119-220) in place of the
 * greedy NMS of lfd_postprocess / lfd_multiclass_nms: the same arguments and candidates, plus
 *   method    LFD_SOFT_NMS_LINEAR (score *= 1 - iou when iou > cfg->iou_thr / iou_thr) or LFD_SOFT_NMS_GAUSSIAN (score *= exp(-iou^2 / sigma));
 *             any other value fails with LFD_ERR_INVALID
 *   min_score a reweighted candidate whose score is < min_score is dropped (the selected one never is).
 * One CTA per image runs the reference's loop (nms_cpu.cpp:76-206) over all classes in one array, starting from the candidates in source
 * order (src ascending); the class offsets are those of the greedy path.  Outputs as there, except: rows in selection order and d[4] = the
 * decayed score at selection.  Linear mode is bit-exact with the reference; gaussian mode rounds exp(double) to fp32.
 * Up to 8192 candidates per image live in shared memory, more in the workspace.  No allocation, no host synchronisation. */
enum { LFD_SOFT_NMS_LINEAR = 1, LFD_SOFT_NMS_GAUSSIAN = 2 };
size_t lfd_postprocess_soft_nms_workspace_bytes(const lfd_post_cfg* cfg);
int lfd_postprocess_soft_nms(const lfd_post_cfg* cfg, const float* cls, const float* reg, const float* img_w, const float* img_h,
                             const float* resize_scale, void* workspace, float* dets, int32_t* labels, int32_t* src, int32_t* count,
                             int32_t* overflow, int method, float sigma, float min_score, lfd_stream stream);
size_t lfd_multiclass_soft_nms_workspace_bytes(int cap);
int lfd_multiclass_soft_nms(const float* boxes, int box_per_class, const float* scores, int score_stride, const int32_t* labels_in, int n, int C,
                            float score_thr, float iou_thr, int class_agnostic, int cap, void* workspace, float* dets, int32_t* labels, int32_t* src,
                            int32_t* count, int32_t* overflow, int method, float sigma, float min_score, lfd_stream stream);

size_t lfd_nms_workspace_bytes(int n);
/* dets device float[n][5]; keep device int64[n] (first *n_keep valid, score-descending); n_keep device int32[1]. */
int lfd_nms(const float* dets, int n, float iou_thr, void* workspace, int64_t* keep, int32_t* n_keep, lfd_stream stream);

/* ------------------------------------------------------------------------------------------ training losses */
typedef struct lfd_levels {
    int32_t num_levels;
    int32_t off[LFD_MAX_LEVELS], w[LFD_MAX_LEVELS], stride[LFD_MAX_LEVELS];
    float lo[LFD_MAX_LEVELS], hi[LFD_MAX_LEVELS];   /* regression range of the level */
    float glo[LFD_MAX_LEVELS], ghi[LFD_MAX_LEVELS]; /* gray range (after int() truncation, lfd.py:49-50) */
} lfd_levels;

enum { LFD_ASSIGN_DIST = 0, LFD_ASSIGN_LONGER = 1, LFD_ASSIGN_SHORTER = 2 };

/* gt_boxes device float[N][gmax][4] (x,y,w,h), gt_labels int[N][gmax], gt_count int[N].
 * cls_target float[N][P][C], reg_target float[N][P][4], label int[N][P] (-1 ignore, C background),
 * counters int[2] = {n_pos, n_valid} (zeroed inside). */
int lfd_assign_targets(const lfd_levels* lv, int N, int P, int C, int gmax, int assign_mode, int independent,
                       const float* gt_boxes, const int32_t* gt_labels, const int32_t* gt_count, float* cls_target,
                       float* reg_target, int32_t* label, int32_t* counters, lfd_stream stream);

/* Losses of LFD.get_loss (lfd/model/lfd.py:326-387) and their gradients w.r.t. the network outputs.
 * classification (over the non-gray rows, avg_factor = n_pos + 1): sigmoid focal (FocalLoss), cross entropy over C+1 logits
 * (CrossEntropyLoss), BCE with logits against the soft targets (BCEWithLogitsLoss), quality focal (QualityFocalLoss, beta in `gamma`,
 * quality = the point's maximal centre score); regression (positives, avg_factor = n_pos): -log IoU / GIoU / DIoU / CIoU on the decoded
 * boxes (bbox_mode sigmoid | exp), SmoothL1 / MSE on the raw outputs against the range-normalised targets (bbox_mode independent). */
enum { LFD_CLS_BCE = 2, LFD_CLS_QFL = 3 }; /* continues LFD_CLS_SIGMOID = 0, LFD_CLS_SOFTMAX = 1 */
enum { LFD_REG_IOU = 0, LFD_REG_GIOU = 1, LFD_REG_DIOU = 2, LFD_REG_CIOU = 3, LFD_REG_SMOOTH_L1 = 4, LFD_REG_MSE = 5 };
typedef struct lfd_loss_cfg {
    int32_t N, P, C;
    int32_t cls_mode, bbox_mode, reg_loss;
    float gamma, alpha;          /* focal: gamma, alpha; quality focal: beta in gamma */
    float reg_eps;               /* IoU family eps */
    float smooth_l1_beta;
    float cls_weight, reg_weight;
    int32_t max_ctas;            /* 0 = default.  > 0: stands in for the SM count the two loss launches are sized from (4 * max_ctas blocks
                                    each), so every thread walks more of its grid-stride loop (tests) */
} lfd_loss_cfg;
/* loss_sums double[2] = {sum of element-wise cls loss over valid rows, sum of the regression loss over positives} (zeroed inside);
 * the reference's normalisation is loss = sums[0]/(n_pos+1) + sums[1]/n_pos.  grad_cls / grad_reg (optional) receive
 * d loss / d cls_logits and d loss / d reg with that normalisation and the loss weights applied.  cls_target (N, P, C): the soft
 * targets of lfd_assign_targets, needed by BCE / QFL only (may be NULL otherwise). */
int lfd_detection_loss(const lfd_levels* lv, const lfd_loss_cfg* cfg, const float* cls_logits, const float* reg, const float* cls_target,
                       const float* reg_target, const int32_t* label, const int32_t* counters, float* grad_cls, float* grad_reg,
                       double* loss_sums, lfd_stream stream);

/* enable_classification_weight / enable_regression_weight of the reference's LFD (lfd/model/lfd.py:322-384).  The weight of a positive
 * row is its maximal classification target (the row maximum of cls_target, >= 0.001), and weight_sum is their sum over the batch.
 *   lfd_loss_weight_sum: *weight_sum (device double[1]) = that sum over the rows with 0 <= label < C, in a fixed order (per-block
 *       partials in `workspace`, of lfd_loss_weight_sum_workspace_bytes(cfg) bytes, then one block adds them up; no atomics), so
 *       repeated calls give the same bits.  Reads cfg->N, P, C and max_ctas.  Data-parallel callers sum *weight_sum over their ranks
 *       before the loss, as they do the counters.
 *   lfd_detection_loss_weighted: lfd_detection_loss with the two switches (0 or 1 each; anything else is LFD_ERR_INVALID):
 *       cls_weighted: classification avg_factor = *weight_sum instead of n_pos + 1 (no per-element weight, every cls_mode);
 *       reg_weighted: each positive's regression loss times its weight (loss_sums[1] is then sum w_i * loss_i), avg_factor =
 *       *weight_sum instead of n_pos; without positives the regression loss and its gradient are 0, as unweighted.
 *       reg_weighted needs cls_target and is LFD_ERR_INVALID with SmoothL1 / MSE: there the reference multiplies the (n, 4) element
 *       loss by the (n,) weight, which does not broadcast.
 *   With both switches 0 it is lfd_detection_loss, bit for bit, and weight_sum may be NULL.  A zero *weight_sum (no positives) with
 *   cls_weighted divides by zero, as the reference does: the classification gradients are +-inf (NaN where the element's own is 0). */
size_t lfd_loss_weight_sum_workspace_bytes(const lfd_loss_cfg* cfg);
int lfd_loss_weight_sum(const lfd_loss_cfg* cfg, const float* cls_target, const int32_t* label, void* workspace, double* weight_sum,
                        lfd_stream stream);
int lfd_detection_loss_weighted(const lfd_levels* lv, const lfd_loss_cfg* cfg, const float* cls_logits, const float* reg,
                                const float* cls_target, const float* reg_target, const int32_t* label, const int32_t* counters,
                                float* grad_cls, float* grad_reg, double* loss_sums, int cls_weighted, int reg_weighted,
                                const double* weight_sum, lfd_stream stream);

/* Element-wise box losses of the stand-alone IoULoss / GIoULoss / DIoULoss / CIoULoss modules (lfd/model/losses/iou_loss.py:105-283,
 * before the reduction): pred / target float[n][4] xyxy, kind = LFD_REG_IOU .. LFD_REG_CIOU; loss float[n], grad_pred float[n][4]
 * (d loss_i / d pred_i, optional). */
int lfd_box_loss(int kind, const float* pred, const float* target, int n, float eps, float* loss, float* grad_pred, lfd_stream stream);

int lfd_sigmoid_focal_loss_forward(const float* logits, const int64_t* targets, int M, int C, float gamma, float alpha,
                                   float* losses, lfd_stream stream);
int lfd_sigmoid_focal_loss_backward(const float* logits, const int64_t* targets, const float* d_losses, int M, int C,
                                    float gamma, float alpha, float* d_logits, lfd_stream stream);

/* ------------------------------------------------------------------------------------------ training step
 * What the reference gets from autograd over its conv / BatchNorm2d / GroupNorm / ReLU modules in train mode
 * (lfd/model/backbone/lfd_resnet.py:96-154,354-473, neck/simple_neck.py:35-74, head/lfd_head.py:85-185), i.e. the body of
 * Executor.train's `model(x)` ... `loss.backward()` (lfd/execution/executor.py:185-214), and from
 * clip_grad_norm_ + torch.optim.SGD.step (lfd/execution/hooks/optimizer_hook.py:21-36).
 *
 * A training plan is an ordered list of lfd_top ops over ONE workspace (bf16 NHWC activations, their bf16 gradients, fp64
 * statistics, packed bf16 weight operands, fp32 weight-gradient staging); parameters, their gradients and the BatchNorm
 * running statistics are the caller's fp32 device tensors, referenced by absolute pointers that stay fixed for the plan's
 * lifetime.  off[] are byte offsets into the workspace (-1 = unused), ptr[] absolute device pointers:
 *
 *   kind             off[0]   off[1]  off[2]  off[3]   off[4]     off[5]   off[6]  off[7]   ptr[0..3]
 *   PACK             -        -       -       -        -          -        -       -        table (lfd_pack_desc[n_desc], device)
 *   STEM0 / CONV     in       out     res     gnstats  packed w   -        -       -        -          (as lfd_op; STEM0 reads the run-time input;
 *                                                                                                        CONV is also the data-gradient conv: in = dz
 *                                                                                                        (zero-inserted for stride 2), packed w = PACK_CONV_DGRAD,
 *                                                                                                        res = out accumulates into an existing gradient)
 *   BN_STATS         z        -       -       sums     -          -        -       -        -
 *   BN_APPLY         z        y       res     sums     -          -        -       -        gamma, beta, running_mean, running_var
 *   GN_APPLY         in       out     -       gnstats  -          -        -       -        gamma, beta
 *   HEAD_FINAL       raw      -       -       gnstats  staging    -        -       -        gamma, beta, cls out, reg out
 *   HEAD_FINAL_BWD   raw      dact    -       gnstats  staging    dstage   dscale  -        gamma, beta, grad cls, grad reg
 *   NORM_BWD_REDUCE  dy       y       z       fsums    bsums      -        -       -        gamma, beta, -, -, running_mean, running_var (frozen)
 *   NORM_BWD_APPLY   dy       y       z       fsums    bsums      dz       dz_up   dres     gamma, beta, dgamma, dbeta, running_mean, running_var (frozen)
 *   WGRAD            x        dz      -       -        -          dstage   -       -        -
 *   WGRAD_STEM       x27      dz      -       -        -          dstage   -       -        -          (x = the run-time input image; x27 >= 0: scratch
 *                                                                                                        bf16 [N][Ho][Wo][32] for the im2col + tensor-core path, dstage then has 32 rows;
 *                                                                                                        x27 = -1 or impl = SIMT: the SIMT kernel, 27 rows;
 *                                                                                                        Cin = 1 (gray): 9 rows [tap][co], x27 zero past column 9)
 *   UNPACK           -        -       -       -        -          -        -       -        table (lfd_unpack_desc[n_desc], device)
 *   ZERO             begin    bytes   -       -        -          -        -       -        -          (cudaMemsetAsync of a workspace region)
 *   INFER            in       out     res     ds_out   -          -        -       -        op (const lfd_op*, HOST memory, read by lfd_train_plan_create)
 *                                                                                                        one inference op inside the training plan: STEM0 / CONV
 *                                                                                                        (with tail and fused shortcut) / STEM4, bf16, no GroupNorm
 *                                                                                                        statistics.  Its weight / shift pointers are the caller's
 *                                                                                                        packed operands (lfd_op conventions); off[0..3] replace the
 *                                                                                                        op's in_off / out_off / res_off / ds_out_off, max_ctas its
 *                                                                                                        max_ctas.  The frozen backbone prefix of a fine-tuning step
 *                                                                                                        (BatchNorm folded, no statistics, no backward) runs on it.
 *
 * head staging (fp32): w[n_out][C] (bf16-rounded values), scale[n_out], shift[n_out] = bias * scale, bias[n_out];
 * head dstage (fp32): dW[n_out][C], dbias[n_out]; dscale (fp32): the level's Scale gradient [1].  wgrad dstage (fp32): [ksize^2][Cin][Cout].
 * BatchNorm statistics are taken over the STORED bf16 conv output; GroupNorm ones come from the conv epilogue as in inference. */
enum { LFD_TOP_PACK = 0, LFD_TOP_STEM0 = 1, LFD_TOP_CONV = 2, LFD_TOP_BN_STATS = 3, LFD_TOP_BN_APPLY = 4, LFD_TOP_GN_APPLY = 5,
       LFD_TOP_HEAD_FINAL = 6, LFD_TOP_HEAD_FINAL_BWD = 7, LFD_TOP_NORM_BWD_REDUCE = 8, LFD_TOP_NORM_BWD_APPLY = 9, LFD_TOP_WGRAD = 10,
       LFD_TOP_WGRAD_STEM = 11, LFD_TOP_UNPACK = 12, LFD_TOP_ZERO = 13, LFD_TOP_INFER = 14 };
enum { LFD_WGRAD_UMMA = 0, LFD_WGRAD_SIMT = 1 }; /* SIMT = cross-check kernel, validation only */

typedef struct lfd_top {
    int32_t kind;
    int32_t N, H, W, Cin, Ho, Wo, Cout, ksize, stride;
    int32_t relu, groups, cc, n_cls, n_reg, point_off, P, cls_stride;
    int32_t accumulate;   /* NORM_BWD_APPLY: dres += g instead of dres = g */
    int32_t upH, upW;     /* NORM_BWD_APPLY with dz_up: size of the zero-inserted gradient map (the stride-2 conv's input size) */
    int32_t n_desc, max_n;/* PACK / UNPACK: table entries, largest element count of an entry */
    int32_t impl;         /* WGRAD: LFD_WGRAD_UMMA | LFD_WGRAD_SIMT; CONV: LFD_CONV_UMMA | LFD_CONV_SIMT */
    int32_t frozen;       /* BN_APPLY / NORM_BWD_* (BatchNorm): the module is in eval mode -- normalise with the running statistics
                             (ptr[2..3] of BN_APPLY, ptr[4..5] of NORM_BWD_*), do not update them, no batch-statistics terms in dz */
    int32_t branch, wait_mask; /* as in lfd_op: branch 0 = the caller's stream, ops of branch b > 0 run on side stream b (forked after the
                                  main-stream op preceding the branch's first op, joined at the end of the plan); wait_mask bit w = wait for
                                  everything enqueued so far on branch w.  The per-level neck / head chains of the forward and of the
                                  backward are independent of the backbone's smaller stages: lfd/_train.py derives the masks from the
                                  read / write / accumulate role of every off[] entry. */
    int32_t max_ctas;  /* CONV / WGRAD: upper bound on the persistent CTAs (0 = all), as in lfd_op.  BN_* / GN_APPLY / HEAD_FINAL* /
                          NORM_BWD_* / WGRAD_STEM size their grids from the SM count: max_ctas > 0 stands in for it (so a kernel with
                          k blocks per SM gets k * max_ctas blocks) and every thread walks more of its grid-stride loop */
    float eps, momentum;
    int64_t off[8];
    const void* ptr[6];
    /* STEM0 / WGRAD_STEM on a LFD_INPUT_U8_NHWC image: the input transform, as in lfd_op (all zero = simple_normalize on BGR).  The forward's
     * STEM0 and the backward's WGRAD_STEM of one step must carry the same one. */
    int32_t in_swap_rb;
    float in_mean[3];
    float in_scale[3];
    int32_t pad2_;
} lfd_top;

/* entries of the PACK / UNPACK tables (device memory, absolute pointers) */
enum { LFD_PACK_CONV_FWD = 0, LFD_PACK_CONV_DGRAD = 1, LFD_PACK_STEM = 2, LFD_PACK_ROUND_F32 = 3, LFD_PACK_SCALE_SHIFT = 4 };
typedef struct lfd_pack_desc {
    int32_t kind;
    int32_t Cout, Cin, k, cc; /* conv: OIHW dims of the fp32 parameter, cc = channel chunk of the packed operand (lfd_conv_query) */
    int32_t n;                /* destination elements */
    const float* src;         /* the parameter; SCALE_SHIFT: the bias [n] (or NULL) */
    const float* src2;        /* SCALE_SHIFT: the level's scalar Scale parameter (or NULL = 1) */
    void* dst;                /* CONV_FWD: bf16 [Cin/cc][k*k][cc/8][Cout][8]; CONV_DGRAD: the transposed conv's operand
                                 bf16 [Cout/cc][k*k][cc/8][Cin][8] with flipped taps; STEM: bf16 [kh][2][Cout][8] of a
                                 [Cout][Cin][3][3] weight, Cin = 3 or 1 (gray: channel-0 lanes, zeros elsewhere);
                                 ROUND_F32: fp32 copy holding bf16-rounded values; SCALE_SHIFT: scale[n] */
    void* dst2;               /* SCALE_SHIFT: shift[n] = bias * scale */
    void* dst3;               /* SCALE_SHIFT: bias[n] */
} lfd_pack_desc;
enum { LFD_UNPACK_CONV = 0, LFD_UNPACK_ADD = 1 };
typedef struct lfd_unpack_desc {
    int32_t kind;
    int32_t Cout, Cin, kk;    /* UNPACK_CONV: staging [kk][Cin][Cout] -> gradient [Cout][Cin][kk] (+=) */
    int32_t n;                /* elements */
    int32_t pad_;
    const float* src;
    float* dst;               /* dst[i] += ... */
} lfd_unpack_desc;

typedef struct lfd_train_plan lfd_train_plan;
int lfd_train_plan_create(const lfd_top* ops, int n_ops, int64_t workspace_bytes, lfd_train_plan** out);
int lfd_train_plan_destroy(lfd_train_plan* plan);
int lfd_train_plan_num_ops(const lfd_train_plan* plan);
/* Enqueues every op in order on `stream`.  use_graph != 0: captured into a CUDA graph on first use per (input, workspace). */
int lfd_train_plan_run(lfd_train_plan* plan, const void* input, int input_format, void* workspace, int use_graph, lfd_stream stream);
/* one eager pass with a CUDA event pair around every op (synchronises): ms_per_op float[lfd_train_plan_num_ops()] (host) */
int lfd_train_plan_profile(lfd_train_plan* plan, const void* input, int input_format, void* workspace, float* ms_per_op, lfd_stream stream);
/* run a single op (tests) */
int lfd_run_top(const lfd_top* op, const void* input, int input_format, void* workspace, lfd_stream stream);

/* sqnorm double[1] (device) = sum of grads^2 (zeroed inside) -- the total_norm^2 of clip_grad_norm_(norm_type=2) */
int lfd_grad_sqnorm(const float* grads, int64_t n, double* sqnorm, lfd_stream stream);
/* torch.optim.SGD.step over flat fp32 buffers, preceded by the clip: g *= grad_scale; if max_norm > 0:
 * g *= min(1, max_norm / (grad_scale * sqrt(*sqnorm) + 1e-6)) (written back, like clip_grad_norm_); g += weight_decay * p;
 * buf = momentum * buf + (1 - dampening) * g; p -= lr * (nesterov ? g + momentum * buf : buf).  momentum_buf may be NULL. */
int lfd_sgd_step(float* params, float* grads, float* momentum_buf, int64_t n, float lr, float momentum, float dampening,
                 float weight_decay, int nesterov, float max_norm, float grad_scale, const double* sqnorm, lfd_stream stream);

/* ------------------------------------------------------------------------------------------ training input batch
 * One launch builds a batch of training crops from uint8 source windows, the pixel work of the reference's data loader
 * (RandomBBoxCropRegionSampler & co. lfd/data_pipeline/sampler/region_sampler.py, crop_from_image :280-300, the gray -> 3 channel
 * tile data_loader.py:122-124, HorizontalFlip / BGR2RGB / Normalize, _image_batch_postprocess data_loader.py:68-83), and the
 * 1-channel batches of gray models (num_input_channels = 1):
 *   R = cv2.resize(S, (0, 0), fx = s, fy = s) (INTER_LINEAR on uint8, bit-exact; INTER_AREA when 1/s == 2; a copy when the size is kept),
 *   crop[y][x] = R[crop_y + y][crop_x + x] inside R, 0 outside; out[y][x] = crop[y][out_w - 1 - x] when flipped.
 * R is never materialised. */
enum { LFD_RESIZE_COPY = 0, LFD_RESIZE_LINEAR = 1, LFD_RESIZE_AREA2 = 2 };
enum { LFD_INPUT_OUT_U8_NHWC = 0, LFD_INPUT_OUT_F32_NCHW = 1, LFD_INPUT_OUT_U8_GRAY = 2, LFD_INPUT_OUT_F32_GRAY = 3 };
typedef struct lfd_input_desc {
    int64_t src_off;          /* byte offset in src of the window's first pixel */
    double inv_scale;         /* 1 / s */
    int32_t pitch;            /* bytes between window rows (>= win_w * channels) */
    int32_t channels;         /* 1 (gray) or 3 (BGR) */
    int32_t win_x, win_y;     /* window origin inside the full source image */
    int32_t win_w, win_h;     /* window size; it holds every source pixel the crop reads (0 x 0 when the crop misses R) */
    int32_t src_w, src_h;     /* full source image size */
    int32_t dw, dh;           /* size of R: round-half-even(src_w * s), round-half-even(src_h * s) */
    int32_t mode;             /* LFD_RESIZE_*: COPY when (dw, dh) == (src_w, src_h), AREA2 when 1/s == 2 exactly, else LINEAR */
    int32_t crop_x, crop_y;   /* crop origin in R's coordinates (may be negative or beyond R) */
    int32_t out_w, out_h;     /* crop size, <= W, H */
    int32_t flip;             /* 1: horizontal flip of the crop */
} lfd_input_desc;
/* descs: device lfd_input_desc[n]; src: device bytes holding every window.
 * out_mode LFD_INPUT_OUT_U8_NHWC: out uint8 [n, H, W, 3]; LFD_INPUT_OUT_F32_NCHW: out float32 [n, 3, H, W] with
 * out = (v - mean[c]) * scale[c] (albumentations' Normalize: mean[c] = mean * max_pixel, scale[c] = float32(1 / (std * max_pixel))).
 * Pixels outside an image's out_w x out_h are 0 in both modes (the zero padding of mixed-size batches).  swap_rb: BGR -> RGB; a
 * 1-channel source is replicated to 3.  mean / scale: host float[3], unused in the uint8 mode.  W <= 6144.
 * The gray modes, for 1-channel models: LFD_INPUT_OUT_U8_GRAY: out uint8 [n, H, W]; LFD_INPUT_OUT_F32_GRAY: out float32 [n, 1, H, W]
 * with out = (v - mean[0]) * scale[0].  A gray source is read as it is; a BGR source is converted first, as cv2.cvtColor(S,
 * COLOR_BGR2GRAY) does on uint8 ((3735 B + 19235 G + 9798 R + 16384) >> 15), and R is cv2.resize of that gray image.  Padding is 0
 * as above.  swap_rb != 0 with a gray mode is LFD_ERR_INVALID; only mean[0] and scale[0] are read.
 * Every argument is checked before anything is enqueued: an invalid call writes nothing. */
int lfd_input_batch(const lfd_input_desc* descs, int n, const uint8_t* src, void* out, int out_mode, int swap_rb, int H, int W,
                    const float* mean, const float* scale, lfd_stream stream);

/* ------------------------------------------------------------------------------------------ model files
 * A model file (written by lfd/_engine.py InferencePlan.export, lfd.deployment.export_model) is one inference plan with its weights and
 * its post-process, so that a program that links only this library and cudart runs a trained model: the same kernels, launches and
 * results as the Python plan it was exported from.  Little-endian; DESIGN.md "Model files" has the layout:
 *   header   48 bytes: "LFDMODEL", format version (LFD_MODEL_FORMAT_VERSION), lfd_abi_version(), target "sm_90a", sizeof(lfd_op),
 *            sizeof(lfd_post_cfg), payload bytes, CRC-32 of the payload (zlib's), a zero word
 *   payload  the plan (capacity, P, cls_channels, dtype, conv_impl, op count, statistics region, workspace bytes, input transform,
 *            NMS type and Soft-NMS arguments, blob sizes; 120 bytes), the lfd_post_cfg, the lfd_op records, per op (index of the op that
 *            produces its input or -1, head level or -1), the fp32 blob, the 16-bit blob.
 * In an lfd_op record every pointer field holds ((blob + 1) << 56) | byte offset into the blob (blob 0 = fp32, 1 = 16-bit), or 0 for NULL.
 *
 * lfd_engine_open validates the whole file before keeping it (host only, no device needed): header fields, struct sizes, checksum, sizes
 * and bounds of the plan, every op (kind, geometry as lfd_plan_create and the wgmma kernel's configuration take it, the image op at the
 * capacity, the input transform on the image op only and equal to the plan's, branch, every workspace range against the workspace, every
 * (blob, offset) range against its blob, the producer / level table with each op reading an output of its producer of matching size and
 * channels) and the post-process configuration.  A file it refuses gives LFD_ERR_INVALID (or
 * LFD_ERR_UNSUPPORTED: another format version, ABI or target, a SIMT plan) and an lfd_last_error() that names the field. */
#define LFD_MODEL_FORMAT_VERSION 1
typedef struct lfd_engine lfd_engine;
typedef struct lfd_engine_desc {
    int32_t N, H, W;              /* capacity: frames of up to H x W, N per call */
    int32_t P, cls_channels;      /* points and classification channels at the capacity */
    int32_t num_classes, dtype, n_ops;
    int32_t cap;                  /* detections per image (dets / labels rows) */
    int32_t soft_nms;             /* 0 greedy NMS, 1 Soft-NMS */
    int64_t weights_bytes;        /* device buffer for lfd_engine_bind's weights */
    int64_t workspace_bytes;      /* forward workspace, including the engine's own cls / reg region */
    int64_t post_workspace_bytes; /* post-process workspace */
} lfd_engine_desc;
int lfd_engine_open(const void* bytes, size_t n, lfd_engine** out);
int lfd_engine_close(lfd_engine* engine);
int lfd_engine_info(const lfd_engine* engine, lfd_engine_desc* out);
/* op i of the file as stored (pointer fields in the (blob, offset) encoding above); src_op / level may be NULL */
int lfd_engine_op(const lfd_engine* engine, int i, lfd_op* op, int32_t* src_op, int32_t* level);
/* Copies the weights into `weights` (asynchronously on `stream`: the caller's later work on `stream` sees them), resolves the ops'
 * pointers and creates the plan (lfd_plan_create: needs the device).  The buffers stay the caller's and must outlive the engine or the
 * next bind; a buffer smaller than lfd_engine_info reports fails with LFD_ERR_CAPACITY, one not aligned to 256 bytes (what cudaMalloc
 * returns; the weights are bulk-copied and the activations reached through TMA) with LFD_ERR_INVALID, before anything is copied.  Like
 * lfd_plan_*, the engine's plan keeps its side streams, events and CUDA graphs, and on the first frame below the capacity a device
 * geometry table and a pinned staging ring for it (lfd_plan_forward_extent); everything sized by the model is in the caller's buffers. */
int lfd_engine_bind(lfd_engine* engine, void* weights, size_t weights_bytes, void* workspace, size_t workspace_bytes, void* post_workspace,
                    size_t post_workspace_bytes, lfd_stream stream);
/* One batch: lfd_plan_forward_extent on N frames of h x w (<= the capacity) in the capacity layout of input_format (see
 * lfd_plan_forward_extent), then lfd_postprocess / lfd_postprocess_soft_nms with image size w x h and resize scale 1.  The geometry table
 * of a smaller frame is derived from the file.  Outputs (device): dets float[N][cap][5] = x1, y1, x2, y2, score; labels int32[N][cap];
 * count int32[N + 1] (count[N] = 1: an image had more than cap candidates).  cls_out float[N][P][cls_channels] / reg_out float[N][P][4]
 * receive the frame's network outputs (laid out as lfd_plan_forward_extent lays them out), or are NULL: the engine's region of the
 * workspace holds them then.  use_graph: the forward is replayed as a CUDA graph (lfd_plan_forward).  No host synchronisation; every
 * argument is checked before anything is enqueued.  The calls of one engine share its workspaces: the caller orders them (one stream,
 * or events between streams), as for one lfd_plan. */
int lfd_engine_detect(lfd_engine* engine, const void* input, int input_format, int h, int w, float* dets, int32_t* labels, int32_t* count,
                      float* cls_out, float* reg_out, int use_graph, lfd_stream stream);
int lfd_engine_num_launches(const lfd_engine* engine); /* lfd_plan_num_launches of the bound plan (0 before lfd_engine_bind) */

#ifdef __cplusplus
}
#endif
#endif /* LFD_B200_H_ */
