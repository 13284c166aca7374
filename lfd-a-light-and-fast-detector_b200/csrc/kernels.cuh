// kernels.cuh -- parameter blocks and launchers of the non-GEMM kernels (internal, not part of the C-ABI).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "image.cuh"

namespace lfd {

static constexpr int kMaxLevels = 8;

struct Stem0Params {
    ImageIn img;
    __nv_bfloat16* out;        // bf16 NHWC
    const __nv_bfloat16* w;    // packed [kh][2][Cout][8]: element (kh, kc, n, j) = weight (n, ci = j % 4, kh, kw = 2 kc + j / 4), 0 for kw = 3 or ci = 3
    const float* shift;        // fp32 [Cout] or null (BatchNorm scale is folded into w); applied as bf16
    int N, Ho, Wo, Cout, relu;
    int f16;                   // 16-bit type of weights / output: 0 = bf16, 1 = fp16
};
cudaError_t stem0_launch(const Stem0Params& p, cudaStream_t st);

struct GnApplyParams {
    const __nv_bfloat16* in;
    __nv_bfloat16* out;
    const double* stats;       // [N][groups][2]
    const float* gamma;
    const float* beta;
    int N, HW, C, groups;
    float eps;
    int f16;
    unsigned long long* tl;    // debugging time-line slot or null
    // null: all HW pixels.  Otherwise device int2 (h, w), read when the kernel starts: only the top-left h x w of the map (row pitch W) is
    // valid -- the GroupNorm count is h * w; the first h rows are written (the pixels right of w are outside the valid extent)
    const int* ext = nullptr;
    int W = 0;
};
cudaError_t gn_apply_launch(const GnApplyParams& p, int num_sms, cudaStream_t st);

struct HeadFinalParams {
    const __nv_bfloat16* in;   // pre-GN tower output [N][HW][C]
    const double* stats;
    const float* gamma;
    const float* beta;
    const float* w;            // [n_out][C] fp32 holding bf16-rounded values
    const float* scale;        // [n_out]
    const float* shift;        // [n_out]
    float* cls;                // (N, P, cls_stride) or null
    float* reg;                // (N, P, 4) or null
    int N, HW, C, groups, n_out, n_cls, P, point_off, cls_stride;
    float eps;
    int f16;
    unsigned long long* tl;    // debugging time-line slot or null
    // null: all HW pixels.  Otherwise device int[6] (h, w, -, -, point_off, P), read when the kernel starts: the top-left h x w of the map
    // (row pitch W) is valid; pixel (y, x) goes to point point_off + y * w + x of a (N, P, .) output -- the layout of a plan built for the frame
    const int* ext = nullptr;
    int W = 0;
};
cudaError_t head_final_launch(const HeadFinalParams& p, int num_sms, cudaStream_t st);

struct LevelTable {
    int num_levels;
    int off[kMaxLevels], w[kMaxLevels], stride[kMaxLevels];
    float lo[kMaxLevels], hi[kMaxLevels], glo[kMaxLevels], ghi[kMaxLevels];
};

struct PostParams {
    const float* cls;          // (N, P, cls_stride)
    const float* reg;          // (N, P, 4)
    const float* img_w;        // [N] clamp bounds (resized width / height), lfd.py:440-441
    const float* img_h;
    const float* resize_scale; // [N]
    int N, P, C, cls_stride, cls_mode, bbox_mode, num_levels, cap;
    int level_off[kMaxLevels], level_w[kMaxLevels], level_stride[kMaxLevels];
    float level_hi[kMaxLevels];
    float score_thr;
    float* cand_box;           // [N][cap][4]
    float* cand_score;         // [N][cap]
    int* cand_src;             // [N][cap]
    int* cand_count;           // [N]
};
cudaError_t candidates_launch(const PostParams& p, int num_sms, cudaStream_t st);

struct NmsParams {
    const float* cand_box;
    const float* cand_score;
    const int* cand_src;
    const int* cand_count;
    uint8_t* scratch;
    size_t scratch_stride;
    int cap, cap_pow2, C, class_agnostic;
    float iou_thr;
    float* out_dets;           // [N][cap][5]
    int* out_label;            // [N][cap]
    int* out_src;              // [N][cap]
    int* out_count;            // [N]
    int* overflow;             // single flag
};
size_t nms_scratch_stride(int cap, int cap_pow2);
cudaError_t box_candidates_launch(const float* boxes, int box_per_class, const float* scores, int score_stride, const int* labels_in, int n, int C,
                                  float score_thr, int cap, float* cand_box, float* cand_score, int* cand_src, int* cand_count, cudaStream_t st);
cudaError_t nms_launch(const NmsParams& p, int n_images, cudaStream_t st);
// Soft-NMS on the same candidates, scratch and outputs (nms.iou_thr = the linear threshold; outputs in selection order, scores decayed)
struct SoftNmsParams {
    NmsParams nms;
    int method;                // 1 linear, 2 gaussian (the reference's codes)
    float sigma, min_score;
};
cudaError_t soft_nms_launch(const SoftNmsParams& p, int n_images, cudaStream_t st);

struct AssignParams {
    LevelTable lv;
    const float* gt_boxes;     // [N][gmax][4] xywh
    const int* gt_labels;      // [N][gmax]
    const int* gt_count;       // [N]
    int N, P, C, gmax, assign_mode, independent;
    float* cls_target;         // [N][P][C]
    float* reg_target;         // [N][P][4]
    int* label;                // [N][P]  -1 ignore, C background
    int* counters;             // [0] n_pos, [1] n_valid  (zeroed by the caller)
};
cudaError_t assign_targets_launch(const AssignParams& p, cudaStream_t st);

cudaError_t focal_forward_launch(const float* logits, const long long* targets, int M, int C, float gamma, float alpha,
                                 float* losses, cudaStream_t st);
cudaError_t focal_backward_launch(const float* logits, const long long* targets, const float* d_losses, int M, int C,
                                  float gamma, float alpha, float* d_logits, cudaStream_t st);

struct ClsLossParams {
    const float* logits;       // (N, P, C')
    const float* cls_target;   // (N, P, C) soft targets (BCE / QFL only)
    const int* label;
    const int* counters;
    float* grad;               // (N, P, C') or null
    double* loss_sum;          // zeroed by the caller
    int N, P, C, cls_mode;     // 0 sigmoid focal, 1 cross entropy (C+1 logits), 2 BCE-with-logits on the soft targets, 3 quality focal (beta = gamma)
    float gamma, alpha, loss_weight;
    int weighted;              // 1: avg_factor = *weight_sum (the sum of the positives' weights) instead of n_pos + 1
    const double* weight_sum;
};
cudaError_t cls_loss_launch(const ClsLossParams& p, int num_sms, cudaStream_t st);
// sum over the positive rows (0 <= label < C) of the row maximum of cls_target, in a fixed order: one partial per block of
// loss_weight_partials_kernel (blocks of them, into `partials`), then one block adds the partials in index order into *weight_sum
int loss_weight_blocks(int num_sms);
cudaError_t loss_weight_sum_launch(const float* cls_target, const int* label, size_t rows, int C, int num_sms, double* partials,
                                   double* weight_sum, cudaStream_t st);

struct RegLossParams {
    LevelTable lv;
    const float* reg;          // (N, P, 4) raw outputs
    const float* reg_target;
    const int* label;
    const int* counters;
    float* grad;
    double* loss_sum;
    int N, P, C, bbox_mode;    // 0 sigmoid * range, 1 exp, 2 independent (raw outputs against targets / range)
    int loss_kind;             // 0 IoU (-log), 1 GIoU, 2 DIoU, 3 CIoU, 4 SmoothL1, 5 MSE (4, 5: bbox_mode 2 only)
    float eps, loss_weight, beta;
    int weighted;              // 1: each positive's loss times its weight (row maximum of cls_target), avg_factor = *weight_sum
    const double* weight_sum;
    const float* cls_target;   // (N, P, C), read when weighted
};
cudaError_t iou_loss_launch(const RegLossParams& p, int num_sms, cudaStream_t st);
// element-wise IoU-family loss (kind 0..3) + d loss / d pred on explicit box pairs
cudaError_t box_loss_launch(int kind, const float* pred, const float* target, int n, float eps, float* loss, float* grad, cudaStream_t st);

// input.cu: descs = device lfd_input_desc[n] (include/lfd_b200.h, lfd_input_batch)
cudaError_t input_batch_launch(const void* descs, int n, const uint8_t* src, void* out, int out_mode, int swap_rb, int H, int W,
                               const float* mean, const float* scale, cudaStream_t st);

}  // namespace lfd
