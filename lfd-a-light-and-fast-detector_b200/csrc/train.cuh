// train.cuh -- parameter blocks and launchers of the training-side kernels (internal, not part of the C-ABI).
//
// Training replaces, for the LFD hot path, what the reference gets from autograd over nn.Conv2d / nn.BatchNorm2d /
// nn.GroupNorm / ReLU in train mode (lfd/model/backbone/lfd_resnet.py:96-154,354-473, neck/simple_neck.py:35-74,
// head/lfd_head.py:85-185) plus torch.optim.SGD + clip_grad_norm_ (lfd/execution/hooks/optimizer_hook.py:21-36).
// Activations and their gradients are bf16 NHWC, statistics and weight gradients fp32 / fp64.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

#include "../../include/lfd_b200.h"
#include "kernels.cuh"

namespace lfd {

// ---------------------------------------------------------------------------------------------------
// parameter staging: fp32 master parameters -> the operand formats of the kernels (and back for the gradients)
// ---------------------------------------------------------------------------------------------------
enum { PACK_CONV_FWD = LFD_PACK_CONV_FWD, PACK_CONV_DGRAD = LFD_PACK_CONV_DGRAD, PACK_STEM = LFD_PACK_STEM, PACK_ROUND_F32 = LFD_PACK_ROUND_F32,
       PACK_SCALE_SHIFT = LFD_PACK_SCALE_SHIFT };
typedef lfd_pack_desc PackDesc;     // one entry of the device-side table (include/lfd_b200.h)
cudaError_t pack_launch(const PackDesc* table, int n_desc, int max_n, cudaStream_t st);

enum { UNPACK_CONV = LFD_UNPACK_CONV, UNPACK_ADD = LFD_UNPACK_ADD };
typedef lfd_unpack_desc UnpackDesc;
cudaError_t unpack_launch(const UnpackDesc* table, int n_desc, int max_n, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------
// BatchNorm, training mode (batch statistics): z = conv(x) stored as bf16, statistics over the stored values
// ---------------------------------------------------------------------------------------------------
struct BnStatsParams {
    const __nv_bfloat16* z;    // [M][C]
    double* sums;              // [C][2] (sum, sum of squares); zeroed by the caller
    long long M;
    int C;
};
cudaError_t bn_stats_launch(const BnStatsParams& p, int num_sms, cudaStream_t st);

struct BnApplyParams {
    const __nv_bfloat16* z;
    const __nv_bfloat16* res;  // optional residual (added before the ReLU)
    __nv_bfloat16* y;
    const double* sums;
    const float* gamma;
    const float* beta;
    float* running_mean;       // optional: updated with `momentum` (unbiased variance), like nn.BatchNorm2d
    float* running_var;
    long long M;
    int C, relu;
    int frozen;                // 1: normalise with the running statistics and leave them alone (a BatchNorm2d in eval mode inside a training step)
    float eps, momentum;
};
cudaError_t bn_apply_launch(const BnApplyParams& p, int num_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------
// normalisation backward (BatchNorm: groups == 0, GroupNorm: groups == 16 with 8 channels per group), two phases
// ---------------------------------------------------------------------------------------------------
struct NormBwdParams {
    const __nv_bfloat16* dy;   // gradient w.r.t. the layer output (after the ReLU)
    const __nv_bfloat16* y;    // BatchNorm: the stored output (ReLU mask = y > 0); GroupNorm: null (the mask is recomputed)
    const __nv_bfloat16* z;    // the stored conv output the normalisation read
    const double* fsums;       // forward statistics: BN [C][2], GN [N][groups][2]
    double* bsums;             // backward sums: [C][2] = (sum g, sum g * zhat) (+ GN: [N][groups][2] = (sum g*gamma, sum g*gamma*zhat) behind it)
    const float* gamma;
    const float* beta;
    __nv_bfloat16* dz;         // gradient w.r.t. z (compact)
    __nv_bfloat16* dz_up;      // optional: the same, zero-inserted to [N][upH][upW][C] (dgrad of a stride-2 conv = stride-1 conv on this)
    __nv_bfloat16* dres;       // optional: g = dy * mask, the gradient of the residual input
    float* dgamma;             // parameter gradients (+=)
    float* dbeta;
    int N, H, W, C, groups, relu;
    int upH, upW;
    int dres_accumulate;       // 1: dres += g
    int frozen;                // BatchNorm in eval mode: statistics = running_mean / running_var, no batch-statistics terms in dz
    const float* running_mean;
    const float* running_var;
    float eps;
};
cudaError_t norm_bwd_reduce_launch(const NormBwdParams& p, int num_sms, cudaStream_t st);
cudaError_t norm_bwd_apply_launch(const NormBwdParams& p, int num_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------
// head final backward: gradients of the final 1x1 convs (+ Scale) and of the tower activation
// ---------------------------------------------------------------------------------------------------
struct HeadFinalBwdParams {
    const __nv_bfloat16* raw;  // pre-GN tower output [N][HW][C]
    const double* stats;       // forward GN statistics
    const float* gamma;
    const float* beta;
    const float* w;            // staging: [n_out][C] (bf16-rounded values), then scale[n_out], shift[n_out], bias[n_out]
    const float* gcls;         // (N, P, cls_stride) or null
    const float* greg;         // (N, P, 4) or null
    __nv_bfloat16* dact;       // gradient w.r.t. the post-GN/ReLU activation [N][HW][C]
    float* dstage;             // [n_out][C] weight gradients, [n_out] bias gradients (+=, atomics; shared by the levels of a shared head)
    float* dscale;             // [1] gradient of the level's Scale parameter (+=) or null
    int N, HW, C, groups, n_out, n_cls, P, point_off, cls_stride;
    float eps;
};
cudaError_t head_final_bwd_launch(const HeadFinalBwdParams& p, int num_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------
// weight gradients
// ---------------------------------------------------------------------------------------------------
struct WgradGeom { int N, H, W, Cin, Ho, Wo, Cout, ksize, stride; };
// wgmma kernel (wgrad_umma.cu): dstage[tap][Cin][Cout] += sum over pixels x_tap[pixel][ci] * dz[pixel][co]
int wgrad_umma_supported(const WgradGeom& g);
cudaError_t wgrad_umma_launch(const WgradGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dz, float* dstage, int num_sms, cudaStream_t st);
// SIMT cross-check (validation only)
cudaError_t wgrad_simt_launch(const WgradGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dz, float* dstage, cudaStream_t st);
// the stem conv: the raw image (image.cuh), normalised + rounded to bf16 like the forward does
// im2col of the stem conv's input for the tensor-core path: X27 bf16 [N][Ho][Wo][32] (27 (tap, ci) values + 5 zeros per output pixel)
cudaError_t stem_im2col_launch(const WgradGeom& g, const ImageIn& img, __nv_bfloat16* x27, int num_sms, cudaStream_t st);
cudaError_t wgrad_stem_launch(const WgradGeom& g, const ImageIn& img, const __nv_bfloat16* dz, float* dstage, int num_sms, cudaStream_t st);

// ---------------------------------------------------------------------------------------------------
// optimizer: clip_grad_norm_ + SGD(momentum, weight decay) over flat fp32 buffers
// ---------------------------------------------------------------------------------------------------
cudaError_t sqnorm_launch(const float* g, long long n, double* out, int num_sms, cudaStream_t st);   // *out += sum g^2
struct SgdParams {
    float* p;
    float* g;
    float* m;                  // momentum buffer (zero-initialised) or null
    long long n;
    float lr, momentum, dampening, weight_decay;
    int nesterov;
    float max_norm;            // > 0: gradients are scaled by min(1, max_norm / (sqrt(*sqnorm) + 1e-6)) first (written back to g)
    const double* sqnorm;
    float grad_scale;          // multiplied into g before everything else (1 / world size for an averaged all-reduce)
};
cudaError_t sgd_launch(const SgdParams& p, int num_sms, cudaStream_t st);

}  // namespace lfd
