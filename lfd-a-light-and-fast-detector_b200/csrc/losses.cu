// losses.cu -- label assignment and the classification / regression losses of LFD.get_loss, on the device.
//
//   assign_targets_kernel   lfd/model/lfd.py:155-259 (`_generate_target_for_single_image`): the reference builds
//                           P x G dense tensors on the CPU, sorts them and scatters with fancy indexing, image by
//                           image; here one thread owns one (image, point) and walks the image's gt boxes keeping
//                           the per-class best green score, the gray flag and the best-scoring green gt's deltas.
//                           Tie rule (reference: unspecified): highest score, then lowest gt index.
//   focal kernels           sigmoid focal loss, formulas of
//                           lfd/model/losses/build/sigmoid_focal_loss/src/cuda/sigmoid_focal_loss_cuda.cu:24-97
//                           (`lfd_sigmoid_focal_loss_{forward,backward}` mirror the pybind module 1:1), plus the
//                           fused row-masked forward+backward+reduction used by get_loss.
//   ce_loss_kernel          F.cross_entropy(reduction='none') + gradient (losses/cross_entropy_loss.py:12-22).
//   iou_loss_kernel         decode (lfd.py:261-282,353-378) + -log(IoU) (losses/iou_loss.py:66-80,98-123) + analytic
//                           gradient w.r.t. the raw regression outputs.
//   loss_weight_*_kernel    weight.sum() of enable_classification_weight / enable_regression_weight (lfd.py:322-324), the
//                           avg_factor of the weighted losses, summed in a fixed order.
// All label-assignment arithmetic uses _rn intrinsics (no FMA contraction) so that scores / deltas are
// bit-identical to the reference's separately rounded fp32 tensor ops.
#include <cfloat>

#include "kernels.cuh"
#include "ptx.cuh"

namespace lfd {

struct PointGeom {
    float px, py, half, lo, hi, glo, ghi;
};

__device__ __forceinline__ PointGeom point_geom(const LevelTable& lv, int pt) {
    int level = 0;
    for (int l = 1; l < lv.num_levels; ++l)
        if (pt >= lv.off[l]) level = l;
    const int local = pt - lv.off[level];
    PointGeom g;
    g.px = (float)((local % lv.w[level]) * lv.stride[level]);
    g.py = (float)((local / lv.w[level]) * lv.stride[level]);
    g.half = __fdiv_rn((float)lv.stride[level], 2.0f);
    g.lo = lv.lo[level]; g.hi = lv.hi[level]; g.glo = lv.glo[level]; g.ghi = lv.ghi[level];
    return g;
}

__device__ __forceinline__ float center_score(float d, float half) {  // lfd.py:190-198
    float s = __fdiv_rn(fabsf(d), half);
    s = s >= 1.0f ? s : 1.0f;
    return __fsqrt_rn(__fdiv_rn(1.0f, s));
}

__global__ void __launch_bounds__(256) assign_targets_kernel(const AssignParams p) {
    const int n = blockIdx.y;
    const int pt = blockIdx.x * blockDim.x + threadIdx.x;
    if (pt >= p.P) return;
    const PointGeom pg = point_geom(p.lv, pt);
    const int G = p.gt_count[n];
    const float4* boxes = reinterpret_cast<const float4*>(p.gt_boxes) + (size_t)n * p.gmax;
    const int* labels = p.gt_labels + (size_t)n * p.gmax;
    float* cls_row = p.cls_target + ((size_t)n * p.P + pt) * p.C;
    for (int c = 0; c < p.C; ++c) cls_row[c] = 0.f;
    float best = 0.f;
    float4 best_delta = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int pass = 0; pass < 2; ++pass) {  // pass 0: green (max score per class); pass 1: gray overrides with -1
        for (int g = 0; g < G; ++g) {
            const float4 b = boxes[g];  // x, y, w, h
            const float d0 = __fsub_rn(pg.px, b.x), d1 = __fsub_rn(pg.py, b.y);
            const float d2 = __fsub_rn(__fsub_rn(__fadd_rn(b.x, b.z), 1.0f), pg.px);
            const float d3 = __fsub_rn(__fsub_rn(__fadd_rn(b.y, b.w), 1.0f), pg.py);
            float measure;
            if (p.assign_mode == 0) measure = fmaxf(fmaxf(d0, d1), fmaxf(d2, d3));  // 'dist'
            else if (p.assign_mode == 1) measure = fmaxf(b.z, b.w);                 // 'longer'
            else measure = fminf(b.z, b.w);                                         // 'shorter'
            const bool hit = fminf(fminf(d0, d1), fminf(d2, d3)) >= 0.f;
            if (!hit) continue;
            const int lab = labels[g];
            if (pass == 0) {
                if (pg.lo <= measure && measure <= pg.hi) {
                    const float cx = __fadd_rn(b.x, __fdiv_rn(b.z, 2.0f)), cy = __fadd_rn(b.y, __fdiv_rn(b.w, 2.0f));
                    const float sc = __fmul_rn(center_score(__fsub_rn(pg.px, cx), pg.half), center_score(__fsub_rn(pg.py, cy), pg.half));
                    cls_row[lab] = fmaxf(cls_row[lab], sc);
                    if (sc > best) {
                        best = sc;
                        if (p.independent) {  // lfd.py:219-220
                            best_delta = make_float4(__fdiv_rn(d0, pg.hi), __fdiv_rn(d1, pg.hi), __fdiv_rn(d2, pg.hi), __fdiv_rn(d3, pg.hi));
                        } else {
                            best_delta = make_float4(d0, d1, d2, d3);
                        }
                    }
                }
            } else {
                const bool gray = (pg.glo <= measure && measure < pg.lo) || (pg.hi < measure && measure <= pg.ghi);
                if (gray) cls_row[lab] = -1.0f;
            }
        }
    }
    reinterpret_cast<float4*>(p.reg_target)[(size_t)n * p.P + pt] = best_delta;
    // row summary for the losses (lfd.py:314-329): ignore if any class is gray, positive if max score >= 0.001
    float mn = cls_row[0], mxv = cls_row[0];
    int arg = 0;
    for (int c = 1; c < p.C; ++c) {
        const float v = cls_row[c];
        mn = fminf(mn, v);
        if (v > mxv) { mxv = v; arg = c; }
    }
    int label;
    if (mn < 0.f) label = -1;
    else if (mxv >= 0.001f) label = arg;
    else label = p.C;
    p.label[(size_t)n * p.P + pt] = label;
    const bool pos = label >= 0 && label < p.C, valid = label >= 0;
    const unsigned mp = __ballot_sync(__activemask(), pos), mv = __ballot_sync(__activemask(), valid);
    const unsigned act = __activemask();
    if ((threadIdx.x & 31) == __ffs(act) - 1) {
        if (mp) atomicAdd(p.counters + 0, __popc(mp));
        if (mv) atomicAdd(p.counters + 1, __popc(mv));
    }
}

// ---------------------------------------------------------------------------------------------------
// sigmoid focal loss
__device__ __forceinline__ void focal_terms(float x, float gamma, float* p_out, float* log1mp) {
    *p_out = 1.0f / (1.0f + expf(-x));
    const float pos = x >= 0.f ? 1.0f : 0.0f;
    *log1mp = -1.0f * x * pos - logf(1.0f + expf(x - 2.0f * x * pos));
}
__device__ __forceinline__ float focal_fwd(float x, int t, int d, float gamma, float alpha) {
    float pr, l1;
    focal_terms(x, gamma, &pr, &l1);
    const float c1 = (t == d) ? 1.f : 0.f, c2 = (t >= 0 && t != d) ? 1.f : 0.f;
    const float term1 = powf(1.0f - pr, gamma) * logf(fmaxf(pr, FLT_MIN));
    const float term2 = powf(pr, gamma) * l1;
    return -c1 * term1 * alpha - c2 * term2 * (1.0f - alpha);
}
__device__ __forceinline__ float focal_bwd(float x, int t, int d, float gamma, float alpha) {
    float pr, l1;
    focal_terms(x, gamma, &pr, &l1);
    const float c1 = (t == d) ? 1.f : 0.f, c2 = (t >= 0 && t != d) ? 1.f : 0.f;
    const float term1 = powf(1.0f - pr, gamma) * (1.0f - pr - (pr * gamma * logf(fmaxf(pr, FLT_MIN))));
    const float term2 = powf(pr, gamma) * (l1 * (1.0f - pr) * gamma - pr);
    return -c1 * term1 * alpha - c2 * term2 * (1.0f - alpha);
}

__global__ void __launch_bounds__(512) focal_forward_kernel(int nthreads, const float* logits, const long long* targets,
                                                           int C, float gamma, float alpha, float* losses) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nthreads; i += blockDim.x * gridDim.x)
        losses[i] = focal_fwd(logits[i], (int)targets[i / C], i % C, gamma, alpha);
}
__global__ void __launch_bounds__(512) focal_backward_kernel(int nthreads, const float* logits, const long long* targets,
                                                            const float* d_losses, int C, float gamma, float alpha, float* d_logits) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nthreads; i += blockDim.x * gridDim.x)
        d_logits[i] = focal_bwd(logits[i], (int)targets[i / C], i % C, gamma, alpha) * d_losses[i];
}
cudaError_t focal_forward_launch(const float* logits, const long long* targets, int M, int C, float gamma, float alpha,
                                 float* losses, cudaStream_t st) {
    const int total = M * C;
    if (total == 0) return cudaSuccess;
    int grid = (total + 511) / 512;
    if (grid > 4096) grid = 4096;  // sigmoid_focal_loss_cuda.cu:112-114
    focal_forward_kernel<<<grid, 512, 0, st>>>(total, logits, targets, C, gamma, alpha, losses);
    return cudaGetLastError();
}
cudaError_t focal_backward_launch(const float* logits, const long long* targets, const float* d_losses, int M, int C,
                                  float gamma, float alpha, float* d_logits, cudaStream_t st) {
    const int total = M * C;
    if (total == 0) return cudaSuccess;
    int grid = (total + 511) / 512;
    if (grid > 4096) grid = 4096;
    focal_backward_kernel<<<grid, 512, 0, st>>>(total, logits, targets, d_losses, C, gamma, alpha, d_logits);
    return cudaGetLastError();
}

__device__ __forceinline__ double block_sum(double v, double* sh) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[w] = v;
    __syncthreads();
    double r = 0;
    if (threadIdx.x == 0)
        for (int i = 0; i < nw; ++i) r += sh[i];
    return r;  // valid on thread 0
}

// weight of a positive row (lfd.py:322-324): its maximal classification target, the centre score of its best green gt.  Read from
// the soft targets rather than stored by assign_targets_kernel, so the assignment and its callers stay as they are; the loss
// kernels read the row only for the few positive points.
__device__ __forceinline__ float row_weight(const float* cls_target, size_t r, int C) {
    const float* row = cls_target + r * C;
    float w = row[0];
    for (int c = 1; c < C; ++c) w = fmaxf(w, row[c]);
    return w;
}

// sum of the positives' weights (the reference's weight.sum()): per-block partials in a fixed order, then one block adds them up in
// index order -- no floating-point atomics, so repeated steps give the same bits
__global__ void __launch_bounds__(256) loss_weight_partials_kernel(const float* __restrict__ cls_target, const int* __restrict__ label, size_t rows,
                                                                   int C, double* __restrict__ partials) {
    __shared__ double sh[8];
    double acc = 0.0;
    for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (size_t)gridDim.x * blockDim.x) {
        const int t = label[r];
        if (t >= 0 && t < C) acc += (double)row_weight(cls_target, r, C);
    }
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}
__global__ void __launch_bounds__(256) loss_weight_final_kernel(const double* __restrict__ partials, int n, double* __restrict__ weight_sum) {
    __shared__ double sh[8];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partials[i];
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) *weight_sum = s;
}

// classification loss of get_loss (lfd.py:326-341): rows with label -1 are dropped, avg_factor = n_pos + 1 (weighted: the sum of the
// positives' weights, enable_classification_weight).  cls_mode 0: sigmoid focal over C logits; 1: cross entropy over C+1 logits.
// Writes d loss / d logit.
__global__ void __launch_bounds__(256) cls_loss_kernel(const ClsLossParams p) {
    __shared__ double sh[8];
    const int Cp = p.cls_mode == 1 ? p.C + 1 : p.C;
    const float inv_avg = p.weighted ? 1.0f / (float)*p.weight_sum : 1.0f / (float)(p.counters[0] + 1);
    double acc = 0.0;
    const size_t rows = (size_t)p.N * p.P;
    if (p.cls_mode != 1) {
        const size_t total = rows * Cp;
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
            const int t = p.label[i / Cp];
            float l = 0.f, g = 0.f;
            if (t >= 0) {
                const int d = (int)(i % Cp);
                const float x = p.logits[i];
                if (p.cls_mode == 0) {
                    l = focal_fwd(x, t, d, p.gamma, p.alpha);
                    g = focal_bwd(x, t, d, p.gamma, p.alpha);
                } else {
                    // binary cross entropy with logits against a target q (ATen's stable form): max(x,0) - x q + log(1 + exp(-|x|))
                    const float sg = 1.0f / (1.0f + expf(-x));
                    const float sp = fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));      // softplus(x) = BCE(x, 0)
                    if (p.cls_mode == 2) {                                          // losses/bce_with_logits_loss.py:28-44, soft targets
                        const float q = p.cls_target[i];
                        l = sp - x * q;
                        g = sg - q;
                    } else if (d != t) {                                            // quality focal, negatives: BCE(x, 0) * sigmoid^beta
                        const float m = powf(sg, p.gamma);                          // (losses/gfocal_loss.py:32-38)
                        l = sp * m;
                        g = sg * m + sp * p.gamma * m * (1.0f - sg);
                    } else {                                                        // positives: BCE(x, score) * |score - sigmoid|^beta (:41-46)
                        const float* row = p.cls_target + (i / Cp) * Cp;
                        float q = row[0];
                        for (int c = 1; c < Cp; ++c) q = fmaxf(q, row[c]);          // quality = the point's (maximal) centre score
                        const float a = fabsf(q - sg), bce = sp - x * q;
                        const float m = powf(a, p.gamma);
                        l = bce * m;
                        g = (sg - q) * m + (a > 0.f ? bce * p.gamma * powf(a, p.gamma - 1.0f) * (q > sg ? -1.f : 1.f) * sg * (1.0f - sg) : 0.f);
                    }
                }
                g *= inv_avg * p.loss_weight;
            }
            if (p.grad) p.grad[i] = g;
            acc += (double)l;
        }
    } else {
        for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (size_t)gridDim.x * blockDim.x) {
            const int t = p.label[r];
            const float* x = p.logits + r * Cp;
            float* g = p.grad ? p.grad + r * Cp : nullptr;
            if (t < 0) {
                if (g) for (int c = 0; c < Cp; ++c) g[c] = 0.f;
                continue;
            }
            float mx = x[0];
            for (int c = 1; c < Cp; ++c) mx = fmaxf(mx, x[c]);
            float den = 0.f;
            for (int c = 0; c < Cp; ++c) den += expf(x[c] - mx);
            const float lden = logf(den);
            acc += (double)(-(x[t] - mx - lden));
            if (g && p.weighted) {
                // as autograd's log_softmax backward, softmax * s - onehot * s: without positives s = inf and the target logit's
                // gradient is NaN, the others +inf, exactly as the reference's
                const float s = inv_avg * p.loss_weight;
                for (int c = 0; c < Cp; ++c) g[c] = expf(x[c] - mx) / den * s - (c == t ? s : 0.f);
            } else if (g) {
                for (int c = 0; c < Cp; ++c) g[c] = (expf(x[c] - mx) / den - (c == t ? 1.f : 0.f)) * inv_avg * p.loss_weight;
            }
        }
    }
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) atomicAdd(p.loss_sum, s);
}


// ---------------------------------------------------------------------------------------------------
// forward-mode derivatives w.r.t. the four predicted box coordinates (x1, y1, x2, y2): the GIoU / DIoU / CIoU losses are written
// exactly like the reference's functions (losses/iou_loss.py:125-283) on this type, so value AND gradient follow the same formula
struct Dual {
    float v, d[4];
};
__device__ __forceinline__ Dual dc(float c) { Dual r; r.v = c; r.d[0] = r.d[1] = r.d[2] = r.d[3] = 0.f; return r; }
__device__ __forceinline__ Dual dvar(float v, int i) { Dual r = dc(v); r.d[i] = 1.f; return r; }
__device__ __forceinline__ Dual operator+(Dual a, Dual b) { Dual r; r.v = a.v + b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] + b.d[i]; return r; }
__device__ __forceinline__ Dual operator-(Dual a, Dual b) { Dual r; r.v = a.v - b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] - b.d[i]; return r; }
__device__ __forceinline__ Dual operator*(Dual a, Dual b) { Dual r; r.v = a.v * b.v; for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i]; return r; }
__device__ __forceinline__ Dual operator/(Dual a, Dual b) {
    Dual r; r.v = a.v / b.v;
    const float inv = 1.0f / b.v;
    for (int i = 0; i < 4; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv;
    return r;
}
__device__ __forceinline__ Dual dmax(Dual a, Dual b) {   // torch.max(a, b): ties share the gradient
    if (a.v > b.v) return a;
    if (b.v > a.v) return b;
    Dual r; r.v = a.v; for (int i = 0; i < 4; ++i) r.d[i] = 0.5f * (a.d[i] + b.d[i]); return r;
}
__device__ __forceinline__ Dual dmin(Dual a, Dual b) {
    if (a.v < b.v) return a;
    if (b.v < a.v) return b;
    Dual r; r.v = a.v; for (int i = 0; i < 4; ++i) r.d[i] = 0.5f * (a.d[i] + b.d[i]); return r;
}
__device__ __forceinline__ Dual dclamp0(Dual a) { return a.v >= 0.f ? a : dc(0.f); }   // clamp(min=0): gradient where a >= 0
__device__ __forceinline__ Dual datan(Dual a) { Dual r; r.v = atanf(a.v); const float k = 1.0f / (1.0f + a.v * a.v); for (int i = 0; i < 4; ++i) r.d[i] = a.d[i] * k; return r; }

// kind 1 GIoU, 2 DIoU, 3 CIoU; pr = predicted box (variables), tg = target box (constants)
__device__ __forceinline__ Dual iou_family_loss(int kind, const Dual* pr, const float* tgf, float eps) {
    const Dual tg[4] = {dc(tgf[0]), dc(tgf[1]), dc(tgf[2]), dc(tgf[3])};
    const Dual w = dclamp0(dmin(pr[2], tg[2]) - dmax(pr[0], tg[0])), h = dclamp0(dmin(pr[3], tg[3]) - dmax(pr[1], tg[1]));
    const Dual overlap = w * h;
    const Dual ap = (pr[2] - pr[0]) * (pr[3] - pr[1]), ag = (tg[2] - tg[0]) * (tg[3] - tg[1]);
    const Dual uni = ap + ag - overlap + dc(eps);
    const Dual ious = overlap / uni;
    const Dual cw = dclamp0(dmax(pr[2], tg[2]) - dmin(pr[0], tg[0])), ch = dclamp0(dmax(pr[3], tg[3]) - dmin(pr[1], tg[1]));
    if (kind == 1) {
        const Dual area = cw * ch + dc(eps);
        return dc(1.f) - (ious - (area - uni) / area);
    }
    const Dual c2 = cw * cw + ch * ch + dc(eps);
    const Dual dx = (tg[0] + tg[2]) - (pr[0] + pr[2]), dy = (tg[1] + tg[3]) - (pr[1] + pr[3]);
    const Dual rho2 = (dx * dx) / dc(4.f) + (dy * dy) / dc(4.f);
    if (kind == 2) return dc(1.f) - (ious - rho2 / c2);
    const Dual w1 = pr[2] - pr[0], h1 = pr[3] - pr[1] + dc(eps);
    const Dual w2 = tg[2] - tg[0], h2 = tg[3] - tg[1] + dc(eps);
    const Dual da = datan(w2 / h2) - datan(w1 / h1);
    const Dual v = dc(0.40528473456935109f) * da * da;          // 4 / pi^2
    // v = 0 (equal aspect ratios): the term and its derivatives are 0.  Evaluated, it is 0 / 0 when the fp32 IoU rounds to 1 (identical
    // boxes whose area swamps eps), where the reference's value in exact arithmetic is 0 / (eps / (area + eps)) = 0.
    const Dual vt = v.v == 0.f ? dc(0.f) : (v * v) / (dc(1.f) - ious + v);
    return dc(1.f) - (ious - (rho2 / c2 + vt));
}

// regression loss of get_loss (lfd.py:343-387): positives, avg_factor = n_pos.  loss_kind 0: -log IoU (analytic gradient);
// 1..3: GIoU / DIoU / CIoU through forward-mode derivatives; 4, 5: SmoothL1 / MSE on the raw outputs ('independent' targets).
// weighted (enable_regression_weight, weight_reduce_loss of losses/utils.py:28-53): the row loss times the row's weight, avg_factor =
// the sum of the weights; no positives: loss and gradients 0 either way (lfd.py:386-387).
__global__ void __launch_bounds__(256) iou_loss_kernel(const RegLossParams p) {
    __shared__ double sh[8];
    const size_t rows = (size_t)p.N * p.P;
    const int npos = p.counters[0];
    const float inv_avg = npos > 0 ? (p.weighted ? 1.0f / (float)*p.weight_sum : 1.0f / (float)npos) : 0.f;
    double acc = 0.0;
    for (size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (size_t)gridDim.x * blockDim.x) {
        const int t = p.label[r];
        float4 g4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (t >= 0 && t < p.C) {
            float sc = inv_avg * p.loss_weight, wt = 1.0f;   // wt = 1: the product below is exact, the unweighted sums keep their bits
            if (p.weighted) {
                wt = row_weight(p.cls_target, r, p.C);
                sc *= wt;
            }
            const int pt = (int)(r % p.P);
            const PointGeom pg = point_geom(p.lv, pt);
            const float4 rv = reinterpret_cast<const float4*>(p.reg)[r];
            const float4 tv = reinterpret_cast<const float4*>(p.reg_target)[r];
            float raw[4] = {rv.x, rv.y, rv.z, rv.w}, d[4], dd[4];  // dd = d(distance)/d(raw)
            if (p.loss_kind >= 4) {   // 'independent': element-wise loss between the raw outputs and the range-normalised targets (lfd.py:353-358)
                const float tg[4] = {tv.x, tv.y, tv.z, tv.w};
                float gk[4], ls = 0.f;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float df = raw[k] - tg[k], ad = fabsf(df);
                    if (p.loss_kind == 4) {                      // losses/smooth_l1_loss.py:10-28
                        if (ad < p.beta) { ls += 0.5f * ad * ad / p.beta; gk[k] = df / p.beta; }
                        else { ls += ad - 0.5f * p.beta; gk[k] = df > 0.f ? 1.f : -1.f; }
                    } else { ls += df * df; gk[k] = 2.f * df; }  // F.mse_loss(reduction='none')
                }
                acc += (double)(ls * wt);
                if (p.grad) reinterpret_cast<float4*>(p.grad)[r] = make_float4(gk[0] * sc, gk[1] * sc, gk[2] * sc, gk[3] * sc);
                continue;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (p.bbox_mode == 0) { const float s = 1.0f / (1.0f + expf(-raw[k])); d[k] = s * pg.hi; dd[k] = pg.hi * s * (1.0f - s); }
                else { d[k] = expf(raw[k]); dd[k] = d[k]; }
            }
            const float px1 = pg.px - d[0], py1 = pg.py - d[1], px2 = pg.px + d[2], py2 = pg.py + d[3];
            const float tx1 = pg.px - tv.x, ty1 = pg.py - tv.y, tx2 = pg.px + tv.z, ty2 = pg.py + tv.w;
            if (p.loss_kind >= 1) {
                const Dual pr[4] = {dvar(px1, 0), dvar(py1, 1), dvar(px2, 2), dvar(py2, 3)};
                const float tg[4] = {tx1, ty1, tx2, ty2};
                const Dual ls = iou_family_loss(p.loss_kind, pr, tg, p.eps);
                acc += (double)(ls.v * wt);
                if (p.grad) reinterpret_cast<float4*>(p.grad)[r] = make_float4(-ls.d[0] * dd[0] * sc, -ls.d[1] * dd[1] * sc, ls.d[2] * dd[2] * sc, ls.d[3] * dd[3] * sc);
                continue;
            }
            const float ltx = fmaxf(px1, tx1), lty = fmaxf(py1, ty1), rbx = fminf(px2, tx2), rby = fminf(py2, ty2);
            const float rw = rbx - ltx, rh = rby - lty;
            const float w = fmaxf(rw, 0.f), h = fmaxf(rh, 0.f);
            const float ov = w * h;
            const float pw = px2 - px1, ph = py2 - py1;
            const float ap = pw * ph, at = (tx2 - tx1) * (ty2 - ty1);
            const float ur = ap + at - ov;
            const float un = fmaxf(ur, 1e-6f);
            const float iou = ov / un;
            const float iouc = fmaxf(iou, p.eps);
            acc += (double)(-logf(iouc) * wt);
            if (p.grad) {
                const float g_iou = iou >= p.eps ? -1.0f / iouc : 0.f;
                const float un_live = ur > 1e-6f ? 1.f : 0.f;
                const float g_ov = g_iou * (1.0f / un + un_live * ov / (un * un));
                const float g_ap = -g_iou * un_live * ov / (un * un);
                const float g_w = rw > 0.f ? g_ov * h : 0.f, g_h = rh > 0.f ? g_ov * w : 0.f;
                float g_px1 = -g_ap * ph, g_px2 = g_ap * ph, g_py1 = -g_ap * pw, g_py2 = g_ap * pw;
                // torch.max / torch.min of the reference's bbox_overlaps: a predicted edge equal to the target edge gets half the gradient
                if (px2 < tx2) g_px2 += g_w; else if (px2 == tx2) g_px2 += 0.5f * g_w;
                if (px1 > tx1) g_px1 -= g_w; else if (px1 == tx1) g_px1 -= 0.5f * g_w;
                if (py2 < ty2) g_py2 += g_h; else if (py2 == ty2) g_py2 += 0.5f * g_h;
                if (py1 > ty1) g_py1 -= g_h; else if (py1 == ty1) g_py1 -= 0.5f * g_h;
                g4 = make_float4(-g_px1 * dd[0] * sc, -g_py1 * dd[1] * sc, g_px2 * dd[2] * sc, g_py2 * dd[3] * sc);
            }
        }
        if (p.grad) reinterpret_cast<float4*>(p.grad)[r] = g4;
    }
    const double s = block_sum(acc, sh);
    if (threadIdx.x == 0) atomicAdd(p.loss_sum, s);
}

// element-wise box losses on explicit (pred, target) xyxy pairs: the stand-alone IoULoss / GIoULoss / DIoULoss / CIoULoss modules
// (losses/iou_loss.py:105-283 before the reduction).  kind 0: -log(max(IoU, eps)) with IoU = overlap / max(union, 1e-6).
__global__ void __launch_bounds__(256) box_loss_kernel(int kind, const float* __restrict__ pred, const float* __restrict__ target, int n, float eps,
                                                       float* __restrict__ loss, float* __restrict__ grad) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 pv = reinterpret_cast<const float4*>(pred)[i], tv = reinterpret_cast<const float4*>(target)[i];
        const Dual pr[4] = {dvar(pv.x, 0), dvar(pv.y, 1), dvar(pv.z, 2), dvar(pv.w, 3)};
        const float tg[4] = {tv.x, tv.y, tv.z, tv.w};
        Dual ls;
        if (kind == 0) {
            const Dual t4[4] = {dc(tg[0]), dc(tg[1]), dc(tg[2]), dc(tg[3])};
            const Dual w = dclamp0(dmin(pr[2], t4[2]) - dmax(pr[0], t4[0])), h = dclamp0(dmin(pr[3], t4[3]) - dmax(pr[1], t4[1]));
            const Dual ov = w * h;
            Dual un = (pr[2] - pr[0]) * (pr[3] - pr[1]) + (t4[2] - t4[0]) * (t4[3] - t4[1]) - ov;
            if (un.v < 1e-6f) un = dc(1e-6f);
            Dual iou = ov / un;
            if (iou.v < eps) iou = dc(eps);
            ls = dc(-logf(iou.v));
            for (int k = 0; k < 4; ++k) ls.d[k] = -iou.d[k] / iou.v;
        } else {
            ls = iou_family_loss(kind, pr, tg, eps);
        }
        loss[i] = ls.v;
        if (grad) reinterpret_cast<float4*>(grad)[i] = make_float4(ls.d[0], ls.d[1], ls.d[2], ls.d[3]);
    }
}
cudaError_t box_loss_launch(int kind, const float* pred, const float* target, int n, float eps, float* loss, float* grad, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    int grid = (n + 255) / 256;
    if (grid > 4096) grid = 4096;
    box_loss_kernel<<<grid, 256, 0, st>>>(kind, pred, target, n, eps, loss, grad);
    return cudaGetLastError();
}

cudaError_t assign_targets_launch(const AssignParams& p, cudaStream_t st) {
    assign_targets_kernel<<<dim3((p.P + 255) / 256, p.N), 256, 0, st>>>(p);
    return cudaGetLastError();
}
cudaError_t cls_loss_launch(const ClsLossParams& p, int num_sms, cudaStream_t st) {
    cls_loss_kernel<<<num_sms * 4, 256, 0, st>>>(p);
    return cudaGetLastError();
}
cudaError_t iou_loss_launch(const RegLossParams& p, int num_sms, cudaStream_t st) {
    iou_loss_kernel<<<num_sms * 4, 256, 0, st>>>(p);
    return cudaGetLastError();
}
int loss_weight_blocks(int num_sms) { return num_sms * 4; }
cudaError_t loss_weight_sum_launch(const float* cls_target, const int* label, size_t rows, int C, int num_sms, double* partials,
                                   double* weight_sum, cudaStream_t st) {
    const int blocks = loss_weight_blocks(num_sms);
    loss_weight_partials_kernel<<<blocks, 256, 0, st>>>(cls_target, label, rows, C, partials);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    loss_weight_final_kernel<<<1, 256, 0, st>>>(partials, blocks, weight_sum);
    return cudaGetLastError();
}

}  // namespace lfd
