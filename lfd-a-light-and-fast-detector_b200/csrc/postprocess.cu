// postprocess.cu -- score (sigmoid | softmax) + threshold + distance->box decode + class-aware greedy NMS.
//
// Replaces lfd/model/lfd.py:434-509 (`_get_results_for_single_image`), :577-641 (predict path),
// lfd/model/utils/nms.py:119-220 (`batched_nms`, `multiclass_nms`) and the native
// lfd/model/utils/build/nms/src/{cpu/nms_cpu.cpp:8-66, cuda/nms_kernel.cu:24-138}.
// The reference's CUDA NMS copies an n x n/64 bitmask to the host and sweeps it on the CPU
// (nms_kernel.cu:104-131); here everything stays on the device:
//   candidates_kernel : one thread per point -- scores, strict `> thr` filter, decode, clamp, /resize_scale,
//                       warp-aggregated append to the image's candidate list.
//   nms_kernel        : one CTA per image, warp-cooperative -- class offsets (label * (max_coord + 1), added in
//                       fp32 exactly like nms.py:145-150), bitonic sort by (score desc, source index asc),
//                       greedy sweep with strict `iou > thr`, IoU without +1 / epsilon; writes kept rows in
//                       score-descending order.
// Arithmetic that decides kept indices is written with explicit _rn intrinsics so that nvcc cannot contract
// it into FMAs (the reference computes every step in separately rounded fp32).
#include "conv_common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace lfd {

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// 32-bit key that sorts ASCENDING when the float sorts DESCENDING (total order incl. negatives)
__device__ __forceinline__ uint32_t desc_key(float f) {
    uint32_t u = __float_as_uint(f);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ~u;
}

// ---------------------------------------------------------------------------------------------------
// distance2bbox (+ clamp to the image, / resize scale) of one point: lfd.py:468-488
__device__ __forceinline__ void decode_point(const PostParams& p, int n, int pt, float* box) {
    int level = 0;
    for (int l = 1; l < p.num_levels; ++l)
        if (pt >= p.level_off[l]) level = l;
    const int local = pt - p.level_off[level];
    const float4 r = *reinterpret_cast<const float4*>(p.reg + ((size_t)n * p.P + pt) * 4);
    const int W = p.level_w[level];
    const float px = (float)((local % W) * p.level_stride[level]);
    const float py = (float)((local / W) * p.level_stride[level]);
    float d[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (p.bbox_mode == 0) d[k] = __fmul_rn(sigmoid_f(d[k]), p.level_hi[level]);   // lfd.py:481-486
        else if (p.bbox_mode == 1) d[k] = expf(d[k]);                                  // :478-480
        else d[k] = __fmul_rn(d[k], p.level_hi[level]);                                // 'independent' :468-476
    }
    const float iw = p.img_w[n], ih = p.img_h[n], rs = p.resize_scale[n];
    box[0] = __fdiv_rn(fminf(fmaxf(__fsub_rn(px, d[0]), 0.f), iw), rs);
    box[1] = __fdiv_rn(fminf(fmaxf(__fsub_rn(py, d[1]), 0.f), ih), rs);
    box[2] = __fdiv_rn(fminf(fmaxf(__fadd_rn(px, d[2]), 0.f), iw), rs);
    box[3] = __fdiv_rn(fminf(fmaxf(__fadd_rn(py, d[3]), 0.f), ih), rs);
}

// warp-aggregated slot claim in the image's candidate list
__device__ __forceinline__ void claim_candidate(const PostParams& p, int n, bool pass, const float* box, float score, int src) {
    const unsigned m = __ballot_sync(0xffffffffu, pass);
    if (!m) return;
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(p.cand_count + n, __popc(m));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (pass) {
        const int slot = base + __popc(m & ((1u << lane) - 1));
        if (slot < p.cap) {
            const size_t o = (size_t)n * p.cap + slot;
            reinterpret_cast<float4*>(p.cand_box)[o] = make_float4(box[0], box[1], box[2], box[3]);
            p.cand_score[o] = score;
            p.cand_src[o] = src;
        }
    }
}

// One thread per point, looping over the classes: single-class heads (the face configs) and the softmax head (needs the row).
__global__ void __launch_bounds__(256) candidates_kernel(const PostParams p) {
    const int n = blockIdx.y;
    const int pt = blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = pt < p.P;
    float box[4] = {0, 0, 0, 0};
    bool decoded = false;
    const float* cls = p.cls + ((size_t)n * p.P + (active ? pt : 0)) * p.cls_stride;
    float smax = 0.f, sden = 1.f;
    if (active && p.cls_mode == 1) {  // softmax over C+1 logits, background (last) dropped (lfd.py:450-452)
        smax = cls[0];
        for (int c = 1; c <= p.C; ++c) smax = fmaxf(smax, cls[c]);
        sden = 0.f;
        for (int c = 0; c <= p.C; ++c) sden += expf(cls[c] - smax);
    }
    for (int c = 0; c < p.C; ++c) {
        float score = 0.f;
        bool pass = false;
        if (active) {
            score = p.cls_mode == 1 ? expf(cls[c] - smax) / sden : sigmoid_f(cls[c]);
            pass = score > p.score_thr;
        }
        if (pass && !decoded) {
            decode_point(p, n, pt, box);
            decoded = true;
        }
        claim_candidate(p, n, pass, box, score, pt * p.C + c);
    }
}

// Softmax heads (TT100K: 45 classes + background): one thread per point as above, but the block's 128 logit rows are first brought into
// shared memory with coalesced loads (thread-per-row loads touch 32 different rows of C + 1 floats per instruction).
static constexpr int kRowsPts = 128;
__global__ void __launch_bounds__(kRowsPts) candidates_rows_kernel(const PostParams p) {
    extern __shared__ float rows[];
    const int n = blockIdx.y;
    const int pt0 = blockIdx.x * kRowsPts;
    const int npts = min(kRowsPts, p.P - pt0);
    const float* src = p.cls + ((size_t)n * p.P + pt0) * p.cls_stride;
    for (int i = threadIdx.x; i < npts * p.cls_stride; i += kRowsPts) rows[i] = src[i];
    __syncthreads();
    const bool active = (int)threadIdx.x < npts;
    const int pt = pt0 + threadIdx.x;
    const float* cls = rows + (active ? threadIdx.x : 0) * p.cls_stride;
    float box[4] = {0, 0, 0, 0};
    bool decoded = false;
    float smax = 0.f, sden = 1.f;
    if (active && p.cls_mode == 1) {  // softmax over C+1 logits, background (last) dropped (lfd.py:450-452)
        smax = cls[0];
        for (int c = 1; c <= p.C; ++c) smax = fmaxf(smax, cls[c]);
        sden = 0.f;
        for (int c = 0; c <= p.C; ++c) sden += expf(cls[c] - smax);
    }
    for (int c = 0; c < p.C; ++c) {
        float score = 0.f;
        bool pass = false;
        if (active) {
            score = p.cls_mode == 1 ? expf(cls[c] - smax) / sden : sigmoid_f(cls[c]);
            pass = score > p.score_thr;
        }
        if (pass && !decoded) {
            decode_point(p, n, pt, box);
            decoded = true;
        }
        claim_candidate(p, n, pass, box, score, pt * p.C + c);
    }
}

// Sigmoid heads with several classes (TT100K: 45): one thread per (point, class) logit, so that a warp reads 128 contiguous bytes of the
// (N, P, C) score tensor per load instead of 32 rows of C floats; the box is decoded only for the few logits that pass.
__global__ void __launch_bounds__(256) candidates_flat_kernel(const PostParams p) {
    const int n = blockIdx.y;
    const long long total = (long long)p.P * p.cls_stride;
    const float* cls = p.cls + (size_t)n * total;
    const long long rounds = (total + (long long)gridDim.x * 256 - 1) / ((long long)gridDim.x * 256);
    for (long long r = 0; r < rounds; ++r) {      // every lane of a warp runs the same number of rounds (the claim is warp-collective)
        const long long e = (r * gridDim.x + blockIdx.x) * 256 + threadIdx.x;
        float score = 0.f, box[4] = {0, 0, 0, 0};
        bool pass = false;
        int pt = 0, c = 0;
        if (e < total) {
            pt = (int)(e / p.cls_stride);
            c = (int)(e - (long long)pt * p.cls_stride);
            if (c < p.C) {
                score = sigmoid_f(cls[e]);
                pass = score > p.score_thr;
            }
        }
        if (pass) decode_point(p, n, pt, box);
        claim_candidate(p, n, pass, box, score, pt * p.C + c);
    }
}

// Candidates from explicit (already decoded) boxes: the entry of multiclass_nms / batched_nms (utils/nms.py:119-220).
//   labels_in == null: rows x classes grid, candidate (i, c) when scores[i * score_stride + c] > score_thr (strict, nms.py:204),
//                      box = boxes[i] (box_per_class 0) or boxes[i][c]
//   labels_in != null: one candidate per row: (boxes[i], scores[i], labels_in[i]), no threshold
__global__ void __launch_bounds__(256) box_candidates_kernel(const float* __restrict__ boxes, int box_per_class, const float* __restrict__ scores,
                                                             int score_stride, const int* __restrict__ labels_in, int n, int C, float score_thr, int cap,
                                                             float* cand_box, float* cand_score, int* cand_src, int* cand_count) {
    const long long total = labels_in ? (long long)n : (long long)n * C;
    for (long long idx = (long long)blockIdx.x * 256 + threadIdx.x; idx < total; idx += (long long)gridDim.x * 256) {
        int i, c;
        float sc;
        if (labels_in) { i = (int)idx; c = labels_in[i]; sc = scores[i]; }
        else { i = (int)(idx / C); c = (int)(idx % C); sc = scores[(size_t)i * score_stride + c]; if (!(sc > score_thr)) continue; }
        const int slot = atomicAdd(cand_count, 1);
        if (slot >= cap) continue;                   // the NMS kernel reports the overflow
        const float4 b = reinterpret_cast<const float4*>(boxes)[box_per_class ? (size_t)i * C + c : (size_t)i];
        reinterpret_cast<float4*>(cand_box)[slot] = b;
        cand_score[slot] = sc;
        cand_src[slot] = i * C + c;
    }
}
cudaError_t box_candidates_launch(const float* boxes, int box_per_class, const float* scores, int score_stride, const int* labels_in, int n, int C,
                                  float score_thr, int cap, float* cand_box, float* cand_score, int* cand_src, int* cand_count, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    const long long total = labels_in ? (long long)n : (long long)n * C;
    long long blocks = (total + 255) / 256;
    if (blocks > 2048) blocks = 2048;
    box_candidates_kernel<<<(int)blocks, 256, 0, st>>>(boxes, box_per_class, scores, score_stride, labels_in, n, C, score_thr, cap, cand_box, cand_score, cand_src,
                                                      cand_count);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// One CTA per image.
//   cand_*   : unsorted candidates (count K, K <= cap)
//   scratch  : per image  [cap_pow2] u64 keys | [cap_pow2] u32 payload | [cap] float4 sorted boxes | [cap] u8 flags
//   outputs  : dets [cap][5], labels [cap], src [cap] (index into the (point, class) grid, or the input row for
//              raw mode), count
static constexpr int kNmsThreads = 1024;
static constexpr int kNmsSmemSort = 4096;   // candidates sortable / sweepable entirely in shared memory
static constexpr int kNmsMaskMax = 1024;    // candidates for which the K x K suppression bit matrix fits in shared memory
static constexpr size_t kNmsMaskOff = 32768;   // smem offset of the bit matrix (behind the 1024-entry sort arrays, 29 KB)

__device__ __forceinline__ float iou_ref(const float4 a, const float aa, const float4 b, const float ab) {
    const float xx1 = fmaxf(a.x, b.x), yy1 = fmaxf(a.y, b.y), xx2 = fminf(a.z, b.z), yy2 = fminf(a.w, b.w);
    const float w = fmaxf(0.f, __fsub_rn(xx2, xx1)), h = fmaxf(0.f, __fsub_rn(yy2, yy1));
    const float inter = __fmul_rn(w, h);
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ab), inter));  // nms_cpu.cpp:57-61
}
__device__ __forceinline__ float box_area(const float4 b) { return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y)); }

// largest and smallest coordinate over the K candidate boxes (nms.py:148 `bboxes.max()`), every thread gets both
__device__ __forceinline__ void block_box_extent(const float4* cbox, int K, float* s_red, float* s_red2, float& mx, float& mn) {
    const int tid = threadIdx.x;
    mx = -3.4e38f; mn = 3.4e38f;
    for (int i = tid; i < K; i += kNmsThreads) {
        const float4 b = cbox[i];
        mx = fmaxf(mx, fmaxf(fmaxf(b.x, b.y), fmaxf(b.z, b.w)));
        mn = fminf(mn, fminf(fminf(b.x, b.y), fminf(b.z, b.w)));
    }
    for (int o = 16; o; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    }
    if ((tid & 31) == 0) { s_red[tid >> 5] = mx; s_red2[tid >> 5] = mn; }
    __syncthreads();
    mx = s_red[0];
    mn = s_red2[0];
    for (int i = 1; i < kNmsThreads / 32; ++i) { mx = fmaxf(mx, s_red[i]); mn = fminf(mn, s_red2[i]); }
}

// ascending bitonic sort of Kp (a power of two) 64-bit keys, with an optional 32-bit payload
__device__ __forceinline__ void block_bitonic_sort(unsigned long long* keys, uint32_t* pay, int Kp) {
    const int tid = threadIdx.x;
    for (int size = 2; size <= Kp; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < (Kp >> 1); i += kNmsThreads) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const bool up = (lo & size) == 0;
                const unsigned long long a = keys[lo], b = keys[hi];
                if ((a > b) == up) {
                    keys[lo] = b; keys[hi] = a;
                    if (pay) { const uint32_t t = pay[lo]; pay[lo] = pay[hi]; pay[hi] = t; }
                }
            }
            __syncthreads();
        }
}

// exclusive prefix of v over the block's threads; the total lands in s_scan[32]
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_scan) {
    const int tid = threadIdx.x;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= o) incl += t;
    }
    __syncthreads();
    if ((tid & 31) == 31) s_scan[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
        int w = s_scan[tid], wi = w;
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, wi, o);
            if (tid >= o) wi += t;
        }
        s_scan[tid] = wi - w;
        if (tid == 31) s_scan[32] = wi;
    }
    __syncthreads();
    return s_scan[tid >> 5] + incl - v;
}

// output row k of image n: the box with its class offset taken off again (nms.py:155, the fp32 round trip kept), score, label, source
__device__ __forceinline__ void write_det(const NmsParams& p, int n, int k, float4 ob, float score, int src, float offmul) {
    if (!p.class_agnostic) {
        const float off = __fmul_rn((float)(src % p.C), offmul);
        ob.x = __fsub_rn(ob.x, off); ob.y = __fsub_rn(ob.y, off); ob.z = __fsub_rn(ob.z, off); ob.w = __fsub_rn(ob.w, off);
    }
    float* d = p.out_dets + ((size_t)n * p.cap + k) * 5;
    d[0] = ob.x; d[1] = ob.y; d[2] = ob.z; d[3] = ob.w; d[4] = score;
    p.out_label[(size_t)n * p.cap + k] = src % p.C;
    p.out_src[(size_t)n * p.cap + k] = src;
}

__global__ void __launch_bounds__(kNmsThreads) nms_kernel(const NmsParams p) {
    extern __shared__ __align__(16) uint8_t nsm[];
    __shared__ float s_red[32], s_red2[32];
    __shared__ int s_keep, s_scan[33];
    const int n = blockIdx.x;
    const int tid = threadIdx.x;
    int K = p.cand_count[n];
    if (K > p.cap) {  // capacity overflow: report, process the first cap (host turns this into an error)
        if (tid == 0) atomicExch(p.overflow, 1);
        K = p.cap;
    }
    if (K == 0) {
        if (tid == 0) p.out_count[n] = 0;
        return;
    }
    int Kp = 1;
    while (Kp < K) Kp <<= 1;
    const bool in_smem = Kp <= kNmsSmemSort;
    const bool use_mask = Kp <= kNmsMaskMax;          // the common case: bit-matrix sweep (step 4a)
    const size_t L = use_mask ? kNmsMaskMax : kNmsSmemSort;   // entries the shared-memory arrays are laid out for
    uint8_t* gscr = p.scratch + (size_t)n * p.scratch_stride;
    unsigned long long* keys = in_smem ? reinterpret_cast<unsigned long long*>(nsm)
                                       : reinterpret_cast<unsigned long long*>(gscr);
    uint32_t* pay = in_smem ? reinterpret_cast<uint32_t*>(nsm + L * 8)
                            : reinterpret_cast<uint32_t*>(gscr + (size_t)p.cap_pow2 * 8);
    float4* sbox = in_smem ? reinterpret_cast<float4*>(nsm + L * 12)
                           : reinterpret_cast<float4*>(gscr + (size_t)p.cap_pow2 * 12);
    uint8_t* removed = in_smem ? nsm + L * 28 : gscr + (size_t)p.cap_pow2 * 12 + (size_t)p.cap * 16;
    const float4* cbox = reinterpret_cast<const float4*>(p.cand_box) + (size_t)n * p.cap;
    const float* cscore = p.cand_score + (size_t)n * p.cap;
    const int* csrc = p.cand_src + (size_t)n * p.cap;

    // 1. max coordinate over the candidate boxes (nms.py:148 `bboxes.max()`)
    float mx = -3.4e38f, mn = 3.4e38f;
    if (!p.class_agnostic) block_box_extent(cbox, K, s_red, s_red2, mx, mn);
    const float offmul = __fadd_rn(mx, 1.0f);

    // 2. sort keys: score descending, source index ascending (deterministic total order)
    for (int i = tid; i < Kp; i += kNmsThreads) {
        unsigned long long k = ~0ull;
        if (i < K) k = ((unsigned long long)desc_key(cscore[i]) << 32) | (unsigned)csrc[i];
        keys[i] = k;
        pay[i] = (uint32_t)i;
    }
    __syncthreads();
    block_bitonic_sort(keys, pay, Kp);

    // 3. sorted, class-offset boxes
    for (int i = tid; i < K; i += kNmsThreads) {
        const int s = (int)pay[i];
        float4 b = cbox[s];
        if (!p.class_agnostic) {
            const float off = __fmul_rn((float)(csrc[s] % p.C), offmul);
            b.x = __fadd_rn(b.x, off); b.y = __fadd_rn(b.y, off); b.z = __fadd_rn(b.z, off); b.w = __fadd_rn(b.w, off);
        }
        sbox[i] = b;
        removed[i] = 0;
    }
    if (tid == 0) s_keep = 0;
    __syncthreads();

    // 4a. K <= 1024: all pairwise decisions first (mask[i] bit j = "i suppresses j", j > i; fully parallel), then ONE warp walks
    //     the rows in score order OR-ing the masks of the kept boxes into a 1024-bit register bitmap (one word per lane).
    //     Same decisions as the sweep below (a box is dropped iff an earlier KEPT box overlaps it by more than iou_thr).
    if (use_mask) {
        uint32_t* mask = reinterpret_cast<uint32_t*>(nsm + kNmsMaskOff);   // [K][32 words]
        int* keep_list = reinterpret_cast<int*>(keys);                    // the sort keys are dead by now
        const int nw = (K + 31) >> 5;
        for (int idx = tid; idx < K * nw; idx += kNmsThreads) {
            const int i = idx / nw, w = idx - i * nw;
            uint32_t bits = 0;
            if (w >= (i >> 5)) {
                const float4 bi = sbox[i];
                const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
                const int j0 = w << 5;
                for (int b = 0; b < 32; ++b) {
                    const int j = j0 + b;
                    if (j > i && j < K) {
                        const float4 bj = sbox[j];
                        const float aj = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
                        if (iou_ref(bi, ai, bj, aj) > p.iou_thr) bits |= 1u << b;
                    }
                }
            }
            mask[i * 32 + w] = bits;
        }
        __syncthreads();
        if (tid < 32) {
            uint32_t rem = 0;     // lane l: boxes 32 l .. 32 l + 31
            int nkeep = 0;
            for (int i = 0; i < K; ++i) {
                const uint32_t wv = __shfl_sync(0xffffffffu, rem, i >> 5);
                if ((wv >> (i & 31)) & 1u) continue;   // uniform
                if (tid == 0) keep_list[nkeep] = i;
                ++nkeep;
                if (tid < nw) rem |= mask[i * 32 + tid];
            }
            if (tid == 0) s_keep = nkeep;
        }
        __syncthreads();
        const int nkeep = s_keep;
        for (int k = tid; k < nkeep; k += kNmsThreads) {
            const int i = keep_list[k];
            const int s = (int)pay[i];
            write_det(p, n, k, sbox[i], cscore[s], csrc[s], offmul);
        }
        if (tid == 0) p.out_count[n] = nkeep;
        return;
    }

    // 4c. K > 1024 with several classes: boxes of different classes never suppress each other (after the class offsets they cannot
    //     overlap when every coordinate is >= 0, which the decode's clamp guarantees), so the greedy sweep factors into one sweep per class
    //     -- same arithmetic on the same offset boxes, same decisions, but 32 classes at a time (one warp each) instead of K lock-step
    //     rounds of the whole CTA.  The candidates are re-sorted by (class, global rank); kept boxes are emitted in global rank order.
    const size_t seg_off = in_smem ? ((L * 29 + 15) & ~(size_t)15) : 0;
    const size_t seg_cap = ((size_t)kNmsMaskOff + (size_t)kNmsMaskMax * 128 - seg_off) / 4;
    if (!p.class_agnostic && p.C > 1 && mn >= 0.f && (size_t)K <= seg_cap) {
        int* seg = reinterpret_cast<int*>(nsm + seg_off);
        for (int i = tid; i < Kp; i += kNmsThreads)
            keys[i] = i < K ? (((unsigned long long)(unsigned)(csrc[pay[i]] % p.C) << 32) | (unsigned)i) : ~0ull;
        __syncthreads();
        block_bitonic_sort(keys, nullptr, Kp);
        // segment starts, in order (block-wide exclusive scan of the boundary flags; each thread owns a run of consecutive positions)
        const int per = (K + kNmsThreads - 1) / kNmsThreads;
        const int i0 = min(tid * per, K), i1 = min(i0 + per, K);
        int cnt = 0;
        for (int i = i0; i < i1; ++i) cnt += (i == 0 || (keys[i] >> 32) != (keys[i - 1] >> 32)) ? 1 : 0;
        int pos = block_exclusive_scan(cnt, s_scan);
        const int nseg = s_scan[32];
        for (int i = i0; i < i1; ++i)
            if (i == 0 || (keys[i] >> 32) != (keys[i - 1] >> 32)) seg[pos++] = i;
        __syncthreads();
        constexpr int kLongSeg = 512;
        const int lane = tid & 31, warp = tid >> 5;
        for (int j = warp; j < nseg; j += kNmsThreads / 32) {      // one warp per class
            const int a = seg[j], b = j + 1 < nseg ? seg[j + 1] : K;
            if (b - a > kLongSeg) continue;
            for (int ii = a; ii < b; ++ii) {
                const int ri = (int)(unsigned)keys[ii];
                if (removed[ri]) continue;                         // uniform over the warp
                const float4 bi = sbox[ri];
                const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
                for (int jj = ii + 1 + lane; jj < b; jj += 32) {
                    const int rj = (int)(unsigned)keys[jj];
                    if (removed[rj]) continue;
                    const float4 bj = sbox[rj];
                    const float aj = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
                    if (iou_ref(bi, ai, bj, aj) > p.iou_thr) removed[rj] = 1;
                }
                __syncwarp();
            }
        }
        __syncthreads();
        for (int j = 0; j < nseg; ++j) {                           // classes with many candidates: the whole CTA in lock step
            const int a = seg[j], b = j + 1 < nseg ? seg[j + 1] : K;
            if (b - a <= kLongSeg) continue;
            for (int ii = a; ii < b; ++ii) {
                const int ri = (int)(unsigned)keys[ii];
                if (removed[ri]) continue;                         // uniform (written only between barriers)
                const float4 bi = sbox[ri];
                const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
                for (int jj = ii + 1 + tid; jj < b; jj += kNmsThreads) {
                    const int rj = (int)(unsigned)keys[jj];
                    if (removed[rj]) continue;
                    const float4 bj = sbox[rj];
                    const float aj = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
                    if (iou_ref(bi, ai, bj, aj) > p.iou_thr) removed[rj] = 1;
                }
                __syncthreads();
            }
        }
        // kept boxes in global rank (score) order
        cnt = 0;
        for (int i = i0; i < i1; ++i) cnt += removed[i] ? 0 : 1;
        int k = block_exclusive_scan(cnt, s_scan);
        for (int i = i0; i < i1; ++i) {
            if (removed[i]) continue;
            const int sidx = (int)pay[i];
            write_det(p, n, k, sbox[i], cscore[sidx], csrc[sidx], offmul);
            ++k;
        }
        if (tid == 0) p.out_count[n] = s_scan[32];
        return;
    }

    // 4b. greedy sweep (whole CTA in lock step; `removed` is only written between barriers)
    for (int i = 0; i < K; ++i) {
        if (removed[i]) continue;  // uniform
        const float4 bi = sbox[i];
        const float ai = __fmul_rn(__fsub_rn(bi.z, bi.x), __fsub_rn(bi.w, bi.y));
        if (tid == 0) {
            const int s = (int)pay[i];
            write_det(p, n, s_keep++, bi, cscore[s], csrc[s], offmul);
        }
        for (int j = i + 1 + tid; j < K; j += kNmsThreads) {
            if (removed[j]) continue;
            const float4 bj = sbox[j];
            const float aj = __fmul_rn(__fsub_rn(bj.z, bj.x), __fsub_rn(bj.w, bj.y));
            if (iou_ref(bi, ai, bj, aj) > p.iou_thr) removed[j] = 1;
        }
        __syncthreads();
    }
    if (tid == 0) p.out_count[n] = s_keep;
}

// ---------------------------------------------------------------------------------------------------
// Soft-NMS (nms_cpu.cpp:76-206 behind utils/nms.py:62-158): one CTA per image runs the reference's in-place loop over ONE array
// holding every class (per-class CTAs would differ: the swaps of one class move positions that decide the ties of another).
//   0. the candidates are sorted by source index, which is the reference's initial order (input rows, or nonzero() of the
//      thresholded (point, class) grid); class-aware mode adds label * (max coordinate + 1) in fp32 as the hard path does
//   per iteration i over the n live positions:
//   1. select: one block reduction of key = desc_key(score) << 32 | position over [i, n) -- the FIRST position of the maximum
//      (the reference scans with `max < s[pos]`, so -0 ties +0, a NaN at i is selected, a NaN behind i never is)
//   2. swap the selected element m with i (only the element at i has to move: position i is never read again) and emit row i
//   3. reweight (i, n): linear w = ovr > thr ? 1 - ovr : 1, gaussian w = (float)exp((double)(-(ovr * ovr) / sigma)); an element
//      whose new score is < min_score is removed
//   4. only when the block votes a removal: reproduce the reference's swap-with-last compaction as a permutation -- the j-th lowest
//      removed position below the new count receives the j-th highest surviving position at or above it (the weights do not depend
//      on the position, so reweighting everything first and permuting afterwards gives the same array)
// Layout (shared memory up to kSoftSmem entries, else the image's global scratch): box float4 [L] (class-offset boxes; areas are
// recomputed) | (score, src) float2 [Lp] (the u64 sort keys before step 0 ends) | hole table int [L / 2 + 1] | removed flags u8 [L].
// Arithmetic that decides the results uses _rn intrinsics: linear mode is bit-exact against the reference's fp32 loop.
static constexpr int kSoftSmem = 8192;
static constexpr size_t kSoftSmemBytes = (size_t)kSoftSmem * 24 + ((size_t)kSoftSmem / 2 + 1) * 4 + kSoftSmem;   // 216 KB

__global__ void __launch_bounds__(kNmsThreads) soft_nms_kernel(const SoftNmsParams sp) {
    extern __shared__ __align__(16) uint8_t ssm[];
    __shared__ float s_red[32], s_red2[32];
    __shared__ unsigned long long s_min[32];
    __shared__ int s_scan[33];
    const NmsParams& p = sp.nms;
    const int n = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31;
    int K = p.cand_count[n];
    if (K > p.cap) {  // capacity overflow: report, process the first cap (host turns this into an error)
        if (tid == 0) atomicExch(p.overflow, 1);
        K = p.cap;
    }
    if (K == 0) {
        if (tid == 0) p.out_count[n] = 0;
        return;
    }
    int Kp = 1;
    while (Kp < K) Kp <<= 1;
    const bool in_smem = K <= kSoftSmem;
    const size_t L = in_smem ? kSoftSmem : p.cap, Lp = in_smem ? kSoftSmem : p.cap_pow2;
    uint8_t* base = in_smem ? ssm : p.scratch + (size_t)n * p.scratch_stride;
    float4* box = reinterpret_cast<float4*>(base);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(base + L * 16);
    float2* ss = reinterpret_cast<float2*>(keys);
    int* holes = reinterpret_cast<int*>(base + L * 16 + Lp * 8);
    uint8_t* gone = reinterpret_cast<uint8_t*>(holes + L / 2 + 1);
    const float4* cbox = reinterpret_cast<const float4*>(p.cand_box) + (size_t)n * p.cap;
    const float* cscore = p.cand_score + (size_t)n * p.cap;
    const int* csrc = p.cand_src + (size_t)n * p.cap;

    float mx = -3.4e38f, mn = 3.4e38f;
    if (!p.class_agnostic) block_box_extent(cbox, K, s_red, s_red2, mx, mn);
    const float offmul = __fadd_rn(mx, 1.0f);

    // 0. reference order: sort by source index (unique per image), candidate slot in the low word
    for (int i = tid; i < Kp; i += kNmsThreads)
        keys[i] = i < K ? (((unsigned long long)(unsigned)csrc[i] << 32) | (unsigned)i) : ~0ull;
    __syncthreads();
    block_bitonic_sort(keys, nullptr, Kp);
    for (int i = tid; i < K; i += kNmsThreads) {
        const int c = (int)(unsigned)keys[i];     // ss[i] overwrites keys[i]: same thread, same address
        const int src = csrc[c];
        float4 b = cbox[c];
        if (!p.class_agnostic) {
            const float off = __fmul_rn((float)(src % p.C), offmul);
            b.x = __fadd_rn(b.x, off); b.y = __fadd_rn(b.y, off); b.z = __fadd_rn(b.z, off); b.w = __fadd_rn(b.w, off);
        }
        box[i] = b;
        ss[i] = make_float2(cscore[c], __int_as_float(src));
    }
    __syncthreads();

    const float thr = p.iou_thr, sigma = sp.sigma, min_score = sp.min_score;
    const bool linear = sp.method == 1;
    int cnt = K;   // live positions (block-uniform)
    for (int i = 0; i < cnt; ++i) {
        // 1. selection
        unsigned long long best = ~0ull;
        for (int q = i + tid; q < cnt; q += kNmsThreads) {
            const float s = ss[q].x;
            unsigned long long k;
            if (s != s) k = q == i ? (unsigned long long)(unsigned)i : ~0ull;   // desc_key never yields 0 for a number
            else k = ((unsigned long long)desc_key(s == 0.f ? 0.f : s) << 32) | (unsigned)q;
            best = k < best ? k : best;
        }
        for (int o = 16; o; o >>= 1) {
            const unsigned long long t = __shfl_xor_sync(0xffffffffu, best, o);
            best = t < best ? t : best;
        }
        if (lane == 0) s_min[tid >> 5] = best;
        __syncthreads();
        best = s_min[0];
        for (int w = 1; w < kNmsThreads / 32; ++w) best = s_min[w] < best ? s_min[w] : best;
        const int m = (int)(unsigned)best;
        const float4 bm = box[m];
        const float2 em = ss[m];
        const float am = box_area(bm);
        if (tid == 0) write_det(p, n, i, bm, em.x, __float_as_int(em.y), offmul);
        __syncthreads();   // position m is rewritten below

        // 2 + 3. the element at i moves to m; reweight (i, cnt)
        bool any_gone = false;
        for (int q = i + 1 + tid; q < cnt; q += kNmsThreads) {
            const int from = q == m ? i : q;
            const float4 b = box[from];
            float2 e = ss[from];
            const float ovr = iou_ref(bm, am, b, box_area(b));
            float w = 1.f;
            if (linear) {
                if (ovr > thr) w = __fsub_rn(1.f, ovr);
            } else {
                w = (float)exp((double)__fdiv_rn(-__fmul_rn(ovr, ovr), sigma));
            }
            e.x = __fmul_rn(w, e.x);
            const bool g = e.x < min_score;
            if (q == m) box[q] = b;
            ss[q] = e;
            gone[q] = g;
            any_gone |= g;
        }
        if (!__syncthreads_or(any_gone)) continue;

        // 4. compaction (each thread owns a run of consecutive positions of (i, cnt))
        const int a = i + 1, len = cnt - a;
        const int per = (len + kNmsThreads - 1) / kNmsThreads;
        const int q0 = min(a + tid * per, cnt), q1 = min(q0 + per, cnt);
        int c = 0;
        for (int q = q0; q < q1; ++q) c += gone[q];
        const int before = block_exclusive_scan(c, s_scan);   // removed positions in [a, q0)
        const int removed = s_scan[32];
        const int n2 = cnt - removed, survivors = len - removed;
        int r = before;
        for (int q = q0; q < q1; ++q)
            if (gone[q]) {
                if (q < n2) holes[r] = q;                      // removed positions below n2 come first: rank among the holes = r
                ++r;
            }
        __syncthreads();
        r = before;
        for (int q = q0; q < q1; ++q) {
            if (gone[q]) { ++r; continue; }
            if (q >= n2) {
                const int h = holes[survivors - ((q - a + 1) - r)];   // rank from the top = survivors in (q, cnt)
                box[h] = box[q];
                ss[h] = ss[q];
            }
        }
        __syncthreads();
        cnt = n2;
    }
    if (tid == 0) p.out_count[n] = cnt;
}

cudaError_t soft_nms_launch(const SoftNmsParams& p, int n_images, cudaStream_t st) {
    static bool attr[kMaxDevices] = {};   // per-device function attribute
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!attr[dev]) {
        cudaError_t e = cudaFuncSetAttribute(soft_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSoftSmemBytes);
        if (e != cudaSuccess) return e;
        attr[dev] = true;
    }
    soft_nms_kernel<<<n_images, kNmsThreads, kSoftSmemBytes, st>>>(p);
    return cudaGetLastError();
}

cudaError_t candidates_launch(const PostParams& p, int num_sms, cudaStream_t st) {
    if (p.cls_mode == 0 && p.C > 1) {
        const long long total = (long long)p.P * p.cls_stride;
        long long blocks = (total + 255) / 256;
        const long long cap = (long long)(num_sms > 0 ? num_sms : 132) * 8;     // grid-stride beyond 8 blocks per SM and image
        if (blocks > cap) blocks = cap;
        candidates_flat_kernel<<<dim3((unsigned)blocks, p.N), 256, 0, st>>>(p);
    } else if (p.cls_stride > 1 && (size_t)kRowsPts * p.cls_stride * 4 <= 48 * 1024) {
        candidates_rows_kernel<<<dim3((p.P + kRowsPts - 1) / kRowsPts, p.N), kRowsPts, (size_t)kRowsPts * p.cls_stride * 4, st>>>(p);
    } else {
        candidates_kernel<<<dim3((p.P + 255) / 256, p.N), 256, 0, st>>>(p);
    }
    return cudaGetLastError();
}

size_t nms_scratch_stride(int cap, int cap_pow2) {
    size_t s = (size_t)cap_pow2 * 12 + (size_t)cap * 16 + (size_t)cap;
    return (s + 255) & ~(size_t)255;
}

cudaError_t nms_launch(const NmsParams& p, int n_images, cudaStream_t st) {
    const size_t smem = kNmsMaskOff + (size_t)kNmsMaskMax * 128;   // 160 KB (>= the 4096-entry sweep layout, 116 KB)
    static bool attr[kMaxDevices] = {};   // per-device function attribute
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!attr[dev]) {
        cudaError_t e = cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        attr[dev] = true;
    }
    nms_kernel<<<n_images, kNmsThreads, smem, st>>>(p);
    return cudaGetLastError();
}

}  // namespace lfd
