// input.cu -- the training input batch (lfd_input_batch): resize + crop + flip + channel order + normalisation of every image of a
// batch in one launch, bit-exact against cv2.resize (INTER_LINEAR / the INTER_AREA special case for 1/s == 2) and crop_from_image.
//
// One CTA per (image, band of kBandRows output rows).  The CTA first builds a per-output-column table in shared memory (source
// column and weights, or "zero" / "padding"), then each thread produces four consecutive pixels of a row: it reads their 2x2 source
// neighbourhoods directly from the window (the resized image is never materialised) and writes 12 bytes (uint8 NHWC) or one float4
// per channel plane (fp32 NCHW), so consecutive threads store consecutive addresses.  The gray modes (uint8 [n,H,W], fp32 [n,1,H,W])
// convert a BGR source to gray at every tap they read, then resize the gray values; they store 4 bytes or one float4.
#include "../../include/lfd_b200.h"
#include "kernels.cuh"

namespace lfd {
namespace {

constexpr int kBandRows = 4;
constexpr int kThreads = 256;
constexpr int kPad = -2, kZero = -1;   // column / row table: outside the image's out size, outside R (raw pixel 0)

// cv2's source coordinate of resized index d: f = float((d + 0.5) * (1/s) - 0.5) in double, i = floor(f), a = f - i
__device__ __forceinline__ void src_coord(int d, double inv, int* i, float* a) {
    const float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, inv), 0.5);
    *i = (int)floorf(f);
    *a = f - (float)*i;
}
__device__ __forceinline__ int weight(float a) { return __float2int_rn(a * 2048.f); }   // saturate_cast<short>(a * 2048): round half to even

// column entry: x = source column of the first tap relative to the window (or kZero / kPad);
// y = a0 | a1 << 12 | (second tap exists) << 24 (LINEAR: a1 > 0 reads column x + 1; AREA2: the block has two columns)
__device__ int2 column_entry(const lfd_input_desc& d, int x) {
    if (x >= d.out_w) return make_int2(kPad, 0);
    const int c = d.crop_x + (d.flip ? d.out_w - 1 - x : x);
    if (c < 0 || c >= d.dw) return make_int2(kZero, 0);
    if (d.mode == LFD_RESIZE_COPY) return make_int2(c - d.win_x, 2048);
    if (d.mode == LFD_RESIZE_AREA2) return make_int2(2 * c - d.win_x, (2 * c + 1 < d.src_w) << 24);
    int i;
    float a;
    src_coord(c, d.inv_scale, &i, &a);
    if (i < 0) i = 0, a = 0.f;                                   // cv2 clamps the tap and zeroes its weight at both borders
    if (i >= d.src_w - 1) i = d.src_w - 1, a = 0.f;
    const int a0 = weight(1.f - a), a1 = weight(a);
    return make_int2(i - d.win_x, a0 | a1 << 12 | (a1 > 0) << 24);
}

struct RowInfo {
    const uint8_t* r0;   // first source row (window relative), null for kZero / kPad rows
    const uint8_t* r1;   // second source row
    int b0, b1;          // LINEAR: vertical weights; AREA2: b1 = 1 when the block has two rows
    int kind;            // 0 = pixel row, kZero, kPad
};

__device__ RowInfo row_info(const lfd_input_desc& d, const uint8_t* win, int y) {
    RowInfo ri{nullptr, nullptr, 2048, 0, 0};
    if (y >= d.out_h) { ri.kind = kPad; return ri; }
    const int r = d.crop_y + y;
    if (r < 0 || r >= d.dh || d.win_h <= 0) { ri.kind = kZero; return ri; }
    int y0 = r, y1 = r;
    if (d.mode == LFD_RESIZE_AREA2) {
        y0 = 2 * r;
        y1 = min(y0 + 1, d.src_h - 1);
        ri.b1 = y0 + 1 < d.src_h;
    } else if (d.mode == LFD_RESIZE_LINEAR) {
        int i;
        float a;
        src_coord(r, d.inv_scale, &i, &a);
        ri.b0 = weight(1.f - a);                                 // rows clamp the indices only (clip() in cv2's resize invoker)
        ri.b1 = weight(a);
        y0 = min(max(i, 0), d.src_h - 1);
        y1 = min(max(i + 1, 0), d.src_h - 1);
    }
    // a descriptor whose window misses a row it needs gives wrong pixels, never an out-of-bounds read
    y0 = min(max(y0 - d.win_y, 0), d.win_h - 1);
    y1 = min(max(y1 - d.win_y, 0), d.win_h - 1);
    ri.r0 = win + (size_t)y0 * d.pitch;
    ri.r1 = win + (size_t)y1 * d.pitch;
    return ri;
}

// one channel of one output pixel of the gray modes from its source taps: tap(row, x) is the value the resize reads at window column x
// of a source row.  The same arithmetic as pixel() below, which the 3-channel modes run.
template <class Tap>
__device__ __forceinline__ int resample(const lfd_input_desc& d, const RowInfo& ri, int2 col, int x0, int x1, Tap tap) {
    const int two = col.y >> 24 & 1;
    const int p00 = tap(ri.r0, x0);
    if (d.mode == LFD_RESIZE_COPY) return p00;
    if (d.mode == LFD_RESIZE_AREA2) {
        int sum = p00 + (two ? tap(ri.r0, x1) : 0);
        if (ri.b1) sum += tap(ri.r1, x0) + (two ? tap(ri.r1, x1) : 0);
        const int count = (1 + two) * (1 + ri.b1);
        return count == 4 ? (sum + 2) >> 2 : __float2int_rn((float)sum / (float)count);   // partial blocks: sum / count, half to even
    }
    const int a0 = col.y & 0xfff, a1 = col.y >> 12 & 0xfff;
    const int h0 = p00 * a0 + (two ? tap(ri.r0, x1) * a1 : 0);
    const int h1 = tap(ri.r1, x0) * a0 + (two ? tap(ri.r1, x1) * a1 : 0);
    return min((((h0 >> 4) * ri.b0 >> 16) + ((h1 >> 4) * ri.b1 >> 16) + 2) >> 2, 255);
}

// one output pixel: channel k of the source order in bits 8k..8k+7 (a gray source replicated)
__device__ __forceinline__ uint32_t pixel(const lfd_input_desc& d, const RowInfo& ri, int2 col) {
    if (ri.kind != 0 || col.x < 0 || d.win_w <= 0) return 0u;
    const int C = d.channels, wmax = d.win_w - 1;
    const int x0 = min(max(col.x, 0), wmax);
    const int x1 = min(max(col.x + 1, 0), wmax);
    const int two = col.y >> 24 & 1;
    uint32_t packed = 0u;
    for (int k = 0; k < C; ++k) {
        const int p00 = ri.r0[x0 * C + k];
        int out;
        if (d.mode == LFD_RESIZE_COPY) {
            out = p00;
        } else if (d.mode == LFD_RESIZE_AREA2) {
            int sum = p00 + (two ? ri.r0[x1 * C + k] : 0);
            if (ri.b1) sum += ri.r1[x0 * C + k] + (two ? ri.r1[x1 * C + k] : 0);
            const int count = (1 + two) * (1 + ri.b1);
            out = count == 4 ? (sum + 2) >> 2 : __float2int_rn((float)sum / (float)count);   // partial blocks: sum / count, half to even
        } else {
            const int a0 = col.y & 0xfff, a1 = col.y >> 12 & 0xfff;
            const int h0 = p00 * a0 + (two ? ri.r0[x1 * C + k] * a1 : 0);
            const int h1 = ri.r1[x0 * C + k] * a0 + (two ? ri.r1[x1 * C + k] * a1 : 0);
            out = min((((h0 >> 4) * ri.b0 >> 16) + ((h1 >> 4) * ri.b1 >> 16) + 2) >> 2, 255);
        }
        packed |= (uint32_t)out << (8 * k);
    }
    return C == 1 ? packed * 0x010101u : packed;
}

// one output pixel of a gray mode: the gray value, a BGR source converted tap by tap (bgr_to_gray) before the resize arithmetic of
// pixel(), as cv2.resize of cv2.cvtColor(BGR2GRAY) computes it.  The 3-channel modes keep pixel() as it is, so their code does not change.
__device__ __forceinline__ uint32_t gray_pixel(const lfd_input_desc& d, const RowInfo& ri, int2 col) {
    if (ri.kind != 0 || col.x < 0 || d.win_w <= 0) return 0u;
    const int wmax = d.win_w - 1;
    const int x0 = min(max(col.x, 0), wmax);
    const int x1 = min(max(col.x + 1, 0), wmax);
    if (d.channels == 1) return resample(d, ri, col, x0, x1, [](const uint8_t* r, int x) { return (int)r[x]; });
    return resample(d, ri, col, x0, x1, [](const uint8_t* r, int x) { return (int)bgr_to_gray(r[3 * x], r[3 * x + 1], r[3 * x + 2]); });
}

template <int OUT_MODE>
__global__ void __launch_bounds__(kThreads) input_batch_kernel(const lfd_input_desc* __restrict__ descs, const uint8_t* __restrict__ src,
                                                               void* __restrict__ out, int swap_rb, int H, int W, float3 mean, float3 scale) {
    extern __shared__ int2 cols[];   // [W]
    const int img = blockIdx.y;
    const lfd_input_desc d = descs[img];
    for (int x = threadIdx.x; x < W; x += kThreads) cols[x] = column_entry(d, x);
    __syncthreads();
    const uint8_t* win = src + d.src_off;
    const int groups = (W + 3) >> 2;
    const int y_begin = blockIdx.x * kBandRows;
    const int rows = min(kBandRows, H - y_begin);
    for (int t = threadIdx.x; t < rows * groups; t += kThreads) {
        const int y = y_begin + t / groups, x = (t % groups) * 4;
        const RowInfo ri = row_info(d, win, y);
        constexpr bool gray = OUT_MODE == LFD_INPUT_OUT_U8_GRAY || OUT_MODE == LFD_INPUT_OUT_F32_GRAY;
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            v[j] = x + j < W ? (gray ? gray_pixel(d, ri, cols[x + j]) : pixel(d, ri, cols[x + j])) : 0u;
            if (!gray && swap_rb) v[j] = (v[j] & 0x00ff00u) | (v[j] >> 16 & 0xffu) | (v[j] & 0xffu) << 16;
        }
        const int n = min(4, W - x);
        if constexpr (OUT_MODE == LFD_INPUT_OUT_U8_NHWC) {
            uint8_t* o = reinterpret_cast<uint8_t*>(out) + (((size_t)img * H + y) * W + x) * 3;
            if (n == 4 && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
                uint32_t* ow = reinterpret_cast<uint32_t*>(o);
                ow[0] = v[0] | v[1] << 24;
                ow[1] = v[1] >> 8 | v[2] << 16;
                ow[2] = v[2] >> 16 | v[3] << 8;
            } else {
                for (int j = 0; j < n * 3; ++j) o[j] = (uint8_t)(v[j / 3] >> (8 * (j % 3)));
            }
        } else if constexpr (OUT_MODE == LFD_INPUT_OUT_F32_NCHW) {
            const float m[3] = {mean.x, mean.y, mean.z}, s[3] = {scale.x, scale.y, scale.z};
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float f[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int2 e = x + j < W ? cols[x + j] : make_int2(kPad, 0);
                    f[j] = (ri.kind == kPad || e.x == kPad) ? 0.f : __fmul_rn(__fsub_rn((float)(v[j] >> (8 * c) & 0xffu), m[c]), s[c]);
                }
                float* o = reinterpret_cast<float*>(out) + (((size_t)img * 3 + c) * H + y) * W + x;
                if (n == 4 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
                    *reinterpret_cast<float4*>(o) = make_float4(f[0], f[1], f[2], f[3]);
                } else {
                    for (int j = 0; j < n; ++j) o[j] = f[j];
                }
            }
        } else if constexpr (OUT_MODE == LFD_INPUT_OUT_U8_GRAY) {
            uint8_t* o = reinterpret_cast<uint8_t*>(out) + ((size_t)img * H + y) * W + x;
            if (n == 4 && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
                *reinterpret_cast<uint32_t*>(o) = v[0] | v[1] << 8 | v[2] << 16 | v[3] << 24;
            } else {
                for (int j = 0; j < n; ++j) o[j] = (uint8_t)v[j];
            }
        } else {   // LFD_INPUT_OUT_F32_GRAY: one plane, one constant pair (mean.x, scale.x)
            float f[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int2 e = x + j < W ? cols[x + j] : make_int2(kPad, 0);
                f[j] = (ri.kind == kPad || e.x == kPad) ? 0.f : __fmul_rn(__fsub_rn((float)v[j], mean.x), scale.x);
            }
            float* o = reinterpret_cast<float*>(out) + ((size_t)img * H + y) * W + x;
            if (n == 4 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
                *reinterpret_cast<float4*>(o) = make_float4(f[0], f[1], f[2], f[3]);
            } else {
                for (int j = 0; j < n; ++j) o[j] = f[j];
            }
        }
    }
}

}  // namespace

cudaError_t input_batch_launch(const void* descs, int n, const uint8_t* src, void* out, int out_mode, int swap_rb, int H, int W,
                               const float* mean, const float* scale, cudaStream_t st) {
    const dim3 grid((H + kBandRows - 1) / kBandRows, n);
    const size_t smem = (size_t)W * sizeof(int2);
    const lfd_input_desc* d = reinterpret_cast<const lfd_input_desc*>(descs);
    const float3 zero = make_float3(0.f, 0.f, 0.f);
    if (out_mode == LFD_INPUT_OUT_U8_NHWC) {
        input_batch_kernel<LFD_INPUT_OUT_U8_NHWC><<<grid, kThreads, smem, st>>>(d, src, out, swap_rb, H, W, zero, zero);
    } else if (out_mode == LFD_INPUT_OUT_F32_NCHW) {
        input_batch_kernel<LFD_INPUT_OUT_F32_NCHW><<<grid, kThreads, smem, st>>>(d, src, out, swap_rb, H, W, make_float3(mean[0], mean[1], mean[2]),
                                                                              make_float3(scale[0], scale[1], scale[2]));
    } else if (out_mode == LFD_INPUT_OUT_U8_GRAY) {
        input_batch_kernel<LFD_INPUT_OUT_U8_GRAY><<<grid, kThreads, smem, st>>>(d, src, out, 0, H, W, zero, zero);
    } else {
        input_batch_kernel<LFD_INPUT_OUT_F32_GRAY><<<grid, kThreads, smem, st>>>(d, src, out, 0, H, W, make_float3(mean[0], 0.f, 0.f),
                                                                              make_float3(scale[0], 0.f, 0.f));
    }
    return cudaGetLastError();
}

}  // namespace lfd
