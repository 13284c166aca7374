// image.cuh -- what a pixel of the input image is, for every kernel that reads the image (internal, not part of the C-ABI).
// The device code that knows the formats (LFD_INPUT_*), the input transform and the channel order for every reader but the MODE_STEM
// producer of conv_umma.cu, which keeps its own loader on the same ImageIn (routed through these helpers, its stem op ran about 12 %
// slower on uint8 BGR frames; DESIGN.md, section 1, "Gray (1-channel) models").  A reader loads a pixel's raw
// words (image_load, or image_load_words + image_unpack_word), decodes them to the three network-channel values (image_decode) and,
// for the stem's wgmma operand, packs those (pack_px).  The channel count CH (3 = BGR, 1 = gray) and the format FMT are template
// parameters: a reader picks its body once per launch (image_dispatch), and no pixel pays a run-time format or channel branch.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/lfd_b200.h"
#include "ptx.cuh"

namespace lfd {

// What every kernel that reads a uint8 image makes of it: network input channel c of a pixel = apply(m, byte[m]) with m = swap ? 2 - c : c,
// in fp32 one subtract, then one multiply: albumentations' Normalize after an optional BGR -> RGB, with the constants Normalize itself
// computes.  mean / scale are indexed by the byte's position m IN MEMORY (api.cu permutes the C-ABI's per-network-channel constants once),
// so a loader normalises the three bytes where they lie and a swap only exchanges two finished floats.  Pixels outside the image are 0
// AFTER this (the conv's zero padding), not the image of byte 0.
struct InputTransform {
    int swap;
    float mean[3], scale[3];
    __host__ __device__ __forceinline__ float apply(int m, uint32_t byte) const { return ((float)byte - mean[m]) * scale[m]; }
};

// LFD_INPUT_U8_NV12: the three bytes (B, G, R) of a pixel from its Y byte and the (U, V) pair of its 2x2 block -- BT.601 limited
// range in 20-bit fixed point, bit for bit what cv2.cvtColor(f, COLOR_YUV2BGR_NV12) gives.  The only code that knows the constants.
__host__ __device__ __forceinline__ uint32_t nv12_sat8(int v) { return (uint32_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
__host__ __device__ __forceinline__ void nv12_to_bgr(uint32_t Y, uint32_t U, uint32_t V, uint32_t bgr[3]) {
    const int y = ((int)Y > 16 ? (int)Y - 16 : 0) * 1220542 + (1 << 19);     // max(0, Y - 16) * 1220542 + the rounding half
    const int u = (int)U - 128, v = (int)V - 128;
    bgr[0] = nv12_sat8((y + 2116026 * u) >> 20);                           // arithmetic shifts
    bgr[1] = nv12_sat8((y - 852492 * v - 409993 * u) >> 20);
    bgr[2] = nv12_sat8((y + 1673527 * v) >> 20);
}

// uint8 B, G, R -> gray in 15-bit fixed point, bit for bit what cv2.cvtColor(img, COLOR_BGR2GRAY) gives on uint8 (all 2^24 triples; the
// often-quoted 14-bit constants 1868 / 9617 / 4899 differ on 43 864 of them).  The training input kernel's gray modes (input.cu).
__host__ __device__ __forceinline__ uint32_t bgr_to_gray(uint32_t b, uint32_t g, uint32_t r) {
    return (3735u * b + 19235u * g + 9798u * r + 16384u) >> 15;
}

// The input image of a batch: fp32 NCHW float[N][ch][H][W], uint8 NHWC uint8[N][H][W][ch], or NV12 (image n = an H x W Y plane, then the
// interleaved (U, V) plane of H / 2 rows at the same pitch; ch = 1 reads the Y plane only).  H x W is the tensor's (the pitch); a smaller
// frame lies in its top-left corner.  xf.swap is 0 for fp32 input: its planes are taken as they are.
struct ImageIn {
    const void* data;
    int format;                 // LFD_INPUT_F32_NCHW, LFD_INPUT_U8_NHWC or LFD_INPUT_U8_NV12
    int ch;                     // 3 (BGR) or 1 (gray)
    int H, W;
    InputTransform xf;
};

// f(CH, FMT) with the image's channel count and format as std::integral_constant: the body a reader runs for this image
template <class F>
LFD_DEVINL void image_dispatch(const ImageIn& im, F&& f) {
    using C1 = std::integral_constant<int, 1>;
    using C3 = std::integral_constant<int, 3>;
    using NV12 = std::integral_constant<int, LFD_INPUT_U8_NV12>;
    using U8 = std::integral_constant<int, LFD_INPUT_U8_NHWC>;
    using F32 = std::integral_constant<int, LFD_INPUT_F32_NCHW>;
    if (im.ch == 1) {
        if (im.format == LFD_INPUT_U8_NV12) f(C1(), NV12());
        else if (im.format == LFD_INPUT_U8_NHWC) f(C1(), U8());
        else f(C1(), F32());
    } else {
        if (im.format == LFD_INPUT_U8_NV12) f(C3(), NV12());
        else if (im.format == LFD_INPUT_U8_NHWC) f(C3(), U8());
        else f(C3(), F32());
    }
}

// The offset of pixel (y, x) from the first pixel of its image, in the units image_load takes: bytes for uint8 NHWC, elements of a plane
// otherwise.  Linear in (y, x), so a loader may keep the offsets of its pixels relative to a patch origin precomputed.  An int: exact
// while one image has fewer than 2^31 / 3 pixels (the image offset n * H * W is taken in ptrdiff_t by the loaders).
template <int CH, int FMT>
LFD_DEVINL int image_px(const ImageIn& im, int y, int x) { return (y * im.W + x) * (FMT == LFD_INPUT_U8_NHWC ? CH : 1); }

// The raw words of pixel (y, x) of image n at offset o = image_px(y, x): fp32 the CH values as bits, one plane apart; uint8 the CH
// bytes; NV12 the Y byte and, for CH = 3, the U and V bytes of its 2x2 block.  A pixel outside the image (inside = false) loads image
// n's first pixel instead, so the loads need no predicate; image_decode zeroes it.
template <int CH, int FMT>
LFD_DEVINL void image_load(const ImageIn& im, int n, int o, int y, int x, bool inside, uint32_t (&raw)[CH]) {
    const ptrdiff_t plane = (ptrdiff_t)im.H * im.W;
    if (!inside) o = 0;
    if constexpr (FMT == LFD_INPUT_U8_NV12) {
        const uint8_t* img = static_cast<const uint8_t*>(im.data) + n * (plane + (plane >> 1));
        raw[0] = __ldg(img + o);
        if constexpr (CH == 3) {
            const uint8_t* uv = img + plane + (inside ? (ptrdiff_t)(y >> 1) * im.W + (x & ~1) : 0);
            raw[1] = __ldg(uv);
            raw[2] = __ldg(uv + 1);
        }
    } else if constexpr (FMT == LFD_INPUT_U8_NHWC) {
        const uint8_t* src = static_cast<const uint8_t*>(im.data) + n * plane * CH + o;
#pragma unroll
        for (int k = 0; k < CH; ++k) raw[k] = __ldg(src + k);
    } else {
        const float* src = static_cast<const float*>(im.data) + n * plane * CH + o;
#pragma unroll
        for (int k = 0; k < CH; ++k) raw[k] = __float_as_uint(__ldg(src + k * plane));
    }
}

// The word loader of a uint8 image with W % 4 == 0 at a 4-byte aligned address: the aligned words of the 4 pixels x .. x + 3 (x % 4 == 0)
// of row y -- BGR 3 words, gray 1 word; NV12 the Y word and, for CH = 3, the UV word U0 V0 U1 V1 of their two 2x2 blocks (aligned too:
// the NV12 image pitch H * W * 3 / 2 is then a multiple of 4, H being even).  A group outside the image loads nothing and reads as 0.
template <int CH, int FMT>
LFD_DEVINL void image_load_words(const ImageIn& im, int n, int y, int x, bool inside, uint32_t (&wd)[CH]) {
    const ptrdiff_t plane = (ptrdiff_t)im.H * im.W;
    if constexpr (FMT == LFD_INPUT_U8_NV12) {
        const uint8_t* img = static_cast<const uint8_t*>(im.data) + n * (plane + (plane >> 1));
        wd[0] = inside ? __ldg(reinterpret_cast<const uint32_t*>(img + (ptrdiff_t)y * im.W + x)) : 0u;
        if constexpr (CH == 3) {
            wd[1] = inside ? __ldg(reinterpret_cast<const uint32_t*>(img + plane + (ptrdiff_t)(y >> 1) * im.W + x)) : 0u;
            wd[2] = 0u;
        }
    } else {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(static_cast<const uint8_t*>(im.data) + (n * plane + (ptrdiff_t)y * im.W + x) * CH);
#pragma unroll
        for (int k = 0; k < CH; ++k) wd[k] = inside ? __ldg(src + k) : 0u;
    }
}

// Pixel k (0..3) of such a group: its raw words, as image_load gives them
template <int CH, int FMT>
__host__ __device__ __forceinline__ void image_unpack_word(const uint32_t (&wd)[CH], int k, uint32_t (&raw)[CH]) {
    if constexpr (CH == 1) {
        raw[0] = (wd[0] >> (8 * k)) & 0xffu;
    } else if constexpr (FMT == LFD_INPUT_U8_NV12) {
        raw[0] = (wd[0] >> (8 * k)) & 0xffu;
        raw[1] = (wd[1] >> (8 * (k & 2))) & 0xffu;
        raw[2] = (wd[1] >> (8 * (k & 2) + 8)) & 0xffu;
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) raw[c] = (wd[(3 * k + c) >> 2] >> (8 * ((3 * k + c) & 3))) & 0xffu;
    }
}

// Raw words -> the three network-channel values of the pixel: NV12 -> (B, G, R) bytes, uint8 bytes through xf by byte position, fp32 as
// it is, 0 outside the image (the conv's zero padding, after the transform); BGR -> RGB exchanges two finished floats (a swap of the bytes
// costs the stem4 producers a stack frame); gray is (v, 0, 0).
template <int CH, int FMT>
LFD_DEVINL void image_decode(const ImageIn& im, const uint32_t (&raw)[CH], bool inside, float (&f)[3]) {
    constexpr bool u8 = FMT != LFD_INPUT_F32_NCHW;
    if constexpr (CH == 1) {
        f[0] = inside ? (u8 ? im.xf.apply(0, raw[0]) : __uint_as_float(raw[0])) : 0.f;
        f[1] = f[2] = 0.f;
    } else {
        uint32_t b[3] = {raw[0], raw[1], raw[2]};
        if constexpr (FMT == LFD_INPUT_U8_NV12) nv12_to_bgr(raw[0], raw[1], raw[2], b);
        float v[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) v[k] = inside ? (u8 ? im.xf.apply(k, b[k]) : __uint_as_float(b[k])) : 0.f;
        const bool sw = im.xf.swap;
        f[0] = sw ? v[2] : v[0];
        f[1] = v[1];
        f[2] = sw ? v[0] : v[2];
    }
}

// The stem's wgmma operand: one pixel as [c0 c1 c2 0] in the 16-bit type, rounded here (rounding point R0)
template <bool F16>
LFD_DEVINL uint2 pack_px(const float (&f)[3]) { return make_uint2(pack2<F16>(f[0], f[1]), pack2<F16>(f[2], 0.f)); }

}  // namespace lfd
