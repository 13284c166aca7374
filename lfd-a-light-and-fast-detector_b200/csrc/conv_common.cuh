// conv_common.cuh -- shared declarations of the convolution kernels (internal, not part of the C-ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>
#include "kernels.cuh"

namespace lfd {

// MODE_STEM4: the four convolutions of the 'faster' stem (3x3/s2 3->64, 1x1, 3x3/s2 64->64, 1x1) in one kernel (stem4_kernel)
enum { MODE_FLAT = 0, MODE_3X3S1 = 1, MODE_3X3S2 = 2, MODE_1X1S2 = 3, MODE_STEM = 4, MODE_STEM4 = 5 };

static constexpr int kMaxStages = 8;
static constexpr int kMaxDevices = 64;   // per-device state (function attributes, SM counts) is indexed by the device ordinal
// dynamic shared memory map of conv_umma_kernel (bytes)
static constexpr int kSmemBarOff = 0;        // mbarriers
static constexpr int kSmemTableOff = 512;    // first per-layer region
// from there, at offsets chosen per layer (UmmaConvParams::smem_*_off): halo pixel table (modes that need it), the fp32 shifts
// of the conv and of the fused tail, then the 1024-byte aligned staging regions [warpgroup][buffer]

struct ConvGeom {
    int N, H, W, Cin, Ho, Wo, Cout, ksize, stride;
    int tail_cout;   // > 0: a 1x1/s1 conv (Cout -> tail_cout) is fused behind this conv (second GEMM in the same kernel)
    int ds_cout;     // > 0 (3x3/s2 only): the residual block's 1x1/s2 shortcut conv (Cin -> ds_cout == Cout) is fused: second output tensor
    int stem;   // 1: 3x3/s2 conv on the raw 3- or 1-channel image (K = 27 padded to 32), operand built by the producers
    int stem4;  // 1: the fused four-conv stem (MODE_STEM4); H x W = the image, Ho x Wo = the stem3 output, Cout = tail_cout = 64
};

struct alignas(64) UmmaConvParams {
    CUtensorMap tm_out;         // TMA descriptor of the stored tensor (epilogue tile store)
    CUtensorMap tm_res;         // TMA descriptor of the residual tensor (same geometry)
    CUtensorMap tm_out3;        // TMA descriptor of the fused shortcut conv's output (same geometry)
    int stg_nbuf;               // staging buffers per warpgroup (2: the store of tile t overlaps the conversion of tile t+1)
    int solo;                   // 1: conv_umma_solo_kernel (one consumer warpgroup per tile, see umma_conv_configure)
    const __nv_bfloat16* in;
    __nv_bfloat16* out;
    const __nv_bfloat16* res;   // optional residual (same shape as out)
    const __nv_bfloat16* w;     // packed [cc][tap][kc][Cout][8]
    const float* shift;         // [Cout] fp32 or null; rounded to the 16-bit type and added to the accumulator (BatchNorm scale is folded into w)
    // fused trailing 1x1 conv ("tail"): out = act2(scale2 * (W2 . act(scale * conv(x) + shift)) + shift2); `out`, `res`,
    // `stats` then refer to the tail's output (Cf channels) and the intermediate never leaves the SM
    const __nv_bfloat16* w2;    // packed [Cout/8][Cout2][8]
    const float* shift2;
    int Cout2, relu2, Cf;       // Cf = channels of the stored tensor (Cout2 with a tail, else Cout)
    // fused 1x1/s2 shortcut conv (MODE_3X3S2, no tail): out3 = W3 . x[centre tap] + shift3; its weights / shift travel in w2 / shift2
    int Cout3;
    __nv_bfloat16* out3;
    uint32_t smem_w2_off;
    double* stats;              // optional [N][groups][2] (sum, sumsq) of the stored output
    unsigned long long* tl;     // debugging: [start, end] of the launch in %globaltimer ns (LFD_B200_TIMELINE builds), normally null
    long long* trace;           // debugging: clock64() timeline of CTA 0 ([role 0..3][entry < 32][4], see conv_umma.cu), normally null
    int N, H, W, Cin, Ho, Wo, Cout;
    int relu, gn_groups, mode;
    int tiles_x, tiles_per_img, num_tiles;
    unsigned long long magic_tpi, magic_tx;   // ceil(2^40 / d) for division-free tile decomposition
    int n_px;                   // halo pixels loaded per stage
    int Cc, stages, b_resident;
    int log2_cpc, log2_cpr;
    uint32_t lbo_a, sbo_a;
    uint32_t a_stage_bytes, b_slice_bytes, stage_bytes, w_total_bytes;
    uint32_t smem_table_off, smem_bias_off, smem_bias2_off, smem_staging_off;
    uint32_t smem_w_off, smem_ring_off;
    ImageIn img;                // MODE_STEM / MODE_STEM4: the image (read from the constant bank)
    int f16;                    // activation / weight type: 0 = bf16, 1 = IEEE fp16 (same bytes, same tensor-core rate)
    // MODE_STEM4: stem0 = w / shift / relu, stem1 = w2 / shift2 / relu2 (the tail fields), stem2 = its 3x3/s2 weights packed
    // [9][8][64][8] + shift + ReLU, stem3 = its 1x1 weights packed [8][64][8] + shift + ReLU; H1 x W1 = the stem1 map
    const __nv_bfloat16* w_s2;
    const float* shift_s2;
    const __nv_bfloat16* w_s3;
    const float* shift_s3;
    int relu_s2, relu_s3, H1, W1;
    int in_words;               // MODE_STEM4: u8 NHWC image with W % 4 == 0 at a 4-byte aligned address -> the producer loads aligned words
    // null: the launch covers the whole tensors (H .. Wo).  Otherwise int4 (H, W, Ho, Wo) in device memory, read when the kernel starts: the
    // valid extent of a smaller frame in the top-left corner of the same tensors (the pitches, the tensor maps and the grid stay those of
    // H .. Wo; bounds, zero padding, statistics and the tile walk follow the valid extent)
    const int* ext;
};

// returns 0 when the geometry is supported by the wgmma kernel
int umma_conv_configure(const ConvGeom& g, int num_sms, UmmaConvParams* out, size_t* smem_bytes, int* grid);
cudaError_t umma_conv_launch(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st);
// fills p->tm_out / p->tm_res from p->out / p->res (host, no launch); returns 0 on success
int umma_conv_encode_maps(UmmaConvParams* p);

// SIMT cross-check kernel (same packed weights, same epilogue semantics); debugging / validation only.
cudaError_t simt_conv_launch(const ConvGeom& g, int Cc, const __nv_bfloat16* in, __nv_bfloat16* out,
                             const __nv_bfloat16* res, const __nv_bfloat16* w, const float* shift,
                             double* stats, int gn_groups, int relu, int f16, cudaStream_t st);

}  // namespace lfd
