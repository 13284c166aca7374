// conv_simt.cu -- the bandwidth-bound / narrow kernels of the LFD forward that are not GEMM shaped, plus a
// SIMT cross-check of the wgmma convolution:
//   stem0_kernel       3x3 stride-2 conv on the 3-channel (or gray) image (K = 27): direct, fused BN scale/shift + ReLU,
//                      reads fp32 NCHW (reference `forward(x)` input) or uint8 HWC BGR with the
//                      (x/255-0.5)/0.5 normalisation fused (reference predict path,
//                      lfd/data_pipeline/augmentation/augmentation_pipeline.py:31-36); writes bf16 NHWC.
//                      Reference: lfd/model/backbone/lfd_resnet.py:356-366 (first conv+BN+ReLU of every stem).
//   gn_apply_kernel    GroupNorm apply + ReLU of a tower layer (lfd/model/head/lfd_head.py:95-106); statistics
//                      were accumulated by the producing conv's epilogue.
//   head_final_kernel  second GroupNorm apply + ReLU fused with the narrow final 1x1 convs (cls C' channels,
//                      reg 4 channels, bias, per-level Scale; lfd_head.py:137-143,164-185) writing fp32 straight
//                      into the (N, P, C') / (N, P, 4) layout of lfd/model/lfd.py:526-540.
//   simt_conv_kernel   direct convolution with the same packed weights and epilogue semantics as conv_umma.cu;
//                      used only to cross-check the tensor-core kernel (tests, conv_impl = LFD_CONV_SIMT).
#include "conv_common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace lfd {

// ===================================================================================================
// stem0
// ===================================================================================================
static constexpr int kS0Threads = 256;
static constexpr int kS0TileH = 4, kS0TileW = 32;        // 128 output pixels per block
static constexpr int kS0PatchH = 2 * kS0TileH + 1;       // 9
static constexpr int kS0PatchW = 2 * kS0TileW + 1;       // 65
static constexpr int kS0PatchPitch = 66;

template <int NG>  // NG = Cout / 8 channel groups
__global__ void __launch_bounds__(kS0Threads) stem0_kernel(const __grid_constant__ Stem0Params p) {
    constexpr int PXP = kS0Threads / NG;   // pixels per pass
    constexpr int PASSES = (128 + PXP - 1) / PXP;
    // NG = 6 (48 channels): 42 pixels per pass, 4 passes, and the last 4 threads idle; the power-of-two widths tile 128 exactly
    constexpr bool kRagged = PXP * PASSES != 128 || PXP * NG != kS0Threads;
    __shared__ float patch[3 * kS0PatchH * kS0PatchPitch];
    __shared__ __align__(16) float wsm[27 * 64];
    const int tid = threadIdx.x;
    const int n = blockIdx.z;
    const int oy0 = blockIdx.y * kS0TileH, ox0 = blockIdx.x * kS0TileW;
    const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
    const int Cout = NG * 8;
    for (int i = tid; i < 27 * Cout; i += kS0Threads) {
        const int k = i / Cout, nn = i % Cout;
        const int kh = k / 9, kw = (k / 3) % 3, ci = k % 3;   // packed [kh][kw / 2][Cout][(kw % 2) * 4 + ci]
        wsm[i] = up_lo_rt((uint32_t)reinterpret_cast<const unsigned short*>(p.w)[(((kh * 2 + (kw >> 1)) * Cout + nn) * 8) + (kw & 1) * 4 + ci], p.f16);
    }
    // input patch -> smem, rounded to bf16 (rounding point R0 of DESIGN.md); a gray image fills channels 1 and 2 with 0
    image_dispatch(p.img, [&](auto ch_c, auto fmt_c) {
        constexpr int CH = decltype(ch_c)::value, FMT = decltype(fmt_c)::value;
        for (int i = tid; i < kS0PatchH * kS0PatchW; i += kS0Threads) {
            const int r = i / kS0PatchW, c = i % kS0PatchW;
            const int y = iy0 + r, x = ix0 + c;
            const bool inside = y >= 0 && y < p.img.H && x >= 0 && x < p.img.W;
            uint32_t raw[CH];
            float f[3];
            image_load<CH, FMT>(p.img, n, image_px<CH, FMT>(p.img, y, x), y, x, inside, raw);
            image_decode<CH, FMT>(p.img, raw, inside, f);
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) patch[(ci * kS0PatchH + r) * kS0PatchPitch + c] = round16_rt(f[ci], p.f16);
        }
    });
    __syncthreads();
    const int g = tid % NG, lp0 = tid / NG;
    float acc[PASSES][8];
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[ps][j] = 0.f;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
        const int kh = tap / 3, kw = tap % 3;
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
            const float4 w0 = *reinterpret_cast<const float4*>(&wsm[(tap * 3 + ci) * Cout + g * 8]);
            const float4 w1 = *reinterpret_cast<const float4*>(&wsm[(tap * 3 + ci) * Cout + g * 8 + 4]);
#pragma unroll
            for (int ps = 0; ps < PASSES; ++ps) {
                const int lp = ps * PXP + lp0;
                if (kRagged && (lp0 >= PXP || lp >= 128)) continue;
                const int ly = lp / kS0TileW, lx = lp % kS0TileW;
                const float x = patch[(ci * kS0PatchH + 2 * ly + kh) * kS0PatchPitch + 2 * lx + kw];
                acc[ps][0] = fmaf(x, w0.x, acc[ps][0]); acc[ps][1] = fmaf(x, w0.y, acc[ps][1]);
                acc[ps][2] = fmaf(x, w0.z, acc[ps][2]); acc[ps][3] = fmaf(x, w0.w, acc[ps][3]);
                acc[ps][4] = fmaf(x, w1.x, acc[ps][4]); acc[ps][5] = fmaf(x, w1.y, acc[ps][5]);
                acc[ps][6] = fmaf(x, w1.z, acc[ps][6]); acc[ps][7] = fmaf(x, w1.w, acc[ps][7]);
            }
        }
    }
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = 1.0f; sh[j] = p.shift ? round16_rt(p.shift[g * 8 + j], p.f16) : 0.f; }
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps) {
        const int lp = ps * PXP + lp0;
        if (kRagged && (lp0 >= PXP || lp >= 128)) continue;
        const int oy = oy0 + lp / kS0TileW, ox = ox0 + lp % kS0TileW;
        if (oy >= p.Ho || ox >= p.Wo) continue;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j] = fmaf(acc[ps][j], sc[j], sh[j]);
            if (p.relu) o[j] = fmaxf(o[j], 0.f);
        }
        uint4 ov;
        ov.x = pack2_rt(o[0], o[1], p.f16); ov.y = pack2_rt(o[2], o[3], p.f16);
        ov.z = pack2_rt(o[4], o[5], p.f16); ov.w = pack2_rt(o[6], o[7], p.f16);
        *reinterpret_cast<uint4*>(p.out + (((size_t)n * p.Ho + oy) * p.Wo + ox) * Cout + g * 8) = ov;
    }
}

cudaError_t stem0_launch(const Stem0Params& p, cudaStream_t st) {
    dim3 grid((p.Wo + kS0TileW - 1) / kS0TileW, (p.Ho + kS0TileH - 1) / kS0TileH, p.N);
    switch (p.Cout) {
        case 64: stem0_kernel<8><<<grid, kS0Threads, 0, st>>>(p); break;
        case 48: stem0_kernel<6><<<grid, kS0Threads, 0, st>>>(p); break;
        case 32: stem0_kernel<4><<<grid, kS0Threads, 0, st>>>(p); break;
        case 16: stem0_kernel<2><<<grid, kS0Threads, 0, st>>>(p); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// ===================================================================================================
// GroupNorm apply (+ReLU), bf16 -> bf16.  Group size must be 8 channels (one 16-byte chunk).
// ===================================================================================================
__device__ __forceinline__ void gn_mean_rstd(const double* stats, int n, int g, int groups, double count, float eps,
                                             float* mean, float* rstd) {
    const double s1 = stats[((size_t)n * groups + g) * 2], s2 = stats[((size_t)n * groups + g) * 2 + 1];
    const double m = s1 / count;
    double var = s2 / count - m * m;
    if (var < 0) var = 0;
    *mean = (float)m;
    *rstd = (float)(1.0 / sqrt(var + (double)eps));
}

template <bool F16>
__global__ void __launch_bounds__(256) gn_apply_kernel(const GnApplyParams p) {
    __shared__ float s_mean[32], s_rstd[32];
    LFD_TL_BEGIN(p.tl);
    const int n = blockIdx.y;
    const int cpr = p.C >> 3;
    int count = p.HW;
    size_t total = (size_t)p.HW * cpr;
    if (p.ext) {
        count = p.ext[0] * p.ext[1];
        total = (size_t)p.ext[0] * p.W * cpr;
    }
    if (threadIdx.x < p.groups)
        gn_mean_rstd(p.stats, n, threadIdx.x, p.groups, (double)count * 8.0, p.eps, &s_mean[threadIdx.x], &s_rstd[threadIdx.x]);
    __syncthreads();
    const uint4* in = reinterpret_cast<const uint4*>(p.in + (size_t)n * p.HW * p.C);
    uint4* out = reinterpret_cast<uint4*>(p.out + (size_t)n * p.HW * p.C);
#pragma unroll 4
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % cpr);
        const uint4 q = in[i];
        float f[8] = {up_lo<F16>(q.x), up_hi<F16>(q.x), up_lo<F16>(q.y), up_hi<F16>(q.y), up_lo<F16>(q.z), up_hi<F16>(q.z), up_lo<F16>(q.w), up_hi<F16>(q.w)};
        const float m = s_mean[g], r = s_rstd[g];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float y = (f[j] - m) * r;
            y = fmaf(y, p.gamma[g * 8 + j], p.beta[g * 8 + j]);
            f[j] = fmaxf(y, 0.f);
        }
        uint4 o;
        o.x = pack2<F16>(f[0], f[1]); o.y = pack2<F16>(f[2], f[3]); o.z = pack2<F16>(f[4], f[5]); o.w = pack2<F16>(f[6], f[7]);
        out[i] = o;
    }
    LFD_TL_END(p.tl);
}

cudaError_t gn_apply_launch(const GnApplyParams& p, int num_sms, cudaStream_t st) {
    if (p.C != p.groups * 8 || p.groups > 32) return cudaErrorInvalidValue;
    const size_t total = (size_t)p.HW * (p.C >> 3);
    int bx = (int)((total + 255) / 256);
    const int cap = (8 * num_sms + p.N - 1) / p.N;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    if (p.f16) gn_apply_kernel<true><<<dim3(bx, p.N), 256, 0, st>>>(p);
    else gn_apply_kernel<false><<<dim3(bx, p.N), 256, 0, st>>>(p);
    return cudaGetLastError();
}

// ===================================================================================================
// head final: GN apply + ReLU (bf16 round) -> narrow 1x1 convs -> fp32 (N, P, C') / (N, P, 4)
// ===================================================================================================
static constexpr int kHfThreads = 256;
static constexpr int kHfPpt = 4;                       // pixels per thread
static constexpr int kHfPixPerBlock = (kHfThreads / 8) * kHfPpt;   // 128
static constexpr int kHfMaxC = 128;

// 8 threads share one pixel (16 channels each): coalesced 256-byte rows, the 16-channel weight slice of every output
// is a broadcast-friendly 64-byte shared-memory read, partial dot products are combined with 3 warp shuffles.
template <bool F16>
__global__ void __launch_bounds__(kHfThreads) head_final_kernel(const HeadFinalParams p) {
    extern __shared__ __align__(16) float hf_smem[];
    float* wsm = hf_smem;                                 // [n_out][C]
    float* s_mean = wsm + (size_t)p.n_out * p.C;          // [groups]
    float* s_rstd = s_mean + 32;
    LFD_TL_BEGIN(p.tl);
    const int n = blockIdx.y;
    int HW = p.HW, vw = p.W, P = p.P, point_off = p.point_off;      // valid pixels, valid width, output geometry
    if (p.ext) {
        vw = p.ext[1]; HW = p.ext[0] * vw; point_off = p.ext[4]; P = p.ext[5];
    }
    for (int i = threadIdx.x; i < p.n_out * p.C; i += kHfThreads) wsm[i] = p.w[i];
    const bool gn = p.groups > 0;      // groups == 0: the tower has no norm layers, the input is the already activated tensor
    if (gn && threadIdx.x < p.groups)
        gn_mean_rstd(p.stats, n, threadIdx.x, p.groups, (double)HW * 8.0, p.eps, &s_mean[threadIdx.x], &s_rstd[threadIdx.x]);
    __syncthreads();
    const int sl = threadIdx.x & 7;                       // channel slice: channels [16 sl, 16 sl + 16)
    float ga[16], be[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { ga[j] = gn ? p.gamma[sl * 16 + j] : 1.f; be[j] = gn ? p.beta[sl * 16 + j] : 0.f; }
    const float m0 = gn ? s_mean[2 * sl] : 0.f, r0 = gn ? s_rstd[2 * sl] : 1.f, m1 = gn ? s_mean[2 * sl + 1] : 0.f, r1 = gn ? s_rstd[2 * sl + 1] : 1.f;
    // persistent over 128-pixel tiles: the raw rows of the NEXT tile are fetched into registers before the current tile is evaluated, so the
    // loads of tile t+1 fly while tile t computes (one wave of blocks instead of HW / 128 short-lived ones, each paying the weight fetch)
    const uint4* rows = reinterpret_cast<const uint4*>(p.in + (size_t)n * p.HW * p.C + sl * 16);
    const int row_u4 = p.C >> 3;                          // uint4 per pixel row
    uint4 nxt[kHfPpt][2];
    auto fetch = [&](int tile) {
#pragma unroll
        for (int k = 0; k < kHfPpt; ++k) {
            const int pix = tile * kHfPixPerBlock + (threadIdx.x >> 3) + k * (kHfThreads / 8);
            nxt[k][0] = make_uint4(0, 0, 0, 0); nxt[k][1] = nxt[k][0];
            if (pix < HW) {
                const size_t row = vw == p.W ? (size_t)pix : (size_t)(pix / vw) * p.W + pix % vw;   // valid pixel -> row of the map
                nxt[k][0] = rows[row * row_u4]; nxt[k][1] = rows[row * row_u4 + 1];
            }
        }
    };
    const int n_tiles = (HW + kHfPixPerBlock - 1) / kHfPixPerBlock;
    if ((int)blockIdx.x < n_tiles) fetch(blockIdx.x);
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int pix0 = tile * kHfPixPerBlock + (threadIdx.x >> 3);
    float a[kHfPpt][16];
#pragma unroll
    for (int k = 0; k < kHfPpt; ++k) {
        const uint4 q0 = nxt[k][0], q1 = nxt[k][1];
        float f[16] = {up_lo<F16>(q0.x), up_hi<F16>(q0.x), up_lo<F16>(q0.y), up_hi<F16>(q0.y), up_lo<F16>(q0.z), up_hi<F16>(q0.z), up_lo<F16>(q0.w), up_hi<F16>(q0.w),
                       up_lo<F16>(q1.x), up_hi<F16>(q1.x), up_lo<F16>(q1.y), up_hi<F16>(q1.y), up_lo<F16>(q1.z), up_hi<F16>(q1.z), up_lo<F16>(q1.w), up_hi<F16>(q1.w)};
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            float y = (f[j] - (j < 8 ? m0 : m1)) * (j < 8 ? r0 : r1);
            y = fmaf(y, ga[j], be[j]);
            a[k][j] = round16<F16>(fmaxf(y, 0.f));        // rounding point Rg
        }
    }
    if (tile + (int)gridDim.x < n_tiles) fetch(tile + gridDim.x);
    for (int o0 = 0; o0 < p.n_out; o0 += 8) {
        float acc[8][kHfPpt];
#pragma unroll
        for (int o = 0; o < 8; ++o)
#pragma unroll
            for (int k = 0; k < kHfPpt; ++k) acc[o][k] = 0.f;
#pragma unroll
        for (int o = 0; o < 8; ++o) {
            if (o0 + o < p.n_out) {
                const float4* wr = reinterpret_cast<const float4*>(wsm + (size_t)(o0 + o) * p.C + sl * 16);
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    const float4 w4 = wr[v];
#pragma unroll
                    for (int k = 0; k < kHfPpt; ++k) {
                        acc[o][k] = fmaf(a[k][v * 4 + 0], w4.x, acc[o][k]); acc[o][k] = fmaf(a[k][v * 4 + 1], w4.y, acc[o][k]);
                        acc[o][k] = fmaf(a[k][v * 4 + 2], w4.z, acc[o][k]); acc[o][k] = fmaf(a[k][v * 4 + 3], w4.w, acc[o][k]);
                    }
                }
            }
        }
        // combine the 8 channel slices; afterwards lane `sl` owns output o0 + sl
#pragma unroll
        for (int o = 0; o < 8; ++o)
#pragma unroll
            for (int k = 0; k < kHfPpt; ++k) {
                float v = acc[o][k];
                v += __shfl_xor_sync(0xffffffffu, v, 1);
                v += __shfl_xor_sync(0xffffffffu, v, 2);
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                acc[o][k] = v;
            }
        const int o = o0 + sl;
        if (o < p.n_out) {
            const float sc = p.scale[o], sh = p.shift[o];
#pragma unroll
            for (int k = 0; k < kHfPpt; ++k) {
                const int pix = pix0 + k * (kHfThreads / 8);
                if (pix >= HW) continue;
                float v = 0.f;
#pragma unroll
                for (int oo = 0; oo < 8; ++oo) v = (oo == sl) ? acc[oo][k] : v;   // select without dynamic register indexing
                v = fmaf(v, sc, sh);
                if (o < p.n_cls) p.cls[((size_t)n * P + point_off + pix) * p.cls_stride + o] = v;
                else p.reg[((size_t)n * P + point_off + pix) * 4 + (o - p.n_cls)] = v;
            }
        }
    }
    }
    LFD_TL_END(p.tl);
}

cudaError_t head_final_launch(const HeadFinalParams& p, int num_sms, cudaStream_t st) {
    if (p.C != kHfMaxC || (p.groups != 16 && p.groups != 0)) return cudaErrorInvalidValue;   // 128 channels; 16 groups of 8, or no norm
    const size_t smem = ((size_t)p.n_out * p.C + 64) * sizeof(float);
    static bool attr[kMaxDevices] = {};   // per-device function attribute
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!attr[dev]) {
        cudaError_t e = cudaFuncSetAttribute(head_final_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(head_final_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        if (e != cudaSuccess) return e;
        attr[dev] = true;
    }
    if (smem > 64 * 1024) return cudaErrorInvalidValue;
    const int tiles = (p.HW + kHfPixPerBlock - 1) / kHfPixPerBlock;
    int bx = (4 * num_sms + p.N - 1) / p.N;              // about four blocks per SM over all images
    if (bx > tiles) bx = tiles;
    const dim3 grid(bx < 1 ? 1 : bx, p.N);
    if (p.f16) head_final_kernel<true><<<grid, kHfThreads, smem, st>>>(p);
    else head_final_kernel<false><<<grid, kHfThreads, smem, st>>>(p);
    return cudaGetLastError();
}

// ===================================================================================================
// SIMT cross-check convolution (packed weights [cc][tap][kc][Cout][8])
// ===================================================================================================
__global__ void __launch_bounds__(256) simt_conv_kernel(ConvGeom g, int Cc, const __nv_bfloat16* __restrict__ in,
                                                        __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ res,
                                                        const __nv_bfloat16* __restrict__ w, const float* __restrict__ shift,
                                                        double* stats, int gn_groups, int relu, int f16i) {
    const bool f16 = f16i != 0;
    const int ng = g.Cout >> 3;
    const size_t total = (size_t)g.N * g.Ho * g.Wo * ng;
    const int taps = g.ksize * g.ksize, pad = g.ksize / 2, cpc = Cc >> 3, n_cc = g.Cin / Cc;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int og = (int)(idx % ng);
        size_t pix = idx / ng;
        const int ox = (int)(pix % g.Wo), oy = (int)((pix / g.Wo) % g.Ho), n = (int)(pix / ((size_t)g.Wo * g.Ho));
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int cc = 0; cc < n_cc; ++cc)
            for (int tap = 0; tap < taps; ++tap) {
                const int iy = oy * g.stride + tap / g.ksize - pad, ix = ox * g.stride + tap % g.ksize - pad;
                if (iy < 0 || iy >= g.H || ix < 0 || ix >= g.W) continue;
                const __nv_bfloat16* ip = in + (((size_t)n * g.H + iy) * g.W + ix) * g.Cin + cc * Cc;
                for (int kc = 0; kc < cpc; ++kc) {
                    const uint4 xv = *reinterpret_cast<const uint4*>(ip + kc * 8);
                    const float xf[8] = {up_lo_rt(xv.x, f16), up_hi_rt(xv.x, f16), up_lo_rt(xv.y, f16), up_hi_rt(xv.y, f16),
                                         up_lo_rt(xv.z, f16), up_hi_rt(xv.z, f16), up_lo_rt(xv.w, f16), up_hi_rt(xv.w, f16)};
                    const __nv_bfloat16* wp = w + ((((size_t)cc * taps + tap) * cpc + kc) * g.Cout + og * 8) * 8;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const uint4 wv = *reinterpret_cast<const uint4*>(wp + j * 8);
                        acc[j] = fmaf(xf[0], up_lo_rt(wv.x, f16), acc[j]); acc[j] = fmaf(xf[1], up_hi_rt(wv.x, f16), acc[j]);
                        acc[j] = fmaf(xf[2], up_lo_rt(wv.y, f16), acc[j]); acc[j] = fmaf(xf[3], up_hi_rt(wv.y, f16), acc[j]);
                        acc[j] = fmaf(xf[4], up_lo_rt(wv.z, f16), acc[j]); acc[j] = fmaf(xf[5], up_hi_rt(wv.z, f16), acc[j]);
                        acc[j] = fmaf(xf[6], up_lo_rt(wv.w, f16), acc[j]); acc[j] = fmaf(xf[7], up_hi_rt(wv.w, f16), acc[j]);
                    }
                }
            }
        float o[8];
        const size_t off = pix * g.Cout + og * 8;
        uint4 rv = make_uint4(0, 0, 0, 0);
        if (res) rv = *reinterpret_cast<const uint4*>(res + off);
        const float rf[8] = {up_lo_rt(rv.x, f16), up_hi_rt(rv.x, f16), up_lo_rt(rv.y, f16), up_hi_rt(rv.y, f16), up_lo_rt(rv.z, f16), up_hi_rt(rv.z, f16), up_lo_rt(rv.w, f16), up_hi_rt(rv.w, f16)};
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            o[j] = acc[j] + (shift ? round16_rt(shift[og * 8 + j], f16) : 0.f) + rf[j];
            if (relu) o[j] = fmaxf(o[j], 0.f);
            o[j] = round16_rt(o[j], f16);
            s1 += o[j];
            s2 = fmaf(o[j], o[j], s2);
        }
        uint4 ov;
        ov.x = pack2_rt(o[0], o[1], f16); ov.y = pack2_rt(o[2], o[3], f16); ov.z = pack2_rt(o[4], o[5], f16); ov.w = pack2_rt(o[6], o[7], f16);
        *reinterpret_cast<uint4*>(out + off) = ov;
        if (stats) {  // group size 8 == this thread's channel group
            atomicAdd(stats + ((size_t)n * gn_groups + og) * 2, (double)s1);
            atomicAdd(stats + ((size_t)n * gn_groups + og) * 2 + 1, (double)s2);
        }
    }
}

cudaError_t simt_conv_launch(const ConvGeom& g, int Cc, const __nv_bfloat16* in, __nv_bfloat16* out, const __nv_bfloat16* res,
                             const __nv_bfloat16* w, const float* shift, double* stats, int gn_groups,
                             int relu, int f16, cudaStream_t st) {
    const size_t total = (size_t)g.N * g.Ho * g.Wo * (g.Cout >> 3);
    size_t blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) blocks = 1;
    simt_conv_kernel<<<(int)blocks, 256, 0, st>>>(g, Cc, in, out, res, w, shift, stats, gn_groups, relu, f16);
    return cudaGetLastError();
}

}  // namespace lfd
