// wgrad_umma.cu -- convolution weight gradient on Hopper tensor cores (wgmma), sm_90a.
//
// Replaces what autograd's conv backward-weights (cuDNN) computes for every nn.Conv2d of the reference's backbone / neck /
// head towers in training (lfd/model/backbone/lfd_resnet.py:96-154,354-473, neck/simple_neck.py:35-47, head/lfd_head.py:85-135):
//     dW[tap][ci][co] = sum over (n, oy, ox)  x[n, s*oy + kh - pad, s*ox + kw - pad, ci] * dz[n, oy, ox, co]
//
// Formulation: a GEMM whose reduction (K) dimension is the PIXEL index.  With NHWC activations the pixel planes the forward
// kernel already uses -- plane[8-channel chunk][pixel][16 B] -- are exactly the wgmma *MN-major* SWIZZLE_NONE canonical layout
// (core matrix = 8 pixels x 16 B, 8 consecutive channels per 16-byte row; LBO = stride between 8-pixel groups = halo row pitch,
// SBO = stride between 8-channel chunks = plane pitch), so
//   * the x halo of a 16x8 output tile is loaded ONCE (same producers / tables as conv_umma.cu) and the 9 taps are shifted views;
//   * the dz tile is loaded as plane[8-channel chunk][128 pixels][16 B] (the N-major B operand);
//   * one tile = 8 K-steps (16 pixels = two tile rows each) x taps MMAs of M = 64 input channels, N = Cout, K = 16;
//   * the accumulators D[tap][64 x Cout] stay in the registers of the two consumer warpgroups (each owns a subset of the taps)
//     for ALL tiles of the CTA (persistent split-K over pixels) and are flushed once with vector atomics into the fp32
//     staging tensor dstage[tap][Cin][Cout].
// A warpgroup holds at most 128 accumulator registers per thread (256 / Cout taps): the taps of a 3x3 conv are split into groups
// handled by different CTAs, and Cin = 128 into two 64-channel chunks (grid = pixel slices x channel chunks x tap groups).
#include <stdlib.h>

#include "conv_common.cuh"
#include "ptx.cuh"
#include "train.cuh"

namespace lfd {

namespace {

constexpr int kWgProd = 128;                       // producer threads
constexpr int kWgConsumers = 256;                  // two warpgroups
constexpr int kWgThreads = kWgConsumers + kWgProd;
constexpr int kWgMaxStages = 4;
constexpr uint32_t kWgBPitch = 129 * 16;           // pitch between the 8-channel planes of the dz tile (odd multiple of 16 B)

struct WgEntry { uint32_t src_off, dst_off; };
struct WgDelta { int8_t dy, dx; };

struct alignas(16) WgradParams {
    const __nv_bfloat16* x;
    const __nv_bfloat16* dz;
    float* dstage;
    int N, H, W, Cin, Ho, Wo, Cout, mode;
    int tiles_x, tiles_per_img, num_tiles;
    unsigned long long magic_tpi, magic_tx;
    int n_px, Cc, log2_cpc, log2_cpo;
    int n_cich, n_tapg, taps_per_group, n_taps, grid_tiles;
    int stages;
    uint32_t a_plane_pitch, a_row_pitch, a_stage_bytes, stage_bytes;
    uint32_t smem_table_off, smem_ring_off;
};

// taps one consumer warpgroup accumulates: 128 registers per thread of m64 x Cout accumulators
template <int MODE, int COUT>
struct WgTaps { static constexpr int value = (MODE == MODE_3X3S1 || MODE == MODE_3X3S2) ? (256 / COUT < 9 ? 256 / COUT : 9) : 1; };

LFD_DEVINL int wg_fast_div(int x, uint64_t magic) { return (int)(((uint64_t)(uint32_t)x * magic) >> 40); }

template <int MODE>
LFD_DEVINL constexpr int wg_tap_view(int tap) {   // pixel-slot offset of tap's shifted view (same planes as conv_umma.cu)
    if (MODE == MODE_3X3S1) return (tap / 3) * 10 + (tap % 3);
    if (MODE == MODE_3X3S2) {
        const int kh = tap / 3, kw = tap % 3;
        return (kh == 1 ? 0 : 288) + (kw == 1 ? 0 : (kh == 1 ? 144 : 153)) + (kh == 2 ? 9 : 0) + (kw == 2 ? 1 : 0);
    }
    return 0;
}

template <int MODE, int COUT>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_umma_kernel(const __grid_constant__ WgradParams p) {
    constexpr int TPW = WgTaps<MODE, COUT>::value;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem);
    uint64_t* empty = full + kWgMaxStages;
    WgEntry* table = reinterpret_cast<WgEntry*>(smem + p.smem_table_off);
    WgDelta* delta = reinterpret_cast<WgDelta*>(smem + p.smem_table_off + (size_t)p.n_px * sizeof(WgEntry));
    uint8_t* ring = smem + p.smem_ring_off;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // work decomposition: blockIdx = ((tap group * channel chunks) + channel chunk) * pixel slices + pixel slice
    const int slice = blockIdx.x % p.grid_tiles;
    const int cich = (blockIdx.x / p.grid_tiles) % p.n_cich;
    const int tapg = blockIdx.x / (p.grid_tiles * p.n_cich);
    const int tap0 = tapg * p.taps_per_group;
    const int ntap = min(p.taps_per_group, p.n_taps - tap0);
    const int SA = p.stages;

    if (tid == 0) {
        for (int i = 0; i < SA; ++i) { mbar_init(&full[i], kWgProd); mbar_init(&empty[i], kWgConsumers / 32); }
        fence_mbar_init();
    }
    if (MODE != MODE_FLAT) {
        for (int i = tid; i < p.n_px; i += kWgThreads) {
            int dy, dx, slot;
            if (MODE == MODE_3X3S1) { const int r = i / 10, c = i % 10; dy = r - 1; dx = c - 1; slot = i; }
            else if (MODE == MODE_1X1S2) { const int r = i >> 3, c = i & 7; dy = 2 * r; dx = 2 * c; slot = i; }
            else {  // MODE_3X3S2: EE(16x8) | EO(16x9) | OE(17x8) | OO(17x9), every plane with row pitch 9
                int j = i, r, c, base, rodd, codd;
                if (j < 128) { r = j >> 3; c = j & 7; base = 0; rodd = 0; codd = 0; }
                else if ((j -= 128) < 144) { r = j / 9; c = j % 9; base = 144; rodd = 0; codd = 1; }
                else if ((j -= 144) < 136) { r = j >> 3; c = j & 7; base = 288; rodd = 1; codd = 0; }
                else { j -= 136; r = j / 9; c = j % 9; base = 441; rodd = 1; codd = 1; }
                dy = 2 * r - rodd; dx = 2 * c - codd; slot = base + r * 9 + c;
            }
            constexpr int kMin = (MODE == MODE_1X1S2) ? 0 : -1;
            WgEntry e;
            e.src_off = (uint32_t)(((dy - kMin) * p.W + (dx - kMin)) * p.Cin * 2);
            e.dst_off = (uint32_t)slot * 16u;
            table[i] = e;
            WgDelta d;
            d.dy = (int8_t)dy; d.dx = (int8_t)dx;
            delta[i] = d;
        }
    }
    __syncthreads();
    const int HW = p.H * p.W, HoWo = p.Ho * p.Wo;

    if (warp < kWgConsumers / 32) {
        // ============================================================== CONSUMERS: MMAs, then one flush of the accumulators
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        const int wg = warp >> 2;
        // this warpgroup's taps: the first or the second half of the CTA's tap group
        const int half = (ntap + 1) / 2;
        const int t_lo = wg * half, t_n = min(ntap, t_lo + half) - t_lo;
        // MN-major SWIZZLE_NONE: LBO = byte stride between 8-element K groups (pixels), SBO = between 8-element MN chunks (channels)
        const uint64_t adesc0 = wgmma_desc(0, p.a_row_pitch, p.a_plane_pitch);
        const uint64_t bdesc0 = wgmma_desc(0, 128, kWgBPitch);
        const uint32_t a_kstep = (2 * p.a_row_pitch) >> 4;    // one K = 16 step = two tile rows
        float acc[TPW][COUT / 2];
#pragma unroll
        for (int t = 0; t < TPW; ++t)
#pragma unroll
            for (int i = 0; i < COUT / 2; ++i) acc[t][i] = 0.f;
        uint32_t it = 0;
        for (int tile = slice; tile < p.num_tiles; tile += p.grid_tiles, ++it) {
            const uint32_t s = it % SA, ph = (it / SA) & 1;
            mbar_wait(&full[s], ph);
            fence_proxy_async_smem();   // cp.async (generic proxy) writes -> wgmma (async proxy) reads
            const uint32_t a_base = smem_u32(ring) + s * p.stage_bytes;
            const uint32_t b_base = a_base + p.a_stage_bytes;
            const uint64_t ad = adesc0 + (a_base >> 4), bd = bdesc0 + (b_base >> 4);
#pragma unroll
            for (int t = 0; t < TPW; ++t) wgmma_fence_regs<COUT / 2>(acc[t]);
            wgmma_fence();
            for (int kg = 0; kg < 8; ++kg) {
                const uint64_t adk = ad + (uint32_t)(kg * a_kstep), bdk = bd + (uint32_t)(kg * 16);
#pragma unroll
                for (int t = 0; t < TPW; ++t) {
                    if (t >= t_n) break;
                    // tap_view needs a compile-time tap for the 3x3/s2 formula: switch on the run-time tap
                    uint32_t view;
                    if (TPW == 1 && MODE != MODE_3X3S1 && MODE != MODE_3X3S2) view = 0;
                    else {
                        switch (tap0 + t_lo + t) {
                            case 0: view = wg_tap_view<MODE>(0); break; case 1: view = wg_tap_view<MODE>(1); break;
                            case 2: view = wg_tap_view<MODE>(2); break; case 3: view = wg_tap_view<MODE>(3); break;
                            case 4: view = wg_tap_view<MODE>(4); break; case 5: view = wg_tap_view<MODE>(5); break;
                            case 6: view = wg_tap_view<MODE>(6); break; case 7: view = wg_tap_view<MODE>(7); break;
                            default: view = wg_tap_view<MODE>(8); break;
                        }
                    }
                    wgmma_ss<COUT, false, 1, 1>(acc[t], adk + view, bdk, 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int t = 0; t < TPW; ++t) wgmma_fence_regs<COUT / 2>(acc[t]);
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        // flush: thread holds rows (input channels) r0, r0 + 8 and columns (output channels) 8j + 2 (lane % 4) (+1)
        const int r0 = (warp & 3) * 16 + (lane >> 2), tq = lane & 3;
#pragma unroll
        for (int t = 0; t < TPW; ++t) {
            if (t >= t_n) break;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int ci = cich * 64 + r0 + 8 * h;
                if (ci >= p.Cin) continue;
                float* dst = p.dstage + ((size_t)(tap0 + t_lo + t) * p.Cin + ci) * COUT + 2 * tq;
#pragma unroll
                for (int j = 0; j < COUT / 8; ++j) atomicAdd(reinterpret_cast<float2*>(dst + 8 * j), make_float2(acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1]));
            }
        }
    } else {
        // ============================================================== PRODUCERS
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int ptid = tid - kWgConsumers;
        const int cpc = p.Cc >> 3;
        const int ch = ptid & (cpc - 1);
        const int px0 = ptid >> p.log2_cpc;
        const int pstep = kWgProd >> p.log2_cpc;
        const uint32_t ch_dst = ch * p.a_plane_pitch;
        const int my_cnt = (p.n_px - px0 + pstep - 1) / pstep;
        const int cpo = p.Cout >> 3;
        const int chb = ptid & (cpo - 1);
        const int bpx0 = ptid >> p.log2_cpo;
        const int bstep = kWgProd >> p.log2_cpo;
        uint32_t it = 0;
        for (int tile = slice; tile < p.num_tiles; tile += p.grid_tiles, ++it) {
            const int n = wg_fast_div(tile, p.magic_tpi);
            const int t = tile - n * p.tiles_per_img;
            int iy0 = 0, ix0 = 0, oy0 = 0, ox0 = 0;
            if (MODE == MODE_FLAT) ix0 = t * 128;
            else {
                const int ty = wg_fast_div(t, p.magic_tx);
                oy0 = ty * 16; ox0 = (t - ty * p.tiles_x) * 8;
                iy0 = (MODE == MODE_3X3S1) ? oy0 : 2 * oy0;
                ix0 = (MODE == MODE_3X3S1) ? ox0 : 2 * ox0;
            }
            const uint32_t s = it % SA, ph = (it / SA) & 1;
            mbar_wait(&empty[s], ph ^ 1);
            const uint32_t a_base = smem_u32(ring) + s * p.stage_bytes;
            // ---- A: the x halo (zero fill = conv padding)
            const __nv_bfloat16* img = p.x + (size_t)n * HW * p.Cin + cich * 64 + ch * 8;
            constexpr int kDyMin = (MODE == MODE_1X1S2) ? 0 : -1, kDxMin = kDyMin;
            constexpr int kDyMax = (MODE == MODE_3X3S1) ? 16 : ((MODE == MODE_3X3S2) ? 31 : 30);
            constexpr int kDxMax = (MODE == MODE_3X3S1) ? 8 : ((MODE == MODE_3X3S2) ? 15 : 14);
            const bool interior = MODE == MODE_FLAT ? (ix0 + 128 <= HW)
                                                    : (iy0 + kDyMin >= 0 && ix0 + kDxMin >= 0 && iy0 + kDyMax < p.H && ix0 + kDxMax < p.W);
            const uint32_t dst_cc = a_base + ch_dst;
            if (MODE == MODE_FLAT) {
#pragma unroll 4
                for (int pxi = px0; pxi < 128; pxi += pstep) {
                    const int q = ix0 + pxi;
                    const bool ok = q < HW;
                    cp_async16(dst_cc + pxi * 16, img + (size_t)(ok ? q : 0) * p.Cin, ok);
                }
            } else if (interior) {
                const uint8_t* src = reinterpret_cast<const uint8_t*>(img + ((ptrdiff_t)(iy0 + kDyMin) * p.W + ix0 + kDxMin) * p.Cin);
                const WgEntry* tp = table + px0;
#pragma unroll 4
                for (int k = 0; k < my_cnt; ++k, tp += pstep) {
                    const uint2 pe = *reinterpret_cast<const uint2*>(tp);
                    cp_async16_full(dst_cc + pe.y, src + pe.x);
                }
            } else {
#pragma unroll 2
                for (int pxi = px0; pxi < p.n_px; pxi += pstep) {
                    const WgDelta pd = delta[pxi];
                    const int y = iy0 + pd.dy, x = ix0 + pd.dx;
                    const bool ok = ((unsigned)y < (unsigned)p.H) && ((unsigned)x < (unsigned)p.W);
                    cp_async16(dst_cc + table[pxi].dst_off, img + (size_t)(ok ? (y * p.W + x) : 0) * p.Cin, ok);
                }
            }
            // ---- B: the dz tile, 128 pixels (pixels outside the map are ZERO: they must not contribute)
            const uint32_t b_dst = a_base + p.a_stage_bytes + chb * kWgBPitch;
            const __nv_bfloat16* dzi = p.dz + (size_t)n * HoWo * p.Cout + chb * 8;
#pragma unroll 4
            for (int sl = bpx0; sl < 128; sl += bstep) {
                int q;
                bool ok;
                if (MODE == MODE_FLAT) { q = ix0 + sl; ok = q < HoWo; }
                else {
                    const int oy = oy0 + (sl >> 3), ox = ox0 + (sl & 7);
                    ok = oy < p.Ho && ox < p.Wo;
                    q = oy * p.Wo + ox;
                }
                cp_async16(b_dst + sl * 16, dzi + (size_t)(ok ? q : 0) * p.Cout, ok);
            }
            cp_async_mbar_arrive(&full[s]);
        }
        cp_async_wait_all();
    }

}

int wg_mode_of(const WgradGeom& g) {
    if (g.ksize == 1 && g.stride == 1) return MODE_FLAT;
    if (g.ksize == 3 && g.stride == 1) return MODE_3X3S1;
    if (g.ksize == 3 && g.stride == 2) return MODE_3X3S2;
    if (g.ksize == 1 && g.stride == 2) return MODE_1X1S2;
    return -1;
}

int wg_configure(const WgradGeom& g, int num_sms, WgradParams* out, size_t* smem_bytes, int* grid) {
    WgradParams p;
    memset(&p, 0, sizeof(p));
    const int mode = wg_mode_of(g);
    if (mode < 0) return -1;
    if (g.Cin % 32 || g.Cin < 32 || (g.Cin > 64 && g.Cin % 64) || g.Cout % 16 || g.Cout < 16 || g.Cout > 128) return -2;
    const int eh = (g.H + 2 * (g.ksize / 2) - g.ksize) / g.stride + 1, ew = (g.W + 2 * (g.ksize / 2) - g.ksize) / g.stride + 1;
    if (eh != g.Ho || ew != g.Wo) return -3;
    p.mode = mode;
    p.N = g.N; p.H = g.H; p.W = g.W; p.Cin = g.Cin; p.Ho = g.Ho; p.Wo = g.Wo; p.Cout = g.Cout;
    int px_slots, row_slots;
    if (mode == MODE_FLAT) { p.tiles_x = 0; p.tiles_per_img = (g.Ho * g.Wo + 127) / 128; p.n_px = 128; px_slots = 128; row_slots = 8; }
    else {
        p.tiles_x = (g.Wo + 7) / 8;
        p.tiles_per_img = p.tiles_x * ((g.Ho + 15) / 16);
        if (mode == MODE_3X3S1) { p.n_px = 180; px_slots = 180; row_slots = 10; }
        else if (mode == MODE_3X3S2) { p.n_px = 561; px_slots = 594; row_slots = 9; }
        else { p.n_px = 128; px_slots = 128; row_slots = 8; }
    }
    p.num_tiles = p.tiles_per_img * g.N;
    if (p.num_tiles >= (1 << 24) || p.tiles_per_img >= (1 << 16)) return -5;
    p.magic_tpi = ((1ull << 40) + p.tiles_per_img - 1) / p.tiles_per_img;
    p.magic_tx = p.tiles_x ? ((1ull << 40) + p.tiles_x - 1) / p.tiles_x : 0;
    p.a_plane_pitch = (uint32_t)((px_slots | 1) * 16);
    p.a_row_pitch = (uint32_t)(row_slots * 16);
    p.Cc = g.Cin < 64 ? g.Cin : 64;
    auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
    p.log2_cpc = ilog2(p.Cc / 8);
    p.log2_cpo = ilog2(g.Cout / 8);
    if ((1 << p.log2_cpo) != g.Cout / 8) return -2;           // Cout in {16, 32, 64, 128}
    p.n_cich = (g.Cin + 63) / 64;
    p.n_taps = g.ksize * g.ksize;
    // two warpgroups of (at most) 256 / Cout taps per CTA; the groups are balanced (e.g. Cout = 64: 5 + 4 taps, not 8 + 1)
    const int per_wg = p.n_taps == 1 ? 1 : (256 / g.Cout < 9 ? 256 / g.Cout : 9);
    const int max_group = 2 * per_wg;
    p.n_tapg = (p.n_taps + max_group - 1) / max_group;
    p.taps_per_group = (p.n_taps + p.n_tapg - 1) / p.n_tapg;
    // the A stage always provides the 8 planes an M = 64 operand addresses (Cin = 32: the upper 4 are never written, their
    // accumulator rows are never read)
    p.a_stage_bytes = (uint32_t)((8 * (size_t)p.a_plane_pitch + 127) & ~(size_t)127);
    const uint32_t b_stage = (uint32_t)((((size_t)g.Cout / 8) * kWgBPitch + 127) & ~(size_t)127);
    p.stage_bytes = p.a_stage_bytes + b_stage;
    p.smem_table_off = 512;
    const size_t table_bytes = mode == MODE_FLAT ? 0 : (((size_t)p.n_px * 10 + 127) & ~(size_t)127);
    p.smem_ring_off = (uint32_t)((512 + table_bytes + 1023) & ~(size_t)1023);
    const size_t budget = 226 * 1024;
    int st = (int)((budget - p.smem_ring_off) / p.stage_bytes);
    if (st > kWgMaxStages) st = kWgMaxStages;
    if (st < 1) return -7;
    p.stages = st;
    *smem_bytes = p.smem_ring_off + (size_t)st * p.stage_bytes;
    const int per = p.n_cich * p.n_tapg;
    int gt = num_sms / per;
    if (gt < 1) gt = 1;
    if (gt > p.num_tiles) gt = p.num_tiles;
    p.grid_tiles = gt;
    *grid = gt * per;
    *out = p;
    return 0;
}

template <int MODE, int COUT>
cudaError_t wg_launch_t(const WgradParams& p, size_t smem, int grid, cudaStream_t st) {
    static bool configured[kMaxDevices] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_umma_kernel<MODE, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024));
        if (e != cudaSuccess) return e;
        configured[dev] = true;
    }
    wgrad_umma_kernel<MODE, COUT><<<grid, kWgThreads, smem, st>>>(p);
    return cudaGetLastError();
}

template <int MODE>
cudaError_t wg_launch_mode(const WgradParams& p, size_t smem, int grid, cudaStream_t st) {
    switch (p.Cout) {
        case 16: return wg_launch_t<MODE, 16>(p, smem, grid, st);
        case 32: return wg_launch_t<MODE, 32>(p, smem, grid, st);
        case 64: return wg_launch_t<MODE, 64>(p, smem, grid, st);
        case 128: return wg_launch_t<MODE, 128>(p, smem, grid, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace

int wgrad_umma_supported(const WgradGeom& g) {
    WgradParams p;
    size_t smem;
    int grid;
    return wg_configure(g, 132, &p, &smem, &grid) == 0;
}

cudaError_t wgrad_umma_launch(const WgradGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dz, float* dstage, int num_sms, cudaStream_t st) {
    WgradParams p;
    size_t smem = 0;
    int grid = 0;
    if (wg_configure(g, num_sms > 0 ? num_sms : 132, &p, &smem, &grid)) return cudaErrorInvalidValue;
    p.x = x; p.dz = dz; p.dstage = dstage;
    switch (p.mode) {
        case MODE_FLAT: return wg_launch_mode<MODE_FLAT>(p, smem, grid, st);
        case MODE_3X3S1: return wg_launch_mode<MODE_3X3S1>(p, smem, grid, st);
        case MODE_3X3S2: return wg_launch_mode<MODE_3X3S2>(p, smem, grid, st);
        case MODE_1X1S2: return wg_launch_mode<MODE_1X1S2>(p, smem, grid, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace lfd
