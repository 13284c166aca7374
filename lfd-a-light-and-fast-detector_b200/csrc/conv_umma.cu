// conv_umma.cu -- implicit-GEMM convolution on Hopper tensor cores (wgmma), sm_90a.
//
// Replaces, for the LFD hot path, every nn.Conv2d(+BatchNorm2d)(+residual)(+ReLU) of the reference's
// backbone / neck / head towers (lfd/model/backbone/lfd_resnet.py:96-154,354-473,
// lfd/model/neck/simple_neck.py:35-47, lfd/model/head/lfd_head.py:85-135), which the reference runs
// as separate cuDNN / ATen kernels in NCHW fp32.
//
// Formulation (NHWC bf16 activations, fp32 accumulate in registers):
//   D[128 output pixels, Cout] = sum over taps (kh,kw) and channel chunks of  A_tap[128, 16] * W_tap[16, Cout]
//   * persistent CTAs (one per SM), warp-specialised:
//       warpgroups 0, 1  consumers : rows 0..63 / 64..127 of the tile; wgmma.mma_async (m64 x Cout x k16) with pre-built
//                                    descriptors into register accumulators, then the epilogue from the same registers:
//                                    (+shift) (+residual) (+ReLU) -> bf16 -> the warpgroup's own staging rows -> its own TMA
//                                    tensor store (+ optional GroupNorm partial statistics of the stored tensor)
//       warps 8..11      producers : cp.async (16 B, zero-fill = conv padding) of the input halo tile into the A ring;
//                                    completion is signalled by cp.async.mbarrier.arrive (no thread waits on its own copies)
//   * BatchNorm is folded on the host: scale into the bf16 weights; the shift, rounded to the 16-bit type, is added to the
//     fp32 accumulator in the epilogue.
//   * the input halo tile is loaded ONCE per (tile, channel-chunk) into "pixel planes"
//       plane[k-chunk][pixel][8 channels = 16 B]
//     which is exactly the wgmma K-major / no-swizzle canonical layout (8-row core matrices of 16 B rows,
//     SBO between 8-row groups, LBO between 16-byte K chunks).  A 3x3 tap is then just a *shifted view*
//     (start address += tap offset, SBO = halo row pitch), so the 9 taps re-read shared memory, never L2.
//     Stride-2 convolutions de-interleave the halo into 4 row/column parity planes so that every tap is
//     again a unit-stride view.  The plane pitch (LBO) is an ODD multiple of 16 B so that the 8 channel
//     chunks of one pixel land in 8 different bank groups (conflict-free cp.async writes).
//   * MODE_STEM: the 3-channel stem conv's im2col is done by the same address generator (see kStem* below).
//   * optional second GEMM in the same launch: a trailing 1x1 conv whose A operand is the first accumulator, rounded to
//     16 bits, straight from registers ("tail": stem0->stem1, stem2->stem3), or the residual block's 1x1/s2 shortcut conv on
//     the centre tap (MODE_3X3S2, second output tensor).
//   * weights: pre-packed on the host in [channel-chunk][tap][k-chunk][Cout][8] order and brought in by
//     the TMA engine as 1-D bulk copies (cp.async.bulk), either once (resident) or per stage
//     (streamed, for 3x3x128x128 which does not fit next to the A ring).
//   * programmatic dependent launch: the prologue (barriers, weight fetch) overlaps the previous layer.
#include <stdlib.h>

#include <type_traits>

#include "conv_common.cuh"
#include "ptx.cuh"

namespace lfd {

static constexpr int kProdThreads = 128;
static constexpr int kConsumerThreads = 256;                        // two warpgroups
static constexpr int kConvThreads = kConsumerThreads + kProdThreads;

// The role bodies are lambdas that capture many locals by reference.  If the compiler decides NOT to inline one of them the
// closure is materialised in local memory and the kernel runs 2-3x slower (a large stack frame in ptxas -v is the symptom).  Force it.
#define LFD_LAMBDA_INLINE __attribute__((always_inline))

// clock64() timeline of CTA 0 (tests/debug_trace_consumers.py; tests/debug_stem_fusion.py --trace for stem4_kernel); compiled in only with
// -DLFD_B200_TRACE (LFD_B200_TRACE=1 python build.py).
// Buffer [4 roles][32 entries][4 slots]:
//   role 0        producer, per stage                : wait_empty  got_empty  issued  arrived_full (stem: next tile's fetch issued)
//   role 1 + wg   consumer warpgroup wg, per tile    : wait_full  got_full (last chunk)  main_mma_done  tail_mma_done
//   role 3        epilogues, entry 2 * store + wg    : store_entry  after_bulk_wait_read  tma_issued  residual_landed (after the shift loads
//                                                    and the warpgroup barrier; without a residual, after the barrier)
// Only thread 0 of each role stamps.
#ifdef LFD_B200_TRACE
#define LFD_TRACE(role, idx, slot) \
    do { if (p.trace && blockIdx.x == 0 && (idx) < 32) p.trace[((role) * 32 + (idx)) * 4 + (slot)] = clock64(); } while (0)
#define LFD_TRACE_EPI(tr, idx, slot) \
    do { if ((tr) && blockIdx.x == 0 && (idx) < 16) (tr)[(idx) * 8 + (slot)] = clock64(); } while (0)
#else
#define LFD_TRACE(role, idx, slot) ((void)0)
#define LFD_TRACE_EPI(tr, idx, slot) ((void)0)
#endif

// floor(x / d) for 0 <= x < 2^24 via one 32x32->64 multiply; m = ceil(2^40 / d), exact for d < 2^16
LFD_DEVINL int fast_div(int x, uint64_t magic) { return (int)(((uint64_t)(uint32_t)x * magic) >> 40); }

// What one launch covers: the valid extent (input H x W, output Ho x Wo) and the tile grid over it.  Without p.ext that is the host's
// configuration; with it, the extent comes from the plan's geometry table and the grid is recomputed over it exactly as
// configure_with / configure_stem4 compute it for a tensor of that size, so the tiles (and the fused stem's runs) are those of a plan
// built for the frame.  MODE_FLAT tiles walk the first Ho rows of the tensor at its full pitch p.Wo.
struct LaunchGrid {
    int H, W, Ho, Wo;
    int tiles_x, tiles_per_img, num_tiles;
    uint64_t magic_tpi, magic_tx;
};
// EXT is false exactly when p.ext is null: the kernels are instantiated for both, so a launch over the whole tensors keeps the grid
// in the constant bank and runs the code it ran before geometry tables existed
template <int MODE, bool EXT>
LFD_DEVINL LaunchGrid launch_grid(const UmmaConvParams& p) {
    LaunchGrid g;
    if constexpr (!EXT) {
        g.H = p.H; g.W = p.W; g.Ho = p.Ho; g.Wo = p.Wo;
        g.tiles_x = p.tiles_x; g.tiles_per_img = p.tiles_per_img; g.num_tiles = p.num_tiles;
        g.magic_tpi = p.magic_tpi; g.magic_tx = p.magic_tx;
        return g;
    }
    const int4 e = *reinterpret_cast<const int4*>(p.ext);
    g.H = e.x; g.W = e.y; g.Ho = e.z; g.Wo = e.w;
    if (MODE == MODE_FLAT) {
        g.tiles_x = 0; g.magic_tx = 0;
        g.tiles_per_img = (g.Ho * p.Wo + 127) / 128;
    } else {
        g.tiles_x = (g.Wo + 7) / 8;
        g.magic_tx = ((1ull << 40) + (uint64_t)g.tiles_x - 1) / (uint64_t)g.tiles_x;
        g.tiles_per_img = g.tiles_x * ((g.Ho + 15) / 16);
    }
    g.num_tiles = g.tiles_per_img * p.N;
    g.magic_tpi = ((1ull << 40) + (uint64_t)g.tiles_per_img - 1) / (uint64_t)g.tiles_per_img;
    return g;
}

struct PxEntry {  // one halo pixel: where it comes from and where it goes
    uint32_t src_off;  // byte offset of the pixel relative to the halo's top-left pixel (tile origin + (dy_min, dx_min))
    uint32_t dst_off;  // byte offset of its 16-byte slot inside a plane
};
struct PxDelta { int8_t dy, dx; };  // the same pixel relative to the tile's input origin, for tiles that touch the border

// MODE_STEM: the im2col of the 3-channel stem conv is done by the wgmma address generator.  The producers write the raw-image
// patch of one 16x8 output tile (33 rows x 18 pixels) to shared memory as bf16 with the channels padded to 4
// ([row][pixel][b g r 0] = 8 B per pixel, already normalised / rounded = rounding point R0).  Output pixel (oy, ox) and filter row
// kh need the 3 input pixels 2ox-1 .. 2ox+1 of input row 2oy+kh-1 = 12 of the 16 consecutive bf16 values that start at patch
// pixel (2oy + kh, 2ox); consecutive ox are 16 B apart, consecutive oy 2 patch rows.  That is exactly a K-major SWIZZLE_NONE A
// operand with K = 16: core-matrix rows 16 B apart, SBO = 2 rows, LBO (second K chunk) = 16 B (the chunks of neighbouring rows
// overlap, which a read-only view may).  So the conv is 3 MMAs (one per kh, K = 16) per tile against weights packed
// [kh][2][Cout][8] with zeros in the 4th pixel / 4th channel positions; the 18th patch column only meets zero weights but
// must hold finite values.
static constexpr int kStemRows = 33, kStemCols = 18, kStemPix = kStemRows * kStemCols;          // 594
static constexpr int kStemRowBytes = kStemCols * 8;                                             // 144
static constexpr int kStemPerThread = (kStemPix + kProdThreads - 1) / kProdThreads;             // 5
static constexpr int kStemPatchBytes = ((kStemRows * kStemRowBytes + 127) / 128) * 128;         // 4864

// c ? a : b as one selp: the compiler would otherwise select between the two ADDRESSES of an array element in warp_multi_reduce,
// which sends the array to local memory
LFD_DEVINL float selp_f32(bool c, float a, float b) {
    float r;
    asm("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %3, 0;\n\tselp.f32 %0, %1, %2, p;\n\t}" : "=f"(r) : "f"(a), "f"(b), "r"((uint32_t)c));
    return r;
}

// One step of the transposing butterfly of warp_multi_reduce: N live values -> N / 2 (compile-time recursion keeps every array
// index a constant, so the values stay in registers)
template <int NV, int N>
LFD_DEVINL void butterfly_step(float* val, int lane) {
    if constexpr (N > 1) {
        constexpr int off = 16 * N / NV;
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const float lo = val[i], hi = val[i + N / 2];
            const float send = selp_f32(upper, lo, hi);
            const float keep = selp_f32(upper, hi, lo);
            val[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
        butterfly_step<NV, N / 2>(val, lane);
    }
}

// Sums NV per-lane values over the 32 lanes of a warp with NV - 1 + log2(32 / NV) shuffles (transposing butterfly: every step
// halves the number of live values).  Returns, in every lane, the total of value index (lane * NV / 32).
template <int NV>
LFD_DEVINL float warp_multi_reduce(float* val, int lane) {
    butterfly_step<NV, NV>(val, lane);
    float r = val[0];
#pragma unroll
    for (int o = 16 / NV; o >= 1; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    return r;
}

// GroupNorm partial statistics of one warp's NC stored channels: st = [sum per 8-channel chunk | sum of squares per chunk]
template <int NC>
LFD_DEVINL void stats_flush(float* st, int lane, double* dst) {   // dst: (sum, sumsq) pair of the first group
    constexpr int NV = NC / 4, PER = 32 / NV, G = NV / 2;
    const float r = warp_multi_reduce<NV>(st, lane);
    if ((lane & (PER - 1)) == 0) {
        const int idx = lane / PER;
        atomicAdd(dst + (idx & (G - 1)) * 2 + (idx >= G ? 1 : 0), (double)r);
    }
}

template <int MODE>
__device__ __forceinline__ constexpr int tap_view(int tap) {  // pixel offset of tap's shifted view inside a plane
    if (MODE == MODE_3X3S1) return (tap / 3) * 10 + (tap % 3);
    if (MODE == MODE_3X3S2) {
        const int kh = tap / 3, kw = tap % 3;
        return (kh == 1 ? 0 : 288) + (kw == 1 ? 0 : (kh == 1 ? 144 : 153)) + (kh == 2 ? 9 : 0) + (kw == 2 ? 1 : 0);
    }
    if (MODE == MODE_STEM) return tap * (kStemRowBytes / 16);   // "tap" = filter row kh: one patch row further down
    return 0;
}

LFD_DEVINL void wg_bar_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }   // the 128 threads of warpgroup wg

// fused 1x1 tail: acc2[64 x N] = A[64 x K] . W2[K x N], A from registers (K / 16 fragments of 4 packed pairs), W2 resident in shared
// memory as [K / 8][N][8] (LBO = N * 16 B between 8-channel K chunks, SBO = 128 B between 8-column groups)
template <int N, int K, bool F16>
LFD_DEVINL void tail_mma(float* acc2, const uint32_t* a2, uint64_t b2desc0) {
#pragma unroll
    for (int kk = 0; kk < K / 16; ++kk) wgmma_rs<N, F16>(acc2, a2 + 4 * kk, b2desc0 + (uint32_t)((kk * 2 * N * 16) >> 4), kk != 0);
}

// Where the epilogue of one warpgroup writes and what it stores
struct EpiCtx {
    uint32_t stg;          // this warpgroup's staging region: [buffer][64 rows x Cf x 2 B]
    uint32_t stg_bytes;    // bytes of one staging buffer
    int nbuf;
    int r0, tq;            // this thread's first row (second: r0 + 8) within the warpgroup's 64, column pair index (lane % 4)
    int wtid;              // thread index within the warpgroup
    int wg, lane;
#ifdef LFD_B200_TRACE
    long long* tr;         // this warpgroup's first epilogue entry of the trace buffer (null: no trace); its entries are 8 apart
#endif
};

// Register accumulators (rows r0 / r0 + 8, NC <= NCMAX columns) (+shift) (+residual) (+ReLU) -> 16-bit staging rows in the TMA swizzle
// layout -> one TMA tensor store per 64-channel panel (+ GroupNorm partial statistics of the stored values, NC == 128 only).
// Staging rows are laid out the way the TMA engine expects for its swizzle modes: 128-byte panels [panel][64 rows][128 B] with the
// 16-byte chunk index XORed by (row & 7) (SWIZZLE_128B); 64 / 32-byte rows use the 64B / 32B patterns.  The 96-byte rows of a
// 48-channel tensor have no swizzle mode of their width: they are stored plainly, [64 rows][96 B] (SWIZZLE_NONE, see encode_one).
template <int MODE, int NCMAX, bool F16>
LFD_DEVINL void store_tile(const EpiCtx& e, const float* acc, int nc, const float* bias, bool relu, bool res, double* stats,
                           const CUtensorMap* tmap, const CUtensorMap* tmres, int c0, int c1, int n, bool v0, bool v1,
                           uint64_t* res_bar, uint32_t& store_count, uint32_t& res_count) {
    const uint32_t buf = e.stg + (e.nbuf == 2 ? (store_count & 1) * e.stg_bytes : 0u);
#ifdef LFD_B200_TRACE
    const uint32_t tidx = store_count;
#endif
    ++store_count;
    const int row_bytes = nc >= 64 ? 128 : nc * 2;
    const int n_panels = nc >= 64 ? nc / 64 : 1;
    if (e.wtid == 0) {
        LFD_TRACE_EPI(e.tr, tidx, 0);
        // this staging buffer was the source of an earlier store: the TMA engine must be done reading it
        if (e.nbuf == 2) bulk_wait_read<1>(); else bulk_wait_read<0>();
        LFD_TRACE_EPI(e.tr, tidx, 1);
        if (res) {   // residual rows -> staging (out-of-map rows / columns arrive as zeros), added in place below
            mbar_arrive_expect_tx(res_bar, 64u * nc * 2u);
            for (int pn = 0; pn < n_panels; ++pn) {
                if (MODE == MODE_FLAT) tma_load_3d(buf + pn * 8192, tmres, pn * 64, c0, n, res_bar);
                else tma_load_4d(buf + pn * 8192, tmres, pn * 64, c0, c1, n, res_bar);
            }
        }
    }
    // The shifts of this thread's columns are loaded ahead of the staging stores, up to 8 column pairs at a time (4 with 128 columns):
    // the stores' "memory" clobber would otherwise order every load behind the previous store, one shared-memory round trip per pair.
    constexpr int JB = NCMAX / 8 < 8 ? NCMAX / 8 : 4;
    float2 bv[JB];
    auto load_shifts = [&](int j0) LFD_LAMBDA_INLINE {
#pragma unroll
        for (int i = 0; i < JB; ++i)
            if (j0 + i < nc / 8) bv[i] = *reinterpret_cast<const float2*>(bias + 8 * (j0 + i) + 2 * e.tq);
    };
    load_shifts(0);
    wg_bar_sync(e.wg);
    if (res) { mbar_wait(res_bar, res_count & 1); ++res_count; }
    if (e.wtid == 0) LFD_TRACE_EPI(e.tr, tidx, 3);
    float st[NCMAX == 128 ? 32 : 1];
    const bool stat = NCMAX == 128 && stats != nullptr;
#pragma unroll
    for (int j = 0; j < NCMAX / 8; ++j) {
        if (j < nc / 8) {
            if (j > 0 && j % JB == 0) load_shifts(j);
            const float b0 = bv[j % JB].x, b1 = bv[j % JB].y;
            float s1 = 0.f, s2 = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = e.r0 + 8 * h;
                const uint32_t swz = NCMAX == 48 ? 0u : (row_bytes == 128 ? (row & 7) : (row_bytes == 64 ? ((row >> 1) & 3) : ((row >> 2) & 1)));
                const uint32_t addr = buf + (uint32_t)(j >> 3) * 8192u + (uint32_t)(row * row_bytes) + ((((uint32_t)j & 7u) ^ swz) << 4) + 4u * e.tq;
                float x0 = acc[4 * j + 2 * h] + b0, x1 = acc[4 * j + 2 * h + 1] + b1;
                if (res) {
                    uint32_t rv;
                    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rv) : "r"(addr) : "memory");
                    x0 += up_lo<F16>(rv); x1 += up_hi<F16>(rv);
                }
                const uint32_t o = relu ? pack2_relu<F16>(x0, x1) : pack2<F16>(x0, x1);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(o) : "memory");
                if (stat && (h ? v1 : v0)) {
                    const float f0 = up_lo<F16>(o), f1 = up_hi<F16>(o);
                    s1 += f0 + f1;
                    s2 = fmaf(f0, f0, fmaf(f1, f1, s2));
                }
            }
            if (NCMAX == 128) { st[j] = s1; st[16 + j] = s2; }
        }
    }
    fence_proxy_async_smem();             // st.shared (generic proxy) -> TMA store (async proxy)
    wg_bar_sync(e.wg);
    if (e.wtid == 0) {
        for (int pn = 0; pn < n_panels; ++pn) {   // rows / columns outside the map are clipped by the TMA engine
            if (MODE == MODE_FLAT) tma_store_3d(tmap, buf + pn * 8192, pn * 64, c0, n);
            else tma_store_4d(tmap, buf + pn * 8192, pn * 64, c0, c1, n);
        }
        bulk_commit();
        LFD_TRACE_EPI(e.tr, tidx, 2);
    }
    if (NCMAX == 128 && stat) stats_flush<128>(st, e.lane, stats);
}

// The consumers of conv_umma_solo_kernel: MODE_3X3S1, 64 -> 64 channels, resident weights, Cc = 64 (one ring stage per tile), no tail,
// shortcut or statistics.  Consumer warpgroup wg takes the tiles lt = wg, wg + 2, ... of the CTA's sequence and computes all 128 rows
// of each as two m64n64 blocks that share every B descriptor (64 fp32 accumulators per thread), in the k16-outer / tap-inner order of
// conv_umma_body, so every output gets the same sums.  The two warpgroups take turns on the tensor pipe: a warpgroup waits on
// turn[wg] before its first wgmma of a tile and arrives on the other's turn barrier once its MMAs have been waited for, so its epilogue
// runs under the other warpgroup's MMAs.  Warpgroup 0 starts; the alternation follows the tile order, so it never waits for a tile the
// other warpgroup does not have.  The residual rows of a tile are requested at the start of the tile and land under its MMAs.  Each
// warpgroup stages its tile in its own 16 KB region ([box: rows 0-63 | 64-127][64 rows x 128 B], SWIZZLE_128B) and stores it as two
// TMA boxes.
// Trace (LFD_B200_TRACE): role 1 + wg per tile of the warpgroup (k = 0, 1, ...): wait_full  got_full  main_mma_done  got_turn;
// role 3 entry 2 k + wg: epilogue entry  -  tma_issued  residual_landed (after the shift loads and the warpgroup barrier).
template <bool F16, bool EXT>
LFD_DEVINL void solo_consumers(const UmmaConvParams& p, const LaunchGrid& lg, uint64_t* full, uint64_t* empty, uint64_t* wbar,
                               uint64_t* res_bar, uint64_t* turn, const float* bias, uint8_t* staging, uint8_t* wres, uint8_t* ring) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wg = warp >> 2, wtid = tid & 127;
    if (tid == 0) {
        mbar_arrive_expect_tx(wbar, p.w_total_bytes);
        for (uint32_t off = 0; off < p.w_total_bytes; off += 32768) {
            const uint32_t nb = p.w_total_bytes - off < 32768 ? p.w_total_bytes - off : 32768;
            bulk_g2s(smem_u32(wres) + off, reinterpret_cast<const uint8_t*>(p.w) + off, nb, wbar);
        }
    }
    pdl_wait();                                   // residual reads and output stores depend on upstream kernels
    mbar_wait(wbar, 0);

    constexpr uint32_t kBox = 64u * 64u * 2u;     // one 64-row box of 64 channels
    const uint32_t stg = smem_u32(staging) + (uint32_t)wg * 2u * kBox;
    if (wtid == 0 && (stg & 1023u)) __trap();    // swizzle atoms need 1024-byte aligned staging regions
    const int r0 = (warp & 3) * 16 + (lane >> 2), tq = lane & 3;
    const uint64_t adesc0 = wgmma_desc(0, p.lbo_a, p.sbo_a);
    const uint64_t bd = wgmma_desc(0, 64 * 16, 128) + (smem_u32(wres) >> 4);
    const uint32_t a_k16 = (2 * p.lbo_a) >> 4, b_k16 = (2 * 64 * 16) >> 4, b_tap = (8 * 64 * 16) >> 4;
    const uint32_t a_blk = (8u * p.sbo_a) >> 4;  // rows 64..127 start 8 core-matrix rows further down
    const bool has_res = p.res != nullptr, relu = p.relu != 0;
#ifdef LFD_B200_TRACE
    long long* tr = p.trace && wtid == 0 ? p.trace + (3 * 32 + wg) * 4 : nullptr;
#endif

    float acc0[32], acc1[32];
    uint32_t k = 0;                               // tiles of this warpgroup so far
    for (int lt = wg, tile = blockIdx.x + wg * gridDim.x; tile < lg.num_tiles; lt += 2, tile += 2 * gridDim.x, ++k) {
        const int n = fast_div(tile, lg.magic_tpi), t = tile - n * lg.tiles_per_img;
        const int ty = fast_div(t, lg.magic_tx);
        const int c0 = (t - ty * lg.tiles_x) * 8, c1 = ty * 16;
        if (wtid == 0) {
            bulk_wait_read<0>();                  // the previous tile's stores have read the staging region
            if (has_res) {
                mbar_arrive_expect_tx(&res_bar[wg], 2u * kBox);
                tma_load_4d(stg, &p.tm_res, 0, c0, c1, n, &res_bar[wg]);
                tma_load_4d(stg + kBox, &p.tm_res, 0, c0, c1 + 8, n, &res_bar[wg]);
            }
            LFD_TRACE(1 + wg, k, 0);
        }
        const uint32_t s = (uint32_t)lt % p.stages, ph = ((uint32_t)lt / p.stages) & 1;
        mbar_wait(&full[s], ph);
        if (wtid == 0) LFD_TRACE(1 + wg, k, 1);
        if (lt > 0) mbar_wait(&turn[wg], (k - (wg == 0 ? 1u : 0u)) & 1);
        if (wtid == 0) LFD_TRACE(1 + wg, k, 3);
        fence_proxy_async_smem();   // cp.async (generic proxy) writes -> wgmma (async proxy) reads
        const uint64_t ad = adesc0 + ((smem_u32(ring) + s * p.stage_bytes) >> 4);
        wgmma_fence_regs<32>(acc0);
        wgmma_fence_regs<32>(acc1);
        wgmma_fence();
#pragma unroll
        for (int k16 = 0; k16 < 4; ++k16) {
            const uint64_t adk = ad + (uint32_t)(k16 * a_k16), bdk = bd + (uint32_t)(k16 * b_k16);
#pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
                const uint64_t b = bdk + (uint32_t)(tap * b_tap);
                wgmma_ss<64, F16>(acc0, adk + (uint32_t)tap_view<MODE_3X3S1>(tap), b, (k16 | tap) != 0);
                wgmma_ss<64, F16>(acc1, adk + a_blk + (uint32_t)tap_view<MODE_3X3S1>(tap), b, (k16 | tap) != 0);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<32>(acc0);
        wgmma_fence_regs<32>(acc1);
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&empty[s]);               // this warp's part of the stage has been consumed
            mbar_arrive(&turn[wg ^ 1]);           // the tensor pipe is the other warpgroup's
        }
        if (wtid == 0) LFD_TRACE(1 + wg, k, 2);

        // ---- epilogue: (+shift) (+residual) (+ReLU) -> 16-bit staging rows -> two TMA stores
        if (wtid == 0) LFD_TRACE_EPI(tr, k, 0);
        float2 bv[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) bv[j] = *reinterpret_cast<const float2*>(bias + 8 * j + 2 * tq);
        wg_bar_sync(wg);                          // orders thread 0's wait for the staging region before every thread's stores
        if (has_res) mbar_wait(&res_bar[wg], k & 1);
        if (wtid == 0) LFD_TRACE_EPI(tr, k, 3);
        auto stage_box = [&](const float* acc, uint32_t box) LFD_LAMBDA_INLINE {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = r0 + 8 * h;
                    const uint32_t addr = box + (uint32_t)(row * 128) + (((uint32_t)j ^ (uint32_t)(row & 7)) << 4) + 4u * tq;
                    float x0 = acc[4 * j + 2 * h] + bv[j].x, x1 = acc[4 * j + 2 * h + 1] + bv[j].y;
                    if (has_res) {
                        uint32_t rv;
                        asm volatile("ld.shared.b32 %0, [%1];" : "=r"(rv) : "r"(addr) : "memory");
                        x0 += up_lo<F16>(rv); x1 += up_hi<F16>(rv);
                    }
                    const uint32_t o = relu ? pack2_relu<F16>(x0, x1) : pack2<F16>(x0, x1);
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(o) : "memory");
                }
            }
        };
        stage_box(acc0, stg);
        stage_box(acc1, stg + kBox);
        fence_proxy_async_smem();                 // st.shared (generic proxy) -> TMA store (async proxy)
        wg_bar_sync(wg);
        if (wtid == 0) {                          // rows / columns outside the map are clipped by the TMA engine
            tma_store_4d(&p.tm_out, stg, 0, c0, c1, n);
            tma_store_4d(&p.tm_out, stg + kBox, 0, c0, c1 + 8, n);
            bulk_commit();
            LFD_TRACE_EPI(tr, k, 2);
        }
    }
    if (wtid == 0) bulk_wait_all();   // all tile stores have been performed before the CTA retires
}

// DS: the launch carries the fused 1x1/s2 shortcut (MODE_3X3S2, p.Cout3 > 0).  The shortcut and the fused tail never meet in one launch;
// with COUT = 128 a kernel that holds the code of both needs more registers than its 168: it spills and ptxas serialises its wgmmas.
// The body of conv_umma_kernel (COUT = 16 / 32 / 64 / 128), of conv_umma_c48_kernel (COUT = 48) and of conv_umma_solo_kernel (SOLO: the
// consumers are solo_consumers); p is the kernel's parameter.
template <int MODE, int COUT, bool F16, bool EXT, bool DS, bool SOLO = false>
LFD_DEVINL void conv_umma_body(const UmmaConvParams& p) {
    static_assert(!DS || MODE == MODE_3X3S2, "the fused shortcut belongs to a 3x3/s2 conv");
    static_assert(!SOLO || (MODE == MODE_3X3S1 && COUT == 64 && !DS), "the solo schedule is the 64-channel 3x3/s1 conv's");
    constexpr int kProd = kProdThreads;
    constexpr int kThreads = kConvThreads;
    constexpr int TAPS = (MODE == MODE_3X3S1 || MODE == MODE_3X3S2) ? 9 : (MODE == MODE_STEM ? 3 : 1);
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kSmemBarOff);
    uint64_t* empty = full + kMaxStages;
    uint64_t* wbar = empty + kMaxStages;
    uint64_t* res_bar = wbar + 1;     // [2] residual rows of one warpgroup landed (TMA load)
    uint64_t* turn = res_bar + 2;     // [2] SOLO: warpgroup wg may issue its MMAs
    PxEntry* table = reinterpret_cast<PxEntry*>(smem + p.smem_table_off);
    PxDelta* delta = reinterpret_cast<PxDelta*>(smem + p.smem_table_off + (size_t)p.n_px * sizeof(PxEntry));
    float* bias = reinterpret_cast<float*>(smem + p.smem_bias_off);
    float* bias2 = reinterpret_cast<float*>(smem + p.smem_bias2_off);
    uint8_t* staging = smem + p.smem_staging_off;
    uint8_t* wres = smem + p.smem_w_off;        // resident weights (if any)
    uint8_t* ring = smem + p.smem_ring_off;     // stages: [A chunk | B slice (streaming only)]

    // Programmatic dependent launch: let the next kernel of the stream start its prologue (barrier init, weight fetch) while
    // this one is still running; everything that touches upstream results waits at pdl_wait().
    pdl_launch_dependents();
    LFD_TL_BEGIN(p.tl);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int SA = p.stages;
    const int cpc = p.Cc >> 3;  // 16-byte chunks per pixel per stage

    // ------------------------------------------------------------------ one-time setup
    if (tid == 0) {
        for (int i = 0; i < SA; ++i) {
            mbar_init(&full[i], kProd + (p.b_resident ? 0 : 1));
            mbar_init(&empty[i], SOLO ? 4 : kConsumerThreads / 32);   // SOLO: a stage is consumed by the 4 warps of one warpgroup
        }
        mbar_init(wbar, 1);
        mbar_init(&res_bar[0], 1);
        mbar_init(&res_bar[1], 1);
        if (SOLO) {
            mbar_init(&turn[0], 4);
            mbar_init(&turn[1], 4);
        }
        fence_mbar_init();
    }
    // per-channel shifts (folded BatchNorm / bias), rounded to the 16-bit type, added to the fp32 accumulators by the epilogue
    for (int i = tid; i < p.Cout; i += kThreads) bias[i] = p.shift ? round16<F16>(p.shift[i]) : 0.f;
    const int cn2 = p.Cout2 + p.Cout3;      // second GEMM of the launch: fused 1x1 tail or fused 1x1/s2 shortcut (never both)
    for (int i = tid; i < cn2; i += kThreads) bias2[i] = p.shift2 ? round16<F16>(p.shift2[i]) : 0.f;
    // halo pixel table (tile independent)
    if (MODE != MODE_FLAT && MODE != MODE_STEM) {
        for (int i = tid; i < p.n_px; i += kThreads) {
            int dy, dx, slot;
            if (MODE == MODE_3X3S1) {
                int r = i / 10, c = i % 10;
                dy = r - 1; dx = c - 1; slot = i;
            } else if (MODE == MODE_1X1S2) {
                int r = i >> 3, c = i & 7;
                dy = 2 * r; dx = 2 * c; slot = i;
            } else {  // MODE_3X3S2: EE(16x8) | EO(16x9) | OE(17x8) | OO(17x9); all planes use pitch 9
                int j = i, r, c, base, rodd, codd;
                if (j < 128) { r = j >> 3; c = j & 7; base = 0; rodd = 0; codd = 0; }
                else if ((j -= 128) < 144) { r = j / 9; c = j % 9; base = 144; rodd = 0; codd = 1; }
                else if ((j -= 144) < 136) { r = j >> 3; c = j & 7; base = 288; rodd = 1; codd = 0; }
                else { j -= 136; r = j / 9; c = j % 9; base = 441; rodd = 1; codd = 1; }
                dy = 2 * r - rodd; dx = 2 * c - codd; slot = base + r * 9 + c;
            }
            constexpr int kMin = (MODE == MODE_1X1S2) ? 0 : -1;   // smallest dy / dx of the mode
            PxEntry e;
            e.src_off = (uint32_t)(((dy - kMin) * p.W + (dx - kMin)) * p.Cin * 2);
            e.dst_off = (uint32_t)slot * 16u;
            table[i] = e;
            PxDelta d;
            d.dy = (int8_t)dy; d.dx = (int8_t)dx;
            delta[i] = d;
        }
    }
    __syncthreads();

    const int HW = p.H * p.W;              // image stride of the input (its full size; lg.H x lg.W of it is valid)
    const int n_cc = p.Cin / p.Cc;
    const LaunchGrid lg = launch_grid<MODE, EXT>(p);

    if (SOLO && warp < kConsumerThreads / 32) {
        if constexpr (SOLO) solo_consumers<F16, EXT>(p, lg, full, empty, wbar, res_bar, turn, bias, staging, wres, ring);
    } else if (warp < kConsumerThreads / 32) {
        // ============================================================== CONSUMERS (MMA + epilogue)
        // registers move from the producer warpgroup to the accumulators: 2 x 128 x 224 + 128 x 56 = 64512 of 65536
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        const int wg = warp >> 2;
        const uint32_t w2_bytes = p.Cout2 ? (uint32_t)(p.Cout * p.Cout2 * 2) : (p.Cout3 ? (uint32_t)(p.Cin * p.Cout3 * 2) : 0u);
        if ((p.b_resident || w2_bytes) && tid == 0) {
            const uint32_t w1_bytes = p.b_resident ? p.w_total_bytes : 0u;
            mbar_arrive_expect_tx(wbar, w1_bytes + w2_bytes);
            for (uint32_t off = 0; off < w1_bytes; off += 32768) {
                uint32_t nb = w1_bytes - off < 32768 ? w1_bytes - off : 32768;
                bulk_g2s(smem_u32(wres) + off, reinterpret_cast<const uint8_t*>(p.w) + off, nb, wbar);
            }
            if (w2_bytes) bulk_g2s(smem_u32(smem + p.smem_w2_off), p.w2, w2_bytes, wbar);
        }
        pdl_wait();                                   // residual reads, output stores and statistics depend on upstream kernels
        if (p.b_resident || w2_bytes) mbar_wait(wbar, 0);

        EpiCtx e;
        e.stg_bytes = 64u * p.Cf * 2u;
        e.nbuf = p.stg_nbuf;
        e.stg = smem_u32(staging) + (uint32_t)wg * e.nbuf * e.stg_bytes;
        e.r0 = (warp & 3) * 16 + (lane >> 2);
        e.tq = lane & 3;
        e.wtid = tid & 127;
        e.wg = wg;
        e.lane = lane;
#ifdef LFD_B200_TRACE
        e.tr = p.trace && e.wtid == 0 ? p.trace + (3 * 32 + wg) * 4 : nullptr;
#endif
        if (e.wtid == 0 && (e.stg & 1023u)) __trap();    // swizzle atoms need 1024-byte aligned staging regions

        const uint32_t lbo_b = COUT * 16;
        // descriptors differ only in the 14-bit start-address field (bytes >> 4): pre-compute everything else
        const uint64_t adesc0 = wgmma_desc(0, p.lbo_a, p.sbo_a);
        const uint64_t bdesc0 = wgmma_desc(0, lbo_b, 128);
        const uint32_t a_k16 = (2 * p.lbo_a) >> 4;      // address-field step per 16 input channels (A)
        const uint32_t b_k16 = (2 * lbo_b) >> 4;        //   (B)
        const uint32_t b_tap = (cpc * lbo_b) >> 4;      // address-field step per tap (B)
        const uint32_t a_wg = (8u * p.sbo_a * wg) >> 4; // this warpgroup's 64 rows start 8 core-matrix rows further down
        const int nk16 = p.Cc >> 4;
        const uint64_t b2desc0 = wgmma_desc(smem_u32(smem + p.smem_w2_off), cn2 * 16, 128);
        const int flat_valid = lg.Ho * p.Wo;      // MODE_FLAT: the rows of the valid extent, at the full pitch

        float acc[COUT / 2];
        float acc3[DS ? COUT / 2 : 1];
        uint32_t it = 0, store_count = 0, res_count = 0;
        for (int tile = blockIdx.x, lt = 0; tile < lg.num_tiles; tile += gridDim.x, ++lt) {
            for (int cc = 0; cc < n_cc; ++cc, ++it) {
                const uint32_t s = it % SA, ph = (it / SA) & 1;
                if (cc == 0 && e.wtid == 0) LFD_TRACE(1 + wg, lt, 0);
                mbar_wait(&full[s], ph);
                if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 1);
                fence_proxy_async_smem();   // cp.async / st.shared (generic proxy) writes -> wgmma (async proxy) reads
                const uint32_t a_base = smem_u32(ring) + s * p.stage_bytes;
                const uint32_t b_base = p.b_resident ? smem_u32(wres) + cc * p.b_slice_bytes : a_base + p.a_stage_bytes;
                const uint64_t ad = adesc0 + ((a_base >> 4) + a_wg), bd = bdesc0 + (b_base >> 4);
                wgmma_fence_regs<COUT / 2>(acc);
                wgmma_fence();
                for (int k16 = 0; k16 < nk16; ++k16) {
                    const uint64_t adk = ad + (uint32_t)(k16 * a_k16), bdk = bd + (uint32_t)(k16 * b_k16);
#pragma unroll
                    for (int tap = 0; tap < TAPS; ++tap)
                        wgmma_ss<COUT, F16>(acc, adk + (uint32_t)tap_view<MODE>(tap), bdk + (uint32_t)(tap * b_tap), (cc | k16 | tap) != 0);
                }
                if constexpr (DS) {
                    // fused 1x1/s2 shortcut conv of the residual block: its input pixel is this conv's centre tap, so it
                    // is one more MMA per 16 channels on the operand that is already in shared memory
                    wgmma_fence_regs<COUT / 2>(acc3);
                    for (int k16 = 0; k16 < nk16; ++k16)
                        wgmma_ss<COUT, F16>(acc3, ad + (uint32_t)(k16 * a_k16) + (uint32_t)tap_view<MODE>(4),
                                            b2desc0 + (uint32_t)(((cc * cpc + 2 * k16) * COUT * 16) >> 4), (cc | k16) != 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<COUT / 2>(acc);
                if constexpr (DS) wgmma_fence_regs<COUT / 2>(acc3);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);     // this warp's part of the stage has been consumed
            }
            if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 2);

            // ---- epilogue of the tile: this warpgroup's 64 rows
            const int n = fast_div(tile, lg.magic_tpi);
            const int t = tile - n * lg.tiles_per_img;
            int c0, c1 = 0;      // coordinates of the warpgroup's first row: pixel index (flat) or (x, y)
            bool v0, v1;         // this thread's two rows lie inside the valid extent (statistics only; the TMA store clips at the tensor)
            if (MODE == MODE_FLAT) {
                c0 = t * 128 + wg * 64;
                const int q0 = c0 + e.r0, q1 = q0 + 8;
                v0 = q0 < flat_valid && (!EXT || q0 % p.Wo < lg.Wo); v1 = q1 < flat_valid && (!EXT || q1 % p.Wo < lg.Wo);
            } else {
                const int ty = fast_div(t, lg.magic_tx);
                c1 = ty * 16 + wg * 8; c0 = (t - ty * lg.tiles_x) * 8;
                const bool xin = c0 + (e.r0 & 7) < lg.Wo;
                v0 = xin && c1 + (e.r0 >> 3) < lg.Ho; v1 = xin && c1 + (e.r0 >> 3) + 1 < lg.Ho;
            }
            const bool has_res = p.res != nullptr;
            // GroupNorm partial sums are taken over the STORED (16-bit) values, after residual and ReLU; one group = one 16-byte
            // chunk (8 channels)
            double* sdst = p.stats ? p.stats + (size_t)n * p.gn_groups * 2 : nullptr;
            if (!DS && p.Cout2) {
                // fused 1x1 tail: D2[64 x Cout2] = round16(act(D + shift)) . W2, the A operand straight from the accumulator registers
                uint32_t a2[COUT / 4];
#pragma unroll
                for (int kk = 0; kk < COUT / 16; ++kk) {
                    const int c = 16 * kk + 2 * e.tq;
#pragma unroll
                    for (int q = 0; q < 4; ++q) {     // q: (row + 8 (q & 1), column + 8 (q >> 1))
                        const float x0 = acc[8 * kk + 2 * q] + bias[c + 8 * (q >> 1)], x1 = acc[8 * kk + 2 * q + 1] + bias[c + 8 * (q >> 1) + 1];
                        a2[4 * kk + q] = p.relu ? pack2_relu<F16>(x0, x1) : pack2<F16>(x0, x1);
                    }
                }
                // COUT / 16 MMAs of N = Cout2 and the store of Cout2 columns (the widths umma_conv_configure accepts for a stored tensor).
                // Each width has its own accumulator array: with one array shared by MMAs of different N, ptxas runs out of registers
                // for the wgmma pipeline and serialises every wgmma of the kernel (warning C7511), the main loop's included.
                // A 48-channel conv has the 48-channel tail only (the 'fast' stem's 1x1 48->48), the other widths never a 48-channel one.
                auto tail = [&](auto n2) LFD_LAMBDA_INLINE {
                    constexpr int N2 = decltype(n2)::value;
                    float acc2[N2 / 2];
                    wgmma_fence_regs<N2 / 2>(acc2);
                    wgmma_fence();
                    tail_mma<N2, COUT, F16>(acc2, a2, b2desc0);
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs<N2 / 2>(acc2);
                    if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 3);
                    store_tile<MODE, N2, F16>(e, acc2, N2, bias2, (bool)p.relu2, has_res, sdst,
                                              &p.tm_out, &p.tm_res, c0, c1, n, v0, v1, &res_bar[wg], store_count, res_count);
                };
                if constexpr (COUT == 48) {
                    tail(std::integral_constant<int, 48>());
                } else {
                    switch (p.Cout2) {
                        case 16: tail(std::integral_constant<int, 16>()); break;
                        case 32: tail(std::integral_constant<int, 32>()); break;
                        case 64: tail(std::integral_constant<int, 64>()); break;
                        default: tail(std::integral_constant<int, 128>()); break;
                    }
                }
            } else {
                store_tile<MODE, COUT, F16>(e, acc, COUT, bias, (bool)p.relu, has_res, sdst,
                                            &p.tm_out, &p.tm_res, c0, c1, n, v0, v1, &res_bar[wg], store_count, res_count);
                if constexpr (DS)
                    store_tile<MODE, COUT, F16>(e, acc3, COUT, bias2, false, false, nullptr, &p.tm_out3, nullptr, c0, c1, n, v0, v1,
                                                &res_bar[wg], store_count, res_count);
            }
        }
        if (e.wtid == 0) bulk_wait_all();   // all tile stores have been performed before the CTA retires
    } else {
        // ============================================================== PRODUCERS
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int ptid = tid - kConsumerThreads;
        if (MODE == MODE_STEM) {
            // Raw image patch -> normalised bf16 [row][pixel][b g r 0] in the ring stage (see kStem* above).  Every thread owns
            // up to 5 patch pixels; the raw values of the NEXT tile are fetched into registers right after the current patch
            // has been written, so the loads fly while the thread waits for the next free stage.  A gray image (p.img.ch == 1) has
            // one value per pixel (fp32 plane, uint8 byte, NV12's Y byte -- its UV plane is never read -- or a 4:2:2 pixel's Y byte),
            // written as (v, 0, 0, 0): the body is specialised for it at compile time, so the BGR loaders are exactly what they are
            // without it.  The packed formats (4:2:2, 4-byte pixels) have fetch branches of their own, taken once per tile.
            auto stem_producer = [&](auto gray_c) LFD_LAMBDA_INLINE {
                constexpr bool gray = decltype(gray_c)::value;
                const int fmt = p.img.format;
                const bool u8 = fmt != LFD_INPUT_F32_NCHW;   // bytes, normalised by p.img.xf
                const bool nv12 = fmt == LFD_INPUT_U8_NV12;
                const bool yuv422 = fmt == LFD_INPUT_U8_YUY2 || fmt == LFD_INPUT_U8_UYVY;
                const bool px4 = fmt == LFD_INPUT_U8_BGRA || fmt == LFD_INPUT_U8_RGBA;   // RGBA: api.cu permuted p.img.xf
                const int plane = p.H * p.W;
                // source offset of pixel j relative to the patch origin: bytes for BGR, 4:2:2 and 4-byte pixels, elements for gray / fp32 /
                // NV12's Y
                const int bpp = fmt == LFD_INPUT_U8_NHWC && !gray ? 3 : yuv422 ? 2 : px4 ? 4 : 1;
                int rel[kStemPerThread];
                int prc[kStemPerThread];          // (row << 8) | col
#pragma unroll
                for (int j = 0; j < kStemPerThread; ++j) {
                    const int q = min(ptid + j * kProdThreads, kStemPix - 1);
                    const int r = q / kStemCols, c = q - r * kStemCols;
                    prc[j] = (r << 8) | c;
                    rel[j] = (r * p.W + c) * bpp;
                }
                const bool last_ok = ptid + (kStemPerThread - 1) * kProdThreads < kStemPix;   // this thread owns a pixel in the last round
                uint32_t raw[kStemPerThread][gray ? 1 : 3];
                uint32_t okmask = 0;
                auto fetch = [&](int tile) LFD_LAMBDA_INLINE {
                    const int n = fast_div(tile, lg.magic_tpi), t = tile - n * lg.tiles_per_img;
                    const int ty = fast_div(t, lg.magic_tx);
                    const int iy0 = 2 * ty * 16 - 1, ix0 = 2 * (t - ty * lg.tiles_x) * 8 - 1;
                    const bool interior = iy0 >= 0 && ix0 >= 0 && iy0 + kStemRows <= lg.H && ix0 + kStemCols <= lg.W;
                    okmask = 0;
                    if (nv12) {
                        // raw = (Y, U, V): the Y plane, then the interleaved UV plane at the same pitch, UV row = absolute row / 2 (the patch
                        // starts at an odd row), UV column = x & ~1
                        const uint8_t* img = reinterpret_cast<const uint8_t*>(p.img.data) + (size_t)n * (plane + (plane >> 1));
                        const uint8_t* org = img + (ptrdiff_t)iy0 * p.W + ix0;
#pragma unroll
                        for (int j = 0; j < kStemPerThread; ++j) {
                            if (j == kStemPerThread - 1 && !last_ok) break;
                            const int y = iy0 + (prc[j] >> 8), x = ix0 + (prc[j] & 255);
                            const uint8_t* src = org + rel[j];
                            const uint8_t* uv = img + plane + (ptrdiff_t)(y >> 1) * p.W + (x & ~1);
                            const bool ok = interior || ((unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W);
                            if (!ok) { src = img; uv = img + plane; }
                            okmask |= (ok ? 1u : 0u) << j;
                            raw[j][0] = __ldg(src);
                            if constexpr (!gray) { raw[j][1] = __ldg(uv); raw[j][2] = __ldg(uv + 1); }
                        }
                    } else if (yuv422) {
                        // raw = (Y, U, V): the Y byte at byte l of the pixel's 2 (l = 1 for UYVY), U and V at bytes 1 - l and 3 - l of its
                        // pair x & ~1
                        const int l = fmt == LFD_INPUT_U8_UYVY;
                        const uint8_t* img = reinterpret_cast<const uint8_t*>(p.img.data) + (size_t)n * plane * 2;
                        const uint8_t* org = img + ((ptrdiff_t)iy0 * p.W + ix0) * 2;
#pragma unroll
                        for (int j = 0; j < kStemPerThread; ++j) {
                            if (j == kStemPerThread - 1 && !last_ok) break;
                            const int y = iy0 + (prc[j] >> 8), x = ix0 + (prc[j] & 255);
                            const uint8_t* src = org + rel[j];
                            const uint8_t* pair = src - 2 * (x & 1);
                            const bool ok = interior || ((unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W);
                            if (!ok) src = pair = img;
                            okmask |= (ok ? 1u : 0u) << j;
                            raw[j][0] = __ldg(src + l);
                            if constexpr (!gray) { raw[j][1] = __ldg(pair + 1 - l); raw[j][2] = __ldg(pair + 3 - l); }
                        }
                    } else if (u8) {
                        // uint8 BGR / gray (BPP 3 / 1) or 4-byte pixels (BPP 4: bytes 0..2, the alpha byte is never read)
                        auto fetch_bytes = [&](auto bpp_c) LFD_LAMBDA_INLINE {
                            constexpr int BPP = decltype(bpp_c)::value;
                            const uint8_t* img = reinterpret_cast<const uint8_t*>(p.img.data) + (size_t)n * plane * BPP;
                            const uint8_t* org = img + ((ptrdiff_t)iy0 * p.W + ix0) * BPP;
#pragma unroll
                            for (int j = 0; j < kStemPerThread; ++j) {
                                if (j == kStemPerThread - 1 && !last_ok) break;
                                const uint8_t* src = org + rel[j];
                                bool ok = true;
                                if (!interior) {
                                    const int y = iy0 + (prc[j] >> 8), x = ix0 + (prc[j] & 255);
                                    ok = (unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W;
                                    if (!ok) src = img;
                                }
                                okmask |= (ok ? 1u : 0u) << j;
                                raw[j][0] = __ldg(src);
                                if constexpr (!gray) { raw[j][1] = __ldg(src + 1); raw[j][2] = __ldg(src + 2); }
                            }
                        };
                        if constexpr (gray) fetch_bytes(std::integral_constant<int, 1>());
                        else if (px4) fetch_bytes(std::integral_constant<int, 4>());
                        else fetch_bytes(std::integral_constant<int, 3>());
                    } else {
                        const float* img = reinterpret_cast<const float*>(p.img.data) + (size_t)n * plane * (gray ? 1 : 3);
                        const float* org = img + (ptrdiff_t)iy0 * p.W + ix0;
#pragma unroll
                        for (int j = 0; j < kStemPerThread; ++j) {
                            if (j == kStemPerThread - 1 && !last_ok) break;
                            const float* src = org + rel[j];
                            bool ok = true;
                            if (!interior) {
                                const int y = iy0 + (prc[j] >> 8), x = ix0 + (prc[j] & 255);
                                ok = (unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W;
                                if (!ok) src = img;
                            }
                            okmask |= (ok ? 1u : 0u) << j;
                            raw[j][0] = __float_as_uint(__ldg(src));
                            if constexpr (!gray) { raw[j][1] = __float_as_uint(__ldg(src + plane)); raw[j][2] = __float_as_uint(__ldg(src + 2 * plane)); }
                        }
                    }
                };
                uint32_t it = 0;
                pdl_wait();
                if ((int)blockIdx.x < lg.num_tiles) fetch(blockIdx.x);
                for (int tile = blockIdx.x; tile < lg.num_tiles; tile += gridDim.x, ++it) {
                    const uint32_t s = it % SA, ph = (it / SA) & 1;
                    if (ptid == 0) LFD_TRACE(0, it, 0);
                    mbar_wait(&empty[s], ph ^ 1);
                    if (ptid == 0) LFD_TRACE(0, it, 1);
                    const uint32_t dst0 = smem_u32(ring) + s * p.stage_bytes + ptid * 8;
#pragma unroll
                    for (int j = 0; j < kStemPerThread; ++j) {
                        if (j == kStemPerThread - 1 && !last_ok) break;
                        uint32_t lo, hi;
                        if constexpr (gray) {
                            float v = u8 ? p.img.xf.apply(0, raw[j][0]) : __uint_as_float(raw[j][0]);     // NV12 / 4:2:2: the Y byte as it is
                            if (!((okmask >> j) & 1u)) v = 0.f;                                      // conv zero padding
                            lo = pack2<F16>(v, 0.f); hi = pack2<F16>(0.f, 0.f);                       // rounding point R0
                        } else {
                            if (nv12 || yuv422) nv12_to_bgr(raw[j][0], raw[j][1], raw[j][2], raw[j]);   // (Y, U, V) -> the bytes (B, G, R)
                            float f[3];
#pragma unroll
                            for (int k = 0; k < 3; ++k) {
                                f[k] = u8 ? p.img.xf.apply(k, raw[j][k]) : __uint_as_float(raw[j][k]);
                                if (!((okmask >> j) & 1u)) f[k] = 0.f;        // conv zero padding (of the normalised image)
                            }
                            const bool sw = p.img.xf.swap;           // u8 BGR -> RGB: the normalised bytes 0 and 2 change places
                            lo = pack2<F16>(sw ? f[2] : f[0], f[1]); hi = pack2<F16>(sw ? f[0] : f[2], 0.f);   // rounding point R0
                        }
                        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(dst0 + j * (kProdThreads * 8)), "r"(lo), "r"(hi) : "memory");
                    }
                    fence_proxy_async_smem();       // generic-proxy st.shared -> wgmma reads
                    mbar_arrive(&full[s]);
                    if (ptid == 0) LFD_TRACE(0, it, 2);
                    if (tile + (int)gridDim.x < lg.num_tiles) fetch(tile + gridDim.x);
                    if (ptid == 0) LFD_TRACE(0, it, 3);
                }
            };
            if (p.img.ch == 1) stem_producer(std::true_type());
            else stem_producer(std::false_type());
        } else {
        // every thread owns ONE 16-byte channel chunk (cpc divides 128) and walks the halo pixels with a fixed stride
        const int ch = ptid & (cpc - 1);
        const int px0 = ptid >> p.log2_cpc;
        const int pstep = kProd >> p.log2_cpc;
        const uint32_t ch_dst = ch * p.lbo_a;
        const int my_cnt = (p.n_px - px0 + pstep - 1) / pstep;   // halo pixels this thread copies per stage
        uint32_t it = 0;
        pdl_wait();                                   // the input activations are produced by the previous kernel
        for (int tile = blockIdx.x; tile < lg.num_tiles; tile += gridDim.x) {
            const int n = fast_div(tile, lg.magic_tpi);
            const int t = tile - n * lg.tiles_per_img;
            int iy0 = 0, ix0 = 0;
            if (MODE == MODE_FLAT) ix0 = t * 128;
            else {
                const int ty = fast_div(t, lg.magic_tx);
                int oy0 = ty * 16, ox0 = (t - ty * lg.tiles_x) * 8;
                iy0 = (MODE == MODE_3X3S1) ? oy0 : 2 * oy0;
                ix0 = (MODE == MODE_3X3S1) ? ox0 : 2 * ox0;
            }
            const __nv_bfloat16* img = p.in + (size_t)n * HW * p.Cin + ch * 8;
            // tiles whose halo lies inside the valid extent (the vast majority) copy without bounds checks: source = tile origin +
            // a per-pixel offset from the table.  (Flat tiles are pixel-local: they may read the rest of the tensor, whose results
            // land outside the valid extent.)
            constexpr int kDyMin = (MODE == MODE_1X1S2) ? 0 : -1, kDxMin = kDyMin;
            constexpr int kDyMax = (MODE == MODE_3X3S1) ? 16 : ((MODE == MODE_3X3S2) ? 31 : 30);
            constexpr int kDxMax = (MODE == MODE_3X3S1) ? 8 : ((MODE == MODE_3X3S2) ? 15 : 14);
            const bool interior = MODE == MODE_FLAT ? (ix0 + 128 <= HW)
                                                    : (iy0 + kDyMin >= 0 && ix0 + kDxMin >= 0 && iy0 + kDyMax < lg.H && ix0 + kDxMax < lg.W);
            // flat: first pixel of the tile; otherwise the halo's top-left pixel (in range for interior tiles)
            const __nv_bfloat16* org = img + (ptrdiff_t)(MODE == MODE_FLAT ? ix0 : (iy0 + kDyMin) * p.W + ix0 + kDxMin) * p.Cin;
            for (int cc = 0; cc < n_cc; ++cc, ++it) {
                const uint32_t s = it % SA, ph = (it / SA) & 1;
                if (ptid == 0) LFD_TRACE(0, it, 0);
                mbar_wait(&empty[s], ph ^ 1);
                if (ptid == 0) LFD_TRACE(0, it, 1);
                const uint32_t a_base = smem_u32(ring) + s * p.stage_bytes;
                if (!p.b_resident && ptid == 0) {
                    mbar_arrive_expect_tx(&full[s], p.b_slice_bytes);
                    bulk_g2s(a_base + p.a_stage_bytes, reinterpret_cast<const uint8_t*>(p.w) + (size_t)cc * p.b_slice_bytes,
                             p.b_slice_bytes, &full[s]);
                }
                const __nv_bfloat16* src_cc = img + cc * p.Cc;
                const uint32_t dst_cc = a_base + ch_dst;
                if (MODE == MODE_FLAT) {
                    if (interior) {
                        const __nv_bfloat16* src = org + cc * p.Cc + (size_t)px0 * p.Cin;
                        const size_t sstep = (size_t)pstep * p.Cin;
                        uint32_t dst = dst_cc + px0 * 16;
#pragma unroll 4
                        for (int pxi = px0; pxi < 128; pxi += pstep, src += sstep, dst += pstep * 16) cp_async16_full(dst, src);
                    } else {
#pragma unroll 4
                        for (int pxi = px0; pxi < 128; pxi += pstep) {
                            const int q = ix0 + pxi;
                            const bool ok = q < HW;
                            cp_async16(dst_cc + pxi * 16, src_cc + (ok ? q : 0) * p.Cin, ok);
                        }
                    }
                } else if (interior) {
                    const uint8_t* src = reinterpret_cast<const uint8_t*>(org + cc * p.Cc);
                    const PxEntry* tp = table + px0;
#pragma unroll 4
                    for (int k = 0; k < my_cnt; ++k, tp += pstep) {
                        const uint2 pe = *reinterpret_cast<const uint2*>(tp);
                        cp_async16_full(dst_cc + pe.y, src + pe.x);
                    }
                } else {
#pragma unroll 2
                    for (int pxi = px0; pxi < p.n_px; pxi += pstep) {
                        const PxDelta pd = delta[pxi];
                        const int y = iy0 + pd.dy, x = ix0 + pd.dx;
                        const bool ok = ((unsigned)y < (unsigned)lg.H) && ((unsigned)x < (unsigned)lg.W);
                        cp_async16(dst_cc + table[pxi].dst_off, src_cc + (ok ? (y * p.W + x) : 0) * p.Cin, ok);
                    }
                }
                cp_async_mbar_arrive(&full[s]);   // arrives when this thread's copies have landed
                if (ptid == 0) LFD_TRACE(0, it, 2);
            }
        }
        cp_async_wait_all();
        }
    }
    LFD_TL_END(p.tl);
}

template <int MODE, int COUT, bool F16, bool EXT, bool DS>
__global__ void __launch_bounds__(kConvThreads, 1) conv_umma_kernel(const __grid_constant__ UmmaConvParams p) {
    static_assert(COUT != 48, "48-channel outputs run in conv_umma_c48_kernel");
    conv_umma_body<MODE, COUT, F16, EXT, DS>(p);
}

// The 48-channel layers (TrafficLight LFD-S: its stem and stage 0): m64n48k16 MMAs into 24 accumulators per thread, the 48-channel
// tail only, and 96-byte output rows.  A symbol of its own, so that the set of conv_umma_kernel instantiations stays what it was.
template <int MODE, bool F16, bool EXT, bool DS>
__global__ void __launch_bounds__(kConvThreads, 1) conv_umma_c48_kernel(const __grid_constant__ UmmaConvParams p) {
    conv_umma_body<MODE, 48, F16, EXT, DS>(p);
}

// The 64-channel 3x3/s1 convs with one ring stage per tile and more tiles than CTAs: one consumer warpgroup per tile, the two
// warpgroups' MMA phases alternating (solo_consumers).  umma_conv_configure sets p.solo from the geometry.
template <bool F16, bool EXT>
__global__ void __launch_bounds__(kConvThreads, 1) conv_umma_solo_kernel(const __grid_constant__ UmmaConvParams p) {
    conv_umma_body<MODE_3X3S1, 64, F16, EXT, false, true>(p);
}

// ---------------------------------------------------------------------------------------------------
// MODE_STEM4: the 'faster' stem -- stem0 3x3/s2 3->64, stem1 1x1 64->64, stem2 3x3/s2 64->64, stem3 1x1 64->64 -- as ONE kernel.
// Tiles are 16 x 8 pixels of the final (stem3) map, as in MODE_3X3S2.  Each CTA walks a contiguous run of tiles in row-major
// order (floor or ceil of num_tiles / gridDim tiles).  Per tile:
//   producer   the raw-image patch (67 rows x 36 pixels from image (4 oy0 - 3, 4 ox0 - 3)) in the MODE_STEM format -> ring stage;
//   consumers  stem0 + stem1 on the 33 x 17 stem1 pixels stem2's halo needs (rows 2 oy0 - 1 .., columns 2 ox0 - 1 ..), as
//              MODE_STEM m64 blocks (s4_block), two per MMA group; each block's stem1 result (+shift, ReLU, 16-bit) goes into the
//              stem2 parity planes by stmatrix, zeros where the pixel lies outside the stem1 map (stem2's padding); then stem2 as
//              the MODE_3X3S2 main loop (same MMA order as the two-kernel path: k16-major, tap-minor), the stem3 tail and the TMA
//              store of the two-kernel path.
// Column 0 of tile (ty, tx + 1) is column 16 of tile (ty, tx).  So, within a run, a tile whose left neighbour came before it
// inherits that column (copied inside the planes after stem2 of the neighbour, see s4_slot) and computes columns 1..16 only:
// 9 blocks instead of 14.
// The stem1 tensor never exists outside shared memory.  Every wgmma group is waited for before the next barrier / divergent code.
// Trace (LFD_B200_TRACE builds, tests/debug_stem_fusion.py --trace), per tile lt:
//   role 0        producer            : wait_empty  got_empty  patch_written(arrived_full)  -
//   role 1 + wg   consumer warpgroup  : wait_full  got_full  stem01_done  plane_barrier_passed
//   role 3        entry 2 * lt + wg   : store_entry (= tail done)  after_bulk_wait_read  tma_issued  stem2_mma_done
static constexpr int kS4Rows = 67, kS4Cols = 36, kS4Pix = kS4Rows * kS4Cols;                      // 2412 patch pixels
static constexpr int kS4RowBytes = kS4Cols * 8;                                                    // 288
static constexpr int kS4PatchBytes = kS4Pix * 8;                                                   // 19296
static constexpr int kS4PerThread = (kS4Pix + kProdThreads - 1) / kProdThreads;                   // 19
static constexpr int kS4Batch = 5;                                                                 // patch pixels in flight per producer thread
// word loader: a patch row is 10 groups of 4 pixels = 3 aligned 32-bit words (see the producer)
static constexpr int kS4Groups = kS4Rows * 10;                                                     // 670
static constexpr int kS4GroupsPerThread = (kS4Groups + kProdThreads - 1) / kProdThreads;          // 6
static constexpr int kS4GroupBatch = 3;                                                            // groups in flight per producer thread
// The packed row-32 block reads up to 7 stem1 columns past the patch row (rows it discards); the last stage needs this tail.
static constexpr int kS4PatchOverrun = 768;
// Parity planes of the stem1 halo, per 8-channel chunk: [a odd, b odd] 16 x 9 | [a odd, b even] 16 x 9 | [a even, b odd] 17 x 9 |
// [a even, b even] 17 x 9 slots of 16 B (rows of pitch 9).  The even-b plane starts 3 slots (mod 8) after the odd-b plane of the
// same row parity: the 8 pixels b0 .. b0 + 7 (b0 odd) of one stmatrix then fill 8 distinct 16-byte bank groups.
LFD_DEVINL constexpr int s4_slot(int a, int b) {
    return ((a & 1) ? ((b & 1) ? 0 : 147) : ((b & 1) ? 291 : 446)) + (a >> 1) * 9 + (b >> 1);
}
static constexpr int kS4Lbo = 599 * 16;                                                            // plane pitch (odd in 16 B)
// shared-memory map (bytes)
static constexpr int kS4Bar = 0;                    // full[2] | empty[2] | weights | res_bar[2] (unused: no residual)
static constexpr int kS4Shift = 256;                // fp32 shifts of stem0 .. stem3, 64 each
static constexpr int kS4Staging = 2048;             // [warpgroup][64 rows x 64 channels], 1024-byte aligned (TMA swizzle)
static constexpr int kS4W0 = kS4Staging + 2 * 8192; // stem0 [3][2][64][8]
static constexpr int kS4W1 = kS4W0 + 6144;          // stem1 [8][64][8]
static constexpr int kS4W2 = kS4W1 + 8192;          // stem2 [9][8][64][8]
static constexpr int kS4W3 = kS4W2 + 73728;         // stem3 [8][64][8]
static constexpr int kS4Planes = kS4W3 + 8192;      // the parity planes x 8 channel chunks
static constexpr int kS4Ring = kS4Planes + 8 * kS4Lbo;
static constexpr int kS4Smem = kS4Ring + 2 * kS4PatchBytes + kS4PatchOverrun;   // 230720 (<= 227 KB)
static constexpr int kS4WBytes = kS4Planes - kS4W0;
static_assert(kS4Smem <= 227 * 1024, "stem4 shared memory");

// m64 block i of a tile's stem1 cover, origin (halo row a0, column b0):
//   i < 8     rows 8 (i / 2) .. + 7, columns 1 + 8 (i % 2) .. + 7     (every tile)
//   i = 8     row 32 packed: its 8-row groups step along the row (SBO = 8 stem1 columns), columns 1 .. 16 kept
//   9 .. 12   rows 8 (i - 9) .. + 7, columns 0 .. 7                   (tiles that do not inherit column 0)
//   i = 13    row 32 packed, columns 0 .. 15 kept
// Only the first two 8-row groups (warp 0 of the warpgroup) of a packed block are kept.
LFD_DEVINL void s4_block(int i, int& a0, int& b0, bool& packed) {
    packed = i == 8 || i == 13;
    a0 = packed ? 32 : 8 * (i < 8 ? i >> 1 : i - 9);
    b0 = i < 8 ? 1 + 8 * (i & 1) : (i == 8 ? 1 : 0);
}
// This CTA's run of tiles [t0, t1)
LFD_DEVINL void s4_run(int num_tiles, int& t0, int& t1) {
    t0 = (int)((uint64_t)blockIdx.x * (uint32_t)num_tiles / gridDim.x);
    t1 = (int)((uint64_t)(blockIdx.x + 1) * (uint32_t)num_tiles / gridDim.x);
}

LFD_DEVINL void consumers_bar_sync() { asm volatile("bar.sync 3, 256;" ::: "memory"); }   // the two consumer warpgroups

template <bool F16, bool EXT>
__global__ void __launch_bounds__(kConvThreads, 1) stem4_kernel(const __grid_constant__ UmmaConvParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kS4Bar);
    uint64_t* empty = full + 2;
    uint64_t* wbar = empty + 2;
    uint64_t* res_bar = wbar + 1;
    float* shifts = reinterpret_cast<float*>(smem + kS4Shift);
    pdl_launch_dependents();
    LFD_TL_BEGIN(p.tl);
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < 2; ++i) {
            mbar_init(&full[i], kProdThreads);
            mbar_init(&empty[i], kConsumerThreads / 32);
        }
        mbar_init(wbar, 1);
        mbar_init(&res_bar[0], 1);
        mbar_init(&res_bar[1], 1);
        fence_mbar_init();
    }
    if (tid < 256) {
        const int k = tid >> 6;
        const float* s = k == 0 ? p.shift : (k == 1 ? p.shift2 : (k == 2 ? p.shift_s2 : p.shift_s3));
        shifts[tid] = s ? round16<F16>(s[tid & 63]) : 0.f;
    }
    __syncthreads();
    // the valid image, stem3 map and tile grid; the runs and the inherited column below are defined over this grid
    const LaunchGrid lg = launch_grid<MODE_STEM4, EXT>(p);

    if (warp < kConsumerThreads / 32) {
        // ============================================================== CONSUMERS
        asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
        const int wg = warp >> 2;
        if (tid == 0) {
            mbar_arrive_expect_tx(wbar, kS4WBytes);
            auto load_w = [&](uint32_t dst, const __nv_bfloat16* src, uint32_t bytes) LFD_LAMBDA_INLINE {
                for (uint32_t off = 0; off < bytes; off += 32768)
                    bulk_g2s(smem_u32(smem) + dst + off, reinterpret_cast<const uint8_t*>(src) + off, bytes - off < 32768 ? bytes - off : 32768, wbar);
            };
            load_w(kS4W0, p.w, kS4W1 - kS4W0);
            load_w(kS4W1, p.w2, kS4W2 - kS4W1);
            load_w(kS4W2, p.w_s2, kS4W3 - kS4W2);
            load_w(kS4W3, p.w_s3, kS4Planes - kS4W3);
        }
        pdl_wait();
        mbar_wait(wbar, 0);

        EpiCtx e;
        e.stg_bytes = 8192u;
        e.nbuf = 1;
        e.stg = smem_u32(smem + kS4Staging) + (uint32_t)wg * 8192u;
        e.r0 = (warp & 3) * 16 + (lane >> 2);
        e.tq = lane & 3;
        e.wtid = tid & 127;
        e.wg = wg;
        e.lane = lane;
#ifdef LFD_B200_TRACE
        e.tr = p.trace && e.wtid == 0 ? p.trace + (3 * 32 + wg) * 4 : nullptr;
#endif
        const float* sh0 = shifts;
        const float* sh1 = shifts + 64;
        const float* sh2 = shifts + 128;
        const float* sh3 = shifts + 192;
        const uint32_t planes = smem_u32(smem + kS4Planes);
        // descriptors: stem0 A = the patch (MODE_STEM view: SBO = 2 patch rows, LBO = 16 B), B = [kh][2][64][8];
        // stem1 / stem3 B = [8][64][8]; stem2 A = the planes (SBO = pitch-9 rows, LBO = plane pitch), B = [tap][8][64][8]
        const uint64_t adesc_stem = wgmma_desc(0, 16, 2 * kS4RowBytes);
        const uint64_t adesc_row = wgmma_desc(0, 16, 8 * 16);          // packed row 32: 8-row groups 8 stem1 columns apart
        const uint64_t b0desc = wgmma_desc(smem_u32(smem + kS4W0), 64 * 16, 128);
        const uint64_t b1desc = wgmma_desc(smem_u32(smem + kS4W1), 64 * 16, 128);
        const uint64_t b2desc = wgmma_desc(smem_u32(smem + kS4W2), 64 * 16, 128);
        const uint64_t b3desc = wgmma_desc(smem_u32(smem + kS4W3), 64 * 16, 128);
        const uint64_t adesc_pl = wgmma_desc(planes + (uint32_t)wg * 8u * 144u, kS4Lbo, 144);
        // this thread's stem1 pixels inside a block: (row 2 (warp & 3) + h, column lane / 4); its stmatrix row address is the
        // pixel (row 2 (warp & 3) + sh, column sc), channel chunk lane / 16 (+ 2 per stmatrix)
        const int brow = 2 * (warp & 3), bcol = lane >> 2;
        const int sh = (lane >> 3) & 1, sc = lane & 7;

        const int H1 = EXT ? (lg.H - 1) / 2 + 1 : p.H1, W1 = EXT ? (lg.W - 1) / 2 + 1 : p.W1;   // the valid stem1 map
        int tile0, tile1;
        s4_run(lg.num_tiles, tile0, tile1);
        uint32_t store_count = 0, res_count = 0;
        for (int tile = tile0, lt = 0; tile < tile1; ++tile, ++lt) {
            const uint32_t s = lt & 1, ph = (lt >> 1) & 1;
            const int n = fast_div(tile, lg.magic_tpi);
            const int t = tile - n * lg.tiles_per_img;
            const int ty = fast_div(t, lg.magic_tx);
            const int tx = t - ty * lg.tiles_x;
            const int oy0 = ty * 16, ox0 = tx * 8;
            // column 0 was copied from the previous tile / column 16 goes to the next tile
            const bool inherit = tile > tile0 && tx > 0, pass_on = tile + 1 < tile1 && tx + 1 < lg.tiles_x;
            if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 0);
            mbar_wait(&full[s], ph);
            if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 1);
            fence_proxy_async_smem();
            const uint32_t patch = smem_u32(smem + kS4Ring) + s * kS4PatchBytes;

            // ---- stem0 + stem1, two blocks per MMA group: warpgroup 0 takes blocks 0 .. 4 (of 9) or 0 .. 6 (of 14), warpgroup 1
            //      the rest; an odd count repeats its last block (same bits to the same slots)
            const int nblk = inherit ? 9 : 14, half = (nblk + 1) >> 1;
            const int first = wg ? half : 0, cnt = wg ? nblk - half : half;
#pragma unroll 1
            for (int kp = 0; kp < (cnt + 1) >> 1; ++kp) {
                int blk[2] = {first + 2 * kp, first + min(2 * kp + 1, cnt - 1)};
                float c0[2][32];
                wgmma_fence_regs<32>(c0[0]);
                wgmma_fence_regs<32>(c0[1]);
                wgmma_fence();
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    int a0, b0;
                    bool packed;
                    s4_block(blk[q], a0, b0, packed);
                    const uint32_t boff = (uint32_t)(a0 * 2 * kS4RowBytes + b0 * 16);
                    const uint64_t ad = (packed ? adesc_row : adesc_stem) + ((patch + boff) >> 4);
#pragma unroll
                    for (int kh = 0; kh < 3; ++kh)
                        wgmma_ss<64, F16>(c0[q], ad + (uint32_t)(kh * kS4RowBytes / 16), b0desc + (uint32_t)(kh * 2 * 64 * 16 / 16), kh != 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<32>(c0[0]);
                wgmma_fence_regs<32>(c0[1]);
                // stem0 (+shift, ReLU) -> 16 bits -> register A operand of stem1, exactly as the fused tail of the two-kernel path
                uint32_t a1[2][16];
#pragma unroll
                for (int q = 0; q < 2; ++q)
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        const int c = 16 * kk + 2 * e.tq;
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const float x0 = c0[q][8 * kk + 2 * r] + sh0[c + 8 * (r >> 1)], x1 = c0[q][8 * kk + 2 * r + 1] + sh0[c + 8 * (r >> 1) + 1];
                            a1[q][4 * kk + r] = p.relu ? pack2_relu<F16>(x0, x1) : pack2<F16>(x0, x1);
                        }
                    }
                float c1[2][32];
                wgmma_fence_regs<32>(c1[0]);
                wgmma_fence_regs<32>(c1[1]);
                wgmma_fence();
                tail_mma<64, 64, F16>(c1[0], a1[0], b1desc);
                tail_mma<64, 64, F16>(c1[1], a1[1], b1desc);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs<32>(c1[0]);
                wgmma_fence_regs<32>(c1[1]);
                // stem1 (+shift, ReLU) -> 16 bits -> the stem2 parity planes; zeros outside the stem1 map (stem2's padding).
                // One 8x8 stmatrix = 8 channels (one plane chunk) of 8 pixels of one block row, each a 16-byte plane slot.
                float2 bv[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) bv[j] = *reinterpret_cast<const float2*>(sh1 + 8 * j + 2 * e.tq);
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    int a0, b0;
                    bool packed;
                    s4_block(blk[q], a0, b0, packed);
                    if (packed && (warp & 3)) continue;         // warp-uniform: the discarded groups of the packed row
                    uint32_t v[8][2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int a = packed ? a0 : a0 + brow + h, b = b0 + bcol + (packed ? 8 * h : 0);
                        const int y1 = 2 * oy0 - 1 + a, x1 = 2 * ox0 - 1 + b;
                        const bool in = (unsigned)y1 < (unsigned)H1 && (unsigned)x1 < (unsigned)W1;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const float x0 = c1[q][4 * j + 2 * h] + bv[j].x, x1v = c1[q][4 * j + 2 * h + 1] + bv[j].y;
                            const uint32_t w = p.relu2 ? pack2_relu<F16>(x0, x1v) : pack2<F16>(x0, x1v);
                            v[j][h] = in ? w : 0u;
                        }
                    }
                    const int a = packed ? a0 : a0 + brow + sh, b = b0 + sc + (packed ? 8 * sh : 0);
                    const uint32_t addr = planes + (uint32_t)s4_slot(a, b) * 16u + (uint32_t)(lane >> 4) * kS4Lbo;
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        stmatrix_x4(addr + (uint32_t)(2 * k * kS4Lbo), v[2 * k][0], v[2 * k][1], v[2 * k + 1][0], v[2 * k + 1][1]);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);      // this warp's stem0 MMAs have read the patch
            if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 2);
            fence_proxy_async_smem();                   // st.shared (generic proxy) -> wgmma (async proxy) reads of the planes
            consumers_bar_sync();
            if (e.wtid == 0) LFD_TRACE(1 + wg, lt, 3);

            // ---- stem2: the MODE_3X3S2 main loop over the planes
            float acc[32];
            wgmma_fence_regs<32>(acc);
            wgmma_fence();
#pragma unroll
            for (int k16 = 0; k16 < 4; ++k16)
#pragma unroll
                for (int tap = 0; tap < 9; ++tap)
                    wgmma_ss<64, F16>(acc, adesc_pl + (uint32_t)(k16 * 2 * kS4Lbo / 16 + s4_slot(tap / 3, tap % 3)),
                                      b2desc + (uint32_t)((tap * 8 + 2 * k16) * 64 * 16 / 16), (k16 | tap) != 0);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs<32>(acc);
            consumers_bar_sync();                       // both warpgroups are done reading the planes: the next tile may write them
            if (pass_on) {
                // column 16 -> column 0 (even-b slot 8 -> 0) for the next tile.  Each row is copied by the warp that writes its
                // column 16 in the next tile (blocks 1, 3 | 5, 7 and the packed block 8 of warpgroup 0 | 1: warp w writes rows
                // a0 + 2w, + 1), so program order alone keeps the copy ahead of that write; no barrier is needed.
                const int rs = lane >> 3, a = 16 * wg + brow + (rs & 1) + 8 * (rs >> 1);
                const uint32_t src = planes + (uint32_t)(lane & 7) * kS4Lbo + (uint32_t)s4_slot(a, 16) * 16u;
                sts128(src - 8u * 16u, lds128(src));
                if (wg == 1 && brow == 0 && lane < 8) {
                    const uint32_t src32 = planes + (uint32_t)lane * kS4Lbo + (uint32_t)s4_slot(32, 16) * 16u;
                    sts128(src32 - 8u * 16u, lds128(src32));
                }
                __syncwarp();
            }
#ifdef LFD_B200_TRACE
            if (e.wtid == 0 && p.trace && blockIdx.x == 0 && lt < 16) p.trace[(3 * 32 + wg + 2 * lt) * 4 + 3] = clock64();
#endif

            // ---- stem3: fused 1x1 tail and the tile store, as in the two-kernel path
            uint32_t a2[16];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const int c = 16 * kk + 2 * e.tq;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    const float x0 = acc[8 * kk + 2 * r] + sh2[c + 8 * (r >> 1)], x1 = acc[8 * kk + 2 * r + 1] + sh2[c + 8 * (r >> 1) + 1];
                    a2[4 * kk + r] = p.relu_s2 ? pack2_relu<F16>(x0, x1) : pack2<F16>(x0, x1);
                }
            }
            float acc2[32];
            wgmma_fence_regs<32>(acc2);
            wgmma_fence();
            tail_mma<64, 64, F16>(acc2, a2, b3desc);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs<32>(acc2);
            store_tile<MODE_3X3S2, 64, F16>(e, acc2, 64, sh3, (bool)p.relu_s3, false, nullptr, &p.tm_out, &p.tm_res, ox0, oy0 + wg * 8, n,
                                            true, true, &res_bar[wg], store_count, res_count);
        }
        if (e.wtid == 0) bulk_wait_all();
    } else {
        // ============================================================== PRODUCER: raw image patch -> normalised 16-bit [row][pixel][b g r 0]
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int ptid = tid - kConsumerThreads;
        // A gray image (p.img.ch == 1) has one value per pixel, written as (v, 0, 0, 0): the body is specialised for it and for the format
        // at compile time (image.cuh), so the BGR loaders are exactly what they are without it.
        auto s4_producer = [&](auto ch_c, auto fmt_c) LFD_LAMBDA_INLINE {
            constexpr int CH = decltype(ch_c)::value, FMT = decltype(fmt_c)::value;
            pdl_wait();
            int tile0, tile1;
            s4_run(lg.num_tiles, tile0, tile1);
            for (int tile = tile0, lt = 0; tile < tile1; ++tile, ++lt) {
                const uint32_t s = lt & 1, ph = (lt >> 1) & 1;
                const int n = fast_div(tile, lg.magic_tpi), t = tile - n * lg.tiles_per_img;
                const int ty = fast_div(t, lg.magic_tx);
                const int iy0 = 4 * 16 * ty - 3, ix0 = 4 * 8 * (t - ty * lg.tiles_x) - 3;
                const bool interior = iy0 >= 0 && ix0 >= 0 && iy0 + kS4Rows <= lg.H && ix0 + kS4Cols <= lg.W;
                if (ptid == 0) LFD_TRACE(0, lt, 0);
                mbar_wait(&empty[s], ph ^ 1);
                if (ptid == 0) LFD_TRACE(0, lt, 1);
                const uint32_t dst0 = smem_u32(smem + kS4Ring) + s * kS4PatchBytes;
                if (FMT != LFD_INPUT_F32_NCHW && p.in_words) {
                    // ix0 = 1 (mod 4): group g of a patch row = image columns ix0 - 1 + 4g .. + 3 = patch columns 4g - 1 .. 4g + 2, whole
                    // aligned words (image_load_words).  A group lies wholly inside or wholly outside the tensor, so no load touches a byte
                    // outside it; a valid width that is not a multiple of 4 ends inside a group, whose pixels past it are zeroed one by one.
                    // Two batches of 3 groups: all loads of a batch are issued before any is used (6 groups at once do not fit the
                    // producer's 56 registers).
#pragma unroll 1
                    for (int j0 = 0; j0 < kS4GroupsPerThread; j0 += kS4GroupBatch) {
                        uint32_t wd[kS4GroupBatch][kImageWords<CH, FMT>];
                        bool ok[kS4GroupBatch];
#pragma unroll
                        for (int j = 0; j < kS4GroupBatch; ++j) {
                            const int q = ptid + (j0 + j) * kProdThreads;
                            const int r = q / 10, g = q - r * 10;
                            const int y = iy0 + r, x = ix0 - 1 + 4 * g;
                            ok[j] = q < kS4Groups && (unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W;
                            image_load_words<CH, FMT>(p.img, n, y, x, ok[j], wd[j]);
                        }
#pragma unroll
                        for (int j = 0; j < kS4GroupBatch; ++j) {
                            const int q = ptid + (j0 + j) * kProdThreads;
                            if (q >= kS4Groups) break;
                            const int r = q / 10, g = q - r * 10;
                            const int in_cols = lg.W - (ix0 - 1 + 4 * g);    // pixels k < in_cols of the group lie inside the valid width
                            uint2 px[4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                uint32_t raw[CH];
                                float f[3];
                                image_unpack_word<CH, FMT>(wd[j], k, raw);
                                image_decode<CH, FMT>(p.img, raw, ok[j] && (!EXT || k < in_cols), f);
                                px[k] = pack_px<F16>(f);
                            }
                            const uint32_t d = dst0 + (uint32_t)(r * kS4RowBytes + 32 * g);              // patch column 4g, 16-byte aligned
                            if (g > 0) asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(d - 8u), "r"(px[0].x), "r"(px[0].y) : "memory");
                            if (g < 9) {
                                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(d), "r"(px[1].x), "r"(px[1].y), "r"(px[2].x),
                                             "r"(px[2].y) : "memory");
                                asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(d + 16u), "r"(px[3].x), "r"(px[3].y) : "memory");
                            }
                        }
                    }
                } else {
                    // per-pixel loader: fp32 NCHW, or uint8 (BGR / gray / NV12 / 4:2:2 / 4-byte) rows that are not whole aligned words
#pragma unroll 1
                    for (int j0 = 0; j0 < kS4PerThread; j0 += kS4Batch) {
                        uint32_t raw[kS4Batch][CH];
                        bool ok[kS4Batch];
#pragma unroll
                        for (int j = 0; j < kS4Batch; ++j) {
                            const int q = ptid + (j0 + j) * kProdThreads;
                            const int r = q / kS4Cols, c = q - r * kS4Cols;
                            const int y = iy0 + r, x = ix0 + c;
                            ok[j] = q < kS4Pix && (interior || ((unsigned)y < (unsigned)lg.H && (unsigned)x < (unsigned)lg.W));
                            image_load<CH, FMT>(p.img, n, image_px<CH, FMT>(p.img, y, x), y, x, ok[j], raw[j]);
                        }
#pragma unroll
                        for (int j = 0; j < kS4Batch; ++j) {
                            const int q = ptid + (j0 + j) * kProdThreads;
                            if (q >= kS4Pix) break;
                            float f[3];
                            image_decode<CH, FMT>(p.img, raw[j], ok[j], f);
                            const uint2 v = pack_px<F16>(f);
                            asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(dst0 + q * 8), "r"(v.x), "r"(v.y) : "memory");
                        }
                    }
                }
                fence_proxy_async_smem();
                mbar_arrive(&full[s]);
                if (ptid == 0) LFD_TRACE(0, lt, 2);
            }
        };
        image_dispatch(p.img, s4_producer);
    }
    LFD_TL_END(p.tl);
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
// solo: the layout of conv_umma_solo_kernel, whose warpgroups stage all 128 rows of a tile
static int configure_with(const ConvGeom& g, int num_sms, int nbuf, bool solo, UmmaConvParams* out, size_t* smem_bytes, int* grid) {
    UmmaConvParams p;
    memset(&p, 0, sizeof(p));
    p.stg_nbuf = nbuf;
    p.solo = solo ? 1 : 0;
    int mode;
    if (g.stem) {
        if (g.ksize != 3 || g.stride != 2 || g.Cin != 16) return -1;   // "Cin" = K of one filter row: 4 pixels x 4 padded channels
        mode = MODE_STEM;
    } else if (g.ksize == 1 && g.stride == 1) mode = MODE_FLAT;
    else if (g.ksize == 3 && g.stride == 1) mode = MODE_3X3S1;
    else if (g.ksize == 3 && g.stride == 2) mode = MODE_3X3S2;
    else if (g.ksize == 1 && g.stride == 2) mode = MODE_1X1S2;
    else return -1;
    // instantiated output widths (conv_umma_launch): 16 / 32 / 48 / 64 / 128 channels, 3x3 convs from 32
    if (g.Cin % 16 || (g.Cout != 16 && g.Cout != 32 && g.Cout != 48 && g.Cout != 64 && g.Cout != 128)) return -1;
    if ((mode == MODE_3X3S1 || mode == MODE_3X3S2) && g.Cout < 32) return -1;
    p.mode = mode;
    p.N = g.N; p.H = g.H; p.W = g.W; p.Cin = g.Cin; p.Ho = g.Ho; p.Wo = g.Wo; p.Cout = g.Cout;
    const int taps = g.stem ? 3 : g.ksize * g.ksize;   // stem: one MMA group per filter row
    int px_slots;  // plane size in pixels (slots), n_px = pixels actually loaded
    if (mode == MODE_FLAT) {
        p.tiles_x = 0; p.tiles_per_img = (g.Ho * g.Wo + 127) / 128;
        p.n_px = 128; px_slots = 128; p.sbo_a = 128;
    } else {
        p.tiles_x = (g.Wo + 7) / 8;
        p.tiles_per_img = p.tiles_x * ((g.Ho + 15) / 16);
        if (mode == MODE_3X3S1) { p.n_px = 180; px_slots = 180; p.sbo_a = 160; }
        else if (mode == MODE_3X3S2) { p.n_px = 561; px_slots = 594; p.sbo_a = 144; }
        else { p.n_px = 128; px_slots = 128; p.sbo_a = 128; }   // MODE_1X1S2 (and, overridden below, MODE_STEM)
    }
    // plane pitch = odd multiple of 16 B: the 8 chunks of a pixel fall into 8 distinct 16-byte bank groups
    const int plane_slots = px_slots | 1;
    p.lbo_a = plane_slots * 16;
    if (mode == MODE_STEM) { p.lbo_a = 16; p.sbo_a = 2 * kStemRowBytes; }   // overlapping view of the 4-channel patch
    p.num_tiles = p.tiles_per_img * g.N;
    if (p.num_tiles >= (1 << 24) || p.tiles_per_img >= (1 << 16)) return -5;
    p.magic_tpi = ((1ull << 40) + p.tiles_per_img - 1) / p.tiles_per_img;
    p.magic_tx = p.tiles_x ? ((1ull << 40) + p.tiles_x - 1) / p.tiles_x : 0;
    const int Cf = g.tail_cout > 0 ? g.tail_cout : g.Cout;
    if (g.ds_cout && (mode != MODE_3X3S2 || g.tail_cout || g.ds_cout != g.Cout)) return -6;
    if (g.tail_cout && (g.tail_cout % 16 || g.tail_cout > 128 || g.tail_cout < 16)) return -4;
    if (g.tail_cout && (g.tail_cout == 48) != (g.Cout == 48)) return -4;   // a 48-channel conv has the 48-channel tail only
    const size_t staging = (size_t)nbuf * (solo ? 256 : 128) * Cf * 2;   // [warpgroup][buffer][64 rows (solo: 128)][Cf]
    // fixed head of the shared-memory map: barriers | [halo table] | shift | [tail shift] | staging (1 KB aligned)
    size_t hoff = kSmemTableOff;
    p.smem_table_off = (uint32_t)hoff;
    if (mode != MODE_FLAT && mode != MODE_STEM) hoff += ((size_t)p.n_px * 10 + 127) & ~(size_t)127;   // PxEntry[n_px] | PxDelta[n_px]
    p.smem_bias_off = (uint32_t)hoff; hoff += ((size_t)g.Cout * 4 + 15) & ~(size_t)15;
    p.smem_bias2_off = (uint32_t)hoff; hoff += ((size_t)(g.tail_cout + g.ds_cout) * 4 + 15) & ~(size_t)15;
    p.smem_staging_off = (uint32_t)((hoff + 1023) & ~(size_t)1023);
    const size_t fixed = p.smem_staging_off + staging;
    // what lives behind the ring: the weights of the fused tail / shortcut conv
    const size_t w2_bytes = g.tail_cout ? ((size_t)g.Cout * g.tail_cout * 2 + 127) & ~(size_t)127
                                        : (g.ds_cout ? ((size_t)g.Cin * g.ds_cout * 2 + 127) & ~(size_t)127 : 0);
    const size_t post = w2_bytes;
    const size_t budget = 224 * 1024 - post;
    const size_t w_total = (size_t)taps * g.Cin * g.Cout * 2;
    // Choose the channel chunk Cc, weight residency and ring depth.  Preference order:
    //   1. resident weights (loaded once per CTA) with >= 3 A stages, the largest Cc first;
    //   2. otherwise streamed weights: the largest Cc that still gives >= 4 stages (deep ring hides the per-stage
    //      weight fetch), then >= 3, then >= 2.
    const int cands[3] = {64, 32, 16};
    int best_cc = 0, best_res = 0, best_st = 0;
    auto a_bytes = [&](int cc) -> size_t {
        if (mode == MODE_STEM) return kStemPatchBytes;
        return (((size_t)plane_slots * (cc / 8) * 16) + 127) & ~(size_t)127;
    };
    auto stages_for = [&](int cc, int resident) -> int {
        if (g.Cin % cc) return 0;
        const size_t b_slice = (size_t)taps * cc * g.Cout * 2;
        const size_t stage = a_bytes(cc) + (resident ? 0 : b_slice);
        if (fixed + (resident ? w_total : 0) + 2 * stage > budget) return 0;
        int st = (int)((budget - fixed - (resident ? w_total : 0)) / stage);
        if (st > kMaxStages) st = kMaxStages;
        if (st > 4 && stage >= 8192) st = 4;
        return st;
    };
    // (16-channel chunks mean 32-byte global segments per pixel and twice the barrier round trips per tile, so a 2-deep ring of
    //  32-channel stages is preferred to a 4-deep one of 16)
    for (int pass = 0; pass < 3 && !best_cc; ++pass)
        for (int ci = 0; ci < 3 && !best_cc; ++ci) {
            const int want = pass == 0 ? 3 : 2;
            if (pass < 2 && cands[ci] < 32) continue;
            int st = stages_for(cands[ci], 1);
            if (st >= want) { best_cc = cands[ci]; best_res = 1; best_st = st; }
        }
    // Streaming re-reads the whole filter bank from L2 for every tile, so it is taken only when the weights cannot be
    // resident next to a ring of >= 2 stages of >= 32 channels.
    if (!best_cc || (best_st < 3 && best_cc < 32)) {
        for (int want = 4; want >= 2; --want) {
            bool found = false;
            for (int ci = 0; ci < 3 && !found; ++ci) {
                int st = stages_for(cands[ci], 0);
                if (st >= want && (!best_cc || st > best_st)) { best_cc = cands[ci]; best_res = 0; best_st = st; found = true; }
            }
            if (found) break;
        }
    }
    if (!best_cc) return -2;
    p.Cc = best_cc; p.b_resident = best_res; p.stages = best_st;
    p.a_stage_bytes = (uint32_t)a_bytes(best_cc);
    p.b_slice_bytes = (uint32_t)((size_t)taps * best_cc * g.Cout * 2);
    p.stage_bytes = p.a_stage_bytes + (best_res ? 0 : p.b_slice_bytes);
    p.w_total_bytes = (uint32_t)w_total;
    p.smem_w_off = (uint32_t)fixed;
    p.smem_ring_off = (uint32_t)(fixed + (best_res ? w_total : 0));
    auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
    p.log2_cpc = ilog2(p.Cc / 8);
    p.Cf = Cf;
    p.Cout2 = g.tail_cout;
    p.Cout3 = g.ds_cout;
    p.log2_cpr = ilog2(Cf / 8);
    if ((1 << p.log2_cpr) != Cf / 8 && Cf != 48) return -3;       // stored channel count must be 16/32/48/64/128
    size_t off = p.smem_ring_off + (size_t)p.stages * p.stage_bytes;
    p.smem_w2_off = (uint32_t)off; off += w2_bytes;
    *smem_bytes = off;
    *grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
    *out = p;
    return 0;
}

static int configure_stem4(const ConvGeom& g, int num_sms, UmmaConvParams* out, size_t* smem_bytes, int* grid) {
    if ((g.Cin != 3 && g.Cin != 1) || g.ksize != 3 || g.stride != 2 || g.Cout != 64 || g.tail_cout != 64 || g.ds_cout) return -1;
    UmmaConvParams p;
    memset(&p, 0, sizeof(p));
    p.mode = MODE_STEM4;
    p.N = g.N; p.H = g.H; p.W = g.W; p.Cin = 3; p.Cout = 64; p.Cout2 = 64; p.Cf = 64;
    p.H1 = (g.H - 1) / 2 + 1; p.W1 = (g.W - 1) / 2 + 1;           // stem0 / stem1 map
    p.Ho = (p.H1 - 1) / 2 + 1; p.Wo = (p.W1 - 1) / 2 + 1;         // stem2 / stem3 map
    if (g.H < 1 || g.W < 1 || g.Ho != p.Ho || g.Wo != p.Wo) return -1;
    p.tiles_x = (p.Wo + 7) / 8;
    p.tiles_per_img = p.tiles_x * ((p.Ho + 15) / 16);
    p.num_tiles = p.tiles_per_img * g.N;
    if (p.num_tiles >= (1 << 24) || p.tiles_per_img >= (1 << 16)) return -5;
    p.magic_tpi = ((1ull << 40) + p.tiles_per_img - 1) / p.tiles_per_img;
    p.magic_tx = ((1ull << 40) + p.tiles_x - 1) / p.tiles_x;
    p.stg_nbuf = 1; p.stages = 2;
    *smem_bytes = kS4Smem;
    *grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
    *out = p;
    return 0;
}

int umma_conv_configure(const ConvGeom& g, int num_sms, UmmaConvParams* out, size_t* smem_bytes, int* grid) {
    if (g.stem4) return configure_stem4(g, num_sms, out, smem_bytes, grid);
    // a second staging buffer per warpgroup is taken when it costs neither weight residency nor ring depth
    UmmaConvParams p1, p2;
    size_t s1 = 0, s2 = 0;
    int g1 = 0, g2 = 0;
    const int rc = configure_with(g, num_sms, 1, false, &p1, &s1, &g1);
    if (rc) return rc;
    if (configure_with(g, num_sms, 2, false, &p2, &s2, &g2) == 0 && p2.b_resident == p1.b_resident &&
        p2.Cc == p1.Cc && p2.stages >= (p1.stages < 3 ? p1.stages : 3)) {
        *out = p2; *smem_bytes = s2; *grid = g2;
    } else {
        *out = p1; *smem_bytes = s1; *grid = g1;
    }
    // conv_umma_solo_kernel for the 64-channel 3x3/s1 convs with one resident-weight ring stage per tile (a 64-channel conv never has
    // GroupNorm statistics, a 3x3/s1 conv never a shortcut) and more tiles than CTAs, so that the warpgroups have tiles to alternate
    // on (measured on WIDERFACE-S 720p b8: the 45x80 layers, 240 tiles, gain from it; the 23x40 ones, 80 tiles, gain nothing).  One
    // staging region per warpgroup (its stores have drained by the time its next tile, two tiles later, is staged) and a ring of at
    // least 3 stages: two tiles are consumed while the next one fills.
    const bool solo_geom = !g.stem && g.ksize == 3 && g.stride == 1 && g.Cin == 64 && g.Cout == 64 && !g.tail_cout && !g.ds_cout;
    if (solo_geom && out->Cc == 64 && out->b_resident && out->num_tiles > *grid &&
        configure_with(g, num_sms, 1, true, &p1, &s1, &g1) == 0 && p1.b_resident && p1.Cc == 64 && p1.stages >= 3) {
        *out = p1; *smem_bytes = s1; *grid = g1;
    }
    return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// One tensor map per stored tensor; the box is what ONE warpgroup moves: 64 tile rows (64 pixels of a flat tile, 8 x 8 of
// a spatial one) x min(64, Cf) channels, shared-memory side in the matching swizzle mode.  A 48-channel tensor has 96-byte rows, which
// no swizzle mode spans: its box is the whole row, unswizzled, so a store or a residual load covers channels 0-47 of its pixels and
// nothing of the next pixel.
static int encode_one(const UmmaConvParams& p, const void* ptr, CUtensorMap* tm) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return -1;
    const cuuint64_t Cf = p.Cf, HoWo = (cuuint64_t)p.Ho * p.Wo;
    const cuuint32_t inner = p.Cf < 64 ? p.Cf : 64;
    const CUtensorMapSwizzle swz = inner * 2 >= 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : (inner * 2 == 96 ? CU_TENSOR_MAP_SWIZZLE_NONE
                                                    : (inner * 2 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B));
    cuuint64_t dims[4], strides[3];
    cuuint32_t box[4], estr[4] = {1, 1, 1, 1};
    cuuint32_t rank;
    if (p.mode == MODE_FLAT) {
        rank = 3;
        dims[0] = Cf; dims[1] = HoWo; dims[2] = p.N;
        strides[0] = Cf * 2; strides[1] = HoWo * Cf * 2;
        box[0] = inner; box[1] = 64; box[2] = 1;
    } else {
        rank = 4;
        dims[0] = Cf; dims[1] = p.Wo; dims[2] = p.Ho; dims[3] = p.N;
        strides[0] = Cf * 2; strides[1] = (cuuint64_t)p.Wo * Cf * 2; strides[2] = HoWo * Cf * 2;
        box[0] = inner; box[1] = 8; box[2] = 8; box[3] = 1;
    }
    CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : -2;
}

int umma_conv_encode_maps(UmmaConvParams* p) {
    if (encode_one(*p, p->out, &p->tm_out)) return -1;
    if (p->res && encode_one(*p, p->res, &p->tm_res)) return -1;
    if (p->Cout3 && encode_one(*p, p->out3, &p->tm_out3)) return -1;
    return 0;
}

// configured: one flag per device ordinal of the kernel's own (cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute)
static cudaError_t launch_persistent(void (*kernel)(UmmaConvParams), bool* configured, int max_smem, const UmmaConvParams& p, size_t smem,
                                     int grid, cudaStream_t st) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
        if (e != cudaSuccess) return e;
        configured[dev] = true;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(kConvThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, p);
}

template <int MODE, int COUT, bool F16, bool EXT, bool DS>
static cudaError_t launch_mode_t(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    static bool configured[kMaxDevices] = {};
    if constexpr (COUT == 48) return launch_persistent(conv_umma_c48_kernel<MODE, F16, EXT, DS>, configured, 224 * 1024, p, smem, grid, st);
    else return launch_persistent(conv_umma_kernel<MODE, COUT, F16, EXT, DS>, configured, 224 * 1024, p, smem, grid, st);
}

template <int MODE, int COUT, bool F16, bool EXT>
static cudaError_t launch_mode_ds(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    if constexpr (MODE == MODE_3X3S2)
        if (p.Cout3) return launch_mode_t<MODE, COUT, F16, EXT, true>(p, smem, grid, st);
    if constexpr (MODE == MODE_3X3S1 && COUT == 64)
        if (p.solo) {
            static bool configured[kMaxDevices] = {};
            return launch_persistent(conv_umma_solo_kernel<F16, EXT>, configured, 224 * 1024, p, smem, grid, st);
        }
    return launch_mode_t<MODE, COUT, F16, EXT, false>(p, smem, grid, st);
}

template <bool F16, bool EXT>
static cudaError_t launch_stem4_t(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    static bool configured[kMaxDevices] = {};
    return launch_persistent(stem4_kernel<F16, EXT>, configured, kS4Smem, p, smem, grid, st);
}

template <bool F16>
static cudaError_t launch_stem4(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    return p.ext ? launch_stem4_t<F16, true>(p, smem, grid, st) : launch_stem4_t<F16, false>(p, smem, grid, st);
}

template <int MODE, int COUT, bool F16>
static cudaError_t launch_mode_e(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    return p.ext ? launch_mode_ds<MODE, COUT, F16, true>(p, smem, grid, st) : launch_mode_ds<MODE, COUT, F16, false>(p, smem, grid, st);
}

template <int MODE, int COUT>
static cudaError_t launch_mode(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    return p.f16 ? launch_mode_e<MODE, COUT, true>(p, smem, grid, st) : launch_mode_e<MODE, COUT, false>(p, smem, grid, st);
}

// the output widths umma_conv_configure accepts per mode (and only those are instantiated)
template <int MODE>
static cudaError_t launch_cout(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    switch (p.Cout) {
        case 16: if constexpr (MODE != MODE_3X3S1 && MODE != MODE_3X3S2) return launch_mode<MODE, 16>(p, smem, grid, st); break;
        case 32: return launch_mode<MODE, 32>(p, smem, grid, st);
        case 48: return launch_mode<MODE, 48>(p, smem, grid, st);
        case 64: return launch_mode<MODE, 64>(p, smem, grid, st);
        case 128: if constexpr (MODE != MODE_STEM) return launch_mode<MODE, 128>(p, smem, grid, st); break;
    }
    return cudaErrorInvalidValue;
}

cudaError_t umma_conv_launch(const UmmaConvParams& p, size_t smem, int grid, cudaStream_t st) {
    switch (p.mode) {
        case MODE_FLAT: return launch_cout<MODE_FLAT>(p, smem, grid, st);
        case MODE_3X3S1: return launch_cout<MODE_3X3S1>(p, smem, grid, st);
        case MODE_3X3S2: return launch_cout<MODE_3X3S2>(p, smem, grid, st);
        case MODE_1X1S2: return launch_cout<MODE_1X1S2>(p, smem, grid, st);
        case MODE_STEM: return launch_cout<MODE_STEM>(p, smem, grid, st);
        case MODE_STEM4: return p.f16 ? launch_stem4<true>(p, smem, grid, st) : launch_stem4<false>(p, smem, grid, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace lfd
