// train.cu -- the SIMT (HBM-bound) kernels of the training step: parameter staging, BatchNorm batch statistics / apply,
// BatchNorm / GroupNorm backward, the backward of the final head convs, the stem conv's weight gradient, gradient-norm
// clipping + SGD.  The GEMM-shaped parts (forward convs, dgrad, wgrad) run on the tensor cores (wgmma: conv_umma.cu, wgrad_umma.cu).
//
// Reference semantics (what autograd computes for the reference's modules in train mode):
//   BatchNorm2d      lfd/model/backbone/lfd_resnet.py:10-18 (nn.BatchNorm2d defaults: eps 1e-5, momentum 0.1, biased variance
//                    for the normalisation, unbiased for the running estimate)
//   GroupNorm + ReLU lfd/model/head/lfd_head.py:85-135
//   final convs      lfd/model/head/lfd_head.py:137-143,164-185 (Scale multiplies conv output AND bias, :177-180)
//   optimizer step   lfd/execution/hooks/optimizer_hook.py:21-36 (clip_grad_norm_ then torch.optim.SGD.step)
#include <type_traits>

#include "train.cuh"

#include "conv_common.cuh"
#include "ptx.cuh"

namespace lfd {

namespace {

LFD_DEVINL void unpack8(const uint4 q, float* f) {
    f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
    f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
}
LFD_DEVINL uint4 pack8f(const float* f) {
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]); o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
    return o;
}

// Every thread of a 256-thread block holds NV partial sums that belong to "chunk group" (tid % cpr) (cpr = power of two <= 32,
// the number of 16-byte channel chunks per row).  Sums them over the block; afterwards sh[grp * NV + v] holds the totals.
template <int NV>
LFD_DEVINL void block_reduce_groups(float* v, int cpr, float* sh /* [8 warps][cpr <= 32][NV] */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int off = cpr; off < 32; off <<= 1)
#pragma unroll
        for (int i = 0; i < NV; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], off);
    if (lane < cpr)
#pragma unroll
        for (int i = 0; i < NV; ++i) sh[(warp * cpr + lane) * NV + i] = v[i];
    __syncthreads();
    const int total = cpr * NV;
    for (int t = threadIdx.x; t < total; t += 256) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += sh[w * total + t];
        sh[8 * total + t] = s;   // result area behind the per-warp partials
    }
    __syncthreads();
}
static constexpr int kRedFloats(int nv) { return 9 * 32 * nv; }

LFD_DEVINL void mean_rstd_from_sums(const double* sums, int idx, double count, float eps, float* mean, float* rstd, double* var_out = nullptr) {
    const double m = sums[2 * idx] / count;
    double var = sums[2 * idx + 1] / count - m * m;
    if (var < 0) var = 0;
    *mean = (float)m;
    *rstd = (float)(1.0 / sqrt(var + (double)eps));
    if (var_out) *var_out = var;
}

}  // namespace

// ===================================================================================================
// parameter staging
// ===================================================================================================
__global__ void __launch_bounds__(256) pack_kernel(const PackDesc* __restrict__ table) {
    const PackDesc d = table[blockIdx.y];
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= d.n) return;
    if (d.kind == PACK_CONV_FWD || d.kind == PACK_CONV_DGRAD) {
        // destination [Kin/cc][kk][cc/8][Nout][8]; forward: Kin = Cin, Nout = Cout, value = W[n][k][tap];
        // dgrad (the transposed conv): Kin = Cout, Nout = Cin, value = W[k][n][kk-1-tap] (flipped taps)
        const int kk = d.k * d.k;
        const int nout = d.kind == PACK_CONV_FWD ? d.Cout : d.Cin;
        const int cpc = d.cc >> 3;
        const int j = idx & 7;
        int r = idx >> 3;
        const int n = r % nout; r /= nout;
        const int kc = r % cpc; r /= cpc;
        const int tap = r % kk;
        const int c = r / kk;
        const int kch = c * d.cc + kc * 8 + j;
        float v;
        if (d.kind == PACK_CONV_FWD) v = d.src[((size_t)n * d.Cin + kch) * kk + tap];
        else v = d.src[((size_t)kch * d.Cin + n) * kk + (kk - 1 - tap)];
        reinterpret_cast<__nv_bfloat16*>(d.dst)[idx] = __float2bfloat16_rn(v);
    } else if (d.kind == PACK_STEM) {
        // [kh][2][Cout][8]: element (kh, kc, n, j) = W[n][ci = j % 4][kh][kw = 2 kc + j / 4], zero for kw = 3 or ci >= Cin (3, or 1: gray)
        const int j = idx & 7;
        int r = idx >> 3;
        const int n = r % d.Cout; r /= d.Cout;
        const int kc = r & 1;
        const int kh = r >> 1;
        const int ci = j & 3, kw = 2 * kc + (j >> 2);
        const float v = (ci < d.Cin && kw < 3) ? d.src[(((size_t)n * d.Cin + ci) * 3 + kh) * 3 + kw] : 0.f;
        reinterpret_cast<__nv_bfloat16*>(d.dst)[idx] = __float2bfloat16_rn(v);
    } else if (d.kind == PACK_ROUND_F32) {
        reinterpret_cast<float*>(d.dst)[idx] = bf16_round(d.src[idx]);
    } else {  // PACK_SCALE_SHIFT
        const float s = d.src2 ? d.src2[0] : 1.f;
        const float b = d.src ? d.src[idx] : 0.f;
        reinterpret_cast<float*>(d.dst)[idx] = s;
        reinterpret_cast<float*>(d.dst2)[idx] = b * s;
        reinterpret_cast<float*>(d.dst3)[idx] = b;
    }
}

cudaError_t pack_launch(const PackDesc* table, int n_desc, int max_n, cudaStream_t st) {
    if (n_desc <= 0) return cudaSuccess;
    pack_kernel<<<dim3((max_n + 255) / 256, n_desc), 256, 0, st>>>(table);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) unpack_kernel(const UnpackDesc* __restrict__ table) {
    const UnpackDesc d = table[blockIdx.y];
    const int idx = blockIdx.x * 256 + threadIdx.x;   // destination index
    if (idx >= d.n) return;
    if (d.kind == UNPACK_CONV) {
        const int tap = idx % d.kk;
        const int r = idx / d.kk;
        const int ci = r % d.Cin, co = r / d.Cin;
        d.dst[idx] += d.src[((size_t)tap * d.Cin + ci) * d.Cout + co];
    } else {
        d.dst[idx] += d.src[idx];
    }
}

cudaError_t unpack_launch(const UnpackDesc* table, int n_desc, int max_n, cudaStream_t st) {
    if (n_desc <= 0) return cudaSuccess;
    unpack_kernel<<<dim3((max_n + 255) / 256, n_desc), 256, 0, st>>>(table);
    return cudaGetLastError();
}

// ===================================================================================================
// BatchNorm forward (training mode)
// ===================================================================================================
__global__ void __launch_bounds__(256) bn_stats_kernel(const BnStatsParams p) {
    __shared__ float sh[kRedFloats(16)];
    const int cpr = p.C >> 3;
    const size_t total = (size_t)p.M * cpr, stride = (size_t)gridDim.x * 256;
    const uint4* z = reinterpret_cast<const uint4*>(p.z);
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = 0.f;
    // batches of 4 independent 16-byte loads per thread before any arithmetic: the kernel is a pure stream and needs ~64 KB in flight per SM
    auto acc = [&](const uint4 q) {
        float f[8];
        unpack8(q, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) { v[j] += f[j]; v[8 + j] = fmaf(f[j], f[j], v[8 + j]); }
    };
    size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    for (; i + 3 * stride < total; i += 4 * stride) {
        const uint4 q0 = z[i], q1 = z[i + stride], q2 = z[i + 2 * stride], q3 = z[i + 3 * stride];
        acc(q0); acc(q1); acc(q2); acc(q3);
    }
    for (; i < total; i += stride) acc(z[i]);
    block_reduce_groups<16>(v, cpr, sh);
    const float* tot = sh + 8 * cpr * 16;
    for (int t = threadIdx.x; t < cpr * 16; t += 256) {
        const int grp = t >> 4, q = t & 15;
        atomicAdd(p.sums + (size_t)(grp * 8 + (q & 7)) * 2 + (q >> 3), (double)tot[t]);
    }
}

static int elementwise_blocks(size_t chunks, int num_sms) {
    size_t b = (chunks + 256 * 4 - 1) / (256 * 4);
    const size_t cap = (size_t)num_sms * 8;
    if (b > cap) b = cap;
    return b < 1 ? 1 : (int)b;
}
// reductions end with one fp64 atomic per (block, channel, statistic) on a handful of addresses: fewer, longer-running blocks
static int reduce_blocks(size_t chunks, int num_sms) {
    size_t b = (chunks + 256 * 8 - 1) / (256 * 8);
    const size_t cap = (size_t)num_sms * 4;
    if (b > cap) b = cap;
    return b < 1 ? 1 : (int)b;
}
static bool pow2_chunks(int C) { const int cpr = C >> 3; return C % 8 == 0 && cpr >= 1 && cpr <= 32 && (cpr & (cpr - 1)) == 0; }

cudaError_t bn_stats_launch(const BnStatsParams& p, int num_sms, cudaStream_t st) {
    if (!pow2_chunks(p.C)) return cudaErrorInvalidValue;
    bn_stats_kernel<<<reduce_blocks((size_t)p.M * (p.C >> 3), num_sms), 256, 0, st>>>(p);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) bn_apply_kernel(const BnApplyParams p) {
    __shared__ float s_scale[256], s_shift[256];
    for (int c = threadIdx.x; c < p.C; c += 256) {
        float mean, rstd;
        double var;
        if (p.frozen) { mean = p.running_mean[c]; var = (double)p.running_var[c]; rstd = (float)(1.0 / sqrt(var + (double)p.eps)); }
        else mean_rstd_from_sums(p.sums, c, (double)p.M, p.eps, &mean, &rstd, &var);
        const float sc = p.gamma[c] * rstd;
        s_scale[c] = sc;
        s_shift[c] = fmaf(-mean, sc, p.beta[c]);
        if (blockIdx.x == 0 && p.running_mean && p.momentum > 0.f && !p.frozen) {
            const double unbiased = p.M > 1 ? var * (double)p.M / (double)(p.M - 1) : var;
            p.running_mean[c] = (1.f - p.momentum) * p.running_mean[c] + p.momentum * mean;
            p.running_var[c] = (1.f - p.momentum) * p.running_var[c] + p.momentum * (float)unbiased;
        }
    }
    __syncthreads();
    const int cpr = p.C >> 3;
    const size_t total = (size_t)p.M * cpr, stride = (size_t)gridDim.x * 256;
    const int cg = (int)(((size_t)blockIdx.x * 256 + threadIdx.x) % cpr);
    float sc[8], sf[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { sc[j] = s_scale[cg * 8 + j]; sf[j] = s_shift[cg * 8 + j]; }
    const uint4* z = reinterpret_cast<const uint4*>(p.z);
    const uint4* res = reinterpret_cast<const uint4*>(p.res);
    uint4* y = reinterpret_cast<uint4*>(p.y);
    auto apply = [&](size_t i, const uint4 qz, const uint4 qr) {
        float f[8], r[8];
        unpack8(qz, f);
        if (res) unpack8(qr, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float o = fmaf(f[j], sc[j], sf[j]);
            if (res) o += r[j];
            f[j] = p.relu ? fmaxf(o, 0.f) : o;
        }
        y[i] = pack8f(f);
    };
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    for (; i + 3 * stride < total; i += 4 * stride) {      // 4 (8 with a residual) independent loads in flight per thread
        const uint4 z0 = z[i], z1 = z[i + stride], z2 = z[i + 2 * stride], z3 = z[i + 3 * stride];
        uint4 r0 = zero4, r1 = zero4, r2 = zero4, r3 = zero4;
        if (res) { r0 = res[i]; r1 = res[i + stride]; r2 = res[i + 2 * stride]; r3 = res[i + 3 * stride]; }
        apply(i, z0, r0); apply(i + stride, z1, r1); apply(i + 2 * stride, z2, r2); apply(i + 3 * stride, z3, r3);
    }
    for (; i < total; i += stride) apply(i, z[i], res ? res[i] : zero4);
}

cudaError_t bn_apply_launch(const BnApplyParams& p, int num_sms, cudaStream_t st) {
    if (!pow2_chunks(p.C) || p.C > 256) return cudaErrorInvalidValue;
    bn_apply_kernel<<<elementwise_blocks((size_t)p.M * (p.C >> 3), num_sms), 256, 0, st>>>(p);
    return cudaGetLastError();
}

// ===================================================================================================
// BatchNorm / GroupNorm backward
//   g    = dy * [output > 0]                         (ReLU mask; BatchNorm reads the stored output, GroupNorm recomputes it)
//   BN:  dz = gamma * rstd * (g - (S1 + zhat * S2) / M)            S1 = sum g, S2 = sum g * zhat per channel, M = N*H*W
//        dgamma = S2, dbeta = S1, d(residual) = g
//   GN:  dz = rstd * (g * gamma - (T1 + zhat * T2) / Mg)           T1 = sum g*gamma, T2 = sum g*gamma*zhat per (image, group)
//        dgamma = sum g * zhat, dbeta = sum g per channel
// ===================================================================================================
template <bool GN>
__global__ void __launch_bounds__(256) norm_bwd_reduce_kernel(const NormBwdParams p) {
    constexpr int NV = GN ? 18 : 16;
    __shared__ float sh[kRedFloats(NV)];
    __shared__ float s_mean[256], s_rstd[256];
    const int cpr = p.C >> 3;
    const int n = GN ? blockIdx.y : 0;
    const size_t rows = GN ? (size_t)p.H * p.W : (size_t)p.N * p.H * p.W;
    if (GN) {
        if (threadIdx.x < p.groups) mean_rstd_from_sums(p.fsums, n * p.groups + threadIdx.x, (double)rows * 8.0, p.eps, &s_mean[threadIdx.x], &s_rstd[threadIdx.x]);
    } else {
        for (int c = threadIdx.x; c < p.C; c += 256) {
            if (p.frozen) { s_mean[c] = p.running_mean[c]; s_rstd[c] = (float)(1.0 / sqrt((double)p.running_var[c] + (double)p.eps)); }
            else mean_rstd_from_sums(p.fsums, c, (double)rows, p.eps, &s_mean[c], &s_rstd[c]);
        }
    }
    __syncthreads();
    const size_t total = rows * cpr, stride = (size_t)gridDim.x * 256, base = (size_t)n * total;
    const int cg = (int)(((size_t)blockIdx.x * 256 + threadIdx.x) % cpr);
    float mu[8], rs[8], ga[8], be[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        mu[j] = GN ? s_mean[cg] : s_mean[cg * 8 + j];
        rs[j] = GN ? s_rstd[cg] : s_rstd[cg * 8 + j];
        ga[j] = GN ? p.gamma[cg * 8 + j] : 0.f;
        be[j] = GN ? p.beta[cg * 8 + j] : 0.f;
    }
    const uint4* dy = reinterpret_cast<const uint4*>(p.dy) + base;
    const uint4* y = reinterpret_cast<const uint4*>(p.y) + base;
    const uint4* z = reinterpret_cast<const uint4*>(p.z) + base;
    float v[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) v[j] = 0.f;
    const bool need_y = !GN && p.relu;
    auto acc = [&](const uint4 qdy, const uint4 qz, const uint4 qy) {
        float g[8], zf[8], yf[8];
        unpack8(qdy, g);
        unpack8(qz, zf);
        if (need_y) unpack8(qy, yf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float zh = (zf[j] - mu[j]) * rs[j];
            bool on = true;
            if (GN) on = fmaf(zh, ga[j], be[j]) > 0.f;
            else if (p.relu) on = yf[j] > 0.f;
            const float gj = on ? g[j] : 0.f;
            v[j] += gj;                       // dbeta
            v[8 + j] = fmaf(gj, zh, v[8 + j]);   // dgamma
            if (GN) { v[16] = fmaf(gj, ga[j], v[16]); v[17] = fmaf(gj * ga[j], zh, v[17]); }
        }
    };
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    for (; i + stride < total; i += 2 * stride) {      // two rows x three tensors of independent loads in flight per thread
        const uint4 a0 = dy[i], a1 = dy[i + stride], b0 = z[i], b1 = z[i + stride];
        uint4 c0 = zero4, c1 = zero4;
        if (need_y) { c0 = y[i]; c1 = y[i + stride]; }
        acc(a0, b0, c0); acc(a1, b1, c1);
    }
    for (; i < total; i += stride) acc(dy[i], z[i], need_y ? y[i] : zero4);
    block_reduce_groups<NV>(v, cpr, sh);
    const float* tot = sh + 8 * cpr * NV;
    for (int t = threadIdx.x; t < cpr * NV; t += 256) {
        const int grp = t / NV, q = t % NV;
        if (q < 16) atomicAdd(p.bsums + (size_t)(grp * 8 + (q & 7)) * 2 + (q >> 3), (double)tot[t]);
        else atomicAdd(p.bsums + (size_t)p.C * 2 + ((size_t)n * p.groups + grp) * 2 + (q - 16), (double)tot[t]);
    }
}

cudaError_t norm_bwd_reduce_launch(const NormBwdParams& p, int num_sms, cudaStream_t st) {
    if (!pow2_chunks(p.C) || p.C > 256) return cudaErrorInvalidValue;
    if (p.groups) {
        if (p.C != p.groups * 8 || p.groups > 32) return cudaErrorInvalidValue;
        int bx = elementwise_blocks((size_t)p.H * p.W * (p.C >> 3), num_sms);
        const int cap = (4 * num_sms + p.N - 1) / p.N;
        if (bx > cap) bx = cap;
        norm_bwd_reduce_kernel<true><<<dim3(bx, p.N), 256, 0, st>>>(p);
    } else {
        norm_bwd_reduce_kernel<false><<<reduce_blocks((size_t)p.N * p.H * p.W * (p.C >> 3), num_sms), 256, 0, st>>>(p);
    }
    return cudaGetLastError();
}

template <bool GN>
__global__ void __launch_bounds__(256) norm_bwd_apply_kernel(const NormBwdParams p) {
    __shared__ float s_mean[256], s_rstd[256], s_a[256], s_b[256];   // BN: per channel S1 / M, S2 / M; GN: per group T1 / Mg, T2 / Mg
    const int cpr = p.C >> 3;
    const int n = GN ? blockIdx.y : 0;
    const size_t rows = GN ? (size_t)p.H * p.W : (size_t)p.N * p.H * p.W;
    if (GN) {
        if (threadIdx.x < p.groups) {
            const int gi = n * p.groups + threadIdx.x;
            mean_rstd_from_sums(p.fsums, gi, (double)rows * 8.0, p.eps, &s_mean[threadIdx.x], &s_rstd[threadIdx.x]);
            const double* gs = p.bsums + (size_t)p.C * 2 + (size_t)gi * 2;
            s_a[threadIdx.x] = (float)(gs[0] / ((double)rows * 8.0));
            s_b[threadIdx.x] = (float)(gs[1] / ((double)rows * 8.0));
        }
    } else {
        for (int c = threadIdx.x; c < p.C; c += 256) {
            if (p.frozen) {   // constant statistics: dz = gamma * rstd * g
                s_mean[c] = p.running_mean[c]; s_rstd[c] = (float)(1.0 / sqrt((double)p.running_var[c] + (double)p.eps));
                s_a[c] = 0.f; s_b[c] = 0.f;
            } else {
                mean_rstd_from_sums(p.fsums, c, (double)rows, p.eps, &s_mean[c], &s_rstd[c]);
                s_a[c] = (float)(p.bsums[2 * c] / (double)rows);
                s_b[c] = (float)(p.bsums[2 * c + 1] / (double)rows);
            }
        }
    }
    // parameter gradients: one block adds the finished per-channel sums
    if (blockIdx.x == 0 && (!GN || blockIdx.y == 0))
        for (int c = threadIdx.x; c < p.C; c += 256) {
            if (p.dbeta) atomicAdd(p.dbeta + c, (float)p.bsums[2 * c]);
            if (p.dgamma) atomicAdd(p.dgamma + c, (float)p.bsums[2 * c + 1]);
        }
    __syncthreads();
    const size_t total = rows * cpr, stride = (size_t)gridDim.x * 256, base = (size_t)n * total;
    const int cg = (int)(((size_t)blockIdx.x * 256 + threadIdx.x) % cpr);
    float mu[8], rs[8], ga[8], be[8], ca[8], cb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int k = GN ? cg : cg * 8 + j;
        mu[j] = s_mean[k]; rs[j] = s_rstd[k]; ca[j] = s_a[k]; cb[j] = s_b[k];
        ga[j] = p.gamma[cg * 8 + j];
        be[j] = GN ? p.beta[cg * 8 + j] : 0.f;
    }
    const uint4* dy = reinterpret_cast<const uint4*>(p.dy) + base;
    const uint4* y = reinterpret_cast<const uint4*>(p.y) + base;
    const uint4* z = reinterpret_cast<const uint4*>(p.z) + base;
    uint4* dz = reinterpret_cast<uint4*>(p.dz) + base;
    uint4* dres = reinterpret_cast<uint4*>(p.dres) + base;
    uint4* dzu = reinterpret_cast<uint4*>(p.dz_up);
    const int HW = p.H * p.W;
    const bool need_y = !GN && p.relu;
    const bool need_r = p.dres && p.dres_accumulate;
    auto apply = [&](size_t i, const uint4 qdy, const uint4 qz, const uint4 qy, const uint4 qr) {
        float g[8], zf[8], yf[8], o[8];
        unpack8(qdy, g);
        unpack8(qz, zf);
        if (need_y) unpack8(qy, yf);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float zh = (zf[j] - mu[j]) * rs[j];
            bool on = true;
            if (GN) on = fmaf(zh, ga[j], be[j]) > 0.f;
            else if (p.relu) on = yf[j] > 0.f;
            g[j] = on ? g[j] : 0.f;
            if (GN) o[j] = rs[j] * (g[j] * ga[j] - (ca[j] + zh * cb[j]));
            else o[j] = ga[j] * rs[j] * (g[j] - (ca[j] + zh * cb[j]));
        }
        const uint4 ov = pack8f(o);
        dz[i] = ov;
        if (p.dres) {
            if (need_r) {
                float r[8];
                unpack8(qr, r);
#pragma unroll
                for (int j = 0; j < 8; ++j) g[j] += r[j];
            }
            dres[i] = pack8f(g);
        }
        if (p.dz_up) {   // zero-inserted copy (the buffer was cleared by the launcher): pixel (oy, ox) -> (2 oy, 2 ox)
            const size_t row = i / cpr;
            const int nn = (int)(row / HW), rem = (int)(row - (size_t)nn * HW);
            const int oy = rem / p.W, ox = rem - oy * p.W;
            dzu[(((size_t)nn * p.upH + 2 * oy) * p.upW + 2 * ox) * cpr + cg] = ov;
        }
    };
    const uint4 zero4 = make_uint4(0, 0, 0, 0);
    size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    for (; i + stride < total; i += 2 * stride) {      // two rows x up to four tensors of independent loads in flight per thread
        const uint4 a0 = dy[i], a1 = dy[i + stride], b0 = z[i], b1 = z[i + stride];
        uint4 c0 = zero4, c1 = zero4, r0 = zero4, r1 = zero4;
        if (need_y) { c0 = y[i]; c1 = y[i + stride]; }
        if (need_r) { r0 = dres[i]; r1 = dres[i + stride]; }
        apply(i, a0, b0, c0, r0); apply(i + stride, a1, b1, c1, r1);
    }
    for (; i < total; i += stride) apply(i, dy[i], z[i], need_y ? y[i] : zero4, need_r ? dres[i] : zero4);
}

cudaError_t norm_bwd_apply_launch(const NormBwdParams& p, int num_sms, cudaStream_t st) {
    if (!pow2_chunks(p.C) || p.C > 256) return cudaErrorInvalidValue;
    if (p.dz_up) {
        if (p.groups || p.upH < 2 * p.H - 1 || p.upW < 2 * p.W - 1) return cudaErrorInvalidValue;
        cudaError_t e = cudaMemsetAsync(p.dz_up, 0, (size_t)p.N * p.upH * p.upW * p.C * 2, st);
        if (e != cudaSuccess) return e;
    }
    if (p.groups) {
        if (p.C != p.groups * 8 || p.groups > 32) return cudaErrorInvalidValue;
        int bx = elementwise_blocks((size_t)p.H * p.W * (p.C >> 3), num_sms);
        const int cap = (4 * num_sms + p.N - 1) / p.N;
        if (bx > cap) bx = cap;
        norm_bwd_apply_kernel<true><<<dim3(bx, p.N), 256, 0, st>>>(p);
    } else {
        norm_bwd_apply_kernel<false><<<elementwise_blocks((size_t)p.N * p.H * p.W * (p.C >> 3), num_sms), 256, 0, st>>>(p);
    }
    return cudaGetLastError();
}

// ===================================================================================================
// head final backward
//   forward (conv_simt.cu head_final_kernel): t = bf16(relu(gn(raw)));  out_o = scale_o * (W_o . t + b_o)
//   h_o = g_o * scale_o;  dW_o += h_o * t;  db_o += h_o;  dt += h_o * W_o;  dScale += sum over regression rows g_o * (W_o . t + b_o)
// Same thread layout as the forward: 8 threads share a pixel (16 channels each), 4 pixels per thread.
// ===================================================================================================
static constexpr int kHbThreads = 256, kHbPpt = 4, kHbPix = (kHbThreads / 8) * kHbPpt;   // 128 pixels per block iteration

// SMALL: n_out <= 5 (every merged WIDERFACE-style head): the weight-gradient partial sums of a thread stay in registers over all its tiles and
// are flushed once; otherwise (46-class heads) they go through shared-memory atomics per tile.
template <bool SMALL>
__global__ void __launch_bounds__(kHbThreads) head_final_bwd_kernel(const HeadFinalBwdParams p) {
    constexpr int kPpt = SMALL ? 2 : kHbPpt, kPix = (kHbThreads / 8) * kPpt;   // SMALL: fewer pixels per thread, the register room goes to the weight-gradient sums
    extern __shared__ __align__(16) float hb_smem[];
    const int C = p.C, no = p.n_out;
    float* wsm = hb_smem;                       // [no][C]
    float* s_scale = wsm + (size_t)no * C;      // [no]
    float* s_bias = s_scale + no;               // [no]
    float* dWs = s_bias + no;                   // [no][C]
    float* dbs = dWs + (size_t)no * C;          // [no]
    float* dsc = dbs + no;                      // [1]
    float* s_mean = dsc + 1;                    // [32]
    float* s_rstd = s_mean + 32;
    const int n = blockIdx.y;
    for (int i = threadIdx.x; i < no * C; i += kHbThreads) { wsm[i] = p.w[i]; dWs[i] = 0.f; }
    for (int i = threadIdx.x; i < no; i += kHbThreads) {
        s_scale[i] = p.w[(size_t)no * C + i];
        s_bias[i] = p.w[(size_t)no * C + 2 * no + i];
        dbs[i] = 0.f;
    }
    if (threadIdx.x == 0) dsc[0] = 0.f;
    const bool gn = p.groups > 0;      // groups == 0: head without norm layers, `raw` is the already activated tensor
    if (gn && threadIdx.x < p.groups)
        mean_rstd_from_sums(p.stats, n * p.groups + threadIdx.x, (double)p.HW * 8.0, p.eps, &s_mean[threadIdx.x], &s_rstd[threadIdx.x]);
    __syncthreads();
    const int sl = threadIdx.x & 7;
    float ga[16], be[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { ga[j] = gn ? p.gamma[sl * 16 + j] : 1.f; be[j] = gn ? p.beta[sl * 16 + j] : 0.f; }
    const float m0 = gn ? s_mean[2 * sl] : 0.f, r0 = gn ? s_rstd[2 * sl] : 1.f, m1 = gn ? s_mean[2 * sl + 1] : 0.f, r1 = gn ? s_rstd[2 * sl + 1] : 1.f;
    float dscale_acc = 0.f;
    float dwr[SMALL ? 5 : 1][16], dbr[SMALL ? 5 : 1];
#pragma unroll
    for (int o = 0; o < (SMALL ? 5 : 1); ++o) {
        dbr[o] = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) dwr[o][j] = 0.f;
    }
    // SMALL: the activation rows and the upstream gradients of a tile come through a 3-stage cp.async ring (two tiles in flight while one
    // is computed): with ~190 registers per thread only one block fits an SM, so the loads have to be hidden inside the block.
    constexpr int kStages = 3, kStageBytes = kPix * 256 + 5 * kPix * 4;
    const uint32_t ring = (smem_u32(s_rstd + 32) + 15u) & ~15u;
    auto issue = [&](int tile, int stage) {
        if (tile * kPix < p.HW) {
            const uint32_t base = ring + (uint32_t)stage * kStageBytes;
#pragma unroll
            for (int q = 0; q < kPix * 16 / kHbThreads; ++q) {
                const int chunk = threadIdx.x + q * kHbThreads, px = chunk >> 4, part = chunk & 15;
                const int pix = tile * kPix + px;
                const bool ok = pix < p.HW;
                cp_async16(base + px * 256 + part * 16, p.raw + ((size_t)n * p.HW + (ok ? pix : 0)) * C + part * 8, ok);
            }
            for (int idx = threadIdx.x; idx < 5 * kPix; idx += kHbThreads) {
                const int o = idx / kPix, px = idx - o * kPix;
                const int pix = tile * kPix + px;
                const bool ok = o < no && pix < p.HW;
                const size_t pt = (size_t)n * p.P + p.point_off + (ok ? pix : 0);
                const float* src = !ok ? p.w : (o >= p.n_cls ? p.greg + pt * 4 + (o - p.n_cls) : p.gcls + pt * p.cls_stride + o);
                cp_async4(base + kPix * 256 + idx * 4, src, ok);
            }
        }
        cp_async_commit();       // (an empty group past the last tile keeps the group count uniform)
    };
    int t_idx = 0;
    if (SMALL) {
        issue(blockIdx.x, 0);
        issue(blockIdx.x + gridDim.x, 1);
    }
    for (int tile = blockIdx.x; tile * kPix < p.HW; tile += gridDim.x, ++t_idx) {
        const int pix0 = tile * kPix + (threadIdx.x >> 3);
        float a[kPpt][16], dt[kPpt][16];
        uint32_t stage_base = 0;
        if (SMALL) {
            cp_async_wait_group<1>();      // this tile's stage has landed (the next tile's may still be in flight)
            __syncthreads();               // ... for every thread, and everybody is done with the stage about to be refilled
            issue(tile + 2 * gridDim.x, (t_idx + 2) % kStages);
            stage_base = ring + (uint32_t)(t_idx % kStages) * kStageBytes;
        }
        // SMALL: every upstream gradient of the tile is fetched up front, together with the activation rows (ONE memory round trip per tile
        // instead of one per output channel)
        float gpre[SMALL ? 5 : 1][kPpt];
        if (SMALL) {
#pragma unroll
            for (int o = 0; o < 5; ++o)
#pragma unroll
                for (int k = 0; k < kPpt; ++k) {
                    gpre[o][k] = lds32f(stage_base + kPix * 256 + (o * kPix + (threadIdx.x >> 3) + k * (kHbThreads / 8)) * 4);   // zero-filled past the map / n_out
                }
        }
#pragma unroll
        for (int k = 0; k < kPpt; ++k) {
            const int pix = pix0 + k * (kHbThreads / 8);
            uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
            if (SMALL) {
                const uint32_t row = stage_base + ((threadIdx.x >> 3) + k * (kHbThreads / 8)) * 256 + sl * 32;
                q0 = lds128(row); q1 = lds128(row + 16);      // (rows past the map were zero-filled)
            } else if (pix < p.HW) {
                const uint4* src = reinterpret_cast<const uint4*>(p.raw + ((size_t)n * p.HW + pix) * C + sl * 16);
                q0 = src[0]; q1 = src[1];
            }
            float f[16];
            unpack8(q0, f); unpack8(q1, f + 8);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                float yv = (f[j] - (j < 8 ? m0 : m1)) * (j < 8 ? r0 : r1);
                yv = fmaf(yv, ga[j], be[j]);
                a[k][j] = bf16_round(fmaxf(yv, 0.f));
                dt[k][j] = 0.f;
            }
        }
#pragma unroll
        for (int o = 0; o < (SMALL ? 5 : no); ++o) {
            if (SMALL && o >= no) break;
            const bool is_reg = o >= p.n_cls;
            const float sc = s_scale[o];
            float g[kPpt], h[kPpt];
#pragma unroll
            for (int k = 0; k < kPpt; ++k) {
                const int pix = pix0 + k * (kHbThreads / 8);
                float gv = 0.f;
                if (SMALL) gv = gpre[SMALL ? o : 0][k];
                else if (pix < p.HW) {
                    const size_t pt = (size_t)n * p.P + p.point_off + pix;
                    gv = is_reg ? p.greg[pt * 4 + (o - p.n_cls)] : p.gcls[pt * p.cls_stride + o];
                }
                g[k] = gv; h[k] = gv * sc;
            }
            const float4* wr = reinterpret_cast<const float4*>(wsm + (size_t)o * C + sl * 16);
            float hsum = 0.f;
#pragma unroll
            for (int k = 0; k < kPpt; ++k) hsum += h[k];
            float u[kPpt];
#pragma unroll
            for (int k = 0; k < kPpt; ++k) u[k] = 0.f;
#pragma unroll
            for (int v4 = 0; v4 < 4; ++v4) {
                const float4 w4 = wr[v4];
                const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int j = v4 * 4 + e;
                    float dw = 0.f;
#pragma unroll
                    for (int k = 0; k < kPpt; ++k) {
                        dt[k][j] = fmaf(h[k], wv[e], dt[k][j]);
                        dw = fmaf(h[k], a[k][j], dw);
                        if (is_reg) u[k] = fmaf(wv[e], a[k][j], u[k]);
                    }
                    if (SMALL) dwr[SMALL ? o : 0][j] += dw;
                    else {      // the warp's 4 pixel rows first (shuffles), then ONE shared-memory atomic per warp and element (a CAS loop)
                        dw += __shfl_xor_sync(0xffffffffu, dw, 8);
                        dw += __shfl_xor_sync(0xffffffffu, dw, 16);
                        if ((threadIdx.x & 31) < 8 && dw != 0.f) atomicAdd(dWs + (size_t)o * C + sl * 16 + j, dw);
                    }
                }
            }
            if (SMALL) dbr[SMALL ? o : 0] += hsum;
            else {
                hsum += __shfl_xor_sync(0xffffffffu, hsum, 8);
                hsum += __shfl_xor_sync(0xffffffffu, hsum, 16);
                if ((threadIdx.x & 31) == 0 && hsum != 0.f) atomicAdd(dbs + o, hsum);
            }
            if (is_reg) {   // Scale gradient needs the full dot product: combine the 8 channel slices (warp-uniform branch)
#pragma unroll
                for (int k = 0; k < kPpt; ++k) {
                    float v = u[k];
                    v += __shfl_xor_sync(0xffffffffu, v, 1);
                    v += __shfl_xor_sync(0xffffffffu, v, 2);
                    v += __shfl_xor_sync(0xffffffffu, v, 4);
                    if (sl == 0) dscale_acc = fmaf(g[k], v + s_bias[o], dscale_acc);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kPpt; ++k) {
            const int pix = pix0 + k * (kHbThreads / 8);
            if (pix >= p.HW) continue;
            uint4* dst = reinterpret_cast<uint4*>(p.dact + ((size_t)n * p.HW + pix) * C + sl * 16);
            dst[0] = pack8f(dt[k]);
            dst[1] = pack8f(dt[k] + 8);
        }
    }
    if (SMALL) {
        // Block-level reduction of the per-thread weight-gradient sums WITHOUT shared-memory atomics (a float atomicAdd on shared memory is a
        // compare-and-swap loop; with 32 threads per address the old flush cost ~25 us per block, most of the kernel for the small levels):
        // the 4 pixel rows of a warp are combined with two shuffles, the 8 warps through the (now idle) tile ring.
        cp_async_wait_all();
        __syncthreads();
        uint8_t* rb = reinterpret_cast<uint8_t*>(s_rstd + 32);
        rb += (16u - (smem_u32(rb) & 15u)) & 15u;
        float* red = reinterpret_cast<float*>(rb);           // [8 warps][kRedStride]: no * C weight sums, no bias sums, 1 Scale sum
        constexpr int kRedStride = 5 * 128 + 8;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int o = 0; o < 5; ++o) {
            if (o >= no) break;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                float v = dwr[o][j];
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane < 8) red[warp * kRedStride + o * C + sl * 16 + j] = v;
            }
            float b = dbr[o];                                 // identical in the 8 channel-slice lanes of a pixel: take slice 0
            b += __shfl_xor_sync(0xffffffffu, b, 8);
            b += __shfl_xor_sync(0xffffffffu, b, 16);
            if (lane == 0) red[warp * kRedStride + no * C + o] = b;
        }
        float d = dscale_acc;                                 // only the slice-0 lanes carry it
        d += __shfl_xor_sync(0xffffffffu, d, 8);
        d += __shfl_xor_sync(0xffffffffu, d, 16);
        if (lane == 0) red[warp * kRedStride + no * C + no] = d;
        __syncthreads();
        for (int i = threadIdx.x; i < no * C + no + 1; i += kHbThreads) {
            float sum = 0.f;
#pragma unroll
            for (int w = 0; w < kHbThreads / 32; ++w) sum += red[w * kRedStride + i];
            if (sum == 0.f) continue;
            if (i < no * C + no) atomicAdd(p.dstage + i, sum);           // [n_out][C] weights, then [n_out] biases: contiguous in the staging
            else if (p.dscale) atomicAdd(p.dscale, sum);
        }
        return;
    }
    if (dscale_acc != 0.f) atomicAdd(dsc, dscale_acc);
    __syncthreads();
    for (int i = threadIdx.x; i < no * C; i += kHbThreads)
        if (dWs[i] != 0.f) atomicAdd(p.dstage + i, dWs[i]);
    for (int i = threadIdx.x; i < no; i += kHbThreads)
        if (dbs[i] != 0.f) atomicAdd(p.dstage + (size_t)no * C + i, dbs[i]);
    if (threadIdx.x == 0 && p.dscale && dsc[0] != 0.f) atomicAdd(p.dscale, dsc[0]);
}

cudaError_t head_final_bwd_launch(const HeadFinalBwdParams& p, int num_sms, cudaStream_t st) {
    if (p.C != 128 || (p.groups != 16 && p.groups != 0)) return cudaErrorInvalidValue;
    size_t smem = ((size_t)2 * p.n_out * p.C + 3 * p.n_out + 1 + 64) * sizeof(float);
    if (p.n_out <= 5) smem = ((smem + 15) & ~(size_t)15) + 3 * ((kHbThreads / 8) * 2 * 256 + 5 * (kHbThreads / 8) * 2 * 4) + 16;   // + the 3-stage tile ring
    if (smem > 100 * 1024) return cudaErrorInvalidValue;
    static bool attr[kMaxDevices] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return cudaErrorInvalidDevice;
    if (!attr[dev]) {
        cudaError_t e = cudaFuncSetAttribute(head_final_bwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(head_final_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
        if (e != cudaSuccess) return e;
        attr[dev] = true;
    }
    const int pix_per_tile = p.n_out <= 5 ? (kHbThreads / 8) * 2 : kHbPix;
    const int tiles = (p.HW + pix_per_tile - 1) / pix_per_tile;
    int bx = (4 * num_sms + p.N - 1) / p.N;
    if (bx > tiles) bx = tiles;
    if (bx < 1) bx = 1;
    if (p.n_out > 64) return cudaErrorInvalidValue;
    if (p.n_out <= 5) head_final_bwd_kernel<true><<<dim3(bx, p.N), kHbThreads, smem, st>>>(p);
    else head_final_bwd_kernel<false><<<dim3(bx, p.N), kHbThreads, smem, st>>>(p);
    return cudaGetLastError();
}

// ===================================================================================================
// weight gradient of the stem conv (3x3/s2 on the raw image of Cin = 3 or 1 channels): K = 9 Cin, far too narrow for a tensor-core tile.
// dstage[(kh*3+kw)][ci][co] += sum_{n,oy,ox} x(n, ci, 2oy+kh-1, 2ox+kw-1) * dz(n, oy, ox, co), x normalised and rounded to bf16 like
// the forward kernel does (rounding point R0).  Persistent blocks walk 64-pixel output row segments; every thread owns one output
// channel and up to 7 of the 9 Cin (tap, ci) pairs, accumulates in registers and flushes once.
// ===================================================================================================
static constexpr int kWsSeg = 64, kWsCols = 2 * kWsSeg + 1;

__global__ void __launch_bounds__(256) wgrad_stem_kernel(WgradGeom g, const __grid_constant__ ImageIn img, const __nv_bfloat16* __restrict__ dz,
                                                         float* __restrict__ dstage) {
    __shared__ float patch[3][3][kWsCols + 3];   // [ci][kh][column]
    const int Cout = g.Cout;
    const int ngrp = 256 / Cout;                 // (tap, ci) groups
    const int co = threadIdx.x % Cout, grp = threadIdx.x / Cout;
    float acc[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) acc[i] = 0.f;
    const int segs_x = (g.Wo + kWsSeg - 1) / kWsSeg;
    const int n_seg = g.N * g.Ho * segs_x;
    const int K = 9 * g.Cin;
    for (int seg = blockIdx.x; seg < n_seg; seg += gridDim.x) {
        const int sx = seg % segs_x, oy = (seg / segs_x) % g.Ho, n = seg / (segs_x * g.Ho);
        const int ox0 = sx * kWsSeg, ix0 = 2 * ox0 - 1, iy0 = 2 * oy - 1;
        __syncthreads();
        image_dispatch<false>(img, [&](auto ch_c, auto fmt_c) {
            constexpr int CH = decltype(ch_c)::value, FMT = decltype(fmt_c)::value;
            for (int i = threadIdx.x; i < 3 * kWsCols; i += 256) {
                const int c = i % kWsCols, kh = i / kWsCols;
                const int y = iy0 + kh, x = ix0 + c;
                const bool inside = (unsigned)y < (unsigned)g.H && (unsigned)x < (unsigned)g.W;
                uint32_t raw[CH];
                float f[3];
                image_load<CH, FMT>(img, n, image_px<CH, FMT>(img, y, x), y, x, inside, raw);
                image_decode<CH, FMT>(img, raw, inside, f);
#pragma unroll
                for (int ci = 0; ci < CH; ++ci) patch[ci][kh][c] = bf16_round(f[ci]);
            }
        });
        __syncthreads();
        const int npx = min(kWsSeg, g.Wo - ox0);
        const __nv_bfloat16* dzp = dz + (((size_t)n * g.Ho + oy) * g.Wo + ox0) * Cout + co;
        for (int px = 0; px < npx; ++px) {
            const float d = __bfloat162float(dzp[(size_t)px * Cout]);
#pragma unroll
            for (int i = 0; i < 7; ++i) {
                const int q = grp + ngrp * i;   // (kh*3 + kw)*Cin + ci
                if (q < K) {
                    const int ci = g.Cin == 3 ? q % 3 : 0, t = g.Cin == 3 ? q / 3 : q;      // (divisions by a constant)
                    acc[i] = fmaf(d, patch[ci][t / 3][2 * px + t % 3], acc[i]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const int q = grp + ngrp * i;
        if (q < K) atomicAdd(dstage + (size_t)q * Cout + co, acc[i]);
    }
}

cudaError_t wgrad_stem_launch(const WgradGeom& g, const ImageIn& img, const __nv_bfloat16* dz, float* dstage, int num_sms, cudaStream_t st) {
    if ((g.Cin != 3 && g.Cin != 1) || g.ksize != 3 || g.stride != 2 || 256 % g.Cout || g.Cout < 16 || g.Cout > 64) return cudaErrorInvalidValue;
    const int n_seg = g.N * g.Ho * ((g.Wo + kWsSeg - 1) / kWsSeg);
    int blocks = 4 * num_sms;
    if (blocks > n_seg) blocks = n_seg;
    wgrad_stem_kernel<<<blocks, 256, 0, st>>>(g, img, dz, dstage);
    return cudaGetLastError();
}

// im2col of the stem conv for its weight gradient: X27[n][oy][ox][q] with q = (kh*3 + kw)*Cin + ci (q >= 9 Cin: zero; Cin = 3, or 1 for a
// gray image: X9 padded to the same 32 columns) as bf16, the image normalised + rounded like the forward does (R0).  The weight gradient of
// the stem conv is then the weight gradient of a 1x1 conv with 32 input channels over X27, i.e. one launch of the tensor-core wgrad kernel;
// its staging rows [q][co] ARE the [tap][ci][co] layout.  One thread per output pixel: its 9 taps are loaded and decoded once each.
__global__ void __launch_bounds__(256) stem_im2col_kernel(WgradGeom g, const __grid_constant__ ImageIn img, __nv_bfloat16* __restrict__ x27) {
    const size_t total = (size_t)g.N * g.Ho * g.Wo;
    image_dispatch<false>(img, [&](auto ch_c, auto fmt_c) {      // compile-time channel count: every q of a pixel is a fixed register
        constexpr int CH = decltype(ch_c)::value, FMT = decltype(fmt_c)::value;
        for (size_t pix = (size_t)blockIdx.x * 256 + threadIdx.x; pix < total; pix += (size_t)gridDim.x * 256) {
            const int ox = (int)(pix % g.Wo), oy = (int)((pix / g.Wo) % g.Ho), n = (int)(pix / ((size_t)g.Wo * g.Ho));
            float v[32];
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const int y = 2 * oy + t / 3 - 1, x = 2 * ox + t % 3 - 1;
                const bool inside = (unsigned)y < (unsigned)g.H && (unsigned)x < (unsigned)g.W;
                uint32_t raw[CH];
                float f[3];
                image_load<CH, FMT>(img, n, image_px<CH, FMT>(img, y, x), y, x, inside, raw);
                image_decode<CH, FMT>(img, raw, inside, f);
#pragma unroll
                for (int ci = 0; ci < CH; ++ci) v[t * CH + ci] = f[ci];
            }
#pragma unroll
            for (int q = 9 * CH; q < 32; ++q) v[q] = 0.f;
#pragma unroll
            for (int c = 0; c < 4; ++c) reinterpret_cast<uint4*>(x27)[pix * 4 + c] = pack8f(v + 8 * c);
        }
    });
}

cudaError_t stem_im2col_launch(const WgradGeom& g, const ImageIn& img, __nv_bfloat16* x27, int num_sms, cudaStream_t st) {
    if ((g.Cin != 3 && g.Cin != 1) || g.ksize != 3 || g.stride != 2) return cudaErrorInvalidValue;
    const size_t total = (size_t)g.N * g.Ho * g.Wo;
    size_t blocks = (total + 255) / 256;
    if (blocks > (size_t)num_sms * 16) blocks = (size_t)num_sms * 16;
    stem_im2col_kernel<<<(int)blocks, 256, 0, st>>>(g, img, x27);
    return cudaGetLastError();
}

// SIMT cross-check of the tensor-core wgrad: one thread per (tap, ci, co), loop over one image's pixels (grid.y = image)
__global__ void __launch_bounds__(256) wgrad_simt_kernel(WgradGeom g, const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dz,
                                                         float* __restrict__ dstage) {
    const int kk = g.ksize * g.ksize, pad = g.ksize / 2;
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= kk * g.Cin * g.Cout) return;
    const int co = idx % g.Cout, ci = (idx / g.Cout) % g.Cin, tap = idx / (g.Cout * g.Cin);
    const int kh = tap / g.ksize, kw = tap % g.ksize;
    const int n = blockIdx.y;
    float acc = 0.f;
    for (int oy = 0; oy < g.Ho; ++oy) {
        const int iy = oy * g.stride + kh - pad;
        if (iy < 0 || iy >= g.H) continue;
        for (int ox = 0; ox < g.Wo; ++ox) {
            const int ix = ox * g.stride + kw - pad;
            if (ix < 0 || ix >= g.W) continue;
            acc = fmaf(__bfloat162float(x[(((size_t)n * g.H + iy) * g.W + ix) * g.Cin + ci]),
                       __bfloat162float(dz[(((size_t)n * g.Ho + oy) * g.Wo + ox) * g.Cout + co]), acc);
        }
    }
    atomicAdd(dstage + idx, acc);
}

cudaError_t wgrad_simt_launch(const WgradGeom& g, const __nv_bfloat16* x, const __nv_bfloat16* dz, float* dstage, cudaStream_t st) {
    const int total = g.ksize * g.ksize * g.Cin * g.Cout;
    wgrad_simt_kernel<<<dim3((total + 255) / 256, g.N), 256, 0, st>>>(g, x, dz, dstage);
    return cudaGetLastError();
}

// ===================================================================================================
// optimizer
// ===================================================================================================
__global__ void __launch_bounds__(256) sqnorm_kernel(const float* __restrict__ g, long long n, double* out) {
    __shared__ float sh[8];
    float s = 0.f;
    const long long n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
        const float4 v = g4[i];
        s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[(n4 << 2) + threadIdx.x]; s = fmaf(v, v, s); }
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int w = 0; w < 8; ++w) t += (double)sh[w];
        atomicAdd(out, t);
    }
}

cudaError_t sqnorm_launch(const float* g, long long n, double* out, int num_sms, cudaStream_t st) {
    if (((uintptr_t)g & 15) != 0) return cudaErrorInvalidValue;
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 4 * num_sms) blocks = 4 * num_sms;
    if (blocks < 1) blocks = 1;
    sqnorm_kernel<<<(int)blocks, 256, 0, st>>>(g, n, out);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(256) sgd_kernel(const SgdParams p) {
    float coef = p.grad_scale;
    if (p.max_norm > 0.f) {
        const float total = sqrtf((float)(*p.sqnorm)) * fabsf(p.grad_scale);   // norm of the scaled gradients
        const float c = p.max_norm / (total + 1e-6f);
        coef *= c < 1.f ? c : 1.f;
    }
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < p.n; i += (long long)gridDim.x * 256) {
        float g = p.g[i] * coef;
        p.g[i] = g;                                   // clip_grad_norm_ rescales the gradients in place
        const float w = p.p[i];
        g = fmaf(p.weight_decay, w, g);
        if (p.m) {
            const float b = fmaf(p.momentum, p.m[i], (1.f - p.dampening) * g);
            p.m[i] = b;
            g = p.nesterov ? fmaf(p.momentum, b, g) : b;
        }
        p.p[i] = fmaf(-p.lr, g, w);
    }
}

cudaError_t sgd_launch(const SgdParams& p, int num_sms, cudaStream_t st) {
    long long blocks = (p.n + 255) / 256;
    if (blocks > 8 * num_sms) blocks = 8 * num_sms;
    if (blocks < 1) blocks = 1;
    sgd_kernel<<<(int)blocks, 256, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace lfd
