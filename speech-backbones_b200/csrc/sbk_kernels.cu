// sm_90a kernels of the score U-Net step (fp32 CUDA-core path + all fused glue kernels).
//
// Data layout: every activation is NHWC fp32, [B][H][W][C] with H = mel bins (80/40/20),
// W = frames (T, T/2, T/4), C innermost so that one pixel's channels are one contiguous
// 4*C-byte run (coalesced float4 access; K-contiguous operand rows for the implicit GEMM).
// The sampler state xt / mu / z / mask keep the reference's planar [B,80,T] layout.
//
// Stage split (SURVEY.md section 7): every GroupNorm is a grid-wide reduction, so a Block is
// cut at the reduction - the producing conv accumulates per-(sample,group) {sum, sumsq} in its
// epilogue (fp64 atomics of per-CTA fp32 partials), and the consumer applies
// (x-mean)*rstd*gamma+beta -> Mish -> mask (+ time projection) in its operand prologue.
#include "sbk_internal.h"

#include <math.h>
#include <type_traits>

namespace sbk {

// ----------------------------------------------------------------------------------------------
// device helpers
// ----------------------------------------------------------------------------------------------

// Mish, Grad-TTS/model/diffusion.py:16-18: x * tanh(softplus(x)).  With n = e^x,
// tanh(log(1+n)) = n(n+2) / (n(n+2)+2): one exp and one division, no cancellation for x << 0.
// softplus uses torch's threshold 20 (softplus(x) = x beyond it), where tanh is 1 in fp32.
__device__ __forceinline__ float mish_f(float x) {
    float n = expf(fminf(x, 20.f));
    float a = n * (n + 2.f);
    float r = a / (a + 2.f);
    return x > 20.f ? x : x * r;
}

// tensor-core modes: operands are rounded to tf32 anyway, so the activation may use the fast intrinsics
__device__ __forceinline__ float mish_fast_f(float x) {
    const float n = __expf(fminf(x, 20.f));
    const float a = n * (n + 2.f);
    return x > 20.f ? x : x * __fdividef(a, a + 2.f);
}

__device__ __forceinline__ float mish_rt(float x, int exact) { return exact ? mish_f(x) : mish_fast_f(x); }
template <bool EXACT> __device__ __forceinline__ float mish_sel(float x) { return EXACT ? mish_f(x) : mish_fast_f(x); }

__device__ __forceinline__ void gn_mean_rstd(const GnRef& g, int b, int grp, float& mean, float& rstd) {
    const double s = g.stats[(b * kGroups + grp) * 2 + 0];
    const double ss = g.stats[(b * kGroups + grp) * 2 + 1];
    const double m = s * (double)g.inv_count;
    double var = ss * (double)g.inv_count - m * m;
    var = var < 0.0 ? 0.0 : var;
    mean = (float)m;
    rstd = (float)(1.0 / sqrt(var + 1e-5));   // GroupNorm eps, torch default (diffusion.py:53)
}

// fill mean[c], scale[c] = rstd*gamma[c], beta[c] for channels [c_begin, c_begin+n) of a C-channel GN
__device__ __forceinline__ void gn_fill(const GnRef& g, int b, int C, int c_begin, int n,
                                        float* mean, float* scale, float* beta) {
    const int cpg = C / kGroups;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int c = c_begin + i;
        float m, r;
        gn_mean_rstd(g, b, c / cpg, m, r);
        mean[i] = m;
        scale[i] = r * g.gamma[c];
        beta[i] = g.beta[c];
    }
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ----------------------------------------------------------------------------------------------
// implicit-GEMM convolution on CUDA cores (exact fp32)
//   CTA tile 128 pixels x 64 output channels, K chunk = 16 input channels of one filter tap,
//   128 threads, 8x8 register tile per thread, register-prefetch double buffering.
// ----------------------------------------------------------------------------------------------
constexpr int IG_TM = 128, IG_TN = 64, IG_KC = 16, IG_LDA = IG_TM + 4, IG_THREADS = 128;
constexpr int IG_BASE_FLOATS = IG_KC * IG_LDA + IG_KC * IG_TN;

template <int GEOM>
__global__ void __launch_bounds__(IG_THREADS, 3) k_igemm(const IgemmParams p) {
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                       // [KC][LDA]   (k-major, pixel contiguous)
    float* Ws = As + IG_KC * IG_LDA;        // [KC][TN]
    float* ext = Ws + IG_KC * IG_TN;        // prologue / epilogue tables

    const int tid = threadIdx.x;
    const int b = blockIdx.z;
    const int n0 = blockIdx.y * IG_TN;
    const int Cin = p.c0 + p.c1;
    const int Cout = p.Cout;

    int mt = blockIdx.x, phase = 0, HWm;
    if (GEOM == G_UP) {
        const int per = (p.Hin * p.Win + IG_TM - 1) / IG_TM;
        phase = mt / per;
        mt -= phase * per;
        HWm = p.Hin * p.Win;
    } else {
        HWm = p.Hout * p.Wout;
    }
    const int m0 = mt * IG_TM;
    const int ph = phase >> 1, pw = phase & 1;
    const int Wm = (GEOM == G_UP) ? p.Win : p.Wout;   // width of the m index space

    // ---- prologue tables
    float* pg_mean = ext;
    float* pg_scale = pg_mean + Cin;
    float* pg_beta = pg_scale + Cin;
    float* pg_tb = pg_beta + Cin;
    float* ext2 = (p.pro == PRO_GN) ? pg_tb + Cin : ext;
    if (p.pro == PRO_GN) {
        gn_fill(p.pgn, b, Cin, 0, Cin, pg_mean, pg_scale, pg_beta);
        const int row = p.tb_per_sample ? b : *p.step;
        const float* tb = p.tb + (long long)row * p.tb_stride;
        for (int c = tid; c < Cin; c += IG_THREADS) pg_tb[c] = tb[c];
    }
    float* rg_mean = ext2;                  // EPI_RES: [64] x3
    float* rg_scale = rg_mean + IG_TN;
    float* rg_beta = rg_scale + IG_TN;
    if (p.epi == EPI_RES) gn_fill(p.rgn, b, Cout, n0, IG_TN, rg_mean, rg_scale, rg_beta);

    // ---- gather bookkeeping: thread loads pixels (tid>>2)+32*i, channels c4*4..c4*4+3 of the chunk
    const int c4 = tid & 3;
    int g_h[4], g_w[4];
    bool g_ok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + (tid >> 2) + 32 * i;
        g_ok[i] = m < HWm;
        const int mm = g_ok[i] ? m : 0;
        g_h[i] = mm / Wm;
        g_w[i] = mm - g_h[i] * Wm;
    }
    const int w_row = tid >> 4, w_col = (tid & 15) * 4;

    const int cchunks = Cin / IG_KC;
    const int ntaps = (GEOM == G_PW) ? 1 : (GEOM == G_UP ? 4 : 9);
    const int nchunks = ntaps * cchunks;
    const float* wbase = p.w + (long long)b * p.w_bstride;

    float4 ra[4], rw[2];
    float rm[4];

    auto prefetch = [&](int ch) {
        const int tap = ch / cchunks;
        const int cc = (ch - tap * cchunks) * IG_KC;
        int wtap = tap, dh = 0, dw = 0;
        if (GEOM == G_C3 || GEOM == G_DOWN) { dh = tap / 3 - 1; dw = tap % 3 - 1; }
        if (GEOM == G_UP) {
            // ConvTranspose2d(4,2,1): ho = 2*hi - 1 + kh.  For output parity ph the two contributing
            // taps are (kh=1,hi=mh),(kh=3,hi=mh-1) when ph=0 and (kh=0,hi=mh+1),(kh=2,hi=mh) when ph=1.
            const int a = tap >> 1, bb = tap & 1;
            const int kh = ph ? (a ? 2 : 0) : (a ? 3 : 1);
            const int kw = pw ? (bb ? 2 : 0) : (bb ? 3 : 1);
            dh = ph ? (a ? 0 : 1) : (a ? -1 : 0);
            dw = pw ? (bb ? 0 : 1) : (bb ? -1 : 0);
            wtap = kh * 4 + kw;
        }
        const bool second = cc >= p.c0;
        const float* src = second ? p.in1 : p.in0;
        const int cs = second ? p.c1 : p.c0;
        const int co = (second ? cc - p.c0 : cc) + c4 * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int hi, wi;
            if (GEOM == G_DOWN) { hi = 2 * g_h[i] + dh; wi = 2 * g_w[i] + dw; }
            else { hi = g_h[i] + dh; wi = g_w[i] + dw; }
            const bool ok = g_ok[i] && hi >= 0 && hi < p.Hin && wi >= 0 && wi < p.Win;
            if (ok) {
                ra[i] = ldg4(src + ((long long)(b * p.Hin + hi) * p.Win + wi) * cs + co);
                rm[i] = (p.pro != PRO_NONE) ? __ldg(p.mask + (long long)b * p.T + ((long long)wi << p.in_lvl)) : 1.f;
            } else {
                ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                rm[i] = 0.f;
            }
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int row = w_row + 8 * j;
            rw[j] = ldg4(wbase + ((long long)(wtap * Cin + cc + row)) * Cout + n0 + w_col);
        }
    };

    auto stage = [&](int ch) {
        const int cc = (ch % cchunks) * IG_KC + c4 * 4;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float v[4] = {ra[i].x, ra[i].y, ra[i].z, ra[i].w};
            if (p.pro == PRO_MASK) {
#pragma unroll
                for (int q = 0; q < 4; ++q) v[q] *= rm[i];
            } else if (p.pro == PRO_GN) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int c = cc + q;
                    const float y = mish_f((v[q] - pg_mean[c]) * pg_scale[c] + pg_beta[c]) + pg_tb[c];
                    v[q] = rm[i] != 0.f ? y : 0.f;
                }
            }
            const int px = (tid >> 2) + 32 * i;
#pragma unroll
            for (int q = 0; q < 4; ++q) As[(c4 * 4 + q) * IG_LDA + px] = v[q];
        }
#pragma unroll
        for (int j = 0; j < 2; ++j)
            *reinterpret_cast<float4*>(&Ws[(w_row + 8 * j) * IG_TN + w_col]) = rw[j];
    };

    const int ty = tid >> 3, tx = tid & 7;   // pixels ty*8..+7 ; couts tx*4..+3 and 32+tx*4..+3
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    __syncthreads();   // prologue tables visible
    prefetch(0);
    for (int ch = 0; ch < nchunks; ++ch) {
        stage(ch);
        __syncthreads();
        if (ch + 1 < nchunks) prefetch(ch + 1);
#pragma unroll
        for (int k = 0; k < IG_KC; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[k * IG_LDA + ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[k * IG_LDA + ty * 8 + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Ws[k * IG_TN + tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Ws[k * IG_TN + 32 + tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

    // ---- epilogue
    float bia[8];
    {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            bia[j] = p.bias ? p.bias[n0 + tx * 4 + j] : 0.f;
            bia[4 + j] = p.bias ? p.bias[n0 + 32 + tx * 4 + j] : 0.f;
        }
    }

    if (p.epi == EPI_KV) {
        // The N tile holds one head: columns 0..31 = k[d], 32..63 = v[e] (weights packed that way).
        // Compute this tile's softmax partials: m_d = max_px k, Z_d = sum_px exp(k-m_d),
        // S[d][e] = sum_px exp(k[d,px]-m_d) * v[e,px]   (LinearAttention, diffusion.py:95-96).
        float* KVs = ext2;                    // [128][64]
        float* s_m = KVs + IG_TM * IG_TN;     // [32]
        float* s_red = s_m + 32;              // [4][32]
        const int nvalid = min(IG_TM, HWm - m0);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int px = ty * 8 + i;
            *reinterpret_cast<float4*>(&KVs[px * IG_TN + tx * 4]) =
                make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
            *reinterpret_cast<float4*>(&KVs[px * IG_TN + 32 + tx * 4]) =
                make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
        }
        __syncthreads();
        const int d = tid & 31, qr = tid >> 5;     // quarter qr handles pixels qr*32..+31
        float mx = -INFINITY;
        for (int px = qr * 32; px < qr * 32 + 32; ++px)
            if (px < nvalid) mx = fmaxf(mx, KVs[px * IG_TN + d]);
        s_red[qr * 32 + d] = mx;
        __syncthreads();
        if (tid < 32) s_m[tid] = fmaxf(fmaxf(s_red[tid], s_red[32 + tid]), fmaxf(s_red[64 + tid], s_red[96 + tid]));
        __syncthreads();
        const float md = s_m[d];
        float z = 0.f;
        for (int px = qr * 32; px < qr * 32 + 32; ++px) {
            const float e = px < nvalid ? expf(KVs[px * IG_TN + d] - md) : 0.f;
            KVs[px * IG_TN + d] = e;
            z += e;
        }
        s_red[qr * 32 + d] = z;
        __syncthreads();
        float* part = p.kv_part + (((long long)b * gridDim.x + blockIdx.x) * kHeads + blockIdx.y) * kKvPartFloats;
        if (tid < 32) {
            part[tid] = s_m[tid];
            part[32 + tid] = s_red[tid] + s_red[32 + tid] + s_red[64 + tid] + s_red[96 + tid];
        }
        // S: thread owns d = dg*4..+3, e = eg*2..+1
        const int dg = tid & 7, eg = tid >> 3;
        float s[4][2] = {{0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}, {0.f, 0.f}};
        for (int px = 0; px < nvalid; ++px) {
            const float4 pk = *reinterpret_cast<const float4*>(&KVs[px * IG_TN + dg * 4]);
            const float2 vv = *reinterpret_cast<const float2*>(&KVs[px * IG_TN + 32 + eg * 2]);
            s[0][0] = fmaf(pk.x, vv.x, s[0][0]); s[0][1] = fmaf(pk.x, vv.y, s[0][1]);
            s[1][0] = fmaf(pk.y, vv.x, s[1][0]); s[1][1] = fmaf(pk.y, vv.y, s[1][1]);
            s[2][0] = fmaf(pk.z, vv.x, s[2][0]); s[2][1] = fmaf(pk.z, vv.y, s[2][1]);
            s[3][0] = fmaf(pk.w, vv.x, s[3][0]); s[3][1] = fmaf(pk.w, vv.y, s[3][1]);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
            *reinterpret_cast<float2*>(&part[64 + (dg * 4 + q) * 32 + eg * 2]) = make_float2(s[q][0], s[q][1]);
        return;
    }

    const int cpg = Cout / kGroups;
    float st_s[2] = {0.f, 0.f}, st_q[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + ty * 8 + i;
        if (m >= HWm) continue;
        int opix, wo;
        if (GEOM == G_UP) {
            const int mh = m / Wm, mw = m - mh * Wm;
            wo = 2 * mw + pw;
            opix = (2 * mh + ph) * p.Wout + wo;
        } else {
            opix = m;
            wo = m % p.Wout;
        }
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = acc[i][j] + bia[j];
        float* op = p.out + ((long long)b * p.Hout * p.Wout + opix) * Cout + n0;
        if (p.epi == EPI_RES) {
            const float mo = __ldg(p.mask + (long long)b * p.T + ((long long)wo << p.out_lvl));
            if (mo != 0.f) {
                const float* rp = p.rraw + ((long long)b * p.Hout * p.Wout + opix) * Cout + n0;
                const float4 r0 = ldg4(rp + tx * 4), r1 = ldg4(rp + 32 + tx * 4);
                const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int cl = (j < 4) ? tx * 4 + j : 32 + tx * 4 + (j - 4);
                    v[j] += mish_f((rv[j] - rg_mean[cl]) * rg_scale[cl] + rg_beta[cl]);
                }
            }
        } else if (p.ostats) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                st_s[0] += v[j]; st_q[0] = fmaf(v[j], v[j], st_q[0]);
                st_s[1] += v[4 + j]; st_q[1] = fmaf(v[4 + j], v[4 + j], st_q[1]);
            }
        }
        *reinterpret_cast<float4*>(op + tx * 4) = make_float4(v[0], v[1], v[2], v[3]);
        *reinterpret_cast<float4*>(op + 32 + tx * 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
    if (p.epi == EPI_PLAIN && p.ostats) {
        // As is free after the main loop's trailing barrier: use it for the per-CTA group partials
        // (fp64 accumulation: the arrival order of the per-thread fp32 partials then only perturbs the sums at the 1e-16
        //  level, so the fp32 mean / rstd derived from them - and with them the whole sampler - are reproducible run to run)
        double* s_st = reinterpret_cast<double*>(As);   // [8 groups][2]
        if (tid < 16) s_st[tid] = 0.0;
        __syncthreads();
        const int g0 = (n0 + tx * 4) / cpg, g1 = (n0 + 32 + tx * 4) / cpg, gb = n0 / cpg;
        atomicAdd(&s_st[(g0 - gb) * 2 + 0], (double)st_s[0]);
        atomicAdd(&s_st[(g0 - gb) * 2 + 1], (double)st_q[0]);
        atomicAdd(&s_st[(g1 - gb) * 2 + 0], (double)st_s[1]);
        atomicAdd(&s_st[(g1 - gb) * 2 + 1], (double)st_q[1]);
        __syncthreads();
        const int ng = (IG_TN + cpg - 1) / cpg;   // groups this N tile touches (cpg >= 8 -> <= 8)
        if (tid < ng * 2) {
            const int g = gb + (tid >> 1);
            atomicAdd(&p.ostats[((long long)b * kGroups + g) * 2 + (tid & 1)], s_st[tid]);
        }
    }
}

static size_t igemm_smem_bytes(const IgemmParams& p) {
    size_t f = IG_BASE_FLOATS;
    if (p.pro == PRO_GN) f += 4 * (size_t)(p.c0 + p.c1);
    if (p.epi == EPI_RES) f += 3 * IG_TN;
    if (p.epi == EPI_KV) f += IG_TM * IG_TN + 32 + 128;
    return f * sizeof(float);
}

int launch_igemm(const IgemmParams& p, cudaStream_t s) {
    const int mt = igemm_mtiles(p.geom, p.Hout, p.Wout, p.Hin, p.Win);
    dim3 grid(mt, p.Cout / IG_TN, p.B);
    const size_t sm = igemm_smem_bytes(p);
    switch (p.geom) {
        case G_PW:   k_igemm<G_PW><<<grid, IG_THREADS, sm, s>>>(p); break;
        case G_C3:   k_igemm<G_C3><<<grid, IG_THREADS, sm, s>>>(p); break;
        case G_DOWN: k_igemm<G_DOWN><<<grid, IG_THREADS, sm, s>>>(p); break;
        default:     k_igemm<G_UP><<<grid, IG_THREADS, sm, s>>>(p); break;
    }
    return 1;
}

// ----------------------------------------------------------------------------------------------
// first Block conv: planar stack([mu, xt(, s)])*mask -> Conv3x3(cin -> C) + bias, NHWC raw + GN stats
// (GradLogPEstimator2d.forward, diffusion.py:181-186 feeding downs[0][0].block1, :56-58)
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_first_conv(const FirstConvParams p) {
    // CTA = 256 consecutive frames of one mel row x 64 output channels.  The 3-row x 258-frame masked input halo and
    // the 27x64 weights are staged in shared memory.  A thread owns 16 output channels of 4 frames 64 apart: a weight
    // quad is read once for 4 frames (8 FMAs per shared-memory load; the one-frame version was LSU-bound), and for a
    // fixed frame index the lanes of a warp are consecutive frames, so the planar [.][C/4][T][4] stores are 512-byte runs.
    __shared__ __align__(16) float s_w[27 * 64];
    __shared__ float s_in[3][3][258];
    __shared__ float s_b[64];
    __shared__ double s_st[16];     // fp64: order-insensitive accumulation of the warp partials (reproducible GN statistics)
    const int tid = threadIdx.x, b = blockIdx.z, n0 = blockIdx.y * 64;
    const int wtiles = (p.T + 255) / 256;
    const int h = blockIdx.x / wtiles, w0 = (blockIdx.x - h * wtiles) * 256;
    const int K = p.cin * 9;
    const int kreal = p.w_extra ? (p.cin - 1) * 9 : K;       // rows of s_w that come from the shared weight
    for (int i = tid; i < kreal * 64; i += 256) s_w[i] = p.w[(i >> 6) * p.C + n0 + (i & 63)];
    if (p.w_extra) {
        const int row = p.extra_per_sample_row ? 0 : *p.step;
        const float* we = p.w_extra + ((long long)row * p.B + b) * 9 * p.C;
        for (int i = tid; i < 9 * 64; i += 256) s_w[kreal * 64 + i] = we[(i >> 6) * p.C + n0 + (i & 63)];
    }
    if (tid < 64) s_b[tid] = p.bias[n0 + tid];
    if (tid < 16) s_st[tid] = 0.0;
    for (int i = tid; i < p.cin * 3 * 258; i += 256) {
        const int ci = i / 774, rem = i - ci * 774, r = rem / 258, q = rem - r * 258;
        const int hi = h + r - 1, wi = w0 + q - 1;
        float v = 0.f;
        if (hi >= 0 && hi < p.H && wi >= 0 && wi < p.T) {
            const float mk = __ldg(p.mask + (long long)b * p.T + wi);
            const long long idx = ((long long)b * p.H + hi) * p.T + wi;
            const float x = ci == 0 ? __ldg(p.mu + idx) : (ci == 1 ? __ldg(p.xt + idx) : (p.w_extra ? 1.f : __ldg(p.spk_s + b * p.H + hi)));
            v = x * mk;
        }
        s_in[ci][r][q] = v;
    }
    __syncthreads();
    const int pg = tid & 63, cg = tid >> 6;
    float acc[4][16];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[i][j] = s_b[cg * 16 + j];
    for (int ci = 0; ci < p.cin; ++ci) {
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const float* wr = &s_w[(ci * 9 + t) * 64 + cg * 16];
            float4 ww[4];
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4) ww[j4] = *reinterpret_cast<const float4*>(wr + j4 * 4);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float v = s_in[ci][t / 3][pg + 64 * i + t % 3];
#pragma unroll
                for (int j4 = 0; j4 < 4; ++j4) {
                    acc[i][j4 * 4 + 0] = fmaf(v, ww[j4].x, acc[i][j4 * 4 + 0]);
                    acc[i][j4 * 4 + 1] = fmaf(v, ww[j4].y, acc[i][j4 * 4 + 1]);
                    acc[i][j4 * 4 + 2] = fmaf(v, ww[j4].z, acc[i][j4 * 4 + 2]);
                    acc[i][j4 * 4 + 3] = fmaf(v, ww[j4].w, acc[i][j4 * 4 + 3]);
                }
            }
        }
    }
    // GN statistics: each half of the thread's 16 channels lies in one group (8 | C/8)
    const int cpg = p.C / kGroups, gb = n0 / cpg;
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
        float s = 0.f, q = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (w0 + pg + 64 * i < p.T) {
#pragma unroll
                for (int j = 0; j < 8; ++j) { const float v = acc[i][hf * 8 + j]; s += v; q = fmaf(v, v, q); }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
        if ((tid & 31) == 0) {
            const int g = (n0 + cg * 16 + hf * 8) / cpg - gb;
            atomicAdd(&s_st[g * 2], (double)s);
            atomicAdd(&s_st[g * 2 + 1], (double)q);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int w = w0 + pg + 64 * i;
        if (w >= p.T) continue;
        if (p.chw4) {
            float* o = p.out + ((((long long)b * p.H + h) * (p.C / 4) + (n0 + cg * 16) / 4) * p.T + w) * 4;
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4)
                *reinterpret_cast<float4*>(o + (long long)j4 * p.T * 4) = make_float4(acc[i][j4 * 4], acc[i][j4 * 4 + 1], acc[i][j4 * 4 + 2], acc[i][j4 * 4 + 3]);
        } else {
            float* o = p.out + (((long long)b * p.H + h) * p.T + w) * p.C + n0 + cg * 16;
#pragma unroll
            for (int j4 = 0; j4 < 4; ++j4)
                *reinterpret_cast<float4*>(o + j4 * 4) = make_float4(acc[i][j4 * 4], acc[i][j4 * 4 + 1], acc[i][j4 * 4 + 2], acc[i][j4 * 4 + 3]);
        }
    }
    __syncthreads();
    const int ng = (64 + cpg - 1) / cpg;
    if (p.ostats && tid < ng * 2) atomicAdd(&p.ostats[((long long)b * kGroups + gb + (tid >> 1)) * 2 + (tid & 1)], s_st[tid]);
}

int launch_first_conv(const FirstConvParams& p, cudaStream_t s) {
    dim3 grid(((p.T + 255) / 256) * p.H, p.C / 64, p.B);
    k_first_conv<<<grid, 256, 0, s>>>(p);
    return 1;
}

// ----------------------------------------------------------------------------------------------
// ResnetBlock tail for identity / planar-input residuals (ResnetBlock.forward, diffusion.py:77-78):
//   out = Mish(GN(h2raw))*mask + x*mask                      (dim == dim_out)
//   out = Mish(GN(h2raw))*mask + W_res (in*mask) + b_res     (first block, planar cin = 2|3)
// This kernel is the fp32 CUDA-core mode's (NHWC activations, exact Mish); k_resfinal below serves the tensor-core forms.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_resfinal_nhwc(const ResFinalParams p) {
    extern __shared__ __align__(16) float sm[];
    float* mean = sm; float* scale = mean + p.C; float* beta = scale + p.C;
    float* wres = beta + p.C;            // [cin][C] + [C] bias when planar
    const int b = blockIdx.y, tid = threadIdx.x;
    gn_fill(p.gn, b, p.C, 0, p.C, mean, scale, beta);
    if (!p.x) {
        // rows [0, nreal) = shared res_conv weights of the planar channels, row cin = bias (rows in between unused)
        const int nreal = p.r_extra ? p.cin - 1 : p.cin;
        for (int i = tid; i < (p.cin + 1) * p.C; i += 256)
            wres[i] = i < nreal * p.C ? p.wres[i] : (i >= p.cin * p.C ? p.bres[i - p.cin * p.C] : 0.f);
    }
    __syncthreads();
    const int c4n = p.C >> 2;
    const long long n4 = (long long)p.H * p.W * c4n;
    if (p.x) {
        // identity residual: pure streaming (2 reads + 1 write per element); 4 independent units per thread
        constexpr int U = 4;
        for (long long i0 = (long long)blockIdx.x * (256 * U) + tid; i0 < n4; i0 += (long long)gridDim.x * (256 * U)) {
            float4 r[U], xv[U]; float mk[U]; int cc[U]; bool in[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long i = i0 + u * 256;
                in[u] = i < n4;
                int c = 0, w = 0;
                if (in[u]) {
                    const long long pix = i / c4n;
                    c = (int)(i - pix * c4n) * 4;
                    w = (int)(pix % p.W);
                }
                cc[u] = c;
                mk[u] = in[u] ? __ldg(p.mask + (long long)b * p.T + ((long long)w << p.lvl)) : 0.f;
                const bool live = in[u] && mk[u] != 0.f;
                const long long off = ((long long)b * n4 + i) * 4;
                r[u] = live ? ldg4(p.h2raw + off) : make_float4(0.f, 0.f, 0.f, 0.f);
                xv[u] = live ? ldg4(p.x + off) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (!in[u]) continue;
                const int c = cc[u];
                float o[4] = {0.f, 0.f, 0.f, 0.f};
                if (mk[u] != 0.f) {
                    const float rv[4] = {r[u].x, r[u].y, r[u].z, r[u].w};
                    const float xx[4] = {xv[u].x, xv[u].y, xv[u].z, xv[u].w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) o[q] = mish_f((rv[q] - mean[c + q]) * scale[c + q] + beta[c + q]) + xx[q];
                }
                *reinterpret_cast<float4*>(p.out + ((long long)b * n4 + i0 + u * 256) * 4) = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
        return;
    }
    const int nreal = p.r_extra ? p.cin - 1 : p.cin;
    const float* re = p.r_extra ? p.r_extra + ((long long)(p.extra_per_sample_row ? 0 : *p.step) * p.B + b) * p.C : nullptr;
    for (long long i = (long long)blockIdx.x * 256 + tid; i < n4; i += (long long)gridDim.x * 256) {
        // float4 unit i of this sample -> (pixel, channel quad)
        const long long pix = i / c4n;
        const int c = (int)(i - pix * c4n) * 4, w = (int)(pix % p.W), h = (int)(pix / p.W);
        const float mk = __ldg(p.mask + (long long)b * p.T + ((long long)w << p.lvl));
        const long long off = ((long long)b * n4 + i) * 4;
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        if (mk != 0.f) {
            const float4 r = ldg4(p.h2raw + off);
            const float rv[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) o[q] = mish_f((rv[q] - mean[c + q]) * scale[c + q] + beta[c + q]);
        }
        const long long idx = ((long long)b * p.H + h) * p.T + w;
        float in[3];
        in[0] = __ldg(p.mu + idx) * mk;
        in[1] = __ldg(p.xt + idx) * mk;
        in[2] = (p.cin > 2 && !p.r_extra) ? __ldg(p.spk_s + b * p.H + h) * mk : 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float a = wres[p.cin * p.C + c + q];
#pragma unroll
            for (int ci = 0; ci < 3; ++ci)
                if (ci < nreal) a = fmaf(in[ci], wres[ci * p.C + c + q], a);
            if (re) a = fmaf(mk, __ldg(re + c + q), a);
            o[q] += a;
        }
        *reinterpret_cast<float4*>(p.out + off) = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// ----------------------------------------------------------------------------------------------
// Element-wise kernels of the tensor-core forms (enum Form), over planar tensors: the Block activation
//   k_gn_act:    act = mask ? Mish(GN(raw)) + tproj : 0
// (Block.forward output * mask, then ResnetBlock's time projection, then the next Block's input mask: diffusion.py:56-58,76;
//  one read + one write per element, so the conv's A path is a pure copy), and the ResnetBlock tail
//   k_resfinal:  out = mask ? Mish(GN(h2raw)) + x : 0                                   (identity residual)
//                out = (W_res (in*mask) + b_res + (mask ? Mish(GN(h2raw)) : 0)) (*mask)  (first block: planar inputs)
// A CTA owns ONE output channel chunk, whose GN / time / residual parameters live in registers for the whole kernel, and
// walks mel bins 4 at a time; a thread owns frame(s) w, so the mask is read once and every index is 32-bit and
// division-free (a generic flat loop was issue-bound on 64-bit divisions).  In the fp32 forms a chunk is 4 channels and a
// lane owns a frame.  In bf16 a chunk is 8 channels and a LANE PAIR owns a frame: lane half h handles the fp32 raw chunk
// 2*ch+h (the same register footprint as the fp32 forms) and writes its 8-byte half of the 16-byte bf16 chunk, so loads are
// two interleaved 256-byte runs per warp and stores one contiguous 256-byte run.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2_f(float lo, float hi) {
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ float bf16_lo_f(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi_f(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }
__device__ __forceinline__ float4 opnd_f32(float4 v) { return v; }
__device__ __forceinline__ float4 opnd_f32(uint2 v) { return make_float4(bf16_lo_f(v.x), bf16_hi_f(v.x), bf16_lo_f(v.y), bf16_hi_f(v.y)); }
__device__ __forceinline__ float rna_tf32(float x) {
    uint32_t t;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(x));
    return __uint_as_float(t);
}

enum Tail { TAIL_ACT, TAIL_ID, TAIL_PLANAR };
__host__ __device__ constexpr int lanes_per_frame(int form) { return form == FORM_BF16 ? 2 : 1; }

// grid.x = (channel chunks) x (mel-bin groups); a 256-thread CTA covers min(W, F) frames x F / min(W, F) bin sub-groups
// (F = 256 / lanes per frame), each walking 4 bins per pass, ~2 passes per thread
static int planar_ew_grid(int form, int H, int W, int C) {
    const int lanes = lanes_per_frame(form), F = 256 / lanes;
    const int nsub = W >= F ? 1 : F / W;
    int nhg = (H + 8 * nsub - 1) / (8 * nsub);
    if (nhg < 1) nhg = 1;
    return C / (4 * lanes) * nhg;
}

template <int FORM, int TAIL, class P>
__device__ __forceinline__ void planar_ew(const P& p, const float* raw) {
    constexpr bool B16 = FORM == FORM_BF16, X3 = FORM == FORM_X3;
    constexpr int LPF = lanes_per_frame(FORM), F = 256 / LPF;
    constexpr int U = 4;                         // independent 16-byte loads in flight per thread
    using Unit = typename std::conditional<B16, uint2, float4>::type;   // a thread's 4 channels of an operand tensor
    extern __shared__ __align__(16) float sm[];
    float* mean = sm; float* scale = mean + p.C; float* beta = scale + p.C;
    float* ext = beta + p.C;                     // TAIL_ACT: time projection [C]; TAIL_PLANAR: res_conv [cin][C] + bias [C]
    const int b = blockIdx.y, tid = threadIdx.x;
    gn_fill(p.gn, b, p.C, 0, p.C, mean, scale, beta);
    if constexpr (TAIL == TAIL_ACT) {
        const int row = p.tb_per_sample ? b : *p.step;
        const float* tb = p.tb + (long long)row * p.tb_stride;
        for (int c = tid; c < p.C; c += 256) ext[c] = tb[c];
    } else if constexpr (TAIL == TAIL_PLANAR) {
        // rows [0, nreal) = shared res_conv weights of the planar channels, row cin = bias (rows in between unused)
        const int nreal = p.r_extra ? p.cin - 1 : p.cin;
        for (int i = tid; i < (p.cin + 1) * p.C; i += 256)
            ext[i] = i < nreal * p.C ? p.wres[i] : (i >= p.cin * p.C ? p.bres[i - p.cin * p.C] : 0.f);
    }
    __syncthreads();
    const int c4n = p.C >> 2, ncc = p.C >> (1 + LPF);                  // fp32 chunks, output chunks
    const int ch = blockIdx.x % ncc, hg = blockIdx.x / ncc, nhg = gridDim.x / ncc;
    const int half = tid & (LPF - 1), q = tid >> (LPF - 1);
    const int tw = p.W >= F ? F : p.W, nsub = F / tw, sub = q / tw, wl = q - sub * tw;
    if (sub >= nsub) return;
    const int c4 = LPF * ch + half;                                      // this thread's fp32 chunk
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 pm = reinterpret_cast<const float4*>(mean)[c4], ps = reinterpret_cast<const float4*>(scale)[c4];
    const float4 pb = reinterpret_cast<const float4*>(beta)[c4];
    const float* rawb = raw + ((long long)b * p.H * c4n + c4) * p.W * 4;
    const int hs4 = c4n * p.W * 4;                                       // floats between mel bins (raw)
    // out and the identity residual x, in Units: mel bins are c4n * W Units apart in every form, frames LPF Units
    const long long obase = B16 ? ((long long)b * p.H * ncc + ch) * p.W * 2 + half : ((long long)b * p.H * c4n + c4) * p.W;
    const int ohs = c4n * p.W;
    float4 pt = z4, rx = z4;
    bool has_spk = false;
    if constexpr (TAIL == TAIL_ACT) pt = reinterpret_cast<const float4*>(ext)[c4];
    if constexpr (TAIL == TAIL_PLANAR) {
        // first ResnetBlock: res_conv over the 2-3 planar network inputs (+ DiffVC's folded conditioning channel)
        if (p.r_extra) rx = ldg4(p.r_extra + ((long long)(p.extra_per_sample_row ? 0 : *p.step) * p.B + b) * p.C + c4 * 4);
        has_spk = p.cin > 2 && !p.r_extra;      // = a third real weight row
    }
    // this chunk's res_conv bias and weight rows: bf16, whose launch bounds leave room, holds them in registers; the fp32
    // forms re-read them from shared memory per element (broadcast loads), which keeps them under the registers of the
    // fp32 kernels this walk replaced
    float4 wb = z4, w0 = z4, w1 = z4, w2 = z4;
    auto res_w = [&](const auto& q) {             // q = p (generic, so that only TAIL_PLANAR instantiates it)
        wb = reinterpret_cast<const float4*>(ext + q.cin * q.C)[c4];
        w0 = reinterpret_cast<const float4*>(ext)[c4];
        w1 = reinterpret_cast<const float4*>(ext + q.C)[c4];
        w2 = has_spk ? reinterpret_cast<const float4*>(ext + 2 * q.C)[c4] : z4;
    };
    if constexpr (TAIL == TAIL_PLANAR && B16) res_w(p);
    for (int w = wl; w < p.W; w += tw) {
        const float mk = __ldg(p.mask + (long long)b * p.T + ((long long)w << p.lvl));
        for (int h0 = (hg * nsub + sub) * U; h0 < p.H; h0 += nhg * nsub * U) {
            float4 r[U]; Unit xv[U]; float i0[U], i1[U], i2[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const bool live = mk != 0.f && h0 + u < p.H;
                r[u] = live ? ldg4(rawb + (long long)(h0 + u) * hs4 + w * 4) : z4;
                if constexpr (TAIL == TAIL_ID)
                    xv[u] = live ? __ldg(reinterpret_cast<const Unit*>(p.x) + obase + (long long)(h0 + u) * ohs + w * LPF) : Unit{};
                if constexpr (TAIL == TAIL_PLANAR) {
                    const long long idx = ((long long)b * p.H + h0 + u) * p.T + w;
                    i0[u] = live ? __ldg(p.mu + idx) * mk : 0.f;
                    i1[u] = live ? __ldg(p.xt + idx) * mk : 0.f;
                    i2[u] = (live && has_spk) ? __ldg(p.spk_s + b * p.H + h0 + u) * mk : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (h0 + u >= p.H) continue;
                float4 o = z4;
                if constexpr (TAIL == TAIL_PLANAR) {
                    if constexpr (!B16) res_w(p);
                    o.x = fmaf(mk, rx.x, fmaf(i2[u], w2.x, fmaf(i1[u], w1.x, fmaf(i0[u], w0.x, wb.x))));
                    o.y = fmaf(mk, rx.y, fmaf(i2[u], w2.y, fmaf(i1[u], w1.y, fmaf(i0[u], w0.y, wb.y))));
                    o.z = fmaf(mk, rx.z, fmaf(i2[u], w2.z, fmaf(i1[u], w1.z, fmaf(i0[u], w0.z, wb.z))));
                    o.w = fmaf(mk, rx.w, fmaf(i2[u], w2.w, fmaf(i1[u], w1.w, fmaf(i0[u], w0.w, wb.w))));
                    if (mk != 0.f) {
                        o.x += mish_sel<X3>((r[u].x - pm.x) * ps.x + pb.x);
                        o.y += mish_sel<X3>((r[u].y - pm.y) * ps.y + pb.y);
                        o.z += mish_sel<X3>((r[u].z - pm.z) * ps.z + pb.z);
                        o.w += mish_sel<X3>((r[u].w - pm.w) * ps.w + pb.w);
                    }
                    if (p.out_mask) { o.x *= mk; o.y *= mk; o.z *= mk; o.w *= mk; }
                } else if (mk != 0.f) {
                    float4 a;
                    if constexpr (TAIL == TAIL_ACT) a = pt; else a = opnd_f32(xv[u]);
                    o.x = mish_sel<X3>((r[u].x - pm.x) * ps.x + pb.x) + a.x;
                    o.y = mish_sel<X3>((r[u].y - pm.y) * ps.y + pb.y) + a.y;
                    o.z = mish_sel<X3>((r[u].z - pm.z) * ps.z + pb.z) + a.z;
                    o.w = mish_sel<X3>((r[u].w - pm.w) * ps.w + pb.w) + a.w;
                    if constexpr (FORM == FORM_TF32 && TAIL == TAIL_ACT) o = make_float4(rna_tf32(o.x), rna_tf32(o.y), rna_tf32(o.z), rna_tf32(o.w));
                }
                const long long oi = obase + (long long)(h0 + u) * ohs + w * LPF;
                if constexpr (B16) {
                    reinterpret_cast<uint2*>(p.out)[oi] = make_uint2(pack_bf16x2_f(o.x, o.y), pack_bf16x2_f(o.z, o.w));
                } else {
                    reinterpret_cast<float4*>(p.out)[oi] = o;
                }
            }
        }
    }
}

template <int FORM>
__global__ void __launch_bounds__(256) k_gn_act(const GnActParams p) { planar_ew<FORM, TAIL_ACT>(p, p.raw); }

// the bf16 identity tail keeps to 64 registers for 4 CTAs per SM; its planar-input tail needs more and runs 2 (0: no minimum)
template <int FORM, bool PLANAR>
__global__ void __launch_bounds__(256, FORM == FORM_BF16 ? (PLANAR ? 2 : 4) : 0) k_resfinal(const ResFinalParams p) {
    planar_ew<FORM, PLANAR ? TAIL_PLANAR : TAIL_ID>(p, p.h2raw);
}

int launch_gn_act(const GnActParams& p, cudaStream_t s) {
    const dim3 grid(planar_ew_grid(p.form, p.H, p.W, p.C), p.B);
    const size_t sm = 4 * p.C * sizeof(float);
    switch (p.form) {
        case FORM_TF32: k_gn_act<FORM_TF32><<<grid, 256, sm, s>>>(p); return 1;
        case FORM_X3:   k_gn_act<FORM_X3><<<grid, 256, sm, s>>>(p); return 1;
        case FORM_BF16: k_gn_act<FORM_BF16><<<grid, 256, sm, s>>>(p); return 1;
    }
    return -1;
}

template <int FORM>
static void launch_resfinal_planar(const ResFinalParams& p, size_t sm, cudaStream_t s) {
    const dim3 grid(planar_ew_grid(FORM, p.H, p.W, p.C), p.B);
    if (p.x) k_resfinal<FORM, false><<<grid, 256, sm, s>>>(p);
    else k_resfinal<FORM, true><<<grid, 256, sm, s>>>(p);
}

int launch_resfinal(const ResFinalParams& p, cudaStream_t s) {
    const size_t sm = (3 * p.C + (p.x ? 0 : (p.cin + 1) * p.C)) * sizeof(float);
    switch (p.form) {
        case FORM_NHWC: {
            const long long n4 = (long long)p.H * p.W * (p.C / 4);
            int gx = p.x ? (int)((n4 + 256 * 4 * 8 - 1) / (256 * 4 * 8)) : (int)((n4 + 256 * 4 - 1) / (256 * 4));
            if (gx < 1) gx = 1;
            if (gx > 4096) gx = 4096;
            k_resfinal_nhwc<<<dim3(gx, p.B), 256, sm, s>>>(p);
            return 1;
        }
        case FORM_TF32: launch_resfinal_planar<FORM_TF32>(p, sm, s); return 1;
        case FORM_X3:   launch_resfinal_planar<FORM_X3>(p, sm, s); return 1;
        case FORM_BF16: launch_resfinal_planar<FORM_BF16>(p, sm, s); return 1;
    }
    return -1;
}

// ----------------------------------------------------------------------------------------------
// LinearAttention: merge per-tile partials into the normalised context (diffusion.py:95-96)
// ----------------------------------------------------------------------------------------------
// One CTA per (head, sample), 1024 threads: the tile loop is split four ways (and the max pass 32 ways) so that the
// ~1.4 MB of partials a level-0 sample carries is read with enough loads in flight; partial sums meet in shared memory.
__global__ void __launch_bounds__(1024) k_attn_ctx(const AttnCtxParams p) {
    __shared__ float s_red[32 * 33];
    __shared__ float s_M[32];
    __shared__ __align__(16) float s_acc[3][256][5];
    const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const float* base = p.kv_part + ((long long)b * p.mtiles * kHeads + h) * kKvPartFloats;
    const long long tstride = (long long)kHeads * kKvPartFloats;
    {
        const int w = tid >> 5, lane = tid & 31;
        float mx = -INFINITY;
        for (int i = w; i < p.mtiles; i += 32) mx = fmaxf(mx, base[i * tstride + lane]);
        s_red[w * 33 + lane] = mx;
    }
    __syncthreads();
    if (tid < 32) {
        float mx = s_red[tid];
        for (int w = 1; w < 32; ++w) mx = fmaxf(mx, s_red[w * 33 + tid]);
        s_M[tid] = mx;
    }
    __syncthreads();
    const int sub = tid >> 8, u = tid & 255;
    const int d = u >> 3, e0 = (u & 7) * 4;
    const float M = s_M[d];
    float z = 0.f, a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 2
    for (int i = sub; i < p.mtiles; i += 4) {
        const float* pt = base + i * tstride;
        const float f = expf(pt[d] - M);
        z = fmaf(f, pt[32 + d], z);
        const float4 sv = *reinterpret_cast<const float4*>(pt + 64 + d * 32 + e0);
        a0 = fmaf(f, sv.x, a0); a1 = fmaf(f, sv.y, a1); a2 = fmaf(f, sv.z, a2); a3 = fmaf(f, sv.w, a3);
    }
    if (sub > 0) { float* q = s_acc[sub - 1][u]; q[0] = z; q[1] = a0; q[2] = a1; q[3] = a2; q[4] = a3; }
    __syncthreads();
    if (sub == 0) {
#pragma unroll
        for (int j = 0; j < 3; ++j) { const float* q = s_acc[j][u]; z += q[0]; a0 += q[1]; a1 += q[2]; a2 += q[3]; a3 += q[4]; }
        const float inv = 1.f / z;
        float* o = p.ctx + (((long long)b * kHeads + h) * 32 + d) * 32 + e0;
        *reinterpret_cast<float4*>(o) = make_float4(a0 * inv, a1 * inv, a2 * inv, a3 * inv);
    }
}

int launch_attn_ctx(const AttnCtxParams& p, cudaStream_t s) {
    k_attn_ctx<<<dim3(kHeads, p.B), 1024, 0, s>>>(p);
    return 1;
}


// out = to_out(context^T q) is linear in q = Wq x, so for each sample the whole second half of
// LinearAttention + Rezero + Residual (diffusion.py:45-46,97-100,108-110) collapses to a per-sample
// 1x1 conv:  x + g*(Wout blockdiag(ctx_h^T) Wq x + bout) = (I + g P_b) x + g bout.
// This kernel builds (I + g P_b) in the implicit-GEMM weight layout [ci][co].
__global__ void __launch_bounds__(256) k_attn_mix(const AttnMixParams p) {
    // 48 KB static: Mb transposed [j = h*32+d][cl] (16 KB) + a 32 KB union: the contexts in phase 1, a 128 x 64 tile of Wq
    // in phase 2 (Wq used to be read from global inside the j loop: 128 dependent L2 round trips per 64 input channels made
    // this tiny kernel 80 us at C = 256)
    __shared__ __align__(16) float s_mb[128 * 32];
    __shared__ __align__(16) float s_u[128 * 64];
    float* s_ctx = s_u;                                 // [kHeads*32][33]
    float* s_wq = s_u;                                  // [128][64]
    const int cb = blockIdx.x * 32, b = blockIdx.y, tid = threadIdx.x, C = p.C;
    for (int i = tid; i < kHeads * 32 * 32; i += 256)
        s_ctx[(i >> 5) * 33 + (i & 31)] = p.ctx[(long long)b * kHeads * 1024 + i];
    __syncthreads();
    {   // Mb[cl][h*32+d] = sum_e wout[c][h*32+e] * ctx[h][d][e]; stored j-major so the next phase reads float4 rows
        const int j = tid & 127, hh = j >> 5, cl0 = (tid >> 7) * 16;
        float cr[32];
#pragma unroll
        for (int e = 0; e < 32; ++e) cr[e] = s_ctx[j * 33 + e];
        for (int cl = cl0; cl < cl0 + 16; ++cl) {
            const float4* wo4 = reinterpret_cast<const float4*>(p.wout + (long long)(cb + cl) * kAttnHidden + hh * 32);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
            for (int e4 = 0; e4 < 8; ++e4) {
                const float4 w = __ldg(wo4 + e4);
                a0 = fmaf(w.x, cr[4 * e4 + 0], a0); a1 = fmaf(w.y, cr[4 * e4 + 1], a1);
                a2 = fmaf(w.z, cr[4 * e4 + 2], a2); a3 = fmaf(w.w, cr[4 * e4 + 3], a3);
            }
            s_mb[j * 32 + cl] = (a0 + a1) + (a2 + a3);
        }
    }
    const float g = __ldg(p.g);
    // P[cl][c'] = sum_j Mb[cl][j] * Wq[j][c']: thread = (input channel c' within a block of 64, group of 8 output rows)
    const int cq = tid >> 6, cl0 = cq * 8, cpl = tid & 63;
    for (int cp0 = 0; cp0 < C; cp0 += 64) {
        __syncthreads();                                // phase 1 readers of s_ctx / previous block's readers of s_wq are done
#pragma unroll
        for (int i = 0; i < 8; ++i) {                   // 128 rows x 16 float4, coalesced 256-byte rows
            const int idx = tid + i * 256, row = idx >> 4, c4 = idx & 15;
            *reinterpret_cast<float4*>(&s_wq[row * 64 + c4 * 4]) = ldg4(p.wq + (long long)row * C + cp0 + c4 * 4);
        }
        __syncthreads();
        const int cp = cp0 + cpl;
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
#pragma unroll 8
        for (int j = 0; j < kAttnHidden; ++j) {
            const float wq = s_wq[j * 64 + cpl];
            const float4 m0 = *reinterpret_cast<const float4*>(&s_mb[j * 32 + cl0]);
            const float4 m1 = *reinterpret_cast<const float4*>(&s_mb[j * 32 + cl0 + 4]);
            acc[0] = fmaf(m0.x, wq, acc[0]); acc[1] = fmaf(m0.y, wq, acc[1]); acc[2] = fmaf(m0.z, wq, acc[2]); acc[3] = fmaf(m0.w, wq, acc[3]);
            acc[4] = fmaf(m1.x, wq, acc[4]); acc[5] = fmaf(m1.y, wq, acc[5]); acc[6] = fmaf(m1.z, wq, acc[6]); acc[7] = fmaf(m1.w, wq, acc[7]);
        }
        if (p.nt) {
            // g*P only (see AttnMixParams), this sample's image of the 1x1 conv's weights (sbk_internal.h: conv_tc_wimg)
            const ConvTcWImg wi = conv_tc_wimg(G_PW, p.form, p.nt, C);
            const int epc = form_epc(p.form), cps = wi.kch * epc;
            const int ks = cp / cps, kc = (cp % cps) / epc, e = cp % epc;
            uint8_t* wb = reinterpret_cast<uint8_t*>(p.w_eff) + (long long)b * conv_tc_wimg_bytes(wi, C);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int co = cb + cl0 + i;
                float v = g * acc[i];
                const long long idx = conv_tc_wimg_index(wi, co, ks, 0, kc, e);
                if (p.form == FORM_X3) {
                    // tf32 (RNA) main image and the correction chunk {w[c0..c3], w_lo[c0..c3] * 2^12} of the f16 MMA
                    // (sbk_internal.h: corr_chunk)
                    uint32_t uh;
                    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(uh) : "f"(v));
                    reinterpret_cast<float*>(wb)[idx] = __uint_as_float(uh);
                    unsigned short* cb16 = reinterpret_cast<unsigned short*>(wb) + 2 * conv_tc_wimg_index(wi, co, ks, 0, kc, 0, 1);
                    cb16[e] = (unsigned short)(f16x2_sat(v, 0.f) & 0xFFFFu);
                    cb16[4 + e] = (unsigned short)(f16x2_sat((v - __uint_as_float(uh)) * kCorrUp, 0.f) & 0xFFFFu);
                } else if (p.form == FORM_BF16) {
                    reinterpret_cast<unsigned short*>(wb)[idx] = (unsigned short)(pack_bf16x2_f(v, 0.f) & 0xFFFFu);
                } else {
                    uint32_t u; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
                    reinterpret_cast<float*>(wb)[idx] = __uint_as_float(u);
                }
            }
        } else {
            float* o = p.w_eff + ((long long)b * C + cp) * C + cb + cl0;
#pragma unroll
            for (int i = 0; i < 8; i += 4) {
                float4 v = make_float4(g * acc[i], g * acc[i + 1], g * acc[i + 2], g * acc[i + 3]);
                if (cb + cl0 + i + 0 == cp) v.x += 1.f;
                if (cb + cl0 + i + 1 == cp) v.y += 1.f;
                if (cb + cl0 + i + 2 == cp) v.z += 1.f;
                if (cb + cl0 + i + 3 == cp) v.w += 1.f;
                *reinterpret_cast<float4*>(o + i) = v;
            }
        }
    }
    if (b == 0 && tid < 32) p.b_eff[cb + tid] = g * p.bout[cb + tid];
}

int launch_attn_mix(const AttnMixParams& p, cudaStream_t s) {
    k_attn_mix<<<dim3(p.C / 32, p.B), 256, 0, s>>>(p);
    return 1;
}

// ----------------------------------------------------------------------------------------------
// final_block tail + final_conv + Euler(-Maruyama) update (diffusion.py:213-216,264-274)
//   est  = mask ? (sum_c wfin[c]*Mish(GN(raw))[c] + bfin) : 0
//   mode 1: xt' = (xt - (0.5*(mu - xt - est))*beta*h) * mask
//   mode 2: xt' = (xt - ((0.5*(mu - xt) - est)*beta*h + eps*sqrt(beta*h))) * mask
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_final(const FinalParams p) {
    extern __shared__ __align__(16) float sm[];
    float* mean = sm; float* scale = mean + p.C; float* beta = scale + p.C; float* wf = beta + p.C;
    const int b = blockIdx.y, tid = threadIdx.x;
    gn_fill(p.gn, b, p.C, 0, p.C, mean, scale, beta);
    for (int i = tid; i < p.C; i += 256) wf[i] = p.wfin[i];
    __syncthreads();
    const int HW = p.H * p.T;
    const int lane16 = tid & 15, pl = tid >> 4;
    const float bf = __ldg(p.bfin);
    float4 cf = make_float4(0.f, 0.f, 0.f, 0.f);
    int srow = 0;
    if (p.mode != 0) { srow = *p.step; cf = p.coef[srow]; }
    auto update = [&](long long idx, float mk, float dot) {
        const float est = mk != 0.f ? dot + bf : 0.f;
        if (p.mode == 0) {
            p.xt_out[idx] = est;
        } else {
            const float xt = p.xt_in[idx], mu = __ldg(p.mu + idx);
            float dxt;
            if (p.mode == 1) {
                dxt = ((0.5f * ((mu - xt) - est)) * cf.x) * cf.y;
            } else if (p.mode == 3) {
                // DiffVC pf / em / ml (DiffVC/model/diffusion.py:177-194): coef = {A, Bc, sigma}
                dxt = (mu - xt) * cf.x - est * cf.y;
                if (cf.z != 0.f) dxt += __ldg(*p.noise_pp + (long long)srow * p.B * HW + idx) * cf.z;
            } else {
                const float eps = __ldg(*p.noise_pp + (long long)srow * p.B * HW + idx);
                dxt = ((0.5f * (mu - xt) - est) * cf.x) * cf.y + eps * cf.z;
            }
            p.xt_out[idx] = (xt - dxt) * mk;
        }
    };
    if (p.chw4) {
        // [B][H][C/4][T][4]: one thread per frame; per channel chunk a warp reads 32 frames x 16 B = 512 contiguous bytes
        const int c4n = p.C / 4;
        for (int m = blockIdx.x * 256 + tid; m < HW; m += gridDim.x * 256) {
            const int h = m / p.T, w = m - h * p.T;
            const float mk = __ldg(p.mask + (long long)b * p.T + w);
            float dot = 0.f;
            if (mk != 0.f) {
                const float* rp = p.raw + ((((long long)b * p.H + h) * c4n) * p.T + w) * 4;
#pragma unroll 4
                for (int ch = 0; ch < c4n; ++ch) {
                    const float4 r = ldg4(rp + (long long)ch * p.T * 4);
                    const int c = ch * 4;
                    dot = fmaf(wf[c + 0], mish_rt((r.x - mean[c + 0]) * scale[c + 0] + beta[c + 0], p.exact), dot);
                    dot = fmaf(wf[c + 1], mish_rt((r.y - mean[c + 1]) * scale[c + 1] + beta[c + 1], p.exact), dot);
                    dot = fmaf(wf[c + 2], mish_rt((r.z - mean[c + 2]) * scale[c + 2] + beta[c + 2], p.exact), dot);
                    dot = fmaf(wf[c + 3], mish_rt((r.w - mean[c + 3]) * scale[c + 3] + beta[c + 3], p.exact), dot);
                }
            }
            update((long long)b * HW + m, mk, dot);
        }
        return;
    }
    for (int base = blockIdx.x * 128; base < HW; base += gridDim.x * 128) {
#pragma unroll
        for (int it = 0; it < 8; ++it) {
            const int m = base + it * 16 + pl;
            const bool inb = m < HW;        // shuffles below run for the full warp regardless
            const int w = inb ? m % p.T : 0;
            const float mk = inb ? __ldg(p.mask + (long long)b * p.T + w) : 0.f;
            float dot = 0.f;
            if (mk != 0.f) {
                const float* rp = p.raw + ((long long)b * HW + m) * p.C;
                for (int c = lane16 * 4; c < p.C; c += 64) {
                    const float4 r = ldg4(rp + c);
                    dot = fmaf(wf[c + 0], mish_f((r.x - mean[c + 0]) * scale[c + 0] + beta[c + 0]), dot);
                    dot = fmaf(wf[c + 1], mish_f((r.y - mean[c + 1]) * scale[c + 1] + beta[c + 1]), dot);
                    dot = fmaf(wf[c + 2], mish_f((r.z - mean[c + 2]) * scale[c + 2] + beta[c + 2]), dot);
                    dot = fmaf(wf[c + 3], mish_f((r.w - mean[c + 3]) * scale[c + 3] + beta[c + 3]), dot);
                }
            }
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o, 16);
            if (lane16 == 0 && inb) update((long long)b * HW + m, mk, dot);
        }
    }
}

int launch_final(const FinalParams& p, cudaStream_t s) {
    int gx = p.chw4 ? (p.H * p.T + 255) / 256 : (p.H * p.T + 127) / 128;
    if (gx > 2048) gx = 2048;
    k_final<<<dim3(gx, p.B), 256, 4 * p.C * sizeof(float), s>>>(p);
    return 1;
}

// ----------------------------------------------------------------------------------------------
// time conditioning for a table of rows (diffusion.py:118-125,143-144,178-179 and ResnetBlock.mlp :64-65,76)
// Everything here depends on t only, never on xt, so it is evaluated for all N steps before the loop.
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_time_table(const TimeTableParams p) {
    extern __shared__ float sm[];
    float* emb = sm; float* hid = emb + p.dim; float* tm = hid + 4 * p.dim;
    const int r = blockIdx.x, tid = threadIdx.x, dim = p.dim, half = dim / 2;
    const float a = p.pe_scale * p.t_rows[r];
    for (int j = tid; j < half; j += 256) {
        const float arg = a * p.freqs[j];
        emb[j] = sinf(arg);
        emb[half + j] = cosf(arg);
    }
    __syncthreads();
    for (int o = tid; o < 4 * dim; o += 256) {
        float acc = p.b0[o];
        for (int k = 0; k < dim; ++k) acc = fmaf(p.w0[o * dim + k], emb[k], acc);
        hid[o] = mish_f(acc);
    }
    __syncthreads();
    for (int o = tid; o < dim; o += 256) {
        float acc = p.b2[o];
        for (int k = 0; k < 4 * dim; ++k) acc = fmaf(p.w2[o * 4 * dim + k], hid[k], acc);
        tm[o] = mish_f(acc);            // ResnetBlock.mlp starts with Mish (diffusion.py:64)
    }
    __syncthreads();
    for (int k = 0; k < p.nproj; ++k) {
        for (int o = tid; o < p.pc[k]; o += 256) {
            float acc = p.pb[k][o];
            for (int j = 0; j < dim; ++j) acc = fmaf(p.pw[k][o * dim + j], tm[j], acc);
            p.tb[(long long)r * p.tb_stride + p.poff[k] + o] = acc;
        }
    }
}

int launch_time_table(const TimeTableParams& p, cudaStream_t s) {
    k_time_table<<<p.rows, 256, 6 * p.dim * sizeof(float), s>>>(p);
    return 1;
}

// spk_mlp (diffusion.py:140-141,175-176): Linear(E,4E) -> Mish -> Linear(4E,n_feats); t-independent, once per call
__global__ void __launch_bounds__(256) k_spk(const SpkParams p) {
    extern __shared__ float sm[];
    float* x = sm; float* hid = sm + p.E;
    const int b = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < p.E; i += 256) x[i] = p.spk[b * p.E + i];
    __syncthreads();
    for (int o = tid; o < 4 * p.E; o += 256) {
        float acc = p.b0[o];
        for (int k = 0; k < p.E; ++k) acc = fmaf(p.w0[o * p.E + k], x[k], acc);
        hid[o] = mish_f(acc);
    }
    __syncthreads();
    for (int o = tid; o < p.n_feats; o += 256) {
        float acc = p.b2[o];
        for (int k = 0; k < 4 * p.E; ++k) acc = fmaf(p.w2[o * 4 * p.E + k], hid[k], acc);
        p.out[b * p.n_feats + o] = acc;
    }
}

int launch_spk(const SpkParams& p, cudaStream_t s) {
    k_spk<<<p.B, 256, 5 * p.E * sizeof(float), s>>>(p);
    return 1;
}

// DiffVC conditioning fold (see CondFoldParams): grid (rows*B), 256 threads
__global__ void __launch_bounds__(256) k_cond_fold(const CondFoldParams p) {
    extern __shared__ float s_c[];                      // cond vector [dc]
    const int rb = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < p.dc; i += 256) s_c[i] = p.cond[(long long)rb * p.dc + i];
    __syncthreads();
    const int cin = 2 + p.dc;
    for (int o = tid; o < 10 * p.C; o += 256) {
        const int t = o / p.C, co = o - t * p.C;        // t < 9: conv tap, t == 9: res_conv
        float a = 0.f;
        if (t < 9) {
            const float* w = p.w1 + ((long long)co * cin + 2) * 9 + t;
            for (int ci = 0; ci < p.dc; ++ci) a = fmaf(s_c[ci], __ldg(w + (long long)ci * 9), a);
            p.w_extra[((long long)rb * 9 + t) * p.C + co] = a;
        } else {
            const float* w = p.wres + (long long)co * cin + 2;
            for (int ci = 0; ci < p.dc; ++ci) a = fmaf(s_c[ci], __ldg(w + ci), a);
            p.r_extra[(long long)rb * p.C + co] = a;
        }
    }
}

int launch_cond_fold(const CondFoldParams& p, cudaStream_t s) {
    k_cond_fold<<<p.rows * p.B, 256, p.dc * sizeof(float), s>>>(p);
    return 1;
}

// ----------------------------------------------------------------------------------------------
// DiffVC RefBlock glue (tensor-core modes; the six 3x3 convs themselves run on k_conv_tc<G_C3>)
// ----------------------------------------------------------------------------------------------
__global__ void k_diff_mean(const DiffMeanParams p) {
    const long long n = (long long)p.B * p.H * p.T;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int w = (int)(i % p.T);
    const long long b = i / ((long long)p.H * p.T);
    p.out[i] = (p.ref[i] * p.g + p.mean_ref[i] * (1.0f - p.g)) * p.mask[b * p.T + w];
}
int launch_diff_mean(const DiffMeanParams& p, cudaStream_t s) {
    const long long n = (long long)p.B * p.H * p.T;
    k_diff_mean<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p);
    return 1;
}

// InstanceNorm2d statistics: one CTA per (16-byte channel chunk, sample); the chunk's rows are contiguous float4 runs
__global__ void __launch_bounds__(256) k_chan_stats(const ChanStatsParams p) {
    __shared__ double s_s[8][8];
    const int ch = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, c4n = p.C / 4;
    float sx[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
    double ds[4] = {0, 0, 0, 0}, dq[4] = {0, 0, 0, 0};
    for (int h = 0; h < p.H; ++h) {
        const float* row = p.x + ((((long long)b * p.H + h) * c4n + ch) * p.W) * 4;
        for (int w = tid; w < p.W; w += 256) {
            const float4 v = ldg4(row + (long long)w * 4);
            sx[0] += v.x; sx[1] += v.y; sx[2] += v.z; sx[3] += v.w;
            sq[0] = fmaf(v.x, v.x, sq[0]); sq[1] = fmaf(v.y, v.y, sq[1]); sq[2] = fmaf(v.z, v.z, sq[2]); sq[3] = fmaf(v.w, v.w, sq[3]);
        }
        if ((h & 7) == 7 || h == p.H - 1) {      // flush the fp32 partials into fp64 every 8 rows
#pragma unroll
            for (int q = 0; q < 4; ++q) { ds[q] += sx[q]; dq[q] += sq[q]; sx[q] = 0.f; sq[q] = 0.f; }
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { ds[q] += __shfl_xor_sync(0xffffffffu, ds[q], o); dq[q] += __shfl_xor_sync(0xffffffffu, dq[q], o); }
    }
    if ((tid & 31) == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) { s_s[tid >> 5][q] = ds[q]; s_s[tid >> 5][4 + q] = dq[q]; }
    }
    __syncthreads();
    if (tid < 8) {
        double a = 0;
        for (int wv = 0; wv < 8; ++wv) a += s_s[wv][tid];
        const int q = tid & 3, which = tid >> 2;
        p.stats[((long long)b * p.C + ch * 4 + q) * 2 + which] = a;
    }
}
int launch_chan_stats(const ChanStatsParams& p, cudaStream_t s) {
    k_chan_stats<<<dim3(p.C / 4, p.B), 256, 0, s>>>(p);
    return 1;
}

// InstanceNorm2d(affine) + GLU(dim=1) (+ time bias) * mask, written in operand form (tf32-rounded)
__global__ void __launch_bounds__(256) k_in_glu(const InGluParams p) {
    extern __shared__ float sm[];
    float* mean = sm; float* scale = mean + p.C; float* beta = scale + p.C; float* tbv = beta + p.C;   // tbv: [C/2]
    const int b = blockIdx.y, tid = threadIdx.x, Ch = p.C / 2;
    const double inv = 1.0 / ((double)p.H * p.W);
    for (int c = tid; c < p.C; c += 256) {
        const double s = p.stats[((long long)b * p.C + c) * 2], ss = p.stats[((long long)b * p.C + c) * 2 + 1];
        const double m = s * inv;
        double var = ss * inv - m * m;
        var = var < 0.0 ? 0.0 : var;
        mean[c] = (float)m;
        scale[c] = (float)(1.0 / sqrt(var + 1e-5)) * p.gamma[c];
        beta[c] = p.beta[c];
    }
    for (int c = tid; c < Ch; c += 256) tbv[c] = p.tb ? p.tb[c] : 0.f;
    __syncthreads();
    const int o4n = Ch / 4, i4n = p.C / 4;            // output / input channel chunks
    const long long n4 = (long long)p.H * p.W * o4n;
    for (long long i = (long long)blockIdx.x * 256 + tid; i < n4; i += (long long)gridDim.x * 256) {
        const long long hc = i / p.W;
        const int w = (int)(i - hc * p.W);
        const int h = (int)(hc / o4n), ch = (int)(hc - (long long)h * o4n);
        const float mk = __ldg(p.mask + (long long)b * p.T + w);
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        if (mk != 0.f) {
            const float* rowa = p.raw + ((((long long)b * p.H + h) * i4n + ch) * p.W + w) * 4;
            const float4 a = ldg4(rowa), g = ldg4(rowa + (long long)o4n * p.W * 4);      // gate half: channel c + C/2
            const float av[4] = {a.x, a.y, a.z, a.w}, gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int c = ch * 4 + q;
                const float xa = (av[q] - mean[c]) * scale[c] + beta[c];
                const float xg = (gv[q] - mean[Ch + c]) * scale[Ch + c] + beta[Ch + c];
                if (p.form == FORM_X3) {
                    o[q] = xa * (1.f / (1.f + expf(-xg))) + tbv[c];          // fp32x3 mode: exact sigmoid, no operand rounding
                } else {
                    float y = xa * __fdividef(1.f, 1.f + __expf(-xg)) + tbv[c];
                    uint32_t t; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(y));
                    o[q] = __uint_as_float(t);
                }
            }
        }
        *reinterpret_cast<float4*>(p.out + ((long long)b * n4 + i) * 4) = make_float4(o[0], o[1], o[2], o[3]);
    }
}
int launch_in_glu(const InGluParams& p, cudaStream_t s) {
    const long long n4 = (long long)p.H * p.W * (p.C / 8);
    int gx = (int)((n4 + 256 * 8 - 1) / (256 * 8));
    if (gx < 1) gx = 1;
    if (gx > 4096) gx = 4096;
    k_in_glu<<<dim3(gx, p.B), 256, (3 * p.C + p.C / 2) * sizeof(float), s>>>(p);
    return 1;
}

// conditioning vector of one step: [sinusoid(1000 t) | ref_block.final_conv(mean-pooled y) | c] -> cond_block
__global__ void __launch_bounds__(256) k_vc_cond(const VcCondParams p) {
    extern __shared__ float sm[];
    const int b = blockIdx.x, tid = threadIdx.x, dim = p.dim, dc = p.dc, half = dim / 2;
    const int n_in = dim + (p.use_ref ? dc : 0) + 256;
    float* in = sm;                 // [n_in]
    float* ybar = in + n_in;        // [dc]
    float* hid = ybar + dc;         // [4*dc]
    const float a = 1000.0f * p.t;  // SinusoidalPosEmb hard-codes the scale (modules.py:123)
    for (int j = tid; j < half; j += 256) {
        const float arg = a * p.freqs[j];
        in[j] = sinf(arg);
        in[half + j] = cosf(arg);
    }
    if (p.use_ref) {
        float msum = 0.f;
        for (int w = 0; w < p.Tr; ++w) msum += p.mask[(long long)b * p.Tr + w];
        const double den = (double)msum * p.H;
        for (int c = tid; c < dc; c += 256) ybar[c] = (float)(p.ysum[((long long)b * dc + c) * 2] / den);
    }
    for (int j = tid; j < 256; j += 256) in[dim + (p.use_ref ? dc : 0) + j] = p.c[(long long)b * 256 + j];
    __syncthreads();
    if (p.use_ref) {
        for (int o = tid; o < dc; o += 256) {
            float acc = p.bf[o];
            for (int k = 0; k < dc; ++k) acc = fmaf(p.wf[o * dc + k], ybar[k], acc);
            in[dim + o] = acc;
        }
        __syncthreads();
    }
    for (int o = tid; o < 4 * dc; o += 256) {
        float acc = p.b0[o];
        for (int k = 0; k < n_in; ++k) acc = fmaf(p.w0[(long long)o * n_in + k], in[k], acc);
        hid[o] = mish_f(acc);
    }
    __syncthreads();
    for (int o = tid; o < dc; o += 256) {
        float acc = p.b2[o];
        for (int k = 0; k < 4 * dc; ++k) acc = fmaf(p.w2[o * 4 * dc + k], hid[k], acc);
        p.out[(long long)b * dc + o] = acc;
    }
}
int launch_vc_cond(const VcCondParams& p, cudaStream_t s) {
    const int n_in = p.dim + (p.use_ref ? p.dc : 0) + 256;
    k_vc_cond<<<p.B, 256, (n_in + p.dc + 4 * p.dc) * sizeof(float), s>>>(p);
    return 1;
}

// zero the GroupNorm statistics arena and advance the device-side step counter
// ----------------------------------------------------------------------------------------------
// GradTTS.forward, the lines between the text encoder and the decoder (Grad-TTS/model/tts.py:82-94, model/utils.py:26-39).
// The reference builds the 0/1 alignment `attn` [B,Tx,Ty] with five full-size elementwise passes (zeros, sequence_mask over
// B*Tx rows, pad, subtract, mask) and then multiplies it with mu_x as a dense batched GEMM.  attn^T @ mu_x^T with a 0/1
// matrix that has at most one 1 per output frame is a gather, so one thread per output frame finds its token by binary
// search in the cumulative durations and copies that token's F features: one pass, exact.
//   path[i][t] = [t < cum_i] - [t < cum_(i-1)]  (float compares against the frame index, utils.py:33-37), * x_mask_i * y_mask_t
// ----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_prior_expand(const PriorExpandParams p) {
    extern __shared__ __align__(16) float s_cum[];         // [Tx] cumulative durations of this sample
    const int b = blockIdx.y, tid = threadIdx.x;
    if (tid == 0) {
        // torch.cumsum on the CPU reference accumulates sequentially in double (at::acc_type<float, false>) and rounds each
        // prefix to fp32; durations are non-integers when length_scale != 1 and prefixes such as 100 x 0.91 land next to
        // an integer, so the accumulation type decides which frame a token boundary falls on
        double c = 0.0;
        const float* w = p.w_ceil + (long long)b * p.Tx;
        for (int i = 0; i < p.Tx; ++i) { c += (double)w[i]; s_cum[i] = (float)c; }
    }
    __syncthreads();
    const int t = blockIdx.x * 256 + tid;
    if (t >= p.Ty) return;
    const float tf = (float)t;
    // first token whose cumulative duration exceeds t (cum is non-decreasing): path[i][t] = 1 exactly for that token
    int lo = 0, hi = p.Tx;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (tf < s_cum[mid]) hi = mid; else lo = mid + 1; }
    const int tok = lo;                                    // == Tx: frame beyond the last token
    const float ym = (long long)t < p.y_len[b] ? 1.f : 0.f;
    const float am = tok < p.Tx ? __ldg(p.x_mask + (long long)b * p.Tx + tok) * ym : 0.f;   // attn_mask at (tok, t)
    p.y_mask[(long long)b * p.Ty + t] = ym;
    const float* mx = p.mu_x + (long long)b * p.F * p.Tx + (tok < p.Tx ? tok : 0);
    const float* nz = p.noise_tf ? p.noise_tf + ((long long)b * p.Ty + t) * p.F : nullptr;
    for (int f = 0; f < p.F; ++f) {
        // attn is exactly 0 or 1: the reference's matmul adds one product and Tx-1 zeros
        const float m = am != 0.f ? __ldg(mx + (long long)f * p.Tx) * am : 0.f;
        const long long o = ((long long)b * p.F + f) * p.Ty + t;
        p.mu_y[o] = m;
        p.z[o] = nz ? m + __fdiv_rn(nz[f], p.temperature) : m;
    }
    if (p.attn) {
        float* ap = p.attn + (long long)b * p.Tx * p.Ty + t;
        for (int i = 0; i < p.Tx; ++i) ap[(long long)i * p.Ty] = (i == tok) ? am : 0.f;
    }
}

int launch_prior_expand(const PriorExpandParams& p, cudaStream_t s) {
    k_prior_expand<<<dim3((p.Ty + 255) / 256, p.B), 256, (size_t)p.Tx * sizeof(float), s>>>(p);
    return 1;
}

__global__ void k_step_begin(const StepBeginParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n_doubles) p.stats[i] = 0.0;
    if (i == 0) {
        const int cur = *p.step_next;
        *p.step_cur = cur;
        *p.step_next = cur + 1;
    }
}

int launch_step_begin(const StepBeginParams& p, cudaStream_t s) {
    const int n = p.n_doubles > 0 ? p.n_doubles : 1;
    k_step_begin<<<(n + 255) / 256, 256, 0, s>>>(p);
    return 1;
}

// xt0 = z * mask (diffusion.py:256)
__global__ void k_scale_mask(const float* z, const float* mask, float* out, int H, int T, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int w = (int)(i % T);
    const long long b = i / ((long long)H * T);
    out[i] = z[i] * mask[b * T + w];
}

int launch_scale_mask(const float* z, const float* mask, float* out, long long, int B, int H, int T, cudaStream_t s) {
    const long long n = (long long)B * H * T;
    k_scale_mask<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(z, mask, out, H, T, n);
    return 1;
}

}  // namespace sbk
