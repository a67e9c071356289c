// Grad-TTS text encoder (token ids -> mu_x, logw, x_mask): Grad-TTS/model/text_encoder.py:281-326 (TextEncoder) with its
// ConvReluNorm prenet (:32-64), the relative-position transformer encoder (:96-278) and the duration predictor (:67-93),
// eval mode.  SURVEY.md 8(f) rank 4: the module whose outputs feed `sbk_prior_expand` and the sampler; it runs once per
// utterance (7.3 M MACs per token: 0.07 % of the 50-step decoder's work), so the design goal is few launches and exact fp32
// arithmetic, not tensor-core throughput.
//
// Activations are token-major fp32 [B][T][C] (a token's channels are contiguous: the natural layout for 1-D convs over few
// channels).  Everything a conv feeds is fused into its epilogue: bias, ReLU, the x_mask multiplies, the residual add and
// the channel LayerNorm (eps 1e-4, biased variance, :11-29) - a CTA owns TE_TOK tokens x ALL output channels, so the
// LayerNorm reduction never leaves the CTA.  39 launches per forward (the reference issues ~330 ATen kernels):
//   k_te_embed                      emb(x) * sqrt(C)                                            (:313)
//   k_te_conv x4                    prenet: 3 x relu(LN(conv5(x*mask))), then (org + proj(x)) * mask   (:57-64)
//   per layer: k_te_conv (q|k|v as one 3C-channel 1x1), k_te_attn, k_te_conv (conv_o + residual + LN),
//              k_te_conv (ffn conv_1 + relu + mask), k_te_conv (ffn conv_2 + mask + residual + LN)      (:267-278)
//   k_te_conv                       proj_m(x*mask) * mask -> mu_x, written planar [B][n_feats][T]       (:321)
//   k_te_conv x3                    duration predictor: 2 x LN(relu(conv3(x*mask))), proj -> logw       (:83-93)
// k_te_attn: one warp per (utterance, head, query): scores over all keys with the windowed relative-position logits
// q_i.E_k[j-i+w] added for |j-i| <= w (:151-157 restated directly instead of through the pad/reshape skewing), the
// reference's masked_fill(-1e4), softmax, p.V plus the relative-value term sum_j p_ij E_v[j-i+w] (:164-169).
#include "sbk_host.h"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

using namespace sbk;

namespace {

constexpr int TE_TOK = 8;            // tokens per CTA of k_te_conv
constexpr int TE_MAXCO = 3;          // output channels per thread (Cout <= 768)

struct TeConvParams {
    const float* in; int Cin;        // [B][T][Cin], or the reference's planar [B][Cin][T] when in_planar
    int in_planar;
    const float* spk; int E;         // optional: Cin..Cin+E-1 are the speaker embedding [B][E], constant over T (:317-318)
    const float* w;                  // packed [K][Cin+E][Cout]
    const float* bias;               // [Cout]
    int K, Cout, B, T;
    const float* mask;               // x_mask [B][T]
    int in_mask;                     // the conv reads x * x_mask
    int relu1, mask1;                // after the bias: ReLU, then * x_mask
    const float* res; int res_mask;  // + residual (optionally residual * x_mask)
    const float* ln_g; const float* ln_b;   // channel LayerNorm when non-null
    int relu2, mask2;                // after the LayerNorm: ReLU, then * x_mask
    float* out; int out_planar;      // [B][T][Cout], or the reference's planar [B][Cout][T]
};

__global__ void k_te_embed(const long long* ids, const float* emb, float* out, int n_tok, int C, int V, float scale) {
    const long long n = (long long)n_tok * (C / 4);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long tok = i / (C / 4); const int c4 = (int)(i - tok * (C / 4));
        long long id = ids[tok];
        id = id < 0 ? 0 : (id >= V ? V - 1 : id);
        const float4 e = __ldg(reinterpret_cast<const float4*>(emb + id * C) + c4);
        reinterpret_cast<float4*>(out)[i] = make_float4(e.x * scale, e.y * scale, e.z * scale, e.w * scale);
    }
}

__global__ void k_te_mask(const long long* lengths, float* mask, int B, int T) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < B * T) mask[i] = (i % T) < lengths[i / T] ? 1.f : 0.f;            // sequence_mask (model/utils.py:6-10)
}

__global__ void __launch_bounds__(256) k_te_conv(const TeConvParams p) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x, b = blockIdx.y, t0 = blockIdx.x * TE_TOK;
    const int Ci = p.Cin + p.E, pad = p.K / 2, NPOS = TE_TOK + p.K - 1;
    float* s_in = sm;                                   // [NPOS][Ci]; reused as [TE_TOK][Cout] by the LayerNorm
    __shared__ float s_mk[TE_TOK + 8];
    __shared__ float s_mean[TE_TOK], s_rstd[TE_TOK];
    for (int i = tid; i < NPOS * Ci; i += 256) {
        const int pos = i / Ci, ci = i - pos * Ci, t = t0 + pos - pad;
        float v = 0.f;
        if (t >= 0 && t < p.T) {
            v = ci >= p.Cin ? p.spk[(long long)b * p.E + ci - p.Cin]
                : p.in_planar ? p.in[((long long)b * p.Cin + ci) * p.T + t] : p.in[((long long)b * p.T + t) * p.Cin + ci];
            if (p.in_mask) v *= p.mask[(long long)b * p.T + t];
        }
        s_in[i] = v;
    }
    if (tid < TE_TOK) s_mk[tid] = (t0 + tid < p.T) ? p.mask[(long long)b * p.T + t0 + tid] : 0.f;
    __syncthreads();
    float acc[TE_MAXCO][TE_TOK];
    int co[TE_MAXCO];
#pragma unroll
    for (int o = 0; o < TE_MAXCO; ++o) {
        co[o] = tid + 256 * o;
        const float bb = co[o] < p.Cout ? p.bias[co[o]] : 0.f;
#pragma unroll
        for (int k = 0; k < TE_TOK; ++k) acc[o][k] = bb;
    }
    for (int k = 0; k < p.K; ++k) {
        const float* wk = p.w + (long long)k * Ci * p.Cout;
        for (int ci = 0; ci < Ci; ++ci) {
            float x[TE_TOK];
#pragma unroll
            for (int q = 0; q < TE_TOK; ++q) x[q] = s_in[(q + k) * Ci + ci];
#pragma unroll
            for (int o = 0; o < TE_MAXCO; ++o) {
                if (co[o] < p.Cout) {
                    const float w = __ldg(wk + (long long)ci * p.Cout + co[o]);
#pragma unroll
                    for (int q = 0; q < TE_TOK; ++q) acc[o][q] = fmaf(x[q], w, acc[o][q]);
                }
            }
        }
    }
    // ---- epilogue
#pragma unroll
    for (int o = 0; o < TE_MAXCO; ++o) {
        if (co[o] >= p.Cout) continue;
#pragma unroll
        for (int q = 0; q < TE_TOK; ++q) {
            const int t = t0 + q;
            float v = acc[o][q];
            if (p.relu1) v = fmaxf(v, 0.f);
            if (p.mask1) v *= s_mk[q];
            if (p.res && t < p.T) {
                const float r = p.res[((long long)b * p.T + t) * p.Cout + co[o]];
                v += p.res_mask ? r * s_mk[q] : r;
            }
            acc[o][q] = v;
        }
    }
    if (p.ln_g) {
        __syncthreads();                                // s_in is dead: reuse it for the LayerNorm exchange
        float* s_v = sm;                                // [TE_TOK][Cout]
#pragma unroll
        for (int o = 0; o < TE_MAXCO; ++o)
            if (co[o] < p.Cout)
#pragma unroll
                for (int q = 0; q < TE_TOK; ++q) s_v[q * p.Cout + co[o]] = acc[o][q];
        __syncthreads();
        {   // warp q reduces token q: mean, then the biased variance of (x - mean) (two passes, as the reference computes it)
            const int q = tid >> 5, lane = tid & 31;
            float s = 0.f;
            for (int c = lane; c < p.Cout; c += 32) s += s_v[q * p.Cout + c];
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
            const float mean = s / (float)p.Cout;
            float vs = 0.f;
            for (int c = lane; c < p.Cout; c += 32) { const float d = s_v[q * p.Cout + c] - mean; vs = fmaf(d, d, vs); }
#pragma unroll
            for (int m = 16; m > 0; m >>= 1) vs += __shfl_xor_sync(0xffffffffu, vs, m);
            if (lane == 0) { s_mean[q] = mean; s_rstd[q] = 1.0f / sqrtf(vs / (float)p.Cout + 1e-4f); }
        }
        __syncthreads();
#pragma unroll
        for (int o = 0; o < TE_MAXCO; ++o)
            if (co[o] < p.Cout) {
                const float g = p.ln_g[co[o]], be = p.ln_b[co[o]];
#pragma unroll
                for (int q = 0; q < TE_TOK; ++q) acc[o][q] = (acc[o][q] - s_mean[q]) * s_rstd[q] * g + be;
            }
    }
#pragma unroll
    for (int o = 0; o < TE_MAXCO; ++o) {
        if (co[o] >= p.Cout) continue;
#pragma unroll
        for (int q = 0; q < TE_TOK; ++q) {
            const int t = t0 + q;
            if (t >= p.T) continue;
            float v = acc[o][q];
            if (p.relu2) v = fmaxf(v, 0.f);
            if (p.mask2) v *= s_mk[q];
            if (p.out_planar) p.out[((long long)b * p.Cout + co[o]) * p.T + t] = v;
            else p.out[((long long)b * p.T + t) * p.Cout + co[o]] = v;
        }
    }
}

// Self-attention with windowed relative positions (:143-171).  qkv: [B][T][3C] (q | k | v), head h = channels [h*d, (h+1)*d).
__global__ void __launch_bounds__(256) k_te_attn(const float* qkv, const float* mask, const float* ek, const float* ev,
                                                 float* out, int B, int T, int C, int H, int win) {
    extern __shared__ __align__(16) float sm[];
    const int d = C / H, nrel = 2 * win + 1;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * 8 + warp, h = blockIdx.y, b = blockIdx.z;
    if (i >= T) return;                                   // (no block-wide barrier below)
    const int Tp = (T + 3) & ~3;                          // keeps every warp's slice 16-byte aligned
    float* s_q = sm + (size_t)warp * (d + Tp + 32);
    float* s_p = s_q + d;
    float* s_qe = s_p + Tp;
    const long long row = (long long)b * T;
    const float* qp = qkv + (row + i) * 3 * C + h * d;
    for (int c = lane; c < d; c += 32) s_q[c] = qp[c];
    __syncwarp();
    const float scale = 1.0f / sqrtf((float)d);
    if (lane < nrel) {
        float a = 0.f;
        for (int c = 0; c < d; ++c) a = fmaf(s_q[c], ek[lane * d + c], a);
        s_qe[lane] = a;
    }
    __syncwarp();
    const float mi = mask[row + i];
    float mx = -INFINITY;
    for (int j = lane; j < T; j += 32) {
        const float4* kp = reinterpret_cast<const float4*>(qkv + (row + j) * 3 * C + C + h * d);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int c4 = 0; c4 < d / 4; ++c4) {
            const float4 kv = __ldg(kp + c4);
            const float4 qv = *reinterpret_cast<const float4*>(s_q + c4 * 4);
            a0 = fmaf(qv.x, kv.x, a0); a1 = fmaf(qv.y, kv.y, a1); a2 = fmaf(qv.z, kv.z, a2); a3 = fmaf(qv.w, kv.w, a3);
        }
        float sc = ((a0 + a1) + (a2 + a3)) * scale;
        const int rel = j - i;
        if (rel >= -win && rel <= win) sc += s_qe[rel + win] * scale;
        if (mi * mask[row + j] == 0.f) sc = -1e4f;        // masked_fill(mask == 0, -1e4)
        s_p[j] = sc;
        mx = fmaxf(mx, sc);
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
    float z = 0.f;
    for (int j = lane; j < T; j += 32) { const float e = expf(s_p[j] - mx); s_p[j] = e; z += e; }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) z += __shfl_xor_sync(0xffffffffu, z, m);
    const float inv = 1.0f / z;
    __syncwarp();
    for (int c = lane; c < d; c += 32) {
        float a = 0.f;
        const float* vp = qkv + row * 3 * C + 2 * C + h * d + c;
        for (int j = 0; j < T; ++j) a = fmaf(s_p[j], __ldg(vp + (long long)j * 3 * C), a);
        float r = 0.f;
        for (int q = 0; q < nrel; ++q) {
            const int j = i + q - win;
            if (j >= 0 && j < T) r = fmaf(s_p[j], ev[q * d + c], r);
        }
        out[(row + i) * C + h * d + c] = (a + r) * inv;
    }
}

__global__ void k_te_concat_spk(const float* h, const float* spk, float* out, int B, int T, int C, int E) {
    const long long n = (long long)B * T * (C + E);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % (C + E)); const long long tok = i / (C + E);
        out[i] = c < C ? h[tok * C + c] : spk[(tok / T) * E + c - C];
    }
}

}  // namespace

struct sbk_textenc {
    sbk_textenc_config cfg;
    WeightSet w;
    Workspace ws;
    bool is_packed = false;
    int64_t last_launches = 0;
    // debug capture (fmt: 0 token-major fp32 [B][T][C], 1 planar fp32 [B][C][T])
    Snapshots snaps;
    int enc_ch() const { return cfg.n_channels + (cfg.n_spks > 1 ? cfg.spk_emb_dim : 0); }
};

extern "C" int sbk_textenc_create(const sbk_textenc_config* cfg, sbk_textenc** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_textenc_create: null argument");
    const int C = cfg->n_channels, Ce = C + (cfg->n_spks > 1 ? cfg->spk_emb_dim : 0);
    if (C <= 0 || C % 4 != 0 || Ce % 4 != 0) return fail(SBK_ERR_ARG, "sbk_textenc_create: channel counts must be multiples of 4");
    if (cfg->n_heads <= 0 || Ce % cfg->n_heads != 0 || (Ce / cfg->n_heads) % 4 != 0) return fail(SBK_ERR_ARG, "sbk_textenc_create: channels / heads must be a multiple of 4");
    if (3 * Ce > 256 * TE_MAXCO || cfg->filter_channels > 256 * TE_MAXCO || cfg->filter_channels_dp > 256 * TE_MAXCO || cfg->n_feats > 256 * TE_MAXCO)
        return fail(SBK_ERR_UNSUPPORTED, "sbk_textenc_create: at most %d output channels per conv", 256 * TE_MAXCO);
    if (cfg->kernel_size < 1 || cfg->kernel_size % 2 == 0 || cfg->kernel_size > 9) return fail(SBK_ERR_ARG, "sbk_textenc_create: kernel_size must be odd and <= 9");
    if (cfg->window_size < 1 || cfg->window_size > 15) return fail(SBK_ERR_UNSUPPORTED, "sbk_textenc_create: window_size must be in 1..15 (relative-position attention)");
    sbk_textenc* e = new sbk_textenc();
    e->cfg = *cfg;
    auto add = [&](const std::string& n, std::vector<int64_t> s) { e->w.add(n, std::move(s)); };
    const int F = cfg->filter_channels, Fd = cfg->filter_channels_dp, K = cfg->kernel_size, d = Ce / cfg->n_heads, nrel = 2 * cfg->window_size + 1;
    const bool mel = cfg->kind == 1;         // DiffVC MelEncoder (DiffVC/model/encoder.py:257-284): init_proj | prenet | encoder | term_proj
    if (mel && cfg->n_spks > 1) { delete e; return fail(SBK_ERR_ARG, "sbk_textenc_create: the mel encoder has no speaker input"); }
    if (mel) { add("init_proj.weight", {C, cfg->n_feats, 1}); add("init_proj.bias", {C}); }
    else add("emb.weight", {cfg->n_vocab, C});
    for (int i = 0; i < 3; ++i) {
        const std::string p = "prenet.";
        add(p + "conv_layers." + std::to_string(i) + ".weight", {C, C, 5}); add(p + "conv_layers." + std::to_string(i) + ".bias", {C});
        add(p + "norm_layers." + std::to_string(i) + ".gamma", {C}); add(p + "norm_layers." + std::to_string(i) + ".beta", {C});
    }
    add("prenet.proj.weight", {C, C, 1}); add("prenet.proj.bias", {C});
    for (int i = 0; i < cfg->n_layers; ++i) {
        const std::string a = "encoder.attn_layers." + std::to_string(i), n = std::to_string(i);
        add(a + ".emb_rel_k", {1, nrel, d}); add(a + ".emb_rel_v", {1, nrel, d});
        for (const char* c : {"conv_q", "conv_k", "conv_v", "conv_o"}) { add(a + "." + c + ".weight", {Ce, Ce, 1}); add(a + "." + c + ".bias", {Ce}); }
        add("encoder.norm_layers_1." + n + ".gamma", {Ce}); add("encoder.norm_layers_1." + n + ".beta", {Ce});
        add("encoder.ffn_layers." + n + ".conv_1.weight", {F, Ce, K}); add("encoder.ffn_layers." + n + ".conv_1.bias", {F});
        add("encoder.ffn_layers." + n + ".conv_2.weight", {Ce, F, K}); add("encoder.ffn_layers." + n + ".conv_2.bias", {Ce});
        add("encoder.norm_layers_2." + n + ".gamma", {Ce}); add("encoder.norm_layers_2." + n + ".beta", {Ce});
    }
    if (mel) {
        add("term_proj.weight", {cfg->n_feats, C, 1}); add("term_proj.bias", {cfg->n_feats});
    } else {
        add("proj_m.weight", {cfg->n_feats, Ce, 1}); add("proj_m.bias", {cfg->n_feats});
        add("proj_w.conv_1.weight", {Fd, Ce, K}); add("proj_w.conv_1.bias", {Fd});
        add("proj_w.norm_1.gamma", {Fd}); add("proj_w.norm_1.beta", {Fd});
        add("proj_w.conv_2.weight", {Fd, Fd, K}); add("proj_w.conv_2.bias", {Fd});
        add("proj_w.norm_2.gamma", {Fd}); add("proj_w.norm_2.beta", {Fd});
        add("proj_w.proj.weight", {1, Fd, 1}); add("proj_w.proj.bias", {1});
    }
    *out = e;
    return SBK_OK;
}

extern "C" void sbk_textenc_destroy(sbk_textenc* e) {
    delete e;
}
extern "C" int sbk_textenc_num_weights(const sbk_textenc* e) { return e ? e->w.count() : 0; }
extern "C" const char* sbk_textenc_weight_name(const sbk_textenc* e, int i) { return e ? e->w.name(i) : nullptr; }

extern "C" int sbk_textenc_set_weight(sbk_textenc* e, const char* name, const void* data, const int64_t* shape, int ndim) {
    if (!e || !name || !data || !shape) return fail(SBK_ERR_ARG, "sbk_textenc_set_weight: null argument");
    TRY(e->w.set(name, data, shape, ndim, e->cfg.device, "sbk_textenc_set_weight"));
    e->is_packed = false;
    return SBK_OK;
}

// conv weights [co][ci][k] (one or several stacked along co) -> [k][ci][co_total]
static int te_pack(sbk_textenc* e, const std::vector<std::string>& srcs, const std::string& key, bool bias) {
    std::vector<std::vector<float>> ws; std::vector<std::vector<int64_t>> shapes;
    int64_t co_total = 0;
    for (auto& n : srcs) {
        std::vector<float> w;
        TRY(e->w.fetch(n, w));
        const std::vector<int64_t>& shape = e->w.find(n)->shape;
        ws.push_back(std::move(w)); shapes.push_back(shape); co_total += shape[0];
    }
    std::vector<float> outw;
    if (bias) {
        for (auto& w : ws) outw.insert(outw.end(), w.begin(), w.end());
    } else {
        const int64_t ci = shapes[0][1], K = shapes[0][2];
        outw.resize((size_t)K * ci * co_total);
        int64_t off = 0;
        for (size_t m = 0; m < ws.size(); ++m) {
            const int64_t co = shapes[m][0];
            for (int64_t o = 0; o < co; ++o) for (int64_t i = 0; i < ci; ++i) for (int64_t k = 0; k < K; ++k)
                outw[((size_t)k * ci + i) * co_total + off + o] = ws[m][((size_t)o * ci + i) * K + k];
            off += co;
        }
    }
    return upload(e->w.packed, key, outw.size() * 4, outw.data());
}

extern "C" int sbk_textenc_pack(sbk_textenc* e) {
    if (!e) return fail(SBK_ERR_ARG, "sbk_textenc_pack: null handle");
    TRY(e->w.require_all("sbk_textenc_pack"));
    CU(cudaSetDevice(e->cfg.device));
    for (int i = 0; i < 3; ++i) TRY(te_pack(e, {"prenet.conv_layers." + std::to_string(i) + ".weight"}, "prenet.conv" + std::to_string(i), false));
    TRY(te_pack(e, {"prenet.proj.weight"}, "prenet.proj", false));
    for (int i = 0; i < e->cfg.n_layers; ++i) {
        const std::string a = "encoder.attn_layers." + std::to_string(i), n = std::to_string(i);
        TRY(te_pack(e, {a + ".conv_q.weight", a + ".conv_k.weight", a + ".conv_v.weight"}, a + ".qkv.w", false));
        TRY(te_pack(e, {a + ".conv_q.bias", a + ".conv_k.bias", a + ".conv_v.bias"}, a + ".qkv.b", true));
        TRY(te_pack(e, {a + ".conv_o.weight"}, a + ".o.w", false));
        TRY(te_pack(e, {"encoder.ffn_layers." + n + ".conv_1.weight"}, "ffn" + n + ".1", false));
        TRY(te_pack(e, {"encoder.ffn_layers." + n + ".conv_2.weight"}, "ffn" + n + ".2", false));
    }
    if (e->cfg.kind == 1) {
        TRY(te_pack(e, {"init_proj.weight"}, "init_proj", false));
        TRY(te_pack(e, {"term_proj.weight"}, "term_proj", false));
    } else {
        TRY(te_pack(e, {"proj_m.weight"}, "proj_m", false));
        TRY(te_pack(e, {"proj_w.conv_1.weight"}, "dp.1", false));
        TRY(te_pack(e, {"proj_w.conv_2.weight"}, "dp.2", false));
        TRY(te_pack(e, {"proj_w.proj.weight"}, "dp.p", false));
    }
    e->is_packed = true;
    return SBK_OK;
}

// shared body of TextEncoder.forward (x, x_lengths given; mel == nullptr) and MelEncoder.forward (mel, mask_in given)
static int te_forward(sbk_textenc* e, const int64_t* x, const int64_t* x_lengths, const float* spk, const float* mel, const float* mask_in,
                      float* mu_x, float* logw, float* x_mask, int B, int Tx, void* stream) {
    if (!e->is_packed) return fail(SBK_ERR_STATE, "sbk_textenc_forward: weights not packed");
    if (B <= 0 || Tx <= 0) return fail(SBK_ERR_ARG, "sbk_textenc_forward: B and Tx must be positive");
    const sbk_textenc_config& c = e->cfg;
    if (c.n_spks > 1 && !spk) return fail(SBK_ERR_ARG, "sbk_textenc_forward: spk is required when n_spks > 1");
    // k_te_attn keeps one (d + Tx + 32)-float slice per warp in shared memory: a longer sequence is refused here, before
    // anything is launched or written
    const int d = e->enc_ch() / c.n_heads;
    const size_t asm_ = (size_t)8 * (d + ((Tx + 3) & ~3) + 32) * sizeof(float);
    if (asm_ > 200 * 1024) return fail(SBK_ERR_UNSUPPORTED, "sbk_textenc_forward: Tx = %d tokens exceeds the attention kernel's shared-memory budget", Tx);
    CU(cudaSetDevice(c.device));
    cudaStream_t s = (cudaStream_t)stream;
    const int C = c.n_channels, Ce = e->enc_ch(), F = c.filter_channels, Fd = c.filter_channels_dp, K = c.kernel_size;
    const size_t ntok = (size_t)B * Tx;
    const size_t wide = (size_t)std::max(std::max(3 * Ce, F), Fd);
    // three token-major [B][Tx][Ce] activations and two [B][Tx][wide] scratch buffers (q|k|v, the hidden layers)
    float *h0, *h1, *h2, *wa, *wb;
    auto carve = [&](Arena& ar) {
        auto take = [&](size_t floats) { return (float*)ar.take(floats * sizeof(float)); };
        h0 = take(ntok * Ce); h1 = take(ntok * Ce); h2 = take(ntok * Ce); wa = take(ntok * wide); wb = take(ntok * wide);
    };
    Arena probe;
    carve(probe);
    if (e->ws.reserve(probe.bytes())) return fail(SBK_ERR_CUDA, "out of memory: text-encoder workspace %zu bytes", probe.bytes());
    Arena ar = e->ws.arena();
    carve(ar);
    int64_t n = 0;
    // debug capture: the activations are rewritten within the call, so each tensor is copied right after the launch that wrote it
    e->snaps.begin();
    auto snap = [&](const std::string& name, const float* src, size_t channels, int fmt) { e->snaps.record(name, src, ntok * channels, fmt, s); };
    auto conv = [&](const float* in, int Cin, const float* spk_in, int E, const std::string& wkey, const std::string& bkey, int Kk, int Cout,
                    int in_mask, int relu1, int mask1, const float* res, int res_mask, const std::string& ln, int relu2, int mask2,
                    float* out, int planar, int in_planar = 0) {
        TeConvParams p; memset(&p, 0, sizeof(p));
        p.in = in; p.Cin = Cin; p.in_planar = in_planar; p.spk = spk_in; p.E = E; p.w = e->w.get(wkey); p.bias = e->w.get(bkey); p.K = Kk; p.Cout = Cout; p.B = B; p.T = Tx;
        p.mask = x_mask; p.in_mask = in_mask; p.relu1 = relu1; p.mask1 = mask1; p.res = res; p.res_mask = res_mask;
        if (!ln.empty()) { p.ln_g = e->w.get(ln + ".gamma"); p.ln_b = e->w.get(ln + ".beta"); }
        p.relu2 = relu2; p.mask2 = mask2; p.out = out; p.out_planar = planar;
        const size_t smem = sizeof(float) * std::max((size_t)(TE_TOK + Kk - 1) * (Cin + E), (size_t)TE_TOK * Cout);
        k_te_conv<<<dim3((Tx + TE_TOK - 1) / TE_TOK, B), 256, smem, s>>>(p);
        ++n;
    };
    static bool attr_done[64] = {};
    if (c.device >= 0 && c.device < 64 && !attr_done[c.device]) {
        CU(cudaFuncSetAttribute(k_te_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        CU(cudaFuncSetAttribute(k_te_attn, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr_done[c.device] = true;
    }
    if (mel) {
        // MelEncoder (DiffVC/model/encoder.py:279-284): x = init_proj(x * x_mask); the caller's mask is used as is
        x_mask = const_cast<float*>(mask_in);
        conv(mel, c.n_feats, nullptr, 0, "init_proj", "init_proj.bias", 1, C, 1, 0, 0, nullptr, 0, "", 0, 0, h0, 0, 1);
        snap("init_proj", h0, C, 0);
    } else {
        k_te_mask<<<(B * Tx + 255) / 256, 256, 0, s>>>(reinterpret_cast<const long long*>(x_lengths), x_mask, B, Tx); ++n;
        snap("mask", x_mask, 1, 0);
        k_te_embed<<<(int)std::min<size_t>((ntok * (C / 4) + 255) / 256, 8 * (size_t)sbk::device_sm_count()), 256, 0, s>>>(reinterpret_cast<const long long*>(x), e->w.get("emb.weight"), h0, (int)ntok, C, c.n_vocab, sqrtf((float)C)); ++n;
        snap("embed", h0, C, 0);
    }
    // ---- prenet (ConvReluNorm, :57-64): x = relu(LN(conv5(x * mask))) x3; x = (x_org + proj(x)) * mask
    const float* cur = h0; float* pp[2] = {h1, h2};
    for (int i = 0; i < 3; ++i) {
        conv(cur, C, nullptr, 0, "prenet.conv" + std::to_string(i), "prenet.conv_layers." + std::to_string(i) + ".bias", 5, C,
             1, 0, 0, nullptr, 0, "prenet.norm_layers." + std::to_string(i), 1, 0, pp[i & 1], 0);
        cur = pp[i & 1];
        snap("prenet." + std::to_string(i), cur, C, 0);
    }
    float* hx = cur == h1 ? h2 : h1;
    conv(cur, C, nullptr, 0, "prenet.proj", "prenet.proj.bias", 1, C, 0, 0, 0, h0, 0, "", 0, 1, hx, 0);
    snap("prenet.proj", hx, C, 0);
    // (multi-speaker: the speaker embedding is concatenated to every token after the prenet, :317-318)
    float* h = hx;
    if (c.n_spks > 1) {
        // h0 is free now but sized for Ce as well: concatenate into it
        k_te_concat_spk<<<(int)std::min<size_t>((ntok * Ce + 255) / 256, 8 * (size_t)sbk::device_sm_count()), 256, 0, s>>>(hx, spk, h0, B, Tx, C, c.spk_emb_dim); ++n;
        h = h0;
        snap("spk_concat", h0, Ce, 0);
    }
    float* other[2];
    { int k = 0; for (float* q : {h0, h1, h2}) if (q != h && k < 2) other[k++] = q; }
    // ---- encoder (:267-278)
    for (int i = 0; i < c.n_layers; ++i) {
        const std::string a = "encoder.attn_layers." + std::to_string(i), nn = std::to_string(i), q = "enc." + nn;
        conv(h, Ce, nullptr, 0, a + ".qkv.w", a + ".qkv.b", 1, 3 * Ce, 1, 0, 0, nullptr, 0, "", 0, 0, wa, 0);          // x = x * mask; q|k|v
        snap(q + ".qkv", wa, 3 * Ce, 0);
        k_te_attn<<<dim3((Tx + 7) / 8, c.n_heads, B), 256, asm_, s>>>(wa, x_mask, e->w.get(a + ".emb_rel_k"), e->w.get(a + ".emb_rel_v"), wb, B, Tx, Ce, c.n_heads, c.window_size); ++n;
        snap(q + ".attn", wb, Ce, 0);
        conv(wb, Ce, nullptr, 0, a + ".o.w", a + ".conv_o.bias", 1, Ce, 0, 0, 0, h, 1, "encoder.norm_layers_1." + nn, 0, 0, other[0], 0);   // LN(x*mask + attn)
        snap(q + ".ln1", other[0], Ce, 0);
        conv(other[0], Ce, nullptr, 0, "ffn" + nn + ".1", "encoder.ffn_layers." + nn + ".conv_1.bias", K, F, 1, 1, 1, nullptr, 0, "", 0, 0, wa, 0);
        snap(q + ".ffn1", wa, F, 0);
        conv(wa, F, nullptr, 0, "ffn" + nn + ".2", "encoder.ffn_layers." + nn + ".conv_2.bias", K, Ce, 0, 0, 1, other[0], 0, "encoder.norm_layers_2." + nn, 0, 0, other[1], 0);
        snap(q + ".ln2", other[1], Ce, 0);
        float* t = h; h = other[1]; other[1] = t;
    }
    auto done = [&]() -> int {
        if (const cudaError_t err = e->snaps.finish()) return fail(SBK_ERR_CUDA, "sbk_textenc_forward: debug capture failed: %s", cudaGetErrorString(err));
        CU(cudaGetLastError());
        e->last_launches = n;
        return SBK_OK;
    };
    if (mel) {
        // x = term_proj(x * x_mask): no output mask (DiffVC/model/encoder.py:283)
        conv(h, Ce, nullptr, 0, "term_proj", "term_proj.bias", 1, c.n_feats, 1, 0, 0, nullptr, 0, "", 0, 0, mu_x, 1);
        snap("out", mu_x, c.n_feats, 1);
        return done();
    }
    // ---- x = x * mask; mu = proj_m(x) * mask; logw = DurationPredictor(x, mask)  (:278, :321-324, :83-93)
    conv(h, Ce, nullptr, 0, "proj_m", "proj_m.bias", 1, c.n_feats, 1, 0, 0, nullptr, 0, "", 0, 1, mu_x, 1);
    snap("mu", mu_x, c.n_feats, 1);
    conv(h, Ce, nullptr, 0, "dp.1", "proj_w.conv_1.bias", K, Fd, 1, 1, 0, nullptr, 0, "proj_w.norm_1", 0, 0, wa, 0);
    snap("dp.1", wa, Fd, 0);
    conv(wa, Fd, nullptr, 0, "dp.2", "proj_w.conv_2.bias", K, Fd, 1, 1, 0, nullptr, 0, "proj_w.norm_2", 0, 0, wb, 0);
    snap("dp.2", wb, Fd, 0);
    conv(wb, Fd, nullptr, 0, "dp.p", "proj_w.proj.bias", 1, 1, 1, 0, 0, nullptr, 0, "", 0, 1, logw, 1);
    snap("logw", logw, 1, 1);
    return done();
}

extern "C" int sbk_textenc_forward(sbk_textenc* e, const int64_t* x, const int64_t* x_lengths, const float* spk,
                                   float* mu_x, float* logw, float* x_mask, int B, int Tx, void* stream) {
    if (!e || !x || !x_lengths || !mu_x || !logw || !x_mask) return fail(SBK_ERR_ARG, "sbk_textenc_forward: null argument");
    if (e->cfg.kind != 0) return fail(SBK_ERR_ARG, "sbk_textenc_forward: this handle is a mel encoder, use sbk_melenc_forward");
    return te_forward(e, x, x_lengths, spk, nullptr, nullptr, mu_x, logw, x_mask, B, Tx, stream);
}

// MelEncoder.forward(x, x_mask) (DiffVC/model/encoder.py:279-284): x [B,n_feats,T], x_mask [B,1,T] -> out [B,n_feats,T]
extern "C" int sbk_melenc_forward(sbk_textenc* e, const float* x, const float* x_mask, float* out, int B, int T, void* stream) {
    if (!e || !x || !x_mask || !out) return fail(SBK_ERR_ARG, "sbk_melenc_forward: null argument");
    if (e->cfg.kind != 1) return fail(SBK_ERR_ARG, "sbk_melenc_forward: this handle is a text encoder, use sbk_textenc_forward");
    return te_forward(e, nullptr, nullptr, nullptr, x, x_mask, out, nullptr, nullptr, B, T, stream);
}

extern "C" int64_t sbk_textenc_last_launch_count(const sbk_textenc* e) { return e ? e->last_launches : 0; }

extern "C" int sbk_textenc_debug_capture(sbk_textenc* e, int on) {
    if (!e) return fail(SBK_ERR_ARG, "sbk_textenc_debug_capture: null handle");
    e->snaps.on = on != 0;
    return SBK_OK;
}
extern "C" int sbk_textenc_debug_num(const sbk_textenc* e) { return e ? (int)e->snaps.list.size() : 0; }
extern "C" const char* sbk_textenc_debug_name(const sbk_textenc* e, int i) {
    if (!e || i < 0 || i >= (int)e->snaps.list.size()) return nullptr;
    return e->snaps.list[i].name.c_str();
}
extern "C" int sbk_textenc_debug_op_layout(const sbk_textenc* e, const char* name) {
    const Snapshots::Snap* sn = e && name ? e->snaps.find(name) : nullptr;
    return sn ? sn->fmt : -1;
}
extern "C" int sbk_textenc_debug_read(sbk_textenc* e, const char* name, void* dst, int64_t* numel) {
    if (!e || !name) return fail(SBK_ERR_ARG, "sbk_textenc_debug_read: null argument");
    return e->snaps.read(name, dst, numel, e->cfg.device, "sbk_textenc_debug_read");
}
