// HiFi-GAN generator (mel -> waveform), the step immediately after the sampler: Grad-TTS/hifi-gan/models.py:77-128 (Generator),
// :13-49 (ResBlock1) or :53-74 (ResBlock2, HiFi-GAN V3), called at Grad-TTS/inference.py:81.  SURVEY.md 8(f) rank 3.
//
// Mapping onto the sampler's wgmma kernels (sbk_conv_tc.cu), all activations fp32 [B][C/4][L][4] (the 2-D layout with H = 1):
//   * Conv1d(K in {3,5,7,11}, dilation d) -> k_conv_tc<G_C1K*>: one strip of 128 + 64 samples per channel chunk in shared memory
//                                            (128 + 128, G_C1K*W, for a launch whose halo (K-1)*d exceeds 64), tap t of the
//                                            wgmma A operand = descriptor start + t*d samples; bias, LeakyReLU and the ResBlock
//                                            residual (x + conv2(...), models.py:47; x + conv_d(...), :68) live in its epilogue,
//                                            which also writes lrelu(x) - the next conv's operand - so no activation pass exists;
//   * ConvTranspose1d(k = 2u, stride u)   -> ONE 1x1 GEMM (k_conv_tc<G_PW>) to k*Cout channels, Z[i][t][co] = sum_ci x[i][ci] w[ci][co][t],
//                                            then k_ct_fold adds the two taps that reach each output sample (o = u*i - p + t), the
//                                            bias and the LeakyReLU.  (A transposed conv with k = 2u is exactly a 2-tap overlap-add.)
//   * MRF mean (xs / num_kernels, :112)   -> k_mrf: (r0 + r1 + r2) / 3 and the next stage's LeakyReLU in one pass;
//   * conv_post (C -> 1, K = 7) + tanh    -> k_post on CUDA cores (224 MACs per sample).
// Precision (sbk_vocoder_set_precision), the same launches in every mode:
//   tf32 (default)  tf32 operands (weights rounded to nearest at pack time, activations truncated by the tensor core), fp32
//                   accumulation and fp32 everywhere else - the arithmetic PyTorch's own GPU convs use by default;
//   fp32x3 (and fp32)  x*w = x_hi*w_hi + one f16 correction MMA (sbk_internal.h: corr_chunk), chunked accumulation: the
//                   conv inputs are the tf32 mode's fp32 tensors, and the conv kernel derives the correction operand in
//                   shared memory;
//   bf16            bf16 weights, and the conv inputs (the LeakyReLU operands mel_in, SA, A0, A1, A2, Hb) stored as bf16
//                   [B][C/8][L][8]; the residual stream x (X0, X1, X2, R[j]), the GEMM output Z and conv_post's input stay fp32.
// conv_post, tanh, the folds and the MRF mean are fp32 in every mode.
// Ragged batches (sbk_vocoder_forward_lengths): each utterance's Conv1d strips, transposed-conv fold and conv_post end at its
// own length times the stage's samples per frame, as in a call on that utterance alone, and the Conv1d tiles past it are
// skipped (DESIGN.md 4.2.1).
#include "sbk_host.h"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

using namespace sbk;

int sbk::device_sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    return n;
}

namespace {

constexpr float kSlope = 0.1f;        // LRELU_SLOPE, models.py:10

// An activation operand (a conv input) in the mode's form.  The 4 channels v of element i = bc*L + l of a [B][C/4][L][4]
// tensor (bc = b*C/4 + channel chunk) go to
//   bf16 = 0: out[i] fp32 (tf32 and fp32x3);
//   bf16 = 1: half of the 16-byte chunk (b, c/8, l) of a bf16 [B][C/8][L][8] tensor (C/4 even), round to nearest even.
__device__ __forceinline__ void store_operand(float4 v, long long bc, long long l, long long L, void* out, int bf16) {
    if (bf16) {
        uint32_t lo, hi;
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(v.y), "f"(v.x));
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(v.w), "f"(v.z));
        reinterpret_cast<uint2*>(out)[((bc >> 1) * L + l) * 2 + (bc & 1)] = make_uint2(lo, hi);
    } else {
        reinterpret_cast<float4*>(out)[bc * L + l] = v;
    }
}

__device__ __forceinline__ float4 lrelu4(float4 v, float slope) {
    return make_float4(v.x > 0.f ? v.x : v.x * slope, v.y > 0.f ? v.y : v.y * slope, v.z > 0.f ? v.z : v.z * slope, v.w > 0.f ? v.w : v.w * slope);
}

// mel [B][F][T] (the reference's planar layout) -> the operand [B][F/4][T][4], or bf16 [B][F/8][T][8]
__global__ void k_voc_mel_in(const float* mel, void* out, int B, int F, int T, int bf16) {
    const long long n = (long long)B * (F / 4) * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long bc = i / T;
        const int ch = (int)(bc % (F / 4)); const long long b = bc / (F / 4);
        const float* src = mel + ((b * F + ch * 4) * T) + t;
        store_operand(make_float4(src[0], src[T], src[2 * (long long)T], src[3 * (long long)T]), bc, t, T, out, bf16);
    }
}

// ConvTranspose1d(k = 2u, stride u, padding u/2) overlap-add (models.py:108): output sample o = u*q + r receives tap
// t1 = (o + p) mod u of input i1 = (o + p) / u and tap t1 + u of input i1 - 1 (p = u/2).
//   z: [B][(2u*C)/4][Lin][4], channel index t*C + co;  x (raw): [B][C/4][Lin*u][4];  a = lrelu(x) in operand form (store_operand)
// A ragged batch (lengths, lmul = input samples per mel frame): input i1 exists only below utterance b's own edge Lin_b,
// as in a call on that utterance alone.  (i1 - 1 < Lin_b for every o < Lin_b * u; outputs past that edge are not read.)
__global__ void k_voc_ct_fold(const float* z, const float* bias, float* x, void* a, int B, int C, int Lin, int u, float slope, int bf16,
                              const int64_t* lengths, int lmul) {
    const int Lout = Lin * u, c4n = C / 4, p = u / 2;
    const long long n = (long long)B * c4n * Lout;
    const long long zc = (long long)Lin * 4;                       // floats between consecutive channel chunks of z
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(i % Lout);
        const long long bc = i / Lout;
        const int ch = (int)(bc % c4n); const long long b = bc / c4n;
        const int i1 = (o + p) / u, t1 = (o + p) - i1 * u;
        const float* zb = z + b * (long long)(2 * u * c4n) * zc;
        float4 v = __ldg(reinterpret_cast<const float4*>(bias) + ch);
        if (i1 < ragged_edge(lengths, b, Lin, lmul)) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(zb + ((long long)t1 * c4n + ch) * zc + (long long)i1 * 4));
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        if (i1 >= 1) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(zb + ((long long)(t1 + u) * c4n + ch) * zc + (long long)(i1 - 1) * 4));
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        reinterpret_cast<float4*>(x)[i] = v;
        store_operand(lrelu4(v, slope), bc, o, Lout, a, bf16);
    }
}

// Multi-receptive-field fusion (models.py:109-114): x = ((r0 + r1) + r2) / 3, written as the next consumer's operand lrelu(x)
// (store_operand over [B][C/4][L][4] chunks, i = bc*L + l; conv_post's input is plain fp32: bf16 = 0)
__global__ void k_voc_mrf(const float4* r0, const float4* r1, const float4* r2, void* a, long long n4, int L, float inv, float slope,
                          int bf16) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 p = __ldg(r0 + i), q = __ldg(r1 + i), r = __ldg(r2 + i);
        float4 v = make_float4(((p.x + q.x) + r.x) * inv, ((p.y + q.y) + r.y) * inv, ((p.z + q.z) + r.z) * inv, ((p.w + q.w) + r.w) * inv);
        const long long bc = bf16 ? i / L : 0;
        store_operand(lrelu4(v, slope), bc, bf16 ? i - bc * L : i, L, a, bf16);
    }
}

// conv_post (Conv1d C -> 1, K = 7, padding 3) + tanh (models.py:116-117) on a = lrelu(x, 0.01): [B][C/4][L][4] -> wav [B][1][L].
// A ragged batch (lengths, lmul = samples per mel frame): utterance b's signal ends at L_b, its taps past L_b read zero
// padding and its samples from L_b on are 0.
__global__ void __launch_bounds__(256) k_voc_post(const float* a, const float* w /*[C][7]*/, const float* bias, float* wav, int B, int C, int L,
                                                  const int64_t* lengths, int lmul) {
    extern __shared__ float s_w[];                       // [7][C]
    for (int i = threadIdx.x; i < 7 * C; i += blockDim.x) { const int t = i / C, c = i - t * C; s_w[i] = w[c * 7 + t]; }
    __syncthreads();
    const float bb = __ldg(bias);
    const int c4n = C / 4;
    const long long n = (long long)B * L;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int l = (int)(i % L); const long long b = i / L;
        const int Lb = ragged_edge(lengths, b, L, lmul);
        const float* ab = a + b * (long long)c4n * L * 4;
        float acc = bb;
#pragma unroll
        for (int t = 0; t < 7; ++t) {
            const int li = l + t - 3;
            if (li < 0 || li >= Lb) continue;
            for (int ch = 0; ch < c4n; ++ch) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(ab + ((long long)ch * L + li) * 4));
                const float* ww = s_w + t * C + ch * 4;
                acc = fmaf(v.x, ww[0], acc); acc = fmaf(v.y, ww[1], acc); acc = fmaf(v.z, ww[2], acc); acc = fmaf(v.w, ww[3], acc);
            }
        }
        wav[i] = l < Lb ? tanhf(acc) : 0.f;
    }
}

// the tensor-core form of each mode: fp32 and fp32x3 run the fp32x3 split, bf16 its bf16 operands, tf32 tf32 operands
bool prec_bf16(int precision) { return precision == SBK_PREC_BF16; }

}  // namespace

struct sbk_vocoder {
    sbk_vocoder_config_ex cfg;
    int precision = SBK_PREC_TF32;
    WeightSet w;                             // raw: reference layout (after remove_weight_norm); packed: tensor-core stage images
    float* zero = nullptr;
    Workspace ws;
    bool is_packed = false;
    int64_t last_launches = 0;
    // test hook (sbk_vocoder_debug_*): the last forward's intermediates; fmt 1 = fp32 [B][C/4][L][4] (wav: [B][1][L]),
    // 2 = bf16 [B][C/8][L][8]
    Snapshots snaps;
    int n_res() const { return cfg.n_kernels; }
    bool x3() const { return prec_runs_x3(precision); }
    bool bf16() const { return prec_bf16(precision); }
    int form() const { return x3() ? FORM_X3 : (bf16() ? FORM_BF16 : FORM_TF32); }
};

// the Conv1d geometry of a kernel size: the 64-sample-halo strip, or the 128-sample one when the launch's halo (K-1)*dil
// needs it (both read the weight image packed for the narrow geometry); -1 for an unsupported size
static int voc_geom(int k, int halo = 0) {
    const bool wide = halo > conv_tc_c1_halo(G_C1K3);
    switch (k) {
        case 3:  return wide ? G_C1K3W : G_C1K3;
        case 5:  return wide ? G_C1K5W : G_C1K5;
        case 7:  return wide ? G_C1K7W : G_C1K7;
        case 11: return wide ? G_C1K11W : G_C1K11;
        default: return -1;
    }
}

// dilations a ResBlock applies: ResBlock1 all three, ResBlock2 the first two (models.py:13-74)
static int voc_ndil(const sbk_vocoder_config_ex& c) { return c.resblock == 2 ? 2 : 3; }

extern "C" int sbk_vocoder_create_ex(const sbk_vocoder_config_ex* cfg, sbk_vocoder** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_vocoder_create: null argument");
    if (cfg->resblock != 1 && cfg->resblock != 2) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: resblock %d (HiFi-GAN defines ResBlock1 and ResBlock2)", cfg->resblock);
    if (cfg->n_ups < 1 || cfg->n_ups > 4 || cfg->n_kernels != 3) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: needs 1..4 upsample stages and 3 resblock kernels (got %d, %d)", cfg->n_ups, cfg->n_kernels);
    if (cfg->num_mels <= 0 || cfg->num_mels % 8 != 0) return fail(SBK_ERR_ARG, "sbk_vocoder_create: num_mels must be a multiple of 8 (one K stage), got %d", cfg->num_mels);
    int ch = cfg->upsample_initial_channel;
    if (ch % 64 != 0) return fail(SBK_ERR_ARG, "sbk_vocoder_create: upsample_initial_channel must be a multiple of 64");
    for (int i = 0; i < cfg->n_ups; ++i) {
        const int u = cfg->upsample_rates[i], k = cfg->upsample_kernel_sizes[i];
        if (k != 2 * u || u % 2 != 0) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d: ConvTranspose1d needs k = 2*stride and an even stride (got k=%d, u=%d)", i, k, u);
        if (ch % 32 != 0) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d input channels %d: need a multiple of 32", i, ch);
        ch /= 2;
        if (ch % 32 != 0) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d has %d channels; the Conv1d tiles need a multiple of 32 (HiFi-GAN V2's 16- and 8-channel stages are not supported)", i, ch);
    }
    const int halo_max = conv_tc_c1_halo(G_C1K3W);
    for (int j = 0; j < 3; ++j) {
        const int k = cfg->resblock_kernel_sizes[j];
        if (voc_geom(k) < 0) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: resblock kernel %d (supported: 3, 5, 7, 11)", k);
        for (int d = 0; d < voc_ndil(*cfg); ++d) {
            const int dil = cfg->resblock_dilations[j][d];
            if (dil < 1) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: resblock kernel %d: dilation %d", j, dil);
            if ((k - 1) * dil > halo_max) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: halo (k-1)*d = %d exceeds %d samples", (k - 1) * dil, halo_max);
        }
    }
    sbk_vocoder* v = new sbk_vocoder();
    v->cfg = *cfg;
    auto add = [&](const std::string& n, std::vector<int64_t> s) { v->w.add(n, std::move(s)); };
    const int c0 = cfg->upsample_initial_channel;
    add("conv_pre.weight", {c0, cfg->num_mels, 7}); add("conv_pre.bias", {c0});
    for (int i = 0; i < cfg->n_ups; ++i) {
        add("ups." + std::to_string(i) + ".weight", {c0 >> i, c0 >> (i + 1), cfg->upsample_kernel_sizes[i]});
        add("ups." + std::to_string(i) + ".bias", {c0 >> (i + 1)});
    }
    int n = 0;
    // ResBlock1: convs1.d, convs2.d (d < 3); ResBlock2: convs.d (d < 2)
    const std::vector<const char*> groups = cfg->resblock == 2 ? std::vector<const char*>{"convs"} : std::vector<const char*>{"convs1", "convs2"};
    for (int i = 0; i < cfg->n_ups; ++i) {
        const int c = c0 >> (i + 1);
        for (int j = 0; j < 3; ++j, ++n)
            for (const char* grp : groups)
                for (int d = 0; d < voc_ndil(*cfg); ++d) {
                    const std::string q = "resblocks." + std::to_string(n) + "." + grp + "." + std::to_string(d);
                    add(q + ".weight", {c, c, cfg->resblock_kernel_sizes[j]}); add(q + ".bias", {c});
                }
    }
    add("conv_post.weight", {1, c0 >> cfg->n_ups, 7}); add("conv_post.bias", {1});
    *out = v;
    return SBK_OK;
}

// The V1 entry point: a ResBlock1 generator with its documented 64-sample halo limit.
extern "C" int sbk_vocoder_create(const sbk_vocoder_config* cfg, sbk_vocoder** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_vocoder_create: null argument");
    sbk_vocoder_config_ex ex;
    memset(&ex, 0, sizeof(ex));
    ex.device = cfg->device; ex.num_mels = cfg->num_mels; ex.upsample_initial_channel = cfg->upsample_initial_channel;
    ex.n_ups = cfg->n_ups; ex.n_kernels = cfg->n_kernels; ex.resblock = 1;
    memcpy(ex.upsample_rates, cfg->upsample_rates, sizeof(ex.upsample_rates));
    memcpy(ex.upsample_kernel_sizes, cfg->upsample_kernel_sizes, sizeof(ex.upsample_kernel_sizes));
    memcpy(ex.resblock_kernel_sizes, cfg->resblock_kernel_sizes, sizeof(ex.resblock_kernel_sizes));
    memcpy(ex.resblock_dilations, cfg->resblock_dilations, sizeof(ex.resblock_dilations));
    for (int j = 0; j < 3; ++j)
        for (int d = 0; d < 3; ++d) {
            const int halo = (cfg->resblock_kernel_sizes[j] - 1) * cfg->resblock_dilations[j][d];
            if (halo > conv_tc_c1_halo(G_C1K3)) return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: halo (k-1)*d = %d exceeds 64 samples (sbk_vocoder_create_ex takes up to 128)", halo);
        }
    return sbk_vocoder_create_ex(&ex, out);
}

extern "C" void sbk_vocoder_destroy(sbk_vocoder* v) {
    if (!v) return;
    if (v->zero) cudaFree(v->zero);
    delete v;
}

// Host logic only (no device work): the mode's tiling rules, then the packed state is dropped.
extern "C" int sbk_vocoder_set_precision(sbk_vocoder* v, int32_t precision) {
    if (!v) return fail(SBK_ERR_ARG, "sbk_vocoder_set_precision: null handle");
    if (precision == SBK_PREC_F16)
        return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_set_precision: fp16 is a sampler mode; the vocoder has no fp16 kernels "
                                         "(use tf32, bf16 or fp32x3)");
    if (precision < SBK_PREC_FP32 || precision > SBK_PREC_FP32X3) return fail(SBK_ERR_ARG, "sbk_vocoder_set_precision: unknown precision %d", precision);
    if (prec_bf16(precision)) {
        // bf16 K stages hold 16 input channels (Conv1d) and 64 (GEMM, sbk_conv_tc.cu conv_tc_stage_channels).  Every stage
        // has a multiple of 32 channels (sbk_vocoder_create), so its GEMM reads a multiple of 64: only conv_pre can fail.
        const int c1 = conv_tc_stage_channels(G_C1K3, FORM_BF16);
        if (v->cfg.num_mels % c1 != 0)
            return fail(SBK_ERR_UNSUPPORTED, "sbk_vocoder_set_precision: bf16 needs num_mels to be a multiple of %d, got %d", c1, v->cfg.num_mels);
    }
    v->precision = precision;
    v->is_packed = false;
    return SBK_OK;
}

extern "C" int sbk_vocoder_num_weights(const sbk_vocoder* v) { return v ? v->w.count() : 0; }
extern "C" const char* sbk_vocoder_weight_name(const sbk_vocoder* v, int i) { return v ? v->w.name(i) : nullptr; }

extern "C" int sbk_vocoder_set_weight(sbk_vocoder* v, const char* name, const void* data, const int64_t* shape, int ndim) {
    if (!v || !name || !data || !shape) return fail(SBK_ERR_ARG, "sbk_vocoder_set_weight: null argument");
    TRY(v->w.set(name, data, shape, ndim, v->cfg.device, "sbk_vocoder_set_weight"));
    v->is_packed = false;
    return SBK_OK;
}

// logical [co][ci][taps] -> the conv kernel's per-stage shared-memory image in the handle's mode (conv_tc_pack_image: tf32
// RNA, bf16 RNE, or fp32x3 (w_hi, correction) stage pairs)
static int voc_pack(sbk_vocoder* v, const std::vector<float>& w, const std::string& key, int cout, int cin, int geom) {
    const int form = v->form(), NT = conv_tc_ntile(geom, cout, form), CPS = conv_tc_stage_channels(geom, form);
    if (cin % CPS != 0 || cout % NT != 0) return fail(SBK_ERR_UNSUPPORTED, "vocoder pack '%s': %d -> %d channels do not tile (K stage %d, N tile %d)", key.c_str(), cin, cout, CPS, NT);
    std::vector<uint8_t> img(conv_tc_pack_image(w.data(), cout, cin, geom, form, NT, nullptr));
    conv_tc_pack_image(w.data(), cout, cin, geom, form, NT, img.data());
    return upload(v->w.packed, key, img.size(), img.data());
}

extern "C" int sbk_vocoder_pack(sbk_vocoder* v) {
    if (!v) return fail(SBK_ERR_ARG, "sbk_vocoder_pack: null handle");
    TRY(v->w.require_all("sbk_vocoder_pack"));
    CU(cudaSetDevice(v->cfg.device));
    v->is_packed = false;
    for (auto& s : v->w.spec) {
        if (s.name.size() < 7 || s.name.compare(s.name.size() - 7, 7, ".weight") != 0 || s.name == "conv_post.weight") continue;
        std::vector<float> w;
        TRY(v->w.fetch(s.name, w));
        const std::string key = s.name.substr(0, s.name.size() - 7) + ".wtc";
        int rc;
        if (s.name.compare(0, 4, "ups.") == 0) {
            // ConvTranspose1d [ci][co][k] -> 1x1 GEMM to k*co channels: W'[t*co_n + co][ci]
            const int ci_n = (int)s.shape[0], co_n = (int)s.shape[1], k = (int)s.shape[2];
            std::vector<float> g((size_t)k * co_n * ci_n);
            for (int ci = 0; ci < ci_n; ++ci) for (int co = 0; co < co_n; ++co) for (int t = 0; t < k; ++t)
                g[((size_t)t * co_n + co) * ci_n + ci] = w[((size_t)ci * co_n + co) * k + t];
            rc = voc_pack(v, g, key, k * co_n, ci_n, G_PW);
        } else {
            rc = voc_pack(v, w, key, (int)s.shape[0], (int)s.shape[1], voc_geom((int)s.shape[2]));
        }
        if (rc != SBK_OK) return rc;
    }
    if (!v->zero) { CU(cudaMalloc(&v->zero, 8192)); CU(cudaMemset(v->zero, 0, 8192)); }
    v->is_packed = true;
    return SBK_OK;
}

namespace {

// The workspace of one (B, T) in the handle's mode: 11 activation buffers of the largest stage, the transposed-conv GEMM
// output and the re-laid-out mel.  SA, A0, A1, A2, Hb and the mel are conv inputs: bf16 in the bf16 mode, fp32 in the
// others.  Over a null-base arena only the size is computed.
struct VocBufs {
    void* melc; float* Z;
    void *SA, *A0, *A1, *A2, *Hb;
    float *X0, *X1, *X2, *R[3];
};

size_t voc_carve(const sbk_vocoder* v, int B, int T, Arena& ar, VocBufs* o) {
    const sbk_vocoder_config_ex& c = v->cfg;
    size_t big = 0, zmax = 0;
    { long long L = T; int ch = c.upsample_initial_channel; big = (size_t)B * ch * L;
      for (int i = 0; i < c.n_ups; ++i) { zmax = std::max<size_t>(zmax, (size_t)B * c.upsample_kernel_sizes[i] * (ch / 2) * L); L *= c.upsample_rates[i]; ch /= 2; big = std::max<size_t>(big, (size_t)B * ch * L); } }
    const size_t ob = v->bf16() ? 2 : 4;            // bytes per element of an operand tensor
    auto take = [&](size_t bytes) { return (char*)ar.take(bytes); };
    VocBufs b{};
    b.melc = take((size_t)B * c.num_mels * T * ob);
    b.Z = (float*)take(zmax * 4);
    // SA: the stage input lrelu(x) (conv_pre / MRF output);  X0|A0: the stage's x after the transposed conv and lrelu(x);
    // X1|A1, X2|A2: the running x of a ResBlock after its first / second dilation;  Hb: lrelu(conv1(.));  R[j]: ResBlock outputs
    b.SA = take(big * ob); b.X0 = (float*)take(big * 4); b.A0 = take(big * ob); b.X1 = (float*)take(big * 4); b.A1 = take(big * ob);
    b.X2 = (float*)take(big * 4); b.A2 = take(big * ob); b.Hb = take(big * ob);
    for (int j = 0; j < 3; ++j) b.R[j] = (float*)take(big * 4);
    if (o) *o = b;
    return ar.bytes();
}

}  // namespace

extern "C" size_t sbk_vocoder_workspace_bytes(const sbk_vocoder* v, int B, int T) {
    if (!v || B <= 0 || T <= 0) return 0;
    Arena probe;
    return voc_carve(v, B, T, probe, nullptr);
}

// lengths (device, nullable): each utterance's mel frames.  Every stage runs on the batch's T frames, except that the
// Conv1d strips, the transposed-conv fold and conv_post treat utterance b's signal as ending at its own length (clamped to
// [0, T]) times the stage's samples per frame, and the Conv1d tiles past that edge are skipped; the GEMMs, the mel re-layout
// and the MRF mean still compute the padded samples, which no valid output reads.
extern "C" int sbk_vocoder_forward_lengths(sbk_vocoder* v, const float* mel, const int64_t* lengths, float* wav, int B, int T, void* stream) {
    if (!v || !mel || !wav) return fail(SBK_ERR_ARG, "sbk_vocoder_forward: null argument");
    if (!v->is_packed) return fail(SBK_ERR_STATE, "sbk_vocoder_forward: weights not packed for the current precision (sbk_vocoder_set_weight for every key, then sbk_vocoder_pack)");
    if (B <= 0 || T <= 0) return fail(SBK_ERR_ARG, "sbk_vocoder_forward: B and T must be positive (got %d, %d)", B, T);
    CU(cudaSetDevice(v->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const sbk_vocoder_config_ex& c = v->cfg;
    const size_t need = sbk_vocoder_workspace_bytes(v, B, T);
    if (v->ws.reserve(need)) return fail(SBK_ERR_CUDA, "out of memory: the vocoder workspace for (B=%d, T=%d) needs %zu bytes", B, T, need);
    VocBufs wb;
    Arena ar = v->ws.arena();
    voc_carve(v, B, T, ar, &wb);
    const bool bf = v->bf16();
    const int ofmt = bf ? 2 : 1;                     // debug layout of the operand tensors
    void *melc = wb.melc, *SA = wb.SA, *A0 = wb.A0, *A1 = wb.A1, *A2 = wb.A2, *Hb = wb.Hb;
    float *Z = wb.Z, *X0 = wb.X0, *X1 = wb.X1, *X2 = wb.X2, **R = wb.R;
    int64_t n = 0;
    int rcl = 0;
    int mul = 1;                                     // samples per mel frame at the current stage
    // act_out: out = lrelu(conv + bias), the next conv's operand; otherwise out = conv + bias (+ addin) in fp32 and
    // a_out = lrelu(out) in operand form
    auto conv = [&](int geom, const std::string& pre, const void* in, int cin, int cout, int L, int dil, void* out, int act_out,
                    const float* addin, void* a_out) {
        ConvTcParams p; memset(&p, 0, sizeof(p));
        p.geom = geom; p.in0 = in; p.c0 = cin; p.H = 1; p.W = L; p.B = B; p.Ho = 1; p.Wo = L;
        p.wpk = v->w.get(pre + ".wtc"); p.bias = geom == G_PW ? nullptr : v->w.get(pre + ".bias"); p.out = (float*)out; p.Cout = cout; p.epi = EPI_PLAIN;
        p.zero_page = v->zero; p.dil = dil; p.pad = geom == G_PW ? 0 : (conv_tc_taps(geom) - 1) * dil / 2;
        p.slope = kSlope; p.act_out = act_out; p.addin = addin; p.act = a_out;
        p.form = v->form(); p.nt = conv_tc_ntile(geom, cout, p.form);      // as voc_pack packed it
        p.voc = 1;
        p.lengths = lengths; p.len_mul = mul;                               // (the GEMM ignores them: it computes every row)
        const int k = launch_conv_tc(p, s);
        if (k < 0) rcl = -1; else n += k;
    };
    // debug capture (the name is pre + suf, put together only when capturing)
    v->snaps.begin();
    auto snap = [&](const std::string& pre, const char* suf, const void* src, size_t numel, int fmt) {
        if (v->snaps.on) v->snaps.record(pre + suf, src, numel, fmt, s);
    };
    const size_t bn = (size_t)B;
    k_voc_mel_in<<<ew_grid((long long)B * (c.num_mels / 4) * T), 256, 0, s>>>(mel, melc, B, c.num_mels, T, bf ? 1 : 0); ++n;
    snap("mel_in", "", melc, bn * c.num_mels * T, ofmt);
    int ch = c.upsample_initial_channel; int L = T;
    // conv_pre + the first stage's leaky_relu (models.py:105,107)
    conv(G_C1K7, "conv_pre", melc, c.num_mels, ch, L, 1, SA, 1, nullptr, nullptr);
    snap("conv_pre", "", SA, bn * ch * L, ofmt);
    int rb = 0;
    const float* post_in = nullptr;
    for (int i = 0; i < c.n_ups; ++i) {
        const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i], co = ch / 2;
        const std::string up = "ups." + std::to_string(i);
        conv(G_PW, up, SA, ch, k * co, L, 1, Z, 0, nullptr, nullptr);    // Z[i][t*co + c] (models.py:108)
        snap(up, ".z", Z, bn * k * co * L, 1);
        const int Lo = L * u;
        k_voc_ct_fold<<<ew_grid((long long)B * (co / 4) * Lo), 256, 0, s>>>(Z, v->w.get(up + ".bias"), X0, A0, B, co, L, u, kSlope, bf ? 1 : 0,
                                                                       lengths, mul); ++n;
        snap(up, ".x", X0, bn * co * Lo, 1); snap(up, ".a", A0, bn * co * Lo, ofmt);
        ch = co; L = Lo; mul *= u;
        const size_t na = bn * ch * L;
        for (int j = 0; j < 3; ++j, ++rb) {
            const int k = c.resblock_kernel_sizes[j];
            const std::string rp = "resblocks." + std::to_string(rb);
            if (c.resblock == 2) {
                // per dilation d: x = conv_d(lrelu(x)) + x   (models.py:64-69); the second conv's x is the block output
                const int d0 = c.resblock_dilations[j][0], d1 = c.resblock_dilations[j][1];
                conv(voc_geom(k, (k - 1) * d0), rp + ".convs.0", A0, ch, ch, L, d0, X1, 0, X0, A1);
                snap(rp, ".convs.0.x", X1, na, 1); snap(rp, ".convs.0.a", A1, na, ofmt);
                conv(voc_geom(k, (k - 1) * d1), rp + ".convs.1", A1, ch, ch, L, d1, R[j], 0, X1, nullptr);
                snap(rp, ".convs.1.x", R[j], na, 1);
                continue;
            }
            const int geom = voc_geom(k);
            // per dilation d: xt = conv2(lrelu(conv1_d(lrelu(x)))); x = xt + x   (models.py:42-47); the dilated convs1 pick
            // their strip from the halo
            auto g1 = [&](int d) { return voc_geom(k, (k - 1) * c.resblock_dilations[j][d]); };
            conv(g1(0), rp + ".convs1.0", A0, ch, ch, L, c.resblock_dilations[j][0], Hb, 1, nullptr, nullptr);
            snap(rp, ".convs1.0", Hb, na, ofmt);
            conv(geom, rp + ".convs2.0", Hb, ch, ch, L, 1, X1, 0, X0, A1);
            snap(rp, ".convs2.0.x", X1, na, 1); snap(rp, ".convs2.0.a", A1, na, ofmt);
            conv(g1(1), rp + ".convs1.1", A1, ch, ch, L, c.resblock_dilations[j][1], Hb, 1, nullptr, nullptr);
            snap(rp, ".convs1.1", Hb, na, ofmt);
            conv(geom, rp + ".convs2.1", Hb, ch, ch, L, 1, X2, 0, X1, A2);
            snap(rp, ".convs2.1.x", X2, na, 1); snap(rp, ".convs2.1.a", A2, na, ofmt);
            conv(g1(2), rp + ".convs1.2", A2, ch, ch, L, c.resblock_dilations[j][2], Hb, 1, nullptr, nullptr);
            snap(rp, ".convs1.2", Hb, na, ofmt);
            conv(geom, rp + ".convs2.2", Hb, ch, ch, L, 1, R[j], 0, X2, nullptr);
            snap(rp, ".convs2.2.x", R[j], na, 1);
        }
        // x = xs / num_kernels, then the next consumer's leaky_relu: LRELU_SLOPE before the next ups, torch's default 0.01
        // before conv_post (models.py:107,114-115).  SA is free again: its only reader was this stage's GEMM.  conv_post's
        // input is fp32 in every mode and goes to X0 (its last reader, this stage's first convs2, is done).
        const long long n4 = (long long)B * (ch / 4) * L;
        const bool last = i + 1 == c.n_ups;
        void* mo = last ? (void*)X0 : SA;
        k_voc_mrf<<<ew_grid(n4), 256, 0, s>>>(reinterpret_cast<const float4*>(R[0]), reinterpret_cast<const float4*>(R[1]), reinterpret_cast<const float4*>(R[2]),
                                               mo, n4, L, 1.0f / 3.0f, last ? 0.01f : kSlope, (bf && !last) ? 1 : 0); ++n;
        if (v->snaps.on) snap("mrf." + std::to_string(i), "", mo, na, last ? 1 : ofmt);
        if (last) post_in = X0;
    }
    k_voc_post<<<ew_grid((long long)B * L), 256, 7 * ch * sizeof(float), s>>>(post_in, v->w.get("conv_post.weight"), v->w.get("conv_post.bias"), wav, B, ch, L,
                                                                           lengths, mul); ++n;
    snap("wav", "", wav, bn * L, 1);
    const cudaError_t snap_err = v->snaps.finish();
    if (rcl < 0) return fail(SBK_ERR_CUDA, "sbk_vocoder_forward: a tensor-core launch was refused (device attribute / geometry)");
    if (snap_err != cudaSuccess) return fail(SBK_ERR_CUDA, "sbk_vocoder_forward: debug capture failed: %s", cudaGetErrorString(snap_err));
    CU(cudaGetLastError());
    v->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_vocoder_forward(sbk_vocoder* v, const float* mel, float* wav, int B, int T, void* stream) {
    return sbk_vocoder_forward_lengths(v, mel, nullptr, wav, B, T, stream);
}

extern "C" int64_t sbk_vocoder_last_launch_count(const sbk_vocoder* v) { return v ? v->last_launches : 0; }

extern "C" int sbk_vocoder_debug_capture(sbk_vocoder* v, int on) {
    if (!v) return fail(SBK_ERR_ARG, "sbk_vocoder_debug_capture: null handle");
    v->snaps.on = on != 0;
    return SBK_OK;
}
extern "C" int sbk_vocoder_debug_num(const sbk_vocoder* v) { return v ? (int)v->snaps.list.size() : 0; }
extern "C" const char* sbk_vocoder_debug_name(const sbk_vocoder* v, int i) {
    if (!v || i < 0 || i >= (int)v->snaps.list.size()) return nullptr;
    return v->snaps.list[i].name.c_str();
}
extern "C" int sbk_vocoder_debug_op_layout(const sbk_vocoder* v, const char* name) {
    const Snapshots::Snap* sn = v && name ? v->snaps.find(name) : nullptr;
    return sn ? sn->fmt : -1;
}
extern "C" int sbk_vocoder_debug_read(sbk_vocoder* v, const char* name, float* dst, int64_t* numel) {
    if (!v || !name) return fail(SBK_ERR_ARG, "sbk_vocoder_debug_read: null argument");
    return v->snaps.read(name, dst, numel, v->cfg.device, "sbk_vocoder_debug_read");
}
