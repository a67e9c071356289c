// HiFi-GAN generator (mel -> waveform), the step immediately after the sampler: Grad-TTS/hifi-gan/models.py:77-128 (Generator),
// :13-49 (ResBlock1), called at Grad-TTS/inference.py:81.  SURVEY.md 8(f) rank 3.
//
// Mapping onto the sampler's wgmma kernels (sbk_conv_tc.cu), all activations fp32 [B][C/4][L][4] (the 2-D layout with H = 1):
//   * Conv1d(K in {3,7,11}, dilation d)   -> k_conv_tc<G_C1K*>: one strip of 128 + 64 samples per channel chunk in shared memory,
//                                            tap t of the wgmma A operand = descriptor start + t*d samples; bias, LeakyReLU and
//                                            the ResBlock residual (x + conv2(...), models.py:47) live in its epilogue, which
//                                            also writes lrelu(x) - the next conv's operand - so no activation pass exists;
//   * ConvTranspose1d(k = 2u, stride u)   -> ONE 1x1 GEMM (k_conv_tc<G_PW>) to k*Cout channels, Z[i][t][co] = sum_ci x[i][ci] w[ci][co][t],
//                                            then k_ct_fold adds the two taps that reach each output sample (o = u*i - p + t), the
//                                            bias and the LeakyReLU.  (A transposed conv with k = 2u is exactly a 2-tap overlap-add.)
//   * MRF mean (xs / num_kernels, :112)   -> k_mrf: (r0 + r1 + r2) / 3 and the next stage's LeakyReLU in one pass;
//   * conv_post (C -> 1, K = 7) + tanh    -> k_post on CUDA cores (224 MACs per sample).
// tf32 operands (weights rounded to nearest at pack time, activations truncated by the tensor core), fp32 accumulation and
// fp32 everywhere else - the arithmetic PyTorch's own GPU convs use by default.
#include "../../include/sbk.h"
#include "sbk_internal.h"

#include <math.h>
#include <stdarg.h>
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

int sbk_set_error(int code, const char* fmt, ...);     // sbk_api.cu: fills the thread-local error text

#define VCU(x)                                                                                              \
    do {                                                                                                    \
        cudaError_t e_ = (x);                                                                               \
        if (e_ != cudaSuccess)                                                                              \
            return sbk_set_error(SBK_ERR_CUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

namespace {

constexpr float kSlope = 0.1f;        // LRELU_SLOPE, models.py:10

// mel [B][F][T] (the reference's planar layout) -> [B][F/4][T][4]
__global__ void k_voc_mel_in(const float* mel, float* out, int B, int F, int T) {
    const long long n = (long long)B * (F / 4) * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long bc = i / T;
        const int ch = (int)(bc % (F / 4)); const long long b = bc / (F / 4);
        const float* src = mel + ((b * F + ch * 4) * T) + t;
        reinterpret_cast<float4*>(out)[i] = make_float4(src[0], src[T], src[2 * (long long)T], src[3 * (long long)T]);
    }
}

// ConvTranspose1d(k = 2u, stride u, padding u/2) overlap-add (models.py:108): output sample o = u*q + r receives tap
// t1 = (o + p) mod u of input i1 = (o + p) / u and tap t1 + u of input i1 - 1 (p = u/2).
//   z: [B][(2u*C)/4][Lin][4], channel index t*C + co;  x (raw) and a = lrelu(x): [B][C/4][Lin*u][4]
__global__ void k_voc_ct_fold(const float* z, const float* bias, float* x, float* a, int B, int C, int Lin, int u, float slope) {
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
        if (i1 < Lin) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(zb + ((long long)t1 * c4n + ch) * zc + (long long)i1 * 4));
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        if (i1 >= 1) {
            const float4 w = __ldg(reinterpret_cast<const float4*>(zb + ((long long)(t1 + u) * c4n + ch) * zc + (long long)(i1 - 1) * 4));
            v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
        }
        reinterpret_cast<float4*>(x)[i] = v;
        reinterpret_cast<float4*>(a)[i] = make_float4(v.x > 0.f ? v.x : v.x * slope, v.y > 0.f ? v.y : v.y * slope,
                                                      v.z > 0.f ? v.z : v.z * slope, v.w > 0.f ? v.w : v.w * slope);
    }
}

// Multi-receptive-field fusion (models.py:109-114): x = ((r0 + r1) + r2) / 3, written as the next consumer's operand lrelu(x)
__global__ void k_voc_mrf(const float4* r0, const float4* r1, const float4* r2, float4* a, long long n4, float inv, float slope) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 p = __ldg(r0 + i), q = __ldg(r1 + i), r = __ldg(r2 + i);
        float4 v = make_float4(((p.x + q.x) + r.x) * inv, ((p.y + q.y) + r.y) * inv, ((p.z + q.z) + r.z) * inv, ((p.w + q.w) + r.w) * inv);
        a[i] = make_float4(v.x > 0.f ? v.x : v.x * slope, v.y > 0.f ? v.y : v.y * slope, v.z > 0.f ? v.z : v.z * slope, v.w > 0.f ? v.w : v.w * slope);
    }
}

// conv_post (Conv1d C -> 1, K = 7, padding 3) + tanh (models.py:116-117) on a = lrelu(x, 0.01): [B][C/4][L][4] -> wav [B][1][L]
__global__ void __launch_bounds__(256) k_voc_post(const float* a, const float* w /*[C][7]*/, const float* bias, float* wav, int B, int C, int L) {
    extern __shared__ float s_w[];                       // [7][C]
    for (int i = threadIdx.x; i < 7 * C; i += blockDim.x) { const int t = i / C, c = i - t * C; s_w[i] = w[c * 7 + t]; }
    __syncthreads();
    const float bb = __ldg(bias);
    const int c4n = C / 4;
    const long long n = (long long)B * L;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int l = (int)(i % L); const long long b = i / L;
        const float* ab = a + b * (long long)c4n * L * 4;
        float acc = bb;
#pragma unroll
        for (int t = 0; t < 7; ++t) {
            const int li = l + t - 3;
            if (li < 0 || li >= L) continue;
            for (int ch = 0; ch < c4n; ++ch) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(ab + ((long long)ch * L + li) * 4));
                const float* ww = s_w + t * C + ch * 4;
                acc = fmaf(v.x, ww[0], acc); acc = fmaf(v.y, ww[1], acc); acc = fmaf(v.z, ww[2], acc); acc = fmaf(v.w, ww[3], acc);
            }
        }
        wav[i] = tanhf(acc);
    }
}

// grid-stride elementwise kernels: 256-thread blocks, at most 16 blocks per SM
int ew_grid(long long n) {
    const long long g = (n + 255) / 256, cap = 16LL * device_sm_count();
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

uint32_t f32_to_tf32_rna(float x) {
    uint32_t u; memcpy(&u, &x, 4);
    if ((u & 0x7F800000u) != 0x7F800000u) u += 0x1000u;
    return u & 0xFFFFE000u;
}

struct VWSpec { std::string name; std::vector<int64_t> shape; };

}  // namespace

struct sbk_vocoder {
    sbk_vocoder_config cfg;
    std::vector<VWSpec> spec;
    std::map<std::string, float*> raw;       // device copies, reference layout (after remove_weight_norm)
    std::map<std::string, float*> packed;    // tensor-core stage images
    float* zero = nullptr;
    void* mem = nullptr; size_t cap = 0;
    bool is_packed = false;
    int64_t last_launches = 0;
    int n_res() const { return cfg.n_kernels; }
};

static int voc_geom(int k) { return k == 3 ? G_C1K3 : (k == 7 ? G_C1K7 : (k == 11 ? G_C1K11 : -1)); }

extern "C" int sbk_vocoder_create(const sbk_vocoder_config* cfg, sbk_vocoder** out) {
    if (!cfg || !out) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_create: null argument");
    if (cfg->n_ups < 1 || cfg->n_ups > 4 || cfg->n_kernels != 3) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: needs 1..4 upsample stages and 3 resblock kernels (HiFi-GAN V1/V2 layout)");
    if (cfg->num_mels <= 0 || cfg->num_mels % 8 != 0) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_create: num_mels must be a multiple of 8 (one K stage), got %d", cfg->num_mels);
    int ch = cfg->upsample_initial_channel;
    if (ch % 64 != 0) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_create: upsample_initial_channel must be a multiple of 64");
    for (int i = 0; i < cfg->n_ups; ++i) {
        const int u = cfg->upsample_rates[i], k = cfg->upsample_kernel_sizes[i];
        if (k != 2 * u || u % 2 != 0) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d: ConvTranspose1d needs k = 2*stride and an even stride (got k=%d, u=%d)", i, k, u);
        if (ch % 32 != 0) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d input channels %d: need a multiple of 32", i, ch);
        ch /= 2;
        if (ch % 32 != 0) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: stage %d has %d channels; the tensor-core path needs multiples of 32 (HiFi-GAN V1)", i, ch);
    }
    for (int j = 0; j < 3; ++j) {
        if (voc_geom(cfg->resblock_kernel_sizes[j]) < 0) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: resblock kernel %d (supported: 3, 7, 11)", cfg->resblock_kernel_sizes[j]);
        for (int d = 0; d < 3; ++d) {
            const int dil = cfg->resblock_dilations[j][d];
            if (dil < 1 || (cfg->resblock_kernel_sizes[j] - 1) * dil > 64) return sbk_set_error(SBK_ERR_UNSUPPORTED, "sbk_vocoder_create: halo (k-1)*d = %d exceeds 64 samples", (cfg->resblock_kernel_sizes[j] - 1) * dil);
        }
    }
    sbk_vocoder* v = new sbk_vocoder();
    v->cfg = *cfg;
    auto add = [&](const std::string& n, std::vector<int64_t> s) { v->spec.push_back({n, s}); };
    const int c0 = cfg->upsample_initial_channel;
    add("conv_pre.weight", {c0, cfg->num_mels, 7}); add("conv_pre.bias", {c0});
    for (int i = 0; i < cfg->n_ups; ++i) {
        add("ups." + std::to_string(i) + ".weight", {c0 >> i, c0 >> (i + 1), cfg->upsample_kernel_sizes[i]});
        add("ups." + std::to_string(i) + ".bias", {c0 >> (i + 1)});
    }
    int n = 0;
    for (int i = 0; i < cfg->n_ups; ++i) {
        const int c = c0 >> (i + 1);
        for (int j = 0; j < 3; ++j, ++n)
            for (const char* grp : {"convs1", "convs2"})
                for (int d = 0; d < 3; ++d) {
                    const std::string q = "resblocks." + std::to_string(n) + "." + grp + "." + std::to_string(d);
                    add(q + ".weight", {c, c, cfg->resblock_kernel_sizes[j]}); add(q + ".bias", {c});
                }
    }
    add("conv_post.weight", {1, c0 >> cfg->n_ups, 7}); add("conv_post.bias", {1});
    *out = v;
    return SBK_OK;
}

extern "C" void sbk_vocoder_destroy(sbk_vocoder* v) {
    if (!v) return;
    for (auto& kv : v->raw) cudaFree(kv.second);
    for (auto& kv : v->packed) cudaFree(kv.second);
    if (v->zero) cudaFree(v->zero);
    if (v->mem) cudaFree(v->mem);
    delete v;
}

extern "C" int sbk_vocoder_num_weights(const sbk_vocoder* v) { return v ? (int)v->spec.size() : 0; }
extern "C" const char* sbk_vocoder_weight_name(const sbk_vocoder* v, int i) {
    if (!v || i < 0 || i >= (int)v->spec.size()) return nullptr;
    return v->spec[i].name.c_str();
}

extern "C" int sbk_vocoder_set_weight(sbk_vocoder* v, const char* name, const void* data, const int64_t* shape, int ndim) {
    if (!v || !name || !data || !shape) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_set_weight: null argument");
    const VWSpec* ws = nullptr;
    for (auto& s : v->spec) if (s.name == name) { ws = &s; break; }
    if (!ws) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_set_weight: unexpected key '%s' (strict)", name);
    if ((int)ws->shape.size() != ndim) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_set_weight: '%s' rank %d, expected %d", name, ndim, (int)ws->shape.size());
    size_t numel = 1;
    for (int i = 0; i < ndim; ++i) {
        if (ws->shape[i] != shape[i]) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_set_weight: '%s' dim %d is %lld, expected %lld", name, i, (long long)shape[i], (long long)ws->shape[i]);
        numel *= (size_t)shape[i];
    }
    VCU(cudaSetDevice(v->cfg.device));
    float*& dst = v->raw[name];
    if (!dst) VCU(cudaMalloc(&dst, numel * sizeof(float)));
    VCU(cudaMemcpy(dst, data, numel * sizeof(float), cudaMemcpyDefault));
    v->is_packed = false;
    return SBK_OK;
}

// logical [co][ci][taps] -> the conv kernel's per-stage shared-memory image [ntile][kstage][tap][16 B chunk][co % NT][4], tf32 (RNA)
static int voc_pack(sbk_vocoder* v, const std::vector<float>& w, const std::string& key, int cout, int cin, int geom) {
    const int taps = conv_tc_taps(geom), NT = conv_tc_ntile(geom, cout), CPS = conv_tc_stage_channels(geom, 0), KCHK = CPS / 4;
    if (cin % CPS != 0 || cout % NT != 0) return sbk_set_error(SBK_ERR_UNSUPPORTED, "vocoder pack '%s': %d -> %d channels do not tile (K stage %d, N tile %d)", key.c_str(), cin, cout, CPS, NT);
    const int ksteps = cin / CPS;
    std::vector<uint32_t> img((size_t)cout * cin * taps);
    for (int nt = 0; nt < cout / NT; ++nt) for (int ks = 0; ks < ksteps; ++ks) for (int tap = 0; tap < taps; ++tap)
        for (int k = 0; k < KCHK; ++k) for (int col = 0; col < NT; ++col) for (int e = 0; e < 4; ++e) {
            const int co = nt * NT + col, ci = ks * CPS + k * 4 + e;
            img[(((((size_t)nt * ksteps + ks) * taps + tap) * KCHK + k) * NT + col) * 4 + e] = f32_to_tf32_rna(w[((size_t)co * cin + ci) * taps + tap]);
        }
    float*& d = v->packed[key];
    if (!d) VCU(cudaMalloc(&d, img.size() * 4));
    VCU(cudaMemcpy(d, img.data(), img.size() * 4, cudaMemcpyHostToDevice));
    return SBK_OK;
}

extern "C" int sbk_vocoder_pack(sbk_vocoder* v) {
    if (!v) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_pack: null handle");
    for (auto& s : v->spec) if (!v->raw.count(s.name)) return sbk_set_error(SBK_ERR_STATE, "sbk_vocoder_pack: missing key '%s' (strict)", s.name.c_str());
    VCU(cudaSetDevice(v->cfg.device));
    for (auto& s : v->spec) {
        if (s.name.size() < 7 || s.name.compare(s.name.size() - 7, 7, ".weight") != 0 || s.name == "conv_post.weight") continue;
        size_t numel = 1; for (auto d : s.shape) numel *= (size_t)d;
        std::vector<float> w(numel);
        VCU(cudaMemcpy(w.data(), v->raw[s.name], numel * 4, cudaMemcpyDeviceToHost));
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
    if (!v->zero) { VCU(cudaMalloc(&v->zero, 8192)); VCU(cudaMemset(v->zero, 0, 8192)); }
    v->is_packed = true;
    return SBK_OK;
}

extern "C" size_t sbk_vocoder_workspace_bytes(const sbk_vocoder* v, int B, int T) {
    if (!v || B <= 0 || T <= 0) return 0;
    const sbk_vocoder_config& c = v->cfg;
    size_t big = 0, zmax = 0;
    long long L = T; int ch = c.upsample_initial_channel;
    big = (size_t)B * ch * L;
    for (int i = 0; i < c.n_ups; ++i) {
        zmax = std::max<size_t>(zmax, (size_t)B * c.upsample_kernel_sizes[i] * (ch / 2) * L);
        L *= c.upsample_rates[i]; ch /= 2;
        big = std::max<size_t>(big, (size_t)B * ch * L);
    }
    return (11 * big + zmax + (size_t)B * c.num_mels * T) * sizeof(float) + 16 * 256;
}

extern "C" int sbk_vocoder_forward(sbk_vocoder* v, const float* mel, float* wav, int B, int T, void* stream) {
    if (!v || !mel || !wav) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_forward: null argument");
    if (!v->is_packed) return sbk_set_error(SBK_ERR_STATE, "sbk_vocoder_forward: weights not packed (sbk_vocoder_set_weight for every key, then sbk_vocoder_pack)");
    if (B <= 0 || T <= 0) return sbk_set_error(SBK_ERR_ARG, "sbk_vocoder_forward: B and T must be positive (got %d, %d)", B, T);
    VCU(cudaSetDevice(v->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const sbk_vocoder_config& c = v->cfg;
    const size_t need = sbk_vocoder_workspace_bytes(v, B, T);
    if (need > v->cap) {
        if (v->mem) { cudaFree(v->mem); v->mem = nullptr; v->cap = 0; }
        const cudaError_t e = cudaMalloc(&v->mem, need);
        if (e != cudaSuccess) { v->mem = nullptr; cudaGetLastError(); return sbk_set_error(SBK_ERR_CUDA, "out of memory: the vocoder workspace for (B=%d, T=%d) needs %zu bytes", B, T, need); }
        v->cap = need;
    }
    // ---- carve: 10 activation buffers of the largest stage + the transposed-conv GEMM output + the re-laid-out mel
    size_t big = 0, zmax = 0;
    { long long L = T; int ch = c.upsample_initial_channel; big = (size_t)B * ch * L;
      for (int i = 0; i < c.n_ups; ++i) { zmax = std::max<size_t>(zmax, (size_t)B * c.upsample_kernel_sizes[i] * (ch / 2) * L); L *= c.upsample_rates[i]; ch /= 2; big = std::max<size_t>(big, (size_t)B * ch * L); } }
    char* base = (char*)v->mem; size_t off = 0;
    auto take = [&](size_t floats) { off = (off + 255) & ~size_t(255); float* r = (float*)(base + off); off += floats * sizeof(float); return r; };
    float* melc = take((size_t)B * c.num_mels * T);
    float* Z = take(zmax);
    // SA: the stage input lrelu(x) (conv_pre / MRF output);  X0|A0: the stage's x after the transposed conv and lrelu(x);
    // X1|A1, X2|A2: the running x of a ResBlock after its first / second dilation;  Hb: lrelu(conv1(.));  R[j]: ResBlock outputs
    float *SA = take(big), *X0 = take(big), *A0 = take(big), *X1 = take(big), *A1 = take(big), *X2 = take(big), *A2 = take(big), *Hb = take(big);
    float* R[3] = {take(big), take(big), take(big)};
    auto W = [&](const std::string& k) -> const float* { auto it = v->packed.find(k); if (it != v->packed.end()) return it->second; auto i2 = v->raw.find(k); return i2 != v->raw.end() ? i2->second : nullptr; };
    int64_t n = 0;
    int rcl = 0;
    auto conv = [&](int geom, const std::string& pre, const float* in, int cin, int cout, int L, int dil, float* out, int act_out,
                    const float* addin, float* out2) {
        ConvTcParams p; memset(&p, 0, sizeof(p));
        p.geom = geom; p.in0 = in; p.c0 = cin; p.H = 1; p.W = L; p.B = B; p.Ho = 1; p.Wo = L;
        p.wpk = W(pre + ".wtc"); p.bias = geom == G_PW ? nullptr : W(pre + ".bias"); p.out = out; p.Cout = cout; p.epi = EPI_PLAIN;
        p.zero_page = v->zero; p.dil = dil; p.pad = geom == G_PW ? 0 : (conv_tc_taps(geom) - 1) * dil / 2;
        p.slope = kSlope; p.act_out = act_out; p.addin = addin; p.out_lo = out2; p.act_out2 = out2 ? 1 : 0;
        const int k = launch_conv_tc(p, s);
        if (k < 0) rcl = -1; else n += k;
    };
    k_voc_mel_in<<<ew_grid((long long)B * (c.num_mels / 4) * T), 256, 0, s>>>(mel, melc, B, c.num_mels, T); ++n;
    int ch = c.upsample_initial_channel; int L = T;
    // conv_pre + the first stage's leaky_relu (models.py:105,107)
    conv(G_C1K7, "conv_pre", melc, c.num_mels, ch, L, 1, SA, 1, nullptr, nullptr);
    int rb = 0;
    for (int i = 0; i < c.n_ups; ++i) {
        const int u = c.upsample_rates[i], k = c.upsample_kernel_sizes[i], co = ch / 2;
        const std::string up = "ups." + std::to_string(i);
        conv(G_PW, up, SA, ch, k * co, L, 1, Z, 0, nullptr, nullptr);                           // Z[i][t*co + c] (models.py:108)
        const int Lo = L * u;
        k_voc_ct_fold<<<ew_grid((long long)B * (co / 4) * Lo), 256, 0, s>>>(Z, W(up + ".bias"), X0, A0, B, co, L, u, kSlope); ++n;
        ch = co; L = Lo;
        for (int j = 0; j < 3; ++j, ++rb) {
            const int geom = voc_geom(c.resblock_kernel_sizes[j]);
            const std::string rp = "resblocks." + std::to_string(rb);
            // per dilation d: xt = conv2(lrelu(conv1_d(lrelu(x)))); x = xt + x   (models.py:42-47)
            conv(geom, rp + ".convs1.0", A0, ch, ch, L, c.resblock_dilations[j][0], Hb, 1, nullptr, nullptr);
            conv(geom, rp + ".convs2.0", Hb, ch, ch, L, 1, X1, 0, X0, A1);
            conv(geom, rp + ".convs1.1", A1, ch, ch, L, c.resblock_dilations[j][1], Hb, 1, nullptr, nullptr);
            conv(geom, rp + ".convs2.1", Hb, ch, ch, L, 1, X2, 0, X1, A2);
            conv(geom, rp + ".convs1.2", A2, ch, ch, L, c.resblock_dilations[j][2], Hb, 1, nullptr, nullptr);
            conv(geom, rp + ".convs2.2", Hb, ch, ch, L, 1, R[j], 0, X2, nullptr);
        }
        // x = xs / num_kernels, then the next consumer's leaky_relu: LRELU_SLOPE before the next ups, torch's default 0.01
        // before conv_post (models.py:107,114-115).  SA is free again: its only reader was this stage's GEMM.
        const long long n4 = (long long)B * (ch / 4) * L;
        k_voc_mrf<<<ew_grid(n4), 256, 0, s>>>(reinterpret_cast<const float4*>(R[0]), reinterpret_cast<const float4*>(R[1]), reinterpret_cast<const float4*>(R[2]),
                                               reinterpret_cast<float4*>(SA), n4, 1.0f / 3.0f, i + 1 < c.n_ups ? kSlope : 0.01f); ++n;
    }
    k_voc_post<<<ew_grid((long long)B * L), 256, 7 * ch * sizeof(float), s>>>(SA, W("conv_post.weight"), W("conv_post.bias"), wav, B, ch, L); ++n;
    if (rcl < 0) return sbk_set_error(SBK_ERR_CUDA, "sbk_vocoder_forward: a tensor-core launch was refused (device attribute / geometry)");
    VCU(cudaGetLastError());
    v->last_launches = n;
    return SBK_OK;
}

extern "C" int64_t sbk_vocoder_last_launch_count(const sbk_vocoder* v) { return v ? v->last_launches : 0; }
