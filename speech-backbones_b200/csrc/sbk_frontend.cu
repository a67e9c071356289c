// DiffVC's inference front end (DiffVC/inference.ipynb, cell 1): the log-mel analysis `get_mel` (without file decoding or
// resampling) and the post-processing `mel_spectral_subtraction` / `noise_median_smoothing`, per utterance in ragged batches.
//
// Log-mel launch plan (all asynchronous on the caller's stream):
//   1. k_fe_frames: per utterance, truncate to whole 256-sample hops (L_b' = (L_b / 256) * 256), reflect-pad 384 samples at
//      its own two edges and write the framed operand [B][1024/4][T][4] fp32 (frame f = padded samples 256f .. 256f + 1023;
//      the 1x1 wgmma conv's operand form, H = 1, W = T).  The waveform is read only below L_b'; frames from T_b = L_b' / 256
//      on are zeros.
//   2. k_conv_tc<G_PW> in FORM_X3: the windowed DFT as one GEMM, K = 1024 samples, N = the bins the filterbank reads as
//      interleaved (re, im) columns (hann[n] cos 2 pi k n / 1024, -hann[n] sin 2 pi k n / 1024), padded to the N tile.
//      fp32x3 only: the reference's STFT is an fp64 FFT stored as complex64, and a tf32 DFT's error (~1e-3 of the frame's
//      energy) would swamp every quiet bin of a loud frame.
//   3. k_fe_logmel: |X| = sqrt(re^2 + im^2 + 1e-9) (fp32, unfused, as NumPy evaluates it on complex64), the Slaney
//      filterbank as a sparse projection (each filter's contiguous run of nonzero bins, ascending), log(max(mel, 1e-5)),
//      planar [B][80][T]; frames from T_b on are written as 0.
// GEMM rows are independent and each row's accumulation order depends on the K loop only, so every row of a ragged batch is
// bit for bit its own B = 1 call.
//
// Spectral subtraction (k_fe_specsub): one CTA per utterance, on its first T_b frames, as the notebook's function is written.
#include "sbk_host.h"

#include <math.h>
#include <string.h>

#include <vector>

using namespace sbk;

namespace {

constexpr int kNfft = 1024, kHop = 256, kPad = 384, kSr = 22050, kMels = 80;
constexpr double kFmin = 0.0, kFmax = 8000.0;

// utterance b's whole-hop samples: its length clamped to [0, L], truncated to a multiple of the hop
__device__ __forceinline__ int fe_samples(const int64_t* lengths, long long b, int L) {
    long long n = lengths ? lengths[b] : L;
    n = n < 0 ? 0 : (n > L ? L : n);
    return (int)(n / kHop * kHop);
}

__global__ void k_fe_frames(const float* __restrict__ wav, const int64_t* __restrict__ lengths, float* __restrict__ fr, int B, int L,
                            int T) {
    const long long n = (long long)B * (kNfft / 4) * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long r = i / T;
        const int q = (int)(r % (kNfft / 4));
        const long long b = r / (kNfft / 4);
        const int Ls = fe_samples(lengths, b, L), Tb = Ls / kHop;
        // (Tb < 2: no valid reflection; the host refuses such lengths, the kernel writes zeros rather than read outside)
        if (Tb < 2 || t >= Tb) {
            reinterpret_cast<float4*>(fr)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const float* x = wav + b * L;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            int j = t * kHop + 4 * q + e - kPad;               // np.pad(mode='reflect'): the edge sample is not repeated
            j = j < 0 ? -j : (j >= Ls ? 2 * (Ls - 1) - j : j);
            v[e] = __ldg(x + j);
        }
        reinterpret_cast<float4*>(fr)[i] = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// spec: the GEMM's output [B][cout/4][T][4], bin k's (re, im) at columns 2k, 2k + 1
__global__ void k_fe_logmel(const float* __restrict__ spec, const int* __restrict__ mlo, const int* __restrict__ moff,
                            const float* __restrict__ mw, const int64_t* __restrict__ lengths, float* __restrict__ out, int B, int L,
                            int T, int ch4, float log_floor) {
    const long long n = (long long)B * kMels * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long r = i / T;
        const int m = (int)(r % kMels);
        const long long b = r / kMels;
        const int Tb = fe_samples(lengths, b, L) / kHop;
        if (Tb < 2 || t >= Tb) { out[i] = 0.f; continue; }
        const int j0 = __ldg(moff + m), j1 = __ldg(moff + m + 1), k0 = __ldg(mlo + m);
        float acc = 0.f;
        for (int j = j0; j < j1; ++j) {
            const int k = k0 + (j - j0);
            const float2 z = __ldg(reinterpret_cast<const float2*>(spec + ((b * ch4 + (k >> 1)) * T + t) * 4 + 2 * (k & 1)));
            const float p = __fadd_rn(__fadd_rn(__fmul_rn(z.x, z.x), __fmul_rn(z.y, z.y)), 1e-9f);
            acc = fmaf(__ldg(mw + j), sqrtf(p), acc);
        }
        out[i] = acc < 1e-5f ? log_floor : logf(acc);
    }
}

// mel_spectral_subtraction on utterance blockIdx.x's first T_b frames (C channels, planar [B][C][T]); e64: [B][T] fp64 workspace.
// smooth < 0: smoothing_window=None.
__global__ void __launch_bounds__(256) k_fe_specsub(const float* __restrict__ synth, const float* __restrict__ source,
                                                    const int64_t* __restrict__ lengths, float* __restrict__ out,
                                                    double* __restrict__ e64, int C, int T, float floor_, int sw, int smooth) {
    extern __shared__ float s_noise[];                     // [2][C]: the noise floor, then its smoothed copy
    __shared__ double s_e[256 / 32];
    __shared__ int s_i[256 / 32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    long long tl = lengths ? lengths[b] : T;
    const int Tb = (int)(tl < 1 ? 1 : (tl > T ? T : tl));
    const float* src = source + (long long)b * C * T;
    const float* syn = synth + (long long)b * C * T;
    double* col = e64 + (long long)b * T;
    // 1. per-frame energy sum_c exp(2 m) of the source, in fp64, channels in order
    for (int t = tid; t < Tb; t += blockDim.x) {
        double s = 0.0;
        for (int c = 0; c < C; ++c) s += exp(2.0 * (double)src[(long long)c * T + t]);
        col[t] = s;
    }
    __syncthreads();
    // 2. the quietest window: candidates i < T_b - sw scanned from energy_min = 1e5 with a strict '<' (the first minimum wins)
    double best = INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < Tb - sw; i += blockDim.x) {
        double e = 0.0;
        for (int j = 0; j < sw; ++j) e += col[i + j];
        if (e < best) { best = e; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const double oe = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (oe < best || (oe == best && oi < bi)) { best = oe; bi = oi; }
    }
    if (lane == 0) { s_e[warp] = best; s_i[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < (int)(blockDim.x / 32); ++w)
            if (s_e[w] < s_e[0] || (s_e[w] == s_e[0] && s_i[w] < s_i[0])) { s_e[0] = s_e[w]; s_i[0] = s_i[w]; }
        s_i[0] = s_e[0] < 100000.0 ? s_i[0] : 0;
    }
    __syncthreads();
    const int i_min = s_i[0];
    const int nw = Tb - i_min < sw ? Tb - i_min : sw;        // T_b <= sw: the window is the frames that exist
    // 3. per-channel noise floor: min over the window of exp(2 m) of the synthesised mel (fp32, as NumPy on float32)
    float* nz = s_noise;
    float* sm = s_noise + C;
    for (int c = tid; c < C; c += blockDim.x) {
        float v = INFINITY;
        for (int j = 0; j < nw; ++j) v = fminf(v, expf(2.f * syn[(long long)c * T + i_min + j]));
        nz[c] = v;
    }
    __syncthreads();
    // 4. noise_median_smoothing: y[i] = min(x_pad[i + w + 1], median(x_pad[i : i + 2w + 1])) over the edge-padded x, i.e.
    //    channel i + 1 (clamped to the last) against the median of channels i - w .. i + w (clamped): exact selection
    if (smooth >= 0) {
        const int w = smooth;
        for (int c = tid; c < C; c += blockDim.x) {
            auto xp = [&](int j) { j = j < 0 ? 0 : (j >= C ? C - 1 : j); return nz[j]; };
            float med = 0.f;
            for (int k = -w; k <= w; ++k) {
                const float v = xp(c + k);
                int lt = 0, le = 0;
                for (int q = -w; q <= w; ++q) { const float u = xp(c + q); lt += u < v; le += u <= v; }
                if (lt <= w && w < le) { med = v; break; }
            }
            sm[c] = fminf(xp(c + 1), med);
        }
        __syncthreads();
    } else {
        sm = nz;
    }
    // 5. log(sqrt(max(exp(2 m) - noise, floor * noise))) on every frame below T_b, exact zeros after it
    float* o = out + (long long)b * C * T;
    for (long long i = tid; i < (long long)C * T; i += blockDim.x) {
        const int t = (int)(i % T), c = (int)(i / T);
        if (t >= Tb) { o[i] = 0.f; continue; }
        const float nc = sm[c];
        const float d = __fsub_rn(expf(2.f * syn[i]), nc);
        o[i] = logf(sqrtf(fmaxf(d, __fmul_rn(floor_, nc))));
    }
}

// Slaney mel filterbank (librosa.filters.mel(22050, 1024, 80, 0, 8000), htk = False, norm = 1), in double
double hz_to_mel(double f) {
    const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return f >= min_log_hz ? min_log_mel + log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
    const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = log(6.4) / 27.0;
    return m >= min_log_mel ? min_log_hz * exp(logstep * (m - min_log_mel)) : f_sp * m;
}
std::vector<double> mel_basis() {
    const int nb = kNfft / 2 + 1;
    std::vector<double> mf(kMels + 2), w((size_t)kMels * nb, 0.0);
    const double m0 = hz_to_mel(kFmin), m1 = hz_to_mel(kFmax);
    for (int i = 0; i < kMels + 2; ++i) mf[i] = mel_to_hz(m0 + i * (m1 - m0) / (kMels + 1));
    for (int i = 0; i < kMels; ++i) {
        const double enorm = 2.0 / (mf[i + 2] - mf[i]);
        for (int k = 0; k < nb; ++k) {
            const double fk = k * ((double)kSr / 2 / (nb - 1));
            const double lower = -(mf[i] - fk) / (mf[i + 1] - mf[i]), upper = (mf[i + 2] - fk) / (mf[i + 2] - mf[i + 1]);
            const double v = fmax(0.0, fmin(lower, upper));
            w[(size_t)i * nb + k] = v * enorm;
        }
    }
    return w;
}

}  // namespace

struct sbk_frontend {
    sbk_frontend_config cfg;
    // filterbank, sparse: filter m's nonzero weights are mw[moff[m] .. moff[m + 1]) on bins mlo[m] ..
    std::vector<int> mlo, moff;
    std::vector<float> mw;
    int nbins = 0, cout = 0, nt = 0;           // bins the DFT computes (0 .. nbins - 1), its columns padded to the N tile
    BufMap dev;                                 // "dft" (weight image), "mlo", "moff", "mw"
    float* zero = nullptr;
    bool ready = false;
    Workspace ws;
    int64_t last_launches = 0;
};

namespace {

// The framed operand and the DFT's output of a (B, T) log-mel call; a spectral subtraction's [B][T] fp64 energies fit in
// the first.  Over a null-base arena only the size is computed.
size_t fe_carve(const sbk_frontend* h, int B, int T, Arena& ar, float** fr, float** spec) {
    float* a = (float*)ar.take((size_t)B * kNfft * T * sizeof(float));
    float* s = (float*)ar.take((size_t)B * h->cout * T * sizeof(float));
    if (fr) *fr = a;
    if (spec) *spec = s;
    return ar.bytes();
}

// the DFT weight image and the filterbank on the device, and the conv's zero page (first forward on the handle's device)
int fe_prepare(sbk_frontend* h) {
    if (h->ready) return SBK_OK;
    std::vector<float> w((size_t)h->cout * kNfft, 0.f);
    const double tau = 2.0 * M_PI / kNfft;
    for (int n = 0; n < kNfft; ++n) {
        const double hann = 0.5 - 0.5 * cos(tau * n);            // periodic Hann (get_window('hann', 1024, fftbins=True))
        for (int k = 0; k < h->nbins; ++k) {
            const double a = tau * (double)((long long)k * n % kNfft);
            w[(size_t)(2 * k) * kNfft + n] = (float)(hann * cos(a));
            w[(size_t)(2 * k + 1) * kNfft + n] = (float)(-hann * sin(a));
        }
    }
    std::vector<uint8_t> img(conv_tc_pack_image(w.data(), h->cout, kNfft, G_PW, FORM_X3, h->nt, nullptr));
    conv_tc_pack_image(w.data(), h->cout, kNfft, G_PW, FORM_X3, h->nt, img.data());
    TRY(upload(h->dev, "dft", img.size(), img.data()));
    TRY(upload(h->dev, "mlo", h->mlo.size() * sizeof(int), h->mlo.data()));
    TRY(upload(h->dev, "moff", h->moff.size() * sizeof(int), h->moff.data()));
    TRY(upload(h->dev, "mw", h->mw.size() * sizeof(float), h->mw.data()));
    if (!h->zero) { CU(cudaMalloc(&h->zero, 8192)); CU(cudaMemset(h->zero, 0, 8192)); }
    h->ready = true;
    return SBK_OK;
}

const float* fe_get(const sbk_frontend* h, const char* key) { return (const float*)h->dev.at(key).ptr; }

}  // namespace

extern "C" int sbk_frontend_create(const sbk_frontend_config* cfg, sbk_frontend** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_frontend_create: null argument");
    sbk_frontend* h = new sbk_frontend();
    h->cfg = *cfg;
    const int nb = kNfft / 2 + 1;
    const std::vector<double> basis = mel_basis();
    h->moff.push_back(0);
    for (int m = 0; m < kMels; ++m) {
        int lo = nb, hi = -1;
        for (int k = 0; k < nb; ++k)
            if (basis[(size_t)m * nb + k] != 0.0) { lo = lo < k ? lo : k; hi = k; }
        if (hi < lo) lo = hi = 0;                               // (an empty filter: one zero weight)
        h->mlo.push_back(lo);
        for (int k = lo; k <= hi; ++k) h->mw.push_back((float)basis[(size_t)m * nb + k]);
        h->moff.push_back((int)h->mw.size());
        h->nbins = h->nbins > hi + 1 ? h->nbins : hi + 1;
    }
    h->nt = conv_tc_ntile(G_PW, 128, FORM_X3);
    h->cout = (2 * h->nbins + h->nt - 1) / h->nt * h->nt;
    *out = h;
    return SBK_OK;
}

extern "C" void sbk_frontend_destroy(sbk_frontend* h) {
    if (!h) return;
    free_all(h->dev);
    if (h->zero) cudaFree(h->zero);
    delete h;
}

extern "C" int sbk_frontend_dft_bins(const sbk_frontend* h) { return h ? h->nbins : 0; }

extern "C" size_t sbk_frontend_workspace_bytes(const sbk_frontend* h, int B, int T) {
    if (!h || B <= 0 || T <= 0) return 0;
    Arena probe;
    return fe_carve(h, B, T, probe, nullptr, nullptr);
}

extern "C" int sbk_logmel_forward_lengths(sbk_frontend* h, const float* wav, const int64_t* lengths, float* out, int B, int L, int T,
                                          void* stream) {
    if (!h || !wav || !out) return fail(SBK_ERR_ARG, "sbk_logmel_forward: null argument");
    if (B <= 0 || L < 2 * kHop || T < 1 || T > L / kHop)
        return fail(SBK_ERR_ARG, "sbk_logmel_forward: need B >= 1, L >= %d samples and 1 <= T <= L / %d (got B=%d, L=%d, T=%d)", 2 * kHop,
                    kHop, B, L, T);
    CU(cudaSetDevice(h->cfg.device));
    TRY(fe_prepare(h));
    cudaStream_t s = (cudaStream_t)stream;
    const size_t need = sbk_frontend_workspace_bytes(h, B, T);
    if (h->ws.reserve(need)) return fail(SBK_ERR_CUDA, "out of memory: the log-mel workspace for (B=%d, T=%d) needs %zu bytes", B, T, need);
    Arena ar = h->ws.arena();
    float *fr, *spec;
    fe_carve(h, B, T, ar, &fr, &spec);
    int64_t n = 0;
    k_fe_frames<<<ew_grid((long long)B * (kNfft / 4) * T), 256, 0, s>>>(wav, lengths, fr, B, L, T); ++n;
    ConvTcParams p; memset(&p, 0, sizeof(p));
    p.geom = G_PW; p.form = FORM_X3; p.in0 = fr; p.c0 = kNfft; p.H = 1; p.W = T; p.B = B; p.Ho = 1; p.Wo = T;
    p.wpk = h->dev.at("dft").ptr; p.out = spec; p.Cout = h->cout; p.epi = EPI_PLAIN; p.zero_page = h->zero; p.nt = h->nt;
    const int k = launch_conv_tc(p, s);
    if (k < 0) return fail(SBK_ERR_CUDA, "sbk_logmel_forward: the DFT GEMM launch was refused (device attribute / geometry)");
    n += k;
    k_fe_logmel<<<ew_grid((long long)B * kMels * T), 256, 0, s>>>(spec, (const int*)fe_get(h, "mlo"), (const int*)fe_get(h, "moff"),
                                                                  fe_get(h, "mw"), lengths, out, B, L, T, h->cout / 4, (float)log(1e-5));
    ++n;
    CU(cudaGetLastError());
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_spectral_subtraction_lengths(sbk_frontend* h, const float* mel_synth, const float* mel_source, const int64_t* lengths,
                                                float* out, int B, int n_mels, int T, float spectral_floor, int silence_window,
                                                int smoothing_window, void* stream) {
    if (!h || !mel_synth || !mel_source || !out) return fail(SBK_ERR_ARG, "sbk_spectral_subtraction: null argument");
    if (B <= 0 || n_mels <= 0 || n_mels > 4096 || T <= 0)
        return fail(SBK_ERR_ARG, "sbk_spectral_subtraction: need B >= 1, 1 <= n_mels <= 4096, T >= 1 (got %d, %d, %d)", B, n_mels, T);
    if (silence_window < 1) return fail(SBK_ERR_ARG, "sbk_spectral_subtraction: silence_window must be >= 1 (got %d)", silence_window);
    if (smoothing_window < -1 || smoothing_window == 0)
        return fail(SBK_ERR_ARG, "sbk_spectral_subtraction: smoothing_window must be >= 1, or -1 for none (got %d)", smoothing_window);
    CU(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const size_t need = sbk_frontend_workspace_bytes(h, B, T);
    if (h->ws.reserve(need)) return fail(SBK_ERR_CUDA, "out of memory: the spectral subtraction workspace for (B=%d, T=%d) needs %zu bytes", B, T, need);
    Arena ar = h->ws.arena();
    float* fr;
    fe_carve(h, B, T, ar, &fr, nullptr);
    k_fe_specsub<<<B, 256, 2 * (size_t)n_mels * sizeof(float), s>>>(mel_synth, mel_source, lengths, out, (double*)fr, n_mels, T,
                                                                     spectral_floor, silence_window, smoothing_window);
    CU(cudaGetLastError());
    h->last_launches = 1;
    return SBK_OK;
}

extern "C" int64_t sbk_frontend_last_launch_count(const sbk_frontend* h) { return h ? h->last_launches : 0; }
