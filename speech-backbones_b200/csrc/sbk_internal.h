// Internal declarations shared by the kernel translation units and the host-side planner.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace sbk {

constexpr int kGroups = 8;        // GroupNorm groups (Grad-TTS/model/diffusion.py:50)
constexpr int kHeads = 4;         // LinearAttention heads (:83)
constexpr int kDimHead = 32;
constexpr int kAttnHidden = 128;  // heads * dim_head
constexpr int kKvPartFloats = 32 + 32 + 32 * 32;   // per (tile, head): max[32], sum[32], S[32][32]

// G_C1K*: Conv1d with K taps and a runtime dilation over [B][1][C/4][L][4] tensors (the HiFi-GAN vocoder, sbk_vocoder.cu);
// the strip of a G_C1K*W geometry carries a halo (K-1)*dil of up to 128 samples instead of 64 (conv_tc_c1_halo)
// G_C7: 7x7 conv, pad 3, stride 1 (DiffVC's PostNet Block, sbk_postnet.cu): tf32 operands or fp32x3, EPI_PLAIN output
enum Geom { G_PW = 0, G_C3 = 1, G_DOWN = 2, G_UP = 3, G_C1K3 = 4, G_C1K7 = 5, G_C1K11 = 6, G_C7 = 7, G_C1K5 = 8,
            G_C1K3W = 9, G_C1K5W = 10, G_C1K7W = 11, G_C1K11W = 12 };
__host__ __device__ constexpr bool geom_c1_wide(int g) { return g >= G_C1K3W && g <= G_C1K11W; }
__host__ __device__ constexpr bool geom_is_c1(int g) { return (g >= G_C1K3 && g <= G_C1K11) || g == G_C1K5 || geom_c1_wide(g); }
// the largest halo (K-1)*dil, in samples, that a Conv1d geometry's strip carries
__host__ __device__ constexpr int conv_tc_c1_halo(int g) { return geom_c1_wide(g) ? 128 : 64; }
enum Pro { PRO_NONE = 0, PRO_MASK = 1, PRO_GN = 2 };
enum Epi { EPI_PLAIN = 0, EPI_RES = 1, EPI_KV = 2 };

// GroupNorm statistics of one conv output: per (sample, group) {sum, sum of squares} in fp64.
struct GnRef {
    const double* stats;   // [B][8][2]
    const float* gamma;    // [C]
    const float* beta;     // [C]
    float inv_count;       // 1 / ((C/8) * H * W)
};

// Implicit-GEMM convolution over NHWC fp32 activations.
//   out[b][m][co] = epilogue( sum_{tap, ci} prologue(in[b][pix(m,tap)][ci]) * w[tap][ci][co] )
struct IgemmParams {
    int geom;
    // input(s): channel concat of in0 (c0 channels) and in1 (c1 channels, may be 0)
    const float* in0; const float* in1; int c0, c1;
    int Hin, Win, Hout, Wout;
    int B;
    const float* w; long long w_bstride;          // packed [ntaps][Cin][Cout] (+ optional per-sample stride)
    const float* bias;                            // [Cout] or nullptr
    float* out; int Cout;
    // prologue
    int pro;
    const float* mask; int T; int in_lvl;         // mask[b*T + (wi << in_lvl)]
    GnRef pgn;                                    // PRO_GN: statistics of in0
    const float* tb; int tb_stride; int tb_per_sample; const int* step;   // PRO_GN: + time projection row
    // epilogue
    int epi;
    double* ostats;                               // EPI_PLAIN: accumulate GN statistics of `out` (nullable)
    const float* rraw; GnRef rgn; int out_lvl;    // EPI_RES: out = acc + bias + Mish(GN(rraw))*mask
    float* kv_part;                               // EPI_KV: [B][mtiles][4][kKvPartFloats]
};

// Layout and number form of the U-Net's activation tensors, one per precision mode (GnActParams / ResFinalParams::form),
// and, in its tensor-core values, the operand form of a wgmma conv (ConvTcParams::form).
// Raw conv outputs (the GroupNorm inputs) are fp32 in every form: NHWC for FORM_NHWC, else [B][H][C/4][W][4].
enum Form {
    FORM_NHWC = 0,              // fp32 CUDA-core mode: NHWC fp32 [B][H][W][C], exact Mish
    FORM_TF32 = 1,              // fp32 [B][H][C/4][W][4]; the Block activation is rounded to tf32 (cvt.rna), fast Mish
    FORM_X3 = 2,                // fp32 [B][H][C/4][W][4], exact Mish; the convs derive the correction operand (corr_chunk)
    FORM_BF16 = 3,              // bf16 [B][H][C/8][W][8], fast Mish
};

// Tensor-core (wgmma) convolution (sbk_conv_tc.cu).  Inputs are operand-form tensors: already masked / activated, so the
// kernel's A path is a pure copy.  geom = G_C3 (3x3, pad 1) or G_PW (1x1 over the flattened image).
struct ConvTcParams {
    int geom;
    int form;                                       // operand form: FORM_TF32 | FORM_X3 | FORM_BF16
    const void* in0; const void* in1; int c0, c1;   // channel concat of two operand tensors: fp32 [B][H][C/4][W][4], or bf16
                                                    // [B][H][C/8][W][8] in FORM_BF16 (16-byte channel chunks either way)
    int H, W, B;                                    // input grid
    int Ho, Wo;                                     // output grid (G_DOWN: ~H/2 x W/2, G_UP: 2H x 2W; else = H, W)
    const void* wpk; long long w_bstride_bytes;     // weight image conv_tc_pack_image(.., nt, ..) (+ per-sample stride)
    const float* bias; long long bias_bstride;      // per-sample bias stride, 0 in every engine.  Kept: dropping the term
                                                    // reschedules every conv kernel, and bench.py's fp32x3 rate fell 0.4 %
                                                    // without it (H100 80GB HBM3, 700 W)
    float* out; int Cout;                           // FORM_BF16: G_C3 still writes fp32 raw [C/4] (GroupNorm input); the other
                                                    // geometries write bf16 operand tensors [C/8] through this pointer
    int epi;                                        // EPI_PLAIN | EPI_RES | EPI_KV
    double* ostats;                                 // EPI_PLAIN: GroupNorm statistics of the raw output (nullable)
    const float* mask; int T; int lvl; int out_mask;   // out_mask: multiply the stored output by mask[b][wo << lvl]
    const float* rraw; GnRef rgn;                   // EPI_RES: out = acc + bias + Mish(GN(rraw))*mask
    float* kv_part;                                 // EPI_KV: [B][ceil(HW/attn_kv_tile_pixels())][4][kKvPartFloats]
    const float* addin;                             // EPI_PLAIN: out += addin (same shape/layout/dtype as out): residual added in fp32
    const float* zero_page;                         // >= 4 KB of zeros in global memory (out-of-image parts of A tiles; the
                                                    // longest run is a wide Conv1d strip row, 256 samples x 16 B)
    int nt;                                         // N tile: the width the weights were packed with (conv_tc_ntile, or 64 for
                                                    // the U-Net's second 3x3 image, used when 128-wide tiles cannot fill the GPU)
    int rows;                                       // G_C3: output rows per tile, 1 (0 = 1) or 2; 2 runs 64-wide N tiles (nt = 64)
    // Conv1d geometries: dilation and left padding ((K-1)*dil/2) in samples; output activation LeakyReLU(slope) on `out`
    // (act_out) and/or the second output `act`
    int dil, pad; float slope; int act_out;
    // fp32-class mode (FORM_X3): operands are plain fp32; the tensor core reads the top 19 bits of x (= x_hi) by itself and
    // the kernel derives each A tile's correction chunks (corr_chunk below) in shared memory.  Weights are packed as (w_hi,
    // correction) stage pairs and each K stage is issued twice into the same fp32 register accumulator: the f16 correction
    // MMAs (x_lo*w + x*w_lo) first, then the tf32 main MMAs (x_hi*w_hi).
    // The vocoder's output forms (Conv1d geometries, and the transposed convs' 1x1 GEMM when voc = 1).  The output dtype is
    // per output, not per mode: an activated output (act_out) is the next conv's operand and takes the mode's operand form
    // (bf16 mode: bf16 [B][C/8][L][8]); every other output (the residual stream x, the GEMM output Z) stays fp32, with a
    // fp32 addin.
    int voc;
    void* act;                                      // Conv1d: second output lrelu(out) in operand form (fp32, bf16 in bf16 mode)
};

// ---- the wgmma conv's weight image: per N tile and K stage exactly the stage's shared-memory image --------------------
//   [ntile][kstage][main | correction][tap][16-byte chunk][co % nt][e]
// A K stage holds `taps` taps (7x7: the 7 of one kernel row) x `kch` 16-byte chunks of input channels, e = 4 tf32 elements
// per chunk (8 bf16).  FORM_X3 streams a (main, correction) stage pair per K stage: the main stage holds w_hi = tf32(w)
// (RNA), the correction stage per chunk the 8 fp16 {w[c0..c3], (w - w_hi)[c0..c3] * 2^12} that pair with the
// activations' corr_chunk in one f16 MMA.  The other forms have no correction stage.
struct ConvTcWImg { int form, nt, ksteps, taps, kch; };        // ksteps: K stages per N tile

__host__ __device__ constexpr int form_epc(int form) { return form == FORM_BF16 ? 8 : 4; }      // elements per 16-byte chunk
__host__ __device__ constexpr int conv_tc_taps(int geom) {
    return geom == G_PW ? 1 : geom == G_UP ? 16 : geom == G_C1K3 || geom == G_C1K3W ? 3 : geom == G_C1K5 || geom == G_C1K5W ? 5
         : geom == G_C1K7 || geom == G_C1K7W ? 7 : geom == G_C1K11 || geom == G_C1K11W ? 11 : geom == G_C7 ? 49 : 9;
}
__host__ __device__ constexpr int conv_tc_stage_rows(int geom) { return geom == G_C7 ? 7 : 1; }  // weight stages per K step
__host__ __device__ constexpr int conv_tc_kch(int geom) { return geom == G_PW ? 8 : 2; }         // 16-byte chunks per stage
__host__ __device__ constexpr int conv_tc_stage_channels(int geom, int form) { return conv_tc_kch(geom) * form_epc(form); }
__host__ __device__ inline ConvTcWImg conv_tc_wimg(int geom, int form, int nt, int cin) {
    const int rows = conv_tc_stage_rows(geom);
    return {form, nt, cin / conv_tc_stage_channels(geom, form) * rows, conv_tc_taps(geom) / rows, conv_tc_kch(geom)};
}
// elements of one (main or correction) stage
__host__ __device__ inline size_t conv_tc_wimg_stage(const ConvTcWImg& g) { return (size_t)g.taps * g.kch * g.nt * form_epc(g.form); }
// index of element e of chunk ch of output channel co at tap `tap` of K stage ks, in elements of the main stage (4 bytes,
// bf16: 2); corr = 1: the same chunk's place in the correction stage, in 4-byte units
__host__ __device__ inline size_t conv_tc_wimg_index(const ConvTcWImg& g, int co, int ks, int tap, int ch, int e, int corr = 0) {
    return (((size_t)(co / g.nt) * g.ksteps + ks) * (g.form == FORM_X3 ? 2 : 1) + corr) * conv_tc_wimg_stage(g) +
           (((size_t)tap * g.kch + ch) * g.nt + co % g.nt) * form_epc(g.form) + e;
}
__host__ __device__ inline size_t conv_tc_wimg_bytes(const ConvTcWImg& g, int cout) {
    return (size_t)(cout / g.nt) * g.ksteps * (g.form == FORM_X3 ? 2 : 1) * conv_tc_wimg_stage(g) * (g.form == FORM_BF16 ? 2 : 4);
}

// Block activation between the two convs of a ResnetBlock, written once in operand form (diffusion.py:57,76):
//   act = mask ? Mish(GN(raw)) + tproj : 0        (tensor-core forms only: the fp32 mode fuses it into the next conv)
struct GnActParams {
    const float* raw; GnRef gn; const float* tb; int tb_stride; int tb_per_sample; const int* step;
    const float* mask; int T; int lvl;
    float* out; int B, H, W, C;
    int form;                   // FORM_TF32 | FORM_X3 | FORM_BF16
};

struct FirstConvParams {        // Block.conv of downs.0.0.block1 on the planar stack([mu, xt(, s)]) * mask
    const float* mu; const float* xt; const float* spk_s;   // [B][H][T], [B][H][T], [B][H] or nullptr
    const float* mask;          // [B][T]
    const float* w;             // packed [cin*9 + r*3 + s][64]
    const float* bias;
    float* out; double* ostats; // [B][H][T][C] (or [B][H][C/4][T][4] when chw4), [B][8][2]
    int B, H, T, cin, C;
    int chw4;
    // DiffVC: the 128 conditioning channels are spatially constant, so they act as ONE extra input channel whose
    // value is the mask and whose weights are per (row, sample): w_extra[(row*B + b)][9][C] (row = *step or 0)
    const float* w_extra; const int* step; int extra_per_sample_row;
};

struct ResFinalParams {         // out = Mish(GN(h2raw))*mask + res(x*mask)
    const float* h2raw; GnRef gn;
    const float* x;             // identity residual source (NHWC, same C) or nullptr for the planar first block
    const float* mu; const float* xt; const float* spk_s;   // planar inputs for downs.0.0.res_conv
    const float* wres; const float* bres; int cin;          // [cin][C], [C]
    const float* r_extra; const int* step; int extra_per_sample_row;   // DiffVC: + mask * r_extra[(row*B + b)][C]
    const float* mask; int T; int lvl;
    float* out;
    int B, H, W, C;
    int out_mask;               // planar first block in a tensor-core form: store out*mask (operand form for the next conv)
    int form;                   // layout and number form of x and out (enum Form)
};

struct AttnCtxParams {          // merge per-tile softmax partials -> normalised context [B][4][32][32]
    const float* kv_part; int mtiles; float* ctx; int B;
};

struct AttnMixParams {          // A_b = I + g * Wout * blockdiag(ctx^T) * Wq ; packed as [ci][co]; bias' = g*bout
    const float* ctx;           // [B][4][32][32]
    const float* wq;            // [128][C]   (rows 0..127 of to_qkv)
    const float* wout;          // [C][128]
    const float* bout;          // [C]
    const float* g;             // [1]
    float* w_eff;               // [B][C(ci)][C(co)]
    float* b_eff;               // [C]
    int B, C;
    int nt;                     // != 0: write g*P only (the identity/residual is added in fp32 by the conv epilogue), as the
                                // 1x1 conv's weight image of N tile nt in operand form `form` (conv_tc_wimg), per sample
    int form;
};

struct FinalParams {            // final_block GN+Mish, final_conv 1x1 -> 1, mask, Euler(-Maruyama) update
    const float* raw; GnRef gn; // [B][H][T][C]
    const float* wfin; const float* bfin;
    const float* mask; const float* mu;
    const float* xt_in; float* xt_out;   // Euler mode: xt_out = (xt - dxt)*mask ; estimator mode: xt_out = est
    const float* const* noise_pp;   // stoc: device cell holding a base such that step i's slab is base + i*B*H*T
    const float4* coef;         // per step {beta, h, sqrt(beta*h), 0}
    const int* step;
    int mode;                   // 0: estimator output, 1: deterministic Euler, 2: Euler-Maruyama (Grad-TTS),
                                // 3: DiffVC  xt' = (xt - ((mean-xt)*A - est*Bc + eps*sigma))*mask, coef = {A, Bc, sigma}
    int B, H, T, C;
    int chw4;
    int exact;                  // fp32x3 mode: exact Mish (expf + IEEE division) instead of the fast intrinsics
};

struct TimeTableParams {        // SinusoidalPosEmb + mlp + the 12 per-ResnetBlock projections
    const float* t_rows; int rows;     // t value per row
    const float* freqs;                // [dim/2] host-computed exp(-j*ln(1e4)/(dim/2-1))
    float pe_scale; int dim;
    const float* w0; const float* b0;  // [4*dim][dim], [4*dim]
    const float* w2; const float* b2;  // [dim][4*dim], [dim]
    int nproj;
    const float* pw[16]; const float* pb[16]; int pc[16]; int poff[16];   // Linear(dim -> pc[k]) per ResnetBlock
    float* tb; int tb_stride;
};

struct SpkParams {              // spk_mlp: Linear(E,4E) -> Mish -> Linear(4E, n_feats)
    const float* spk; const float* w0; const float* b0; const float* w2; const float* b2;
    float* out; int B, E, n_feats;
};

// DiffVC: fold the conditioning vector into the first ResnetBlock (diffusion.py:73-76 of DiffVC: condition is
// broadcast over the grid and concatenated as 128 extra channels): per (row, sample)
//   w_extra[tap][co] = sum_ci cond[ci] * W1[co][2+ci][tap],   r_extra[co] = sum_ci cond[ci] * Wres[co][2+ci]
struct CondFoldParams {
    const float* cond;      // [rows][B][dc]
    const float* w1;        // raw block1 conv weight [C][2+dc][3][3]
    const float* wres;      // raw res_conv weight [C][2+dc]
    float* w_extra;         // [rows*B][9][C]
    float* r_extra;         // [rows*B][C]
    int rows, B, dc, C;
};
int launch_cond_fold(const CondFoldParams& p, cudaStream_t s);

// ---- DiffVC RefBlock / conditioning branch (DiffVC/model/modules.py:128-166, diffusion.py:62-71), tensor-core modes ----
struct DiffMeanParams {          // xt_ref = (ref*g + mean_ref*(1-g)) * ref_mask  (compute_diffused_mean, diffusion.py:151-155)
    const float* ref; const float* mean_ref; const float* mask; float* out; float g; int B, H, T;
};
struct ChanStatsParams {         // per (sample, channel) {sum, sum of squares} over H*W of a [B][H][C/4][W][4] tensor (InstanceNorm2d)
    const float* x; double* stats; int B, H, W, C;
};
struct InGluParams {             // y = mask ? tf32( IN(raw[c]) * sigmoid(IN(raw[c + C/2])) + tb[c] ) : 0   -> C/2 channels
    const float* raw; const double* stats; const float* gamma; const float* beta;   // InstanceNorm2d affine, eps 1e-5
    const float* tb;             // [C/2] time bias (mlp1 / mlp2 row of this step) or nullptr
    const float* mask; int T;    // ref_mask [B][T]
    float* out; int B, H, W, C;  // C = raw channels
    int form;                    // FORM_TF32: fast sigmoid, out rounded to tf32; FORM_X3: exact sigmoid, out unrounded
};
struct VcCondParams {            // cond_block( [sinusoid(t) | final_conv(mean-pooled RefBlock) | c] )  (diffusion.py:62-71)
    const double* ysum;          // [B][dc][2] channel sums of the masked RefBlock output (before final_conv)
    const float* mask; int Tr; int H;
    const float* wf; const float* bf;         // ref_block.final_conv [dc][dc], [dc]
    const float* c;              // [B][256] speaker embedding
    const float* freqs; float t; int dim;     // sinusoid
    const float* w0; const float* b0; const float* w2; const float* b2;   // cond_block
    float* out;                  // [B][dc] (row of this step)
    int B, dc, use_ref;
};
int launch_diff_mean(const DiffMeanParams& p, cudaStream_t s);
int launch_chan_stats(const ChanStatsParams& p, cudaStream_t s);
int launch_in_glu(const InGluParams& p, cudaStream_t s);
int launch_vc_cond(const VcCondParams& p, cudaStream_t s);

// GradTTS.forward glue before the decoder (Grad-TTS/model/tts.py:82-94): alignment path + aligned prior + terminal sample
struct PriorExpandParams {
    const float* mu_x;          // [B][F][Tx]
    const float* w_ceil;        // [B][Tx]
    const float* x_mask;        // [B][Tx]
    const long long* y_len;     // [B]
    const float* noise_tf;      // [B][Ty][F] or nullptr
    float temperature;
    int B, F, Tx, Ty;
    float* mu_y; float* z;      // [B][F][Ty]
    float* y_mask;              // [B][Ty]
    float* attn;                // [B][Tx][Ty] or nullptr
};
int launch_prior_expand(const PriorExpandParams& p, cudaStream_t s);

struct StepBeginParams { double* stats; int n_doubles; int* step_cur; int* step_next; };

// launchers (all asynchronous on `s`); return the number of kernels launched
int launch_igemm(const IgemmParams& p, cudaStream_t s);
int launch_first_conv(const FirstConvParams& p, cudaStream_t s);
int launch_conv_tc(const ConvTcParams& p, cudaStream_t s);
// N tile of a conv: the width its weights are packed with and its launch runs (ConvTcParams::nt)
int conv_tc_ntile(int geom, int Cout, int form);
// host: logical weights [cout][cin][taps] -> the conv kernel's weight image for N tile nt (conv_tc_wimg).  Returns the
// image size in bytes; dst may be null to query it.
size_t conv_tc_pack_image(const float* w, int cout, int cin, int geom, int form, int nt, uint8_t* dst);
// host: the k and v rows of to_qkv [384][C] -> k_attn_kv_wg's weight image (sbk_conv_tc.cu).  Returns its size in bytes;
// dst may be null to query it.
size_t attn_kv_pack_image(const float* qkv, int C, int form, uint8_t* dst);
int launch_gn_act(const GnActParams& p, cudaStream_t s);
int launch_resfinal(const ResFinalParams& p, cudaStream_t s);
int launch_attn_ctx(const AttnCtxParams& p, cudaStream_t s);
// fused k|v projection + softmax + context partials (sbk_attn_x3.cu), one partial per item of attn_kv_tile_pixels() pixels:
// p.kv_part = [B][items per sample][4][kKvPartFloats]; tf32 / bf16 operands, or fp32-class (fp32x3 mode)
int attn_kv_tile_pixels();
int launch_attn_kv(const ConvTcParams& p, cudaStream_t s);
int launch_attn_mix(const AttnMixParams& p, cudaStream_t s);
int launch_final(const FinalParams& p, cudaStream_t s);
int launch_time_table(const TimeTableParams& p, cudaStream_t s);
int launch_spk(const SpkParams& p, cudaStream_t s);
int launch_step_begin(const StepBeginParams& p, cudaStream_t s);
int device_sm_count();      // SMs of the current device (grid caps of the grid-stride kernels)
int launch_scale_mask(const float* z, const float* mask, float* out, long long n_per_b_row, int B, int H, int T, cudaStream_t s);

// the part of an fp32 value the tensor core's tf32 operand path drops (low 13 mantissa bits): exact in fp32
__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// ---- fp32x3 mode: the correction operand ------------------------------------------------------------------------------
// x*w = x_hi*w_hi + (x_lo*w + x*w_lo) + O(2^-23): the first product runs as a tf32 MMA on the fp32 tensor itself (the
// tensor core reads the top 19 bits = x_hi), the bracket is ONE f16 MMA over a packed correction operand.  For every
// 16-byte chunk of 4 channels of an A tile the conv kernel derives, in shared memory, a 16-byte chunk of eight fp16 values
//     { x_lo[c0..c3] , x[c0..c3] * 2^-12 }            with x_lo = x - trunc_tf32(x)  (|x_lo| <= 2^-10 |x|)
// and the weight packers write the matching K order { w[c0..c3] , w_lo[c0..c3] * 2^12 } (w_lo = w - tf32(w)), so one
// K = 16 fp16 MMA over two chunks adds x_lo*w + x*w_lo for 8 channels.  fp16 carries the same 11 significant bits as tf32;
// the exact 2^-12 / 2^12 scaling keeps x in fp16's range up to |x| = 2.7e8 and keeps w_lo (~2^-12 |w|) out of its subnormals.
// Two MMAs per algorithmic MAC instead of the
// three of a 3xTF32 split, at the same modelled accuracy (CPU operand-rounding model: 1.1e-6 vs 1.2e-6 per estimator call).
constexpr float kCorrDown = 1.f / 4096.f;     // 2^-12 (activation side)
constexpr float kCorrUp = 4096.f;             // 2^12  (weight side)
__device__ __forceinline__ uint32_t f16x2_sat(float e0, float e1) {     // e0 in the low half (= the lower K index)
    uint32_t d;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(e1), "f"(e0));
    return d;
}
__device__ __forceinline__ float4 corr_chunk(float x0, float x1, float x2, float x3) {
    return make_float4(__uint_as_float(f16x2_sat(tf32_lo(x0), tf32_lo(x1))), __uint_as_float(f16x2_sat(tf32_lo(x2), tf32_lo(x3))),
                       __uint_as_float(f16x2_sat(x0 * kCorrDown, x1 * kCorrDown)), __uint_as_float(f16x2_sat(x2 * kCorrDown, x3 * kCorrDown)));
}

inline int igemm_mtiles(int geom, int Hout, int Wout, int Hin, int Win) {
    const int TM = 128;
    if (geom == G_UP) return 4 * ((Hin * Win + TM - 1) / TM);
    return (Hout * Wout + TM - 1) / TM;
}

}  // namespace sbk
