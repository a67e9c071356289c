/*
 * sbk.h - C ABI of the H100-native score-based mel sampler (libsbk.so).
 *
 * The reference (huawei-noah/Speech-Backbones) has no FFI layer: its boundary for this
 * path is the Python class `Diffusion` (Grad-TTS/model/diffusion.py:227-279) and its
 * estimator `GradLogPEstimator2d` (:128-216).  This header is the boundary a binding
 * for that class would call; every entry point cites the reference interface it replaces.
 * Plain pointers and sizes only; no torch types.  All tensors are contiguous fp32 in the
 * reference's own layouts ([B,n_feats,T], [B,1,T], [B], [B,spk_emb_dim]).
 *
 * Ownership: the caller owns every buffer passed in/out and the CUDA stream; the library
 * owns packed weights, workspaces and CUDA graphs.  Calls on one handle are not re-entrant.
 * Work is enqueued asynchronously on `stream` (stream-ordered with the caller's next op)
 * except for the *_host entry points, which synchronise before returning.
 * Errors: 0 on success, non-zero otherwise; text via sbk_last_error().  No exceptions.
 */
#ifndef SBK_H_
#define SBK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sbk_handle sbk_handle;

enum { SBK_OK = 0, SBK_ERR_ARG = 1, SBK_ERR_CUDA = 2, SBK_ERR_STATE = 3, SBK_ERR_UNSUPPORTED = 4 };

/* arithmetic of the dense contractions (3x3/1x1 convs); GN / softmax / Mish / Euler are always fp32 */
enum { SBK_PREC_FP32 = 0,   /* CUDA-core FFMA, fp32 operands (bit-faithful class of the CPU reference)   */
       SBK_PREC_TF32 = 1,   /* wgmma tf32, fp32 accumulate in registers (PyTorch's default GPU class) */
       SBK_PREC_BF16 = 2,   /* wgmma bf16 on bf16 operand tensors (conv inputs + weights stored as bf16),
                               fp32 accumulate; raw conv outputs, GN statistics, softmax, sampler state fp32
                               (BASELINE config 3); both models                                             */
       SBK_PREC_FP32X3 = 3 };/* fp32-class arithmetic on wgmma: x*w = x_hi*w_hi (tf32, the tensor core reads
                               the top 19 bits of x) + (x_lo*w + x*w_lo) as ONE f16 MMA over packed fp16
                               correction chunks - two MMAs per MAC; fp32 accumulation in registers, cut into short runs
                               that are summed in round-to-nearest fp32 (the tensor core truncates its accumulator);
                               softmax / Mish / GN exact fp32.  The default of the drop-in modules: matches the
                               reference's fp32 CPU arithmetic to 2-3e-6 per estimator call                   */
enum { SBK_PREC_F16 = 4 };  /* wgmma f16 on fp16 operand tensors: SBK_PREC_BF16's layout, tiling and launches with
                               fp16 elements (11 significant bits, tf32's, instead of bf16's 8), rounded to nearest
                               even and saturated to +-65504; fp32 accumulate, raw conv outputs, GN statistics,
                               softmax and sampler state fp32.  tf32-class error at bf16's operand bytes and MMA
                               rate.  Both models' samplers (DiffVC's RefBlock branch runs tf32 operands, as in the
                               bf16 mode) and the PostNet (tf32 operands); the vocoder refuses it               */

enum { SBK_MODEL_GRADTTS = 0, SBK_MODEL_DIFFVC = 1 };

/* Constructor arguments of Diffusion.__init__ (Grad-TTS/model/diffusion.py:228-230). */
typedef struct sbk_config {
    int32_t model;        /* SBK_MODEL_*                                                    */
    int32_t n_feats;      /* 80                                                             */
    int32_t dim;          /* 64 (Grad-TTS dec_dim, params.py:40)                            */
    int32_t n_spks;       /* 1 => no speaker channel; >1 => spk_mlp + third input channel   */
    int32_t spk_emb_dim;  /* 64                                                             */
    float beta_min;       /* 0.05                                                           */
    float beta_max;       /* 20.0                                                           */
    float pe_scale;       /* 1000.0                                                         */
    int32_t device;       /* CUDA device ordinal                                            */
    int32_t precision;    /* SBK_PREC_*                                                     */
    int32_t use_graph;    /* 1: capture one reverse step as a CUDA graph and replay it      */
    /* SBK_MODEL_DIFFVC only (DiffVC/model/diffusion.py:110, DiffVC/params.py:26-28); `dim` is dim_unet (256) */
    int32_t dim_cond;     /* dim_spk = 128: width of the conditioning vector                */
    int32_t use_ref_t;    /* 1: the state_dict carries ref_block.* (strict loading)         */
} sbk_config;

/* Diffusion.__init__ / GradLogPEstimator2d.__init__ (diffusion.py:128-172,228-242). */
int sbk_create(const sbk_config* cfg, sbk_handle** out);
void sbk_destroy(sbk_handle* h);

/* nn.Module.load_state_dict(strict=True) (Grad-TTS/inference.py:53): one call per state_dict
 * entry under `estimator.` with the reference name (e.g. "estimator.downs.0.0.block1.block.0.weight")
 * and shape.  `data` may be a host or device pointer to contiguous fp32.  sbk_pack() then checks
 * that every expected tensor was supplied (strict) and builds the kernel layouts. */
int sbk_set_weight(sbk_handle* h, const char* ref_name, const void* data, const int64_t* shape, int ndim);
int sbk_pack(sbk_handle* h);
/* number of tensors the strict loader expects / name of the i-th one (host logic; no GPU work) */
int sbk_num_weights(const sbk_handle* h);
const char* sbk_weight_name(const sbk_handle* h, int i);

/* bytes of device workspace a (B,T) problem needs (activations, statistics, time tables) */
size_t sbk_workspace_bytes(const sbk_handle* h, int B, int T);          /* for n_timesteps <= 1024 */
/* the same for a given number of steps: the per-step tables (time projections, coefficients, DiffVC conditioning vectors
 * and folded first-conv weights) have max(64, B, n_timesteps) rows, so N = 2000 or DiffVC at large N * B needs more */
size_t sbk_workspace_bytes_n(const sbk_handle* h, int B, int T, int n_timesteps);

/* GradLogPEstimator2d.forward(x, mask, mu, t, spk) (diffusion.py:174-216).
 * x, mu, out: [B,n_feats,T]; mask: [B,1,T] in {0,1}; t: [B]; spk: NULL or [B,spk_emb_dim]. Device pointers. */
int sbk_estimator(sbk_handle* h, const float* x, const float* mask, const float* mu, const float* t,
                  const float* spk, float* out, int B, int T, void* stream);
/* Ragged batches.  lengths: NULL (the dense call above: sbk_estimator, sbk_reverse_diffusion and sbk_reverse_steps are these
 * entry points with lengths = NULL) or device int64 [B], each utterance's valid frames, such as Grad-TTS's y_lengths.
 * Utterance b is computed on its own grid of T_b = fix_len_compatibility(lengths[b]) frames (a multiple of 4, <= T):
 * out[b, :, :T_b] is the call on x[b:b+1, :, :T_b], mask[b:b+1, :, :T_b], mu[b:b+1, :, :T_b] (and noise[:, b, :, :T_b],
 * spk[b:b+1]) - its GroupNorm statistics, attention softmax and conv borders see its own T_b frames only - and
 * out[b, :, T_b:] is 0.  Nothing at or past T_b is read.  The kernels clamp each length to [1, T]; validating them is the
 * caller's job.  The plan keeps its own device copy of lengths, refreshed on the stream by every call, so the captured
 * graphs never hold the caller's pointer; a ragged loop is still one host launch.  tf32 and bf16 rows are bit for bit their
 * own B = 1 calls; fp32x3 and fp32 rows agree with them to fp32 rounding. */
int sbk_estimator_lengths(sbk_handle* h, const float* x, const float* mask, const float* mu, const float* t,
                          const float* spk, const int64_t* lengths, float* out, int B, int T, void* stream);

/* Diffusion.reverse_diffusion(z, mask, mu, n_timesteps, stoc, spk) (diffusion.py:254-275).
 * noise: NULL when stoc==0, else [N,B,n_feats,T] pre-drawn N(0,1) (the reference draws it with
 * torch.randn inside the loop, :267; the binding draws it in the same order and passes it in).
 * out may alias z.  Device pointers. */
int sbk_reverse_diffusion(sbk_handle* h, const float* z, const float* mask, const float* mu, const float* spk,
                          const float* noise, float* out, int B, int T, int n_timesteps, int stoc, void* stream);
/* the same over a ragged batch (lengths: see sbk_estimator_lengths) */
int sbk_reverse_diffusion_lengths(sbk_handle* h, const float* z, const float* mask, const float* mu, const float* spk,
                                  const float* noise, const int64_t* lengths, float* out, int B, int T, int n_timesteps,
                                  int stoc, void* stream);

/* ---- rolling batches (Grad-TTS; DiffVC through sbk_vc_rolling_reserve / sbk_vc_rolling_admit) ---------------
 * A slot plan of `capacity` rows (slots) at T = max_frames keeps running while requests join and leave it: slot b holds
 * one request - the arguments of one B = 1 Diffusion.forward call - at its own step i_b of its own n_timesteps N_b, and
 * runs as a ragged row of its T_b frames (sbk_estimator_lengths).  Step i_b uses t = 1 - (i_b + 0.5)/N_b and the
 * coefficients every other sampler call uses for it.  A finished request's mel is its own B = 1 sbk_reverse_diffusion
 * (bit for bit in tf32 and bf16, within fp32 rounding in fp32x3 and fp32) and, in every mode bit for bit, row b of a
 * sbk_reverse_diffusion_lengths call at (capacity, max_frames) with N_b steps, whatever the other slots hold and whenever
 * the request was admitted.  An empty slot runs as a 4-frame row of zeros and is read by no other row.
 * The schedule is deterministic: the caller knows when each slot finishes without reading device memory.
 * The plan is the handle's one plan: another sampler call on the handle replaces it, and the rolling entry points then fail
 * with SBK_ERR_STATE until the next sbk_rolling_reserve (sbk_vc_rolling_reserve).  sbk_rolling_reserve and sbk_rolling_admit
 * take Grad-TTS handles only (SBK_ERR_ARG for DiffVC); sbk_rolling_advance / read / release serve the slot plans of both
 * models. */
/* (Re)build the slot plan at (capacity >= 1, max_frames a multiple of 4) with every slot empty. */
int sbk_rolling_reserve(sbk_handle* h, int capacity, int max_frames, void* stream);
/* Admit a request into an empty slot (SBK_ERR_STATE if it is busy): z, mu [1,n_feats,T_b], mask [1,1,T_b] (copied on the
 * stream: they may be reused after the call), T_b a multiple of 4 in [4, max_frames], n_timesteps >= 1, spk [1,spk_emb_dim]
 * when n_spks > 1, and for stoc = 1 noise [n_timesteps,1,n_feats,T_b], the reference's per-step draws, which the slot reads
 * until it finishes: the caller keeps it alive until then.  Only this slot's rows and schedule are written. */
int sbk_rolling_admit(sbk_handle* h, int slot, const float* z, const float* mask, const float* mu, const float* spk,
                      const float* noise, int T_b, int n_timesteps, int stoc, void* stream);
/* Run `steps` >= 1 steps of every slot that has steps left (a finished or empty slot is left as it is).  One host launch
 * of a CUDA graph (sbk_last_host_launches() == 1) where the driver supports conditional nodes. */
int sbk_rolling_advance(sbk_handle* h, int steps, void* stream);
/* Copy a finished slot's mel into out [1,n_feats,T_b] (device, stream-ordered, no host synchronisation); SBK_ERR_STATE if
 * the slot holds no finished request. */
int sbk_rolling_read(sbk_handle* h, int slot, float* out, void* stream);
/* Empty a slot (finished or not) so that a new request can be admitted into it. */
int sbk_rolling_release(sbk_handle* h, int slot, void* stream);

/* Rolling DiffVC batches: the same slot plan on a DiffVC handle (SBK_ERR_ARG for Grad-TTS), advanced, read and released with
 * sbk_rolling_advance / read / release.  Slot b holds the arguments of one B = 1 sbk_vc_reverse_diffusion call at its own
 * step i_b of its own N_b: step i_b uses t = 1 - i_b/N_b, the {A, Bc, sigma} coefficients of every other DiffVC sampler call
 * and row i_b of the request's own conditioning table, gathered into a [1][capacity] table and folded into the first
 * ResnetBlock per slot.  A finished request's mel is, in every mode bit for bit, row b of a sbk_vc_reverse_diffusion_lengths
 * call at (capacity, max_frames) with the same N_b, mode, cond rows and noise, whatever the other slots hold and whenever it
 * was admitted; and its own B = 1 sbk_vc_reverse_diffusion where the two plans pick the same 3x3 tile layout (SBK_CONV3_ROWS
 * pins it): bit for bit in tf32 and bf16, within fp32 rounding in fp32x3 and fp32. */
/* (Re)build a DiffVC slot plan at (capacity >= 1, max_frames a multiple of 4) with every slot empty. */
int sbk_vc_rolling_reserve(sbk_handle* h, int capacity, int max_frames, void* stream);
/* Admit a request into an empty slot (SBK_ERR_STATE if it is busy): z, mean [1,n_feats,T_b], mask [1,1,T_b], T_b a multiple of
 * 4 in [4, max_frames], n_timesteps >= 1, cond [n_timesteps][1][dim_cond] (sbk_vc_conditioning at B = 1), mode 0 pf, 1 em,
 * 2 ml.  z, mask, mean and cond are copied on the stream.  For em / ml, noise [n_timesteps,1,n_feats,T_b], the reference's
 * per-step draws, which the slot reads until it finishes: the caller keeps it alive until then; NULL for pf.  Only this
 * slot's rows and schedule are written. */
int sbk_vc_rolling_admit(sbk_handle* h, int slot, const float* z, const float* mask, const float* mean, const float* cond,
                         const float* noise, int T_b, int n_timesteps, int mode, void* stream);

/* ---- DiffVC (SBK_MODEL_DIFFVC) ------------------------------------------------------------------------------
 * GradLogPEstimator.forward (DiffVC/model/diffusion.py:61-106) with the xt-independent conditioning vector
 * (time sinusoid | RefBlock | speaker embedding -> cond_block, :62-71) supplied by the caller: cond [B][dim_cond].
 * x, mean, out: [B,n_feats,T]; mask [B,1,T]; t [B].  Device pointers. */
int sbk_vc_estimator(sbk_handle* h, const float* x, const float* mask, const float* mean, const float* cond,
                     const float* t, float* out, int B, int T, void* stream);
/* A ragged DiffVC batch: lengths (device int64 [B], NULL = sbk_vc_estimator) holds each utterance's valid frames L_b (DiffVC's
 * x_lengths); the kernels clamp them to [1, T].  As for Grad-TTS (sbk_estimator_lengths), utterance b runs on its own
 * T_b = fix_len_compatibility(L_b) frames: out[b, :, :T_b] is what sbk_vc_estimator computes on the [:T_b] slices of row b
 * with the same cond row (bit for bit in tf32 and bf16, within fp32 rounding in fp32x3 and fp32), out[b, :, T_b:] is 0, and
 * x, mean and mask at or past T_b are not read. */
int sbk_vc_estimator_lengths(sbk_handle* h, const float* x, const float* mask, const float* mean, const float* cond,
                             const float* t, const int64_t* lengths, float* out, int B, int T, void* stream);

/* Diffusion.reverse_diffusion (DiffVC/model/diffusion.py:164-196), mode 0 = 'pf', 1 = 'em', 2 = 'ml';
 * t_i = 1 - i/N.  cond: [N][B][dim_cond], the conditioning vector of every step (it depends on t, ref and c only,
 * never on xt, so the binding evaluates it for all N steps before the loop).  noise: [N][B][n_feats][T] for
 * 'em'/'ml' (the reference draws randn_like(z) per step, :194), NULL for 'pf'.  out may alias z. */
int sbk_vc_reverse_diffusion(sbk_handle* h, const float* z, const float* mask, const float* mean, const float* cond,
                             const float* noise, float* out, int B, int T, int n_timesteps, int mode, void* stream);
/* the same over a ragged batch (lengths: see sbk_vc_estimator_lengths).  Row b equals the call on its [:T_b] slices given the
 * same draws noise[:, b, :, :T_b]; z, mean, mask and noise at or past T_b are not read, and out there is 0. */
int sbk_vc_reverse_diffusion_lengths(sbk_handle* h, const float* z, const float* mask, const float* mean, const float* cond,
                                     const float* noise, const int64_t* lengths, float* out, int B, int T, int n_timesteps,
                                     int mode, void* stream);

/* The hoisted conditioning branch natively: for every step i (t_i = 1 - i/N)
 * xt_ref = compute_diffused_mean(ref, ref_mask, mean_ref, t_i) (:151-155) -> RefBlock (modules.py:156-166: a CUDA-core
 * first Conv3x3, five Conv3x3 on wgmma, each + InstanceNorm2d + GLU, two time biases, 1x1 conv, masked mean) -> cond_block
 * over [sinusoid(t_i) | RefBlock | c] (:62-71).  ref, mean_ref: [B,n_feats,Tr]; ref_mask: [B,1,Tr]; c: [B,256];
 * cond_out: [N][B][dim_cond], ready for sbk_vc_reverse_diffusion.  Every precision mode runs it: tf32 and bf16 handles
 * with tf32 operands, fp32x3 and fp32 handles with the fp32x3 split (so each pair computes the same table).
 * SBK_ERR_UNSUPPORTED if a RefBlock conv has no tensor-core kernel. */
int sbk_vc_conditioning(sbk_handle* h, const float* ref, const float* ref_mask, const float* mean_ref, const float* c,
                        float* cond_out, int B, int Tr, int n_timesteps, void* stream);
/* A ragged reference batch: ref_lengths (device int64 [B], NULL = sbk_vc_conditioning) holds each reference's valid frames
 * R_b (DiffVC's x_ref_lengths); the kernels clamp them to [1, Tr].  Sample b's cond rows are bit for bit what
 * sbk_vc_conditioning computes for ref[b, :, :R_b], mean_ref[b, :, :R_b] with an all-ones mask (B = 1, the reference's own
 * call): the diffused reference, the block11 conv, the five 3x3 convs, the InstanceNorm statistics and divisor (H * R_b),
 * the GLU outputs and the mean pooling all stop at R_b, with no rounding of the length.  ref and mean_ref at or past R_b
 * are not read; ref_mask must be 1 below R_b.  Same workspace and launches as sbk_vc_conditioning. */
int sbk_vc_conditioning_lengths(sbk_handle* h, const float* ref, const float* ref_mask, const float* mean_ref, const float* c,
                                const int64_t* ref_lengths, float* cond_out, int B, int Tr, int n_timesteps, void* stream);
/* test hook: with sbk_debug_capture on, sbk_vc_conditioning copies every tensor the RefBlock branch writes right after the
 * launch that wrote it into a per-name device buffer (the copies do not count as launches).  Each step overwrites the
 * previous step's copies, so they hold the LAST step (t = 1/N).  Names in launch order: ref_block.xt_ref [B][H][Tr];
 * ref_block.tb (the step's time-bias row, [3 * dim_cond / 4]: mlp1 then mlp2); then per block11, block12, block21, block22,
 * block31, block32: ref_block.<blk>.raw (conv output), .stats ([B][C][2] float64 sums of x and x^2), .act (InstanceNorm +
 * GLU (+ time bias) * mask); last ref_block.ysum ([B][dim_cond][2] float64).  No names when use_ref_t is 0. */
int sbk_vc_cond_debug_num(const sbk_handle* h);
const char* sbk_vc_cond_debug_name(const sbk_handle* h, int i);
/* 0 = fp32 array, 1 = fp32 [B][H][C/4][Tr][4], 3 = float64 array, -1 = no such name */
int sbk_vc_cond_debug_op_layout(const sbk_handle* h, const char* name);
/* copy a snapshot to `dst` (host or device) in its own dtype (float64 for layout 3, else fp32); returns its element count
 * through *numel; dst may be NULL to query it */
int sbk_vc_cond_debug_read(sbk_handle* h, const char* name, void* dst, int64_t* numel);

/* The same loop in slices: runs steps [step_begin, step_end) of an n_timesteps-step trajectory in place
 * on xt (which must already hold z*mask at step 0, or the previous slice's result).  noise, when stoc,
 * holds (step_end-step_begin) slabs of [B,n_feats,T].  Lets a caller stream noise for large N. */
int sbk_reverse_steps(sbk_handle* h, float* xt, const float* mask, const float* mu, const float* spk,
                      const float* noise, int B, int T, int n_timesteps, int step_begin, int step_end,
                      int stoc, void* stream);
/* the same over a ragged batch (lengths: see sbk_estimator_lengths); xt at or past T_b is neither read nor kept (0 after) */
int sbk_reverse_steps_lengths(sbk_handle* h, float* xt, const float* mask, const float* mu, const float* spk,
                              const float* noise, const int64_t* lengths, int B, int T, int n_timesteps, int step_begin,
                              int step_end, int stoc, void* stream);

/* Diffusion.forward with HOST buffers (the call `GradTTS.forward` makes at tts.py:96 when the caller's
 * tensors live on the CPU): copies z/mask/mu(/spk/noise) to the device, runs the loop, copies the result
 * back into out, and synchronises.  Pinned host memory gives asynchronous copies. */
int sbk_reverse_diffusion_host(sbk_handle* h, const float* z, const float* mask, const float* mu, const float* spk,
                               const float* noise, float* out, int B, int T, int n_timesteps, int stoc);

/* ---- the step before the path (SURVEY.md 8f rank 2): GradTTS.forward, Grad-TTS/model/tts.py:82-94 -----------------
 * From the encoder outputs build, in ONE pass and without materialising [B,Tx,Ty] intermediates,
 *   attn  = generate_path(w_ceil, x_mask (x) y_mask)            (model/utils.py:26-39, tts.py:83-85)
 *   mu_y  = (attn^T @ mu_x^T)^T  - a 0/1 matrix product, i.e. an exact gather of encoder frames   (tts.py:88-89)
 *   z     = mu_y + noise / temperature                          (tts.py:94; IEEE division as on the reference's CPU path)
 *   y_mask = sequence_mask(y_lengths, Ty)                       (tts.py:83)
 * mu_x: [B,F,Tx]; w_ceil: [B,Tx] = ceil(exp(logw) * x_mask) * length_scale (tts.py:77-78, computed by the caller with the
 * reference's own ops so that the token durations are the reference's bit for bit); x_mask: [B,Tx] in {0,1};
 * y_lengths: [B] int64 = clamp_min(sum(w_ceil), 1) (tts.py:79); Ty = fix_len_compatibility(max(y_lengths)) (tts.py:80-81).
 * noise_tf: [B][Ty][F] standard normal draws - the MEMORY order in which the reference's randn_like(mu_y) fills its
 * transposed mu_y - or NULL (then z = mu_y).  Outputs: mu_y, z: [B,F,Ty] contiguous (the layout sbk_reverse_diffusion
 * takes); y_mask: [B,Ty]; attn: NULL or [B,Tx,Ty].  Cumulative durations are accumulated sequentially in double and rounded
 * to fp32 per prefix, exactly as torch.cumsum does on the reference's CPU path.  No handle: the op has no weights.  Device pointers; asynchronous on `stream`. */
int sbk_prior_expand(const float* mu_x, const float* w_ceil, const float* x_mask, const int64_t* y_lengths,
                     const float* noise_tf, float temperature, int B, int F, int Tx, int Ty,
                     float* mu_y, float* z, float* y_mask, float* attn, void* stream);

/* number of kernel launches the last sbk_estimator / sbk_reverse_* call enqueued (graph nodes count) */
int64_t sbk_last_launch_count(const sbk_handle* h);
/* number of HOST launches the Euler loop of the last sbk_reverse_* call took: 1 when the whole loop ran as one CUDA graph
 * (a conditional WHILE node around one captured reverse step - the reference's Python loop, diffusion.py:258-274, issues
 * ~350 kernel launches per step), n_steps when it fell back to one graph launch per step, n_steps * kernels without graphs */
int sbk_last_host_launches(const sbk_handle* h);

/* measurement hook: run ONE step of the current plan (the (B,T) of the last call) launch by launch with a CUDA
 * event between launches, on the library's stream, and return per-launch milliseconds plus the algorithmic
 * FLOPs / HBM bytes of each launch (names via sbk_debug_name).  Advances the library's xt copy by one step. */
int sbk_profile_ops(sbk_handle* h, float* ms, double* flops, double* bytes, int cap, int* n_ops);

/* test hook: copy a named intermediate of the last sbk_estimator call (NHWC fp32) to `dst` (host or device).
 * Returns the element count through *numel; dst may be NULL to query the size only. */
int sbk_debug_read(sbk_handle* h, const char* name, float* dst, int64_t* numel);
/* test hook: when on, sbk_estimator snapshots every launch's output right after the launch (workspace buffers
 * are reused across stages, so later stages would otherwise overwrite earlier intermediates) */
int sbk_debug_capture(sbk_handle* h, int on);
/* test hook: layout of the intermediates sbk_debug_read returns: 0 = NHWC [B][H][W][C] (fp32 mode),
 * 1 = channel-chunk planar [B][H][C/4][W][4] (tensor-core modes) */
int sbk_debug_layout(const sbk_handle* h);
/* test hook: layout of ONE named intermediate (the bf16 mode mixes fp32 raw outputs with bf16 operand tensors):
 * 0 / 1 as above, 2 = [B][H][C/8][W][8] stored as bf16, 4 = the same stored as fp16 (sbk_debug_read widens both to fp32;
 * dst must be host memory), -1 = unknown name */
int sbk_debug_op_layout(const sbk_handle* h, const char* name);
/* test hook: enumerate intermediate names */
int sbk_debug_num(const sbk_handle* h);
const char* sbk_debug_name(const sbk_handle* h, int i);

/* ---- the step after the path (SURVEY.md 8f rank 3): the HiFi-GAN generator, mel -> waveform ----------------------------
 * Grad-TTS/hifi-gan/models.py:77-128 (Generator) with ResBlock1 (:13-49) or ResBlock2 (:53-74, sbk_vocoder_create_ex), built
 * from Grad-TTS/checkpts/hifigan-config.json (or the public HiFi-GAN V3 config) and
 * called as `vocoder.forward(y_dec)` at Grad-TTS/inference.py:81 after `remove_weight_norm()` (:63).  The fields below are that
 * JSON's; weights are the generator's state_dict AFTER remove_weight_norm ("conv_pre.weight" [C0,num_mels,7],
 * "ups.i.weight" [Cin,Cout,k], "resblocks.n.convs{1,2}.j.weight" [C,C,k], "conv_post.weight" [1,C,7] and the biases).
 * Dense contractions run on wgmma, by default with tf32 operands and fp32 accumulation; everything else is fp32.
 * sbk_vocoder_set_precision selects the operand arithmetic of the convs and transposed convs:
 *   SBK_PREC_TF32 (a fresh handle)  tf32 operands;
 *   SBK_PREC_FP32X3 (and FP32, which maps to it)  fp32-class: x*w = x_hi*w_hi + one f16 correction MMA, chunked accumulation;
 *   SBK_PREC_BF16  bf16 weights and bf16 conv inputs (the LeakyReLU operands); the residual stream stays fp32.
 *   SBK_PREC_F16 is a sampler mode: the vocoder refuses it (SBK_ERR_UNSUPPORTED).
 * In every mode conv_post + tanh, the transposed convs' overlap-add, the MRF mean and the waveform are fp32, and the forward
 * makes the same launches. */
typedef struct sbk_vocoder sbk_vocoder;
typedef struct sbk_vocoder_config {
    int32_t device;
    int32_t num_mels;                     /* 80                                                        */
    int32_t upsample_initial_channel;     /* 512                                                       */
    int32_t n_ups;                        /* len(upsample_rates) = 4                                   */
    int32_t upsample_rates[4];            /* [8, 8, 2, 2]                                              */
    int32_t upsample_kernel_sizes[4];     /* [16, 16, 4, 4]  (must be 2 * rate)                        */
    int32_t n_kernels;                    /* len(resblock_kernel_sizes) = 3                            */
    int32_t resblock_kernel_sizes[3];     /* [3, 7, 11]                                                */
    int32_t resblock_dilations[3][3];     /* [[1,3,5],[1,3,5],[1,3,5]]                                 */
} sbk_vocoder_config;
/* Generator.__init__, models.py:78-101, for a ResBlock1 generator (HiFi-GAN V1).  SBK_ERR_UNSUPPORTED unless there are 1..4
 * upsample stages with k = 2 * rate and an even rate, every stage has a multiple of 32 channels, there are 3 resblock
 * kernels, and every halo (k-1)*d is at most 64 samples.  Equivalent to sbk_vocoder_create_ex with resblock = 1 under that
 * tighter halo limit. */
int sbk_vocoder_create(const sbk_vocoder_config* cfg, sbk_vocoder** out);
/* The fields of sbk_vocoder_config plus the config's "resblock": 1 (ResBlock1, models.py:13-49: convs1 / convs2 at all three
 * dilations) or 2 (ResBlock2, :53-74: two convs, at the first two dilations of each kernel; HiFi-GAN V3).  ResBlock2
 * weights are "resblocks.n.convs.j.weight" [C,C,k] (j < 2) and their biases. */
typedef struct sbk_vocoder_config_ex {
    int32_t device;
    int32_t num_mels;
    int32_t upsample_initial_channel;
    int32_t n_ups;
    int32_t upsample_rates[4];
    int32_t upsample_kernel_sizes[4];
    int32_t n_kernels;
    int32_t resblock_kernel_sizes[3];     /* each 3, 5, 7 or 11                                        */
    int32_t resblock_dilations[3][3];     /* ResBlock2 reads [j][0] and [j][1]                         */
    int32_t resblock;                     /* 1 or 2                                                    */
} sbk_vocoder_config_ex;
/* The limits of sbk_vocoder_create, except that a halo (k-1)*d may reach 128 samples (a launch whose halo exceeds 64 runs on
 * the wide Conv1d strip); d >= 1.  SBK_ERR_UNSUPPORTED names the rule a refused config breaks (HiFi-GAN V2's 16- and
 * 8-channel stages break the 32-channel rule). */
int sbk_vocoder_create_ex(const sbk_vocoder_config_ex* cfg, sbk_vocoder** out);
void sbk_vocoder_destroy(sbk_vocoder* v);
int sbk_vocoder_num_weights(const sbk_vocoder* v);
const char* sbk_vocoder_weight_name(const sbk_vocoder* v, int i);
/* load_state_dict(strict) + remove_weight_norm (inference.py:61-63): one call per effective tensor, host or device fp32 */
int sbk_vocoder_set_weight(sbk_vocoder* v, const char* name, const void* data, const int64_t* shape, int ndim);
int sbk_vocoder_pack(sbk_vocoder* v);
/* SBK_PREC_* (host logic only, no device work).  Drops the packed weights: sbk_vocoder_forward returns SBK_ERR_STATE until
 * sbk_vocoder_pack runs again.  SBK_ERR_UNSUPPORTED for a configuration the mode cannot tile (bf16: num_mels a multiple of
 * 16); the handle then keeps its previous precision. */
int sbk_vocoder_set_precision(sbk_vocoder* v, int32_t precision);
/* device bytes of one forward at (B, T) in the current precision */
size_t sbk_vocoder_workspace_bytes(const sbk_vocoder* v, int B, int T);
/* Generator.forward (models.py:104-119): mel [B,num_mels,T] -> wav [B,1,T*prod(upsample_rates)] in (-1,1).  Device pointers,
 * asynchronous on `stream`.  Equivalent to sbk_vocoder_forward_lengths with lengths = NULL. */
int sbk_vocoder_forward(sbk_vocoder* v, const float* mel, float* wav, int B, int T, void* stream);
/* A ragged batch: lengths (device int64 [B], NULL = every utterance T frames) holds each utterance's valid mel frames T_b,
 * as Grad-TTS's y_lengths or DiffVC's x_lengths.  wav[b, :, :T_b*hop] is bit for bit what sbk_vocoder_forward computes for
 * mel[b, :, :T_b] alone (B = 1, the reference's own call), and wav[b, :, T_b*hop:] is 0 (hop = prod(upsample_rates)); the
 * mel's frames past T_b do not affect it.  The Conv1d work past each utterance's end is skipped.  The kernels clamp
 * each length to [0, T] (no host read of the lengths; callers validate them: an utterance of 0 frames gives a zero
 * waveform).  Same workspace and launches as sbk_vocoder_forward. */
int sbk_vocoder_forward_lengths(sbk_vocoder* v, const float* mel, const int64_t* lengths, float* wav, int B, int T, void* stream);
int64_t sbk_vocoder_last_launch_count(const sbk_vocoder* v);
/* test hook: when on, sbk_vocoder_forward copies every tensor it writes right after the launch that wrote it (the workspace
 * buffers are reused within a call) into a per-name device buffer; the copies do not count as launches.  Names in launch
 * order: mel_in, conv_pre, ups.i.{z,x,a}, resblocks.n.convs1.d, resblocks.n.convs2.d.x (and .a for d < 2), mrf.i, wav;
 * a ResBlock2 generator captures resblocks.n.convs.0.x, resblocks.n.convs.0.a, resblocks.n.convs.1.x for each block.
 * Activations keep the kernel layout (sbk_vocoder_debug_op_layout); wav is [B][1][L].  fp32x3 captures the same fp32
 * tensors as tf32: its correction chunks are derived inside the conv kernels and never stored. */
int sbk_vocoder_debug_capture(sbk_vocoder* v, int on);
int sbk_vocoder_debug_num(const sbk_vocoder* v);                                  /* names captured by the last forward */
const char* sbk_vocoder_debug_name(const sbk_vocoder* v, int i);
/* copy a captured tensor to `dst` (host or device) as fp32, bf16 snapshots widened exactly, element order unchanged; returns
 * its element count through *numel; dst may be NULL to query it */
int sbk_vocoder_debug_read(sbk_vocoder* v, const char* name, float* dst, int64_t* numel);
/* layout of a captured tensor: 1 = fp32 [B][C/4][L][4] (wav: [B][1][L]), 2 = bf16 [B][C/8][L][8] (the conv inputs in the bf16
 * mode), -1 = no such name */
int sbk_vocoder_debug_op_layout(const sbk_vocoder* v, const char* name);

/* ---- the module in front of the glue (SURVEY.md 8f rank 4): the Grad-TTS text encoder -------------------------------
 * TextEncoder (Grad-TTS/model/text_encoder.py:281-326): embedding, ConvReluNorm prenet, relative-position transformer
 * encoder, proj_m and the duration predictor; eval mode.  Called as `self.encoder(x, x_lengths, spk)` at tts.py:75; its
 * outputs are exactly sbk_prior_expand's inputs.  Constructor arguments as in text_encoder.py:282-284 (p_dropout is
 * irrelevant in eval mode); weights under the reference's state_dict names.  Exact fp32 arithmetic on CUDA cores. */
typedef struct sbk_textenc sbk_textenc;
typedef struct sbk_textenc_config {
    int32_t device;
    int32_t n_vocab, n_feats, n_channels, filter_channels, filter_channels_dp, n_heads, n_layers, kernel_size, window_size;
    int32_t n_spks, spk_emb_dim;
    int32_t kind;      /* 0: TextEncoder; 1: DiffVC MelEncoder(n_feats, channels, filters, heads, layers, kernel, dropout, window_size)
                          (DiffVC/model/encoder.py:257-284: init_proj | prenet | encoder | term_proj; n_vocab / filter_channels_dp unused) */
} sbk_textenc_config;
int sbk_textenc_create(const sbk_textenc_config* cfg, sbk_textenc** out);
void sbk_textenc_destroy(sbk_textenc* e);
int sbk_textenc_num_weights(const sbk_textenc* e);
const char* sbk_textenc_weight_name(const sbk_textenc* e, int i);
int sbk_textenc_set_weight(sbk_textenc* e, const char* name, const void* data, const int64_t* shape, int ndim);
int sbk_textenc_pack(sbk_textenc* e);
/* TextEncoder.forward(x, x_lengths, spk) (:312-326): x [B,Tx] int64 token ids, x_lengths [B] int64, spk NULL or
 * [B,spk_emb_dim] -> mu_x [B,n_feats,Tx], logw [B,1,Tx], x_mask [B,1,Tx].  Device pointers, asynchronous on `stream`. */
int sbk_textenc_forward(sbk_textenc* e, const int64_t* x, const int64_t* x_lengths, const float* spk,
                        float* mu_x, float* logw, float* x_mask, int B, int Tx, void* stream);
/* MelEncoder.forward(x, x_mask) (DiffVC/model/encoder.py:279-284, called at DiffVC/model/vc.py:39,45): x [B,n_feats,T],
 * x_mask [B,1,T] in {0,1} -> out [B,n_feats,T] (the "average voice" mel; not masked, as in the reference).  kind = 1 handles. */
int sbk_melenc_forward(sbk_textenc* e, const float* x, const float* x_mask, float* out, int B, int T, void* stream);
/* Both forwards check every argument, the attention kernel's sequence limit included (SBK_ERR_UNSUPPORTED once
 * 8 * (d + Tx rounded up to 4 + 32) floats exceed 200 KB, i.e. Tx > 6272 at head dim 96), before anything is launched or
 * written. */
int64_t sbk_textenc_last_launch_count(const sbk_textenc* e);
/* test hook: with capture on, both forwards copy every tensor right after the launch that wrote it into a per-name device
 * buffer (the copies do not count as launches; outputs and kernels are unchanged).  Names in launch order: mask (text
 * encoder only: x_mask [B][Tx]), embed (emb(x) * sqrt(C)) or init_proj (mel encoder), prenet.{0,1,2}, prenet.proj,
 * spk_concat (n_spks > 1), then per layer i: enc.i.qkv (q | k | v), enc.i.attn (attention before conv_o), enc.i.ln1,
 * enc.i.ffn1 (relu(conv_1) * mask), enc.i.ln2; then mu, dp.1, dp.2, logw (text encoder) or out (mel encoder). */
int sbk_textenc_debug_capture(sbk_textenc* e, int on);
int sbk_textenc_debug_num(const sbk_textenc* e);
const char* sbk_textenc_debug_name(const sbk_textenc* e, int i);
/* 0 = token-major fp32 [B][Tx][C], 1 = planar fp32 [B][C][Tx] (mu, logw, out), -1 = no such name */
int sbk_textenc_debug_op_layout(const sbk_textenc* e, const char* name);
/* copy a snapshot to `dst` (host or device) as fp32; returns its element count through *numel; dst may be NULL to query it */
int sbk_textenc_debug_read(sbk_textenc* e, const char* name, void* dst, int64_t* numel);

/* ---- DiffVC's PostNet: the second half of the "average voice" encoder --------------------------------------------------
 * FwdDiffusion (DiffVC/model/vc.py:19-48) is MelEncoder (above, kind = 1) followed by PostNet (DiffVC/model/postnet.py:40-53):
 * init_conv 1x1 (1 -> dim), a ResnetBlock of two Block(7x7 Conv2d(dim, dim, padding 3), GroupNorm(groups, dim), Mish) plus a
 * 1x1 residual conv (postnet.py:15-37), final_conv 1x1 (dim -> 1), over the [n_feats, T] mel grid as a one-channel image.
 * The 7x7 convs run on wgmma (tf32 operands, or the fp32x3 split); GroupNorm statistics cover the whole grid, padded columns
 * included, as the reference's do. */
typedef struct sbk_postnet sbk_postnet;
typedef struct sbk_postnet_config {
    int32_t device;
    int32_t dim;          /* PostNet(dim) (vc.py:34; DiffVC enc_dim = 128): 64, 128 or a multiple of 256                  */
    int32_t groups;       /* GroupNorm groups (postnet.py:16,27,41, default 8): must be 8                                       */
    int32_t precision;    /* SBK_PREC_*: FP32X3 and FP32 run the fp32x3 split, TF32, BF16 and F16 run tf32 operands      */
} sbk_postnet_config;
/* PostNet.__init__ (postnet.py:41-45).  SBK_ERR_UNSUPPORTED for any other dim / groups. */
int sbk_postnet_create(const sbk_postnet_config* cfg, sbk_postnet** out);
void sbk_postnet_destroy(sbk_postnet* p);
/* the 14 tensors of PostNet.state_dict() (init_conv.*, res_block.block{1,2}.block.{0,1}.*, res_block.res.*, final_conv.*):
 * count / name of the i-th one (host logic; no GPU work) */
int sbk_postnet_num_weights(const sbk_postnet* p);
const char* sbk_postnet_weight_name(const sbk_postnet* p, int i);
/* load_state_dict(strict) (vc.py:77-79 loads the encoder's checkpoint): one call per tensor, host or device fp32; then pack */
int sbk_postnet_set_weight(sbk_postnet* p, const char* name, const void* data, const int64_t* shape, int ndim);
int sbk_postnet_pack(sbk_postnet* p);
/* device workspace of a (B, n_feats, T) call (allocated by sbk_postnet_forward, grow-only) */
size_t sbk_postnet_workspace_bytes(const sbk_postnet* p, int B, int n_feats, int T);
/* PostNet.forward(x, mask) (postnet.py:47-53, called at vc.py:40,46): x [B,n_feats,T], mask [B,1,T] in {0,1} -> out
 * [B,n_feats,T].  The output is not masked, as in the reference: a padded column equals final_conv.bias.  Device pointers,
 * asynchronous on `stream`; a refused kernel launch fails the call. */
int sbk_postnet_forward(sbk_postnet* p, const float* x, const float* mask, float* out, int B, int n_feats, int T, void* stream);
/* A ragged batch: lengths (device int64 [B], NULL = every utterance T frames, as sbk_postnet_forward) holds each utterance's
 * valid frames L_b, as DiffVC's x_lengths or x_ref_lengths.  out[b, :, :L_b] is bit for bit what sbk_postnet_forward computes
 * for x[b, :, :L_b] with an all-ones mask (B = 1, the reference's own call: its GroupNorm statistics and 7x7 borders see
 * exactly L_b frames, no rounding of the length), and out[b, :, L_b:] is 0 - not final_conv.bias, since the utterance's own
 * call has no such columns.  x at or past L_b is not read; mask must be 1 below L_b.  The kernels clamp each length to
 * [1, T] (no host read of the lengths; callers validate them).  Same workspace and launches as sbk_postnet_forward. */
int sbk_postnet_forward_lengths(sbk_postnet* p, const float* x, const float* mask, const int64_t* lengths, float* out, int B,
                                int n_feats, int T, void* stream);
/* kernel launches (and memsets) the last sbk_postnet_forward enqueued */
int64_t sbk_postnet_last_launch_count(const sbk_postnet* p);
/* test hook: with capture on, sbk_postnet_forward copies every intermediate right after the launch that wrote it into a
 * per-name device buffer (the copies do not count as launches; outputs and kernels are unchanged).  Names in launch order:
 * a0 (init_conv(x*mask)*mask), block1.raw (7x7 conv output), block1.stats ([B][groups][2] float64 sums of x and x^2),
 * block1.act (Mish(GN(raw)) * mask), block2.raw, block2.stats, res (the residual conv's output, final_conv's input).  The
 * call's own output is not copied.  All are whole [B, n_feats, T] grids, past a ragged batch's edges included. */
int sbk_postnet_debug_capture(sbk_postnet* p, int on);
int sbk_postnet_debug_num(const sbk_postnet* p);
const char* sbk_postnet_debug_name(const sbk_postnet* p, int i);
/* 1 = fp32 [B][n_feats][dim/4][T][4], 3 = float64 array, -1 = no such name */
int sbk_postnet_debug_op_layout(const sbk_postnet* p, const char* name);
/* copy a snapshot to `dst` (host or device) in its own dtype (float64 for layout 3, else fp32); returns its element count
 * through *numel; dst may be NULL to query it */
int sbk_postnet_debug_read(sbk_postnet* p, const char* name, void* dst, int64_t* numel);

/* ---- DiffVC's inference front end (DiffVC/inference.ipynb: get_mel, mel_spectral_subtraction) ----------------------------
 * A handle without weights: the windowed-DFT basis and the Slaney filterbank are built on the host from the notebook's
 * constants (22050 Hz, n_fft 1024, hop 256, 80 mels, 0 - 8000 Hz).  Creating a handle and sizing its workspace are host logic
 * (no GPU work); the first call uploads the basis to cfg.device. */
typedef struct sbk_frontend sbk_frontend;
typedef struct sbk_frontend_config {
    int32_t device;
} sbk_frontend_config;
int sbk_frontend_create(const sbk_frontend_config* cfg, sbk_frontend** out);
void sbk_frontend_destroy(sbk_frontend* h);
/* bins 0 .. n - 1 the DFT computes: up to the filterbank's last nonzero bin (371 at 8 kHz) */
int sbk_frontend_dft_bins(const sbk_frontend* h);
/* device workspace of a log-mel call of B utterances and T frames (allocated by the calls, grow-only); it also covers a
 * spectral subtraction of [B, n_mels, T] */
size_t sbk_frontend_workspace_bytes(const sbk_frontend* h, int B, int T);
/* get_mel without decoding or resampling: wav [B, L] fp32 at 22050 Hz -> out [B, 80, T] fp32.  lengths (device int64 [B],
 * NULL = every utterance L samples): utterance b is wav[b, :lengths[b]], truncated to T_b = lengths[b] / 256 whole hops and
 * reflect-padded by 384 samples at its own edges; out[b, :, :T_b] is log(max(mel_basis @ |STFT|, 1e-5)) and out[b, :, T_b:]
 * is 0.  Samples at or past lengths[b] are not read.  The DFT runs on wgmma in the fp32x3 split.  Callers validate the
 * lengths (each in 512 .. L) and pass T = max_b T_b (<= L / 256); the kernels clamp a length to [0, L] and write zeros for an
 * utterance of fewer than 2 hops.  Each row is bit for bit the B = 1 call on its own samples.  Asynchronous on `stream`. */
int sbk_logmel_forward_lengths(sbk_frontend* h, const float* wav, const int64_t* lengths, float* out, int B, int L, int T,
                               void* stream);
/* mel_spectral_subtraction(mel_synth, mel_source, spectral_floor, silence_window, smoothing_window) on [B, n_mels, T] fp32,
 * one utterance per CTA: row b is the function on its first lengths[b] frames (device int64 [B], clamped to [1, T]; NULL =
 * all T) followed by zeros.  Window energies accumulate in fp64; smoothing_window = -1 skips noise_median_smoothing.
 * SBK_ERR_ARG for silence_window < 1 or smoothing_window = 0 or < -1. */
int sbk_spectral_subtraction_lengths(sbk_frontend* h, const float* mel_synth, const float* mel_source, const int64_t* lengths,
                                     float* out, int B, int n_mels, int T, float spectral_floor, int silence_window,
                                     int smoothing_window, void* stream);
/* kernel launches the last call enqueued */
int64_t sbk_frontend_last_launch_count(const sbk_frontend* h);

const char* sbk_last_error(void);
const char* sbk_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SBK_H_ */
