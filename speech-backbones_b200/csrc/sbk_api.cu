// Host side of libsbk.so: strict weight loading + packing, workspace arena, the per-step launch
// plan of the Grad-TTS score U-Net, CUDA-graph replay of the Euler(-Maruyama) loop, and the C ABI.
// Mirrors Diffusion / GradLogPEstimator2d (Grad-TTS/model/diffusion.py:128-279); see include/sbk.h.
#include "sbk_host.h"

#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

using namespace sbk;

static thread_local char g_err[1024] = "";
int sbk::fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

namespace {

struct ResnetInfo { std::string prefix; int cin, cout; };
struct AttnInfo { std::string prefix; int c; };

__global__ void k_set_int(int* p, int v) { *p = v; }
__global__ void k_set_ptr(const float** p, const float* v) { *p = v; }
// last node of the WHILE body: run another reverse step iff the step counter has not reached the end of the slice
__global__ void k_loop_cond(cudaGraphConditionalHandle handle, const int* step_next, const int* step_end) {
    cudaGraphSetConditional(handle, *step_next < *step_end ? 1u : 0u);
}

enum OpKind { OP_FIRST, OP_IGEMM, OP_RESFINAL, OP_CTX, OP_MIX, OP_FINAL, OP_CONVTC, OP_GNACT };
struct Op {
    OpKind kind; std::string name;
    FirstConvParams fc; IgemmParams ig; ConvTcParams tc; GnActParams ga; ResFinalParams rf; AttnCtxParams cx; AttnMixParams mx; FinalParams fn;
    const float* dbg_ptr = nullptr; int64_t dbg_numel = 0;
    int dbg_fmt = 0;               // layout of the named output: 0 NHWC fp32, 1 [B][H][C/4][W][4] fp32, 2 [B][H][C/8][W][8] bf16
    double flops = 0, bytes = 0;   // algorithmic work of this launch
    float* dbg_copy = nullptr;     // snapshot taken right after the launch when debug capture is on
};

struct Plan {
    int B = 0, T = 0, tb_rows = 0, noise_cap_steps = 0;
    std::vector<Op> ops;
    int final_op = -1;
    // owned buffers
    float *xt = nullptr, *mu = nullptr, *mask = nullptr, *spk_s = nullptr, *spk_in = nullptr;
    double* stats = nullptr; int n_stat_doubles = 0;
    float *tb = nullptr, *t_rows = nullptr; float4* coef = nullptr;
    int* step_cur = nullptr; int* step_next = nullptr;
    const float** noise_pp = nullptr;
    float *vc_cond = nullptr, *vc_wextra = nullptr, *vc_rextra = nullptr;   // DiffVC conditioning tables [rows][B][...]
    int first_op = -1, first_res_op = -1;
    int tb_stride = 0;
    cudaGraphExec_t gexec[4] = {nullptr, nullptr, nullptr, nullptr};   // one reverse step, per FinalParams.mode
    // the WHOLE loop as one graph: a conditional WHILE node whose body is one reverse step + k_loop_cond, so a sampler
    // call is ONE host launch for any N (N = 1000 needs no 75k-node graph).  loop_state: 0 untried, 1 built, -1 unavailable
    cudaGraphExec_t gloop[4] = {nullptr, nullptr, nullptr, nullptr};
    int loop_state[4] = {0, 0, 0, 0};
    int* step_end = nullptr;
    int launches_per_step = 0;
};

}  // namespace

struct sbk_handle {
    sbk_config cfg;
    WeightSet w;
    std::vector<ResnetInfo> resnets;
    std::vector<AttnInfo> attns;
    float* d_freqs = nullptr;
    float* d_zero = nullptr;                  // zero page for the tensor-core kernels' border copies
    Workspace ws;                             // the plan's arena
    Workspace ref_ws;                         // DiffVC RefBlock workspace
    bool is_packed = false;
    Plan plan;
    cudaStream_t cap_stream = nullptr;
    int64_t last_launches = 0;
    int last_host_launches = 0;               // graph launches the host issued for the loop of the last sampler call
    bool capture = false;
    // sbk_vc_conditioning's debug snapshots (fmt: 0 fp32 array, 1 fp32 [B][H][C/4][Tr][4], 3 float64)
    Snapshots vc_snaps;
    int tb_off[16];
    int tb_total = 0;
};

// ------------------------------------------------------------------------------------------------
// parameter inventory (GradLogPEstimator2d.__init__, diffusion.py:128-172)
// ------------------------------------------------------------------------------------------------
static void build_spec(sbk_handle* h) {
    const sbk_config& c = h->cfg;
    const int dim = c.dim;
    const bool vc = c.model == SBK_MODEL_DIFFVC;
    const int d[4] = {vc ? 2 + c.dim_cond : 2 + (c.n_spks > 1 ? 1 : 0), dim, dim * 2, dim * 4};
    auto add = [&](const std::string& n, std::vector<int64_t> s) { h->w.add(n, std::move(s)); };
    auto resnet = [&](const std::string& p, int cin, int cout) {
        add(p + ".mlp.1.weight", {cout, dim});
        add(p + ".mlp.1.bias", {cout});
        const char* blk[2] = {"block1", "block2"};
        for (int k = 0; k < 2; ++k) {
            const int ci = k == 0 ? cin : cout;
            add(p + "." + blk[k] + ".block.0.weight", {cout, ci, 3, 3});
            add(p + "." + blk[k] + ".block.0.bias", {cout});
            add(p + "." + blk[k] + ".block.1.weight", {cout});
            add(p + "." + blk[k] + ".block.1.bias", {cout});
        }
        if (cin != cout) {
            add(p + ".res_conv.weight", {cout, cin, 1, 1});
            add(p + ".res_conv.bias", {cout});
        }
        h->resnets.push_back({p, cin, cout});
    };
    auto attn = [&](const std::string& p, int ch) {
        add(p + ".fn.g", {1});
        add(p + ".fn.fn.to_qkv.weight", {kAttnHidden * 3, ch, 1, 1});
        add(p + ".fn.fn.to_out.weight", {ch, kAttnHidden, 1, 1});
        add(p + ".fn.fn.to_out.bias", {ch});
        h->attns.push_back({p, ch});
    };
    if (c.n_spks > 1) {
        add("estimator.spk_mlp.0.weight", {c.spk_emb_dim * 4, c.spk_emb_dim});
        add("estimator.spk_mlp.0.bias", {c.spk_emb_dim * 4});
        add("estimator.spk_mlp.2.weight", {c.n_feats, c.spk_emb_dim * 4});
        add("estimator.spk_mlp.2.bias", {c.n_feats});
    }
    add("estimator.mlp.0.weight", {dim * 4, dim});
    add("estimator.mlp.0.bias", {dim * 4});
    add("estimator.mlp.2.weight", {dim, dim * 4});
    add("estimator.mlp.2.bias", {dim});
    if (vc) {
        // RefBlock + cond_block (DiffVC/model/modules.py:128-154, diffusion.py:28-33): accepted by the strict loader;
        // this round the binding evaluates them (they are xt-independent and hoisted out of the loop)
        const int dc = c.dim_cond, base = dc / 4;
        int cond_total = dim + 256;
        if (c.use_ref_t) {
            add("estimator.ref_block.mlp1.1.weight", {base, dim}); add("estimator.ref_block.mlp1.1.bias", {base});
            add("estimator.ref_block.mlp2.1.weight", {2 * base, dim}); add("estimator.ref_block.mlp2.1.bias", {2 * base});
            const char* nm[6] = {"block11", "block12", "block21", "block22", "block31", "block32"};
            const int ci[6] = {1, base, base, 2 * base, 2 * base, 4 * base}, co[6] = {2 * base, 2 * base, 4 * base, 4 * base, 8 * base, 8 * base};
            for (int k = 0; k < 6; ++k) {
                const std::string q = std::string("estimator.ref_block.") + nm[k];
                add(q + ".0.weight", {co[k], ci[k], 3, 3}); add(q + ".0.bias", {co[k]});
                add(q + ".1.weight", {co[k]}); add(q + ".1.bias", {co[k]});
            }
            add("estimator.ref_block.final_conv.weight", {dc, 4 * base, 1, 1});
            add("estimator.ref_block.final_conv.bias", {dc});
            cond_total += dc;
        }
        add("estimator.cond_block.0.weight", {4 * dc, cond_total}); add("estimator.cond_block.0.bias", {4 * dc});
        add("estimator.cond_block.2.weight", {dc, 4 * dc}); add("estimator.cond_block.2.bias", {dc});
    }
    for (int l = 0; l < 3; ++l) {
        const std::string p = "estimator.downs." + std::to_string(l);
        resnet(p + ".0", d[l], d[l + 1]);
        resnet(p + ".1", d[l + 1], d[l + 1]);
        attn(p + ".2", d[l + 1]);
        if (l < 2) {
            add(p + ".3.conv.weight", {d[l + 1], d[l + 1], 3, 3});
            add(p + ".3.conv.bias", {d[l + 1]});
        }
    }
    resnet("estimator.mid_block1", d[3], d[3]);
    attn("estimator.mid_attn", d[3]);
    resnet("estimator.mid_block2", d[3], d[3]);
    const int up_in[2] = {d[2], d[1]}, up_out[2] = {d[3], d[2]};
    for (int j = 0; j < 2; ++j) {
        const std::string p = "estimator.ups." + std::to_string(j);
        resnet(p + ".0", up_out[j] * 2, up_in[j]);
        resnet(p + ".1", up_in[j], up_in[j]);
        attn(p + ".2", up_in[j]);
        add(p + ".3.conv.weight", {up_in[j], up_in[j], 4, 4});
        add(p + ".3.conv.bias", {up_in[j]});
    }
    add("estimator.final_block.block.0.weight", {dim, dim, 3, 3});
    add("estimator.final_block.block.0.bias", {dim});
    add("estimator.final_block.block.1.weight", {dim});
    add("estimator.final_block.block.1.bias", {dim});
    add("estimator.final_conv.weight", {1, dim, 1, 1});
    add("estimator.final_conv.bias", {1});
    int off = 0;
    for (size_t k = 0; k < h->resnets.size(); ++k) { h->tb_off[k] = off; off += h->resnets[k].cout; }
    h->tb_total = off;
}

// ------------------------------------------------------------------------------------------------
// C ABI: lifecycle + strict loading
// ------------------------------------------------------------------------------------------------
extern "C" const char* sbk_last_error(void) { return g_err; }
extern "C" const char* sbk_version(void) { return "sbk 0.1 (sm_90a)"; }

extern "C" int sbk_create(const sbk_config* cfg, sbk_handle** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_create: null argument");
    if (cfg->model != SBK_MODEL_GRADTTS && cfg->model != SBK_MODEL_DIFFVC) return fail(SBK_ERR_UNSUPPORTED, "sbk_create: model %d not supported", cfg->model);
    if (cfg->model == SBK_MODEL_DIFFVC && (cfg->dim_cond <= 0 || cfg->dim_cond % 4 != 0)) return fail(SBK_ERR_ARG, "sbk_create: DiffVC needs dim_cond > 0 (multiple of 4), got %d", cfg->dim_cond);
    if (cfg->model == SBK_MODEL_DIFFVC && cfg->use_ref_t && cfg->dim_cond % 128 != 0)
        return fail(SBK_ERR_ARG, "sbk_create: the native RefBlock needs dim_cond to be a multiple of 128 (its first conv writes 64-channel "
                                 "tiles and every conv reads 32-channel K stages), got %d", cfg->dim_cond);
    // Past the planar network inputs (k_first_conv and the first block's res_conv), every U-Net channel count, concatenations
    // included, is a multiple of dim, and no tensor-core conv reads a K stage of more than 64 channels
    // (conv_tc_stage_channels).  A multiple of 64 therefore lets every other U-Net conv of the tensor-core modes run on the
    // tensor cores: the CUDA-core convs serve the fp32 mode alone.
    if (cfg->dim <= 0 || cfg->dim % 64 != 0) return fail(SBK_ERR_ARG, "sbk_create: dim must be a positive multiple of 64 (got %d)", cfg->dim);
    if (cfg->n_feats <= 0 || cfg->n_feats % 4 != 0) return fail(SBK_ERR_ARG, "sbk_create: n_feats must be a multiple of 4 (two stride-2 levels), got %d", cfg->n_feats);
    if (cfg->n_spks < 1 || cfg->spk_emb_dim <= 0) return fail(SBK_ERR_ARG, "sbk_create: bad speaker configuration");
    if (cfg->precision < SBK_PREC_FP32 || cfg->precision > SBK_PREC_FP32X3) return fail(SBK_ERR_ARG, "sbk_create: unknown precision %d", cfg->precision);
    sbk_handle* h = new sbk_handle();
    h->cfg = *cfg;
    build_spec(h);
    *out = h;
    return SBK_OK;
}

// drop the launch plan and its graphs (the arena h->ws is grow-only: a new (B,T) whose layout fits its capacity is laid out
// inside it without a cudaFree/cudaMalloc pair)
static void free_plan(sbk_handle* h) {
    Plan& p = h->plan;
    for (int i = 0; i < 4; ++i) if (p.gexec[i]) { cudaGraphExecDestroy(p.gexec[i]); p.gexec[i] = nullptr; }
    for (int i = 0; i < 4; ++i) if (p.gloop[i]) { cudaGraphExecDestroy(p.gloop[i]); p.gloop[i] = nullptr; }
    for (auto& op : p.ops) if (op.dbg_copy) cudaFree(op.dbg_copy);
    p = Plan();
}

extern "C" void sbk_destroy(sbk_handle* h) {
    if (!h) return;
    free_plan(h);
    cudaFree(h->d_freqs);
    cudaFree(h->d_zero);
    if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
    delete h;
}

extern "C" int sbk_num_weights(const sbk_handle* h) { return h ? h->w.count() : 0; }
extern "C" const char* sbk_weight_name(const sbk_handle* h, int i) { return h ? h->w.name(i) : nullptr; }

extern "C" int sbk_set_weight(sbk_handle* h, const char* name, const void* data, const int64_t* shape, int ndim) {
    if (!h || !name || !data || !shape) return fail(SBK_ERR_ARG, "sbk_set_weight: null argument");
    TRY(h->w.set(name, data, shape, ndim, h->cfg.device, "sbk_set_weight"));
    h->is_packed = false;
    return SBK_OK;
}

// copy a raw tensor to the host, repack with `f(dst, src)`, upload under `key`
template <class F>
static int repack(sbk_handle* h, const std::string& src, const std::string& key, size_t out_floats, F f) {
    std::vector<float> hs, hd(out_floats);
    TRY(h->w.fetch(src, hs));
    f(hd.data(), hs.data(), h->w.find(src)->shape);
    return upload(h->w.packed, key, out_floats * sizeof(float), hd.data());
}


// logical weights [cout][cin][taps] -> the conv kernel's weight image for N tile nt, uploaded under `key`
static int pack_tc_host(sbk_handle* h, const std::vector<float>& hs, const std::string& key, int cout, int cin, int geom, int form, int nt) {
    std::vector<uint8_t> hd(conv_tc_pack_image(hs.data(), cout, cin, geom, form, nt, nullptr));
    conv_tc_pack_image(hs.data(), cout, cin, geom, form, nt, hd.data());
    return upload(h->w.packed, key, hd.size(), hd.data());
}
static int pack_tc(sbk_handle* h, const std::string& src, const std::string& key, int cout, int cin, int geom, int form) {
    std::vector<float> hs;
    TRY(h->w.fetch(src, hs));
    const int nt = conv_tc_ntile(geom, cout, form);
    TRY(pack_tc_host(h, hs, key, cout, cin, geom, form, nt));
    // 3x3 convs with >= 128 output channels also get a 64-wide N-tile image: the two-row tiles run 64 channels wide, and
    // small batches have too few 128-wide tiles to fill the GPU's SMs, so the planner switches those launches to twice as
    // many half-width tiles
    if (geom == G_C3 && nt == 128) TRY(pack_tc_host(h, hs, key + "64", cout, cin, geom, form, 64));
    return SBK_OK;
}
// the k and v rows of to_qkv for k_attn_kv_wg (sbk_attn_x3.cu)
static int pack_tc_kv(sbk_handle* h, const std::string& src, const std::string& key, int C, int form) {
    std::vector<float> q;
    TRY(h->w.fetch(src, q));
    std::vector<uint8_t> m(attn_kv_pack_image(q.data(), C, form, nullptr));
    attn_kv_pack_image(q.data(), C, form, m.data());
    return upload(h->w.packed, key, m.size(), m.data());
}
// ConvTranspose2d weight [ci][co][4][4] -> logical [co][ci][kh*4+kw]
static int pack_tc_up(sbk_handle* h, const std::string& src, const std::string& key, int C, int form) {
    std::vector<float> w, m((size_t)C * C * 16);
    TRY(h->w.fetch(src, w));
    for (int ci = 0; ci < C; ++ci) for (int co = 0; co < C; ++co) for (int t = 0; t < 16; ++t)
        m[((size_t)co * C + ci) * 16 + t] = w[((size_t)ci * C + co) * 16 + t];
    return pack_tc_host(h, m, key, C, C, G_UP, form, conv_tc_ntile(G_UP, C, form));
}

extern "C" int sbk_pack(sbk_handle* h) {
    if (!h) return fail(SBK_ERR_ARG, "sbk_pack: null handle");
    TRY(h->w.require_all("sbk_pack"));
    CU(cudaSetDevice(h->cfg.device));
    // conv KxK [co][ci][r][s] -> [r*K+s][ci][co]
    auto conv_pack = [](float* d, const float* s, const std::vector<int64_t>& sh) {
        const int64_t co = sh[0], ci = sh[1], kk = sh[2] * sh[3];
        for (int64_t o = 0; o < co; ++o) for (int64_t i = 0; i < ci; ++i) for (int64_t t = 0; t < kk; ++t)
            d[(t * ci + i) * co + o] = s[(o * ci + i) * kk + t];
    };
    // ConvTranspose2d [ci][co][kh][kw] -> [kh*4+kw][ci][co]
    auto convt_pack = [](float* d, const float* s, const std::vector<int64_t>& sh) {
        const int64_t ci = sh[0], co = sh[1], kk = sh[2] * sh[3];
        for (int64_t i = 0; i < ci; ++i) for (int64_t o = 0; o < co; ++o) for (int64_t t = 0; t < kk; ++t)
            d[(t * ci + i) * co + o] = s[(i * co + o) * kk + t];
    };
    // first conv [co][ci][3][3] -> [ci*9+t][co]
    auto first_pack = [](float* d, const float* s, const std::vector<int64_t>& sh) {
        const int64_t co = sh[0], ci = sh[1];
        for (int64_t o = 0; o < co; ++o) for (int64_t i = 0; i < ci; ++i) for (int64_t t = 0; t < 9; ++t)
            d[(i * 9 + t) * co + o] = s[(o * ci + i) * 9 + t];
    };
    // to_qkv [384][C] -> k/v part as [ci][head*64 + {d | 32+e}]
    auto kv_pack = [](float* d, const float* s, const std::vector<int64_t>& sh) {
        const int64_t C = sh[1];
        for (int64_t ci = 0; ci < C; ++ci) for (int hd = 0; hd < kHeads; ++hd) for (int x = 0; x < 32; ++x) {
            d[ci * 256 + hd * 64 + x] = s[(128 + hd * 32 + x) * C + ci];
            d[ci * 256 + hd * 64 + 32 + x] = s[(256 + hd * 32 + x) * C + ci];
        }
    };
    // the first ResnetBlock's block1 conv (k_first_conv) and res_conv (the planar-input tail) run on CUDA cores in every mode
    const ResnetInfo& r0 = h->resnets[0];
    TRY(repack(h, r0.prefix + ".block1.block.0.weight", r0.prefix + ".block1.w", (size_t)r0.cin * 9 * r0.cout, first_pack));
    TRY(repack(h, r0.prefix + ".res_conv.weight", r0.prefix + ".res.w", (size_t)r0.cin * r0.cout, conv_pack));
    const bool x3 = h->cfg.precision == SBK_PREC_FP32X3;
    if (h->cfg.precision == SBK_PREC_FP32) {
        for (size_t k = 0; k < h->resnets.size(); ++k) {
            const ResnetInfo& r = h->resnets[k];
            if (k != 0) TRY(repack(h, r.prefix + ".block1.block.0.weight", r.prefix + ".block1.w", (size_t)r.cin * 9 * r.cout, conv_pack));
            TRY(repack(h, r.prefix + ".block2.block.0.weight", r.prefix + ".block2.w", (size_t)r.cout * 9 * r.cout, conv_pack));
            if (k != 0 && r.cin != r.cout) TRY(repack(h, r.prefix + ".res_conv.weight", r.prefix + ".res.w", (size_t)r.cin * r.cout, conv_pack));
        }
        for (auto& a : h->attns) TRY(repack(h, a.prefix + ".fn.fn.to_qkv.weight", a.prefix + ".kv.w", (size_t)a.c * 256, kv_pack));
        for (int l = 0; l < 2; ++l) {
            const std::string p = "estimator.downs." + std::to_string(l) + ".3.conv";
            const int c = h->cfg.dim << l;
            TRY(repack(h, p + ".weight", p + ".w", (size_t)c * c * 9, conv_pack));
        }
        for (int j = 0; j < 2; ++j) {
            const std::string p = "estimator.ups." + std::to_string(j) + ".3.conv";
            const int c = h->cfg.dim << (1 - j);
            TRY(repack(h, p + ".weight", p + ".w", (size_t)c * c * 16, convt_pack));
        }
        TRY(repack(h, "estimator.final_block.block.0.weight", "estimator.final_block.w", (size_t)h->cfg.dim * h->cfg.dim * 9, conv_pack));
    } else {
        const int form = h->cfg.precision == SBK_PREC_BF16 ? FORM_BF16 : (x3 ? FORM_X3 : FORM_TF32);
        for (size_t k = 0; k < h->resnets.size(); ++k) {
            const ResnetInfo& r = h->resnets[k];
            if (k != 0) TRY(pack_tc(h, r.prefix + ".block1.block.0.weight", r.prefix + ".block1.wtc", r.cout, r.cin, G_C3, form));
            TRY(pack_tc(h, r.prefix + ".block2.block.0.weight", r.prefix + ".block2.wtc", r.cout, r.cout, G_C3, form));
            if (k != 0 && r.cin != r.cout) TRY(pack_tc(h, r.prefix + ".res_conv.weight", r.prefix + ".res.wtc", r.cout, r.cin, G_PW, form));
        }
        TRY(pack_tc(h, "estimator.final_block.block.0.weight", "estimator.final_block.wtc", h->cfg.dim, h->cfg.dim, G_C3, form));
        for (auto& a : h->attns) TRY(pack_tc_kv(h, a.prefix + ".fn.fn.to_qkv.weight", a.prefix + ".kv.wtc", a.c, form));
        for (int l = 0; l < 2; ++l) {
            const std::string p = "estimator.downs." + std::to_string(l) + ".3.conv";
            TRY(pack_tc(h, p + ".weight", p + ".wtc", h->cfg.dim << l, h->cfg.dim << l, G_DOWN, form));
        }
        for (int j = 0; j < 2; ++j) {
            const std::string p = "estimator.ups." + std::to_string(j) + ".3.conv";
            TRY(pack_tc_up(h, p + ".weight", p + ".wtc", h->cfg.dim << (1 - j), form));
        }
    }
    if (h->cfg.model == SBK_MODEL_DIFFVC && h->cfg.use_ref_t) {
        const int base = h->cfg.dim_cond / 4;
        const char* nm[5] = {"block12", "block21", "block22", "block31", "block32"};
        const int ci[5] = {base, base, 2 * base, 2 * base, 4 * base}, co[5] = {2 * base, 4 * base, 4 * base, 8 * base, 8 * base};
        for (int k = 0; k < 5; ++k) {
            const std::string q = std::string("estimator.ref_block.") + nm[k];
            // the hoisted RefBlock branch (sbk_vc_conditioning) runs once per call outside the loop, on the tensor cores in
            // every precision: tf32 operands with fp32 activations for the tf32 / bf16 handles, (w_hi, correction) image pairs for
            // the fp32-class handles (fp32x3 and the CUDA-core fp32 mode, whose U-Net kernels have no InstanceNorm/GLU path)
            TRY(pack_tc(h, q + ".0.weight", q + ".wtc", co[k], ci[k], G_C3, prec_runs_x3(h->cfg.precision) ? FORM_X3 : FORM_TF32));
        }
        TRY(repack(h, "estimator.ref_block.block11.0.weight", "estimator.ref_block.block11.w", (size_t)9 * 2 * base, first_pack));
    }
    // sinusoid frequencies, SinusoidalPosEmb.forward (diffusion.py:121-122): fp32 exp of fp32(j) * fp32(-ln(1e4)/(half-1))
    {
        const int half = h->cfg.dim / 2;
        std::vector<float> f(half);
        const float neg = (float)(-(log(10000.0) / (double)(half - 1)));
        for (int j = 0; j < half; ++j) f[j] = expf((float)j * neg);
        if (!h->d_freqs) CU(cudaMalloc(&h->d_freqs, half * sizeof(float)));
        CU(cudaMemcpy(h->d_freqs, f.data(), half * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (!h->d_zero) {
        CU(cudaMalloc(&h->d_zero, 8192));
        CU(cudaMemset(h->d_zero, 0, 8192));
    }
    free_plan(h);   // packed pointers may have changed; the arena itself stays
    h->is_packed = true;
    return SBK_OK;
}

// ------------------------------------------------------------------------------------------------
// workspace layout + launch plan
// ------------------------------------------------------------------------------------------------
namespace {
struct Bufs {
    float *A[3], *Bf[3], *X[3], *Y[3], *S[3], *D[3], *U1;
    float *kv_part, *ctx, *w_eff, *b_eff;
};
}

static size_t layout(const sbk_handle* h, int B, int T, int tb_rows, Arena& ar, Bufs* bf, Plan* pl) {
    const sbk_config& c = h->cfg;
    const int dim = c.dim, H = c.n_feats;
    const size_t P[3] = {(size_t)H * T, (size_t)(H / 2) * (T / 2), (size_t)(H / 4) * (T / 4)};
    const int C[3] = {dim, dim * 2, dim * 4};
    auto f = [&](size_t n) { return (float*)ar.take(n * sizeof(float)); };
    // operand-form tensors (conv inputs): fp32, or bf16 in the bf16 mode; A[] holds the raw conv outputs (always fp32)
    const size_t osz = c.precision == SBK_PREC_BF16 ? 2 : 4;
    const bool x3 = c.precision == SBK_PREC_FP32X3;
    Bufs b{};
    // (fp32x3 keeps no correction twin of these: the conv kernels derive the correction operand in shared memory)
    auto fo = [&](size_t n) { return (float*)ar.take(n * osz); };
    for (int l = 0; l < 3; ++l) {
        const size_t n = (size_t)B * P[l] * C[l];
        b.A[l] = f(n); b.Bf[l] = fo(n); b.X[l] = fo(n); b.Y[l] = fo(n);
        b.S[l] = l > 0 ? fo(n) : nullptr;
        b.D[l] = l > 0 ? fo((size_t)B * P[l] * C[l - 1]) : nullptr;
    }
    b.U1 = fo((size_t)B * P[1] * C[1]);
    const size_t mt0 = (P[0] + attn_kv_tile_pixels() - 1) / attn_kv_tile_pixels();     // attention partials: level 0 has the most items
    b.kv_part = f((size_t)B * mt0 * kHeads * kKvPartFloats);
    b.ctx = f((size_t)B * kHeads * 1024);
    b.w_eff = f((size_t)B * C[2] * C[2] * (x3 ? 2 : 1));
    b.b_eff = f(C[2]);
    if (bf) *bf = b;
    Plan dummy;
    Plan& p = pl ? *pl : dummy;
    p.xt = f((size_t)B * H * T); p.mu = f((size_t)B * H * T); p.mask = f((size_t)B * T);
    p.spk_s = f((size_t)B * H); p.spk_in = f((size_t)B * c.spk_emb_dim);
    p.n_stat_doubles = 25 * B * kGroups * 2;
    p.stats = (double*)ar.take(p.n_stat_doubles * sizeof(double));
    p.tb_stride = h->tb_total;
    p.tb = f((size_t)tb_rows * h->tb_total);
    p.t_rows = f(tb_rows);
    p.coef = (float4*)ar.take((size_t)tb_rows * sizeof(float4));
    p.step_cur = (int*)ar.take(sizeof(int));
    p.step_next = (int*)ar.take(sizeof(int));
    p.step_end = (int*)ar.take(sizeof(int));
    p.noise_pp = (const float**)ar.take(sizeof(float*));
    if (c.model == SBK_MODEL_DIFFVC) {
        p.vc_cond = f((size_t)tb_rows * B * c.dim_cond);
        p.vc_wextra = f((size_t)tb_rows * B * 9 * dim);
        p.vc_rextra = f((size_t)tb_rows * B * dim);
    }
    return ar.bytes();
}

// rows of the per-step tables (time projections, coefficients, DiffVC conditioning): the same rule ensure_plan uses
static int table_rows(int B, int n_timesteps) { const int r = B > n_timesteps ? B : n_timesteps; return r < 64 ? 64 : r; }

extern "C" size_t sbk_workspace_bytes_n(const sbk_handle* h, int B, int T, int n_timesteps) {
    if (!h || B <= 0 || T <= 0 || T % 4 != 0 || n_timesteps < 1) return 0;
    Arena ar;
    return layout(h, B, T, table_rows(B, n_timesteps), ar, nullptr, nullptr);
}
extern "C" size_t sbk_workspace_bytes(const sbk_handle* h, int B, int T) { return sbk_workspace_bytes_n(h, B, T, 1024); }

static int build_plan(sbk_handle* h, int B, int T, int tb_rows) {
    free_plan(h);
    Plan& pl = h->plan;
    const sbk_config& c = h->cfg;
    Arena probe;
    const size_t bytes = layout(h, B, T, tb_rows, probe, nullptr, nullptr);
    if (const cudaError_t e = h->ws.reserve(bytes))
        return fail(SBK_ERR_CUDA, "out of memory: the (B=%d, T=%d) workspace needs %zu bytes (%s); free cached blocks "
                                  "(torch.cuda.empty_cache()) or split the batch", B, T, bytes, cudaGetErrorString(e));
    Arena ar = h->ws.arena();
    Bufs bf;
    layout(h, B, T, tb_rows, ar, &bf, &pl);
    pl.B = B; pl.T = T; pl.tb_rows = tb_rows;

    const int dim = c.dim, H0 = c.n_feats;
    const int Hs[3] = {H0, H0 / 2, H0 / 4}, Ws[3] = {T, T / 2, T / 4};
    const bool vc = c.model == SBK_MODEL_DIFFVC;
    const int cin0 = vc ? 3 : 2 + (c.n_spks > 1 ? 1 : 0);     // DiffVC: {mean, xt, folded conditioning channel}
    int gn_slot = 0;
    auto stats_slot = [&]() { return pl.stats + (size_t)(gn_slot++) * B * kGroups * 2; };
    auto gnref = [&](const double* st, const std::string& blk, int C, int lvl) {
        GnRef g; g.stats = st; g.gamma = h->w.get(blk + ".block.1.weight"); g.beta = h->w.get(blk + ".block.1.bias");
        g.inv_count = 1.0f / ((float)(C / kGroups) * (float)Hs[lvl] * (float)Ws[lvl]);
        return g;
    };
    auto base_ig = [&](int geom, int lvl_in, int lvl_out) {
        IgemmParams p; memset(&p, 0, sizeof(p));
        p.geom = geom; p.B = B; p.T = T;
        p.Hin = Hs[lvl_in]; p.Win = Ws[lvl_in]; p.Hout = Hs[lvl_out]; p.Wout = Ws[lvl_out];
        p.in_lvl = lvl_in; p.out_lvl = lvl_out; p.mask = pl.mask; p.step = pl.step_cur;
        return p;
    };
    const bool use_tc = c.precision != SBK_PREC_FP32;
    const bool x3 = c.precision == SBK_PREC_FP32X3;
    const int num_sms = device_sm_count();
    const char* rows_env = getenv("SBK_CONV3_ROWS");
    const int conv_rows_env = rows_env ? atoi(rows_env) : 0;
    const bool b16 = c.precision == SBK_PREC_BF16;          // operand tensors in bf16 [B][H][C/8][W][8]
    const double osz = b16 ? 2.0 : 4.0;                     // bytes per operand-tensor element
    const int fmt_raw = use_tc ? 1 : 0, fmt_opnd = b16 ? 2 : fmt_raw;
    const int form = b16 ? FORM_BF16 : (x3 ? FORM_X3 : (use_tc ? FORM_TF32 : FORM_NHWC));
    auto push = [&](Op& op, const float* dbg, int64_t numel) {
        op.dbg_ptr = dbg; op.dbg_numel = numel;
        // raw Block-conv outputs (and the attention contexts) are fp32; every other named output is an operand tensor
        // (the CUDA-core ops run in the fp32 mode only, where both formats are NHWC fp32)
        const bool raw_out = op.kind == OP_FIRST || op.kind == OP_CTX || (op.kind == OP_CONVTC && op.tc.geom == G_C3);
        op.dbg_fmt = raw_out ? fmt_raw : fmt_opnd;
        if (op.kind == OP_IGEMM) {
            const IgemmParams& p = op.ig;
            const double cin = p.c0 + p.c1, opx = (double)B * p.Hout * p.Wout, ipx = (double)B * p.Hin * p.Win;
            const double taps = p.geom == G_PW ? 1 : (p.geom == G_UP ? 4 : 9);
            op.flops = 2.0 * opx * p.Cout * cin * taps;
            op.bytes = 4.0 * (ipx * cin + (p.epi == EPI_KV ? 0.0 : opx * p.Cout) + (p.epi == EPI_RES ? opx * p.Cout : 0.0));
        } else if (op.kind == OP_FIRST) {
            op.flops = 2.0 * B * H0 * T * op.fc.C * op.fc.cin * 9;
            op.bytes = 4.0 * B * H0 * T * (op.fc.cin + op.fc.C);
        } else if (op.kind == OP_RESFINAL) {
            op.bytes = (4.0 + (op.rf.x ? osz : 0.0) + osz) * B * op.rf.H * op.rf.W * op.rf.C;
        } else if (op.kind == OP_FINAL) {
            op.flops = 2.0 * B * H0 * T * op.fn.C;
            op.bytes = 4.0 * B * H0 * T * (op.fn.C + 3.0);
        }
        pl.ops.push_back(op);
    };
    auto npix = [&](int lvl) { return (int64_t)B * Hs[lvl] * Ws[lvl]; };

    // In the tensor-core modes every conv input is kept in HBM in "operand form" (already masked; Block activations
    // already GroupNorm-ed/Mish-ed/time-biased), so a conv's A path is a pure copy.  `store_masked` marks outputs
    // whose consumers all multiply by the mask anyway (everything except the tensors fed to LinearAttention, which
    // reads the unmasked x, diffusion.py:192,202,210).
    auto tc_conv = [&](const std::string& name, int geom, const std::string& wkey, const std::string& bkey, int lvl,
                       const float* in0, int c0, const float* in1, int c1, int cout, float* out, double* st) {
        Op op; op.name = name; op.kind = OP_CONVTC;
        ConvTcParams& p = op.tc; memset(&p, 0, sizeof(p));
        p.geom = geom; p.in0 = in0; p.c0 = c0; p.in1 = in1; p.c1 = c1; p.H = Hs[lvl]; p.W = Ws[lvl]; p.B = B;
        p.Ho = p.H; p.Wo = p.W;
        p.wpk = h->w.get(wkey); p.bias = bkey.empty() ? nullptr : h->w.get(bkey); p.out = out; p.Cout = cout;
        p.epi = EPI_PLAIN; p.ostats = st; p.mask = pl.mask; p.T = T; p.lvl = lvl; p.zero_page = h->d_zero;
        p.form = form; p.nt = conv_tc_ntile(geom, cout, form);
        if (geom == G_C3) {
            // Two-row tiles (2 rows x 128 pixels x 64 channels) bring a third less operand traffic from L2 per MAC than
            // one-row tiles, but there are half as many per 64 channels.  A persistent grid runs ceil(tiles / SMs) waves,
            // so they are used only from 4 waves on, where the last wave's round-up costs at most a quarter of a wave
            // more than in the one-row layout.  SBK_CONV3_ROWS = 1 | 2 overrides the choice (A/B runs of one process).
            const long long wt = (Ws[lvl] + 127) / 128;
            const long long tiles2 = (long long)B * wt * ((Hs[lvl] + 1) / 2) * (cout / 64);
            bool two = tiles2 >= 4LL * num_sms;
            if (conv_rows_env == 1 || conv_rows_env == 2) two = conv_rows_env == 2;
            const bool wide = p.nt == 128;
            if (two && (!wide || h->w.packed.count(wkey + "64"))) {
                p.rows = 2;
                if (wide) { p.nt = 64; p.wpk = h->w.get(wkey + "64"); }
            } else if (wide) {
                // tiles of one row x 128 pixels x 128 channels; when they cannot fill half the SMs, use 64-wide N tiles instead
                const long long tiles = (long long)B * wt * Hs[lvl] * (cout / 128);
                if (tiles * 2 <= num_sms && h->w.packed.count(wkey + "64")) { p.nt = 64; p.wpk = h->w.get(wkey + "64"); }
            }
        }
        const double taps = geom == G_PW ? 1.0 : (geom == G_UP ? 4.0 : 9.0);
        op.flops = 2.0 * B * Hs[lvl] * Ws[lvl] * cout * (c0 + c1) * taps;
        op.bytes = (double)B * Hs[lvl] * Ws[lvl] * (osz * (c0 + c1) + (geom == G_C3 ? 4.0 : osz) * cout);
        return op;
    };
    // one Block conv (Conv3x3 + bias + GN statistics of the raw output) on the CUDA-core path
    auto ffma_block_conv = [&](const std::string& name, const std::string& wkey, const std::string& bkey, int lvl,
                               const float* in0, int c0, const float* in1, int c1, int cout, float* out, double* st,
                               int pro, const GnRef* pgn, int tb_k) {
        Op op; op.name = name; op.kind = OP_IGEMM;
        op.ig = base_ig(G_C3, lvl, lvl);
        IgemmParams& p = op.ig;
        p.in0 = in0; p.c0 = c0; p.in1 = in1; p.c1 = c1; p.w = h->w.get(wkey); p.bias = h->w.get(bkey);
        p.out = out; p.Cout = cout; p.pro = pro; p.epi = EPI_PLAIN; p.ostats = st;
        if (pgn) { p.pgn = *pgn; p.tb = pl.tb + h->tb_off[tb_k]; p.tb_stride = pl.tb_stride; }
        push(op, out, npix(lvl) * cout);
    };
    // ResnetBlock (diffusion.py:74-79) at level lvl: in (in0|in1) -> out
    auto resnet = [&](int k, int lvl, const float* in0, int c0, const float* in1, int c1, float* out, bool store_masked) {
        const ResnetInfo& r = h->resnets[k];
        float* A = bf.A[lvl]; float* Bb = bf.Bf[lvl];
        double* st1 = stats_slot(); double* st2 = stats_slot();
        // ---- block1 conv -> raw h1 (A)
        if (k == 0) {
            Op op; op.kind = OP_FIRST; op.name = r.prefix + ".block1.raw";
            FirstConvParams& p = op.fc; memset(&p, 0, sizeof(p));
            p.mu = pl.mu; p.xt = pl.xt; p.spk_s = pl.spk_s; p.mask = pl.mask;
            p.w = h->w.get(r.prefix + ".block1.w"); p.bias = h->w.get(r.prefix + ".block1.block.0.bias");
            p.out = A; p.ostats = st1; p.B = B; p.H = H0; p.T = T; p.cin = cin0; p.C = r.cout; p.chw4 = use_tc ? 1 : 0;
            if (vc) { p.w_extra = pl.vc_wextra; p.step = pl.step_cur; }
            pl.first_op = (int)pl.ops.size();
            push(op, A, npix(lvl) * r.cout);
        } else if (use_tc) {
            Op op = tc_conv(r.prefix + ".block1.raw", G_C3, r.prefix + ".block1.wtc", r.prefix + ".block1.block.0.bias", lvl,
                            in0, c0, in1, c1, r.cout, A, st1);
            push(op, A, npix(lvl) * r.cout);
        } else {
            ffma_block_conv(r.prefix + ".block1.raw", r.prefix + ".block1.w", r.prefix + ".block1.block.0.bias", lvl,
                            in0, c0, in1, c1, r.cout, A, st1, PRO_MASK, nullptr, k);
        }
        // ---- block2 conv -> raw h2 (FFMA: A -> Bb with the GN/Mish prologue fused; TC: A -> act (Bb) -> A)
        const GnRef g1 = gnref(st1, r.prefix + ".block1", r.cout, lvl);
        float* h2 = Bb;
        if (use_tc) {
            {
                Op op; op.kind = OP_GNACT; op.name = r.prefix + ".block1.act";
                GnActParams& p = op.ga; memset(&p, 0, sizeof(p));
                p.raw = A; p.gn = g1; p.tb = pl.tb + h->tb_off[k]; p.tb_stride = pl.tb_stride; p.step = pl.step_cur;
                p.mask = pl.mask; p.T = T; p.lvl = lvl; p.out = Bb; p.B = B; p.H = Hs[lvl]; p.W = Ws[lvl]; p.C = r.cout;
                p.form = form;
                op.bytes = (4.0 + osz) * npix(lvl) * r.cout;
                push(op, nullptr, 0);
            }
            Op op = tc_conv(r.prefix + ".block2.raw", G_C3, r.prefix + ".block2.wtc", r.prefix + ".block2.block.0.bias", lvl,
                            Bb, r.cout, nullptr, 0, r.cout, A, st2);
            push(op, A, npix(lvl) * r.cout);
            h2 = A;
        } else {
            ffma_block_conv(r.prefix + ".block2.raw", r.prefix + ".block2.w", r.prefix + ".block2.block.0.bias", lvl,
                            A, r.cout, nullptr, 0, r.cout, Bb, st2, PRO_GN, &g1, k);
        }
        // ---- tail: out = Mish(GN(h2))*mask + res(x*mask)
        const GnRef g2 = gnref(st2, r.prefix + ".block2", r.cout, lvl);
        if (k == 0 || r.cin == r.cout) {
            Op op; op.kind = OP_RESFINAL; op.name = r.prefix + ".out";
            ResFinalParams& p = op.rf; memset(&p, 0, sizeof(p));
            p.h2raw = h2; p.gn = g2;
            p.mask = pl.mask; p.T = T; p.lvl = lvl; p.out = out; p.B = B; p.H = Hs[lvl]; p.W = Ws[lvl]; p.C = r.cout;
            p.out_mask = store_masked ? 1 : 0; p.form = form;
            if (k == 0) {
                p.x = nullptr; p.mu = pl.mu; p.xt = pl.xt; p.spk_s = pl.spk_s; p.cin = cin0;
                p.wres = h->w.get(r.prefix + ".res.w"); p.bres = h->w.get(r.prefix + ".res_conv.bias");
                if (vc) { p.r_extra = pl.vc_rextra; p.step = pl.step_cur; }
                pl.first_res_op = (int)pl.ops.size();
            } else {
                p.x = in0;
            }
            op.bytes = (4.0 + (k == 0 ? 0.0 : osz) + osz) * npix(lvl) * r.cout;
            push(op, out, npix(lvl) * r.cout);
        } else if (use_tc) {
            Op op = tc_conv(r.prefix + ".out", G_PW, r.prefix + ".res.wtc", r.prefix + ".res_conv.bias", lvl,
                            in0, c0, in1, c1, r.cout, out, nullptr);
            op.tc.epi = EPI_RES; op.tc.rraw = h2; op.tc.rgn = g2; op.tc.out_mask = store_masked ? 1 : 0;
            op.bytes += 4.0 * npix(lvl) * r.cout;          // + the fp32 h2raw side input
            push(op, out, npix(lvl) * r.cout);
        } else {
            Op op; op.kind = OP_IGEMM; op.name = r.prefix + ".out";
            op.ig = base_ig(G_PW, lvl, lvl);
            IgemmParams& p = op.ig;
            p.in0 = in0; p.c0 = c0; p.in1 = in1; p.c1 = c1;
            p.w = h->w.get(r.prefix + ".res.w"); p.bias = h->w.get(r.prefix + ".res_conv.bias");
            p.out = out; p.Cout = r.cout; p.pro = PRO_MASK; p.epi = EPI_RES;
            p.rraw = h2; p.rgn = g2;
            push(op, out, npix(lvl) * r.cout);
        }
    };
    // Residual(Rezero(LinearAttention)) (diffusion.py:39-46,82-110)
    auto attention = [&](int k, int lvl, const float* x, float* out) {
        const AttnInfo& a = h->attns[k];
        int mt = igemm_mtiles(G_PW, Hs[lvl], Ws[lvl], Hs[lvl], Ws[lvl]);
        if (use_tc) {
            // k|v projection, softmax and context partials fused on the tensor cores (k_attn_kv_wg): k and v never reach
            // HBM.  One partial per item of attn_kv_tile_pixels() pixels x 4 heads: an utterance is cut at the same pixels
            // whatever batch it sits in.
            Op op = tc_conv(a.prefix + ".kvpart", G_PW, a.prefix + ".kv.wtc", "", lvl, x, a.c, nullptr, 0, 256, nullptr, nullptr);
            op.tc.epi = EPI_KV; op.tc.kv_part = bf.kv_part;
            op.bytes = osz * npix(lvl) * a.c;
            op.flops += 2.0 * npix(lvl) * 4096.0;
            mt = (Hs[lvl] * Ws[lvl] + attn_kv_tile_pixels() - 1) / attn_kv_tile_pixels();
            push(op, nullptr, 0);
        } else {
            Op op; op.kind = OP_IGEMM; op.name = a.prefix + ".kvpart";
            op.ig = base_ig(G_PW, lvl, lvl);
            IgemmParams& p = op.ig;
            p.in0 = x; p.c0 = a.c; p.w = h->w.get(a.prefix + ".kv.w"); p.Cout = 256; p.pro = PRO_NONE; p.epi = EPI_KV;
            p.kv_part = bf.kv_part; p.out = nullptr;
            push(op, nullptr, 0);
        }
        {
            Op op; op.kind = OP_CTX; op.name = a.prefix + ".ctx";
            op.cx.kv_part = bf.kv_part; op.cx.mtiles = mt; op.cx.ctx = bf.ctx; op.cx.B = B;
            push(op, bf.ctx, (int64_t)B * kHeads * 1024);
        }
        {
            Op op; op.kind = OP_MIX; op.name = a.prefix + ".mix";
            AttnMixParams& p = op.mx; memset(&p, 0, sizeof(p));
            p.ctx = bf.ctx; p.wq = h->w.get(a.prefix + ".fn.fn.to_qkv.weight"); p.wout = h->w.get(a.prefix + ".fn.fn.to_out.weight");
            p.bout = h->w.get(a.prefix + ".fn.fn.to_out.bias"); p.g = h->w.get(a.prefix + ".fn.g");
            p.w_eff = bf.w_eff; p.b_eff = bf.b_eff; p.B = B; p.C = a.c;
            if (use_tc) { p.nt = conv_tc_ntile(G_PW, a.c, form); p.form = form; }
            push(op, nullptr, 0);
        }
        if (use_tc) {
            // the per-sample (I + g P_b) matrix is written by k_attn_mix directly in the tensor-core weight-stage layout
            Op op = tc_conv(a.prefix + ".out", G_PW, "", "", lvl, x, a.c, nullptr, 0, a.c, out, nullptr);
            op.tc.wpk = bf.w_eff; op.tc.bias = bf.b_eff;
            op.tc.w_bstride_bytes = (long long)conv_tc_wimg_bytes(conv_tc_wimg(G_PW, form, op.tc.nt, a.c), a.c);
            op.tc.out_mask = 1; op.tc.addin = x;
            op.bytes += osz * npix(lvl) * a.c;
            push(op, out, npix(lvl) * a.c);
        } else {
            Op op; op.kind = OP_IGEMM; op.name = a.prefix + ".out";
            op.ig = base_ig(G_PW, lvl, lvl);
            IgemmParams& p = op.ig;
            p.in0 = x; p.c0 = a.c; p.w = bf.w_eff; p.w_bstride = (long long)a.c * a.c; p.bias = bf.b_eff;
            p.out = out; p.Cout = a.c; p.pro = PRO_NONE; p.epi = EPI_PLAIN;
            push(op, out, npix(lvl) * a.c);
        }
    };
    auto resample = [&](int geom, const std::string& pre, int lvl_in, int lvl_out, const float* x, int C, float* out) {
        if (use_tc) {
            Op op = tc_conv(pre + ".out", geom, pre + ".conv.wtc", pre + ".conv.bias", lvl_in, x, C, nullptr, 0, C, out, nullptr);
            op.tc.Ho = Hs[lvl_out]; op.tc.Wo = Ws[lvl_out]; op.tc.lvl = lvl_out; op.tc.out_mask = 1;
            op.flops = 2.0 * npix(lvl_out) * C * C * (geom == G_UP ? 4.0 : 9.0);
            op.bytes = osz * C * (npix(lvl_in) + npix(lvl_out));
            push(op, out, npix(lvl_out) * C);
            return;
        }
        Op op; op.kind = OP_IGEMM; op.name = pre + ".out";
        op.ig = base_ig(geom, lvl_in, lvl_out);
        IgemmParams& p = op.ig;
        p.in0 = x; p.c0 = C; p.w = h->w.get(pre + ".conv.w"); p.bias = h->w.get(pre + ".conv.bias");
        p.out = out; p.Cout = C; p.pro = PRO_MASK; p.epi = EPI_PLAIN;
        push(op, out, npix(lvl_out) * C);
    };

    const int C1 = dim, C2 = dim * 2, C3 = dim * 4;
    // downs (diffusion.py:190-197)
    const bool sm = use_tc;     // store-masked convention only in the tensor-core modes
    resnet(0, 0, nullptr, cin0, nullptr, 0, bf.X[0], sm);
    resnet(1, 0, bf.X[0], C1, nullptr, 0, bf.Y[0], false);          // feeds attention: unmasked
    attention(0, 0, bf.Y[0], bf.X[0]);
    resample(G_DOWN, "estimator.downs.0.3", 0, 1, bf.X[0], C1, bf.D[1]);
    resnet(2, 1, bf.D[1], C1, nullptr, 0, bf.X[1], sm);
    resnet(3, 1, bf.X[1], C2, nullptr, 0, bf.Y[1], false);
    attention(1, 1, bf.Y[1], bf.S[1]);
    resample(G_DOWN, "estimator.downs.1.3", 1, 2, bf.S[1], C2, bf.D[2]);
    resnet(4, 2, bf.D[2], C2, nullptr, 0, bf.X[2], sm);
    resnet(5, 2, bf.X[2], C3, nullptr, 0, bf.Y[2], false);
    attention(2, 2, bf.Y[2], bf.S[2]);
    // mid (:199-203); Identity()(x*mask) is absorbed by the consumers' masking
    resnet(6, 2, bf.S[2], C3, nullptr, 0, bf.X[2], false);
    attention(3, 2, bf.X[2], bf.Y[2]);
    resnet(7, 2, bf.Y[2], C3, nullptr, 0, bf.X[2], sm);
    // ups (:205-211): cat(x, skip) is pure addressing (two input pointers)
    resnet(8, 2, bf.X[2], C3, bf.S[2], C3, bf.Y[2], sm);
    resnet(9, 2, bf.Y[2], C2, nullptr, 0, bf.X[2], false);
    attention(4, 2, bf.X[2], bf.Y[2]);
    resample(G_UP, "estimator.ups.0.3", 2, 1, bf.Y[2], C2, bf.U1);
    resnet(10, 1, bf.U1, C2, bf.S[1], C2, bf.X[1], sm);
    resnet(11, 1, bf.X[1], C1, nullptr, 0, bf.Y[1], false);
    attention(5, 1, bf.Y[1], bf.X[1]);
    resample(G_UP, "estimator.ups.1.3", 1, 0, bf.X[1], C1, bf.Y[0]);
    // final_block + final_conv + update (:213-216)
    double* stf = stats_slot();
    if (use_tc) {
        Op op = tc_conv("estimator.final_block.raw", G_C3, "estimator.final_block.wtc", "estimator.final_block.block.0.bias", 0,
                        bf.Y[0], C1, nullptr, 0, C1, bf.A[0], stf);
        push(op, bf.A[0], npix(0) * C1);
    } else {
        ffma_block_conv("estimator.final_block.raw", "estimator.final_block.w", "estimator.final_block.block.0.bias", 0,
                        bf.Y[0], C1, nullptr, 0, C1, bf.A[0], stf, PRO_MASK, nullptr, 0);
    }
    {
        Op op; op.kind = OP_FINAL; op.name = "estimator.out";
        FinalParams& p = op.fn; memset(&p, 0, sizeof(p));
        p.raw = bf.A[0]; p.gn = gnref(stf, "estimator.final_block", C1, 0);
        p.wfin = h->w.get("estimator.final_conv.weight"); p.bfin = h->w.get("estimator.final_conv.bias");
        p.mask = pl.mask; p.mu = pl.mu; p.xt_in = pl.xt; p.xt_out = pl.xt;
        p.coef = pl.coef; p.step = pl.step_cur; p.B = B; p.H = H0; p.T = T; p.C = C1; p.chw4 = use_tc ? 1 : 0; p.exact = x3 ? 1 : 0;
        pl.final_op = (int)pl.ops.size();
        push(op, nullptr, 0);
    }
    pl.launches_per_step = (int)pl.ops.size() + 1;
    return SBK_OK;
}

static int launch_op(const Op& op, cudaStream_t s) {
    switch (op.kind) {
        case OP_FIRST: return launch_first_conv(op.fc, s);
        case OP_IGEMM: return launch_igemm(op.ig, s);
        case OP_RESFINAL: return launch_resfinal(op.rf, s);
        case OP_CTX: return launch_attn_ctx(op.cx, s);
        case OP_MIX: return launch_attn_mix(op.mx, s);
        case OP_FINAL: return launch_final(op.fn, s);
        case OP_CONVTC: return launch_conv_tc(op.tc, s);
        case OP_GNACT: return launch_gn_act(op.ga, s);
    }
    return -1;
}

// enqueue one estimator evaluation (+ update); returns the number of launches, or -1 when a launcher refused (a
// per-device attribute could not be set, an unsupported layout): the caller turns that into SBK_ERR_CUDA
static int run_ops(sbk_handle* h, cudaStream_t s) {
    Plan& pl = h->plan;
    StepBeginParams sb{pl.stats, pl.n_stat_doubles, pl.step_cur, pl.step_next};
    int n = launch_step_begin(sb, s);
    for (auto& op : pl.ops) {
        const int k = launch_op(op, s);
        if (k < 0) { fail(SBK_ERR_CUDA, "launch of '%s' was refused (device attribute / layout)", op.name.c_str()); return -1; }
        n += k;
        if (h->capture && op.dbg_ptr && op.dbg_numel > 0) {
            const size_t esz = snap_elem_bytes(op.dbg_fmt);
            if (!op.dbg_copy) cudaMalloc(&op.dbg_copy, op.dbg_numel * esz);
            cudaMemcpyAsync(op.dbg_copy, op.dbg_ptr, op.dbg_numel * esz, cudaMemcpyDeviceToDevice, s);
        }
    }
    return n;
}

static int ensure_plan(sbk_handle* h, int B, int T, int rows) {
    if (!h->is_packed) return fail(SBK_ERR_STATE, "weights not packed: call sbk_set_weight for every key, then sbk_pack");
    if (B <= 0 || T <= 0 || T % 4 != 0) return fail(SBK_ERR_ARG, "B must be > 0 and T a positive multiple of 4 (fix_len_compatibility), got B=%d T=%d", B, T);
    CU(cudaSetDevice(h->cfg.device));
    Plan& pl = h->plan;
    if (pl.B == B && pl.T == T && pl.tb_rows >= rows) return SBK_OK;     // (a freed plan has B = 0)
    int cap = rows < 64 ? 64 : rows;
    if (pl.B == B && pl.T == T && cap < pl.tb_rows) cap = pl.tb_rows;
    return build_plan(h, B, T, cap);
}

static int time_table(sbk_handle* h, int rows, cudaStream_t s) {
    Plan& pl = h->plan;
    TimeTableParams p; memset(&p, 0, sizeof(p));
    p.t_rows = pl.t_rows; p.rows = rows; p.freqs = h->d_freqs; p.pe_scale = h->cfg.pe_scale; p.dim = h->cfg.dim;
    p.w0 = h->w.get("estimator.mlp.0.weight"); p.b0 = h->w.get("estimator.mlp.0.bias");
    p.w2 = h->w.get("estimator.mlp.2.weight"); p.b2 = h->w.get("estimator.mlp.2.bias");
    p.nproj = (int)h->resnets.size();
    for (int k = 0; k < p.nproj; ++k) {
        p.pw[k] = h->w.get(h->resnets[k].prefix + ".mlp.1.weight");
        p.pb[k] = h->w.get(h->resnets[k].prefix + ".mlp.1.bias");
        p.pc[k] = h->resnets[k].cout; p.poff[k] = h->tb_off[k];
    }
    p.tb = pl.tb; p.tb_stride = pl.tb_stride;
    return launch_time_table(p, s);
}

static int speaker(sbk_handle* h, const float* spk, int B, cudaStream_t s) {
    if (h->cfg.n_spks < 2) return 0;
    Plan& pl = h->plan;
    SpkParams p; p.spk = spk; p.B = B; p.E = h->cfg.spk_emb_dim; p.n_feats = h->cfg.n_feats; p.out = pl.spk_s;
    p.w0 = h->w.get("estimator.spk_mlp.0.weight"); p.b0 = h->w.get("estimator.spk_mlp.0.bias");
    p.w2 = h->w.get("estimator.spk_mlp.2.weight"); p.b2 = h->w.get("estimator.spk_mlp.2.bias");
    return launch_spk(p, s);
}

static void set_mode(Plan& pl, int mode, bool per_sample_t, float* out) {
    for (auto& op : pl.ops)
        if (op.kind == OP_IGEMM && op.ig.pro == PRO_GN) op.ig.tb_per_sample = per_sample_t ? 1 : 0;
    for (auto& op : pl.ops)
        if (op.kind == OP_GNACT) op.ga.tb_per_sample = per_sample_t ? 1 : 0;
    if (pl.first_op >= 0) pl.ops[pl.first_op].fc.extra_per_sample_row = per_sample_t ? 1 : 0;
    if (pl.first_res_op >= 0) pl.ops[pl.first_res_op].rf.extra_per_sample_row = per_sample_t ? 1 : 0;
    FinalParams& f = pl.ops[pl.final_op].fn;
    f.mode = mode; f.xt_out = out; f.noise_pp = pl.noise_pp;
}

extern "C" int sbk_estimator(sbk_handle* h, const float* x, const float* mask, const float* mu, const float* t,
                             const float* spk, float* out, int B, int T, void* stream) {
    if (!h || !x || !mask || !mu || !t || !out) return fail(SBK_ERR_ARG, "sbk_estimator: null argument");
    if (h->cfg.model != SBK_MODEL_GRADTTS) return fail(SBK_ERR_ARG, "sbk_estimator: this handle is a DiffVC model, use sbk_vc_*");
    if (h->cfg.n_spks > 1 && !spk) return fail(SBK_ERR_ARG, "sbk_estimator: spk is required when n_spks > 1");
    TRY(ensure_plan(h, B, T, B));
    cudaStream_t s = (cudaStream_t)stream;
    Plan& pl = h->plan;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    CU(cudaMemcpyAsync(pl.xt, x, nb, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.mu, mu, nb, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.mask, mask, (size_t)B * T * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.t_rows, t, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, s));
    int64_t n = 0;
    n += speaker(h, spk, B, s);
    n += time_table(h, B, s);
    set_mode(pl, 0, true, out);
    k_set_int<<<1, 1, 0, s>>>(pl.step_next, 0); ++n;
    { const int k = run_ops(h, s); if (k < 0) return SBK_ERR_CUDA; n += k; }
    CU(cudaGetLastError());
    h->last_launches = n;
    return SBK_OK;
}

// host-side coefficients of step i, with the reference's fp32 rounding order (diffusion.py:259-263,269,273)
static void step_coefs(const sbk_config& c, int n_timesteps, int i, float* t_out, float4* cf) {
    const double hd = 1.0 / n_timesteps;
    const float t = (float)(1.0 - (i + 0.5) * hd);             // python double scalar * ones(fp32)
    const float beta = c.beta_min + (float)((double)c.beta_max - (double)c.beta_min) * t;
    const float hf = (float)hd;
    *t_out = t;
    *cf = make_float4(beta, hf, sqrtf(beta * hf), 0.f);
}

// Build (once per plan and sampler mode) the single-launch loop graph.  Returns false - and the caller falls back to one
// graph launch per step - if this driver / toolkit refuses conditional nodes; the reason is kept in sbk_last_error().
static bool build_loop_graph(sbk_handle* h, int mode) {
    Plan& pl = h->plan;
    if (pl.loop_state[mode] != 0) return pl.loop_state[mode] > 0;
    pl.loop_state[mode] = -1;
    if (!h->cap_stream && cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking) != cudaSuccess) return false;
    cudaGraph_t g = nullptr;
    cudaGraphExec_t exec = nullptr;
    bool ok = false;
    do {
        if (cudaGraphCreate(&g, 0) != cudaSuccess) break;
        cudaGraphConditionalHandle handle;
        // default 1 at every launch: the body runs at least once (callers never launch an empty slice)
        if (cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault) != cudaSuccess) break;
        cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};     // (the union has no default constructor)
        np.type = cudaGraphNodeTypeConditional;
        np.conditional.handle = handle;
        np.conditional.type = cudaGraphCondTypeWhile;
        np.conditional.size = 1;
        cudaGraphNode_t node;
        if (cudaGraphAddNode(&node, g, nullptr, 0, &np) != cudaSuccess) break;
        cudaGraph_t body = np.conditional.phGraph_out[0];
        if (cudaStreamBeginCaptureToGraph(h->cap_stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal) != cudaSuccess) break;
        const int k = run_ops(h, h->cap_stream);
        k_loop_cond<<<1, 1, 0, h->cap_stream>>>(handle, pl.step_next, pl.step_end);
        cudaGraph_t dummy = nullptr;
        if (cudaStreamEndCapture(h->cap_stream, &dummy) != cudaSuccess || k < 0) break;
        if (cudaGraphInstantiate(&exec, g, 0) != cudaSuccess) break;
        ok = true;
    } while (0);
    if (!ok) {
        const cudaError_t e = cudaGetLastError();
        fail(SBK_ERR_CUDA, "single-launch loop graph unavailable (%s): falling back to one graph launch per step", cudaGetErrorString(e));
        if (exec) cudaGraphExecDestroy(exec);
    } else {
        pl.gloop[mode] = exec;
        pl.loop_state[mode] = 1;
    }
    if (g) cudaGraphDestroy(g);
    return ok;
}

static int run_steps(sbk_handle* h, const float* noise, int B, int T, int N, int s0, int s1, int stoc, cudaStream_t s, int64_t* launches) {
    Plan& pl = h->plan;
    const int mode = h->cfg.model == SBK_MODEL_DIFFVC ? 3 : (stoc ? 2 : 1);
    set_mode(pl, mode, false, pl.xt);
    // the kernel indexes noise by absolute step: bias the base so slab s0 is the first one supplied
    const float* nbase = noise ? noise - (long long)s0 * B * h->cfg.n_feats * T : nullptr;
    k_set_int<<<1, 1, 0, s>>>(pl.step_next, s0);
    k_set_ptr<<<1, 1, 0, s>>>(pl.noise_pp, nbase);
    *launches += 2;
    h->last_host_launches = s1 - s0;
    if (h->cfg.use_graph && s1 > s0 && build_loop_graph(h, mode)) {
        // one host launch: WHILE(step_next < step_end) { one reverse step }
        k_set_int<<<1, 1, 0, s>>>(pl.step_end, s1);
        CU(cudaGraphLaunch(pl.gloop[mode], s));
        *launches += 1 + (int64_t)(s1 - s0) * (pl.launches_per_step + 1);
        h->last_host_launches = 1;
    } else if (h->cfg.use_graph) {
        if (!pl.gexec[mode]) {
            if (!h->cap_stream) CU(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
            cudaGraph_t g = nullptr;
            CU(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
            const int k = run_ops(h, h->cap_stream);
            CU(cudaStreamEndCapture(h->cap_stream, &g));
            if (k < 0) { if (g) cudaGraphDestroy(g); return SBK_ERR_CUDA; }
            CU(cudaGraphInstantiate(&pl.gexec[mode], g, 0));
            CU(cudaGraphDestroy(g));
        }
        for (int i = s0; i < s1; ++i) CU(cudaGraphLaunch(pl.gexec[mode], s));
        *launches += (int64_t)(s1 - s0) * pl.launches_per_step;
    } else {
        for (int i = s0; i < s1; ++i) { const int k = run_ops(h, s); if (k < 0) return SBK_ERR_CUDA; *launches += k; }
    }
    CU(cudaGetLastError());
    (void)N;
    return SBK_OK;
}

static int prepare_loop(sbk_handle* h, const float* mask, const float* mu, const float* spk, int B, int T, int N,
                        cudaStream_t s, int64_t* launches) {
    Plan& pl = h->plan;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    if (mu != pl.mu) CU(cudaMemcpyAsync(pl.mu, mu, nb, cudaMemcpyDeviceToDevice, s));
    if (mask != pl.mask) CU(cudaMemcpyAsync(pl.mask, mask, (size_t)B * T * sizeof(float), cudaMemcpyDeviceToDevice, s));
    std::vector<float> tr(N); std::vector<float4> cf(N);
    for (int i = 0; i < N; ++i) step_coefs(h->cfg, N, i, &tr[i], &cf[i]);
    // pageable-source async copies are staged before returning, so the vectors may die at scope exit
    CU(cudaMemcpyAsync(pl.t_rows, tr.data(), N * sizeof(float), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(pl.coef, cf.data(), N * sizeof(float4), cudaMemcpyHostToDevice, s));
    *launches += speaker(h, spk, B, s);
    *launches += time_table(h, N, s);
    return SBK_OK;
}

extern "C" int sbk_reverse_steps(sbk_handle* h, float* xt, const float* mask, const float* mu, const float* spk,
                                 const float* noise, int B, int T, int n_timesteps, int step_begin, int step_end,
                                 int stoc, void* stream) {
    if (!h || !xt || !mask || !mu) return fail(SBK_ERR_ARG, "sbk_reverse_steps: null argument");
    if (n_timesteps < 1 || step_begin < 0 || step_end > n_timesteps || step_begin > step_end)
        return fail(SBK_ERR_ARG, "sbk_reverse_steps: bad step range [%d,%d) of %d", step_begin, step_end, n_timesteps);
    if (stoc && !noise) return fail(SBK_ERR_ARG, "sbk_reverse_steps: stoc=1 needs a noise buffer");
    if (h->cfg.model != SBK_MODEL_GRADTTS) return fail(SBK_ERR_ARG, "sbk_reverse_steps: this handle is a DiffVC model, use sbk_vc_*");
    if (h->cfg.n_spks > 1 && !spk) return fail(SBK_ERR_ARG, "sbk_reverse_steps: spk is required when n_spks > 1");
    TRY(ensure_plan(h, B, T, n_timesteps));
    cudaStream_t s = (cudaStream_t)stream;
    Plan& pl = h->plan;
    int64_t n = 0;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    CU(cudaMemcpyAsync(pl.xt, xt, nb, cudaMemcpyDeviceToDevice, s));
    TRY(prepare_loop(h, mask, mu, spk, B, T, n_timesteps, s, &n));
    TRY(run_steps(h, noise, B, T, n_timesteps, step_begin, step_end, stoc, s, &n));
    CU(cudaMemcpyAsync(xt, pl.xt, nb, cudaMemcpyDeviceToDevice, s));
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_reverse_diffusion(sbk_handle* h, const float* z, const float* mask, const float* mu, const float* spk,
                                     const float* noise, float* out, int B, int T, int n_timesteps, int stoc, void* stream) {
    if (!h || !z || !mask || !mu || !out) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion: null argument");
    if (n_timesteps < 1) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion: n_timesteps must be >= 1");
    if (stoc && !noise) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion: stoc=1 needs a noise buffer");
    if (h->cfg.model != SBK_MODEL_GRADTTS) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion: this handle is a DiffVC model, use sbk_vc_*");
    if (h->cfg.n_spks > 1 && !spk) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion: spk is required when n_spks > 1");
    TRY(ensure_plan(h, B, T, n_timesteps));
    cudaStream_t s = (cudaStream_t)stream;
    Plan& pl = h->plan;
    int64_t n = 0;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    TRY(prepare_loop(h, mask, mu, spk, B, T, n_timesteps, s, &n));
    n += launch_scale_mask(z, pl.mask, pl.xt, 0, B, h->cfg.n_feats, T, s);     // xt = z * mask (:256)
    TRY(run_steps(h, noise, B, T, n_timesteps, 0, n_timesteps, stoc, s, &n));
    CU(cudaMemcpyAsync(out, pl.xt, nb, cudaMemcpyDeviceToDevice, s));
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_reverse_diffusion_host(sbk_handle* h, const float* z, const float* mask, const float* mu, const float* spk,
                                          const float* noise, float* out, int B, int T, int n_timesteps, int stoc) {
    if (!h || !z || !mask || !mu || !out) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion_host: null argument");
    if (n_timesteps < 1) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion_host: n_timesteps must be >= 1");
    if (stoc && !noise) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion_host: stoc=1 needs a noise buffer");
    if (h->cfg.model != SBK_MODEL_GRADTTS) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion_host: this handle is a DiffVC model, use sbk_vc_*");
    if (h->cfg.n_spks > 1 && !spk) return fail(SBK_ERR_ARG, "sbk_reverse_diffusion_host: spk is required when n_spks > 1");
    TRY(ensure_plan(h, B, T, n_timesteps));
    if (!h->cap_stream) CU(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    cudaStream_t s = h->cap_stream;
    Plan& pl = h->plan;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    float* d_z = nullptr; float* d_noise = nullptr;
    CU(cudaMallocAsync(&d_z, nb, s));
    CU(cudaMemcpyAsync(d_z, z, nb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(pl.mu, mu, nb, cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(pl.mask, mask, (size_t)B * T * sizeof(float), cudaMemcpyHostToDevice, s));
    if (spk) CU(cudaMemcpyAsync(pl.spk_in, spk, (size_t)B * h->cfg.spk_emb_dim * sizeof(float), cudaMemcpyHostToDevice, s));
    if (stoc) {
        CU(cudaMallocAsync(&d_noise, nb * n_timesteps, s));
        CU(cudaMemcpyAsync(d_noise, noise, nb * n_timesteps, cudaMemcpyHostToDevice, s));
    }
    int64_t n = 0;
    TRY(prepare_loop(h, pl.mask, pl.mu, spk ? pl.spk_in : nullptr, B, T, n_timesteps, s, &n));
    n += launch_scale_mask(d_z, pl.mask, pl.xt, 0, B, h->cfg.n_feats, T, s);
    TRY(run_steps(h, d_noise, B, T, n_timesteps, 0, n_timesteps, stoc, s, &n));
    CU(cudaMemcpyAsync(out, pl.xt, nb, cudaMemcpyDeviceToHost, s));
    CU(cudaFreeAsync(d_z, s));
    if (d_noise) CU(cudaFreeAsync(d_noise, s));
    CU(cudaStreamSynchronize(s));
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_profile_ops(sbk_handle* h, float* ms, double* flops, double* bytes, int cap, int* n_ops) {
    if (!h || !ms || !n_ops) return fail(SBK_ERR_ARG, "sbk_profile_ops: null argument");
    Plan& pl = h->plan;
    if (pl.ops.empty()) return fail(SBK_ERR_STATE, "sbk_profile_ops: no plan yet (run a sampler call first)");
    const int n = (int)pl.ops.size();
    if (cap < n) return fail(SBK_ERR_ARG, "sbk_profile_ops: need room for %d launches", n);
    CU(cudaSetDevice(h->cfg.device));
    if (!h->cap_stream) CU(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    cudaStream_t s = h->cap_stream;
    CU(cudaDeviceSynchronize());
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) CU(cudaEventCreate(&e));
    StepBeginParams sb{pl.stats, pl.n_stat_doubles, pl.step_cur, pl.step_next};
    k_set_int<<<1, 1, 0, s>>>(pl.step_next, 0);
    launch_step_begin(sb, s);
    for (int i = 0; i < n; ++i) {
        CU(cudaEventRecord(ev[i], s));
        if (launch_op(pl.ops[i], s) < 0) return fail(SBK_ERR_CUDA, "sbk_profile_ops: launch of '%s' was refused", pl.ops[i].name.c_str());
    }
    CU(cudaEventRecord(ev[n], s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    for (int i = 0; i < n; ++i) {
        CU(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
        if (flops) flops[i] = pl.ops[i].flops;
        if (bytes) bytes[i] = pl.ops[i].bytes;
    }
    for (auto& e : ev) cudaEventDestroy(e);
    *n_ops = n;
    return SBK_OK;
}

// ------------------------------------------------------------------------------------------------
// DiffVC entry points (DiffVC/model/diffusion.py:61-106, 164-196)
// ------------------------------------------------------------------------------------------------
// host scalars of step i with the reference's double-precision scalar math (get_gamma / get_mu / get_nu / get_sigma,
// diffusion.py:124-149, 169-193): dxt = (mean - xt)*A - est*Bc + eps*sigma
static void vc_step_coefs(const sbk_config& c, int N, int i, int mode, float* t_out, float4* cf) {
    const double h = 1.0 / N, t = 1.0 - i * h;
    const double bmin = c.beta_min, bmax = c.beta_max;
    auto gamma = [&](double s, double tt, double p) {
        double bi = bmin + 0.5 * (bmax - bmin) * (tt + s);
        bi *= (tt - s);
        return exp(-0.5 * p * bi);
    };
    const double beta_t = bmin + (bmax - bmin) * t;
    double A, Bc, sigma;
    if (mode == 0) { A = 0.5 * beta_t * h; Bc = 0.5 * beta_t * h; sigma = 0.0; }
    else if (mode == 2) {
        double kappa = gamma(0, t - h, 1.0) * (1.0 - gamma(t - h, t, 2.0));
        kappa /= (gamma(0, t, 1.0) * beta_t * h);
        kappa -= 1.0;
        const double ct = 1.0 - gamma(0, t, 2.0);
        const double nu = gamma(0, t - h, 1.0) * (1.0 - gamma(t - h, t, 2.0)) / ct;
        const double mu = gamma(t - h, t, 1.0) * (1.0 - gamma(0, t - h, 2.0)) / ct;
        double omega = nu / gamma(0, t, 1.0);
        omega += mu;
        omega -= (0.5 * beta_t * h + 1.0);
        sigma = sqrt((1.0 - gamma(0, t - h, 2.0)) * (1.0 - gamma(t - h, t, 2.0)) / ct);
        A = 0.5 * beta_t * h + omega; Bc = (1.0 + kappa) * (beta_t * h);
    } else { A = 0.5 * beta_t * h; Bc = beta_t * h; sigma = sqrt(beta_t * h); }
    *t_out = (float)t;
    *cf = make_float4((float)A, (float)Bc, (float)sigma, 0.f);
}

static int vc_fold(sbk_handle* h, const float* cond, int rows, int B, cudaStream_t s) {
    Plan& pl = h->plan;
    const sbk_config& c = h->cfg;
    CU(cudaMemcpyAsync(pl.vc_cond, cond, (size_t)rows * B * c.dim_cond * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CondFoldParams p;
    p.cond = pl.vc_cond; p.w1 = h->w.get("estimator.downs.0.0.block1.block.0.weight");
    p.wres = h->w.get("estimator.downs.0.0.res_conv.weight");
    p.w_extra = pl.vc_wextra; p.r_extra = pl.vc_rextra; p.rows = rows; p.B = B; p.dc = c.dim_cond; p.C = c.dim;
    return launch_cond_fold(p, s);
}

extern "C" int sbk_vc_estimator(sbk_handle* h, const float* x, const float* mask, const float* mean, const float* cond,
                                const float* t, float* out, int B, int T, void* stream) {
    if (!h || !x || !mask || !mean || !cond || !t || !out) return fail(SBK_ERR_ARG, "sbk_vc_estimator: null argument");
    if (h->cfg.model != SBK_MODEL_DIFFVC) return fail(SBK_ERR_ARG, "sbk_vc_estimator: this handle is not a DiffVC model");
    TRY(ensure_plan(h, B, T, B));
    cudaStream_t s = (cudaStream_t)stream;
    Plan& pl = h->plan;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    CU(cudaMemcpyAsync(pl.xt, x, nb, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.mu, mean, nb, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.mask, mask, (size_t)B * T * sizeof(float), cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.t_rows, t, (size_t)B * sizeof(float), cudaMemcpyDeviceToDevice, s));
    int64_t n = 0;
    n += vc_fold(h, cond, 1, B, s);               // one row: the per-sample conditioning vectors
    n += time_table(h, B, s);
    set_mode(pl, 0, true, out);
    k_set_int<<<1, 1, 0, s>>>(pl.step_next, 0); ++n;
    { const int k = run_ops(h, s); if (k < 0) return SBK_ERR_CUDA; n += k; }
    CU(cudaGetLastError());
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_vc_reverse_diffusion(sbk_handle* h, const float* z, const float* mask, const float* mean, const float* cond,
                                        const float* noise, float* out, int B, int T, int n_timesteps, int mode, void* stream) {
    if (!h || !z || !mask || !mean || !cond || !out) return fail(SBK_ERR_ARG, "sbk_vc_reverse_diffusion: null argument");
    if (h->cfg.model != SBK_MODEL_DIFFVC) return fail(SBK_ERR_ARG, "sbk_vc_reverse_diffusion: this handle is not a DiffVC model");
    if (mode < 0 || mode > 2) return fail(SBK_ERR_ARG, "sbk_vc_reverse_diffusion: mode must be 0 (pf), 1 (em) or 2 (ml)");
    if (n_timesteps < 1) return fail(SBK_ERR_ARG, "sbk_vc_reverse_diffusion: n_timesteps must be >= 1");
    if (mode != 0 && !noise) return fail(SBK_ERR_ARG, "sbk_vc_reverse_diffusion: modes em/ml need a noise buffer");
    TRY(ensure_plan(h, B, T, n_timesteps));
    cudaStream_t s = (cudaStream_t)stream;
    Plan& pl = h->plan;
    const int N = n_timesteps;
    const size_t nb = (size_t)B * h->cfg.n_feats * T * sizeof(float);
    int64_t n = 0;
    CU(cudaMemcpyAsync(pl.mu, mean, nb, cudaMemcpyDeviceToDevice, s));
    CU(cudaMemcpyAsync(pl.mask, mask, (size_t)B * T * sizeof(float), cudaMemcpyDeviceToDevice, s));
    std::vector<float> tr(N); std::vector<float4> cf(N);
    for (int i = 0; i < N; ++i) vc_step_coefs(h->cfg, N, i, mode, &tr[i], &cf[i]);
    CU(cudaMemcpyAsync(pl.t_rows, tr.data(), N * sizeof(float), cudaMemcpyHostToDevice, s));
    CU(cudaMemcpyAsync(pl.coef, cf.data(), N * sizeof(float4), cudaMemcpyHostToDevice, s));
    n += vc_fold(h, cond, N, B, s);
    n += time_table(h, N, s);
    n += launch_scale_mask(z, pl.mask, pl.xt, 0, B, h->cfg.n_feats, T, s);
    TRY(run_steps(h, noise, B, T, N, 0, N, mode != 0, s, &n));
    CU(cudaMemcpyAsync(out, pl.xt, nb, cudaMemcpyDeviceToDevice, s));
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_vc_conditioning(sbk_handle* h, const float* ref, const float* ref_mask, const float* mean_ref, const float* c,
                                   float* cond_out, int B, int Tr, int n_timesteps, void* stream) {
    if (!h || !ref || !ref_mask || !mean_ref || !c || !cond_out) return fail(SBK_ERR_ARG, "sbk_vc_conditioning: null argument");
    if (h->cfg.model != SBK_MODEL_DIFFVC) return fail(SBK_ERR_ARG, "sbk_vc_conditioning: this handle is not a DiffVC model");
    if (!h->is_packed) return fail(SBK_ERR_STATE, "sbk_vc_conditioning: weights not packed");
    if (h->cfg.use_ref_t && h->cfg.dim_cond % 128 != 0) return fail(SBK_ERR_ARG, "sbk_vc_conditioning: dim_cond must be a multiple of 128");
    // fp32-class handles (fp32x3 and the CUDA-core fp32 mode) run the RefBlock convs with the tf32 + fp16-correction split and exact IN / GLU
    const int form = prec_runs_x3(h->cfg.precision) ? FORM_X3 : FORM_TF32;
    if (B <= 0 || Tr <= 0 || n_timesteps < 1) return fail(SBK_ERR_ARG, "sbk_vc_conditioning: bad sizes");
    CU(cudaSetDevice(h->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const sbk_config& cf = h->cfg;
    const int H = cf.n_feats, dc = cf.dim_cond, base = dc / 4, N = n_timesteps, dim = cf.dim;
    const size_t px = (size_t)B * H * Tr;
    // ---- workspace
    float *xt_ref, *raw, *act, *tb, *trows; double *st, *ys;
    auto carve = [&](Arena& ar) {
        xt_ref = (float*)ar.take(px * sizeof(float));
        raw = (float*)ar.take(px * 8 * base * sizeof(float));
        act = (float*)ar.take(px * 4 * base * sizeof(float));
        st = (double*)ar.take((size_t)B * 8 * base * 2 * sizeof(double));
        ys = (double*)ar.take((size_t)B * dc * 2 * sizeof(double));
        tb = (float*)ar.take((size_t)N * 3 * base * sizeof(float));
        trows = (float*)ar.take((size_t)N * sizeof(float));
    };
    Arena probe;
    carve(probe);
    if (const cudaError_t e = h->ref_ws.reserve(probe.bytes()))
        return fail(SBK_ERR_CUDA, "out of memory: the RefBlock workspace for (B=%d, Tr=%d) needs %zu bytes (%s)", B, Tr, probe.bytes(), cudaGetErrorString(e));
    Arena ar = h->ref_ws.arena();
    carve(ar);
    // ---- time values + the two RefBlock time biases (mlp1, mlp2: Mish -> Linear on the time-MLP output) for all steps
    std::vector<float> tr(N);
    for (int i = 0; i < N; ++i) tr[i] = (float)(1.0 - i * (1.0 / N));
    CU(cudaMemcpyAsync(trows, tr.data(), N * sizeof(float), cudaMemcpyHostToDevice, s));
    int64_t n = 0;
    if (cf.use_ref_t) {
        TimeTableParams tp; memset(&tp, 0, sizeof(tp));
        tp.t_rows = trows; tp.rows = N; tp.freqs = h->d_freqs; tp.pe_scale = 1000.0f; tp.dim = dim;
        tp.w0 = h->w.get("estimator.mlp.0.weight"); tp.b0 = h->w.get("estimator.mlp.0.bias");
        tp.w2 = h->w.get("estimator.mlp.2.weight"); tp.b2 = h->w.get("estimator.mlp.2.bias");
        tp.nproj = 2;
        tp.pw[0] = h->w.get("estimator.ref_block.mlp1.1.weight"); tp.pb[0] = h->w.get("estimator.ref_block.mlp1.1.bias"); tp.pc[0] = base; tp.poff[0] = 0;
        tp.pw[1] = h->w.get("estimator.ref_block.mlp2.1.weight"); tp.pb[1] = h->w.get("estimator.ref_block.mlp2.1.bias"); tp.pc[1] = 2 * base; tp.poff[1] = base;
        tp.tb = tb; tp.tb_stride = 3 * base;
        n += launch_time_table(tp, s);
    }
    auto gamma0 = [&](double t) {       // get_gamma(0, t), diffusion.py:124-131
        double bi = cf.beta_min + 0.5 * ((double)cf.beta_max - cf.beta_min) * t;
        bi *= t;
        return exp(-0.5 * bi);
    };
    auto conv = [&](const char* name, int cin, int cout) {
        ConvTcParams p; memset(&p, 0, sizeof(p));
        const std::string q = std::string("estimator.ref_block.") + name;
        p.geom = G_C3; p.in0 = act; p.c0 = cin; p.H = H; p.W = Tr; p.B = B; p.Ho = H; p.Wo = Tr;
        p.wpk = h->w.get(q + ".wtc"); p.bias = h->w.get(q + ".0.bias"); p.out = raw; p.Cout = cout; p.epi = EPI_PLAIN;
        p.mask = ref_mask; p.T = Tr; p.zero_page = h->d_zero;
        p.form = form; p.nt = conv_tc_ntile(G_C3, cout, p.form);     // as sbk_pack packed it
        return launch_conv_tc(p, s);
    };
    // debug capture: every step writes the same workspace buffers, so the last step's tensors are recorded
    h->vc_snaps.begin();
    bool last_step = false;
    auto snap = [&](const char* name, const char* suf, const void* src, size_t numel, int fmt) {
        if (h->vc_snaps.on && last_step) h->vc_snaps.record(std::string("ref_block.") + name + suf, src, numel, fmt, s);
    };
    auto norm_glu = [&](const char* name, int C, const float* tbias) {
        const std::string q = std::string("estimator.ref_block.") + name;
        ChanStatsParams cs{raw, st, B, H, Tr, C};
        int k = launch_chan_stats(cs, s);
        snap(name, ".stats", st, (size_t)B * C * 2, 3);
        InGluParams g; memset(&g, 0, sizeof(g));
        g.raw = raw; g.stats = st; g.gamma = h->w.get(q + ".1.weight"); g.beta = h->w.get(q + ".1.bias"); g.tb = tbias;
        g.mask = ref_mask; g.T = Tr; g.out = act; g.B = B; g.H = H; g.W = Tr; g.C = C; g.form = form;
        k += launch_in_glu(g, s);
        snap(name, ".act", act, px * C / 2, 1);
        return k;
    };
    // the five wgmma convs, each followed by its InstanceNorm + GLU; tb_off: offset of the stage's time bias in a tb row
    struct Stage { const char* name; int cin, cout, tb_off; };
    const Stage stages[5] = {{"block12", base, 2 * base, 0}, {"block21", base, 4 * base, -1}, {"block22", 2 * base, 4 * base, base},
                             {"block31", 2 * base, 8 * base, -1}, {"block32", 4 * base, 8 * base, -1}};
    for (int i = 0; i < N; ++i) {
        last_step = i + 1 == N;
        if (cf.use_ref_t) {
            const float* tb_row = tb + (size_t)i * 3 * base;
            DiffMeanParams dm{ref, mean_ref, ref_mask, xt_ref, (float)gamma0(1.0 - i * (1.0 / N)), B, H, Tr};
            n += launch_diff_mean(dm, s);
            snap("xt_ref", "", xt_ref, px, 0);
            snap("tb", "", tb_row, (size_t)3 * base, 0);
            FirstConvParams fc; memset(&fc, 0, sizeof(fc));
            fc.mu = xt_ref; fc.xt = xt_ref; fc.mask = ref_mask; fc.w = h->w.get("estimator.ref_block.block11.w");
            fc.bias = h->w.get("estimator.ref_block.block11.0.bias"); fc.out = raw; fc.ostats = nullptr;
            fc.B = B; fc.H = H; fc.T = Tr; fc.cin = 1; fc.C = 2 * base; fc.chw4 = 1;
            n += launch_first_conv(fc, s);
            snap("block11", ".raw", raw, px * 2 * base, 1);
            n += norm_glu("block11", 2 * base, nullptr);
            for (const Stage& sg : stages) {
                const int k = conv(sg.name, sg.cin, sg.cout);
                if (k < 0) return fail(SBK_ERR_UNSUPPORTED, "sbk_vc_conditioning: the tensor-core conv of %s was refused", sg.name);
                n += k;
                snap(sg.name, ".raw", raw, px * sg.cout, 1);
                n += norm_glu(sg.name, sg.cout, sg.tb_off < 0 ? nullptr : tb_row + sg.tb_off);
            }
            ChanStatsParams ysm{act, ys, B, H, Tr, 4 * base};
            n += launch_chan_stats(ysm, s);
            snap("ysum", "", ys, (size_t)B * dc * 2, 3);
        }
        VcCondParams vp; memset(&vp, 0, sizeof(vp));
        vp.ysum = ys; vp.mask = ref_mask; vp.Tr = Tr; vp.H = H;
        vp.wf = h->w.get("estimator.ref_block.final_conv.weight"); vp.bf = h->w.get("estimator.ref_block.final_conv.bias");
        vp.c = c; vp.freqs = h->d_freqs; vp.t = tr[i]; vp.dim = dim;
        vp.w0 = h->w.get("estimator.cond_block.0.weight"); vp.b0 = h->w.get("estimator.cond_block.0.bias");
        vp.w2 = h->w.get("estimator.cond_block.2.weight"); vp.b2 = h->w.get("estimator.cond_block.2.bias");
        vp.out = cond_out + (size_t)i * B * dc; vp.B = B; vp.dc = dc; vp.use_ref = cf.use_ref_t ? 1 : 0;
        n += launch_vc_cond(vp, s);
    }
    if (const cudaError_t e = h->vc_snaps.finish()) return fail(SBK_ERR_CUDA, "sbk_vc_conditioning: debug capture failed: %s", cudaGetErrorString(e));
    CU(cudaGetLastError());
    h->last_launches = n;
    return SBK_OK;
}

extern "C" int sbk_vc_cond_debug_num(const sbk_handle* h) { return h ? (int)h->vc_snaps.list.size() : 0; }
extern "C" const char* sbk_vc_cond_debug_name(const sbk_handle* h, int i) {
    if (!h || i < 0 || i >= (int)h->vc_snaps.list.size()) return nullptr;
    return h->vc_snaps.list[i].name.c_str();
}
extern "C" int sbk_vc_cond_debug_op_layout(const sbk_handle* h, const char* name) {
    const Snapshots::Snap* sn = h && name ? h->vc_snaps.find(name) : nullptr;
    return sn ? sn->fmt : -1;
}
extern "C" int sbk_vc_cond_debug_read(sbk_handle* h, const char* name, void* dst, int64_t* numel) {
    if (!h || !name) return fail(SBK_ERR_ARG, "sbk_vc_cond_debug_read: null argument");
    return h->vc_snaps.read(name, dst, numel, h->cfg.device, "sbk_vc_cond_debug_read");
}

extern "C" int sbk_prior_expand(const float* mu_x, const float* w_ceil, const float* x_mask, const int64_t* y_lengths,
                                const float* noise_tf, float temperature, int B, int F, int Tx, int Ty,
                                float* mu_y, float* z, float* y_mask, float* attn, void* stream) {
    if (!mu_x || !w_ceil || !x_mask || !y_lengths || !mu_y || !z || !y_mask) return fail(SBK_ERR_ARG, "sbk_prior_expand: null argument");
    if (B <= 0 || F <= 0 || Tx <= 0 || Ty <= 0) return fail(SBK_ERR_ARG, "sbk_prior_expand: bad sizes B=%d F=%d Tx=%d Ty=%d", B, F, Tx, Ty);
    if (Tx > 12000) return fail(SBK_ERR_ARG, "sbk_prior_expand: Tx=%d exceeds the 12000-token shared-memory table", Tx);
    if (noise_tf && !(temperature > 0.f)) return fail(SBK_ERR_ARG, "sbk_prior_expand: temperature must be > 0");
    PriorExpandParams p;
    p.mu_x = mu_x; p.w_ceil = w_ceil; p.x_mask = x_mask; p.y_len = reinterpret_cast<const long long*>(y_lengths);
    p.noise_tf = noise_tf; p.temperature = temperature; p.B = B; p.F = F; p.Tx = Tx; p.Ty = Ty;
    p.mu_y = mu_y; p.z = z; p.y_mask = y_mask; p.attn = attn;
    launch_prior_expand(p, (cudaStream_t)stream);
    CU(cudaGetLastError());
    return SBK_OK;
}

extern "C" int64_t sbk_last_launch_count(const sbk_handle* h) { return h ? h->last_launches : 0; }
extern "C" int sbk_last_host_launches(const sbk_handle* h) { return h ? h->last_host_launches : 0; }

extern "C" int sbk_debug_capture(sbk_handle* h, int on) {
    if (!h) return fail(SBK_ERR_ARG, "sbk_debug_capture: null handle");
    h->capture = h->vc_snaps.on = on != 0;
    return SBK_OK;
}
extern "C" int sbk_debug_layout(const sbk_handle* h) { return (h && h->cfg.precision != SBK_PREC_FP32) ? 1 : 0; }
// layout of one named intermediate: 0 [B][H][W][C] fp32, 1 [B][H][C/4][W][4] fp32, 2 [B][H][C/8][W][8] (bf16 in HBM;
// sbk_debug_read widens it to fp32), -1 unknown name
extern "C" int sbk_debug_op_layout(const sbk_handle* h, const char* name) {
    if (!h || !name) return -1;
    for (auto& op : h->plan.ops) if (op.name == name) return op.dbg_fmt;
    return -1;
}
extern "C" int sbk_debug_num(const sbk_handle* h) { return h ? (int)h->plan.ops.size() : 0; }
extern "C" const char* sbk_debug_name(const sbk_handle* h, int i) {
    if (!h || i < 0 || i >= (int)h->plan.ops.size()) return nullptr;
    return h->plan.ops[i].name.c_str();
}
extern "C" int sbk_debug_read(sbk_handle* h, const char* name, float* dst, int64_t* numel) {
    if (!h || !name) return fail(SBK_ERR_ARG, "sbk_debug_read: null argument");
    for (auto& op : h->plan.ops) {
        if (op.name != name) continue;
        if (numel) *numel = op.dbg_numel;
        if (dst && op.dbg_ptr && op.dbg_numel > 0) {
            CU(cudaDeviceSynchronize());
            const void* src = op.dbg_copy ? (const void*)op.dbg_copy : (const void*)op.dbg_ptr;
            return read_widened(dst, src, op.dbg_numel, op.dbg_fmt);
        }
        return SBK_OK;
    }
    return fail(SBK_ERR_ARG, "sbk_debug_read: no intermediate named '%s'", name);
}
