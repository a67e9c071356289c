// DiffVC's PostNet (DiffVC/model/postnet.py:40-53), the second half of the "average voice" encoder FwdDiffusion
// (DiffVC/model/vc.py:19-48: MelEncoder followed by PostNet), over the [n_feats x T] mel grid as a one-channel image:
//   init_conv 1x1 (1 -> dim) -> ResnetBlock(dim) [Block(7x7 conv, GroupNorm(8), Mish) x 2 + 1x1 res conv] -> final_conv 1x1 (dim -> 1)
//
// Launch plan (all asynchronous on the caller's stream):
//   1. zero the two blocks' GroupNorm statistics
//   2. k_pn_init: a0 = init_conv(x*mask)*mask in operand form [B][n_feats][dim/4][T][4] - the
//      input of block1 AND of the residual conv (ResnetBlock.forward multiplies both by the mask, postnet.py:22,36)
//   3. k_conv_tc<G_C7>: block1 conv -> raw1 + GroupNorm partials (fixed-order, fp64)
//   4. k_gn_act: act = mask ? Mish(GN(raw1)) : 0 (no time bias: tb is the zero page, postnet.py:22-23)
//   5. k_conv_tc<G_C7>: block2 conv -> raw2 + GroupNorm partials
//   6. k_conv_tc<G_PW, RES>: y = (res(a0) + bias + Mish(GN(raw2))*mask) * mask   (postnet.py:36 and final_conv's input mask, :52)
//   7. k_pn_final: out = final_conv(y) + bias, planar [B][n_feats][T], NOT masked (as in the reference: a padded column
//      equals final_conv.bias).  A separate CUDA-core pass: dim MACs per pixel, < 1 % of the PostNet's time; the 1x1 res
//      conv's epilogue would need a new template variant for it.
// GroupNorm statistics cover the whole n_feats x T grid, padded columns included, as the reference's GroupNorm does.
#include "sbk_host.h"

#include <math.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

using namespace sbk;

namespace {

// a0 = (w*(x*m) + b)*m per channel, written as [B][H][C/4][T][4] operand chunks; tf32 mode rounds to nearest (as k_gn_act),
// fp32x3 mode keeps fp32.  RAG (a ragged batch): frames at or past the utterance's length are written as 0, x is not read there.
template <bool RAG>
__device__ __forceinline__ void pn_init(const float* x, const float* mask, const float* w, const float* bias, float* out, int B, int H,
                                        int C, int T, int round_tf32, const int64_t* lengths) {
    const int c4n = C / 4;
    const long long n = (long long)B * H * c4n * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long r = i / T;
        const int ch = (int)(r % c4n);
        const long long bh = r / c4n;                       // b*H + h
        const long long b = bh / H;
        if (RAG && t >= grid_edge(lengths, b, T, 0, 1)) {
            reinterpret_cast<float4*>(out)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
            continue;
        }
        const float m = __ldg(mask + b * T + t);
        const float xv = __ldg(x + bh * T + t) * m;
        const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + ch), bv = __ldg(reinterpret_cast<const float4*>(bias) + ch);
        float o[4] = {(wv.x * xv + bv.x) * m, (wv.y * xv + bv.y) * m, (wv.z * xv + bv.z) * m, (wv.w * xv + bv.w) * m};
        if (round_tf32) {
#pragma unroll
            for (int q = 0; q < 4; ++q) { uint32_t u; asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(o[q])); o[q] = __uint_as_float(u); }
        }
        reinterpret_cast<float4*>(out)[i] = make_float4(o[0], o[1], o[2], o[3]);
    }
}
__global__ void k_pn_init(const float* x, const float* mask, const float* w, const float* bias, float* out, int B, int H, int C, int T,
                          int round_tf32) {
    pn_init<false>(x, mask, w, bias, out, B, H, C, T, round_tf32, nullptr);
}
__global__ void k_pn_init_ragged(const float* x, const float* mask, const float* w, const float* bias, float* out, int B, int H, int C,
                                 int T, int round_tf32, const int64_t* lengths) {
    pn_init<true>(x, mask, w, bias, out, B, H, C, T, round_tf32, lengths);
}

// final_conv (dim -> 1, postnet.py:52): out[b][h][t] = bias + sum_c w[c] * y[b][h][c][t], channels summed in order.
// RAG: frames at or past the utterance's length are written as 0 (its own call has no such frames), y is not read there.
template <bool RAG>
__device__ __forceinline__ void pn_final(const float* y, const float* w, const float* bias, float* out, int B, int H, int C, int T,
                                         const int64_t* lengths) {
    const int c4n = C / 4;
    const long long n = (long long)B * H * T;
    const float bb = __ldg(bias);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % T);
        const long long bh = i / T;
        if (RAG && t >= grid_edge(lengths, bh / H, T, 0, 1)) { out[i] = 0.f; continue; }
        const float* yp = y + (bh * c4n * T + t) * 4;
        float acc = 0.f;
        for (int ch = 0; ch < c4n; ++ch) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(yp + (long long)ch * T * 4));
            const float4 wv = __ldg(reinterpret_cast<const float4*>(w) + ch);
            acc = fmaf(v.x, wv.x, acc); acc = fmaf(v.y, wv.y, acc); acc = fmaf(v.z, wv.z, acc); acc = fmaf(v.w, wv.w, acc);
        }
        out[i] = acc + bb;
    }
}
__global__ void k_pn_final(const float* y, const float* w, const float* bias, float* out, int B, int H, int C, int T) {
    pn_final<false>(y, w, bias, out, B, H, C, T, nullptr);
}
__global__ void k_pn_final_ragged(const float* y, const float* w, const float* bias, float* out, int B, int H, int C, int T,
                                  const int64_t* lengths) {
    pn_final<true>(y, w, bias, out, B, H, C, T, lengths);
}

// The workspace of one (B, n_feats, T), the same in every mode: a0, raw (raw1, then raw2), act (act1, then the res conv's
// output y), and the two blocks' [B][8][2] fp64 GroupNorm statistics.  Over a null-base arena only the size is computed.
struct PnBufs { float *a0, *raw, *act; double* st; };
size_t pn_carve(int B, int H, int C, int T, Arena& ar, PnBufs* o) {
    const size_t big = (size_t)B * H * C * T * sizeof(float);
    PnBufs b;
    b.a0 = (float*)ar.take(big);
    b.raw = (float*)ar.take(big);
    b.act = (float*)ar.take(big);
    b.st = (double*)ar.take(2 * (size_t)B * kGroups * 2 * sizeof(double));
    if (o) *o = b;
    return ar.bytes();
}

}  // namespace

struct sbk_postnet {
    // precision: the fp32-class modes run the fp32x3 path (prec_runs_x3), tf32, bf16 and fp16 the tf32 path (16-bit operands
    // are not implemented for the 7x7 geometry)
    sbk_postnet_config cfg;
    WeightSet w;                             // raw: reference layout; packed: tensor-core stage images
    float* zero = nullptr;                   // zero page: A-tile borders, and k_gn_act's (absent) time bias
    Workspace ws;
    bool is_packed = false;
    int64_t last_launches = 0;
    // debug capture (fmt: 1 fp32 [B][H][C/4][T][4], 3 float64 [B][groups][2])
    Snapshots snaps;
};

extern "C" int sbk_postnet_create(const sbk_postnet_config* cfg, sbk_postnet** out) {
    if (!cfg || !out) return fail(SBK_ERR_ARG, "sbk_postnet_create: null argument");
    if (cfg->groups != kGroups)
        return fail(SBK_ERR_UNSUPPORTED, "sbk_postnet_create: groups = %d; the GroupNorm kernels are built for %d groups", cfg->groups, kGroups);
    // the conv epilogue reduces GroupNorm partials per 32-channel block: a group must be 8 or 16 channels wide (dim 64, 128)
    // or a whole number of blocks (dim a multiple of 256); channels come in 64-wide N tiles
    const int d = cfg->dim;
    if (d <= 0 || d % 64 != 0 || (d > 128 && d % 256 != 0))
        return fail(SBK_ERR_UNSUPPORTED, "sbk_postnet_create: dim = %d; supported: 64, 128 and multiples of 256", d);
    if (cfg->precision < SBK_PREC_FP32 || cfg->precision > SBK_PREC_F16)
        return fail(SBK_ERR_ARG, "sbk_postnet_create: unknown precision %d", cfg->precision);
    sbk_postnet* p = new sbk_postnet();
    p->cfg = *cfg;
    auto add = [&](const std::string& n, std::vector<int64_t> s) { p->w.add(n, std::move(s)); };
    add("init_conv.weight", {d, 1, 1, 1}); add("init_conv.bias", {d});
    for (const char* blk : {"block1", "block2"}) {
        const std::string q = std::string("res_block.") + blk + ".block.";
        add(q + "0.weight", {d, d, 7, 7}); add(q + "0.bias", {d});
        add(q + "1.weight", {d}); add(q + "1.bias", {d});
    }
    add("res_block.res.weight", {d, d, 1, 1}); add("res_block.res.bias", {d});
    add("final_conv.weight", {1, d, 1, 1}); add("final_conv.bias", {1});
    *out = p;
    return SBK_OK;
}

extern "C" void sbk_postnet_destroy(sbk_postnet* p) {
    if (!p) return;
    if (p->zero) cudaFree(p->zero);
    delete p;
}

extern "C" int sbk_postnet_num_weights(const sbk_postnet* p) { return p ? p->w.count() : 0; }
extern "C" const char* sbk_postnet_weight_name(const sbk_postnet* p, int i) { return p ? p->w.name(i) : nullptr; }

extern "C" int sbk_postnet_set_weight(sbk_postnet* p, const char* name, const void* data, const int64_t* shape, int ndim) {
    if (!p || !name || !data || !shape) return fail(SBK_ERR_ARG, "sbk_postnet_set_weight: null argument");
    TRY(p->w.set(name, data, shape, ndim, p->cfg.device, "sbk_postnet_set_weight"));
    p->is_packed = false;
    return SBK_OK;
}

static int pn_pack(sbk_postnet* p, const std::string& name, int geom) {
    const int d = p->cfg.dim;
    std::vector<float> w;
    TRY(p->w.fetch(name, w));
    const int form = prec_runs_x3(p->cfg.precision) ? FORM_X3 : FORM_TF32, nt = conv_tc_ntile(geom, d, form);
    std::vector<uint8_t> img(conv_tc_pack_image(w.data(), d, d, geom, form, nt, nullptr));
    conv_tc_pack_image(w.data(), d, d, geom, form, nt, img.data());
    return upload(p->w.packed, name, img.size(), img.data());
}

extern "C" int sbk_postnet_pack(sbk_postnet* p) {
    if (!p) return fail(SBK_ERR_ARG, "sbk_postnet_pack: null handle");
    TRY(p->w.require_all("sbk_postnet_pack"));
    CU(cudaSetDevice(p->cfg.device));
    TRY(pn_pack(p, "res_block.block1.block.0.weight", G_C7));
    TRY(pn_pack(p, "res_block.block2.block.0.weight", G_C7));
    TRY(pn_pack(p, "res_block.res.weight", G_PW));
    if (!p->zero) { CU(cudaMalloc(&p->zero, 8192)); CU(cudaMemset(p->zero, 0, 8192)); }
    p->is_packed = true;
    return SBK_OK;
}

extern "C" size_t sbk_postnet_workspace_bytes(const sbk_postnet* p, int B, int n_feats, int T) {
    if (!p || B <= 0 || n_feats <= 0 || T <= 0) return 0;
    Arena probe;
    return pn_carve(B, n_feats, p->cfg.dim, T, probe, nullptr);
}

extern "C" int sbk_postnet_forward(sbk_postnet* p, const float* x, const float* mask, float* out, int B, int n_feats, int T, void* stream) {
    return sbk_postnet_forward_lengths(p, x, mask, nullptr, out, B, n_feats, T, stream);
}

// lengths (device int64 [B], nullable): a ragged batch.  Utterance b runs on its own L_b = lengths[b] frames (clamped to
// [1, T]) exactly as its own call on x[b, :, :L_b] does - no rounding of the length - and its output from L_b on is 0.
extern "C" int sbk_postnet_forward_lengths(sbk_postnet* p, const float* x, const float* mask, const int64_t* lengths, float* out,
                                           int B, int n_feats, int T, void* stream) {
    if (!p || !x || !mask || !out) return fail(SBK_ERR_ARG, "sbk_postnet_forward: null argument");
    if (!p->is_packed) return fail(SBK_ERR_STATE, "sbk_postnet_forward: weights not packed (sbk_postnet_set_weight for every key, then sbk_postnet_pack)");
    if (B <= 0 || n_feats <= 0 || T <= 0) return fail(SBK_ERR_ARG, "sbk_postnet_forward: B, n_feats and T must be positive (got %d, %d, %d)", B, n_feats, T);
    CU(cudaSetDevice(p->cfg.device));
    cudaStream_t s = (cudaStream_t)stream;
    const int C = p->cfg.dim, H = n_feats;
    const bool x3 = prec_runs_x3(p->cfg.precision);
    const int form = x3 ? FORM_X3 : FORM_TF32;
    const size_t need = sbk_postnet_workspace_bytes(p, B, n_feats, T);
    if (p->ws.reserve(need)) return fail(SBK_ERR_CUDA, "out of memory: the PostNet workspace for (B=%d, n_feats=%d, T=%d) needs %zu bytes", B, n_feats, T, need);
    PnBufs wb;
    Arena ar = p->ws.arena();
    pn_carve(B, H, C, T, ar, &wb);
    float *a0 = wb.a0, *raw = wb.raw, *act = wb.act;
    double* st = wb.st;
    double* st1 = st; double* st2 = st + (size_t)B * kGroups * 2;
    auto R = [&](const std::string& k) { return p->w.get(k); };
    const float inv_count = (float)(1.0 / ((double)(C / kGroups) * H * T));
    // a ragged batch: every launch cuts at the utterance's own length (grid_edge, exact rule), and the GroupNorm divisor is
    // the expression above at T = L_b, evaluated per sample in double on the device (gn_inv_count_rag)
    const bool rag = lengths != nullptr;
    int64_t n = 0;
    auto refused = [&](const char* what) {
        return fail(SBK_ERR_CUDA, "sbk_postnet_forward: the %s launch was refused (device attribute / geometry)", what);
    };
    int k;
    // debug capture: raw and act are rewritten within the call, so each tensor is copied right after the launch that wrote it
    const size_t px = (size_t)B * H * T * C;
    p->snaps.begin();
    auto snap = [&](const char* name, const void* src, size_t numel, int fmt) { p->snaps.record(name, src, numel, fmt, s); };

    CU(cudaMemsetAsync(st, 0, 2 * (size_t)B * kGroups * 2 * sizeof(double), s)); ++n;
    if (rag)
        k_pn_init_ragged<<<ew_grid((long long)B * H * (C / 4) * T), 256, 0, s>>>(x, mask, R("init_conv.weight"), R("init_conv.bias"), a0,
                                                                                 B, H, C, T, x3 ? 0 : 1, lengths);
    else
        k_pn_init<<<ew_grid((long long)B * H * (C / 4) * T), 256, 0, s>>>(x, mask, R("init_conv.weight"), R("init_conv.bias"), a0, B, H, C, T,
                                                                          x3 ? 0 : 1);
    ++n;
    snap("a0", a0, px, 1);
    auto conv7 = [&](const char* blk, const float* in, double* ost) {
        ConvTcParams cp; memset(&cp, 0, sizeof(cp));
        const std::string q = std::string("res_block.") + blk + ".block.0.";
        cp.geom = G_C7; cp.in0 = in; cp.c0 = C; cp.H = H; cp.W = T; cp.B = B; cp.Ho = H; cp.Wo = T;
        cp.wpk = R(q + "weight"); cp.bias = R(q + "bias"); cp.out = raw; cp.Cout = C; cp.epi = EPI_PLAIN;
        cp.ostats = ost; cp.mask = mask; cp.T = T; cp.zero_page = p->zero;
        cp.form = form; cp.nt = conv_tc_ntile(G_C7, C, form);     // as pn_pack packed it
        cp.lengths = lengths; cp.exact = 1;
        return launch_conv_tc(cp, s);
    };
    auto gnref = [&](double* stp, const char* blk) {
        const std::string q = std::string("res_block.") + blk + ".block.1.";
        GnRef g; g.stats = stp; g.gamma = R(q + "weight"); g.beta = R(q + "bias"); g.inv_count = inv_count;
        g.lengths = lengths; g.cnt_ch = (float)(C / kGroups) * (float)H; g.T = T; g.lvl = 0; g.exact = 1;
        return g;
    };
    if ((k = conv7("block1", a0, st1)) < 0) return refused("block1 conv");
    n += k;
    snap("block1.raw", raw, px, 1);
    snap("block1.stats", st1, (size_t)B * kGroups * 2, 3);
    {
        GnActParams g; memset(&g, 0, sizeof(g));
        g.raw = raw; g.gn = gnref(st1, "block1"); g.tb = p->zero; g.tb_stride = 0; g.tb_per_sample = 1;
        g.mask = mask; g.T = T; g.lvl = 0; g.out = act; g.B = B; g.H = H; g.W = T; g.C = C;
        g.form = form;
        if ((k = launch_gn_act(g, s)) < 0) return refused("block1 GroupNorm/Mish");
        n += k;
    }
    snap("block1.act", act, px, 1);
    if ((k = conv7("block2", act, st2)) < 0) return refused("block2 conv");
    n += k;
    snap("block2.raw", raw, px, 1);
    snap("block2.stats", st2, (size_t)B * kGroups * 2, 3);
    {
        ConvTcParams cp; memset(&cp, 0, sizeof(cp));
        cp.geom = G_PW; cp.in0 = a0; cp.c0 = C; cp.H = H; cp.W = T; cp.B = B; cp.Ho = H; cp.Wo = T;
        cp.wpk = R("res_block.res.weight"); cp.bias = R("res_block.res.bias"); cp.out = act; cp.Cout = C;
        cp.epi = EPI_RES; cp.rraw = raw; cp.rgn = gnref(st2, "block2"); cp.out_mask = 1;
        cp.mask = mask; cp.T = T; cp.zero_page = p->zero;
        cp.form = form; cp.nt = conv_tc_ntile(G_PW, C, form);
        cp.lengths = lengths; cp.exact = 1;
        if ((k = launch_conv_tc(cp, s)) < 0) return refused("residual conv");
        n += k;
    }
    snap("res", act, px, 1);
    if (rag)
        k_pn_final_ragged<<<ew_grid((long long)B * H * T), 256, 0, s>>>(act, R("final_conv.weight"), R("final_conv.bias"), out, B, H, C, T,
                                                                        lengths);
    else
        k_pn_final<<<ew_grid((long long)B * H * T), 256, 0, s>>>(act, R("final_conv.weight"), R("final_conv.bias"), out, B, H, C, T);
    ++n;
    if (const cudaError_t e = p->snaps.finish()) return fail(SBK_ERR_CUDA, "sbk_postnet_forward: debug capture failed: %s", cudaGetErrorString(e));
    CU(cudaGetLastError());
    p->last_launches = n;
    return SBK_OK;
}

extern "C" int64_t sbk_postnet_last_launch_count(const sbk_postnet* p) { return p ? p->last_launches : 0; }

extern "C" int sbk_postnet_debug_capture(sbk_postnet* p, int on) {
    if (!p) return fail(SBK_ERR_ARG, "sbk_postnet_debug_capture: null handle");
    p->snaps.on = on != 0;
    return SBK_OK;
}
extern "C" int sbk_postnet_debug_num(const sbk_postnet* p) { return p ? (int)p->snaps.list.size() : 0; }
extern "C" const char* sbk_postnet_debug_name(const sbk_postnet* p, int i) {
    if (!p || i < 0 || i >= (int)p->snaps.list.size()) return nullptr;
    return p->snaps.list[i].name.c_str();
}
extern "C" int sbk_postnet_debug_op_layout(const sbk_postnet* p, const char* name) {
    const Snapshots::Snap* sn = p && name ? p->snaps.find(name) : nullptr;
    return sn ? sn->fmt : -1;
}
extern "C" int sbk_postnet_debug_read(sbk_postnet* p, const char* name, void* dst, int64_t* numel) {
    if (!p || !name) return fail(SBK_ERR_ARG, "sbk_postnet_debug_read: null argument");
    return p->snaps.read(name, dst, numel, p->cfg.device, "sbk_postnet_debug_read");
}
