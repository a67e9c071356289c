"""Float64 op replay of one captured estimator call, and a checker that a local defect cannot hide from.

Every op the plan exposes through the debug capture is recomputed in float64 from the GPU's OWN captured inputs (never
from the oracle's chain), so each kernel is judged alone: upstream error can neither mask nor excuse it.  The op semantics
are the oracle's (oracle/gradtts_oracle.py: conv_gn_mish, resnet, rezero_linear_attention, the down/up convs and the
final conv; oracle/diffvc_oracle.py for the DiffVC input stack), restated line for line on float64 copies.

For every linear op the replay also computes the magnitude companion A: the same op on |input| and |weights|, plus |bias|.
`check` then applies two tests:

1. per element  |got - ref| <= kappa * A + floor, with kappa derived from the mode's rounding points (`kappa` below);
2. uniformity: the error, grouped by output column (b, w), by row (b, h) and by 64-channel N-tile block, as
   e_g = ||err_g|| / ||A_g||; the largest e_g may exceed the median of the other groups by at most R_UNIFORM.

Rounding noise is nearly the same in every group (each column has C*H samples), so a defect at one tile seam, one halo row
or one N tile stands out by orders of magnitude even where check 1's worst-case bound is loose (tf32, bf16, fp32x3).

`VocoderReplay` does the same for one HiFi-GAN vocoder call (oracle/hifigan_oracle.py semantics): its [B, C, L] signals
are grouped by sample, 128-sample tile, within-tile phase and N-tile block (`uniformity1d`), and its elementwise kernels
(mel layout, transposed-conv fold, LeakyReLU second outputs, MRF mean) must reproduce their fp32 arithmetic bit for bit.

`RefBlockReplay` and `PostNetReplay` do the same for DiffVC's conditioning branch and PostNet.  With per-utterance lengths,
`Replay`, `RefBlockReplay` and `PostNetReplay` judge each utterance of a ragged call on its own frames.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from helpers import nhwc_to_nchw
from oracle import gradtts_oracle as O
from oracle.precision_model import round_bf16, round_tf32_rna
from speech_backbones_b200.gradtts import fix_len_compatibility

# ---- check 1: kappa, from the rounding points of oracle/precision_model.py ----------------------------------------------
# Operand rounding, relative to |x||w| of one product:
#   tf32    x truncated to 10 mantissa bits (< 2^-10), w round-to-nearest-away (<= 2^-11): 2^-10 + 2^-11 + 2^-21.
#   bf16    (7 fraction bits: RNE <= 2^-8) stored operand tensors are exact bf16 (the capture reads them as stored),
#           weights RNE (<= 2^-8).  The Block
#           activation is rebuilt here and rounded as k_gn_act rounds it (rna tf32 / RNE bf16), so that its rounding - a
#           per-channel constant wherever the time bias dominates, i.e. correlated along a row - is replayed rather than
#           left in the error; the rebuilt fp32 value can still round to the neighbouring value where the GPU's did not,
#           so kappa keeps one activation rounding (<= 2^-8): 2^-7 + 2^-16.
#   fp32x3  x*w = x_hi*w_hi + f16(x_lo)*f16(w) + f16(x*2^-12)*f16(w_lo*2^12): the double-counted x_lo*w_lo (2^-10 * 2^-11)
#           plus four fp16 roundings of 2^-11 on terms of 2^-10 (x_lo, w) and 2^-11 (x*2^-12, w_lo) relative size:
#           3 * 2^-21 + 2 * 2^-22 = 2^-19.
U_OPERAND = {"tf32": 2 ** -10 + 2 ** -11 + 2 ** -21, "bf16": 2 ** -7 + 2 ** -16, "fp32x3": 2 ** -19}
# Accumulation.  A wgmma adds its K-slice (8 tf32 / 16 bf16 or fp16 products) into the fp32 register accumulator: at most
# two roundings of 2^-23 (the inner sum, the accumulator add; round-toward-zero, so 2^-23 rather than 2^-24) on partial
# sums bounded by A, i.e. 2^-22 per MMA.  fp32x3 folds runs of at most 54 MMAs (3x3; 42 for 7x7) round-to-nearest into a
# second fp32 array: 54 * 2^-22 within a run plus 2^-24 per fold.  CUDA-core FFMA chains: the classic gamma_K = K * 2^-24.
K_MMA = {"tf32": 8, "bf16": 16, "fp32x3": 8}
X3_RUN = 54
# GroupNorm / Mish / exp evaluated in fp32 before or after a linear op: __expf is within 2 + 1.16|x| ulp for |x| <= 20
# (< 2^-18 relative), the fast division 2 ulp, the normalisation (v - mean) * scale + beta a few ulp of the magnitudes of
# its terms (not of its result, which can cancel): 2^-17 relative to the companion 1.1 (|v - mean| |scale| + |beta|)
# (|Mish'| <= 1.1), which A contains.
EPS_NL = 2 ** -17
# Inputs recomputed here instead of captured (the multi-speaker embedding MLP, DiffVC's folded conditioning): the GPU's
# fp32 evaluation (K <= 320 FFMA terms) differs by up to 320 * 2^-24 < 2^-15.6 of their magnitude.
EPS_RECOMPUTED = 2 ** -15
# A bf16 operand tensor written by the op: RNE to 7 fraction bits, <= 2^-8 |out| <= 2^-8 A.
EPS_STORE_BF16 = 2 ** -8
# Absolute floor: fp32x3 correction chunks underflow to fp16 subnormals for |x| < 2^-4 (x_lo) or |x| < 2^-2 (x * 2^-12);
# each loses <= 2^-25 absolute, times |w| (or |w_lo| * 2^12 <= 2|w|): 2^-24 * sum |w| over the fan-in.
FLOOR_PER_W = 2 ** -24

# ---- check 2: R ------------------------------------------------------------------------------------------------------
# e_g is a ratio of norms over >= C*H (columns) or C*W (rows) samples, so independent rounding errors make it concentrate
# to a few per cent around the group's RMS level.  What legitimately varies between groups is the number of non-zero
# taps: a column or row at an image or mask edge sees 2 of 3 (or 1 of 3) kernel columns.  Past a mask edge such columns
# are left out (less than half the typical data), and so are the image's first and last rows and columns: there the error
# terms that are constant over a channel (the time bias the GPU evaluates in fp32, against its float64 replay) sum over
# 6 taps instead of 9, which measured up to 6.5x the interior level in the CUDA-core fp32 mode.  Those border groups are
# judged by check 1 alone, which a stale or non-zero padding value fails by 20x or more in every tensor-core mode.
# Among interior groups e_g varies little (measured max/median <= 2.5 on an H100).  R = 4 leaves margin, while one dropped tap
# out of K (or one zeroed halo column) raises its column's e_g by ~ (|x w| / A) / (u / sqrt(K)) = sqrt(K) / (K u) / ~1:
# 2^11 / 24 ~ 85x for a 64-channel tf32 3x3 conv, far more in fp32x3.
R_UNIFORM = 4.0
MIN_GROUP = 32            # groups with fewer elements are too noisy for the ratio (end-to-end PostNet rows of one column)


def kappa(mode, K, tc=True, nl=False, store_bf16=False, extra=0.0, run=X3_RUN):
    """Per-element relative bound of one linear op with fan-in K: operand rounding + accumulation (+ terms above)."""
    if mode == "fp32" or not tc:
        k = K * 2 ** -24
    else:
        n = math.ceil(K / K_MMA[mode])
        if mode == "fp32x3":
            n *= 2                                             # correction MMA + main MMA per K slice
            k = U_OPERAND[mode] + min(n, run) * 2 ** -22 + math.ceil(n / run) * 2 ** -24
        else:
            k = U_OPERAND[mode] + n * 2 ** -22
    if nl:
        k += EPS_NL
    if store_bf16:
        k += EPS_STORE_BF16
    return k + extra


# ---- the checker -----------------------------------------------------------------------------------------------------
def _group_norms(t, dims):
    return t.pow(2).sum(dim=dims).sqrt().flatten()


def groupings(x, ntile=64, period=None):
    """[B,C,H,W] -> {name: (reduce dims or channel-block view)}: columns (b,w), rows (b,h), `ntile`-channel N-tile blocks,
    and with `period`, the column phase w % period over the full period-wide tiles (the image's border columns left out)."""
    B, C, H, W = x.shape
    nb = (C + ntile - 1) // ntile
    out = {"col": lambda t: _group_norms(t, (1, 2)), "row": lambda t: _group_norms(t, (1, 3))}
    if nb > 1:
        pad = nb * ntile - C

        def blk(t):
            t = F.pad(t, (0, 0, 0, 0, 0, pad)) if pad else t
            return t.view(B, nb, ntile, H, W).pow(2).sum(dim=(0, 2, 3, 4)).sqrt()
        out["ntile"] = blk
    sizes = {"col": C * H, "row": C * W, "ntile": B * ntile * H * W}
    # class of each group: 1 for the image's first / last column (row), 0 otherwise
    edge = lambda n: torch.tensor([i in (0, n - 1) for i in range(n)] * B, device=x.device)
    classes = {"col": edge(W), "row": edge(H), "ntile": torch.zeros(nb, dtype=torch.bool, device=x.device)}
    nfull = W // period if period else 0
    if nfull >= 1:
        def phase(t):
            t = t[..., :nfull * period].clone()
            t[..., 0] = 0
            if nfull * period == W:
                t[..., W - 1] = 0
            return t.reshape(B, C, H, nfull, period).pow(2).sum(dim=(0, 1, 2, 3)).sqrt()
        out["phase"] = phase
        sizes["phase"] = B * C * H * nfull
        classes["phase"] = torch.zeros(period, dtype=torch.bool, device=x.device)
    return out, sizes, classes


def uniformity(err, A, Alin=None, min_group=MIN_GROUP, valid=None, ntile=64, period=None):
    """max over groupings of  max_g e_g / median of the other groups' e_g  (0 when the error is zero everywhere).
    `valid` (0/1, the shape of err): groups with fewer than min_group valid elements are left out."""
    Alin = A if Alin is None else Alin
    fns, sizes, classes = groupings(err, ntile, period)
    worst, where = 0.0, ""
    for name, fn in fns.items():
        if sizes[name] < min_group:
            continue
        en, an, ln = fn(err), fn(A), fn(Alin)
        # groups with a full share of data: a column in the padding (only |bias|), or one past a mask edge that sees 1 of 3
        # kernel columns, has a different mix of rounding sources (output rounding against a bias, not a dot product)
        has = ln > 1e-9 * ln.max().clamp_min(1e-300)
        if has.sum() < 2:
            continue
        full = ln >= 0.5 * ln[has].median()
        if valid is not None:
            full &= fn(valid.double()).pow(2) >= min_group
        for cls in (False,):                                    # interior groups only (see R_UNIFORM)
            ok = full & (classes[name] == cls)
            if ok.sum() < 2:
                continue
            r, i = _max_over_median((en[ok] / an[ok]).double())
            if r > worst:
                worst, where = r, f"{name}[{int(ok.nonzero()[i])}]"
    return worst, where


def _max_over_median(e):
    """-> (max e / median of the others, index of the max)"""
    i = int(e.argmax())
    med = torch.cat([e[:i], e[i + 1:]]).median().item()
    emax = e[i].item()
    return (0.0 if emax == 0.0 else (math.inf if med == 0.0 else emax / med)), i


# ---- check 2 on 1-D signals [B, C, L] (the vocoder's Conv1d, GEMM and fold outputs) -------------------------------------
# The Conv1d / 1x1 wgmma kernels tile a signal into TPX = 128-sample strips per N-tile block of output channels
# (sbk_conv_tc.cu).  A defect at a strip seam, in a halo, in one warpgroup half or descriptor offset, or in one N tile shows
# up in one of these groups.  e_g = ||err_g|| / ||Alin_g||: the rounding error scales with the op's own products, while the
# bias and the ResBlock residual that A also carries vary between samples without adding error beyond one fp32 rounding.
# Samples within `pad` of either end see zero-padding taps (a different mix of terms); they are left out here and held to
# check 1, which a stale or non-zero padding value fails many times over.  The same R_UNIFORM applies: on an H100 the
# vocoder's worst ratio was 2.6 (per-sample groups of the 32-channel last stage, the smallest groups), while one dropped
# tap term of a K = 704 Conv1d gives ~80 (test_op_replay.py).
TPX = 128


def groupings1d(x, pad, ntile):
    """[B,C,L] -> {name: fn}: each sample (b, w) over its channels, each 128-sample tile (b, w // 128), each within-tile
    phase w % 128 over the full interior tiles (a defect that repeats in every tile), each `ntile`-channel block."""
    B, C, L = x.shape
    nt = (L + TPX - 1) // TPX

    def tiles(t):
        return F.pad(t, (0, nt * TPX - L)).view(B, C, nt, TPX)
    out = {"sample": lambda t: _group_norms(t, (1,)), "tile": lambda t: _group_norms(tiles(t), (1, 3))}
    inner = [j for j in range(nt) if j * TPX >= pad and (j + 1) * TPX <= L - pad]
    if inner:
        lo, hi = inner[0], inner[-1] + 1
        out["phase"] = lambda t: _group_norms(tiles(t)[:, :, lo:hi], (0, 1, 2))
    if C % ntile == 0 and C // ntile > 1:
        out["ntile"] = lambda t: _group_norms(t.reshape(B, C // ntile, ntile, L), (0, 2, 3))
    return out


def uniformity1d(err, Alin, pad=0, ntile=128, min_group=MIN_GROUP):
    """max over the 1-D groupings of  max_g e_g / median of the other groups' e_g, edge samples left out."""
    B, C, L = err.shape
    valid = torch.zeros(L, dtype=torch.float64, device=err.device)
    valid[pad:max(pad, L - pad)] = 1.0
    valid = valid.expand(B, C, L)
    err, Alin = err * valid, Alin.double() * valid
    worst, where = 0.0, ""
    for name, fn in groupings1d(err, pad, ntile).items():
        en, ln, cnt = fn(err), fn(Alin), fn(valid).pow(2).round()
        ok = (cnt >= min_group) & (ln > 0)
        if ok.sum() < 2:
            continue
        r, i = _max_over_median((en[ok] / ln[ok]).double())
        if r > worst:
            worst, where = r, f"{name}[{int(ok.nonzero()[i])}]"
    return worst, where


def check(got, ref, A, kap, floor=0.0, Alin=None, groups=True, min_group=MIN_GROUP, pad=0, ntile=None, period=None,
          valid=None):
    """-> (elem, unif, where): elem = max |err| / (kappa A + floor) (<= 1 passes), unif = worst max/median group ratio.
    4-D [B,C,H,W] tensors are grouped as images (`ntile`, default 64, `period` and `valid`: groupings / uniformity);
    3-D [B,C,L] tensors as 1-D signals (`pad`, `ntile`, default 128: uniformity1d)."""
    got, ref, A = got.double(), ref.double(), A.double()
    err = (got - ref).abs()
    tiny = torch.finfo(torch.float32).tiny
    elem = (err / (kap * A + floor + tiny)).max().item()
    if groups and err.dim() == 4:
        unif, where = uniformity(err, A, Alin, min_group, valid, ntile=ntile or 64, period=period)
    elif groups and err.dim() == 3:
        unif, where = uniformity1d(err, A if Alin is None else Alin, pad, ntile or 128, min_group)
    else:
        unif, where = 0.0, ""
    return elem, unif, where


def passes(elem, unif):
    return elem <= 1.0 and unif <= R_UNIFORM


# ---- the U-Net graph as the plan builds it (sbk_api.cu build_plan) --------------------------------------------------------
# resnet prefix -> (level, inputs: names of the captured tensors concatenated along C; None = the planar first-block stack)
RESNETS = {
    "downs.0.0": (0, None), "downs.0.1": (0, ["downs.0.0.out"]),
    "downs.1.0": (1, ["downs.0.3.out"]), "downs.1.1": (1, ["downs.1.0.out"]),
    "downs.2.0": (2, ["downs.1.3.out"]), "downs.2.1": (2, ["downs.2.0.out"]),
    "mid_block1": (2, ["downs.2.2.out"]), "mid_block2": (2, ["mid_attn.out"]),
    "ups.0.0": (2, ["mid_block2.out", "downs.2.2.out"]), "ups.0.1": (2, ["ups.0.0.out"]),
    "ups.1.0": (1, ["ups.0.3.out", "downs.1.2.out"]), "ups.1.1": (1, ["ups.1.0.out"]),
}
ATTNS = {"downs.0.2": (0, "downs.0.1.out"), "downs.1.2": (1, "downs.1.1.out"), "downs.2.2": (2, "downs.2.1.out"),
         "mid_attn": (2, "mid_block1.out"), "ups.0.2": (2, "ups.0.1.out"), "ups.1.2": (1, "ups.1.1.out")}
RESAMPLES = {"downs.0.3": ("down", 0, 1, "downs.0.2.out"), "downs.1.3": ("down", 1, 2, "downs.1.2.out"),
             "ups.0.3": ("up", 2, 1, "ups.0.2.out"), "ups.1.3": ("up", 1, 0, "ups.1.2.out")}
# tensors that feed LinearAttention keep their padded columns (test_parity_gpu.py ATTN_INPUTS)
ATTN_INPUTS = {f"estimator.{v}" for _, v in ATTNS.values()}
# plan ops with no captured tensor, and where each is checked instead
SKIP = {
    ".block1.act": "the Block activation in operand form is not captured; block2.raw is replayed from a float64 rebuild "
                   "of it (GN + Mish + time bias of the captured block1.raw), so a wrong activation fails block2.raw",
    ".kvpart": "softmax partials in the kernel's private per-item layout; their merge is checked through .ctx",
    ".mix": "the folded per-sample attention matrix g*Wout*ctx^T*Wq; it is checked through the attention's .out",
}


def skip_reason(name):
    for suf, why in SKIP.items():
        if name.endswith(suf):
            return why
    return None


def ntile_widths(sd, B, H0, T, num_sms):
    """N-tile widths the planner picks for the tensor-core 3x3 convs (sbk_api.cu tc_conv): Cout % 128 == 0 runs 128-wide
    tiles unless B * ceil(W/128) * H * Cout/128 tiles would fill at most half the SMs, then 64-wide."""
    Hs, Ws = (H0, H0 // 2, H0 // 4), (T, T // 2, T // 4)
    convs = []
    for pre, (lvl, ins) in RESNETS.items():
        cout = sd[f"estimator.{pre}.block1.block.0.weight"].shape[0]
        convs += [(lvl, cout)] * (1 if ins is None else 2)    # downs.0.0.block1 runs on CUDA cores
    convs.append((0, sd["estimator.final_block.block.0.weight"].shape[0]))
    widths = set()
    for lvl, cout in convs:
        nt = 64
        if cout % 128 == 0:
            tiles = B * ((Ws[lvl] + 127) // 128) * Hs[lvl] * (cout // 128)
            nt = 64 if tiles * 2 <= num_sms else 128
        widths.add(nt)
    return widths


# ---- the replay ------------------------------------------------------------------------------------------------------
def _lin(fn, x, w, b, **kw):
    """(ref, A, floor, Alin) of one linear op: fn on the values and on the magnitudes (A: plus |bias|; Alin: without)."""
    ref = fn(x, w, b, **kw)
    Alin = fn(x.abs(), w.abs(), None, **kw)
    A = Alin if b is None else Alin + fn(torch.zeros_like(x[:, :1, :1, :1]).expand_as(x), w.abs(), b.abs(), **kw)
    floor = FLOOR_PER_W * w.abs().flatten(1).sum(1).max().item()
    return ref, A, floor, Alin


def _f32(v):
    return v.float().double()


def _gn_mish(p, blk, raw):
    """Block.forward's GN + Mish (oracle conv_gn_mish, after its conv) on a given raw conv output.  F.group_norm's
    statistics, rounded to fp32 where every GN consumer rounds them (sbk_kernels.cu gn_mean_rstd / gn_fill: fp32 mean,
    rstd and rstd * gamma, from an fp32 1/count): that rounding is one constant per (sample, group), an error that is
    correlated over the whole group and so would not average out like the rounding noise check 2 compares."""
    B, C, H, W = raw.shape
    g = raw.view(B, O.GROUPS, -1)
    inv = _f32(torch.tensor(1.0 / g.shape[-1], dtype=torch.float64))
    mean = g.sum(-1) * inv
    var = ((g * g).sum(-1) * inv - mean * mean).clamp_min(0.0)
    rstd = _f32(1.0 / torch.sqrt(var + 1e-5))
    cpg = C // O.GROUPS
    mean = _f32(mean).repeat_interleave(cpg, 1)[:, :, None, None]
    scale = _f32(rstd.repeat_interleave(cpg, 1) * _f32(p[f"{blk}.block.1.weight"])[None])[:, :, None, None]
    beta = p[f"{blk}.block.1.bias"][None, :, None, None]
    y = (raw - mean) * scale + beta
    return O.mish(y), 1.1 * ((raw - mean).abs() * scale.abs() + beta.abs())


def ctx_replay(x, wqkv, mode, tc=True):
    """LinearAttention's context softmax_n(k) v^T over all H*W pixels of x [B,C,H,W] (rezero_linear_attention up to its
    einsum) -> (ref, A, kappa): ref [B, heads, 32, 32]."""
    b, c, hh, ww = x.shape
    K_items = math.ceil(hh * ww / 64)
    kp = kappa(mode, c, tc=tc)                         # the k | v projection
    qkv = F.conv2d(x, wqkv).reshape(b, 3, O.HEADS, -1, hh * ww)
    qkvA = F.conv2d(x.abs(), wqkv.abs()).reshape(b, 3, O.HEADS, -1, hh * ww)
    k, v, kA, vA = qkv[:, 1], qkv[:, 2], qkvA[:, 1], qkvA[:, 2]
    pr = k.softmax(dim=-1)
    ref = torch.einsum("bhdn,bhen->bhde", pr, v)
    # linearised softmax: dp_n = p_n (dk_n - sum_m p_m dk_m), |dk| <= kappa kA, |dv| <= kappa vA
    A = (torch.einsum("bhdn,bhen->bhde", pr, vA) + torch.einsum("bhdn,bhen->bhde", pr * kA, v.abs())
         + (pr * kA).sum(-1)[..., None] * torch.einsum("bhdn,bhen->bhde", pr, v.abs()))
    # + P and V rounded for the context product (tf32 datapath: 2 x 2^-10; fp32x3: the split, 2^-19; fp32: exact
    # operands, 64-pixel FFMA chains) + the merge of one partial per 64-pixel item
    pv = {"tf32": 2 ** -9, "bf16": 2 ** -9, "fp32x3": 2 ** -19, "fp32": 128 * 2 ** -24}[mode]
    return ref, A, kp + pv + K_items * 2 ** -22 + EPS_NL


def crop_utterance(t, b, W):
    """utterance b of a tensor at a ragged call's dense shape [B, ..., W_dense]: its row, its first W columns"""
    return t[b:b + 1, ..., :W]


class Replay:
    """Run one estimator call with debug capture and judge every captured op against its float64 replay.

    model: "gradtts" (x, mask, mu, t, spk) or "diffvc" (x, mask, mean, t, cond).  `sd` is the state_dict the engine holds.

    `lengths` makes it a ragged call (`Engine.estimator / vc_estimator(..., lengths=)`), in which utterance b is the B = 1
    call on its own T_b = fix_len_compatibility(lengths[b]) frames, with its own t and spk (Grad-TTS) or cond (DiffVC) row.  Each utterance is then judged on its own: the inputs
    are sliced to row b and [:T_b], every capture is decoded at the call's dense shape and cropped to [b:b+1, ..., :W_b,l]
    (W_b,l = T_b >> l at level l), and the output to [b, :, :T_b].  The replay judges nothing past an utterance's edge;
    what the call left there is the caller's to check (e.g. that the output is 0)."""

    def __init__(self, eng, sd, mode, model, x, mask, mu, t, spk=None, cond=None, dim=64, pe_scale=1000.0, dev="cuda",
                 lengths=None):
        self.eng, self.mode, self.model, self.dev = eng, mode, model, dev
        self.tc = mode != "fp32"
        self.dim, self.pe_scale = dim, pe_scale
        d = torch.float64
        self.p = {k: v.to(dev, d) for k, v in sd.items()}
        L = None if lengths is None else torch.as_tensor(lengths, dtype=torch.int64).cuda()
        eng.debug_capture(True)
        try:
            if model == "diffvc":
                y = eng.vc_estimator(x.cuda(), mask.cuda(), mu.cuda(), cond.cuda(), t.cuda(), lengths=L)
            else:
                y = eng.estimator(x.cuda(), mask.cuda(), mu.cuda(), t.cuda(), None if spk is None else spk.cuda(),
                                  lengths=L)
            torch.cuda.synchronize()
        finally:
            eng.debug_capture(False)
        self.full = {"y": y.to(dev, d), "x": x.to(dev, d), "mask": mask.to(dev, d), "mu": mu.to(dev, d),
                     "t": t.to(dev, d), "spk": None if spk is None else spk.to(dev, d),
                     "cond": None if cond is None else cond.to(dev, d)}
        B, H0, T = x.shape
        self.dense = (B, (H0, H0 // 2, H0 // 4), (T, T // 2, T // 4))
        # the units judged one by one: the whole call (None), or each utterance (b, T_b) of a ragged one
        self.utts = [None] if lengths is None else [(b, fix_len_compatibility(int(n))) for b, n in enumerate(lengths)]
        self.names = eng.debug_names()
        self.dense_cap = {}                 # captures decoded at the call's shape (fp32, as captured)
        self.nonfinite = []                 # judged captures (cropped) holding a NaN or Inf
        self.select(None if lengths is None else self.utts[0])

    def select(self, utt):
        """Judge `utt` = (b, T_b), utterance b of a ragged call on its own frames, or (None) the whole call."""
        f, self.utt = self.full, utt
        if utt is None:
            row, frames = (lambda v: v), (lambda v: v)
        else:
            b, Tb = utt
            row, frames = (lambda v: v[b:b + 1]), (lambda v: v[b:b + 1, ..., :Tb])
        self.y, self.x, self.mask, self.mu = (frames(f[k]) for k in ("y", "x", "mask", "mu"))
        self.t = row(f["t"])
        self.spk = None if f["spk"] is None else row(f["spk"])
        self.cond = None if f["cond"] is None else row(f["cond"])
        B, H0, T = self.x.shape
        self.B, self.Hs, self.Ws = B, (H0, H0 // 2, H0 // 4), (T, T // 2, T // 4)
        m = self.mask[:, None]
        self.masks = [m, m[..., ::2], m[..., ::4]]
        # the time embedding: GradLogPEstimator2d.forward's first lines (oracle estimator / diffvc conditioning)
        p = self.p
        temb = O.sinusoid(self.t, self.dim, self.pe_scale)
        temb = F.linear(temb, p["estimator.mlp.0.weight"], p["estimator.mlp.0.bias"])
        self.temb = F.linear(O.mish(temb), p["estimator.mlp.2.weight"], p["estimator.mlp.2.bias"])
        self.cap = {}
        self.tag = "" if utt is None else f" b={utt[0]} W=({self.Ws[0]},{self.Ws[1]},{self.Ws[2]})"

    def crop(self, t, lvl):
        """a tensor at the call's shape [B, C, H, W_l] -> the selected unit's part of it"""
        return t if self.utt is None else crop_utterance(t, self.utt[0], self.Ws[lvl])

    def got(self, name, C, lvl):
        if name not in self.cap:
            if name not in self.dense_cap:
                flat = self.eng.debug_read(name)
                assert flat is not None, f"{name}: the plan names it but captured nothing"
                B, Hs, Ws = self.dense
                self.dense_cap[name] = nhwc_to_nchw(flat, B, Hs[lvl], Ws[lvl], C,
                                                    self.eng.debug_layout(name)).to(self.dev)
            self.cap[name] = self.crop(self.dense_cap[name], lvl).to(torch.float64)
        return self.cap[name]

    def got_ctx(self, q):
        """the captured LinearAttention context [B, heads, 32, 32] of attention `q`, the selected unit's rows"""
        name = f"{q}.ctx"
        if name not in self.dense_cap:
            self.dense_cap[name] = self.eng.debug_read(name).view(self.dense[0], O.HEADS, 32, 32).to(self.dev)
        t = self.dense_cap[name]
        return (t if self.utt is None else t[self.utt[0]:self.utt[0] + 1]).to(torch.float64)

    def judged_names(self):
        """the captured ops run() replays (all but SKIP's, and the output, which the call returns)"""
        return [n for n in self.names if skip_reason(n) is None and n != "estimator.out"]

    def hold(self):
        """read every judged capture now: the engine keeps only its last call's, which a later call replaces"""
        utt = self.utt
        for n in self.judged_names():
            self.capture(n)
        self.select(utt)
        return self

    def capture(self, name):
        """the selected unit's capture of a replayed op `name` ([B, C, H, W_l]; a context [B, heads, 32, 32])"""
        if name.endswith(".ctx"):
            return self.got_ctx(name[:-len(".ctx")])
        if name == "estimator.final_block.raw":
            return self.got(name, self.p["estimator.final_block.block.0.weight"].shape[0], 0)
        key = name.replace(".block1.raw", ".out").replace(".block2.raw", ".out")
        return self.got(name, self._chan(key), self._level_of(key))

    def _chan(self, name):
        """channels of a captured resnet / attention / resample output"""
        pre = name[len("estimator."):].rsplit(".", 1)[0]
        if pre in RESNETS:
            return self.p[f"estimator.{pre}.block1.block.0.weight"].shape[0]
        if pre in ATTNS:
            return self.p[f"estimator.{pre}.fn.fn.to_out.weight"].shape[0]
        return self.p[f"estimator.{pre}.conv.weight"].shape[0]

    def _level_of(self, name):
        pre = name[len("estimator."):].rsplit(".", 1)[0]
        if pre in RESNETS:
            return RESNETS[pre][0]
        if pre in ATTNS:
            return ATTNS[pre][0]
        return RESAMPLES[pre][2]

    def captured(self, short):
        name = f"estimator.{short}"
        return self.got(name, self._chan(name), self._level_of(name))

    def first_stack(self):
        """[mu, x(, spk_s)] (oracle estimator) or [mean, x, cond] (diffvc_oracle estimator): the first Block's input."""
        p, mu, x = self.p, self.mu, self.x
        if self.model == "diffvc":
            h = torch.stack([mu, x], 1)
            return torch.cat([h, self.cond[:, :, None, None].expand(-1, -1, h.shape[2], h.shape[3])], 1)
        if self.spk is None:
            return torch.stack([mu, x], 1)
        s = F.linear(self.spk, p["estimator.spk_mlp.0.weight"], p["estimator.spk_mlp.0.bias"])
        s = F.linear(O.mish(s), p["estimator.spk_mlp.2.weight"], p["estimator.spk_mlp.2.bias"])
        return torch.stack([mu, x, s[:, :, None].repeat(1, 1, x.shape[-1])], 1)

    def store_mask(self, name, lvl, ref, A):
        if self.tc and name not in ATTN_INPUTS:
            mk = self.masks[lvl]
            return ref * mk, A * mk
        return ref, A

    # -- one entry per op kind; each returns (got, ref, A, kappa, floor, Alin)
    def resnet_op(self, pre, part):
        p, mode, tc = self.p, self.mode, self.tc
        lvl, ins = RESNETS[pre]
        q = f"estimator.{pre}"
        mk = self.masks[lvl]
        if ins is None:
            xin, recomputed = self.first_stack(), self.spk is not None or self.model == "diffvc"
        else:
            xin, recomputed = torch.cat([self.captured(n) for n in ins], 1), False
        cin, cout = xin.shape[1], p[f"{q}.block1.block.0.weight"].shape[0]
        b16 = mode == "bf16"
        if part == "block1.raw":
            # conv_gn_mish: conv3x3(x*mask) + b; the first Block runs on CUDA cores in every mode
            w, b = p[f"{q}.block1.block.0.weight"], p[f"{q}.block1.block.0.bias"]
            ref, A, floor, Alin = _lin(F.conv2d, xin * mk, w, b, padding=1)
            k = kappa(mode, 9 * cin, tc=tc and ins is not None, extra=EPS_RECOMPUTED if recomputed else 0.0)
            return self.got(f"{q}.block1.raw", cout, lvl), ref, A, k, floor, Alin
        raw1 = self.got(f"{q}.block1.raw", cout, lvl)
        if part == "block2.raw":
            # resnet: h = conv_gn_mish(block1) + mlp(temb); block2 = conv3x3(h*mask) + b
            tb = F.linear(O.mish(self.temb), p[f"{q}.mlp.1.weight"], p[f"{q}.mlp.1.bias"])[:, :, None, None]
            act = (_gn_mish(p, f"{q}.block1", raw1)[0] * mk + tb) * mk
            if mode in ("tf32", "bf16"):                   # k_gn_act's rounding of the operand it writes
                act = (round_tf32_rna if mode == "tf32" else round_bf16)(act.float()).double()
            w, b = p[f"{q}.block2.block.0.weight"], p[f"{q}.block2.block.0.bias"]
            ref, A, floor, Alin = _lin(F.conv2d, act, w, b, padding=1)
            # The CUDA-core fp32 mode forms this conv's input in its prologue from a time bias the GPU evaluates in fp32:
            # that per-channel mismatch with the float64 replay (~1e-7, the same at every pixel) outweighs the conv's own
            # rounding there and measured up to 4x max/median on rows next to the image border, so in that mode
            # block2.raw is held to check 1 only (the path has no wgmma tiles for check 2 to look at).
            groups = Alin if tc else False
            return self.got(f"{q}.block2.raw", cout, lvl), ref, A, kappa(mode, 9 * cout, tc=tc, nl=True), floor, groups
        # part == "out": Mish(GN(raw2))*mask + res(x*mask)
        raw2 = self.got(f"{q}.block2.raw", cout, lvl)
        h, hA = _gn_mish(p, f"{q}.block2", raw2)
        h, hA = h * mk, hA * mk
        wname = f"{q}.res_conv.weight"
        if wname in p:
            res, Ares, floor, Alin = _lin(F.conv2d, xin * mk, p[wname], p[f"{q}.res_conv.bias"])
            # the planar first block's 1x1 runs on CUDA cores; in the tensor-core modes every other 1x1 on the tensor cores
            on_tc = tc and ins is not None
            k = kappa(mode, cin, tc=on_tc, nl=True, store_bf16=b16, extra=EPS_RECOMPUTED if recomputed else 0.0)
        else:
            res, Ares, floor = xin * mk, (xin * mk).abs(), 0.0
            Alin = Ares
            k = kappa(mode, 1, tc=False, nl=True, store_bf16=b16)
        ref, A, Alin = h + res, hA + Ares, hA + Alin
        ref, A = self.store_mask(f"{q}.out", lvl, ref, A)
        _, Alin = self.store_mask(f"{q}.out", lvl, ref, Alin)
        return self.got(f"{q}.out", cout, lvl), ref, A, k, floor, Alin

    def attn_op(self, pre, part):
        """rezero_linear_attention, split at the captured context."""
        p, mode = self.p, self.mode
        lvl, src = ATTNS[pre]
        q = f"estimator.{pre}"
        x = self.captured(src)
        b, c, hh, ww = x.shape
        wqkv = p[f"{q}.fn.fn.to_qkv.weight"]
        if part == "ctx":
            ref, A, k_ctx = ctx_replay(x, wqkv, mode, self.tc)
            got = self.got_ctx(q)
            return got, ref, A, k_ctx, 0.0, False          # [B, heads, 32, 32]: no columns or rows to group
        # part == "out": g * to_out(ctx^T q) + x from the captured ctx
        ctx = self.got_ctx(q)
        wq = wqkv[:O.HEADS * 32]
        g, wo, bo = p[f"{q}.fn.g"], p[f"{q}.fn.fn.to_out.weight"], p[f"{q}.fn.fn.to_out.bias"]
        qq = F.conv2d(x, wq).reshape(b, O.HEADS, -1, hh * ww)
        qA = F.conv2d(x.abs(), wq.abs()).reshape(b, O.HEADS, -1, hh * ww)
        out = torch.einsum("bhde,bhdn->bhen", ctx, qq).reshape(b, -1, hh, ww)
        outA = torch.einsum("bhde,bhdn->bhen", ctx.abs(), qA).reshape(b, -1, hh, ww)
        ref = F.conv2d(out, wo, bo) * g + x
        Alin = F.conv2d(outA, wo.abs()) * g.abs() + x.abs()
        A = Alin + bo.abs()[None, :, None, None] * g.abs()
        # the folded matrix g*Wout*blockdiag(ctx^T)*Wq is formed in fp32 (32 + 128 terms per entry), then applied as a 1x1
        k = kappa(mode, c, tc=self.tc, store_bf16=mode == "bf16", extra=160 * 2 ** -24)
        _, Alin = self.store_mask(f"{q}.out", lvl, ref, Alin)
        ref, A = self.store_mask(f"{q}.out", lvl, ref, A)
        return self.got(f"{q}.out", c, lvl), ref, A, k, 0.0, Alin

    def resample_op(self, pre):
        p, mode = self.p, self.mode
        kind, li, lo, src = RESAMPLES[pre]
        q = f"estimator.{pre}"
        x = self.captured(src) * self.masks[li]
        w, b = p[f"{q}.conv.weight"], p[f"{q}.conv.bias"]
        c = w.shape[0] if kind == "down" else w.shape[1]
        if kind == "down":
            ref, A, floor, Alin = _lin(F.conv2d, x, w, b, stride=2, padding=1)
            K = 9 * x.shape[1]
        else:
            ref, A, floor, Alin = _lin(F.conv_transpose2d, x, w, b, stride=2, padding=1)
            K = 4 * x.shape[1]
        if self.tc:
            ref, A, Alin = ref * self.masks[lo], A * self.masks[lo], Alin * self.masks[lo]
        k = kappa(mode, K, tc=self.tc, store_bf16=mode == "bf16")
        return self.got(f"{q}.out", c, lo), ref, A, k, floor, Alin

    def final_ops(self, name):
        p, mode = self.p, self.mode
        m = self.masks[0]
        if name == "estimator.final_block.raw":
            x = self.got("estimator.ups.1.3.out", self._chan("estimator.ups.1.3.out"), 0) * m
            w, b = p["estimator.final_block.block.0.weight"], p["estimator.final_block.block.0.bias"]
            ref, A, floor, Alin = _lin(F.conv2d, x, w, b, padding=1)
            return self.got(name, w.shape[0], 0), ref, A, kappa(mode, 9 * x.shape[1], tc=self.tc), floor, Alin
        # estimator.out: not captured; the call's own output, from the captured final_block.raw
        C = p["estimator.final_block.block.0.weight"].shape[0]
        h = _gn_mish(p, "estimator.final_block", self.got("estimator.final_block.raw", C, 0))[0] * m
        w, b = p["estimator.final_conv.weight"], p["estimator.final_conv.bias"]
        ref, A, floor, Alin = _lin(F.conv2d, h, w, b)
        return self.y[:, None], ref * m, A * m, kappa(mode, C, tc=False, nl=True), floor, Alin * m

    def run(self):
        """-> rows (name, elem, unif, where), per judged unit (the call, or each utterance: its name carries b and the
        utterance's level widths); raises on an op that is neither replayed nor in SKIP."""
        rows = []
        for utt in self.utts:
            self.select(utt)
            n0 = len(rows)
            for name in self.names:
                why = skip_reason(name)
                if why is not None:
                    continue
                assert name.startswith("estimator."), f"unknown op '{name}': add a replay for it or a reason to SKIP"
                short = name[len("estimator."):]
                pre, _, part = short.partition(".block")
                if short in ("final_block.raw", "out"):
                    r = self.final_ops(name)
                elif part in ("1.raw", "2.raw") and pre in RESNETS:
                    r = self.resnet_op(pre, "block" + part)
                else:
                    pre, part = short.rsplit(".", 1)
                    if pre in RESNETS and part == "out":
                        r = self.resnet_op(pre, "out")
                    elif pre in ATTNS and part in ("ctx", "out"):
                        r = self.attn_op(pre, part)
                    elif pre in RESAMPLES and part == "out":
                        r = self.resample_op(pre)
                    else:
                        raise AssertionError(f"unknown op '{name}': add a replay for it or a reason to SKIP")
                got, ref, A, k, floor, Alin = r
                assert got.shape == ref.shape, f"{name}: captured {tuple(got.shape)} vs replay {tuple(ref.shape)}"
                if not bool(torch.isfinite(got).all()):
                    self.nonfinite.append(name + self.tag)
                elem, unif, where = check(got, ref, A, k, floor, Alin, groups=Alin is not False)
                rows.append((name + self.tag, elem, unif, where))
            assert any(r[0] == "estimator.out" + self.tag for r in rows[n0:]), "the plan no longer names estimator.out"
        return rows


# ---- the HiFi-GAN vocoder (csrc/sbk_vocoder.cu), replayed op by op -------------------------------------------------------
# Every Conv1d, the transposed-conv GEMMs and conv_post are recomputed in float64 from the GPU's captured inputs with the
# semantics of oracle/hifigan_oracle.py.  The Conv1d kernels (k_conv_tc<G_C1K*>) and the GEMMs (k_conv_tc<G_PW>) run tf32
# operands with fp32 accumulation: kappa("tf32", K) with K = Cin * taps.  Their epilogue then adds the fp32 bias (and the
# ResBlock residual) and applies LeakyReLU: each add is one fp32 rounding of <= 2^-24 of a value bounded by A, and x * 0.1f
# one more; LeakyReLU is 1-Lipschitz, so it does not enlarge the error it receives.
EPS_ADD = 2 ** -24
# conv_post + tanh (k_voc_post) runs on CUDA cores: a chain of 7 * C fmaf from the bias, gamma_K = K * 2^-24 of A.  tanh is
# 1-Lipschitz, so that bound carries through it; tanhf adds its own error, at most 2 ulp (CUDA C Programming Guide,
# "Mathematical Functions": tanhf, maximum ulp error 2), and one ulp of y is at most 2^-23 |y|.
TANHF_ULP = 2
VOC_SLOPE = 0.1                         # LRELU_SLOPE (models.py:10); 0.01 (torch's default) before conv_post


def conv1d_ntile(C):
    """N-tile width of k_conv_tc for a Conv1d with C output channels (sbk_conv_tc.cu conv_tc_ntile, tf32 / bf16)"""
    return 128 if C % 128 == 0 else (64 if C % 64 == 0 else 32)


def gemm_ntile(C):
    return 128 if C % 128 == 0 else 64


def lrelu_f32(x, slope):
    """the kernels' LeakyReLU, bit for bit: x > 0 ? x : x * slope (fp32)"""
    x = x.float()
    return torch.where(x > 0, x, x * torch.tensor(slope, dtype=torch.float32, device=x.device))


def ct_fold(z, bias, u):
    """k_voc_ct_fold in fp32: ConvTranspose1d(k = 2u, stride u, padding u/2) as a 2-tap overlap-add of the GEMM output
    z [B, 2u*C, Lin] (channel t*C + c).  Output o (o + u/2 = u*i1 + t1) is (bias + z[t1, i1]) + z[t1 + u, i1 - 1], each
    tap skipped where its input sample lies outside the signal."""
    B, KC, Lin = z.shape
    Cc, p = KC // (2 * u), u // 2
    zz = z.float().view(B, 2 * u, Cc, Lin).permute(0, 2, 1, 3)              # [B, C, tap, Lin]
    o = torch.arange(Lin * u, device=z.device)
    i1, t1 = (o + p) // u, (o + p) % u
    x = bias.float()[None, :, None].expand(B, Cc, Lin * u).clone()
    m = i1 < Lin
    x[:, :, m] = x[:, :, m] + zz[:, :, t1[m], i1[m]]
    m = i1 >= 1
    x[:, :, m] = x[:, :, m] + zz[:, :, t1[m] + u, i1[m] - 1]
    return x


def _bitwise(got, ref):
    """(elem, unif, where) of an op that must reproduce `ref` bit for bit: elem 0 when equal, else inf"""
    same = got.shape == ref.shape and torch.equal(got.float(), ref.float())
    return (0.0 if same else math.inf), 0.0, "bitwise"


class VocoderReplay:
    """Run one vocoder call with debug capture and judge every captured op against its float64 (or bitwise) replay.
    `sd` holds the effective weights the engine was loaded with; `h` its config (oracle/hifigan_oracle.py keys)."""

    def __init__(self, eng, sd, h, mel, dev="cuda"):
        self.eng, self.h, self.dev = eng, h, dev
        self.p = {k: v.to(dev, torch.float64) for k, v in sd.items()}
        self.mel = mel.to(dev, torch.float32).contiguous()
        eng.debug_capture(True)
        try:
            self.wav = eng.forward(self.mel)
            torch.cuda.synchronize()
        finally:
            eng.debug_capture(False)
        self.names = eng.debug_names()
        self.cap = {}

    def got(self, name):
        if name not in self.cap:
            assert name in self.names, f"{name}: the vocoder did not capture it"
            self.cap[name] = self.eng.debug_read(name)
        return self.cap[name]

    def stage_input(self, i):
        """the activation operand a stage's transposed conv reads: lrelu(conv_pre) or lrelu(the previous MRF mean)"""
        return self.got("conv_pre" if i == 0 else f"mrf.{i - 1}")

    def _conv(self, x, w, b, dil, addin=None):
        """(ref, A, Alin, floor): Conv1d 'same' padding + bias (+ residual) on float64 copies, and its magnitude companions"""
        x = x.double()
        pad = (w.shape[2] - 1) * dil // 2
        ref = F.conv1d(x, w, b, padding=pad, dilation=dil)
        Alin = F.conv1d(x.abs(), w.abs(), None, padding=pad, dilation=dil)
        A = Alin + b.abs()[None, :, None]
        if addin is not None:
            ref, A = ref + addin.double(), A + addin.double().abs()
        return ref, A, Alin, FLOOR_PER_W * w.abs().flatten(1).sum(1).max().item()

    def conv_op(self, name):
        """conv_pre, resblocks.n.convs1.d (-> lrelu), resblocks.n.convs2.d.x (+ residual): the Conv1d kernels"""
        p, h = self.p, self.h
        if name == "conv_pre":
            x, w, b, dil, addin, act = self.got("mel_in"), p["conv_pre.weight"], p["conv_pre.bias"], 1, None, True
        else:
            _, n, grp, d = name.split(".")[:4]
            n, d = int(n), int(d)
            st, j = n // 3, n % 3
            pre = f"resblocks.{n}"
            w, b = p[f"{pre}.{grp}.{d}.weight"], p[f"{pre}.{grp}.{d}.bias"]
            if grp == "convs1":
                # input lrelu(x): the fold's second output, then each convs2's
                x = self.got(f"ups.{st}.a" if d == 0 else f"{pre}.convs2.{d - 1}.a")
                dil, addin, act = h["resblock_dilation_sizes"][j][d], None, True
            else:
                x, dil, act = self.got(f"{pre}.convs1.{d}"), 1, False
                addin = self.got(f"ups.{st}.x" if d == 0 else f"{pre}.convs2.{d - 1}.x")
        ref, A, Alin, floor = self._conv(x, w, b, dil, addin)
        if act:
            ref = F.leaky_relu(ref, VOC_SLOPE)
        K = w.shape[1] * w.shape[2]
        # bias add (+ residual add) + LeakyReLU's product, one fp32 rounding each
        k = kappa("tf32", K, extra=EPS_ADD * (1 + (addin is not None) + act))
        pad = (w.shape[2] - 1) * dil // 2
        return self.got(name), ref, A, k, floor, Alin, pad, conv1d_ntile(w.shape[0])

    def gemm_op(self, i):
        """ups.i.z: the transposed conv's 1x1 GEMM to k*co channels, channel t*co + c (sbk_vocoder_pack)"""
        w = self.p[f"ups.{i}.weight"]                                       # [ci, co, k]
        ci, co, k = w.shape
        g = w.permute(2, 1, 0).reshape(k * co, ci, 1)                       # [t*co + c][ci]
        x = self.stage_input(i).double()
        ref, Alin = F.conv1d(x, g), F.conv1d(x.abs(), g.abs())
        floor = FLOOR_PER_W * g.abs().flatten(1).sum(1).max().item()
        return self.got(f"ups.{i}.z"), ref, Alin, kappa("tf32", ci), floor, Alin, 0, gemm_ntile(k * co)

    def fold_vs_convt(self, i):
        """ups.i.x against torch's ConvTranspose1d (models.py:108) on the captured GEMM input: the GEMM's bound plus the
        fold's two fp32 adds"""
        u, k = self.h["upsample_rates"][i], self.h["upsample_kernel_sizes"][i]
        w, b = self.p[f"ups.{i}.weight"], self.p[f"ups.{i}.bias"]
        x = self.stage_input(i).double()
        ref = F.conv_transpose1d(x, w, b, stride=u, padding=(k - u) // 2)
        Alin = F.conv_transpose1d(x.abs(), w.abs(), None, stride=u, padding=(k - u) // 2)
        floor = 2 * FLOOR_PER_W * w.abs().sum(dim=(0, 2)).max().item()
        # the first / last u/2 samples receive one tap instead of two; the fold is elementwise (no N tiles of its own)
        return (self.got(f"ups.{i}.x"), ref, Alin + b.abs()[None, :, None], kappa("tf32", w.shape[0], extra=2 * EPS_ADD),
                floor, Alin, u // 2, w.shape[1])

    def wav_op(self):
        nu = len(self.h["upsample_rates"])
        x = self.got(f"mrf.{nu - 1}").double()
        w, b = self.p["conv_post.weight"], self.p["conv_post.bias"]
        pre = F.conv1d(x, w, b, padding=3)
        A = F.conv1d(x.abs(), w.abs(), b.abs(), padding=3)
        kA = w.shape[1] * w.shape[2] * 2 ** -24 * A
        ref = torch.tanh(pre)
        # per element: the FMA chain's bound through tanh, plus tanhf's 2 ulp of a result no larger than |ref| + kappa A
        bound = kA + TANHF_ULP * 2 ** -23 * (ref.abs() + kA) + torch.finfo(torch.float32).tiny
        return self.got("wav"), ref, bound

    def run(self):
        """-> rows (name, elem, unif, where); raises on a captured name this replay does not know"""
        rows = []
        nu = len(self.h["upsample_rates"])
        for name in self.names:
            parts = name.split(".")
            if name == "mel_in":
                rows.append((name,) + _bitwise(self.got(name), self.mel))
                continue
            if name == "wav":
                got, ref, bound = self.wav_op()
                # CUDA-core chain, no tiles; tanhf's ulp error is not proportional to A, so check 1 only
                rows.append((name,) + check(got, ref, bound, 1.0, groups=False))
                continue
            if parts[0] == "mrf" and len(parts) == 2:
                i = int(parts[1])
                r = [self.got(f"resblocks.{3 * i + j}.convs2.2.x").float() for j in range(3)]
                inv = torch.tensor(1.0 / 3.0, dtype=torch.float32, device=r[0].device)
                ref = lrelu_f32(((r[0] + r[1]) + r[2]) * inv, VOC_SLOPE if i + 1 < nu else 0.01)
                rows.append((name,) + _bitwise(self.got(name), ref))
                continue
            if parts[0] == "ups" and len(parts) == 3 and parts[2] in ("z", "x", "a"):
                i = int(parts[1])
                if parts[2] == "z":
                    r = self.gemm_op(i)
                elif parts[2] == "a":
                    rows.append((name,) + _bitwise(self.got(name), lrelu_f32(self.got(f"ups.{i}.x"), VOC_SLOPE)))
                    continue
                else:
                    u = self.h["upsample_rates"][i]
                    ref = ct_fold(self.got(f"ups.{i}.z"), self.p[f"ups.{i}.bias"].float(), u)
                    rows.append((name,) + _bitwise(self.got(name), ref))
                    got, ref, A, k, floor, Alin, pad, nt = self.fold_vs_convt(i)
                    rows.append((name + "~convT",) + check(got, ref, A, k, floor, Alin, pad=pad, ntile=nt))
                    continue
            elif name == "conv_pre" or (parts[0] == "resblocks" and len(parts) >= 4 and (
                    (parts[2] == "convs1" and len(parts) == 4) or (parts[2] == "convs2" and parts[4:] == ["x"]))):
                r = self.conv_op(name)
            elif parts[0] == "resblocks" and parts[2:3] == ["convs2"] and parts[4:] == ["a"] and int(parts[3]) < 2:
                x = self.got(name[:-2] + ".x")
                rows.append((name,) + _bitwise(self.got(name), lrelu_f32(x, VOC_SLOPE)))
                continue
            else:
                raise AssertionError(f"unknown vocoder op '{name}': add a replay for it")
            got, ref, A, k, floor, Alin, pad, nt = r
            assert got.shape == ref.shape, f"{name}: captured {tuple(got.shape)} vs replay {tuple(ref.shape)}"
            rows.append((name,) + check(got, ref, A, k, floor, Alin, pad=pad, ntile=nt))
        assert rows and rows[-1][0] == "wav", "the vocoder no longer captures wav last"
        return rows


# ---- DiffVC's RefBlock conditioning branch (sbk_api.cu sbk_vc_conditioning), replayed op by op -----------------------------
# One sbk_vc_conditioning call with capture on keeps the tensors of its last step (t = 1/N): the diffused reference, the
# step's time-bias row, and per block the conv output (raw), the InstanceNorm sums (stats) and IN + GLU (+ bias) * mask (act),
# then the masked-mean sums (ysum).  Each is recomputed in float64 from the GPU's own captured inputs with the semantics of
# oracle/diffvc_oracle.py ref_block / conditioning.  The branch runs tf32 operands on tf32 / bf16 handles and the fp32x3
# split on fp32x3 / fp32 handles.
RB_BLOCKS = ("block11", "block12", "block21", "block22", "block31", "block32")
RB_TBIAS = {"block12": (0, 1), "block22": (1, 3)}        # the block's slice of a tb row, in units of base = dim_cond / 4
FIRST_CONV_TILE = 256                                    # k_first_conv: 256 frames of one row per CTA, 64 output channels
TC_TILE = 128                                            # k_conv_tc<G_C3>: 128-pixel tiles of one row
U32 = 2 ** -24
# sinf / cosf: at most 2 ulp (CUDA C Programming Guide, "Mathematical Functions"), one ulp <= 2^-23 of the value
SIN_ULP = 2 * 2 ** -23
# k_in_glu, on top of the operand / activation roundings: fp32 (raw - mean), the fma with scale and beta, the mean and
# rstd * gamma rounded to fp32 from statistics that may land one ulp away from the float64 ones, the sigmoid (2 ulp expf +
# the division, or EPS_NL for __expf / __fdividef), the product with the value half and the time-bias add
IN_GLU_ROUNDINGS = 10


def rb_branch_mode(precision):
    return "fp32x3" if precision in ("fp32", "fp32x3") else "tf32"


def rb_ntile(cout):
    """N tile of the RefBlock's wgmma convs (sbk_conv_tc.cu conv_tc_ntile(G_C3, Cout, form), no planner override)"""
    return 128 if cout % 128 == 0 else 64


def rb_chain(Tr):
    """fp32 terms a k_chan_stats thread sums before it flushes to float64: 8 rows of ceil(Tr / 256) columns.  The ragged
    twin keeps the dense call's partitions of the Tr columns and only drops those at or past R_b, so rb_chain(Tr) bounds its
    chains too."""
    return 8 * math.ceil(Tr / 256)


def rb_conv(x, mask, w, b, got, mode, first=False):
    """blockXY.raw: Conv3x3(x * mask) + bias (ref_block's cig).  block11 runs on CUDA cores (k_first_conv, a 9-term FFMA
    chain from the bias); the others on wgmma (kappa(mode, 9 Cin)).  Uniformity over columns, rows, the conv's N tiles and
    the phase within its pixel tile; the image's border and the columns past a mask edge are left to check 1."""
    m4 = mask[:, None, None, :]
    ref, A, floor, Alin = _lin(F.conv2d, x * m4, w, b, padding=1)
    if first:
        return check(got, ref, A, kappa("fp32", 9 * w.shape[1]), floor, Alin, ntile=64, period=FIRST_CONV_TILE)
    return check(got, ref, A, kappa(mode, 9 * w.shape[1]), floor, Alin, ntile=rb_ntile(w.shape[0]), period=TC_TILE)


def rb_stats(raw, got, Tr):
    """[B,C,2] sums of x and x^2 over all H * Tr pixels (F.instance_norm normalises over the padded columns too).  Each
    k_chan_stats thread runs fp32 chains of rb_chain(Tr) terms (<= that many roundings of 2^-24 of the sum of |terms|),
    flushed into float64 (H * Tr more adds of 2^-53)."""
    s, q = raw.sum((2, 3)), (raw * raw).sum((2, 3))
    ref = torch.stack([s, q], -1)
    A = torch.stack([raw.abs().sum((2, 3)), q], -1)
    k = rb_chain(Tr) * U32 + raw.shape[2] * raw.shape[3] * 2 ** -53
    return check(got, ref, A, k, groups=False)


def rb_var_error(raw, got):
    """worst relative error of the variance k_in_glu derives from the captured sums, against the float64 variance"""
    n = raw.shape[2] * raw.shape[3]
    m = got[..., 0] / n
    var_gpu = (got[..., 1] / n - m * m).clamp_min(0.0)
    var = raw.var(dim=(2, 3), unbiased=False)
    return ((var_gpu - var).abs() / var.clamp_min(1e-300)).max().item()


def in_glu(raw, gamma, beta, tb, mask, mode):
    """k_in_glu on a captured raw [B,C,H,Tr]: InstanceNorm2d(affine) + GLU (+ time bias) * mask, float64 apart from the
    kernel's own roundings: mean and rstd * gamma to fp32, and in the tf32 branch the output to tf32 (rna).
    -> (ref, A): A bounds the magnitudes the rounding errors are relative to.  The reference does not mask the GLU output
    (cig masks the next conv's input instead); the kernel writes zeros there, which the next conv reads."""
    B, C, H, W = raw.shape
    n = H * W
    mean = raw.sum((2, 3)) / n
    var = ((raw * raw).sum((2, 3)) / n - mean * mean).clamp_min(0.0)
    mean_f = _f32(mean)[:, :, None, None]
    scale = _f32(_f32(1.0 / torch.sqrt(var + 1e-5)) * _f32(gamma)[None])[:, :, None, None]
    d = raw - mean_f
    xn = d * scale + beta[None, :, None, None]
    # companion of each normalised value: |raw - mean| |scale| + |beta|, plus |mean| |scale| for the mean's fp32 rounding
    An = (d.abs() + mean_f.abs()) * scale.abs() + beta.abs()[None, :, None, None]
    Ch = C // 2
    xa, xg, Aa, Ag = xn[:, :Ch], xn[:, Ch:], An[:, :Ch], An[:, Ch:]
    sig = torch.sigmoid(xg)
    tbv = torch.zeros(Ch, dtype=raw.dtype, device=raw.device) if tb is None else tb
    m4 = mask[:, None, None, :]
    y = (xa * sig + tbv[None, :, None, None]) * m4
    if mode == "tf32":
        y = round_tf32_rna(y.float()).double()
    # sigmoid' <= 1/4: an error in xg reaches the output as |xa| / 4 of it
    A = (Aa + 0.25 * xa.abs() * Ag + tbv.abs()[None, :, None, None]) * m4
    return y, A


def rb_act(raw, gamma, beta, tb, mask, got, mode):
    ref, A = in_glu(raw, gamma, beta, tb, mask, mode)
    # tf32: the replay rounds its output as the kernel does, so most elements match exactly and the few whose fp32 value
    # lies on the other side of a rounding boundary differ by one tf32 step (<= 2^-10 of the value); that sparse error has
    # no meaningful group ratio (see RB_NO_UNIFORMITY)
    k = IN_GLU_ROUNDINGS * U32 + (EPS_NL + 2 ** -10 if mode == "tf32" else 0.0)
    # groups need RB_MIN_VALID unmasked elements: a row of a one-frame reference holds only C/2 values
    valid = mask[:, None, None, :].expand_as(ref)
    return check(got, ref, A, k, groups=mode != "tf32", min_group=RB_MIN_VALID, valid=valid)


RB_MIN_VALID = 4 * MIN_GROUP


RB_NO_UNIFORMITY = {
    "xt_ref": "elementwise (k_diff_mean, no tiles); held to its per-element bound and to exact zeros past the mask",
    "tb": "one vector per step (k_time_table); no columns or rows",
    "stats": "one pair of sums per (sample, channel); no columns or rows",
    "act.tf32": "the replay is rounded to tf32 as the kernel rounds, so the error is a sparse set of one-step differences",
    "ysum": "one pair of sums per (sample, channel); no columns or rows",
    "cond": "one vector per sample (k_vc_cond); no columns or rows",
}


def _libm_expf():
    import ctypes
    import ctypes.util
    f = ctypes.CDLL(ctypes.util.find_library("m")).expf
    f.argtypes, f.restype = [ctypes.c_float], ctypes.c_float
    return f


def host_freqs(dim):
    """the sinusoid frequencies libsbk uploads (sbk_api.cu sbk_pack): expf((float)j * (float)(-log(10000) / (half - 1)))"""
    import numpy as np
    half = dim // 2
    neg = float(np.float32(-(math.log(10000.0) / (half - 1))))
    expf = _libm_expf()
    return torch.tensor([expf(float(np.float32(np.float32(j) * np.float32(neg)))) for j in range(half)], dtype=torch.float64)


def sinusoid_f32(t32, dim, dev):
    """(emb, bound): [sin | cos] of the fp32 argument fp32(fp32(1000 t) * freq), as k_time_table / k_vc_cond form it"""
    a = torch.tensor(1000.0, dtype=torch.float32) * torch.tensor(t32, dtype=torch.float32)
    arg = (a * host_freqs(dim).float()).double().to(dev)
    emb = torch.cat([arg.sin(), arg.cos()])
    return emb, SIN_ULP * emb.abs() + 2 ** -149


def ffma_layer(x, ex, w, b):
    """y = b + W x as a fp32 FFMA chain of K = fan-in terms from the bias: (ref, bound) for inputs x with error bound ex"""
    y = F.linear(x, w, b)
    prop = F.linear(ex, w.abs())
    A = F.linear(x.abs(), w.abs(), b.abs()) + prop
    return y, prop + (w.shape[1] + 1) * U32 * A


def mish_layer(h, eh):
    """Mish (mish_f, the exact closed form) of a value with error bound eh: |Mish'| <= 1.1, plus EPS_NL of 1.1 |h|"""
    return O.mish(h), 1.1 * eh + EPS_NL * 1.1 * (h.abs() + eh)


class RefBlockReplay:
    """Run one sbk_vc_conditioning call with debug capture and judge every op of its last step against a float64 replay.
    `sd` is the state_dict the engine holds; ref / mean_ref [B,H,Tr], ref_mask [B,1,Tr], c [B,256] (CPU fp32).

    `ref_lengths` makes it a ragged call (`vc_conditioning(..., ref_lengths=)`), in which reference b is the B = 1 call on
    its own R_b frames with an all-ones mask.  Each reference is then judged on its own: the inputs and every capture are
    cropped to [b:b+1, ..., :R_b], so the statistics, InstanceNorm and the masked mean normalise over H * R_b.  Nothing past
    R_b is judged (the caller's mask there is not the reference's own)."""

    def __init__(self, eng, sd, precision, cfg, ref, ref_mask, mean_ref, c, n_timesteps, dev="cuda", ref_lengths=None):
        self.eng, self.cfg, self.dev, self.N = eng, cfg, dev, n_timesteps
        self.mode = rb_branch_mode(precision)
        RL = None if ref_lengths is None else torch.as_tensor(ref_lengths, dtype=torch.int64).cuda()
        eng.debug_capture(True)
        try:
            self.table = eng.vc_conditioning(ref.cuda(), ref_mask.cuda(), mean_ref.cuda(), c.cuda(), n_timesteps,
                                             ref_lengths=RL)
            torch.cuda.synchronize()
        finally:
            eng.debug_capture(False)
        self.names = eng.vc_cond_debug_names()
        d = torch.float64
        self.p = {k: v.to(dev, d) for k, v in sd.items()}
        self.full = {"cap": {n: eng.vc_cond_debug_read(n).to(dev) for n in self.names}, "ref": ref.to(dev, d),
                     "mean_ref": mean_ref.to(dev, d), "c": c.to(dev, d), "mask": ref_mask[:, 0].to(dev, d),
                     "table": self.table.to(dev, d)}
        self.H, self.Tr = ref.shape[1], ref.shape[2]
        # the units judged one by one: the whole call (None), or each reference (b, R_b) of a ragged one
        self.units = [None] if ref_lengths is None else [(b, int(r)) for b, r in enumerate(ref_lengths)]
        self.select(None)
        # the host's scalars of the last step: t as fp32(1 - i / N), gamma(0, t) in double from the fp32 config betas
        i = n_timesteps - 1
        td = 1.0 - i * (1.0 / n_timesteps)
        self.t32 = float(torch.tensor(td, dtype=torch.float32))
        bmin, bmax = (float(torch.tensor(v, dtype=torch.float32)) for v in (cfg.beta_min, cfg.beta_max))
        bi = bmin + 0.5 * (bmax - bmin) * td
        bi *= td
        self.g = float(torch.tensor(math.exp(-0.5 * bi), dtype=torch.float32))
        self.base = cfg.dim_spk // 4

    def select(self, unit):
        """Judge `unit` = (b, R_b), reference b of a ragged call on its own frames, or (None) the whole call."""
        f, self.unit = self.full, unit
        if unit is None:
            row, frames = (lambda v: v), (lambda v: v)
            self.tag = ""
        else:
            b, R = unit
            row, frames = (lambda v: v[b:b + 1]), (lambda v: v[b:b + 1, ..., :R])
            self.tag = f" b={b} R={R}"
        self.ref, self.mean_ref, self.mask = frames(f["ref"]), frames(f["mean_ref"]), frames(f["mask"])
        self.c, self.table_last = row(f["c"]), row(f["table"][-1])
        # stats / ysum [B, C, 2] are per sample; tb is one row for the batch; the rest are [B, (C,) H, Tr] grids
        self.cap = {n: (row(v) if n.endswith((".stats", ".ysum")) else v if n == "ref_block.tb" else frames(v))
                    for n, v in f["cap"].items()}
        self.B = self.ref.shape[0]

    def _w(self, blk, part):
        return self.p[f"estimator.ref_block.{blk}.{part}"]

    def xt_ref(self):
        g = self.g
        m = self.mask[:, None, :]
        ref = (self.ref * g + self.mean_ref * (1.0 - g)) * m
        A = ((self.ref * g).abs() + (self.mean_ref * (1.0 - g)).abs()) * m
        got = self.cap["ref_block.xt_ref"]
        past = (m == 0).expand_as(got)
        assert not past.any() or got[past].abs().max().item() == 0.0, "xt_ref: non-zero past the mask"
        # ref * g, (1 - g), mean_ref * (1 - g) and the sum: four fp32 roundings
        return check(got, ref, A, 4 * U32, groups=False)

    def time_bias(self):
        """tb: k_time_table's Linear(dim, 4 dim) -> Mish -> Linear(4 dim, dim) -> Mish -> mlp1 | mlp2 on this step's t"""
        p = self.p
        emb, e = sinusoid_f32(self.t32, self.cfg.dim_unet, self.dev)
        h, e = ffma_layer(emb, e, p["estimator.mlp.0.weight"], p["estimator.mlp.0.bias"])
        h, e = mish_layer(h, e)
        h, e = ffma_layer(h, e, p["estimator.mlp.2.weight"], p["estimator.mlp.2.bias"])
        h, e = mish_layer(h, e)
        outs = [ffma_layer(h, e, p[f"estimator.ref_block.{m}.1.weight"], p[f"estimator.ref_block.{m}.1.bias"])
                for m in ("mlp1", "mlp2")]
        ref, bound = torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])
        return check(self.cap["ref_block.tb"], ref, bound, 1.0, groups=False)

    def cond(self):
        """the step's cond row from the captured ysum: ybar = ysum / (sum(mask) H) rounded to fp32 as k_vc_cond rounds it,
        final_conv, then cond_block over [sinusoid | final_conv(ybar) | c]"""
        p, dev = self.p, self.dev
        emb, e_emb = sinusoid_f32(self.t32, self.cfg.dim_unet, dev)
        emb, e_emb = emb.expand(self.B, -1), e_emb.expand(self.B, -1)
        parts, errs = [emb], [e_emb]
        if self.cfg.use_ref_t:
            den = self.mask.sum(1, keepdim=True) * self.H
            ybar = _f32(self.cap["ref_block.ysum"][..., 0] / den)
            y, e = ffma_layer(ybar, torch.zeros_like(ybar), p["estimator.ref_block.final_conv.weight"][:, :, 0, 0],
                              p["estimator.ref_block.final_conv.bias"])
            parts.append(y)
            errs.append(e)
        parts.append(self.c)
        errs.append(torch.zeros_like(self.c))
        h, e = ffma_layer(torch.cat(parts, 1), torch.cat(errs, 1), p["estimator.cond_block.0.weight"],
                          p["estimator.cond_block.0.bias"])
        h, e = mish_layer(h, e)
        ref, bound = ffma_layer(h, e, p["estimator.cond_block.2.weight"], p["estimator.cond_block.2.bias"])
        return check(self.table_last, ref, bound, 1.0, groups=False)

    def run(self):
        """-> rows (name, elem, unif, where), per judged unit (the call, or each reference: its name carries b and R_b);
        raises on a captured name this replay does not know, and on a non-zero act past the mask.  Also -> self.var_err:
        {block (+ unit): worst relative error of the variance from the captured sums}.  self.nonfinite lists the judged
        (cropped) captures that hold a NaN or Inf."""
        rows, self.var_err, self.nonfinite = [], {}, []
        known = {"ref_block.xt_ref", "ref_block.tb", "ref_block.ysum"}
        known |= {f"ref_block.{b}.{s}" for b in RB_BLOCKS for s in ("raw", "stats", "act")}
        for name in self.names:
            assert name in known, f"unknown RefBlock op '{name}': add a replay for it"
        for unit in self.units:
            self.select(unit)
            self.nonfinite += [n + self.tag for n, v in self.cap.items() if not bool(torch.isfinite(v).all())]
            rows += [(n + self.tag,) + tuple(r) for n, *r in self._run_unit()]
        return rows

    def _run_unit(self):
        rows = []
        if self.cfg.use_ref_t:
            assert self.names[:2] == ["ref_block.xt_ref", "ref_block.tb"] and self.names[-1] == "ref_block.ysum", self.names
            rows.append(("xt_ref",) + self.xt_ref())
            rows.append(("tb",) + self.time_bias())
            x = self.cap["ref_block.xt_ref"][:, None]
            for blk in RB_BLOCKS:
                raw = self.cap[f"ref_block.{blk}.raw"]
                rows.append((f"{blk}.raw",) + rb_conv(x, self.mask, self._w(blk, "0.weight"), self._w(blk, "0.bias"), raw,
                                                     self.mode, first=blk == "block11"))
                st = self.cap[f"ref_block.{blk}.stats"]
                rows.append((f"{blk}.stats",) + rb_stats(raw, st, self.Tr))
                self.var_err[blk + self.tag] = rb_var_error(raw, st)
                tb = None
                if blk in RB_TBIAS:
                    lo, hi = RB_TBIAS[blk]
                    tb = self.cap["ref_block.tb"][lo * self.base:hi * self.base]
                x = self.cap[f"ref_block.{blk}.act"]
                past = (self.mask == 0)[:, None, None, :].expand_as(x)
                assert not past.any() or x[past].abs().max().item() == 0.0, f"{blk}.act: non-zero past the mask"
                rows.append((f"{blk}.act",) + rb_act(raw, self._w(blk, "1.weight"), self._w(blk, "1.bias"), tb, self.mask, x,
                                                     self.mode))
            rows.append(("ysum",) + rb_stats(x, self.cap["ref_block.ysum"], self.Tr))
        else:
            assert not self.names, f"use_ref_t = False captured {self.names}"
        rows.append(("cond",) + self.cond())
        return rows


# ---- DiffVC's PostNet (csrc/sbk_postnet.cu), replayed op by op --------------------------------------------------------------
# One sbk_postnet_forward call with capture on keeps a0, each block's conv output (raw) and GroupNorm sums (stats), block1's
# Mish(GN) activation, and the residual conv's output (res); the call's own output is the last op.  Each is recomputed in
# float64 from the GPU's own captured inputs with the semantics of oracle/postnet_oracle.py.  fp32x3 / fp32 handles run the
# fp32x3 split, tf32 / bf16 handles tf32 operands (rb_branch_mode).
PN_GROUPS = 8
# fp32 roundings a GroupNorm partial sees before its float64 flush (sbk_conv_tc.cu, the epilogue's statistics): an 8-term
# chain, the 8 -> group-width merge (<= 2), the 32-lane shuffle (5), and the tile's 32-column chunks and passes (<= 8)
PN_STATS_CHAIN = 32
# k_pn_init: one fma, the exact mask product, and on tf32 handles the rna rounding of the stored operand (<= 2^-11 of the
# value; a value just above a power of two attains it, so tf32 a0 rows measure up to 0.999 of this bound on an H100)
PN_A0_TF32 = 2 ** -11


def pn_ntile(C, mode, geom):
    """N tile of the PostNet's wgmma convs (sbk_conv_tc.cu conv_tc_ntile): the 7x7 runs 64 wide in fp32x3"""
    if geom == "c7" and mode == "fp32x3":
        return 64
    return 128 if C % 128 == 0 else 64


def pn_inv_count(C, H, L):
    """the GroupNorm divisor the kernels use: fp32(1 / ((C/8) H L)), for a ragged sample from fp32((C/8) * H) (gn_inv_count_rag)
    - the same value as the dense fp32(1.0 / ((double)(C/8) * H * T)) at L = T"""
    cnt = float(torch.tensor(float(C // PN_GROUPS), dtype=torch.float32) * torch.tensor(float(H), dtype=torch.float32))
    return float(torch.tensor(1.0 / (cnt * L), dtype=torch.float32))


def pn_gn_mish(raw, stats, gamma, beta, inv):
    """Block's GroupNorm(8) + Mish on raw [B,C,H,W] from the GPU's captured sums `stats` [B,8,2] and the kernels' fp32 divisor
    `inv`, as gn_mean_rstd forms them: mean = s inv and var = ss inv - mean^2 in float64, mean and rstd * gamma rounded to
    fp32 (the sums themselves are judged by pn_stats) -> (value, companion 1.1 (|raw - mean| |scale| + |beta|))"""
    C = raw.shape[1]
    mean = stats[..., 0] * inv
    var = (stats[..., 1] * inv - mean * mean).clamp_min(0.0)
    rstd = _f32(1.0 / torch.sqrt(var + 1e-5))
    cpg = C // PN_GROUPS
    mean = _f32(mean).repeat_interleave(cpg, 1)[:, :, None, None]
    scale = _f32(rstd.repeat_interleave(cpg, 1) * _f32(gamma)[None])[:, :, None, None]
    y = (raw - mean) * scale + beta[None, :, None, None]
    return O.mish(y), 1.1 * ((raw - mean).abs() * scale.abs() + beta.abs()[None, :, None, None])


def pn_stats(raw, got):
    """[B, 8, 2] sums of x and x^2 over each group's channels and all H * W pixels of raw [B,C,H,W]"""
    B = raw.shape[0]
    g = raw.reshape(B, PN_GROUPS, -1)
    ref = torch.stack([g.sum(-1), (g * g).sum(-1)], -1)
    A = torch.stack([g.abs().sum(-1), (g * g).sum(-1)], -1)
    return check(got, ref, A, PN_STATS_CHAIN * U32 + g.shape[-1] * 2 ** -53, groups=False)


PN_NO_UNIFORMITY = {
    "a0": "elementwise (k_pn_init, no tiles); held to its per-element bound",
    "stats": "one pair of sums per (sample, group); no columns or rows",
    "act.tf32": "the replay is rounded to tf32 as k_gn_act rounds, so the error is a sparse set of one-step differences",
}


class PostNetReplay:
    """Run one PostNet forward with debug capture and judge every captured op, and the output, against a float64 replay.
    `eng` is a PostNetEngine loaded with `sd`; x [B,H,T], mask [B,1,T] (CPU fp32).

    `lengths` makes it a ragged call (`forward(..., lengths=)`), in which utterance b is the B = 1 call on its own L_b
    frames with an all-ones mask (no rounding of the length).  Each utterance is then judged on its own: every capture and
    the output are cropped to [b:b+1, ..., :L_b], and the GroupNorm count is (C/8) H L_b."""

    def __init__(self, eng, sd, precision, x, mask, lengths=None, dev="cuda"):
        self.eng, self.dev = eng, dev
        self.mode = rb_branch_mode(precision)
        L = None if lengths is None else torch.as_tensor(lengths, dtype=torch.int64).to(dev)
        eng.debug_capture(True)
        try:
            y = eng.forward(x.to(dev), mask.to(dev), L)
            if y.is_cuda:
                torch.cuda.synchronize()
        finally:
            eng.debug_capture(False)
        self.names = eng.debug_names()
        d = torch.float64
        self.p = {k: v.to(dev, d) for k, v in sd.items()}
        self.full = {"cap": {n: eng.debug_read(n).to(dev, d) for n in self.names}, "y": y.to(dev, d), "x": x.to(dev, d),
                     "mask": mask.to(dev, d)}
        self.C = self.p["init_conv.weight"].shape[0]
        self.units = [None] if lengths is None else [(b, int(n)) for b, n in enumerate(lengths)]
        self.select(None)

    def select(self, unit):
        f, self.unit = self.full, unit
        if unit is None:
            frames, self.tag = (lambda v: v), ""
            self.mask = f["mask"][:, :, None]                                  # [B, 1, 1, T]
        else:
            b, L = unit
            frames, self.tag = (lambda v: v[b:b + 1, ..., :L]), f" b={b} L={L}"
            self.mask = torch.ones(1, 1, 1, L, dtype=torch.float64, device=self.dev)
        self.cap = {n: (v[unit[0]:unit[0] + 1] if unit is not None else v) if n.endswith(".stats") else frames(v)
                    for n, v in f["cap"].items()}
        self.x, self.y = frames(f["x"]), frames(f["y"])
        self.B, self.H, self.T = self.x.shape

    def a0(self):
        m = self.mask
        w, b = self.p["init_conv.weight"], self.p["init_conv.bias"]
        x = self.x[:, None] * m
        ref = (F.conv2d(x, w, b)) * m
        A = (F.conv2d(x.abs(), w.abs(), b.abs())) * m
        k = 2 * U32 + (PN_A0_TF32 if self.mode == "tf32" else 0.0)
        return check(self.cap["a0"], ref, A, k, groups=False)

    def conv7(self, blk, xin):
        """blockN.raw: Conv2d 7x7 (padding 3) of the captured input times the mask, + bias: wgmma, K = 49 C (42-MMA fp32x3
        runs).  Uniformity over columns, rows, the conv's N tiles and the phase within its 128-pixel tile."""
        q = f"res_block.{blk}.block"
        w, b = self.p[f"{q}.0.weight"], self.p[f"{q}.0.bias"]
        ref, A, floor, Alin = _lin(F.conv2d, xin * self.mask, w, b, padding=3)
        k = kappa(self.mode, 49 * w.shape[1], run=42)
        return check(self.cap[f"block{blk[-1]}.raw"], ref, A, k, floor, Alin, ntile=pn_ntile(self.C, self.mode, "c7"),
                     period=TC_TILE)

    def act1(self):
        """block1.act = Mish(GN(raw1)) * mask (k_gn_act; tf32 handles round it to tf32 rna)"""
        q = "res_block.block1.block.1"
        raw = self.cap["block1.raw"]
        h, hA = pn_gn_mish(raw, self.cap["block1.stats"], self.p[f"{q}.weight"], self.p[f"{q}.bias"],
                           pn_inv_count(self.C, self.H, self.T))
        ref, A = h * self.mask, hA * self.mask
        if self.mode == "tf32":
            ref = round_tf32_rna(ref.float()).double()
        k = IN_GLU_ROUNDINGS * U32 + EPS_NL + (2 ** -10 if self.mode == "tf32" else 0.0)
        valid = self.mask.expand_as(ref)
        return check(self.cap["block1.act"], ref, A, k, groups=self.mode != "tf32", min_group=RB_MIN_VALID, valid=valid)

    def res(self):
        """res = (res_conv(a0 * mask) + Mish(GN(raw2)) * mask) * mask: the EPI_RES 1x1 (K = C) and its fp32 GN + Mish term"""
        q = "res_block.block2.block.1"
        h, hA = pn_gn_mish(self.cap["block2.raw"], self.cap["block2.stats"], self.p[f"{q}.weight"], self.p[f"{q}.bias"],
                           pn_inv_count(self.C, self.H, self.T))
        m = self.mask
        r, Ar, floor, Alin = _lin(F.conv2d, self.cap["a0"] * m, self.p["res_block.res.weight"], self.p["res_block.res.bias"])
        ref, A, Alin = (r + h * m) * m, (Ar + hA * m) * m, (Alin + hA * m) * m
        k = kappa(self.mode, self.C, nl=True)
        return check(self.cap["res"], ref, A, k, floor, Alin, ntile=pn_ntile(self.C, self.mode, "pw"))

    def out(self):
        """the call's output: final_conv(res) + bias, an fp32 FFMA chain of C terms from 0, then the bias add"""
        w, b = self.p["final_conv.weight"], self.p["final_conv.bias"]
        ref, A, floor, Alin = _lin(F.conv2d, self.cap["res"], w, b)
        return check(self.y[:, None], ref, A, kappa("fp32", self.C + 1), floor, Alin)

    def run(self):
        """-> rows (name, elem, unif, where) per judged unit (the call, or each utterance: its name carries b and L_b);
        raises on a captured name this replay does not know.  self.nonfinite lists judged captures holding a NaN / Inf."""
        want = ["a0", "block1.raw", "block1.stats", "block1.act", "block2.raw", "block2.stats", "res"]
        assert self.names == want, f"PostNet captures {self.names}, the replay knows {want}"
        rows, self.nonfinite = [], []
        for unit in self.units:
            self.select(unit)
            self.nonfinite += [n + self.tag for n, v in self.cap.items() if not bool(torch.isfinite(v).all())]
            if not bool(torch.isfinite(self.y).all()):
                self.nonfinite.append("out" + self.tag)
            r = [("a0",) + self.a0(),
                 ("block1.raw",) + self.conv7("block1", self.cap["a0"]),
                 ("block1.stats",) + pn_stats(self.cap["block1.raw"], self.cap["block1.stats"]),
                 ("block1.act",) + self.act1(),
                 ("block2.raw",) + self.conv7("block2", self.cap["block1.act"]),
                 ("block2.stats",) + pn_stats(self.cap["block2.raw"], self.cap["block2.stats"]),
                 ("res",) + self.res(),
                 ("out",) + self.out()]
            rows += [(n + self.tag,) + tuple(v) for n, *v in r]
        return rows
