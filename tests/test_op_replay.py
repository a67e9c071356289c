"""Self-tests of the op-isolation checker (tests/op_replay.py), CPU only.

A 3x3 conv over an image three 128-pixel tiles wide (W = 260: two full tiles and a ragged one of 4 columns) is emulated in
each tensor-core mode with the rounding primitives of oracle/precision_model.py.  The clean emulation must pass; each
seeded defect - the kinds of mistake a tiled wgmma conv makes at its tile edges - must fail.  The same holds for the 1-D
checks the vocoder uses: a dilated Conv1d over three 128-sample strips in tf32, and the transposed conv's overlap-add fold."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2
from op_replay import (FIRST_CONV_TILE, FLOOR_PER_W, R_UNIFORM, TC_TILE, PostNetReplay, _gn_mish, check, crop_utterance,
                       ct_fold, ctx_replay, kappa, passes, pn_inv_count, rb_act, rb_conv, rb_stats)
from oracle import gradtts_oracle as O
from oracle.precision_model import fp32x3_product, round_bf16, round_tf32_rna, trunc_tf32

B, CIN, COUT, H, W = 1, 64, 128, 6, 260
SEAM = 128                                  # first column of tile 1
MODES = ["tf32", "bf16", "fp32x3"]


@pytest.fixture(scope="module")
def conv():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, CIN, H, W, generator=g)
    w = (torch.rand(COUT, CIN, 3, 3, generator=g) * 2 - 1) / (CIN * 9) ** 0.5
    b = (torch.rand(COUT, generator=g) * 2 - 1) / (CIN * 9) ** 0.5
    d = torch.float64
    ref = F.conv2d(x.to(d), w.to(d), b.to(d), padding=1)
    A = F.conv2d(x.abs().to(d), w.abs().to(d), b.abs().to(d), padding=1)
    return x, w, b, ref, A


def emulate(x, w, b, mode, padding=1):
    """The conv with the mode's operand rounding (precision_model.py), products summed in float64, stored as fp32."""
    if mode == "fp32x3":
        return fp32x3_product(F.conv2d, x, w, 1, padding).double() + b.double()[None, :, None, None]
    if mode == "tf32":
        xq, wq = trunc_tf32(x), round_tf32_rna(w)
    else:
        xq, wq = round_bf16(x), round_bf16(w)
    return F.conv2d(xq.double(), wq.double(), b.double(), padding=padding).float().double()


def only_tap(w, r, s, ci=slice(None)):
    t = torch.zeros_like(w)
    t[:, ci, r, s] = w[:, ci, r, s]
    return t


def defect(name, x, w, b, mode):
    y = emulate(x, w, b, mode)
    if name == "a_dropped_tap":             # one of K = 576 terms (tap r=1, s=0 of input channel 0) lost in column 128
        y[..., SEAM] -= emulate(x, only_tap(w, 1, 0, slice(0, 1)), b * 0, mode)[..., SEAM]
    elif name == "b_zero_halo_at_seam":     # tile 1 reads its left halo (column 127) as zero
        xz = x.clone()
        xz[..., SEAM - 1] = 0
        y[..., SEAM] = emulate(xz, w, b, mode)[..., SEAM]
    elif name == "c_stale_left_padding":    # tile 0's left padding column keeps a value of another tile (column 255)
        xs = torch.zeros(B, CIN, H, 3)
        xs[..., 0] = x[..., 255]
        y[..., 0] += emulate(xs, only_tap(w, 0, 0) + only_tap(w, 1, 0) + only_tap(w, 2, 0), b * 0, mode,
                             padding=(1, 0))[..., 0]
    elif name == "d_no_correction_ntile1":  # fp32x3: N tile 1 (channels 64..127) runs the tf32 main MMAs only
        y[:, 64:] = emulate(x, w, b, "tf32")[:, 64:]
    elif name == "e_missing_bottom_halo":   # output row H-2 misses its bottom halo row (input row H-1)
        xz = x.clone()
        xz[:, :, H - 1] = 0
        y[:, :, H - 2] = emulate(xz, w, b, mode)[:, :, H - 2]
    return y


def _judge(y, ref, A, mode, w):
    floor = FLOOR_PER_W * w.abs().flatten(1).sum(1).max().item()
    return check(y, ref, A, kappa(mode, 9 * CIN), floor)


@pytest.mark.parametrize("mode", MODES)
def test_clean_emulation_passes(conv, mode):
    x, w, b, ref, A = conv
    elem, unif, where = _judge(emulate(x, w, b, mode), ref, A, mode, w)
    print(f"{mode} clean: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
    assert passes(elem, unif), (elem, unif, where)


DEFECTS = ["a_dropped_tap", "b_zero_halo_at_seam", "e_missing_bottom_halo"]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", DEFECTS)
def test_seeded_defect_fails(conv, mode, name):
    x, w, b, ref, A = conv
    y = defect(name, x, w, b, mode)
    elem, unif, where = _judge(y, ref, A, mode, w)
    print(f"{mode} {name}: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert not passes(elem, unif)
    assert unif > R_UNIFORM, "the uniformity check alone must see a local defect"


@pytest.mark.parametrize("mode", MODES)
def test_stale_padding_fails_check1(conv, mode):
    """The image's border columns are judged by the per-element bound alone (op_replay.R_UNIFORM): a stale value in the
    left padding column must exceed it many times over."""
    x, w, b, ref, A = conv
    elem, unif, where = _judge(defect("c_stale_left_padding", x, w, b, mode), ref, A, mode, w)
    print(f"{mode} c_stale_left_padding: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert elem > 10 and not passes(elem, unif)


def test_missing_fp32x3_correction_in_one_ntile_fails(conv):
    x, w, b, ref, A = conv
    y = defect("d_no_correction_ntile1", x, w, b, "fp32x3")
    elem, unif, where = _judge(y, ref, A, "fp32x3", w)
    print(f"fp32x3 d_no_correction_ntile1: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert unif > R_UNIFORM and where.startswith("ntile")
    assert not passes(elem, unif)


def test_global_rel_l2_misses_what_uniformity_sees(conv):
    """Defect (a) in tf32: one dropped tap in one column.  The whole-tensor rel-L2 the stagewise tests use stays far inside
    their tf32 bound (4e-3); the per-column uniformity check does not."""
    x, w, b, ref, A = conv
    y = defect("a_dropped_tap", x, w, b, "tf32")
    g = rel_l2(y, ref)
    elem, unif, where = _judge(y, ref, A, "tf32", w)
    print(f"tf32 dropped tap at column {SEAM}: global rel-L2 {g:.2e} (bound 4e-3: passes) | "
          f"uniformity max/median {unif:.1f} at {where} (bound {R_UNIFORM}: fails)")
    assert g < 4e-3
    assert unif > R_UNIFORM and where == f"col[{SEAM}]"


# ---- the 1-D checker: a dilated Conv1d (K = 11, d = 5, pad 25) over three 128-sample tiles, the last one ragged -----------
L1, CIN1, COUT1, K1, D1 = 300, 64, 128, 11, 5
PAD1 = (K1 - 1) * D1 // 2
NT1 = 32                                    # N-tile width judged here (the vocoder's last stage runs 32-wide tiles)
KAP1 = kappa("tf32", CIN1 * K1, extra=2 ** -24)          # tf32 MMAs + the epilogue's fp32 bias add


@pytest.fixture(scope="module")
def conv1():
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, CIN1, L1, generator=g)
    w = (torch.rand(COUT1, CIN1, K1, generator=g) * 2 - 1) / (CIN1 * K1) ** 0.5
    b = (torch.rand(COUT1, generator=g) * 2 - 1) / (CIN1 * K1) ** 0.5
    d = torch.float64
    ref = F.conv1d(x.to(d), w.to(d), b.to(d), padding=PAD1, dilation=D1)
    Alin = F.conv1d(x.abs().to(d), w.abs().to(d), None, padding=PAD1, dilation=D1)
    return x, w, b, ref, Alin + b.abs().to(d)[None, :, None], Alin


def emulate1d(x, w, b):
    """k_conv_tc<G_C1K11> in tf32: activations truncated, weights rounded to nearest (away), float64 sums, fp32 store"""
    return F.conv1d(trunc_tf32(x).double(), round_tf32_rna(w).double(), b.double(), padding=PAD1, dilation=D1).float().double()


def defect1d(name, x, w, b):
    y = emulate1d(x, w, b)
    if name == "a_dropped_tap":             # one of K = 704 terms (tap 0 of input channel 0) lost at sample 128
        t = torch.zeros_like(w)
        t[:, 0, 0] = w[:, 0, 0]
        y[..., SEAM] -= emulate1d(x, t, b * 0)[..., SEAM]
    elif name == "b_zero_left_halo":        # tile 1 reads its left halo (the 25 samples before 128) as zero
        xz = x.clone()
        xz[..., SEAM - PAD1:SEAM] = 0
        y[..., SEAM:2 * SEAM] = emulate1d(xz, w, b)[..., SEAM:2 * SEAM]
    elif name == "c_stale_right_padding":   # the ragged tile's first padding column keeps a value of another tile
        xs = F.pad(x, (0, 1))
        xs[..., L1] = x[..., 45]
        y[..., 2 * SEAM:] = emulate1d(xs, w, b)[..., 2 * SEAM:L1]
    elif name == "d_ntile_missing_k_stage":  # N block 1 (channels 32..63) misses the last K stage (input channels 56..63)
        xk = x.clone()
        xk[:, CIN1 - 8:] = 0
        y[:, NT1:2 * NT1] = emulate1d(xk, w, b)[:, NT1:2 * NT1]
    return y


def _judge1d(y, conv1):
    x, w, b, ref, A, Alin = conv1
    floor = FLOOR_PER_W * w.abs().flatten(1).sum(1).max().item()
    return check(y, ref, A, KAP1, floor, Alin, pad=PAD1, ntile=NT1)


def test_conv1d_clean_emulation_passes(conv1):
    x, w, b = conv1[:3]
    elem, unif, where = _judge1d(emulate1d(x, w, b), conv1)
    print(f"conv1d tf32 clean: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
    assert passes(elem, unif), (elem, unif, where)


@pytest.mark.parametrize("name", ["a_dropped_tap", "b_zero_left_halo", "c_stale_right_padding", "d_ntile_missing_k_stage"])
def test_conv1d_seeded_defect_fails(conv1, name):
    x, w, b = conv1[:3]
    elem, unif, where = _judge1d(defect1d(name, x, w, b), conv1)
    print(f"conv1d tf32 {name}: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert not passes(elem, unif)
    if name == "c_stale_right_padding":     # only samples within pad of the end see it: check 1 alone must catch it
        assert elem > 1.0
    elif name == "d_ntile_missing_k_stage":
        assert unif > R_UNIFORM and where.startswith("ntile")
    else:
        assert unif > R_UNIFORM, "the uniformity check alone must see a local defect"


def test_conv1d_global_rel_l2_misses_what_uniformity_sees(conv1):
    """One dropped tap term at sample 128: the whole-waveform-style rel-L2 stays under the vocoder's 5e-3 bound, while the
    per-sample uniformity check fails."""
    x, w, b, ref = conv1[:4]
    y = defect1d("a_dropped_tap", x, w, b)
    g = rel_l2(y, ref)
    elem, unif, where = _judge1d(y, conv1)
    print(f"conv1d tf32 dropped tap at sample {SEAM}: global rel-L2 {g:.2e} (bound 5e-3: passes) | "
          f"uniformity max/median {unif:.1f} at {where} (bound {R_UNIFORM}: fails)")
    assert g < 5e-3
    # tile 1 is the only full interior tile here, so its phase 0 group is sample 128 too
    assert unif > R_UNIFORM and where in (f"sample[{SEAM}]", "phase[0]")


# ---- the transposed conv's fold (k_voc_ct_fold) against torch's ConvTranspose1d -------------------------------------------
U, CO_T, LIN_T = 4, 32, 40


@pytest.fixture(scope="module")
def convt():
    g = torch.Generator().manual_seed(13)
    x = torch.randn(1, CIN1, LIN_T, generator=g)
    w = torch.randn(CIN1, CO_T, 2 * U, generator=g) / (CIN1 * 2) ** 0.5
    b = torch.randn(CO_T, generator=g) * 0.02
    # the GEMM to 2u*co channels (channel t*co + c) in tf32, stored fp32
    gw = w.permute(2, 1, 0).reshape(2 * U * CO_T, CIN1, 1)
    z = F.conv1d(trunc_tf32(x).double(), round_tf32_rna(gw).double()).float()
    d = torch.float64
    ref = F.conv_transpose1d(x.to(d), w.to(d), b.to(d), stride=U, padding=U // 2)
    Alin = F.conv_transpose1d(x.abs().to(d), w.abs().to(d), None, stride=U, padding=U // 2)
    return z, b, ref, Alin + b.abs().to(d)[None, :, None], Alin, w


def _judge_fold(y, convt):
    z, b, ref, A, Alin, w = convt
    return check(y, ref, A, kappa("tf32", CIN1, extra=2 * 2 ** -24), 0.0, Alin, pad=U // 2, ntile=CO_T)


def test_fold_clean_passes(convt):
    z, b = convt[:2]
    elem, unif, where = _judge_fold(ct_fold(z, b, U), convt)
    print(f"fold clean: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
    assert passes(elem, unif), (elem, unif, where)


def test_fold_wrong_tap_index_fails(convt):
    """At output phase o % u == 1 the second tap is read from input i1 instead of i1 - 1."""
    z, b = convt[:2]
    y = ct_fold(z, b, U)
    zz = z.view(1, 2 * U, CO_T, LIN_T).permute(0, 2, 1, 3)
    p = U // 2
    for o in range(1, LIN_T * U, U):
        i1, t1 = (o + p) // U, (o + p) % U
        if 1 <= i1 < LIN_T:
            y[:, :, o] += zz[:, :, t1 + U, i1] - zz[:, :, t1 + U, i1 - 1]
    elem, unif, where = _judge_fold(y, convt)
    print(f"fold wrong tap index: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert elem > 1.0 and unif > R_UNIFORM and not passes(elem, unif)


# ---- one RefBlock stage (DiffVC's conditioning branch): tf32 3x3 conv + InstanceNorm + GLU + time bias, and the first conv ---
# Tr = 300 (wgmma tiles 128 | 128 | 44, k_first_conv tiles 256 | 44) with a mask edge at frame 280.  The emulation follows
# the kernels: k_conv_tc<G_C3> on tf32 operands (the activation is already in tf32 form), k_in_glu's fp32 arithmetic with
# the fast sigmoid and an rna tf32 output, zero past the mask; k_first_conv as an fp32 conv of the one-channel xt_ref.
RB_H, RB_TR, RB_LEN, RB_CIN, RB_COUT = 8, 300, 280, 32, 64


@pytest.fixture(scope="module")
def rb_stage():
    g = torch.Generator().manual_seed(17)
    mask = (torch.arange(RB_TR) < RB_LEN).double()[None]
    x = round_tf32_rna(torch.randn(1, RB_CIN, RB_H, RB_TR, generator=g)).double() * mask[:, None, None, :]
    w = (torch.rand(RB_COUT, RB_CIN, 3, 3, generator=g) * 2 - 1) / (RB_CIN * 9) ** 0.5
    b = (torch.rand(RB_COUT, generator=g) * 2 - 1) / (RB_CIN * 9) ** 0.5
    gamma = 1 + 0.1 * torch.randn(RB_COUT, generator=g)
    beta = 0.1 * torch.randn(RB_COUT, generator=g)
    tb = 0.5 * torch.randn(RB_COUT // 2, generator=g)
    xt = torch.randn(1, 1, RB_H, RB_TR, generator=g).double() * mask[:, None, None, :]
    w1 = (torch.rand(RB_COUT, 1, 3, 3, generator=g) * 2 - 1) / 3
    b1 = (torch.rand(RB_COUT, generator=g) * 2 - 1) / 3
    d = torch.float64
    return dict(mask=mask, x=x, w=w.to(d), b=b.to(d), gamma=gamma.to(d), beta=beta.to(d), tb=tb.float().double(),
                xt=xt, w1=w1.to(d), b1=b1.to(d))


def rb_emulate_conv(s, x=None, w_only=None):
    x = s["x"] if x is None else x
    w = round_tf32_rna(s["w"].float()).double() if w_only is None else w_only
    return F.conv2d(x, w, s["b"] if w_only is None else None, padding=1).float().double()


def rb_emulate_in_glu(raw, s, cols=None, swap=False, tb_gate=False):
    """k_in_glu in fp32: statistics over `cols` (default: every column), mean / rstd * gamma rounded to fp32"""
    C = raw.shape[1]
    r = raw if cols is None else raw[..., cols]
    n = r.shape[2] * r.shape[3]
    m = r.sum((2, 3)) / n
    var = ((r * r).sum((2, 3)) / n - m * m).clamp_min(0)
    mean = m.float()[:, :, None, None]
    scale = ((1.0 / torch.sqrt(var + 1e-5)).float() * s["gamma"].float()[None])[:, :, None, None]
    xn = (raw.float() - mean) * scale + s["beta"].float()[None, :, None, None]
    a, gt = (xn[:, C // 2:], xn[:, :C // 2]) if swap else (xn[:, :C // 2], xn[:, C // 2:])
    tb = s["tb"].float()[None, :, None, None]
    y = a * torch.sigmoid(gt + tb) if tb_gate else a * torch.sigmoid(gt) + tb
    return round_tf32_rna(y).double() * s["mask"][:, None, None, :]


def rb_judge_conv(s, raw):
    return rb_conv(s["x"], s["mask"], s["w"], s["b"], raw, "tf32")


def rb_judge_act(s, raw, act):
    return rb_act(raw, s["gamma"], s["beta"], s["tb"], s["mask"], act, "tf32")


def rb_emulate_first(s, xt=None):
    return F.conv2d(s["xt"] if xt is None else xt, s["w1"], s["b1"], padding=1).float().double()


def test_refblock_clean_emulation_passes(rb_stage):
    s = rb_stage
    raw = rb_emulate_conv(s)
    rows = {"raw": rb_judge_conv(s, raw), "act": rb_judge_act(s, raw, rb_emulate_in_glu(raw, s)),
            "first": rb_conv(s["xt"], s["mask"], s["w1"], s["b1"], rb_emulate_first(s), "tf32", first=True)}
    for k, (elem, unif, where) in rows.items():
        print(f"refblock clean {k}: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
        assert passes(elem, unif), (k, elem, unif, where)


def test_refblock_dropped_tap_at_seam_fails(rb_stage):
    """one of K = 288 terms (tap r=1, s=0 of input channel 0) lost in column 128"""
    s = rb_stage
    raw = rb_emulate_conv(s)
    t = torch.zeros_like(s["w"])
    t[:, 0, 1, 0] = round_tf32_rna(s["w"][:, 0, 1, 0].float()).double()
    raw[..., TC_TILE] -= rb_emulate_conv(s, w_only=t)[..., TC_TILE]
    elem, unif, where = rb_judge_conv(s, raw)
    print(f"refblock dropped tap: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert unif > R_UNIFORM and where == f"col[{TC_TILE}]" and not passes(elem, unif)


@pytest.mark.parametrize("name", ["stats_over_valid_columns", "glu_halves_swapped", "time_bias_on_gate", "nonzero_past_mask"])
def test_refblock_in_glu_defect_fails(rb_stage, name):
    s = rb_stage
    raw = rb_emulate_conv(s)
    if name == "stats_over_valid_columns":      # InstanceNorm over the valid frames only: not what F.instance_norm does
        act = rb_emulate_in_glu(raw, s, cols=slice(0, RB_LEN))
    elif name == "glu_halves_swapped":
        act = rb_emulate_in_glu(raw, s, swap=True)
    elif name == "time_bias_on_gate":
        act = rb_emulate_in_glu(raw, s, tb_gate=True)
    else:                                       # the first masked frame keeps its IN + GLU value
        act = rb_emulate_in_glu(raw, s)
        full = rb_emulate_in_glu(raw, dict(s, mask=torch.ones_like(s["mask"])))
        act[..., RB_LEN] = full[..., RB_LEN]
    elem, unif, where = rb_judge_act(s, raw, act)
    print(f"refblock {name}: |err|/(kappa A) max {elem:.3g}")
    assert elem > 10 and not passes(elem, unif)


def test_refblock_stale_halo_at_first_conv_seam_fails(rb_stage):
    """k_first_conv's second 256-frame tile reads its left halo (frame 255) from a stale shared-memory slot (frame 0)"""
    s = rb_stage
    raw = rb_emulate_first(s)
    xs = s["xt"].clone()
    xs[..., FIRST_CONV_TILE - 1] = xs[..., 0]
    raw[..., FIRST_CONV_TILE] = rb_emulate_first(s, xs)[..., FIRST_CONV_TILE]
    elem, unif, where = rb_conv(s["xt"], s["mask"], s["w1"], s["b1"], raw, "tf32", first=True)
    print(f"refblock stale first-conv halo: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert elem > 10 and unif > R_UNIFORM and not passes(elem, unif)


# ---- ragged batches: two utterances of different widths on one dense image, each judged on its own columns ----------------
# A ragged call computes utterance b on its own W_b columns of the dense image (W_b = T_b >> level) and the checker crops
# every capture to [b:b+1, ..., :W_b] (op_replay.Replay with lengths).  Utterance 0 fills the dense width (260: tiles
# 128 | 128 | 4), utterance 1 ends 4 columns past a tile seam (132); past W_b the dense image holds stale values.
RW = (W, 132)


@pytest.fixture(scope="module")
def ragged():
    g = torch.Generator().manual_seed(19)
    x = torch.randn(2, CIN, H, W, generator=g)
    w = (torch.rand(COUT, CIN, 3, 3, generator=g) * 2 - 1) / (CIN * 9) ** 0.5
    b = (torch.rand(COUT, generator=g) * 2 - 1) / (CIN * 9) ** 0.5
    return x, w, b


def _per_utterance(y, judge):
    """judge(b, y cropped to utterance b) -> (elem, unif, where) for each utterance"""
    return [judge(u, crop_utterance(y, u, RW[u])) for u in range(2)]


def _judge_conv_utt(x, w, b, mode):
    def judge(u, got):
        xu = crop_utterance(x, u, RW[u]).double()
        ref, A = F.conv2d(xu, w.double(), b.double(), padding=1), F.conv2d(xu.abs(), w.abs().double(), b.abs().double(), padding=1)
        return _judge(got, ref, A, mode, w)
    return judge


def ragged_conv(x, w, b, mode, stale_edge=False):
    """the ragged 3x3 conv: each utterance's output from its own columns, zero padding at its edge; NaN past it.
    stale_edge: utterance 1's last column reads its right halo (dense column W_1) from the image instead of as zero."""
    y = torch.full((2, COUT, H, W), float("nan"), dtype=torch.float64)
    for u in range(2):
        y[u:u + 1, ..., :RW[u]] = emulate(crop_utterance(x, u, RW[u]), w, b, mode)
    if stale_edge:
        e = RW[1] - 1
        y[1:2, ..., e] = emulate(crop_utterance(x, 1, RW[1] + 1), w, b, mode)[..., e]
    return y


@pytest.mark.parametrize("mode", MODES)
def test_ragged_conv_clean_passes(ragged, mode):
    x, w, b = ragged
    for u, (elem, unif, where) in enumerate(_per_utterance(ragged_conv(x, w, b, mode), _judge_conv_utt(x, w, b, mode))):
        print(f"{mode} ragged conv clean b={u} W={RW[u]}: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
        assert passes(elem, unif), (u, elem, unif, where)


@pytest.mark.parametrize("mode", MODES)
def test_ragged_stale_edge_column_fails(ragged, mode):
    """(a) utterance 1's edge column reads the next column of the dense image instead of zero.  The column is the
    utterance's image border, which check 2 leaves out (op_replay.R_UNIFORM): check 1 alone catches it, by 121x (tf32),
    23x (bf16) and 1.2e4x (fp32x3), while the uniformity ratio stays ~1.1."""
    x, w, b = ragged
    rows = _per_utterance(ragged_conv(x, w, b, mode, stale_edge=True), _judge_conv_utt(x, w, b, mode))
    elem, unif, where = rows[1]
    print(f"{mode} ragged stale edge column b=1 W={RW[1]}: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert passes(*rows[0][:2]) and elem > 10 and not passes(elem, unif)


# (b) GroupNorm + Mish of one Block (the captured raw conv output -> Mish(GN(raw)) * mask), as k_gn_act computes it: the
# group statistics over the utterance's own H x W_b pixels, mean and rstd * gamma rounded to fp32, the rest in fp32, the
# output stored as the mode stores it.  The defect divides the utterance's sums by the dense count C/G * H * W.
def ragged_gn_mish(raw, gamma, beta, mode, dense_count=False):
    y = torch.full_like(raw, float("nan"))
    for u in range(2):
        r = crop_utterance(raw, u, RW[u]).contiguous()
        B_, C_, H_, W_ = r.shape
        g = r.view(1, O.GROUPS, -1)
        n = (C_ // O.GROUPS) * H_ * (W if dense_count else W_)
        mean = g.sum(-1) / n
        var = ((g * g).sum(-1) / n - mean * mean).clamp_min(0.0)
        cpg = C_ // O.GROUPS
        mean_f = mean.float().repeat_interleave(cpg, 1)[:, :, None, None]
        scale = ((1.0 / torch.sqrt(var + 1e-5)).float().repeat_interleave(cpg, 1) * gamma.float()[None])[:, :, None, None]
        h = F.mish((r.float() - mean_f) * scale + beta.float()[None, :, None, None])
        y[u:u + 1, ..., :RW[u]] = (round_bf16(h) if mode == "bf16" else h).double()
    return y


@pytest.fixture(scope="module")
def ragged_gn(ragged):
    x, w, b = ragged
    g = torch.Generator().manual_seed(23)
    raw = torch.cat([emulate(crop_utterance(x, u, W), w, b, "tf32") for u in range(2)], 0)
    gamma, beta = 1 + 0.1 * torch.randn(COUT, generator=g), 0.1 * torch.randn(COUT, generator=g)
    return raw, gamma, beta


def _judge_gn_utt(raw, gamma, beta, mode):
    p = {"blk.block.1.weight": gamma.double(), "blk.block.1.bias": beta.double()}

    def judge(u, got):
        ref, A = _gn_mish(p, "blk", crop_utterance(raw, u, RW[u]).contiguous())
        return check(got, ref, A, kappa(mode, 1, tc=False, nl=True, store_bf16=mode == "bf16"))
    return judge


@pytest.mark.parametrize("mode", MODES)
def test_ragged_group_norm_clean_passes(ragged_gn, mode):
    raw, gamma, beta = ragged_gn
    rows = _per_utterance(ragged_gn_mish(raw, gamma, beta, mode), _judge_gn_utt(raw, gamma, beta, mode))
    for u, (elem, unif, where) in enumerate(rows):
        print(f"{mode} ragged GN clean b={u} W={RW[u]}: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
        assert passes(elem, unif), (u, elem, unif, where)


@pytest.mark.parametrize("mode", MODES)
def test_ragged_group_norm_dense_count_fails(ragged_gn, mode):
    """(b) the GroupNorm count of utterance 1 from the dense W instead of W_b: its mean and variance shrink by ~W_b / W,
    which check 1 sees at every element: it fails by 9.9e4x (tf32, fp32x3) and 195x (bf16)."""
    raw, gamma, beta = ragged_gn
    rows = _per_utterance(ragged_gn_mish(raw, gamma, beta, mode, dense_count=True), _judge_gn_utt(raw, gamma, beta, mode))
    elem, unif, where = rows[1]
    print(f"{mode} ragged GN dense count b=1 W={RW[1]}: |err|/(kappa A) max {elem:.3g}, uniformity {unif:.3g} at {where}")
    assert passes(*rows[0][:2]) and elem > 10 and not passes(elem, unif)


# (c) LinearAttention's context over an utterance's own H x W_b pixels (k_attn_ctx): k | v projected with the mode's operand
# rounding and stored fp32, softmax over the pixels in fp32, P and V rounded for the context product (tf32 datapath in the
# tf32 and bf16 modes), the result stored fp32.  The defect lets the padded pixels of the dense image into the softmax as
# k = 0, v = 0: the numerators keep their value, the denominators grow by n_pad * exp(-max k).  It is visible only where
# exp(-max k) is not negligible against the sum over the valid pixels, i.e. while k stays O(1): here x ~ N(0.5, 1), so k
# is O(1) and v has a mean that the context keeps (for zero-mean v the context is a cancelling sum and the defect smaller).
ATT_C, ATT_H = 64, 4


@pytest.fixture(scope="module")
def ragged_attn():
    g = torch.Generator().manual_seed(29)
    x = torch.randn(2, ATT_C, ATT_H, W, generator=g) + 0.5
    wqkv = torch.randn(3 * O.HEADS * 32, ATT_C, 1, 1, generator=g) / ATT_C ** 0.5
    return x, wqkv


def ragged_ctx(x, wqkv, mode, pad_in_softmax=False):
    out = []
    for u in range(2):
        xu = crop_utterance(x, u, W if pad_in_softmax else RW[u]).clone()
        if mode == "fp32x3":
            kv = fp32x3_product(F.conv2d, xu, wqkv, 1, 0)
        else:
            xq, wq = (trunc_tf32(xu), round_tf32_rna(wqkv)) if mode == "tf32" else (round_bf16(xu), round_bf16(wqkv))
            kv = F.conv2d(xq.double(), wq.double())
        kv = kv.float().reshape(1, 3, O.HEADS, 32, -1)
        k, v = kv[:, 1], kv[:, 2]
        if pad_in_softmax:                  # the pixels at columns >= W_b of every row enter as k = 0, v = 0
            k, v = k.clone(), v.clone()
            k.view(1, O.HEADS, 32, ATT_H, W)[..., RW[u]:] = 0
            v.view(1, O.HEADS, 32, ATT_H, W)[..., RW[u]:] = 0
        pr = k.softmax(-1)
        if mode != "fp32x3":
            pr, v = round_tf32_rna(pr), round_tf32_rna(v)
        out.append(torch.einsum("bhdn,bhen->bhde", pr.double(), v.double()).float().double())
    return out


def _judge_ctx(x, wqkv, mode, got):
    rows = []
    for u in range(2):
        ref, A, k = ctx_replay(crop_utterance(x, u, RW[u]).double(), wqkv.double(), mode)
        rows.append(check(got[u], ref, A, k, groups=False))
    return rows


@pytest.mark.parametrize("mode", MODES)
def test_ragged_attention_context_clean_passes(ragged_attn, mode):
    x, wqkv = ragged_attn
    for u, (elem, unif, where) in enumerate(_judge_ctx(x, wqkv, mode, ragged_ctx(x, wqkv, mode))):
        print(f"{mode} ragged ctx clean b={u} W={RW[u]}: |err|/(kappa A) max {elem:.3f}")
        assert passes(elem, unif), (u, elem)


@pytest.mark.parametrize("mode", MODES)
def test_ragged_attention_padded_pixels_in_softmax_fail(ragged_attn, mode):
    """(c) utterance 1's context with its padded pixels (columns 132..259 of each of the 4 rows: 512 pixels, against
    528 valid ones) in the softmax as k = 0, v = 0.  It fails check 1 by 12.8x (tf32), 4.47x (bf16) and 2.5e3x
    (fp32x3).  The margin shrinks as the keys grow against 0: shifting every k by +c scales the padded pixels' share of
    the denominators by exp(-c), and at c ~ 2.5 bf16's bound (~ 2^-7) no longer separates the defect from rounding
    (float64 estimate: 2.75x at c = 1, 1.35x at c = 2, 0.56x at c = 3).  There the bitwise per-op comparison of a ragged
    call with its B = 1 calls in tf32 and bf16 (test_ragged_decoder_gpu.py) still sees it; fp32x3's bound is ~500x
    tighter than bf16's."""
    x, wqkv = ragged_attn
    rows = _judge_ctx(x, wqkv, mode, ragged_ctx(x, wqkv, mode, pad_in_softmax=True))
    elem, unif, where = rows[1]
    print(f"{mode} ragged ctx padded pixels in softmax b=1 W={RW[1]}: |err|/(kappa A) max {elem:.3g}")
    assert passes(*rows[0][:2]) and elem > 2 and not passes(elem, unif)


# ---- a ragged RefBlock row: reference 0 on its own R = RB_LEN frames of the Tr = RB_TR image (RefBlockReplay crops every
# capture to [b:b+1, ..., :R_b], so its statistics and InstanceNorm normalise over H * R_b).  Past R the dense image holds the
# conv of the whole row (a stale, finite value).
def rb_ragged(s):
    """(raw of the reference's own call [.., :R], the dense image's raw, the stats k_chan_stats_ragged writes)"""
    R = RB_LEN
    x = s["x"][..., :R]
    raw = rb_emulate_conv(dict(s, x=x))
    dense = rb_emulate_conv(dict(s, x=s["x"] + (s["mask"] == 0)[:, None, None, :].double()))
    return raw, dense


def rb_ragged_in_glu(raw, s, n_cols):
    """k_in_glu_ragged on the reference's own columns, the InstanceNorm divisor H * n_cols"""
    C = raw.shape[1]
    n = raw.shape[2] * n_cols
    m = raw.sum((2, 3)) / n
    var = ((raw * raw).sum((2, 3)) / n - m * m).clamp_min(0)
    mean = m.float()[:, :, None, None]
    scale = ((1.0 / torch.sqrt(var + 1e-5)).float() * s["gamma"].float()[None])[:, :, None, None]
    xn = (raw.float() - mean) * scale + s["beta"].float()[None, :, None, None]
    y = xn[:, :C // 2] * torch.sigmoid(xn[:, C // 2:]) + s["tb"].float()[None, :, None, None]
    return round_tf32_rna(y).double()


def rb_judge_ragged(s, raw, stats, act):
    ones = torch.ones(1, raw.shape[-1], dtype=torch.float64)
    return {"stats": rb_stats(raw, stats, RB_TR), "act": rb_act(raw, s["gamma"], s["beta"], s["tb"], ones, act, "tf32")}


def _sums(raw):
    return torch.stack([raw.sum((2, 3)), (raw * raw).sum((2, 3))], -1)


def test_refblock_ragged_clean_passes(rb_stage):
    s = rb_stage
    raw, _ = rb_ragged(s)
    for k, (elem, unif, where) in rb_judge_ragged(s, raw, _sums(raw), rb_ragged_in_glu(raw, s, RB_LEN)).items():
        print(f"refblock ragged clean {k}: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
        assert passes(elem, unif), (k, elem, unif, where)


def test_refblock_ragged_divisor_from_tr_fails(rb_stage):
    """k_in_glu_ragged divides the reference's sums by H * Tr instead of H * R_b: the mean and variance shrink by R_b / Tr
    (280 / 300), which check 1 sees at nearly every element: act fails by ~27x."""
    s = rb_stage
    raw, _ = rb_ragged(s)
    rows = rb_judge_ragged(s, raw, _sums(raw), rb_ragged_in_glu(raw, s, RB_TR))
    elem, unif, _ = rows["act"]
    print(f"refblock ragged divisor H*Tr: act |err|/(kappa A) max {elem:.3g}")
    assert passes(*rows["stats"][:2]) and elem > 10 and not passes(elem, unif)


def test_refblock_ragged_stats_one_column_late_fails(rb_stage):
    """k_chan_stats_ragged sums column R_b (the dense image's value there) too: one column of H in H * R_b terms, an error of
    ~1 / R_b of the sums against a bound of rb_chain(Tr) * 2^-24 ~ 1e-6 of them; stats fail by ~3e4x."""
    s = rb_stage
    raw, dense = rb_ragged(s)
    stats = _sums(raw) + _sums(dense[..., RB_LEN:RB_LEN + 1])
    elem, unif, _ = rb_judge_ragged(s, raw, stats, rb_ragged_in_glu(raw, s, RB_LEN))["stats"]
    print(f"refblock ragged stats one column late: |err|/(kappa A) max {elem:.3g}")
    assert elem > 100 and not passes(elem, unif)


# ---- a ragged PostNet: dim 32 on an 8 x 40 grid, utterances of 40 and 13 frames, driven through PostNetReplay ----------------
# The emulation computes utterance b's own call on its L_b frames in fp32, with k_pn_init's and k_gn_act's tf32 (rna) stores
# on tf32 handles and the kernels' GroupNorm divisor; every capture past L_b is NaN, as a poisoned workspace leaves it.
PN_C, PN_H, PN_T, PN_LENS = 32, 8, 40, [40, 13]


class PostNetEmulation:
    """the engine surface PostNetReplay drives.  defect: "stale_third_zero_column" - utterance 1's block1 conv reads input
    column L_b + 2 (the third of the 7x7's zero columns) from the dense image; "gn_count_from_T" - utterance 1's GroupNorm
    divides by (C/8) H T instead of (C/8) H L_b."""

    def __init__(self, sd, tf32, defect=None):
        self.p, self.tf32, self.defect = {k: v.float() for k, v in sd.items()}, tf32, defect

    def debug_capture(self, on):
        pass

    def debug_names(self):
        return list(self.cap)

    def debug_read(self, name):
        return self.cap[name]

    def forward(self, x, mask, lengths):
        p, B, H, T = self.p, x.shape[0], x.shape[1], x.shape[2]
        rnd = round_tf32_rna if self.tf32 else (lambda v: v)
        big = {k: torch.full((B, PN_C, H, T), float("nan")) for k in ("a0", "block1.raw", "block1.act", "block2.raw", "res")}
        stats = {k: torch.zeros(B, 8, 2, dtype=torch.float64) for k in ("block1.stats", "block2.stats")}
        y = torch.zeros(B, H, T)
        for b, L in enumerate(lengths.tolist()):
            bad = b == 1
            a0_row = rnd(F.conv2d(torch.nan_to_num(x[b:b + 1, None], 1.0), p["init_conv.weight"], p["init_conv.bias"]))
            a0 = a0_row[..., :L]

            def block(i, inp):
                q = f"res_block.block{i}.block"
                w, bias = p[f"{q}.0.weight"], p[f"{q}.0.bias"]
                if i == 1 and bad and self.defect == "stale_third_zero_column":
                    inp = torch.cat([inp, torch.zeros_like(a0_row[..., :3])], -1)
                    inp[..., L + 2] = a0_row[..., L + 2]
                    raw = F.conv2d(F.pad(inp, (3, 0, 3, 3)), w, bias)
                else:
                    raw = F.conv2d(inp, w, bias, padding=3)
                g = raw.double().reshape(1, 8, -1)
                st = torch.stack([g.sum(-1), (g * g).sum(-1)], -1)
                inv = pn_inv_count(PN_C, H, T if bad and self.defect == "gn_count_from_T" else L)
                mean = st[..., 0] * inv
                var = (st[..., 1] * inv - mean * mean).clamp_min(0.0)
                cpg = PN_C // 8
                mean_f = mean.float().repeat_interleave(cpg, 1)[:, :, None, None]
                sc = ((1.0 / torch.sqrt(var + 1e-5)).float().repeat_interleave(cpg, 1) * p[f"{q}.1.weight"][None])[:, :, None, None]
                return raw, st, F.mish((raw - mean_f) * sc + p[f"{q}.1.bias"][None, :, None, None])
            r1, s1, h1 = block(1, a0)
            h1 = rnd(h1)
            r2, s2, h2 = block(2, h1)
            res = F.conv2d(a0, p["res_block.res.weight"], p["res_block.res.bias"]) + h2
            for k, v in (("a0", a0), ("block1.raw", r1), ("block1.act", h1), ("block2.raw", r2), ("res", res)):
                big[k][b:b + 1, ..., :L] = v
            stats["block1.stats"][b], stats["block2.stats"][b] = s1[0], s2[0]
            y[b, :, :L] = F.conv2d(res, p["final_conv.weight"], p["final_conv.bias"])[0, 0]
        names = ("a0", "block1.raw", "block1.stats", "block1.act", "block2.raw", "block2.stats", "res")
        self.cap = {k: big.get(k, stats.get(k)) for k in names}
        return y


def _pn_rows(precision, defect=None):
    from speech_backbones_b200.spec import synthetic_postnet_state_dict
    sd = synthetic_postnet_state_dict(PN_C, 29)
    x = torch.randn(len(PN_LENS), PN_H, PN_T, generator=torch.Generator().manual_seed(31))
    for b, L in enumerate(PN_LENS):
        x[b, :, L:] = float("nan")
    rp = PostNetReplay(PostNetEmulation(sd, precision == "tf32", defect), sd, precision, x,
                       torch.ones(len(PN_LENS), 1, PN_T), lengths=PN_LENS, dev="cpu")
    return {r[0]: r[1:] for r in rp.run()}, rp.nonfinite


@pytest.mark.parametrize("precision", ["tf32", "fp32x3"])
def test_postnet_ragged_clean_passes(precision):
    rows, nonfinite = _pn_rows(precision)
    assert not nonfinite
    for k, (elem, unif, where) in rows.items():
        print(f"postnet {precision} clean {k}: |err|/(kappa A) max {elem:.3f}, uniformity {unif:.2f} at {where}")
        assert passes(elem, unif), (k, elem, unif, where)


@pytest.mark.parametrize("precision", ["tf32", "fp32x3"])
def test_postnet_stale_third_zero_column_fails(precision):
    """utterance 1's 7x7 conv reads input column L_b + 2 from the image instead of as zero: only output column L_b - 1 (the
    utterance's border, which check 2 leaves out) sees it, through one kernel column; check 1 fails it by ~40x (tf32) and
    ~5e3x (fp32x3), and utterance 0 still passes."""
    rows, _ = _pn_rows(precision, "stale_third_zero_column")
    elem, unif, _ = rows["block1.raw b=1 L=13"]
    print(f"postnet {precision} stale third zero column: |err|/(kappa A) max {elem:.3g}")
    assert passes(*rows["block1.raw b=0 L=40"][:2]) and elem > 10 and not passes(elem, unif)


@pytest.mark.parametrize("precision", ["tf32", "fp32x3"])
def test_postnet_group_norm_count_from_t_fails(precision):
    """utterance 1's GroupNorm divides by (C/8) H T instead of (C/8) H L_b: its mean and variance shrink by 13 / 40, which
    check 1 sees at every element of block1.act (fails by ~2e4x in tf32, ~2e6x in fp32x3)."""
    rows, _ = _pn_rows(precision, "gn_count_from_T")
    elem, unif, _ = rows["block1.act b=1 L=13"]
    print(f"postnet {precision} GroupNorm count from T: |err|/(kappa A) max {elem:.3g}")
    assert passes(*rows["block1.act b=0 L=40"][:2]) and elem > 100 and not passes(elem, unif)
