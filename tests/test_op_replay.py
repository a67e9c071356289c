"""Self-tests of the op-isolation checker (tests/op_replay.py), CPU only.

A 3x3 conv over an image three 128-pixel tiles wide (W = 260: two full tiles and a ragged one of 4 columns) is emulated in
each tensor-core mode with the rounding primitives of oracle/precision_model.py.  The clean emulation must pass; each
seeded defect - the kinds of mistake a tiled wgmma conv makes at its tile edges - must fail.  The same holds for the 1-D
checks the vocoder uses: a dilated Conv1d over three 128-sample strips in tf32, and the transposed conv's overlap-add fold."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2
from op_replay import FIRST_CONV_TILE, FLOOR_PER_W, R_UNIFORM, TC_TILE, check, ct_fold, kappa, passes, rb_act, rb_conv
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
