"""Self-tests of the op-isolation checker (tests/op_replay.py), CPU only.

A 3x3 conv over an image three 128-pixel tiles wide (W = 260: two full tiles and a ragged one of 4 columns) is emulated in
each tensor-core mode with the rounding primitives of oracle/precision_model.py.  The clean emulation must pass; each
seeded defect - the kinds of mistake a tiled wgmma conv makes at its tile edges - must fail."""
import pytest
import torch
import torch.nn.functional as F

from helpers import rel_l2
from op_replay import FLOOR_PER_W, R_UNIFORM, check, kappa, passes
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
