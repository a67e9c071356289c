"""fp32x3 without a stored correction twin: the U-Net's convs derive the correction operand (sbk_internal.h: corr_chunk) in
shared memory from the fp32 tile they already load (sbk_conv_tc.cu converter warps, Downsample's consumers,
sbk_attn_x3.cu).

Host: the fp32x3 workspace no longer carries a second copy of every operand tensor.
GPU: every captured fp32x3 op of one estimator call against its float64 replay (tests/op_replay.py) at shapes that put the
converted tile's edges where they can go wrong: a row narrower than the halo, a 4-pixel ragged second tile, an odd-height
two-row tile, ragged masks, and (in every case, the `ups` ResnetBlocks) the in0 | in1 concat boundary between K stages.

Run with -s to see the worst op of each case."""
import pytest
import torch

from op_replay import R_UNIFORM, Replay
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict


def test_fp32x3_workspace_has_no_operand_twin(sbk_lib):
    from speech_backbones_b200.binding import Engine
    ws = {}
    for precision in ("fp32x3", "tf32"):
        eng = Engine(precision=precision)              # host-only: no CUDA call until set_weight
        ws[precision] = eng.workspace_bytes(32, 512)
        eng.close()
    # above tf32 only by the doubled per-sample attention weight image (main + correction stages)
    assert ws["tf32"] < ws["fp32x3"] < 1.1 * ws["tf32"], ws


def _mask(B, T, lengths):
    return (torch.arange(T)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]


# (id, n_feats, B, T, lengths, SBK_CONV3_ROWS)
CASES = [
    ("T4", 80, 2, 4, [4, 3], None),                        # every level's row is narrower than the 130-pixel halo
    ("T132", 80, 1, 132, [132], None),                     # 132 / 66 / 33: a 4-pixel tile after a full one
    ("odd-height-2row", 76, 2, 132, [132, 67], "2"),       # heights 76 / 38 / 19, two-row tiles forced: a missing second row
    ("ragged-B3", 80, 3, 508, [508, 129, 128], None),      # mask edges at the tile seam, tiles 4 / 2 / 1 columns short
    ("one-row", 80, 2, 260, [260, 131], "1"),              # one-row tiles (the 128-wide 3x3 instantiation, three stages)
]


@pytest.mark.gpu
@pytest.mark.parametrize("n_feats,B,T,lengths,rows", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_fp32x3_ops_with_in_sm_correction(sbk_lib, monkeypatch, n_feats, B, T, lengths, rows):
    from speech_backbones_b200.binding import Engine
    if rows is not None:
        monkeypatch.setenv("SBK_CONV3_ROWS", rows)         # read when the engine plans (B, T)
    cfg = UNetConfig(n_feats=n_feats)
    sd = synthetic_state_dict(cfg, 1234)
    eng = Engine(n_feats=n_feats, precision="fp32x3")
    try:
        eng.load_state_dict(sd)
        z, _, mu, _, _ = synthetic_inputs(B, T, n_feats=n_feats)
        mask = _mask(B, T, lengths)
        t = torch.linspace(0.9, 0.2, B)
        res = Replay(eng, sd, "fp32x3", "gradtts", z * mask, mask, mu, t, dim=cfg.dim, pe_scale=cfg.pe_scale).run()
    finally:
        eng.close()
    names = {r[0] for r in res}
    assert any(n.startswith("estimator.ups.0.0.") for n in names), "the two-input ResnetBlocks were not replayed"
    we, wu = max(res, key=lambda r: r[1]), max(res, key=lambda r: r[2])
    print(f"WORST B={B} T={T} H={n_feats}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    bad = [r for r in res if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)
