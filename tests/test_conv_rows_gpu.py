"""Two-row tiles of the tensor-core 3x3 conv (sbk_conv_tc.cu, Geo<G_C3, 2>) against the one-row tiles and float64.

(a) The same estimator call planned with SBK_CONV3_ROWS=1 and =2: each output element sees the same MMA sequence and each
    GroupNorm row total the same fp32 partials, so every 3x3 conv output, and the estimator output, is bit-identical.
(b) n_feats = 76 (level heights 76 / 38 / 19: the last row pair of level 2 has no second row) with two-row tiles forced:
    every op passes its float64 replay (tests/op_replay.py), and the estimator matches the oracle within the mode's
    per-call tolerance.
(c) The planner picks two-row tiles when the two-row grid runs at least 4 waves of num_sms tiles (sbk_api.cu tc_conv)."""
import re

import pytest
import torch

from helpers import rel_l2
from op_replay import R_UNIFORM, Replay
from oracle import gradtts_oracle as O
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
MODES = ["fp32", "fp32x3", "tf32", "bf16"]
EST_TOL = {"fp32": 1e-4, "fp32x3": 1e-5, "tf32": 4e-3, "bf16": 2e-2}     # per estimator call (test_parity / test_fp32x3)


def _mask(B, T, lengths):
    return (torch.arange(T)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]


def _engine(precision, n_feats=80, use_graph=True):
    from speech_backbones_b200.binding import Engine
    cfg = UNetConfig(n_feats=n_feats)
    sd = synthetic_state_dict(cfg, 1234)
    eng = Engine(n_feats=n_feats, precision=precision, use_graph=use_graph)
    eng.load_state_dict(sd)
    return eng, cfg, sd


def _captured_raw(eng, x, mask, mu, t):
    eng.debug_capture(True)
    try:
        y = eng.estimator(x.cuda(), mask.cuda(), mu.cuda(), t.cuda())
        torch.cuda.synchronize()
    finally:
        eng.debug_capture(False)
    raws = {n: eng.debug_read(n).clone() for n in eng.debug_names() if n.endswith(".raw")}
    return y.cpu(), raws


@pytest.mark.parametrize("precision", MODES)
def test_two_row_tiles_bit_identical(sbk_lib, monkeypatch, precision):
    B, T, lengths = 2, 516, [516, 257]
    z, _, mu, _, _ = synthetic_inputs(B, T)
    mask = _mask(B, T, lengths)
    t = torch.linspace(0.9, 0.2, B)
    out = {}
    for rows in ("1", "2"):
        monkeypatch.setenv("SBK_CONV3_ROWS", rows)        # read when the engine plans (B, T)
        eng, _, _ = _engine(precision)
        try:
            out[rows] = _captured_raw(eng, z * mask, mask, mu, t)
        finally:
            eng.close()
    (y1, r1), (y2, r2) = out["1"], out["2"]
    assert r1.keys() == r2.keys() and len(r1) >= 20
    diff = [n for n in r1 if not torch.equal(r1[n], r2[n])]
    assert not diff, "3x3 outputs differ between 1-row and 2-row tiles: " + ", ".join(diff)
    assert torch.equal(y1, y2)


@pytest.mark.parametrize("precision", MODES)
def test_two_row_tiles_odd_height(sbk_lib, monkeypatch, precision):
    monkeypatch.setenv("SBK_CONV3_ROWS", "2")
    B, T, lengths = 2, 516, [516, 257]
    eng, cfg, sd = _engine(precision, n_feats=76)
    try:
        z, _, mu, _, _ = synthetic_inputs(B, T, n_feats=76)
        mask = _mask(B, T, lengths)
        t = torch.linspace(0.9, 0.2, B)
        rp = Replay(eng, sd, precision, "gradtts", z * mask, mask, mu, t, dim=cfg.dim, pe_scale=cfg.pe_scale)
        rows = rp.run()
        for name, elem, unif, where in rows:
            print(f"n_feats=76 {precision} {name:44s} |err|/(kA) {elem:.3e}  max/median {unif:6.2f} {where}")
        bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
        assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)
        sd64 = {k: v.double() for k, v in sd.items()}
        ref = O.estimator(sd64, cfg, (z * mask).double(), mask.double(), mu.double(), t.double())
        err = rel_l2(rp.y.cpu(), ref)
        print(f"n_feats=76 {precision}: estimator rel-L2 vs float64 oracle {err:.3e}")
        assert err <= EST_TOL[precision]
    finally:
        eng.close()


def _conv3_rows_launched(eng, B, T):
    """{1, 2}-subset: tile rows of the 3x3 tensor-core kernels one estimator call launches (kernel names, torch.profiler)."""
    z, mask, mu, _, _ = synthetic_inputs(B, T)
    t = torch.full((B,), 0.5)
    args = [v.cuda() for v in (z * mask, mask, mu, t)]
    eng.estimator(*args)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.estimator(*args)
        torch.cuda.synchronize()
    rows = set()
    for ev in prof.key_averages():
        m = re.search(r"k_conv_tc(?:_x3)?<1,[^>]*, ([12])>", ev.key)      # G_C3 = 1; last template argument = rows
        if m:
            rows.add(int(m.group(1)))
    return rows


def _rule(B, T, num_sms, n_feats=80, dim=64):
    """sbk_api.cu tc_conv: per level, two rows iff B * ceil(W/128) * ceil(H/2) * Cout/64 >= 4 * num_sms."""
    rows = set()
    for lvl, cout in ((0, dim), (1, 2 * dim), (2, 4 * dim)):
        H, W = n_feats >> lvl, T >> lvl
        rows.add(2 if B * ((W + 127) // 128) * ((H + 1) // 2) * (cout // 64) >= 4 * num_sms else 1)
    return rows


@pytest.mark.parametrize("precision", ["fp32x3", "tf32", "bf16"])
def test_planner_picks_two_rows(sbk_lib, monkeypatch, precision):
    monkeypatch.delenv("SBK_CONV3_ROWS", raising=False)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _rule(32, 512, sms) == {2} and _rule(1, 512, sms) == {1}    # the benchmark's shape; B = 1 (too few tiles)
    eng, _, _ = _engine(precision, use_graph=False)
    try:
        for B in (32, 1, 4):                                   # (B = 4 on 132 SMs: level 0 two rows, levels 1-2 one row)
            assert _conv3_rows_launched(eng, B, 512) == _rule(B, 512, sms), B
    finally:
        eng.close()
    monkeypatch.setenv("SBK_CONV3_ROWS", "2")
    eng, _, _ = _engine(precision, use_graph=False)
    try:
        assert _conv3_rows_launched(eng, 1, 512) == {2}        # the override
    finally:
        eng.close()
