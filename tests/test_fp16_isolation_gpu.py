"""The fp16 mode op by op: every captured op of an fp16 estimator call against its float64 replay (tests/op_replay.py), at
the shapes test_op_isolation_gpu.py uses (tile tails at every level, mask edges at tile seams, ragged batches after a NaN
call), and one call whose stored operands exceed fp16's range.

The bounds are the bf16 mode's with fp16's rounding points, as the operand-rounding model has them
(tests/precision_model_fp16.py: the fp16 mode is the bf16 mode with round_f16_sat in place of round_bf16): the replay runs in
its "bf16" structure - the same tensors are 16-bit, the same ones fp32 - with
  * the operand rounding of one product u = 2^-10 + 2^-22 (weights RNE to 10 fraction bits, <= 2^-11; one rebuilt
    activation rounding, <= 2^-11; the stored operand tensors are exact fp16, read as stored), in place of bf16's
    2^-7 + 2^-16, and
  * a 16-bit output store of <= 2^-11 (RNE to 10 fraction bits) in place of bf16's 2^-8,
  * the Block activation rebuilt and rounded as k_gn_act rounds it in this mode (round_f16_sat).
fp16 captures are read through the engine widened to fp32 (debug layout 4, the bf16 layout with fp16 elements)."""
import pytest
import torch

import op_replay
from oracle.precision_model import round_f16_sat
from op_replay import Replay
from speech_backbones_b200 import synthetic_inputs
from speech_backbones_b200.gradtts import fix_len_compatibility
from test_op_isolation_gpu import (DIFFVC_CASES, GRADTTS_CASES, RAGGED_CASES, _mask, _poison_plan, _report_and_assert,
                                   engines)  # noqa: F401  (engines: the module-scoped engine fixture)

pytestmark = pytest.mark.gpu
F16_MAX = 65504.0


class _Fp16Captures:
    """an fp16 engine as the replay reads it: layout 4 (fp16 [B][H][C/8][W][8], widened to fp32 by debug_read) is the
    bf16 layout 2 with other elements"""

    def __init__(self, eng):
        self._eng = eng

    def __getattr__(self, name):
        return getattr(self._eng, name)

    def debug_layout(self, name=None):
        fmt = self._eng.debug_layout(name)
        return 2 if fmt == 4 else fmt


@pytest.fixture
def fp16_bounds(monkeypatch):
    monkeypatch.setitem(op_replay.U_OPERAND, "bf16", 2 ** -10 + 2 ** -22)
    monkeypatch.setattr(op_replay, "EPS_STORE_BF16", 2 ** -11)
    monkeypatch.setattr(op_replay, "round_bf16", round_f16_sat)


@pytest.mark.parametrize("B,T,lengths,n_spks", GRADTTS_CASES, ids=[f"B{c[0]}-T{c[1]}-spk{c[3]}" for c in GRADTTS_CASES])
def test_gradtts_fp16_ops_in_isolation(engines, fp16_bounds, B, T, lengths, n_spks):
    eng, cfg, sd = engines("gradtts", "fp16", n_spks)
    z, _, mu, spk, _ = synthetic_inputs(B, T, n_spks=n_spks)
    mask = _mask(B, T, lengths)
    t = torch.linspace(0.9, 0.2, B)
    rows = Replay(_Fp16Captures(eng), sd, "bf16", "gradtts", z * mask, mask, mu, t, spk=spk, dim=cfg.dim,
                  pe_scale=cfg.pe_scale).run()
    _report_and_assert(f"gradtts fp16 B={B} T={T} spk={n_spks}", rows)


@pytest.mark.parametrize("B,T,lengths,n_spks", RAGGED_CASES, ids=[f"B{c[0]}-T{c[1]}-spk{c[3]}" for c in RAGGED_CASES])
def test_gradtts_fp16_ragged_ops_in_isolation(engines, fp16_bounds, B, T, lengths, n_spks):
    """per utterance on its own frames, after a dense NaN call has filled the plan's workspace, with NaN past every T_b"""
    eng, cfg, sd = engines("gradtts", "fp16", n_spks)
    z, _, mu, spk, _ = synthetic_inputs(B, T, n_spks=n_spks)
    t = torch.linspace(0.9, 0.2, B)
    left = _poison_plan(eng, B, T, t, spk)
    assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
    L = torch.tensor(lengths)
    TB = torch.tensor([fix_len_compatibility(n) for n in lengths])
    frames = torch.arange(T)[None, :]
    past = (frames >= TB[:, None])[:, None]
    mask = torch.where(past, float("nan"), (frames < L[:, None]).float()[:, None])
    x = torch.where(past, float("nan"), z * mask)
    mu = torch.where(past, float("nan"), mu)
    rp = Replay(_Fp16Captures(eng), sd, "bf16", "gradtts", x, mask, mu, t, spk=spk, dim=cfg.dim, pe_scale=cfg.pe_scale,
                lengths=lengths)
    rows = rp.run()
    assert not rp.nonfinite, "NaN / Inf inside an utterance: " + ", ".join(rp.nonfinite)
    for b, Tb in enumerate(TB.tolist()):
        assert torch.count_nonzero(rp.full["y"][b, :, Tb:]) == 0, f"utterance {b}: output not 0 past T_b = {Tb}"
    _report_and_assert(f"gradtts ragged fp16 B={B} T={T} spk={n_spks}", rows)


@pytest.mark.parametrize("B,T", DIFFVC_CASES)
def test_diffvc_fp16_ops_in_isolation(engines, fp16_bounds, B, T):
    from oracle import diffvc_oracle as D
    from speech_backbones_b200.spec import synthetic_diffvc_inputs
    eng, cfg, sd = engines("diffvc", "fp16")
    z, mask, mean, r, rmask, mean_ref, spk = synthetic_diffvc_inputs(B, T, 100, ragged=True)
    if B > 1:
        mask = _mask(B, T, [T] + [T // 2 + 3] * (B - 1))
    t = torch.linspace(0.8, 0.3, B)
    g = D._gamma(cfg, 0, 0.5)
    xt_ref = ((r * g + mean_ref * (1.0 - g)) * rmask)[:, None]
    _, cond = D.conditioning(sd, cfg, xt_ref, rmask, spk, t)
    rows = Replay(_Fp16Captures(eng), sd, "bf16", "diffvc", z * mask, mask, mean, t, cond=cond, dim=cfg.dim_unet).run()
    _report_and_assert(f"diffvc fp16 B={B} T={T}", rows)


def test_stored_operands_beyond_65504_saturate(engines, fp16_bounds, monkeypatch):
    """xt scaled until the first ResnetBlock's output - a stored fp16 operand, its 1x1 res_conv linear in xt - reaches
    4x fp16's largest finite value.  Every captured op is finite, and every op that stores an fp16 operand equals the
    model of the saturating store, its float64 replay clamped to +-65504, within the op's bound; where the replay exceeds
    the range by more than that bound, the capture is exactly +-65504.  Check 1 only: the uniformity check compares
    error levels between column / row groups, and groups of saturated elements have none.  (A numeric case: the
    device's cvt.rn.satfinite store and the host packers' clamp define what an out-of-range value becomes.)"""
    eng, cfg, sd = engines("gradtts", "fp16", 1)
    B, T = 1, 132
    z, _, mu, spk, _ = synthetic_inputs(B, T)
    mask = _mask(B, T, [T])
    t = torch.tensor([0.5])
    eng.debug_capture(True)
    eng.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda())
    first = next(n for n in eng.debug_names() if n.endswith("downs.0.0.out"))
    scale = 4 * F16_MAX / eng.debug_read(first).abs().max().item()
    eng.debug_capture(False)

    saturated = {}
    stored = {"resnet_op": lambda a: a[-1] == "out", "attn_op": lambda a: a[-1] == "out", "resample_op": lambda a: True}
    for meth, is_store in stored.items():
        orig = getattr(Replay, meth)

        def clamped(self, *a, _orig=orig, _is_store=is_store):
            got, ref, A, k, floor, Alin = _orig(self, *a)
            if _is_store(a):
                far = ref.abs() - F16_MAX > k * A              # out of range beyond the op's own error bound
                if bool(far.any()):
                    saturated[a[0]] = int(far.sum())
                    assert bool((got[far].abs() == F16_MAX).all()), f"{a[0]}: out-of-range values not stored as +-65504"
                ref = ref.clamp(-F16_MAX, F16_MAX)
            return got, ref, A, k, floor, Alin
        monkeypatch.setattr(Replay, meth, clamped)
    x = z * mask * scale
    rp = Replay(_Fp16Captures(eng), sd, "bf16", "gradtts", x, mask, mu, t, dim=cfg.dim, pe_scale=cfg.pe_scale)
    rows = rp.run()
    print(f"xt x {scale:.3g}: saturated elements per op {saturated}")
    assert not rp.nonfinite, "non-finite captures: " + ", ".join(rp.nonfinite)
    assert saturated.get("downs.0.0", 0) > 0, saturated
    for name, elem, unif, where in rows:
        print(f"gradtts fp16 saturating {name:44s} |err|/(kA) {elem:.3e}")
    bad = [(n, e) for n, e, _, _ in rows if not e <= 1.0]
    assert not bad, f"ops out of bounds: {bad}"
