"""The HiFi-GAN vocoder in the fp32x3 and bf16 precision modes on the GPU (`Generator(h, precision=...)`).

Bounds, from the CPU operand-rounding model (tests/vocoder_precision_model.py, pinned by tests/test_vocoder_precision.py):
  fp32x3  modelled 9.4e-7 rel-L2 / 1.0e-6 max-abs against the reference goldens; the bound leaves room for the fp32
          accumulation the model does not include: rel-L2 <= 1e-5, max-abs <= 1e-4;
  bf16    modelled 7.4e-3 / 9.2e-3: the project's bf16 per-call bound, rel-L2 <= 2e-2, max-abs <= 5e-2.
The same bounds hold against the CPU oracle (the reference's fp32 arithmetic) at other shapes and on the strip-limit config."""
import os

import pytest
import torch

from helpers import rel_l2
from oracle import hifigan_oracle as H
from speech_backbones_b200.binding import PREC
from speech_backbones_b200.hifigan import Generator, VocoderEngine
from speech_backbones_b200.spec import HIFIGAN_V1, synthetic_hifigan_state_dict
from test_hifigan import HIFIGAN_EDGE

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = ("fp32x3", "bf16")
BOUND = {"fp32x3": (1e-5, 1e-4), "bf16": (2e-2, 5e-2)}        # (rel-L2, max-abs)


@pytest.fixture(scope="module")
def hg_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "hifigan_golden.pt"), weights_only=False)


@pytest.fixture(scope="module")
def vocoders(hg_golden):
    cache = {}

    def get(mode):
        if mode not in cache:
            g = Generator(HIFIGAN_V1, precision=mode).eval()
            g.remove_weight_norm()
            g.load_state_dict(synthetic_hifigan_state_dict(hg_golden["seed"]), strict=True)
            cache[mode] = g.cuda()
        return cache[mode]
    return get


def _within(mode, y, ref, what):
    err, mx = rel_l2(y, ref), (y.double() - ref.double()).abs().max().item()
    print(f"vocoder {mode} {what}: rel-L2 {err:.3e}  max-abs {mx:.3e}")
    assert y.dtype == torch.float32 and y.shape == ref.shape
    assert err <= BOUND[mode][0] and mx <= BOUND[mode][1], (mode, what, err, mx)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("idx", range(3))
def test_vocoder_mode_matches_reference_golden(vocoders, hg_golden, mode, idx):
    c = hg_golden["cases"][idx]
    mel = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(hg_golden["seed"] + c["T"]))
    y = vocoders(mode)(mel.cuda()).cpu()
    _within(mode, y, c["out"], f"golden B={c['B']} T={c['T']}")


@pytest.mark.parametrize("mode", MODES)
def test_vocoder_mode_vs_oracle_long_ragged_batch_independent_repeatable(vocoders, hg_golden, mode):
    """B = 3, T = 301 against the oracle; each batch entry alone gives its row; two identical calls agree bit for bit."""
    g = vocoders(mode)
    sd = synthetic_hifigan_state_dict(hg_golden["seed"])
    mel = torch.randn(3, 80, 301, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = H.generator(sd, mel)
    y = g(mel.cuda())
    _within(mode, y.cpu(), ref, "B=3 T=301 vs oracle")
    y1 = g(mel[1:2].cuda())
    assert rel_l2(y1.cpu(), y[1:2].cpu()) < 1e-6
    y2 = g(mel.cuda())
    assert torch.equal(y2, y)


def test_refused_bf16_switch_keeps_fp32x3():
    """num_mels = 72 does not tile in bf16 (test_vocoder_precision.py): after the refused switch the handle still runs
    fp32x3 - its waveform equals a fresh fp32x3 handle's bit for bit and differs from a tf32 handle's."""
    h72 = dict(HIFIGAN_V1, num_mels=72)
    sd = synthetic_hifigan_state_dict(72, h72)
    mel = torch.randn(1, 72, 16, generator=torch.Generator().manual_seed(72)).cuda()

    def run(precision, refuse_bf16=False):
        eng = VocoderEngine(h72, 0, precision)
        try:
            if refuse_bf16:
                assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC["bf16"]) == 4       # SBK_ERR_UNSUPPORTED
            eng.load_state_dict(sd)
            return eng.forward(mel).cpu()
        finally:
            eng.close()
    y = run("fp32x3", refuse_bf16=True)
    assert torch.equal(y, run("fp32x3"))
    assert not torch.equal(y, run("tf32"))


@pytest.mark.parametrize("mode", MODES)
def test_vocoder_mode_edge_config_vs_oracle(mode):
    """The strip-limit config (64-sample halos, stride-4 folds) at a ragged and at a one-frame input."""
    sd = synthetic_hifigan_state_dict(1234, HIFIGAN_EDGE)
    eng = VocoderEngine(HIFIGAN_EDGE, 0, mode)
    try:
        eng.load_state_dict(sd)
        for B, T in ((2, 17), (1, 1)):
            mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(B * 100 + T))
            with torch.no_grad():
                ref = H.generator(sd, mel, HIFIGAN_EDGE)
            _within(mode, eng.forward(mel.cuda()).cpu(), ref, f"edge B={B} T={T}")
    finally:
        eng.close()


def test_bf16_mode_takes_a_bf16_mel_and_returns_float32(vocoders):
    """bf16 mode: a bfloat16 mel gives the float32 waveform of the same mel widened; the default tf32 mode refuses it."""
    mel16 = torch.randn(2, 80, 23, generator=torch.Generator().manual_seed(11)).bfloat16().cuda()
    g = vocoders("bf16")
    a, b = g(mel16), g(mel16.float())
    assert a.dtype == torch.float32 and torch.equal(a, b)
    with pytest.raises(RuntimeError, match="float32"):
        vocoders("tf32")(mel16)
    with pytest.raises(RuntimeError, match="float32"):
        vocoders("fp32x3")(mel16)


def test_launch_count_is_the_same_in_every_mode(vocoders):
    mel = torch.randn(2, 80, 17, generator=torch.Generator().manual_seed(17)).cuda()
    counts = {}
    for mode in ("tf32", "fp32x3", "bf16"):
        g = vocoders(mode)
        g(mel)
        counts[mode] = g.engine().last_launch_count()
    print("launches per mode", counts)
    assert len(set(counts.values())) == 1, counts


def test_set_precision_needs_a_new_pack(hg_golden):
    """On a packed handle, set_precision drops the packed state (forward: SBK_ERR_STATE); after a pack the handle computes
    exactly what a handle created in that mode computes."""
    sd = synthetic_hifigan_state_dict(hg_golden["seed"])
    mel = torch.randn(1, 80, 9, generator=torch.Generator().manual_seed(9)).cuda()
    eng, fresh = VocoderEngine(HIFIGAN_V1, 0), VocoderEngine(HIFIGAN_V1, 0, "fp32x3")
    try:
        eng.load_state_dict(sd)
        fresh.load_state_dict(sd)
        eng.forward(mel)
        assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC["fp32x3"]) == 0
        with pytest.raises(RuntimeError, match="not packed"):
            eng.forward(mel)
        assert eng.lib.sbk_vocoder_pack(eng.h) == 0
        assert torch.equal(eng.forward(mel), fresh.forward(mel))
    finally:
        eng.close()
        fresh.close()


def test_fp32x3_weight_norm_checkpoint_path():
    """inference.py:60-63 with weight norm attached, then removed: the two effective weights differ in the last fp32 bit,
    which in tf32 flips whole weight roundings (test_hifigan.py); fp32x3 carries each weight to ~2^-22, so the two
    waveforms agree to fp32 class."""
    g = Generator(HIFIGAN_V1, precision="fp32x3").eval()
    with torch.no_grad():
        for n, p in g.named_parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(len(n))) * (0.05 if n.endswith("_v") else 1.0))
    g = g.cuda()
    mel = torch.randn(1, 80, 24, generator=torch.Generator().manual_seed(3)).cuda()
    a = g(mel)
    g.remove_weight_norm()
    b = g(mel)
    err = rel_l2(b.cpu(), a.cpu())
    print("fp32x3 weight-norm path: rel-L2 before/after remove_weight_norm %.3e" % err)
    assert torch.isfinite(a).all() and err <= 1e-5
