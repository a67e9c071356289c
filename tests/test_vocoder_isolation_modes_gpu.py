"""Op isolation for the HiFi-GAN vocoder in the fp32x3 and bf16 precision modes: the five shapes and configs of
tests/test_vocoder_isolation_gpu.py (strip seams, ragged tiles, many-tile persistence, full 64-sample halos), every
captured op against its float64 (or bitwise) replay from the GPU's own captured inputs (tests/vocoder_replay_modes.py:
tests/op_replay.py VocoderReplay with the mode's kappa, weight rounding and operand stores).  Check 1 (|err| <= kappa A)
and check 2 (max/median <= R_UNIFORM) must hold for every op.  Run with -s for the per-op and per-stage figures."""
import pytest
import torch

from speech_backbones_b200.spec import synthetic_hifigan_state_dict
from test_vocoder_isolation_gpu import CASES, CONFIGS, _many_tiles_batch, _report_and_assert, _stage1_tiles
from vocoder_replay_modes import VocoderModeReplay

pytestmark = pytest.mark.gpu
MODES = ("fp32x3", "bf16")


@pytest.fixture(scope="module")
def vocoders(sbk_lib):
    from speech_backbones_b200.hifigan import VocoderEngine
    cache = {}

    def get(cfg, mode):
        if (cfg, mode) not in cache:
            sd = synthetic_hifigan_state_dict(1234, CONFIGS[cfg])
            e = VocoderEngine(CONFIGS[cfg], 0, mode)
            e.load_state_dict(sd)
            cache[(cfg, mode)] = (e, sd)
        return cache[(cfg, mode)]
    yield get
    for e, _ in cache.values():
        e.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg,B,T", CASES, ids=[f"{c}-B{b or 'many'}-T{t}" for c, b, t in CASES])
def test_vocoder_ops_in_isolation_per_mode(vocoders, mode, cfg, B, T):
    if B is None:
        B = _many_tiles_batch()                 # (fp32x3 runs 64-wide Conv1d N tiles: twice the tf32 tile count)
        print(f"B = {B} gives {_stage1_tiles(B, T)} tf32 stage-1 tiles")
    eng, sd = vocoders(cfg, mode)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(1000 * B + T))
    rep = VocoderModeReplay(eng, sd, CONFIGS[cfg], mel, mode)
    if mode == "bf16":
        assert eng.debug_op_layout("conv_pre") == 2 and eng.debug_op_layout("ups.0.x") == 1
    _report_and_assert(f"{mode} {cfg} B={B} T={T}", rep.run())
