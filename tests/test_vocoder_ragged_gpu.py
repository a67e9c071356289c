"""Ragged batches in the HiFi-GAN vocoder on the GPU: `Generator.forward(mel, lengths=...)`.

The reference vocodes one utterance at a time (Grad-TTS/inference.py:81, B = 1), and its convs zero-pad at that utterance's
edges.  With `lengths`, each utterance of a padded batch gets exactly that: wav[b, :, :T_b*hop] is bit for bit the
waveform of the B = 1 call on mel[b:b+1, :, :T_b], and the rest of the row is 0.  The padded mel frames here are random,
not silence, so any read of them into a valid sample would show.

Lengths {97, 1, 16, 17, 50, 96} at T = 97: the full length, a one-frame utterance, stage-0 edges exactly at a 128-sample
Conv1d tile edge (16 x 8) and one frame past it (17 x 8), and odd lengths.  V1 (ResBlock1) and V3 (ResBlock2) in every
precision mode.  Bounds against the CPU oracle are the V1 / V3 tests': rel-L2 5e-3 (tf32), 1e-5 (fp32x3), 2e-2 (bf16)."""
import pytest
import torch

from helpers import rel_l2
from hifigan_v3_oracle import generator as v3_generator
from oracle import hifigan_oracle as H
from speech_backbones_b200.hifigan import Generator
from speech_backbones_b200.spec import HIFIGAN_V1, HIFIGAN_V3, synthetic_hifigan_state_dict

pytestmark = pytest.mark.gpu

T = 97
LENGTHS = [97, 1, 16, 17, 50, 96]
CONFIGS = {"v1": HIFIGAN_V1, "v3": HIFIGAN_V3}
ORACLE = {"v1": lambda sd, mel: H.generator(sd, mel, HIFIGAN_V1), "v3": lambda sd, mel: v3_generator(sd, mel, HIFIGAN_V3)}
MODES = ("tf32", "fp32x3", "fp32", "bf16")
BOUND = {"tf32": 5e-3, "fp32x3": 1e-5, "fp32": 1e-5, "bf16": 2e-2}      # rel-L2 against the oracle
SEED = 4242


def _hop(h):
    hop = 1
    for u in h["upsample_rates"]:
        hop *= u
    return hop


@pytest.fixture(scope="module")
def mel():
    return torch.randn(len(LENGTHS), 80, T, generator=torch.Generator().manual_seed(SEED))


@pytest.fixture(scope="module")
def lengths():
    return torch.tensor(LENGTHS, dtype=torch.int64)


@pytest.fixture(scope="module")
def gens():
    cache = {}

    def get(cfg, mode):
        if (cfg, mode) not in cache:
            g = Generator(CONFIGS[cfg], precision=mode).eval()
            g.remove_weight_norm()
            g.load_state_dict(synthetic_hifigan_state_dict(SEED, CONFIGS[cfg]), strict=True)
            cache[(cfg, mode)] = g.cuda()
        return cache[(cfg, mode)]
    return get


@pytest.fixture(scope="module")
def oracle(mel):
    """each utterance through the CPU oracle at its own length (the reference's B = 1 call), per config"""
    cache = {}

    def get(cfg):
        if cfg not in cache:
            sd = synthetic_hifigan_state_dict(SEED, CONFIGS[cfg])
            with torch.no_grad():
                cache[cfg] = [ORACLE[cfg](sd, mel[b:b + 1, :, :n].contiguous()) for b, n in enumerate(LENGTHS)]
        return cache[cfg]
    return get


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_ragged_rows_equal_single_utterance_calls(gens, mel, lengths, cfg, mode):
    g, hop = gens(cfg, mode), _hop(CONFIGS[cfg])
    wav = g(mel.cuda(), lengths=lengths.cuda())
    assert wav.shape == (len(LENGTHS), 1, T * hop) and wav.dtype == torch.float32
    for b, n in enumerate(LENGTHS):
        one = g(mel[b:b + 1, :, :n].cuda())
        assert torch.equal(wav[b:b + 1, :, :n * hop], one), (cfg, mode, b, n)
        assert not wav[b, :, n * hop:].any(), (cfg, mode, b, n)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_full_lengths_equal_the_call_without_lengths(gens, mel, cfg, mode):
    g = gens(cfg, mode)
    m = mel.cuda()
    full = torch.full((len(LENGTHS),), T, dtype=torch.int64, device="cuda")
    assert torch.equal(g(m, lengths=full), g(m))


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_bf16_mel_with_lengths(gens, mel, lengths, cfg):
    g = gens(cfg, "bf16")
    m16 = mel.bfloat16().cuda()
    a, b = g(m16, lengths=lengths.cuda()), g(m16.float(), lengths=lengths.cuda())
    assert a.dtype == torch.float32 and torch.equal(a, b)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_debug_captures_valid_region_equals_single_calls(gens, mel, lengths, cfg, mode):
    """every captured intermediate, restricted to utterance b's own samples at its stage, equals the B = 1 capture"""
    eng = gens(cfg, mode).engine()
    eng.debug_capture(True)
    try:
        eng.forward(mel.cuda(), lengths.cuda())
        names = eng.debug_names()
        mul = {n: eng._debug_len(n) // T for n in names}          # samples per mel frame of each capture's stage
        ragged = {n: eng.debug_read(n) for n in names}
        for b, n_b in enumerate(LENGTHS):
            eng.forward(mel[b:b + 1, :, :n_b].cuda())
            assert eng.debug_names() == names
            for n in names:
                L = n_b * mul[n]
                one = eng.debug_read(n)
                assert one.shape[-1] == L, (n, one.shape)
                assert torch.equal(ragged[n][b:b + 1, :, :L], one), (cfg, mode, b, n)
    finally:
        eng.debug_capture(False)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_poisoned_workspace_rows_equal_single_calls(gens, mel, lengths, cfg, mode):
    """The ragged call right after a dense NaN-mel call at the same (B, T) - which leaves NaN in every workspace buffer the
    next call at that shape reuses - on mel frames that are NaN past each lengths[b]: each waveform still equals its
    single call bit for bit, and the rest of its row is 0.  A kernel that read a frame past an utterance's edge, or masked
    one by multiplying it by 0, would carry the NaN into the utterance's samples."""
    g, hop = gens(cfg, mode), _hop(CONFIGS[cfg])
    # the single calls first: each plans its own shape, which would replace the poisoned workspace
    single = [g(mel[b:b + 1, :, :n].cuda()) for b, n in enumerate(LENGTHS)]
    assert bool(torch.isnan(g(torch.full_like(mel, float("nan")).cuda())).all())
    past = torch.arange(T)[None, :] >= lengths[:, None]
    wav = g(torch.where(past[:, None], float("nan"), mel).cuda(), lengths=lengths.cuda())
    for b, n in enumerate(LENGTHS):
        assert torch.equal(wav[b:b + 1, :, :n * hop], single[b]), (cfg, mode, b, n)
        assert torch.count_nonzero(wav[b, :, n * hop:]) == 0, (cfg, mode, b, n)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("cfg", sorted(CONFIGS))
def test_ragged_rows_vs_oracle(gens, oracle, mel, lengths, cfg, mode):
    hop = _hop(CONFIGS[cfg])
    wav = gens(cfg, mode)(mel.cuda(), lengths=lengths.cuda()).cpu()
    for b, (n, ref) in enumerate(zip(LENGTHS, oracle(cfg))):
        err = rel_l2(wav[b:b + 1, :, :n * hop], ref)
        print(f"vocoder {cfg} {mode} ragged b={b} T_b={n}: rel-L2 vs oracle {err:.3e}")
        assert err <= BOUND[mode], (cfg, mode, b, n, err)


def test_bad_lengths_raise_before_any_launch(gens, mel):
    """int32, a wrong shape, a CPU (or other-device) tensor, a 0 and a value past T are refused with the reason, and the
    handle runs nothing: the last call's captures are still those of the earlier B = 1 call."""
    g = gens("v3", "tf32")
    eng = g.engine()
    m = mel.cuda()
    eng.debug_capture(True)
    try:
        g(m[:1, :, :5])
        wav_numel = eng.debug_read("wav").numel()
        launches = eng.last_launch_count()
        good = torch.tensor(LENGTHS, dtype=torch.int64)
        cases = [("int64", good.int().cuda()), ("shape", good[:5].cuda()), ("shape", good.view(6, 1).cuda()),
                 ("device", good), ("1\\.\\.97", torch.tensor([3, 0, 5, 5, 5, 5], device="cuda")),
                 ("1\\.\\.97", torch.tensor([3, 98, 5, 5, 5, 5], device="cuda")), ("int64", [97] * 6)]
        if torch.cuda.device_count() > 1:
            cases.append(("device", good.to("cuda:1")))
        for match, ln in cases:
            with pytest.raises(ValueError, match=match):
                g(m, lengths=ln)
            assert eng.debug_read("wav").numel() == wav_numel and eng.last_launch_count() == launches, match
    finally:
        eng.debug_capture(False)
