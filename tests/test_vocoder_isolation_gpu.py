"""Op isolation for the HiFi-GAN vocoder on the GPU: every captured op of one sbk_vocoder_forward call against its float64
(or bitwise) replay from the GPU's own captured inputs (tests/op_replay.py VocoderReplay), at shapes and configs where the
Conv1d strips of k_conv_tc<G_C1K*> break:

  * B=1, T=1: stage 1 is 8 samples long, shorter than the 25-sample pad: one partial tile clipped on both sides, a
    one-sample first fold, conv_pre on one frame;
  * B=2, T=17: stage 1 (136 samples) ends in an 8-sample tile whose left halo lies entirely in the previous tile and whose
    right halo lies entirely in padding; stage 2 (1088) ends in a 64-sample tile;
  * T=301 with the smallest B whose stage-1 convs have more tiles than the device has SMs, so persistent CTAs take a second
    tile with a different border pattern;
  * a second generator (tests/test_hifigan.py HIFIGAN_EDGE) with 60- and 64-sample halos, the latter filling all 192
    strip columns, and stride-4 folds.

V1 runs all three N-tile widths of the Conv1d kernel (256 / 128 channels: 128-wide, 64: 64-wide, 32: 32-wide).

Run with -s to see, per case, op and stage, the worst |err| / (kappa A) (check 1, must be <= 1) and the worst group ratio
max / median (check 2, must be <= R_UNIFORM).  Bitwise ops show 0 (equal) or inf."""
import pytest
import torch

from op_replay import R_UNIFORM, VocoderReplay, conv1d_ntile
from speech_backbones_b200.spec import HIFIGAN_V1, synthetic_hifigan_state_dict
from test_hifigan import HIFIGAN_EDGE

pytestmark = pytest.mark.gpu
CONFIGS = {"v1": HIFIGAN_V1, "edge": HIFIGAN_EDGE}
T_MANY = 301


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _stage1_tiles(B, T, h=HIFIGAN_V1):
    """Conv1d tiles at stage 1: B * ceil(L / 128) strips * N tiles"""
    L, C = T * h["upsample_rates"][0], h["upsample_initial_channel"] // 2
    return B * ((L + 127) // 128) * (C // conv1d_ntile(C))


def _many_tiles_batch():
    """the smallest B for which the stage-1 convs at T = 301 have more tiles than the device has SMs"""
    sms, B = _sm_count(), 1
    while _stage1_tiles(B, T_MANY) <= sms:
        B += 1
    return B


@pytest.fixture(scope="module")
def vocoders(sbk_lib):
    from speech_backbones_b200.hifigan import VocoderEngine
    cache = {}

    def get(cfg):
        if cfg not in cache:
            sd = synthetic_hifigan_state_dict(1234, CONFIGS[cfg])
            e = VocoderEngine(CONFIGS[cfg], 0)
            e.load_state_dict(sd)
            cache[cfg] = (e, sd)
        return cache[cfg]
    yield get
    for e, _ in cache.values():
        e.close()


def _stage(name):
    parts = name.split(".")
    if parts[0] in ("mel_in", "conv_pre"):
        return "pre"
    if parts[0] == "wav":
        return "post"
    return str(int(parts[1]) // 3 if parts[0] == "resblocks" else int(parts[1]))


def _report_and_assert(tag, rows):
    for name, elem, unif, where in rows:
        print(f"{tag} {name:32s} |err|/(kA) {elem:.3e}  max/median {unif:6.2f} {where}")
    for st in dict.fromkeys(_stage(r[0]) for r in rows):
        rs = [r for r in rows if _stage(r[0]) == st and r[3] != "bitwise"]
        if rs:
            we, wu = max(rs, key=lambda r: r[1]), max(rs, key=lambda r: r[2])
            print(f"STAGE {tag} {st:4s}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    we, wu = max(rows, key=lambda r: r[1]), max(rows, key=lambda r: r[2])
    print(f"WORST {tag}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)


CASES = [("v1", 1, 1), ("v1", 2, 17), ("v1", None, T_MANY), ("edge", 2, 17), ("edge", 1, 1)]


@pytest.mark.parametrize("cfg,B,T", CASES, ids=[f"{c}-B{b or 'many'}-T{t}" for c, b, t in CASES])
def test_vocoder_ops_in_isolation(vocoders, cfg, B, T):
    if B is None:
        B = _many_tiles_batch()
        sms = _sm_count()
        assert _stage1_tiles(B, T) > sms >= _stage1_tiles(B - 1, T), (B, sms)
        print(f"device has {sms} SMs: B = {B} gives {_stage1_tiles(B, T)} stage-1 tiles")
    eng, sd = vocoders(cfg)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(1000 * B + T))
    rows = VocoderReplay(eng, sd, CONFIGS[cfg], mel).run()
    _report_and_assert(f"{cfg} B={B} T={T}", rows)


def _expected_names(h):
    names = ["mel_in", "conv_pre"]
    for i in range(len(h["upsample_rates"])):
        names += [f"ups.{i}.z", f"ups.{i}.x", f"ups.{i}.a"]
        for n in range(3 * i, 3 * i + 3):
            for d in range(3):
                names += [f"resblocks.{n}.convs1.{d}", f"resblocks.{n}.convs2.{d}.x"] + ([f"resblocks.{n}.convs2.{d}.a"] if d < 2 else [])
        names.append(f"mrf.{i}")
    return names + ["wav"]


def test_vocoder_capture_is_transparent(vocoders):
    """Capture on changes neither the waveform (bitwise) nor the launch count, and names every written tensor in launch
    order."""
    eng, _ = vocoders("v1")
    mel = torch.randn(2, 80, 17, generator=torch.Generator().manual_seed(17)).cuda()
    off = eng.forward(mel)
    n_off = eng.last_launch_count()
    eng.debug_capture(True)
    try:
        on = eng.forward(mel)
        n_on = eng.last_launch_count()
    finally:
        eng.debug_capture(False)
    torch.cuda.synchronize()
    assert torch.equal(on, off)
    assert n_on == n_off
    assert eng.debug_names() == _expected_names(HIFIGAN_V1)
    assert torch.equal(eng.debug_read("wav"), on)


def test_vocoder_cases_reach_the_edges():
    """V1 runs the 128-, 64- and 32-wide N tiles; the edge config's largest halo fills the 192-sample strip."""
    c0 = HIFIGAN_V1["upsample_initial_channel"]
    assert {conv1d_ntile(c0 >> (i + 1)) for i in range(4)} == {128, 64, 32}
    halo = max((k - 1) * d for k, ds in zip(HIFIGAN_EDGE["resblock_kernel_sizes"], HIFIGAN_EDGE["resblock_dilation_sizes"])
               for d in ds)
    assert 128 + halo == 192
