"""Op isolation for HiFi-GAN V3 (ResBlock2) on the GPU: every captured op of one sbk_vocoder_forward call against its float64
(or bitwise) replay from the GPU's own captured inputs, as tests/test_vocoder_isolation_gpu.py does for V1, in tf32 and in
fp32x3 (whose convs derive the correction operand in shared memory, here on the wide strips too), at shapes where the
Conv1d strips of V3 break:

  * B=1, T=1: stage 0 is 8 samples long, against the 36-sample pad of K = 7 at d = 12 (a wide-strip launch);
  * B=2, T=17: ragged last tiles at every stage;
  * T=301 with the smallest B whose stage-0 convs have more tiles than the device has SMs, so persistent CTAs take a second
    tile with a different border pattern;
  * a config whose largest halo is exactly 128 samples (K = 3 at d = 64), so an interior tile fills all 256 columns of the
    wide strip.

Run with -s to see, per op, the worst |err| / (kappa A) (must be <= 1) and the worst group ratio max / median."""
import pytest
import torch

from op_replay import EPS_ADD, VOC_SLOPE, _bitwise, check, conv1d_ntile, kappa, lrelu_f32
from speech_backbones_b200.spec import HIFIGAN_V3, synthetic_hifigan_state_dict
from test_hifigan_v3 import HIFIGAN_V3_HALO128
from test_vocoder_isolation_gpu import _report_and_assert, _sm_count
from vocoder_replay_modes import VocoderModeReplay, x3_run

pytestmark = pytest.mark.gpu
CONFIGS = {"v3": HIFIGAN_V3, "halo128": HIFIGAN_V3_HALO128}
T_MANY = 301


class ResBlock2Replay(VocoderModeReplay):
    """VocoderModeReplay (tf32, fp32x3) for a ResBlock2 generator: resblocks.n.convs.d.x = conv_d(lrelu(x)) + x, its lrelu
    (.a, d = 0) and the MRF mean over the blocks' convs.1.x; every other op is the V1 replay's."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.all_names = self.names

    def got(self, name):
        if name not in self.cap:
            assert name in self.all_names, f"{name}: the vocoder did not capture it"
            self.cap[name] = self.eng.debug_read(name)
        return self.cap[name]

    def rb2_conv_op(self, name):
        _, n, _, d = name.split(".")[:4]
        n, d = int(n), int(d)
        st, j, pre = n // 3, n % 3, f"resblocks.{n}"
        w, b = self.p[f"{pre}.convs.{d}.weight"], self.p[f"{pre}.convs.{d}.bias"]
        x = self.got(f"ups.{st}.a" if d == 0 else f"{pre}.convs.0.a")
        addin = self.got(f"ups.{st}.x" if d == 0 else f"{pre}.convs.0.x")
        dil = self.h["resblock_dilation_sizes"][j][d]
        ref, A, Alin, floor = self._conv(x, w, b, dil, addin)
        k = kappa(self.mode, w.shape[1] * w.shape[2], extra=2 * EPS_ADD, run=x3_run(w.shape[2]))     # bias add + residual add
        nt = conv1d_ntile(w.shape[0])
        return check(self.got(name), ref, A, k, floor, Alin, pad=(w.shape[2] - 1) * dil // 2,
                     ntile=min(nt, 64) if self.mode == "fp32x3" else nt)

    def run(self):
        nu = len(self.h["upsample_rates"])
        mine = [n for n in self.all_names if n.startswith("resblocks.") or n.startswith("mrf.")]
        rows = []
        for name in mine:
            parts = name.split(".")
            if parts[0] == "mrf":
                i = int(parts[1])
                r = [self.got(f"resblocks.{3 * i + j}.convs.1.x").float() for j in range(3)]
                inv = torch.tensor(1.0 / 3.0, dtype=torch.float32, device=r[0].device)
                rows.append((name,) + _bitwise(self.got(name), lrelu_f32(((r[0] + r[1]) + r[2]) * inv, VOC_SLOPE if i + 1 < nu else 0.01)))
            elif parts[2] == "convs" and parts[4] == "x":
                rows.append((name,) + self.rb2_conv_op(name))
            elif parts[2] == "convs" and parts[3:] == ["0", "a"]:
                rows.append((name,) + _bitwise(self.got(name), lrelu_f32(self.got(name[:-2] + ".x"), VOC_SLOPE)))
            else:
                raise AssertionError(f"unknown vocoder op '{name}': add a replay for it")
        self.names = [n for n in self.all_names if n not in mine]
        try:
            base = super().run()
        finally:
            self.names = self.all_names
        return base[:-1] + rows + base[-1:]


def _stage0_tiles(B, T, h=HIFIGAN_V3):
    L, C = T * h["upsample_rates"][0], h["upsample_initial_channel"] // 2
    return B * ((L + 127) // 128) * (C // conv1d_ntile(C))


def _many_tiles_batch():
    sms, B = _sm_count(), 1
    while _stage0_tiles(B, T_MANY) <= sms:
        B += 1
    return B


@pytest.fixture(scope="module")
def vocoders(sbk_lib):
    from speech_backbones_b200.hifigan import VocoderEngine
    cache = {}

    def get(cfg, mode="tf32"):
        if (cfg, mode) not in cache:
            sd = synthetic_hifigan_state_dict(1234, CONFIGS[cfg])
            e = VocoderEngine(CONFIGS[cfg], 0, mode)
            e.load_state_dict(sd)
            cache[cfg, mode] = (e, sd)
        return cache[cfg, mode]
    yield get
    for e, _ in cache.values():
        e.close()


SHAPES = [("v3", 1, 1), ("v3", 2, 17), ("v3", None, T_MANY), ("halo128", 2, 17), ("halo128", 1, 1)]
CASES = [(c, b, t, m) for m in ("tf32", "fp32x3") for c, b, t in SHAPES]


# (the many-tile batch is counted in tf32's N tiles: fp32x3's are at most 64 wide, so it has at least as many tiles)
@pytest.mark.parametrize("cfg,B,T,mode", CASES,
                         ids=[f"{c}-B{b or 'many'}-T{t}" + ("" if m == "tf32" else f"-{m}") for c, b, t, m in CASES])
def test_v3_vocoder_ops_in_isolation(vocoders, cfg, B, T, mode):
    if B is None:
        B = _many_tiles_batch()
        sms = _sm_count()
        assert _stage0_tiles(B, T) > sms >= _stage0_tiles(B - 1, T), (B, sms)
        print(f"device has {sms} SMs: B = {B} gives {_stage0_tiles(B, T)} stage-0 tiles")
    eng, sd = vocoders(cfg, mode)
    mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(1000 * B + T))
    rows = ResBlock2Replay(eng, sd, CONFIGS[cfg], mel, mode).run()
    names = [r[0] for r in rows]
    assert sum(n.endswith(".x") and ".convs." in n for n in names) == 6 * len(CONFIGS[cfg]["upsample_rates"])
    _report_and_assert(f"{cfg} {mode} B={B} T={T}", rows)


def _expected_names(h):
    names = ["mel_in", "conv_pre"]
    for i in range(len(h["upsample_rates"])):
        names += [f"ups.{i}.z", f"ups.{i}.x", f"ups.{i}.a"]
        for n in range(3 * i, 3 * i + 3):
            names += [f"resblocks.{n}.convs.0.x", f"resblocks.{n}.convs.0.a", f"resblocks.{n}.convs.1.x"]
        names.append(f"mrf.{i}")
    return names + ["wav"]


def test_v3_capture_is_transparent(vocoders):
    """Capture on changes neither the waveform (bitwise) nor the launch count (30), and names every written tensor in
    launch order."""
    eng, _ = vocoders("v3")
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
    assert n_on == n_off == 30
    assert eng.debug_names() == _expected_names(HIFIGAN_V3)
    assert torch.equal(eng.debug_read("wav"), on)


def test_v3_cases_reach_the_edges():
    """V3 runs the 128-, 64- and 32-wide N tiles and the wide strip (halo 72); the halo-128 config fills all 256 columns."""
    c0 = HIFIGAN_V3["upsample_initial_channel"]
    assert {conv1d_ntile(c0 >> (i + 1)) for i in range(3)} == {128, 64, 32}
    halos = lambda h: [(k - 1) * d for k, ds in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]) for d in ds[:2]]
    assert max(halos(HIFIGAN_V3)) == 72
    assert 128 + max(halos(HIFIGAN_V3_HALO128)) == 256
