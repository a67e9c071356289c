"""HiFi-GAN V3 (ResBlock2, Grad-TTS/hifi-gan/models.py:53-74,84) through the drop-in Generator and sbk_vocoder_create_ex.

CPU: the parameter tree is the reference's for a resblock "2" config, the ResBlock2 oracle (tests/hifigan_v3_oracle.py)
reproduces the committed outputs of the UNMODIFIED reference generator (tests/golden/hifigan_v3_golden.pt), and
sbk_vocoder_create_ex accepts and refuses configs by its documented rules (host only, no device work).
GPU: V3 against the reference golden in each precision mode, with the bounds the V1 tests use; a ragged call against the
oracle; the weight-norm checkpoint path; and the V1 waveform is bitwise the same through both create entry points."""
import ctypes as C
import os

import pytest
import torch
from torch.nn.utils import remove_weight_norm

from helpers import rel_l2
from hifigan_v3_oracle import V3, generator, macs_per_mel_frame, param_spec
from speech_backbones_b200.hifigan import Generator, SbkVocoderConfig, SbkVocoderConfigEx, VocoderEngine
from speech_backbones_b200.spec import HIFIGAN_V1, HIFIGAN_V3, hifigan_param_spec, synthetic_hifigan_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SBK_ERR_UNSUPPORTED = 4
BOUND = {"tf32": (5e-3, 2e-2), "fp32x3": (1e-5, 1e-4), "bf16": (2e-2, 5e-2)}        # (rel-L2, max-abs), as for V1


@pytest.fixture(scope="module")
def v3_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "hifigan_v3_golden.pt"), weights_only=False)


def test_v3_config_and_inventory(v3_golden):
    assert HIFIGAN_V3 == V3 == v3_golden["config"]
    spec = hifigan_param_spec(HIFIGAN_V3)
    assert spec == param_spec(V3) and len(spec) == 46
    assert sum(int(torch.tensor(s).prod()) for _, s in spec) == v3_golden["nparams"] == 1_462_273
    assert macs_per_mel_frame(V3) == v3_golden["macs_per_mel_frame"] == 22_482_944
    assert [n for n in dict(spec) if n.startswith("resblocks.0.")] == [
        "resblocks.0.convs.0.weight", "resblocks.0.convs.0.bias", "resblocks.0.convs.1.weight", "resblocks.0.convs.1.bias"]


def test_v3_parameter_tree_matches_reference_names():
    g = Generator(HIFIGAN_V3)
    plain = dict(hifigan_param_spec(HIFIGAN_V3))
    assert set(g.state_dict()) == ({n[:-7] + s for n in plain if n.endswith(".weight") for s in (".weight_g", ".weight_v")}
                                   | {n for n in plain if n.endswith(".bias")})
    with torch.no_grad():
        for p in g.parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(p.numel())))
    eff = g.effective_state_dict()
    g.remove_weight_norm()
    sd = g.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == plain and len(sd) == 46
    for k in sd:
        assert torch.allclose(eff[k], sd[k], rtol=1e-6, atol=1e-7), k
    g.load_state_dict(synthetic_hifigan_state_dict(7, HIFIGAN_V3), strict=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        g(torch.zeros(1, 80, 4))


def test_v3_effective_weights_equal_torch_remove_weight_norm():
    """effective_state_dict on a ResBlock2 conv equals what torch's remove_weight_norm leaves behind"""
    g = Generator(HIFIGAN_V3)
    with torch.no_grad():
        for n, p in g.named_parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(len(n))))
    eff = g.effective_state_dict()
    conv = g.resblocks[4].convs[1]
    remove_weight_norm(conv)
    assert torch.allclose(eff["resblocks.4.convs.1.weight"], conv.weight, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("idx", range(3))
def test_v3_oracle_matches_reference_golden(v3_golden, idx):
    c = v3_golden["cases"][idx]
    sd = synthetic_hifigan_state_dict(v3_golden["seed"], V3)
    mel = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(v3_golden["seed"] + c["T"]))
    with torch.no_grad():
        y = generator(sd, mel, V3)
    assert y.shape == (c["B"], 1, c["T"] * 256)
    assert torch.allclose(y, c["out"], rtol=1e-5, atol=1e-6)      # same build + seeds => bit-exact; slack for BLAS threads


def _fill(cfg, h, resblock=None):
    cfg.device, cfg.num_mels, cfg.upsample_initial_channel = 0, h["num_mels"], h["upsample_initial_channel"]
    cfg.n_ups, cfg.n_kernels = len(h["upsample_rates"]), len(h["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        cfg.upsample_rates[i], cfg.upsample_kernel_sizes[i] = u, k
    for j in range(3):
        cfg.resblock_kernel_sizes[j] = h["resblock_kernel_sizes"][j]
        for d, dil in enumerate(h["resblock_dilation_sizes"][j][:3]):
            cfg.resblock_dilations[j][d] = dil
    if resblock is not None:
        cfg.resblock = resblock
    return cfg


def _create_ex_rc(lib, h, resblock):
    lib.sbk_vocoder_create_ex.argtypes = [C.POINTER(SbkVocoderConfigEx), C.POINTER(C.c_void_p)]
    lib.sbk_vocoder_destroy.argtypes = [C.c_void_p]
    lib.sbk_vocoder_destroy.restype = None
    v = C.c_void_p()
    rc = lib.sbk_vocoder_create_ex(C.byref(_fill(SbkVocoderConfigEx(), h, resblock)), C.byref(v))
    if rc == 0:
        lib.sbk_vocoder_destroy(v)
    return rc


# HiFi-GAN V2 (the public config_v2.json): 128 initial channels, so stages of 64, 32, 16 and 8 channels
HIFIGAN_V2 = dict(HIFIGAN_V1, upsample_initial_channel=128)
# V3 with K = 3 at d = 64: a 128-sample halo, the wide strip's capacity
HIFIGAN_V3_HALO128 = dict(HIFIGAN_V3, resblock_dilation_sizes=[[1, 64], [2, 6], [3, 12]])


def test_create_ex_accepts_and_rejects(sbk_lib):
    """sbk_vocoder_create_ex touches no device: V3, a 128-sample halo and a ResBlock1 config with a 66-sample halo are
    accepted; a 130-sample halo, K = 9, resblock 3, V2's 16-channel stage, k != 2u and dilation 0 are refused."""
    accepted = {
        "V3": (HIFIGAN_V3, 2),
        "halo 128 (K=3, d=64)": (HIFIGAN_V3_HALO128, 2),
        "ResBlock1, halo 66 (K=3, d=33)": (dict(HIFIGAN_V1, resblock_dilation_sizes=[[1, 3, 33], [1, 3, 5], [1, 3, 5]]), 1),
        "V1": (HIFIGAN_V1, 1),
    }
    for what, (h, rb) in accepted.items():
        assert _create_ex_rc(sbk_lib, h, rb) == 0, (what, sbk_lib.sbk_last_error())
    rejected = {
        "halo 130 (K=11, d=13)": (dict(HIFIGAN_V1, resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 13]]), 1),
        "K = 9": (dict(HIFIGAN_V3, resblock_kernel_sizes=[3, 9, 7]), 2),
        "resblock 3": (HIFIGAN_V3, 3),
        "V2 (16-channel stage)": (HIFIGAN_V2, 1),
        "k != 2u": (dict(HIFIGAN_V3, upsample_kernel_sizes=[16, 15, 8]), 2),
        "dilation 0": (dict(HIFIGAN_V3, resblock_dilation_sizes=[[1, 0], [2, 6], [3, 12]]), 2),
    }
    for what, (h, rb) in rejected.items():
        assert _create_ex_rc(sbk_lib, h, rb) == SBK_ERR_UNSUPPORTED, what


def test_engine_refusals_name_the_reason(sbk_lib):
    """VocoderEngine builds through sbk_vocoder_create_ex (host only here): V2 is refused by the 32-channel rule, an unknown
    resblock by name; V3's weight inventory is the reference's."""
    with pytest.raises(RuntimeError, match="16 channels.*multiple of 32"):
        VocoderEngine(HIFIGAN_V2, 0)
    with pytest.raises(RuntimeError, match="resblock '3'"):
        VocoderEngine(dict(HIFIGAN_V3, resblock="3"), 0)
    eng = VocoderEngine(HIFIGAN_V3, 0)
    try:
        assert eng.weight_names() == [n for n, _ in hifigan_param_spec(HIFIGAN_V3)]
    finally:
        eng.close()


# ---- GPU ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def v3_vocoders(v3_golden):
    cache = {}

    def get(mode):
        if mode not in cache:
            g = Generator(HIFIGAN_V3, precision=mode).eval()
            g.remove_weight_norm()
            g.load_state_dict(synthetic_hifigan_state_dict(v3_golden["seed"], HIFIGAN_V3), strict=True)
            cache[mode] = g.cuda()
        return cache[mode]
    return get


def _within(mode, y, ref, what):
    err, mx = rel_l2(y, ref), (y.double() - ref.double()).abs().max().item()
    print(f"vocoder V3 {mode} {what}: rel-L2 {err:.3e}  max-abs {mx:.3e}")
    assert y.dtype == torch.float32 and y.shape == ref.shape
    assert err <= BOUND[mode][0] and mx <= BOUND[mode][1], (mode, what, err, mx)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ("tf32", "fp32x3", "bf16"))
@pytest.mark.parametrize("idx", range(3))
def test_v3_matches_reference_golden(v3_vocoders, v3_golden, mode, idx):
    c = v3_golden["cases"][idx]
    mel = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(v3_golden["seed"] + c["T"]))
    g = v3_vocoders(mode)
    y = g(mel.cuda()).cpu()
    _within(mode, y, c["out"], f"golden B={c['B']} T={c['T']}")
    assert g.engine().last_launch_count() == 30


@pytest.mark.gpu
def test_v3_vs_oracle_long_ragged(v3_vocoders, v3_golden):
    """B = 3, T = 301: strips end mid-tile at every stage; batch entries are independent."""
    sd = synthetic_hifigan_state_dict(v3_golden["seed"], HIFIGAN_V3)
    mel = torch.randn(3, 80, 301, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = generator(sd, mel, V3)
    g = v3_vocoders("tf32")
    y = g(mel.cuda()).cpu()
    _within("tf32", y, ref, "B=3 T=301 vs oracle")
    y1 = g(mel[1:2].cuda()).cpu()
    assert rel_l2(y1, y[1:2]) < 1e-6


@pytest.mark.gpu
def test_v3_weight_norm_checkpoint_path():
    """inference.py:60-63 order with a V3 config: weight-norm parameters -> cuda -> forward, before and after
    remove_weight_norm(); the two differ only by the last-bit differences of the effective weights (tf32 rounding flips)."""
    g = Generator(HIFIGAN_V3).eval()
    with torch.no_grad():
        for n, p in g.named_parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(len(n))) * (0.05 if n.endswith("_v") else 1.0))
    g = g.cuda()
    mel = torch.randn(1, 80, 24, generator=torch.Generator().manual_seed(3)).cuda()
    a = g(mel)
    g.remove_weight_norm()
    b = g(mel)
    assert torch.isfinite(a).all() and rel_l2(b.cpu(), a.cpu()) <= BOUND["tf32"][0]


@pytest.mark.gpu
def test_v1_same_waveform_from_both_create_paths():
    """V1 weights through sbk_vocoder_create and through sbk_vocoder_create_ex(resblock = 1): bitwise the same waveform"""
    sd = synthetic_hifigan_state_dict(2468)
    mel = torch.randn(2, 80, 23, generator=torch.Generator().manual_seed(11)).cuda()
    ex = VocoderEngine(HIFIGAN_V1, 0)
    legacy = VocoderEngine(HIFIGAN_V1, 0)
    try:
        legacy.close()                                    # replace its handle by one from the V1 entry point
        lib = legacy.lib
        lib.sbk_vocoder_create.argtypes = [C.POINTER(SbkVocoderConfig), C.POINTER(C.c_void_p)]
        assert lib.sbk_vocoder_create(C.byref(_fill(SbkVocoderConfig(), HIFIGAN_V1)), C.byref(legacy.h)) == 0
        for e in (ex, legacy):
            e.load_state_dict(sd)
        a, b = ex.forward(mel), legacy.forward(mel)
        torch.cuda.synchronize()
        assert torch.equal(a, b)
        assert ex.last_launch_count() == legacy.last_launch_count() == 87
    finally:
        ex.close()
        legacy.close()
