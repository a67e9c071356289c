"""The HiFi-GAN generator drop-in (SURVEY.md 8f rank 3; Grad-TTS/hifi-gan/models.py:77-128, inference.py:60-63,81).

CPU: the module's parameter tree is the reference's (weight-norm names before, plain names after `remove_weight_norm()`), the
effective weights it hands to libsbk equal what `remove_weight_norm()` produces, and the C ABI exports the vocoder symbols.
GPU: `sbk_vocoder_forward` (dilated Conv1d + transposed-conv GEMMs on wgmma, tf32 operands) against the committed outputs of
the UNMODIFIED reference generator (tests/golden/hifigan_golden.pt) and against the CPU oracle at a ragged size.

Tolerance: tf32 operands through a 15-conv-deep residual stack per stage (the arithmetic PyTorch's own GPU convs use by
default): rel-L2 <= 5e-3 on the waveform, max-abs <= 2e-2 of full scale."""
import os

import pytest
import torch

from helpers import rel_l2
from oracle import hifigan_oracle as H
from speech_backbones_b200.hifigan import Generator
from speech_backbones_b200.spec import HIFIGAN_V1, hifigan_param_spec, synthetic_hifigan_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOC_TOL = 5e-3


@pytest.fixture(scope="module")
def hg_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "hifigan_golden.pt"), weights_only=False)


def test_parameter_tree_matches_reference_names():
    g = Generator(HIFIGAN_V1)
    names = set(g.state_dict())
    plain = dict(hifigan_param_spec())
    # weight-norm parametrised checkpoint format (what Grad-TTS/checkpts/hifigan.pt holds): <conv>.weight_g / .weight_v / .bias
    assert names == {n[:-7] + s for n in plain if n.endswith(".weight") for s in (".weight_g", ".weight_v")} | {n for n in plain if n.endswith(".bias")}
    with torch.no_grad():
        for p in g.parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(p.numel())))
    eff = g.effective_state_dict()
    g.remove_weight_norm()
    sd = g.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == plain
    for k in sd:
        assert torch.allclose(eff[k], sd[k], rtol=1e-6, atol=1e-7), k
    g.load_state_dict(synthetic_hifigan_state_dict(7), strict=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        g(torch.zeros(1, 80, 4))


def test_vocoder_symbols_exported(sbk_lib):
    for sym in ("sbk_vocoder_create", "sbk_vocoder_destroy", "sbk_vocoder_num_weights", "sbk_vocoder_weight_name",
                "sbk_vocoder_set_weight", "sbk_vocoder_pack", "sbk_vocoder_workspace_bytes", "sbk_vocoder_forward",
                "sbk_vocoder_last_launch_count", "sbk_vocoder_debug_capture", "sbk_vocoder_debug_num", "sbk_vocoder_debug_name",
                "sbk_vocoder_debug_read"):
        assert hasattr(sbk_lib, sym), sym


@pytest.fixture(scope="module")
def vocoder(hg_golden):
    g = Generator(HIFIGAN_V1).eval()
    g.remove_weight_norm()
    g.load_state_dict(synthetic_hifigan_state_dict(hg_golden["seed"]), strict=True)
    return g.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(3))
def test_vocoder_matches_reference_golden(vocoder, hg_golden, idx):
    c = hg_golden["cases"][idx]
    gen = torch.Generator().manual_seed(hg_golden["seed"] + c["T"])
    mel = torch.randn(c["B"], 80, c["T"], generator=gen)
    y = vocoder(mel.cuda()).cpu()
    assert y.shape == (c["B"], 1, c["T"] * 256) and y.dtype == torch.float32
    err, mx = rel_l2(y, c["out"]), (y - c["out"]).abs().max().item()
    print("vocoder golden", idx, "B=%d T=%d rel_l2 %.3e max_abs %.3e" % (c["B"], c["T"], err, mx), "launches", vocoder.engine().last_launch_count())
    assert err <= VOC_TOL and mx <= 2e-2


@pytest.mark.gpu
def test_vocoder_vs_oracle_long_ragged(vocoder, hg_golden):
    """T = 301 (not a multiple of any tile: 77056 samples, strips end mid-tile at every stage), B = 3."""
    sd = synthetic_hifigan_state_dict(hg_golden["seed"])
    mel = torch.randn(3, 80, 301, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        ref = H.generator(sd, mel)
    y = vocoder(mel.cuda()).cpu()
    err = rel_l2(y, ref)
    print("vocoder B=3 T=301 rel_l2 %.3e" % err)
    assert err <= VOC_TOL
    # batch entries are independent
    y1 = vocoder(mel[1:2].cuda()).cpu()
    assert rel_l2(y1, y[1:2]) < 1e-6


@pytest.mark.gpu
def test_vocoder_weight_norm_checkpoint_path(hg_golden):
    """inference.py:60-63 order: construct (weight norm attached) -> load a weight-norm checkpoint -> cuda -> forward works
    both before and after remove_weight_norm() and gives the same waveform up to the tf32 operand rounding: the effective
    weights g * v / ||v|| computed by this module and by torch's remove_weight_norm differ in the last fp32 bit, which
    flips tf32 roundings of individual weights (measured 1.2e-3 between the two; the bound is the vocoder's own tolerance)."""
    g = Generator(HIFIGAN_V1).eval()
    with torch.no_grad():
        for n, p in g.named_parameters():
            p.copy_(torch.randn(p.shape, generator=torch.Generator().manual_seed(len(n))) * (0.05 if n.endswith("_v") else 1.0))
    g = g.cuda()
    mel = torch.randn(1, 80, 24, generator=torch.Generator().manual_seed(3)).cuda()
    a = g(mel)
    g.remove_weight_norm()
    b = g(mel)
    assert torch.isfinite(a).all() and rel_l2(b.cpu(), a.cpu()) <= VOC_TOL


# A generator valid for HiFi-GAN and accepted by sbk_vocoder_create that reaches the Conv1d strip's limits, which V1 does
# not: K=3, d=32 gives a 64-sample halo (pad 32: an interior strip fills all 128 + 64 columns), K=7, d=10 and K=11, d=6 a
# 60-sample one; stride-4 transposed convs (k = 8: 2-tap folds with u = 4, GEMMs to 8 * co channels).
HIFIGAN_EDGE = dict(HIFIGAN_V1, upsample_rates=[4, 4, 4, 4], upsample_kernel_sizes=[8, 8, 8, 8],
                    resblock_dilation_sizes=[[1, 8, 32], [1, 5, 10], [1, 3, 6]])


def _voc_create_rc(lib, h):
    import ctypes as C
    from speech_backbones_b200.hifigan import SbkVocoderConfig
    lib.sbk_vocoder_create.argtypes = [C.POINTER(SbkVocoderConfig), C.POINTER(C.c_void_p)]
    lib.sbk_vocoder_destroy.argtypes = [C.c_void_p]
    lib.sbk_vocoder_destroy.restype = None
    cfg = SbkVocoderConfig()
    cfg.device, cfg.num_mels, cfg.upsample_initial_channel = 0, h["num_mels"], h["upsample_initial_channel"]
    cfg.n_ups, cfg.n_kernels = len(h["upsample_rates"]), 3
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        cfg.upsample_rates[i], cfg.upsample_kernel_sizes[i] = u, k
    for j in range(3):
        cfg.resblock_kernel_sizes[j] = h["resblock_kernel_sizes"][j]
        for d in range(3):
            cfg.resblock_dilations[j][d] = h["resblock_dilation_sizes"][j][d]
    v = C.c_void_p()
    rc = lib.sbk_vocoder_create(C.byref(cfg), C.byref(v))
    if rc == 0:
        lib.sbk_vocoder_destroy(v)
    return rc


def test_vocoder_create_accepts_and_rejects_at_the_strip_limits(sbk_lib):
    """sbk_vocoder_create touches no device.  A halo (K-1)*d of 64 samples (the strip's capacity) is accepted and 66 is
    not; so are a transposed conv with k != 2u, an odd stride, and a stage whose channels are not a multiple of 32."""
    SBK_ERR_UNSUPPORTED = 4
    assert _voc_create_rc(sbk_lib, HIFIGAN_V1) == 0
    assert _voc_create_rc(sbk_lib, HIFIGAN_EDGE) == 0
    assert _voc_create_rc(sbk_lib, dict(HIFIGAN_V1, resblock_dilation_sizes=[[1, 3, 32], [1, 3, 5], [1, 3, 5]])) == 0
    rejected = {
        "halo 66 (K=3, d=33)": dict(HIFIGAN_V1, resblock_dilation_sizes=[[1, 3, 33], [1, 3, 5], [1, 3, 5]]),
        "halo 70 (K=11, d=7)": dict(HIFIGAN_V1, resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 7]]),
        "k != 2u": dict(HIFIGAN_V1, upsample_kernel_sizes=[15, 16, 4, 4]),
        "odd u": dict(HIFIGAN_V1, upsample_rates=[8, 8, 3, 2], upsample_kernel_sizes=[16, 16, 6, 4]),
        "48 channels": dict(HIFIGAN_V1, upsample_initial_channel=192, upsample_rates=[8, 8],
                            upsample_kernel_sizes=[16, 16]),
    }
    for what, h in rejected.items():
        assert _voc_create_rc(sbk_lib, h) == SBK_ERR_UNSUPPORTED, what


@pytest.mark.gpu
def test_vocoder_edge_config_vs_oracle():
    """The strip-limit config end to end against the CPU oracle, at a ragged and at a one-frame input."""
    from speech_backbones_b200.hifigan import VocoderEngine
    sd = synthetic_hifigan_state_dict(1234, HIFIGAN_EDGE)
    eng = VocoderEngine(HIFIGAN_EDGE, 0)
    try:
        eng.load_state_dict(sd)
        for B, T in ((2, 17), (1, 1)):
            mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(B * 100 + T))
            with torch.no_grad():
                ref = H.generator(sd, mel, HIFIGAN_EDGE)
            y = eng.forward(mel.cuda()).cpu()
            err = rel_l2(y, ref)
            print("vocoder edge config B=%d T=%d rel_l2 %.3e" % (B, T, err))
            assert y.shape == ref.shape and err <= VOC_TOL
    finally:
        eng.close()
