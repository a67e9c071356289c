"""The HiFi-GAN vocoder's precision modes, CPU side: the public surface (Generator / VocoderEngine `precision`, the
sbk_vocoder_set_precision and sbk_vocoder_debug_op_layout entry points and the host-only rules of set_precision), and the
operand-rounding model (tests/vocoder_precision_model.py) that the GPU bounds of tests/test_vocoder_precision_gpu.py come
from, pinned on the reference goldens."""
import ctypes as C
import os

import pytest
import torch

from helpers import rel_l2
from oracle import hifigan_oracle as H
from speech_backbones_b200.binding import PREC
from speech_backbones_b200.hifigan import Generator
from speech_backbones_b200.spec import HIFIGAN_V1, HIFIGAN_V3, synthetic_hifigan_state_dict
from vocoder_precision_model import vocoder_operand_rounding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SBK_ERR_STATE, SBK_ERR_UNSUPPORTED = 3, 4


def test_generator_accepts_every_prec_name_and_rejects_others():
    for name in PREC:
        assert Generator(HIFIGAN_V1, precision=name).precision == name
    assert Generator(HIFIGAN_V1).precision == "tf32"
    for bad in ("fp16", "TF32", "", None):
        with pytest.raises(ValueError, match="precision"):
            Generator(HIFIGAN_V1, precision=bad)
    with pytest.raises(TypeError):
        Generator(HIFIGAN_V1, "bf16")                  # keyword-only


def test_precision_symbols_exported(sbk_lib):
    for sym in ("sbk_vocoder_set_precision", "sbk_vocoder_debug_op_layout"):
        assert hasattr(sbk_lib, sym), sym


def _engine(h, precision="tf32"):
    from speech_backbones_b200.hifigan import VocoderEngine
    return VocoderEngine(h, 0, precision)


def _forward_rc(eng):
    """sbk_vocoder_forward on an unpacked handle: it returns before touching the (never dereferenced) pointers"""
    fake = C.c_void_p(0x1000)
    return eng.lib.sbk_vocoder_forward(eng.h, fake, fake, 1, 4, None)


def test_set_precision_state_rules_without_a_gpu(sbk_lib):
    """A fresh handle is tf32 and unpacked; set_precision is host logic only and leaves the handle unpacked (forward:
    SBK_ERR_STATE until sbk_vocoder_pack); an unknown precision is an argument error."""
    eng = _engine(HIFIGAN_V1)
    try:
        assert _forward_rc(eng) == SBK_ERR_STATE
        for name in ("fp32x3", "bf16", "fp32", "tf32"):
            assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC[name]) == 0, name
            assert _forward_rc(eng) == SBK_ERR_STATE
            assert b"pack" in eng.lib.sbk_last_error()
        assert eng.lib.sbk_vocoder_set_precision(eng.h, 7) == 1
        assert eng.lib.sbk_vocoder_set_precision(eng.h, -1) == 1
        assert eng.debug_op_layout("mel_in") == -1          # nothing captured yet
    finally:
        eng.close()


def test_bf16_rejects_configs_it_cannot_tile(sbk_lib):
    """bf16 K stages hold 16 channels (Conv1d) and 64 (GEMM): num_mels = 72 is a valid tf32 / fp32x3 vocoder but not a bf16
    one.  (That the handle keeps its precision after the refusal is observed on the GPU, test_vocoder_precision_gpu.py:
    fp32x3 and tf32 have the same workspace, so no host-side figure tells them apart.)"""
    h72 = dict(HIFIGAN_V1, num_mels=72)
    eng = _engine(h72)
    try:
        assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC["fp32x3"]) == 0
        assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC["bf16"]) == SBK_ERR_UNSUPPORTED
        assert b"num_mels" in eng.lib.sbk_last_error()
    finally:
        eng.close()
    with pytest.raises(RuntimeError, match="set_precision"):
        _engine(h72, "bf16")
    _engine(h72, "fp32x3").close()


def test_workspace_same_for_fp32x3_and_shrinks_with_bf16(sbk_lib):
    """fp32x3 stores the tf32 mode's tensors (its convs derive the correction operand in shared memory); bf16 halves the
    conv inputs.  V1 (ResBlock1) and V3 (ResBlock2)."""
    for h in (HIFIGAN_V1, HIFIGAN_V3):
        ws = {}
        for name in ("tf32", "fp32x3", "bf16", "fp32"):
            eng = _engine(h, name)
            try:
                ws[name] = [eng.workspace_bytes(B, T) for B, T in ((1, 1), (2, 17), (32, 512))]
            finally:
                eng.close()
        for i in range(3):
            assert ws["bf16"][i] < ws["tf32"][i] == ws["fp32x3"][i], (h.get("resblock", "1"), ws)
        assert ws["fp32"] == ws["fp32x3"]                  # the same fp32x3 path


# ---- the model behind the GPU bounds ------------------------------------------------------------------------------------
# rel-L2 of each mode's modelled waveform against the golden (the unmodified reference in fp32) and against a float64 run,
# and its max-abs against the golden, over the three hifigan_golden.pt cases (B, T) = (1, 32), (2, 20), (1, 5)
MODEL = {"fp32x3": dict(golden=9.4e-7, fp64=4.85e-7, maxabs=1.03e-6),
         "tf32": dict(golden=2.05e-3, fp64=2.05e-3, maxabs=2.01e-3),
         "bf16": dict(golden=7.43e-3, fp64=7.43e-3, maxabs=9.23e-3)}


@pytest.fixture(scope="module")
def hg_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "hifigan_golden.pt"), weights_only=False)


def test_precision_model_reproduces_its_table(hg_golden):
    """Each case within 20 % of the modelled rel-L2 figures (both columns) and under 1.2x the modelled max-abs."""
    sd = synthetic_hifigan_state_dict(hg_golden["seed"])
    sd64 = {k: v.double() for k, v in sd.items()}
    for c in hg_golden["cases"]:
        mel = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(hg_golden["seed"] + c["T"]))
        with torch.no_grad():
            ref64 = H.generator(sd64, mel.double())
            for mode, m in MODEL.items():
                with vocoder_operand_rounding(mode, sd):
                    y = H.generator(sd, mel)
                e_g, e_64, mx = rel_l2(y, c["out"]), rel_l2(y, ref64), (y - c["out"]).abs().max().item()
                print(f"model {mode:7s} B={c['B']} T={c['T']}: vs golden {e_g:.3e}  vs fp64 {e_64:.3e}  max-abs {mx:.3e}")
                assert 0.8 * m["golden"] <= e_g <= 1.2 * m["golden"], (mode, c["T"], e_g)
                assert 0.8 * m["fp64"] <= e_64 <= 1.2 * m["fp64"], (mode, c["T"], e_64)
                assert mx <= 1.2 * m["maxabs"], (mode, c["T"], mx)
