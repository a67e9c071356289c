"""CPU: the fp16 sampler mode (sbk.h SBK_PREC_F16) - its operand rounding, the operand-rounding model's prediction for it
(tests/precision_model_fp16.py: oracle/precision_model.py's bf16 model with fp16 rounding), the errors measured on the
H100 pinned next to that prediction, and the host rules of the engines that do not run it (the vocoder refuses it, the
PostNet maps it to tf32 operands)."""
import pytest
import torch

from helpers import case_id, case_inputs, rel_l2, stoc_noise
from oracle import gradtts_oracle as O
from oracle import precision_model as P
from oracle.precision_model import round_f16_sat
from precision_model_fp16 import operand_rounding
from speech_backbones_b200.binding import PREC, SAMPLER_PREC

SBK_ERR_UNSUPPORTED = 4


def test_round_f16_sat_is_rne_to_11_bits_and_saturates():
    e = 2.0 ** -10                                              # fp16's unit in the last place at 1.0
    x = torch.tensor([1.0 + e / 2, 1.0 + 3 * e / 2, -(1.0 + e / 2), 1.0 + e / 2 + 2 ** -20])
    assert torch.equal(round_f16_sat(x), torch.tensor([1.0, 1.0 + 2 * e, -1.0, 1.0 + e]))     # ties to even
    big = torch.tensor([65504.0, 65519.0, 65520.0, 1.0e6, float("inf"), -1.0e9, -float("inf")])
    assert torch.equal(round_f16_sat(big), torch.tensor([65504.0, 65504.0, 65504.0, 65504.0, 65504.0, -65504.0, -65504.0]))
    assert torch.isinf(torch.tensor([65520.0]).half().float()).all()           # what saturation prevents
    sub = torch.tensor([2.0 ** -24, 3 * 2.0 ** -25, 2.0 ** -26])
    assert torch.equal(round_f16_sat(sub), torch.tensor([2.0 ** -24, 2.0 ** -23, 0.0]))       # subnormals, ties to even


def _est_cases(golden):
    return [c for c in golden["cases"] if c["kind"] == "est" and c["n_spks"] == 1]


def _model_est(golden, c, mode):
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    with operand_rounding(mode, sd), torch.no_grad():
        y = O.estimator(sd, cfg, z * mask * c["scale"], mask, mu, torch.tensor(c["t"]), spk)
    return rel_l2(y, c["out"])


def test_fp16_model_error_is_tf32_class(golden):
    """fp16 keeps tf32's 11 significant bits: its modelled per-call error is at most 1.3x the tf32 model's on every golden
    estimator case, the x100 stress case included, and far below the bf16 model's."""
    seen = 0
    for c in _est_cases(golden):
        tf32, fp16, bf16 = (_model_est(golden, c, m) for m in ("tf32", "fp16", "bf16"))
        print(f"{case_id(c)}: tf32 {tf32:.3e}  fp16 {fp16:.3e}  bf16 {bf16:.3e}")
        assert fp16 <= 1.3 * tf32, case_id(c)
        assert fp16 <= 0.3 * bf16, case_id(c)
        seen += 1
    assert seen == 6


def test_fp16_model_leaves_the_oracle_unpatched(golden):
    c = _est_cases(golden)[0]
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    r16 = P.round_bf16
    with operand_rounding("fp16", sd):
        assert P.round_bf16 is round_f16_sat
    assert P.round_bf16 is r16
    with torch.no_grad():
        y = O.estimator(sd, cfg, z * mask * c["scale"], mask, mu, torch.tensor(c["t"]), spk)
    assert torch.allclose(y, c["out"], rtol=1e-5, atol=1e-5 * c["out"].abs().max().item())


# rel-L2 vs the reference measured on an H100 80GB HBM3 (700 W) with scripts/gpu_vs_precision_model.py, keyed by case id:
# one estimator call (golden `est` cases, single-speaker) and whole trajectories
MEASURED = {
    "kindest-n_spks1-B2-T32-raggedTrue-t[0.995, 0.5]-scale1.0": 1.445e-03,
    "kindest-n_spks1-B1-T64-raggedFalse-t[0.005]-scale1.0": 1.381e-03,
    "kindest-n_spks1-B2-T32-raggedTrue-t[0.3, 0.7]-scale100.0": 4.010e-03,
    "kindest-n_spks1-B3-T100-raggedTrue-t[0.9, 0.1, 0.5]-scale1.0": 1.457e-03,
    "kindest-n_spks1-B1-T4-raggedFalse-t[0.5]-scale1.0": 1.468e-03,
    "kindest-n_spks1-B1-T256-raggedFalse-t[0.5]-scale1.0": 1.413e-03,
}
MEASURED_TRAJ = {
    "kindtraj-n_spks1-B2-T32-raggedTrue-N1-stocFalse": 6.311e-04,
    "kindtraj-n_spks1-B2-T32-raggedTrue-N10-stocFalse": 5.443e-04,
    "kindtraj-n_spks1-B2-T32-raggedTrue-N5-stocTrue": 7.183e-04,
    "kindtraj-n_spks1-B1-T128-raggedFalse-N10-stocFalse": 4.887e-04,
}


def test_measured_fp16_error_is_explained_by_operand_rounding(golden):
    """test_precision_model.py's rule for tf32 and bf16: at unit scale the measured per-call error is the model's within
    20 %.  At the |xt| x100 stress case the model, coarser through the attention softmax, over-predicts (tf32: 0.73x, fp16:
    0.55x); there the measurement may not exceed the model by more than that test's 45 % slack - a larger error would be a
    bug, a smaller one is the model's coarseness."""
    seen = 0
    for c in _est_cases(golden):
        predicted, measured = _model_est(golden, c, "fp16"), MEASURED[case_id(c)]
        print(f"fp16 {case_id(c)}: model {predicted:.3e}  GPU {measured:.3e}  ratio {measured / predicted:.3f}")
        if c["scale"] == 1.0:
            assert abs(measured / predicted - 1.0) <= 0.20, case_id(c)
        else:
            assert measured / predicted <= 1.45, case_id(c)
        seen += 1
    assert seen == len(MEASURED)


def test_measured_fp16_trajectory_error_is_explained_by_operand_rounding(golden):
    seen = 0
    for c in golden["cases"]:
        if c["kind"] != "traj" or case_id(c) not in MEASURED_TRAJ:
            continue
        cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
        noise = stoc_noise(golden, c) if c["stoc"] else None
        with operand_rounding("fp16", sd), torch.no_grad():
            y = O.reverse_diffusion(sd, cfg, z, mask, mu, c["N"], c["stoc"], spk, noise=noise)
        predicted, measured = rel_l2(y, c["out"]), MEASURED_TRAJ[case_id(c)]
        print(f"fp16 {case_id(c)}: model {predicted:.3e}  GPU {measured:.3e}  ratio {measured / predicted:.3f}")
        assert abs(measured / predicted - 1.0) <= 0.15, case_id(c)
        seen += 1
    assert seen == len(MEASURED_TRAJ)


# ---- the host rules: the samplers take "fp16", the vocoder refuses it, the PostNet runs it as tf32 ------------------------
def test_fp16_is_a_sampler_mode_only():
    assert SAMPLER_PREC["fp16"] == 4 and "fp16" not in PREC
    assert {k: v for k, v in SAMPLER_PREC.items() if k != "fp16"} == PREC


def test_vocoder_module_refuses_fp16_with_the_reason():
    from speech_backbones_b200.hifigan import Generator
    from speech_backbones_b200.spec import HIFIGAN_V1
    with pytest.raises(ValueError, match="sampler mode"):
        Generator(HIFIGAN_V1, precision="fp16")


def test_vocoder_set_precision_refuses_fp16_and_keeps_its_mode(sbk_lib):
    """SBK_ERR_UNSUPPORTED with the reason; the handle keeps its previous precision, observed through the workspace
    (bf16's conv inputs are half tf32's, so a handle still in bf16 reports the smaller figure)."""
    from speech_backbones_b200.hifigan import VocoderEngine
    from speech_backbones_b200.spec import HIFIGAN_V1
    eng = VocoderEngine(HIFIGAN_V1, 0, "bf16")
    try:
        ws_bf16 = eng.workspace_bytes(2, 17)
        assert eng.lib.sbk_vocoder_set_precision(eng.h, SAMPLER_PREC["fp16"]) == SBK_ERR_UNSUPPORTED
        assert b"fp16" in eng.lib.sbk_last_error()
        assert eng.workspace_bytes(2, 17) == ws_bf16
        assert eng.lib.sbk_vocoder_set_precision(eng.h, PREC["tf32"]) == 0
        assert eng.workspace_bytes(2, 17) > ws_bf16
    finally:
        eng.close()
    with pytest.raises(ValueError, match="sampler mode"):
        VocoderEngine(HIFIGAN_V1, 0, "fp16")


def test_postnet_maps_fp16_to_tf32(sbk_lib):
    """The PostNet has no 16-bit 7x7 kernels: "fp16" constructs (so DiffVC(..., precision="fp16") can build its encoder) and
    runs tf32 operands, the workspace of the tf32 and bf16 handles."""
    from speech_backbones_b200.postnet import PostNet, PostNetEngine
    ws = {}
    for precision in ("tf32", "bf16", "fp16"):
        e = PostNetEngine(128, precision=precision)
        try:
            ws[precision] = [int(e.lib.sbk_postnet_workspace_bytes(e.h, B, 80, T)) for B, T in ((1, 1), (2, 17))]
        finally:
            e.close()
    assert ws["fp16"] == ws["tf32"] == ws["bf16"]
    assert PostNet(128, precision="fp16").precision == "fp16"
    with pytest.raises(ValueError, match="precision"):
        PostNet(128, precision="f16")


def test_sampler_modules_accept_fp16():
    from speech_backbones_b200 import diffvc, gradtts
    assert gradtts.Diffusion(80, 64, precision="fp16").precision == "fp16"
    assert diffvc.Diffusion(80, 64, 64, True, 0.05, 20.0, precision="fp16").precision == "fp16"
