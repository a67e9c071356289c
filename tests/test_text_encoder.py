"""The Grad-TTS text-encoder drop-in (SURVEY.md 8f rank 4; Grad-TTS/model/text_encoder.py:281-326, called at tts.py:75).

CPU: the module's parameter tree is the reference's state_dict (names, shapes, 7,200,145 parameters); the C ABI exports the
symbols; CPU tensors are refused.  GPU: `sbk_textenc_forward` (exact fp32, CUDA cores) against the committed outputs of the
UNMODIFIED reference TextEncoder (tests/golden/text_encoder_golden.pt) and, for the multi-speaker variant (speaker embedding
concatenated after the prenet, 256-channel encoder) and a long ragged batch, against the imported reference's restatement.

Tolerance: fp32 sums in a different order than ATen's: rel-L2 <= 2e-5 on mu and logw (12 LayerNorms deep)."""
import os

import pytest
import torch

from helpers import rel_l2
from oracle import text_encoder_oracle as T
from speech_backbones_b200.text_encoder import TextEncoder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TE_TOL = 2e-5
ARGS = (149, 80, 192, 768, 256, 2, 6, 3, 0.1)          # GradTTS(149, 1, 64, 192, 768, 256, 2, 6, 3, 0.1, 4, ...) (params.py)


@pytest.fixture(scope="module")
def te_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "text_encoder_golden.pt"), weights_only=False)


def test_parameter_tree_is_the_reference_state_dict():
    m = TextEncoder(*ARGS, window_size=4)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == dict(T.param_spec())
    assert m.nparams == 7_200_145
    m.load_state_dict(T.synthetic_weights(3), strict=True)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 5, dtype=torch.long), torch.tensor([5]))


def test_textenc_symbols_exported(sbk_lib):
    for sym in ("sbk_textenc_create", "sbk_textenc_destroy", "sbk_textenc_num_weights", "sbk_textenc_weight_name",
                "sbk_textenc_set_weight", "sbk_textenc_pack", "sbk_textenc_forward", "sbk_textenc_last_launch_count",
                "sbk_textenc_debug_capture", "sbk_textenc_debug_num", "sbk_textenc_debug_name", "sbk_textenc_debug_op_layout",
                "sbk_textenc_debug_read"):
        assert hasattr(sbk_lib, sym), sym


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(3))
def test_text_encoder_matches_reference_golden(te_golden, idx):
    c = te_golden["cases"][idx]
    m = TextEncoder(*ARGS, window_size=4).eval()
    m.load_state_dict(T.synthetic_weights(te_golden["seed"]), strict=True)
    m = m.cuda()
    g = torch.Generator().manual_seed(te_golden["seed"] + c["Tx"])
    x = torch.randint(0, 148, (c["B"], c["Tx"]), generator=g)
    mu, logw, mask = m(x.cuda(), torch.tensor(c["lengths"]).cuda())
    assert mask.shape == (c["B"], 1, c["Tx"]) and mask.sum(-1).flatten().tolist() == c["lengths"]
    e_mu, e_w = rel_l2(mu.cpu(), c["mu"]), rel_l2(logw.cpu(), c["logw"])
    print("text encoder golden", idx, "B=%d Tx=%d mu %.3e logw %.3e" % (c["B"], c["Tx"], e_mu, e_w), "launches", m.engine().last_launch_count())
    assert e_mu <= TE_TOL and e_w <= TE_TOL
    assert (mu.cpu() * (1 - mask.cpu())).abs().max().item() == 0.0 and (logw.cpu() * (1 - mask.cpu())).abs().max().item() == 0.0


@pytest.mark.gpu
def test_text_encoder_long_ragged_batch_vs_oracle():
    """B = 5 utterances of up to 221 tokens (config 1's length), ragged: the oracle on the CPU is the checker."""
    sd = T.synthetic_weights(11)
    m = TextEncoder(*ARGS, window_size=4).eval()
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    x = torch.randint(0, 148, (5, 221), generator=torch.Generator().manual_seed(4))
    lengths = torch.tensor([221, 7, 130, 1, 64])
    with torch.no_grad():
        mu_r, w_r, mk_r = T.text_encoder(sd, x, lengths)
    mu, logw, mask = m(x.cuda(), lengths.cuda())
    assert torch.equal(mask.cpu(), mk_r)
    e_mu, e_w = rel_l2(mu.cpu(), mu_r), rel_l2(logw.cpu(), w_r)
    print("text encoder B=5 Tx=221 mu %.3e logw %.3e" % (e_mu, e_w))
    assert e_mu <= TE_TOL and e_w <= TE_TOL
    # utterances are independent: utterance 2 alone (same padded Tx) reproduces its rows
    mu1, w1, _ = m(x[2:3].cuda(), lengths[2:3].cuda())
    assert rel_l2(mu1.cpu(), mu.cpu()[2:3]) < 1e-6 and rel_l2(w1.cpu(), logw.cpu()[2:3]) < 1e-6


@pytest.mark.gpu
def test_text_encoder_multispeaker_vs_oracle():
    """n_spks > 1: the speaker embedding is concatenated after the prenet and the encoder runs on 192 + 64 channels
    (text_encoder.py:305-310,317-318).  The oracle's multi-speaker branch is bit-identical to the unmodified reference
    (checked when it was written: max abs difference 0.0 on mu, logw and the mask)."""
    sd = T.synthetic_weights(5, spk_extra=64)
    m = TextEncoder(*ARGS, window_size=4, spk_emb_dim=64, n_spks=4).eval()
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    x = torch.randint(0, 148, (2, 37), generator=torch.Generator().manual_seed(1))
    lengths = torch.tensor([37, 20])
    spk = torch.randn(2, 64, generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        mu_r, w_r, _ = T.text_encoder(sd, x, lengths, spk=spk)
    mu, logw, _ = m(x.cuda(), lengths.cuda(), spk.cuda())
    e_mu, e_w = rel_l2(mu.cpu(), mu_r), rel_l2(logw.cpu(), w_r)
    print("text encoder n_spks=4 mu %.3e logw %.3e" % (e_mu, e_w))
    assert e_mu <= TE_TOL and e_w <= TE_TOL


# ---- DiffVC's mel encoder (DiffVC/model/encoder.py:257-284): the same kernels behind `MelEncoder`
@pytest.fixture(scope="module")
def mel_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "mel_encoder_golden.pt"), weights_only=False)


def test_mel_encoder_parameter_tree(sbk_lib):
    from speech_backbones_b200.text_encoder import MelEncoder
    m = MelEncoder(80, 192, 768, 2, 6, 3, 0.1, window_size=4)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == dict(T.mel_param_spec())
    assert m.nparams == 6_841_232
    assert hasattr(sbk_lib, "sbk_melenc_forward")
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 80, 8), torch.ones(1, 1, 8))


def test_mel_oracle_matches_reference_golden(mel_golden):
    sd = T.mel_synthetic_weights(mel_golden["seed"])
    for c in mel_golden["cases"]:
        x = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(mel_golden["seed"] + c["T"]))
        mask = (torch.arange(c["T"])[None, :] < torch.tensor(c["lengths"])[:, None]).float()[:, None]
        with torch.no_grad():
            assert torch.allclose(T.mel_encoder(sd, x, mask), c["out"], rtol=1e-4, atol=1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("idx", range(3))
def test_mel_encoder_matches_reference_golden(mel_golden, idx):
    from speech_backbones_b200.text_encoder import MelEncoder
    c = mel_golden["cases"][idx]
    m = MelEncoder(80, 192, 768, 2, 6, 3, 0.1, window_size=4).eval()
    m.load_state_dict(T.mel_synthetic_weights(mel_golden["seed"]), strict=True)
    m = m.cuda()
    x = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(mel_golden["seed"] + c["T"]))
    mask = (torch.arange(c["T"])[None, :] < torch.tensor(c["lengths"])[:, None]).float()[:, None]
    y = m(x.cuda(), mask.cuda()).cpu()
    err = rel_l2(y, c["out"])
    print("mel encoder golden", idx, "B=%d T=%d rel_l2 %.3e" % (c["B"], c["T"], err), "launches", m.engine().last_launch_count())
    assert err <= TE_TOL
