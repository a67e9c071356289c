"""DiffVC's inference front end on the CPU: the float64 oracle (oracle/frontend_oracle.py) against the committed outputs of the
notebook's own cells (tests/golden/frontend_golden.pt), the restated Slaney basis against torchaudio's, the front-end handle's
host logic through the C ABI, and the refusals that happen before any launch."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import frontend_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fg():
    return torch.load(os.path.join(ROOT, "tests", "golden", "frontend_golden.pt"), weights_only=False)


def subtraction_inputs(fg, c):
    """(synth, source) of a spectral-subtraction case; inputs that are frames of a fixture mel are stored as a reference"""
    if "frames" in c:
        k, a, b = c["frames"]
        m = fg["mels"][k][:, a:b].numpy()
        return m, m
    if "source_frames" in c:
        k, a, b = c["source_frames"]
        return c["synth"].numpy(), fg["mels"][k][:, a:b].numpy()
    return c["synth"].numpy(), c["source"].numpy()


def test_oracle_get_mel_matches_notebook_golden(fg):
    basis = O.mel_basis()
    for k, wav in fg["wavs"].items():
        ref = fg["mels"][k].double().numpy()
        got = O.get_mel(wav.numpy(), basis)
        assert got.shape == ref.shape == (80, wav.shape[0] // 256), k
        # the notebook's complex64 STFT and float32 magnitude against float64, then its .float(): well under 1e-6 in log
        assert np.abs(got - ref).max() <= 1e-6, k


def test_oracle_silence_is_the_clip(fg):
    x = fg["wavs"]["silence"].numpy()
    basis = O.mel_basis()
    # every mel of digital silence is sum_k w_mk sqrt(1e-9) <= 1.6e-6, under the 1e-5 clip
    assert (basis.sum(axis=1) * np.sqrt(1e-9)).max() <= 1.6e-6
    assert np.all(O.get_mel(x, basis) == np.log(1e-5))
    assert np.all(fg["mels"]["silence"].numpy() == np.float32(np.log(1e-5)))


def test_oracle_subtraction_matches_notebook_golden(fg):
    for c in fg["subtraction"]:
        synth, source = subtraction_inputs(fg, c)
        got, i_min, _ = O.mel_spectral_subtraction(synth, source, **c["kw"], return_window=True)
        assert i_min == c["i_min"], c["name"]
        ref = c["out"].double().numpy()
        # the notebook computes in float32 (a few ulp of exp and log, amplified by the subtraction's cancellation): within
        # 2.4e-7 (1 + |out|) on these cases
        assert np.all(np.abs(got - ref) <= 1e-6 * (1 + np.abs(ref))), c["name"]


def test_tie_first_index_wins(fg):
    c = [c for c in fg["subtraction"] if c["name"] == "tie_first_wins"][0]
    synth, source = subtraction_inputs(fg, c)
    en = O.window_energies(source)
    assert en[3] == en[12] == en.min() and c["i_min"] == 3


def test_basis_matches_torchaudio(fg):
    import torchaudio.functional as AF
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        ta = AF.melscale_fbanks(513, 0.0, 8000.0, 80, 22050, norm="slaney", mel_scale="slaney").T.numpy()
    finally:
        torch.set_default_dtype(prev)
    basis = O.mel_basis()
    assert np.abs(ta - basis).max() <= 1e-12 * np.abs(basis).max()
    nz = np.nonzero(basis.any(axis=0))[0]
    assert (nz[0], nz[-1], int((basis != 0).sum())) == (1, 371, 727)
    assert fg["crosscheck"]["basis_vs_torchaudio_rel"] < 1e-12 and fg["crosscheck"]["stft_vs_torch_rel"] < 1e-12


def test_stft_matches_torch_stft():
    y = np.random.default_rng(3).standard_normal(256 * 9 + 17)
    ours = O.stft(y)
    yp = np.pad(y[:(len(y) // 256) * 256], 384, mode="reflect")
    ts = torch.stft(torch.from_numpy(yp), 1024, 256, 1024, window=torch.hann_window(1024, periodic=True, dtype=torch.float64),
                    center=False, return_complex=True).numpy()
    assert ours.shape == ts.shape == (513, 9)
    assert np.abs(ours - ts).max() <= 1e-12 * np.abs(ts).max()


def test_handle_host_logic(sbk_lib):
    from speech_backbones_b200.binding import SbkFrontendConfig
    lib = sbk_lib
    h = C.c_void_p()
    assert lib.sbk_frontend_create(C.byref(SbkFrontendConfig(0)), C.byref(h)) == 0
    try:
        assert lib.sbk_frontend_dft_bins(h) == 372
        B, T = 3, 129
        # framed operand [B][1024][T] and the DFT's 768 columns (372 bins as (re, im), padded to the 128-wide N tile), fp32
        need = 4 * B * T * (1024 + 768)
        got = lib.sbk_frontend_workspace_bytes(h, B, T)
        assert need <= got <= need + 3 * 256
        assert lib.sbk_frontend_workspace_bytes(h, 0, T) == 0
        assert lib.sbk_frontend_last_launch_count(h) == 0
        # argument checks come before any CUDA call
        out = C.c_void_p(16)
        assert lib.sbk_logmel_forward_lengths(h, out, None, out, 1, 511, 1, None) == 1
        assert b"L >= 512" in lib.sbk_last_error()
        assert lib.sbk_logmel_forward_lengths(h, out, None, out, 1, 1024, 5, None) == 1
        assert lib.sbk_spectral_subtraction_lengths(h, out, out, None, out, 1, 80, 10, 0.02, 0, 5, None) == 1
        assert b"silence_window" in lib.sbk_last_error()
        assert lib.sbk_spectral_subtraction_lengths(h, out, out, None, out, 1, 80, 10, 0.02, 5, 0, None) == 1
        assert b"smoothing_window" in lib.sbk_last_error()
    finally:
        lib.sbk_frontend_destroy(h)


def test_refusals_before_launch(sbk_lib):
    from speech_backbones_b200.frontend import LogMel, check_wav, mel_spectral_subtraction
    wav = torch.zeros(2, 4096)
    with pytest.raises(ValueError, match="CUDA"):
        LogMel()(wav)
    with pytest.raises(ValueError, match="CUDA"):
        mel_spectral_subtraction(torch.zeros(1, 80, 9), torch.zeros(1, 80, 9))
    with pytest.raises(ValueError, match="CUDA"):
        check_wav(torch.empty(2, 4096, device="meta"))


def test_refusal_reasons_on_validated_inputs(monkeypatch, sbk_lib):
    """The shape / dtype / length rules, reached by letting CPU tensors pass the device rule."""
    from speech_backbones_b200 import frontend as FE
    monkeypatch.setattr(FE, "_check_cuda", lambda t, name: None)
    wav = torch.zeros(2, 4096)
    with pytest.raises(ValueError, match="at least 512 samples"):
        FE.check_wav(torch.zeros(2, 511))
    with pytest.raises(ValueError, match="at least 512 samples"):
        FE.check_wav(wav, torch.tensor([4096, 511]))
    with pytest.raises(ValueError, match="int64"):
        FE.check_wav(wav, torch.tensor([4096, 600], dtype=torch.int32))
    with pytest.raises(ValueError, match="shape"):
        FE.check_wav(wav, torch.tensor([4096]))
    with pytest.raises(ValueError, match="1..4096"):
        FE.check_wav(wav, torch.tensor([4097, 600]))
    with pytest.raises(ValueError, match="1..4096"):
        FE.check_wav(wav, torch.tensor([0, 600]))
    with pytest.raises(ValueError, match="float32"):
        FE.check_wav(wav.double())
    w, lens = FE.check_wav(wav, torch.tensor([4096, 512]))
    assert lens.tolist() == [4096, 512]
    m = torch.zeros(1, 80, 9)
    with pytest.raises(ValueError, match="silence_window"):
        FE.mel_spectral_subtraction(m, m, silence_window=0)
    with pytest.raises(ValueError, match="smoothing_window"):
        FE.mel_spectral_subtraction(m, m, smoothing_window=0)
    with pytest.raises(ValueError, match="must match"):
        FE.mel_spectral_subtraction(m, torch.zeros(1, 80, 8))
