"""DiffVC's inference front end on the GPU (csrc/sbk_frontend.cu) against the notebook's own cells (tests/golden/
frontend_golden.pt) and the float64 oracle (oracle/frontend_oracle.py).

Log-mel error model, per element: the DFT runs in the fp32x3 split with K = 1024 (op_replay.kappa: operand rounding 2^-19,
2^-22 per MMA within a run of 24 MMAs, 2^-24 per fold, times A_t = sum_n hann[n] |x_t[n]|; plus the correction chunks' fp16
subnormal floor 2^-24 sum_n hann[n]) on each of re and im, so |d|X_k|| <= sqrt(2) kappa_t, plus the fp32 magnitude's own
rounding (2^-22 |X_k|).  The filterbank sum in fp32 adds 2^-19 mel, so
    |d log_mel| <= (sum_k w_mk (sqrt(2) kappa_t + 2^-22 |X_k|) + 2^-19 mel) / max(mel, 1e-5) + 2^-22 (|log_mel| + 1).
The notebook's own cells (complex64 STFT, float32 magnitude) differ from float64 by < 1.1e-7 in log (measured by
scripts/make_golden_frontend.py); against the golden the bound grows by 2e-7."""
import math

import numpy as np
import pytest
import torch

from op_replay import kappa
from oracle import frontend_oracle as O
from test_frontend import fg, subtraction_inputs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

KAPPA = kappa("fp32x3", 1024, run=24)
FLOOR = 2 ** -24 * O.hann().sum()


def _logmel(wav, lengths=None):
    from speech_backbones_b200.frontend import LogMel
    return LogMel()(wav, lengths)


def logmel_bound(x, basis):
    """per-element bound on |GPU - float64 oracle| of one utterance's [80, T] log-mel"""
    fr = O.frames(x)                                                     # [T, 1024]
    A = np.abs(fr) @ O.hann()                                            # [T]
    X = np.abs(O.stft(x))                                                # [513, T]
    mag = np.sqrt(X ** 2 + 1e-9)
    kap = math.sqrt(2) * (KAPPA * A + FLOOR)                             # [T]
    mel = basis @ mag
    dmel = basis @ (kap[None, :] + 2 ** -22 * mag) + 2 ** -19 * mel
    ref = np.log(np.clip(mel, 1e-5, None))
    return ref, dmel / np.maximum(mel, 1e-5) + 2 ** -22 * (np.abs(ref) + 1)


def test_logmel_vs_oracle_and_golden(fg):
    basis = O.mel_basis()
    worst = 0.0
    for k, wav in fg["wavs"].items():
        got, ml = _logmel(wav[None].cuda())
        got = got[0].double().cpu().numpy()
        assert ml.tolist() == [wav.shape[0] // 256] and got.shape == (80, wav.shape[0] // 256)
        ref, bound = logmel_bound(wav.numpy(), basis)
        r = np.abs(got - ref) / bound
        g = np.abs(got - fg["mels"][k].double().numpy()) / (bound + 2e-7)
        print(f"{k}: worst |err|/bound vs oracle {r.max():.3f}, vs notebook golden {g.max():.3f}, max |err| "
              f"{np.abs(got - ref).max():.2e}")
        worst = max(worst, r.max(), g.max())
    print(f"worst |err|/bound over the fixture: {worst:.3f}")
    assert worst <= 1.0


def test_silence_is_exactly_the_clip(fg):
    got, _ = _logmel(fg["wavs"]["silence"][None].cuda())
    assert torch.all(got == torch.tensor(np.float32(np.log(1e-5)))).item()


def _ragged_batch(fg, lengths):
    src = torch.cat([fg["wavs"]["crop_6415"], fg["wavs"]["crop_8534"]])
    L = max(lengths) + 300
    wav = torch.full((len(lengths), L), float("nan"))                   # NaN past every utterance's end
    for b, n in enumerate(lengths):
        wav[b, :n] = src[1000 * b:1000 * b + n]
    return wav


# lengths in samples: not multiples of 256, the 512-sample minimum (2 frames, the fewest an utterance can have) and frame
# counts around the 128-row GEMM tile
LENGTHS = [64 * 256 + 100, 65 * 256, 128 * 256 + 255, 129 * 256 + 7, 512, 2 * 256 + 255, 40 * 256 + 3]


def test_ragged_rows_equal_single_calls(fg):
    wav = _ragged_batch(fg, LENGTHS).cuda()
    lens = torch.tensor(LENGTHS, device="cuda")
    # a NaN call first: the workspace (framed operand, DFT output) is full of NaN when the ragged batch runs
    _logmel(torch.full((len(LENGTHS), wav.shape[1]), float("nan"), device="cuda"))
    out, ml = _logmel(wav, lens)
    assert ml.tolist() == [n // 256 for n in LENGTHS] and out.shape[-1] == max(ml.tolist())
    assert torch.isfinite(out).all()
    basis = O.mel_basis()
    for b, n in enumerate(LENGTHS):
        one, _ = _logmel(wav[b:b + 1, :n].contiguous())
        Tb = n // 256
        assert torch.equal(out[b, :, :Tb], one[0]), b
        assert torch.all(out[b, :, Tb:] == 0).item(), b
        ref, bound = logmel_bound(wav[b, :n].cpu().numpy(), basis)
        assert (np.abs(one[0].double().cpu().numpy() - ref) / bound).max() <= 1.0, b


def test_rows_independent_of_batch(fg):
    wav = _ragged_batch(fg, LENGTHS).cuda()
    lens = torch.tensor(LENGTHS, device="cuda")
    full, _ = _logmel(wav, lens)
    perm = [3, 0, 6, 5]
    sub, _ = _logmel(wav[perm].contiguous(), lens[perm].contiguous())
    for i, b in enumerate(perm):
        Tb = LENGTHS[b] // 256
        assert torch.equal(sub[i, :, :Tb], full[b, :, :Tb]), b
    dense, ml = _logmel(wav[:1, :LENGTHS[0]].repeat(3, 1).contiguous())
    assert torch.equal(dense[0], dense[2]) and ml.tolist() == [LENGTHS[0] // 256] * 3


def _oracle_noise(synth, source, kw):
    out, i_min, en = O.mel_spectral_subtraction(synth, source, **kw, return_window=True)
    sw = kw.get("silence_window", 5)
    noise = np.min(np.exp(2.0 * synth.astype(np.float64)[:, i_min:i_min + sw]), axis=-1)
    if kw.get("smoothing_window", 5) is not None:
        noise = O.noise_median_smoothing(noise, kw.get("smoothing_window", 5))
    return out, i_min, en, noise


def subtraction_bound(synth, noise, out, kw):
    """|GPU - float64 oracle| of mel_spectral_subtraction: expf within 2 ulp (2^-22) on e = exp(2m) and on the noise floor,
    one fp32 rounding of e - n and of floor * n, halved by the sqrt inside the log; then sqrtf / logf within 2^-21 (1 + |out|)."""
    fl = kw.get("spectral_floor", 0.02)
    e = np.exp(2.0 * synth.astype(np.float64))
    d = e - noise[:, None]
    fn = fl * noise[:, None]
    dd = 2 ** -22 * (e + 2 * noise[:, None]) + 2 ** -24 * np.abs(d)
    return 0.5 * np.maximum(dd, 2 ** -22 * fn) / np.maximum(d, fn) + 2 ** -21 * (1 + np.abs(out))


def test_subtraction_vs_oracle_and_golden(fg):
    from speech_backbones_b200.frontend import mel_spectral_subtraction
    for c in fg["subtraction"]:
        synth, source = subtraction_inputs(fg, c)
        ref, i_min, en, noise = _oracle_noise(synth, source, c["kw"])
        assert i_min == c["i_min"], c["name"]
        if len(en) > 1:
            s = np.sort(en)
            margin = (s[1] - s[0]) / s[0]
            assert margin > 1e-5 or s[0] == s[1], c["name"]
        got = mel_spectral_subtraction(torch.from_numpy(synth)[None].cuda(), torch.from_numpy(source)[None].cuda(),
                                       **c["kw"])[0].double().cpu().numpy()
        bound = subtraction_bound(synth, noise, ref, c["kw"])
        r = np.abs(got - ref) / bound
        gd = np.abs(got - c["out"].double().numpy()) / (2 * bound)
        print(f"{c['name']}: T={synth.shape[1]} window {i_min}; worst |err|/bound vs oracle {r.max():.3f}, vs golden {gd.max():.3f}")
        assert r.max() <= 1.0 and gd.max() <= 1.0, c["name"]


def test_subtraction_ragged_rows_equal_single_calls(fg):
    from speech_backbones_b200.frontend import mel_spectral_subtraction
    cases = [c for c in fg["subtraction"]]
    for kw in (dict(), dict(smoothing_window=None), dict(smoothing_window=1, silence_window=3, spectral_floor=0.1)):
        ins = [subtraction_inputs(fg, c) for c in cases]
        T = max(s.shape[1] for s, _ in ins)
        B = len(ins)
        sy = torch.full((B, 80, T), float("nan"))
        so = torch.full((B, 80, T), float("nan"))
        for b, (s, r) in enumerate(ins):
            sy[b, :, :s.shape[1]] = torch.from_numpy(s)
            so[b, :, :r.shape[1]] = torch.from_numpy(r)
        lens = torch.tensor([s.shape[1] for s, _ in ins], device="cuda")
        out = mel_spectral_subtraction(sy.cuda(), so.cuda(), **kw, lengths=lens)
        for b, (s, r) in enumerate(ins):
            one = mel_spectral_subtraction(torch.from_numpy(s)[None].cuda(), torch.from_numpy(r)[None].cuda(), **kw)
            Tb = s.shape[1]
            assert torch.equal(out[b, :, :Tb], one[0]), (cases[b]["name"], kw)
            assert torch.all(out[b, :, Tb:] == 0).item()


def test_logmel_feeds_diffvc_ragged(fg):
    from speech_backbones_b200.diffvc import DiffVC
    from speech_backbones_b200.frontend import LogMel, mel_spectral_subtraction
    from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS
    torch.manual_seed(0)
    model = DiffVC(*DIFFVC_MODEL_ARGS).eval().cuda()
    lengths = [40 * 256 + 11, 23 * 256]
    wav = _ragged_batch(fg, lengths).cuda()
    mel, ml = LogMel()(wav, torch.tensor(lengths, device="cuda"))
    c = torch.randn(2, 256, device="cuda")
    mean_x, y = model(mel, ml, mel, ml, c, n_timesteps=2, mode="ml", ragged=True)
    assert y.shape == mel.shape and torch.isfinite(y).all()
    # (random weights give mels far outside a trained model's range, where exp(2 m) overflows as in the notebook: only the
    # layout is checked here)
    den = mel_spectral_subtraction(y, y, smoothing_window=1, lengths=ml)
    for b, n in enumerate(ml.tolist()):
        one = mel_spectral_subtraction(y[b:b + 1, :, :n].contiguous(), y[b:b + 1, :, :n].contiguous(), smoothing_window=1)
        assert torch.allclose(den[b, :, :n], one[0], rtol=0, atol=0, equal_nan=True) and torch.all(den[b, :, n:] == 0).item()
