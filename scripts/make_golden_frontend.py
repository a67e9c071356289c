"""Generate tests/golden/frontend_golden.pt from DiffVC's inference notebook (container only: needs the reference tree).

The notebook's own cells are executed from DiffVC/inference.ipynb's JSON: `get_mel`, `noise_median_smoothing` and
`mel_spectral_subtraction` (cell 1).  librosa is not installed, so `get_mel` runs with three stand-ins:
  * `load` returns the fixture waveform (float32 at 22050 Hz: decoding and resampling are not part of the cell under test);
  * `librosa.core.stft` restates librosa 0.6.0's `center=False` path: frames times a float64 periodic Hann window, np.fft in
    float64, stored as complex64;
  * `mel_basis` is oracle/frontend_oracle.py's float64 restatement of `librosa.filters.mel` 0.6.0 (Slaney, norm=1).
The restatements are cross-checked against torchaudio's Slaney filterbank and float64 torch.stft(center=False); both must
agree to float64 round-off, and the result is stored in the fixture.

Waveforms: two 1.5 s crops of DiffVC/example/*.wav (24 kHz int16) converted to float32 at 22050 Hz with
scipy.signal.resample_poly(x, 147, 160) - NOT librosa's resampler, so these are not the samples `librosa.load` would return -
and seeded synthetic signals.  Outputs are stored as the notebook passes them on: get_mel's float64 log-mel cast by its
`.float()`, mel_spectral_subtraction's float32.

    python scripts/make_golden_frontend.py
"""
import json
import os
import sys
import types

import numpy as np
import scipy.io.wavfile
import scipy.signal
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import frontend_oracle as O, ref_import  # noqa: E402

SR = 22050
SEED = 4242
OUT = os.path.join(ROOT, "tests", "golden", "frontend_golden.pt")


def _stft_librosa060(y, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True, dtype=np.complex64):
    """librosa.core.stft 0.6.0 on its center=False path (the only one the notebook uses)"""
    assert not center and window == "hann" and win_length == n_fft
    w = O.hann(n_fft).reshape(-1, 1)                              # float64 periodic Hann
    n = 1 + (len(y) - n_fft) // hop_length
    frames = np.stack([y[i * hop_length:i * hop_length + n_fft] for i in range(n)], axis=1)
    out = np.empty((1 + n_fft // 2, n), dtype=dtype, order="F")
    out[:] = np.fft.fft(w * frames, axis=0)[:out.shape[0]]
    return out


def notebook_cells(wav_for_load):
    """The notebook's cell-1 functions, executed from the .ipynb JSON with the stand-ins above."""
    src_root, _ = ref_import._roots("diffvc")
    nb = json.load(open(os.path.join(src_root, "inference.ipynb")))
    src = "".join(nb["cells"][1]["source"])
    assert "def get_mel" in src and "def mel_spectral_subtraction" in src and "def noise_median_smoothing" in src
    librosa = types.SimpleNamespace(core=types.SimpleNamespace(stft=_stft_librosa060))
    ns = {"np": np, "librosa": librosa, "mel_basis": O.mel_basis(), "load": lambda path, sr: (wav_for_load[path], sr)}
    exec(compile(src, "DiffVC/inference.ipynb:cell1", "exec"), ns)
    return ns


def crosscheck():
    """The restated basis against torchaudio's, the STFT restatement against float64 torch.stft"""
    import torchaudio.functional as AF
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        ta = AF.melscale_fbanks(513, 0.0, 8000.0, 80, 22050, norm="slaney", mel_scale="slaney").T.numpy()
    finally:
        torch.set_default_dtype(prev)
    basis = O.mel_basis()
    d_basis = float(np.abs(ta - basis).max() / np.abs(basis).max())
    y = np.random.default_rng(SEED).standard_normal(8192)
    ours = np.fft.fft(O.hann()[:, None] * np.stack([y[i * 256:i * 256 + 1024] for i in range(29)], axis=1), axis=0)[:513]
    ts = torch.stft(torch.from_numpy(y), 1024, 256, 1024, window=torch.hann_window(1024, periodic=True, dtype=torch.float64),
                    center=False, return_complex=True).numpy()
    d_stft = float(np.abs(ts - ours).max() / np.abs(ours).max())
    nz = np.nonzero(basis.any(axis=0))[0]
    res = {"basis_vs_torchaudio_rel": d_basis, "stft_vs_torch_rel": d_stft, "first_bin": int(nz[0]), "last_bin": int(nz[-1]),
           "nonzeros": int((basis != 0).sum())}
    print("cross-check:", res)
    assert d_basis < 1e-12 and d_stft < 1e-12, res
    return res


def signals():
    src_root, _ = ref_import._roots("diffvc")
    out = {}
    for name, start in (("6415_111615_000012_000005.wav", 1.0), ("8534_216567_000015_000010.wav", 0.5)):
        sr, x = scipy.io.wavfile.read(os.path.join(src_root, "example", name))
        assert sr == 24000 and x.dtype == np.int16
        x = x.astype(np.float64) / 32768.0
        y = scipy.signal.resample_poly(x, 147, 160)
        s = int(start * SR)
        out["crop_" + name[:4]] = y[s:s + 3 * SR // 2].astype(np.float32)
    rng = np.random.default_rng(SEED)
    n = SR // 4 + 37                                                            # 0.25 s, not a whole number of hops
    t = np.arange(n) / SR
    out["white_noise"] = (0.1 * rng.standard_normal(n)).astype(np.float32)
    out["sine_on_bin"] = (0.5 * np.sin(2 * np.pi * (50 * SR / 1024) * t)).astype(np.float32)
    out["sine_between_bins"] = (0.5 * np.sin(2 * np.pi * (120.5 * SR / 1024) * t + 0.3)).astype(np.float32)
    out["chirp"] = (0.5 * scipy.signal.chirp(t, 100.0, t[-1], 8000.0)).astype(np.float32)
    out["silence"] = np.zeros(n, dtype=np.float32)
    out["loud_plus_quiet"] = (0.9 * np.sin(2 * np.pi * 440.0 * t) + 1e-4 * rng.standard_normal(n)).astype(np.float32)
    return out


def subtraction_cases(ns, crop_mel):
    rng = np.random.default_rng(SEED + 1)
    m = crop_mel[:, 40:100].astype(np.float32)                                     # a converted-mel-like grid, 60 frames
    quiet = (rng.standard_normal((80, 20)) - 6.0).astype(np.float32)
    tie = (rng.standard_normal((80, 20)) * 0.3 + 1.0).astype(np.float32)          # loud frames ...
    tie[:, 3:8] = quiet[:, 0:5]                                                    # ... two identical quietest windows
    tie[:, 12:17] = quiet[:, 0:5]
    tie_synth = (rng.standard_normal((80, 20)) - 1.0).astype(np.float32)           # a different noise floor per window
    cases = [
        dict(name="crop_smooth_none", synth=m, source=m, kw=dict(smoothing_window=None)),
        dict(name="crop_smooth_1", synth=m, source=m, kw=dict(smoothing_window=1)),
        dict(name="crop_smooth_5", synth=m, source=m, kw=dict(smoothing_window=5)),     # (the notebook's default)
        dict(name="distinct_synth_source", synth=(m + 0.25 * rng.standard_normal(m.shape)).astype(np.float32), source=None,
             kw=dict(spectral_floor=0.05, silence_window=3, smoothing_window=2)),
        dict(name="short_T3", synth=(rng.standard_normal((80, 3)) - 2).astype(np.float32),
             source=(rng.standard_normal((80, 3)) - 2).astype(np.float32), kw={}),
        dict(name="short_T5", synth=(rng.standard_normal((80, 5)) - 2).astype(np.float32),
             source=(rng.standard_normal((80, 5)) - 2).astype(np.float32), kw={}),
        dict(name="all_loud", synth=(rng.standard_normal((80, 16)) - 1).astype(np.float32),
             source=(rng.standard_normal((80, 16)) * 0.1 + 3.5).astype(np.float32), kw={}),
        dict(name="tie_first_wins", synth=tie_synth, source=tie, kw={}),
    ]
    for c in cases:
        if c["source"] is None:
            c["source"] = m
        c["out"] = ns["mel_spectral_subtraction"](c["synth"], c["source"], **c["kw"]).astype(np.float32)
        _, i_min, en = O.mel_spectral_subtraction(c["synth"], c["source"], **c["kw"], return_window=True)
        c["i_min"] = i_min
        print(f"subtraction {c['name']}: T={c['synth'].shape[1]} i_min={i_min} "
              f"min energy={en.min() if len(en) else float('nan'):.6g}")
    assert [c for c in cases if c["name"] == "tie_first_wins"][0]["i_min"] == 3
    assert [c for c in cases if c["name"] == "all_loud"][0]["i_min"] == 0
    # frames 40:100 of mels["crop_6415"] are not stored again: the crop cases take them as synth and source (as the notebook
    # calls the function), the distinct case as its source
    for c in cases:
        if c["name"].startswith("crop_"):
            del c["synth"], c["source"]
            c["frames"] = ("crop_6415", 40, 100)
        elif c["source"] is m:
            del c["source"]
            c["source_frames"] = ("crop_6415", 40, 100)
    return [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in c.items()} for c in cases]


def main():
    cc = crosscheck()
    sig = signals()
    ns = notebook_cells(sig)
    mels = {}
    for k, x in sig.items():
        ref = ns["get_mel"](k)
        ora = O.get_mel(x)
        err = float(np.abs(ref - ora).max())
        print(f"get_mel {k}: samples {len(x)} frames {ref.shape[1]}; notebook cell vs float64 oracle max |d log| = {err:.3e}")
        assert ref.shape == ora.shape
        mels[k] = torch.from_numpy(ref).float()                              # the notebook's .float()
    sub = subtraction_cases(ns, mels["crop_6415"].numpy())
    out = {
        "seed": SEED, "sr": SR,
        "note": ("waveforms: crops of DiffVC/example/*.wav resampled 24 kHz -> 22050 Hz with scipy.signal.resample_poly(x, 147, "
                 "160), not librosa's resampler; and seeded synthetic signals.  mels: the notebook's get_mel cell (float64, "
                 "before .float()) with librosa 0.6.0's center=False STFT and Slaney mel basis restated."),
        "crosscheck": cc,
        "wavs": {k: torch.from_numpy(v) for k, v in sig.items()},
        "mels": mels,
        "subtraction": sub,
    }
    torch.save(out, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
