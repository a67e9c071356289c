"""Float64 restatement of DiffVC's inference front end (DiffVC/inference.ipynb, cell 1), per utterance.

`get_mel(wav)` is the notebook's `get_mel` after `librosa.load`: truncate to whole 256-sample hops, reflect-pad 384 samples,
Hann-windowed (periodic) 1024-point STFT with `center=False`, hop 256, `sqrt(re^2 + im^2 + 1e-9)`, the Slaney mel basis of
`librosa.filters.mel(22050, 1024, 80, 0, 8000)` (librosa 0.6.0: `norm=1`, float64), `log(clip(., 1e-5))`.  Everything runs
in float64 here; the notebook stores the STFT as complex64 and squares it in float32.

`mel_spectral_subtraction` and `noise_median_smoothing` restate the notebook's functions in float64, edge rules included.
`mel_spectral_subtraction(..., return_window=True)` also returns the chosen window's first frame and the window energies.
"""
from __future__ import annotations

import numpy as np

SR, N_FFT, HOP, N_MELS, FMIN, FMAX = 22050, 1024, 256, 80, 0.0, 8000.0
PAD = (N_FFT - HOP) // 2          # 384


def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-300) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr=SR, n_fft=N_FFT, n_mels=N_MELS, fmin=FMIN, fmax=FMAX):
    """librosa.filters.mel (0.6.0, htk=False, norm=1) in float64: [n_mels, 1 + n_fft // 2]."""
    fftfreqs = np.linspace(0, float(sr) / 2, int(1 + n_fft // 2), endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, int(1 + n_fft // 2)))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    return weights * enorm[:, None]


def hann(n=N_FFT):
    """scipy.signal.get_window('hann', n, fftbins=True): the periodic window"""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(n) / n)


def frames(wav):
    """[T, 1024] float64 frames of one utterance: truncated to whole hops, reflect-padded by 384 samples"""
    wav = np.asarray(wav, dtype=np.float64)
    wav = wav[:(wav.shape[0] // HOP) * HOP]
    if wav.shape[0] < 2 * HOP:
        raise ValueError(f"an utterance needs at least {2 * HOP} samples (the {PAD}-sample reflection needs {PAD + 1}), "
                         f"got {wav.shape[0]}")
    p = np.pad(wav, PAD, mode="reflect")
    T = 1 + (p.shape[0] - N_FFT) // HOP
    idx = np.arange(T)[:, None] * HOP + np.arange(N_FFT)[None, :]
    return p[idx]


def stft(wav, bins=N_FFT // 2 + 1):
    """complex128 [bins, T]: the windowed rfft of every frame"""
    return np.fft.rfft(frames(wav) * hann()[None, :], axis=1)[:, :bins].T


def get_mel(wav, basis=None):
    """[80, T] float64 log-mel of one utterance (wav: its samples at 22050 Hz)"""
    basis = mel_basis() if basis is None else basis
    X = stft(wav)
    mag = np.sqrt(X.real ** 2 + X.imag ** 2 + 1e-9)
    return np.log(np.clip(basis @ mag, 1e-5, None))


def noise_median_smoothing(x, w=5):
    x = np.asarray(x, dtype=np.float64)
    y = np.copy(x)
    xp = np.pad(x, w, "edge")
    for i in range(y.shape[0]):
        y[i] = min(xp[i + w + 1], np.median(xp[i:i + 2 * w + 1]))
    return y


def window_energies(mel_source, silence_window=5):
    """float64 energy of every candidate window i < T - silence_window"""
    e = np.exp(2.0 * np.asarray(mel_source, dtype=np.float64))
    return np.array([e[:, i:i + silence_window].sum() for i in range(e.shape[-1] - silence_window)])


def mel_spectral_subtraction(mel_synth, mel_source, spectral_floor=0.02, silence_window=5, smoothing_window=5,
                             return_window=False):
    synth = np.asarray(mel_synth, dtype=np.float64)
    energies = window_energies(mel_source, silence_window)
    energy_min, i_min = 100000.0, 0
    for i, e in enumerate(energies):
        if e < energy_min:
            i_min, energy_min = i, e
    noise = np.min(np.exp(2.0 * synth[:, i_min:i_min + silence_window]), axis=-1)
    if smoothing_window is not None:
        noise = noise_median_smoothing(noise, smoothing_window)
    sig = np.exp(2.0 * synth) - noise[:, None]
    with np.errstate(divide="ignore"):
        out = np.log(np.sqrt(np.maximum(sig, spectral_floor * noise[:, None])))
    return (out, i_min, energies) if return_window else out


def get_mel_batch(wav, lengths=None):
    """[B, 80, T] float64 with T = max(lengths // 256) and zeros past each row's frames; wav [B, L]"""
    wav = np.asarray(wav, dtype=np.float64)
    B, L = wav.shape
    lengths = [L] * B if lengths is None else [int(v) for v in lengths]
    mels = [get_mel(wav[b, :lengths[b]]) for b in range(B)]
    T = max(m.shape[1] for m in mels)
    out = np.zeros((B, N_MELS, T))
    for b, m in enumerate(mels):
        out[b, :, :m.shape[1]] = m
    return out
