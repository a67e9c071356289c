"""DiffVC's inference front end on the GPU (DiffVC/inference.ipynb, cell 1): `LogMel` is the notebook's `get_mel` after the
waveform is decoded and resampled to 22050 Hz, `mel_spectral_subtraction` its post-processing of a converted mel.

Both run in libsbk.so (csrc/sbk_frontend.cu): the windowed DFT on wgmma in the fp32x3 split, the magnitude, the Slaney
filterbank and the log on CUDA cores, the spectral subtraction one CTA per utterance.  No CPU path.  Ragged batches: each row
is its own call, exact zeros past its frames, and `LogMel`'s `mel_lengths` is what `DiffVC.forward(..., ragged=True)` takes.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .binding import SbkFrontendConfig, _check, _ptr, check_lengths, load_library

HOP, MIN_SAMPLES, N_MELS = 256, 512, 80


class FrontendEngine:
    """One sbk_frontend handle: no weights; creating it and sizing its workspace are host logic (no GPU work)."""

    def __init__(self, device=0):
        self.lib = lib = load_library()
        self.h = C.c_void_p()
        _check(lib.sbk_frontend_create(C.byref(SbkFrontendConfig(device)), C.byref(self.h)), "sbk_frontend_create")
        self.device = device

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.sbk_frontend_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def dft_bins(self):
        return int(self.lib.sbk_frontend_dft_bins(self.h))

    def workspace_bytes(self, B, T):
        return int(self.lib.sbk_frontend_workspace_bytes(self.h, B, T))

    def last_launch_count(self):
        return int(self.lib.sbk_frontend_last_launch_count(self.h))

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _run(self, fn, what, *args):
        rc = fn(*args)
        if rc != 0 and b"out of memory" in self.lib.sbk_last_error():
            torch.cuda.empty_cache()
            rc = fn(*args)
        _check(rc, what)

    def logmel(self, wav, lengths=None):
        B, L = wav.shape
        mel_lengths = (lengths if lengths is not None else torch.full((B,), L, dtype=torch.int64, device=wav.device)) // HOP
        T = L // HOP if lengths is None else int(mel_lengths.max())
        out = torch.empty((B, N_MELS, T), dtype=torch.float32, device=wav.device)
        with torch.cuda.device(wav.device):
            self._run(self.lib.sbk_logmel_forward_lengths, "sbk_logmel_forward_lengths", self.h, _ptr(wav), _ptr(lengths),
                      _ptr(out), B, L, T, self._stream())
        return out, mel_lengths

    def spectral_subtraction(self, synth, source, lengths, spectral_floor, silence_window, smoothing_window):
        B, Fm, T = synth.shape
        out = torch.empty_like(synth)
        with torch.cuda.device(synth.device):
            self._run(self.lib.sbk_spectral_subtraction_lengths, "sbk_spectral_subtraction_lengths", self.h, _ptr(synth),
                      _ptr(source), _ptr(lengths), _ptr(out), B, Fm, T, float(spectral_floor), int(silence_window),
                      -1 if smoothing_window is None else int(smoothing_window), self._stream())
        return out


_engines: dict[int, FrontendEngine] = {}


def _engine(device) -> FrontendEngine:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _engines:
        _engines[idx] = FrontendEngine(idx)
    return _engines[idx]


def _check_cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise ValueError(f"{name}: expected a torch.Tensor, got {type(t).__name__}")
    if not t.is_cuda:
        raise ValueError(f"{name} lives on {t.device}; the front end runs only on a CUDA device (no CPU path)")


def check_wav(wav, lengths=None):
    """Validates a waveform batch before any launch; returns (wav contiguous, lengths contiguous or None)."""
    _check_cuda(wav, "wav")
    if wav.dim() != 2 or wav.dtype != torch.float32:
        raise ValueError(f"wav: expected float32 [B, L], got {wav.dtype} {tuple(wav.shape)}")
    B, L = wav.shape
    if B < 1:
        raise ValueError("wav: empty batch")
    if lengths is None:
        if L < MIN_SAMPLES:
            raise ValueError(f"an utterance needs at least {MIN_SAMPLES} samples (2 hops of {HOP}; the 384-sample reflection "
                             f"needs 385), got L = {L}")
        return wav.contiguous(), None
    _check_cuda(lengths, "lengths")
    lengths = check_lengths(lengths, B, L, wav.device, "wav")
    lo = int(lengths.min())
    if lo < MIN_SAMPLES:
        raise ValueError(f"an utterance needs at least {MIN_SAMPLES} samples (2 hops of {HOP}; the 384-sample reflection "
                         f"needs 385), got a length of {lo}")
    return wav.contiguous(), lengths


class LogMel(nn.Module):
    """The notebook's `get_mel` on decoded 22050 Hz waveforms: `forward(wav [B, L] float32, lengths=None)` ->
    `(log_mel [B, 80, T], mel_lengths [B])` with mel_lengths = lengths // 256 (L // 256 without lengths), T = max(mel_lengths),
    and exact zeros past each row's frames.  Row b equals `get_mel` on wav[b, :lengths[b]].  No parameters."""

    @torch.no_grad()
    def forward(self, wav, lengths=None):
        wav, lengths = check_wav(wav, lengths)
        return _engine(wav.device).logmel(wav, lengths)


@torch.no_grad()
def mel_spectral_subtraction(mel_synth, mel_source, spectral_floor=0.02, silence_window=5, smoothing_window=5, *,
                             lengths=None):
    """The notebook's `mel_spectral_subtraction` on [B, n_mels, T] float32 CUDA tensors, per utterance: row b is the function
    on its first lengths[b] frames (int64 [B]; None: all T) followed by exact zeros.  The notebook passes the converted mel
    as both arguments."""
    _check_cuda(mel_synth, "mel_synth")
    _check_cuda(mel_source, "mel_source")
    for n, t in (("mel_synth", mel_synth), ("mel_source", mel_source)):
        if t.dim() != 3 or t.dtype != torch.float32:
            raise ValueError(f"{n}: expected float32 [B, n_mels, T], got {t.dtype} {tuple(t.shape)}")
    if mel_synth.shape != mel_source.shape or mel_synth.device != mel_source.device:
        raise ValueError(f"mel_synth {tuple(mel_synth.shape)} on {mel_synth.device} and mel_source {tuple(mel_source.shape)} "
                         f"on {mel_source.device} must match")
    if int(silence_window) != silence_window or silence_window < 1:
        raise ValueError(f"silence_window must be a positive integer, got {silence_window!r}")
    if smoothing_window is not None and (int(smoothing_window) != smoothing_window or smoothing_window < 1):
        raise ValueError(f"smoothing_window must be None or a positive integer, got {smoothing_window!r}")
    B, Fm, T = mel_synth.shape
    if lengths is not None:
        _check_cuda(lengths, "lengths")
        lengths = check_lengths(lengths, B, T, mel_synth.device, "mel")
    return _engine(mel_synth.device).spectral_subtraction(mel_synth.contiguous(), mel_source.contiguous(), lengths,
                                                          spectral_floor, silence_window, smoothing_window)
