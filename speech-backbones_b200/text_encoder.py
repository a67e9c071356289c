"""Drop-in `TextEncoder` for Grad-TTS (replaces Grad-TTS/model/text_encoder.py:281-326 at inference time).

Same constructor, same parameter names and shapes (`emb`, `prenet.conv_layers.i`, `prenet.norm_layers.i.gamma/beta`,
`prenet.proj`, `encoder.attn_layers.i.{emb_rel_k, emb_rel_v, conv_q, conv_k, conv_v, conv_o}`, `encoder.norm_layers_{1,2}.i`,
`encoder.ffn_layers.i.conv_{1,2}`, `proj_m`, `proj_w.{conv_1, norm_1, conv_2, norm_2, proj}`), so
`GradTTS.load_state_dict(strict=True)` keeps working, and the same `forward(x, x_lengths, spk=None)` -> (mu, logw, x_mask)
called at tts.py:75.  The modules below are parameter containers; `forward` runs in libsbk.so (`sbk_textenc_forward`, exact
fp32 on CUDA cores, csrc/sbk_textenc.cu).  Inference only: there is no CPU path and no autograd through this module."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .binding import _check, _NativeHandle, _ptr
from .gradtts import BaseModule


class SbkTextEncConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("device", "n_vocab", "n_feats", "n_channels", "filter_channels", "filter_channels_dp",
                                         "n_heads", "n_layers", "kernel_size", "window_size", "n_spks", "spk_emb_dim", "kind")]


class _ChanNorm(BaseModule):                     # reference name: LayerNorm (text_encoder.py:11-29)
    def __init__(self, channels):
        super().__init__()
        self.gamma = nn.Parameter(torch.ones(channels))
        self.beta = nn.Parameter(torch.zeros(channels))


class _Prenet(BaseModule):                       # reference name: ConvReluNorm (:32-64)
    def __init__(self, ch, kernel_size=5, n_layers=3):
        super().__init__()
        self.conv_layers = nn.ModuleList([nn.Conv1d(ch, ch, kernel_size, padding=kernel_size // 2) for _ in range(n_layers)])
        self.norm_layers = nn.ModuleList([_ChanNorm(ch) for _ in range(n_layers)])
        self.proj = nn.Conv1d(ch, ch, 1)


class _RelAttention(BaseModule):                 # reference name: MultiHeadAttention (:96-215)
    def __init__(self, ch, n_heads, window_size):
        super().__init__()
        d = ch // n_heads
        self.conv_q, self.conv_k, self.conv_v, self.conv_o = (nn.Conv1d(ch, ch, 1) for _ in range(4))
        self.emb_rel_k = nn.Parameter(torch.randn(1, window_size * 2 + 1, d) * d ** -0.5)
        self.emb_rel_v = nn.Parameter(torch.randn(1, window_size * 2 + 1, d) * d ** -0.5)


class _FFN(BaseModule):                          # reference name: FFN (:218-237)
    def __init__(self, ch, filt, kernel_size):
        super().__init__()
        self.conv_1 = nn.Conv1d(ch, filt, kernel_size, padding=kernel_size // 2)
        self.conv_2 = nn.Conv1d(filt, ch, kernel_size, padding=kernel_size // 2)


class _Encoder(BaseModule):                      # reference name: Encoder (:240-278)
    def __init__(self, ch, filt, n_heads, n_layers, kernel_size, window_size):
        super().__init__()
        self.attn_layers = nn.ModuleList([_RelAttention(ch, n_heads, window_size) for _ in range(n_layers)])
        self.norm_layers_1 = nn.ModuleList([_ChanNorm(ch) for _ in range(n_layers)])
        self.ffn_layers = nn.ModuleList([_FFN(ch, filt, kernel_size) for _ in range(n_layers)])
        self.norm_layers_2 = nn.ModuleList([_ChanNorm(ch) for _ in range(n_layers)])


class _DurationPredictor(BaseModule):            # reference name: DurationPredictor (:67-93)
    def __init__(self, ch, filt, kernel_size):
        super().__init__()
        self.conv_1 = nn.Conv1d(ch, filt, kernel_size, padding=kernel_size // 2)
        self.norm_1 = _ChanNorm(filt)
        self.conv_2 = nn.Conv1d(filt, filt, kernel_size, padding=kernel_size // 2)
        self.norm_2 = _ChanNorm(filt)
        self.proj = nn.Conv1d(filt, 1, 1)


class TextEncEngine(_NativeHandle):
    """One sbk_textenc handle (the text encoder, kind 0, or the mel encoder, kind 1).  Its calls are not retried on out of
    memory."""
    PREFIX = "sbk_textenc"
    STATE_DICT = "the text-encoder state_dict"

    def __init__(self, m, device, kind=0):
        super().__init__()
        P, I = C.c_void_p, C.c_int
        self.lib.sbk_textenc_forward.argtypes = [P, P, P, P, P, P, P, I, I, P]
        self.lib.sbk_melenc_forward.argtypes = [P, P, P, P, I, I, P]
        cfg = SbkTextEncConfig(device, m.n_vocab, m.n_feats, m.n_channels, m.filter_channels, m.filter_channels_dp, m.n_heads,
                               m.n_layers, m.kernel_size, m.window_size, m.n_spks, m.spk_emb_dim, kind)
        _check(self._create(cfg), "sbk_textenc_create")
        self.device, self.n_feats, self.n_spks, self.spk_emb_dim = device, m.n_feats, m.n_spks, m.spk_emb_dim

    def forward(self, x, x_lengths, spk=None):
        for n, v in (("x", x), ("x_lengths", x_lengths), ("spk", spk)):
            if v is not None and (not v.is_cuda or v.device.index != self.device):
                raise RuntimeError(f"{n} lives on {v.device}; the text encoder runs only on cuda:{self.device} (no CPU path)")
        if x.dim() != 2 or x.dtype != torch.int64 or x_lengths.dtype != torch.int64 or tuple(x_lengths.shape) != (x.shape[0],):
            raise RuntimeError(f"expected x [B,Tx] int64 and x_lengths [B] int64, got {tuple(x.shape)} {x.dtype}, {tuple(x_lengths.shape)} {x_lengths.dtype}")
        B, Tx = x.shape
        if self.n_spks > 1:
            if spk is None or tuple(spk.shape) != (B, self.spk_emb_dim):
                raise RuntimeError(f"spk [B,{self.spk_emb_dim}] is required for a multi-speaker text encoder")
            spk = spk.to(torch.float32).contiguous()
        else:
            spk = None
        x, x_lengths = x.contiguous(), x_lengths.contiguous()
        mu = torch.empty((B, self.n_feats, Tx), dtype=torch.float32, device=x.device)
        logw = torch.empty((B, 1, Tx), dtype=torch.float32, device=x.device)
        mask = torch.empty((B, 1, Tx), dtype=torch.float32, device=x.device)
        with torch.cuda.device(x.device):
            _check(self.lib.sbk_textenc_forward(self.h, _ptr(x), _ptr(x_lengths), _ptr(spk), _ptr(mu), _ptr(logw), _ptr(mask),
                                                B, Tx, self._stream()), "sbk_textenc_forward")
        return mu, logw, mask

    def forward_mel(self, x, x_mask):
        for n, v in (("x", x), ("x_mask", x_mask)):
            if not v.is_cuda or v.device.index != self.device:
                raise RuntimeError(f"{n} lives on {v.device}; the mel encoder runs only on cuda:{self.device} (no CPU path)")
        B, Fm, T = x.shape
        if Fm != self.n_feats or tuple(x_mask.shape) != (B, 1, T) or x.dtype != torch.float32:
            raise RuntimeError(f"expected x [B,{self.n_feats},T] float32 and x_mask [B,1,T], got {tuple(x.shape)} {x.dtype}, {tuple(x_mask.shape)}")
        x, x_mask = x.contiguous(), x_mask.to(torch.float32).contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            _check(self.lib.sbk_melenc_forward(self.h, _ptr(x), _ptr(x_mask), _ptr(out), B, T, self._stream()), "sbk_melenc_forward")
        return out


class MelEncoder(BaseModule):
    """Drop-in for DiffVC's "average voice" encoder (DiffVC/model/encoder.py:257-284, built at DiffVC/model/vc.py:32 and
    called at :39,45 / :106,108): `MelEncoder(n_feats, channels, filters, heads, layers, kernel, dropout, window_size)`,
    the reference's state_dict (init_proj | prenet | encoder | term_proj, 6,841,232 parameters), `forward(x, x_mask)` in
    libsbk (`sbk_melenc_forward`: the text encoder's kernels, with a 1x1 projection at either end)."""

    def __init__(self, n_feats, channels, filters, heads, layers, kernel, dropout, window_size=None):
        super().__init__()
        if window_size is None:
            raise ValueError("the sm_90a mel encoder implements relative-position attention (DiffVC uses window_size=4)")
        self.n_feats, self.channels, self.filters, self.heads, self.layers = n_feats, channels, filters, heads, layers
        self.kernel, self.dropout, self.window_size = kernel, dropout, window_size
        # the engine reads the text encoder's attribute names
        self.n_vocab, self.n_channels, self.filter_channels, self.filter_channels_dp = 1, channels, filters, 4
        self.n_heads, self.n_layers, self.kernel_size, self.n_spks, self.spk_emb_dim = heads, layers, kernel, 1, 64
        self.init_proj = nn.Conv1d(n_feats, channels, 1)
        self.prenet = _Prenet(channels)
        self.encoder = _Encoder(channels, filters, heads, layers, kernel, window_size)
        self.term_proj = nn.Conv1d(channels, n_feats, 1)
        self._engine = None
        self._engine_sig = None

    def engine(self) -> TextEncEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the mel encoder runs only on a CUDA device (sm_90a); move the module with .cuda() first - "
                               "there is no CPU fallback")
        sig = (dev.index,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = TextEncEngine(self, dev.index, kind=1)
            self._engine_sig = None
        if sig != self._engine_sig:
            with torch.cuda.device(dev):
                self._engine.load_state_dict(self.state_dict())
            self._engine_sig = sig
        return self._engine

    @torch.no_grad()
    def forward(self, x, x_mask):
        return self.engine().forward_mel(x, x_mask)


class TextEncoder(BaseModule):
    def __init__(self, n_vocab, n_feats, n_channels, filter_channels, filter_channels_dp, n_heads, n_layers, kernel_size,
                 p_dropout, window_size=None, spk_emb_dim=64, n_spks=1):
        super().__init__()
        if window_size is None:
            raise ValueError("the sm_90a text encoder implements the relative-position attention Grad-TTS uses (window_size=4)")
        self.n_vocab, self.n_feats, self.n_channels = n_vocab, n_feats, n_channels
        self.filter_channels, self.filter_channels_dp = filter_channels, filter_channels_dp
        self.n_heads, self.n_layers, self.kernel_size = n_heads, n_layers, kernel_size
        self.p_dropout, self.window_size, self.spk_emb_dim, self.n_spks = p_dropout, window_size, spk_emb_dim, n_spks
        ce = n_channels + (spk_emb_dim if n_spks > 1 else 0)
        self.emb = nn.Embedding(n_vocab, n_channels)
        nn.init.normal_(self.emb.weight, 0.0, n_channels ** -0.5)
        self.prenet = _Prenet(n_channels)
        self.encoder = _Encoder(ce, filter_channels, n_heads, n_layers, kernel_size, window_size)
        self.proj_m = nn.Conv1d(ce, n_feats, 1)
        self.proj_w = _DurationPredictor(ce, filter_channels_dp, kernel_size)
        self._engine = None
        self._engine_sig = None

    def engine(self) -> TextEncEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the text encoder runs only on a CUDA device (sm_90a); move the module with .cuda() first - "
                               "there is no CPU fallback")
        sig = (dev.index,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = TextEncEngine(self, dev.index)
            self._engine_sig = None
        if sig != self._engine_sig:
            with torch.cuda.device(dev):
                self._engine.load_state_dict(self.state_dict())
            self._engine_sig = sig
        return self._engine

    @torch.no_grad()
    def forward(self, x, x_lengths, spk=None):
        return self.engine().forward(x, x_lengths, spk)
