"""Drop-in `Generator` for the HiFi-GAN vocoder (replaces Grad-TTS/hifi-gan/models.py:77-128 at inference time).

    from speech_backbones_b200.hifigan import Generator as HiFiGAN          # inference.py:26
    vocoder = HiFiGAN(h)                                                     # :60   (h = AttrDict of hifigan-config.json)
    vocoder.load_state_dict(torch.load(HIFIGAN_CHECKPT)['generator'])        # :61   weight-norm parametrised checkpoint
    _ = vocoder.cuda().eval()                                                # :62
    vocoder.remove_weight_norm()                                             # :63
    audio = vocoder.forward(y_dec)                                           # :81   mel [B,80,T] -> wav [B,1,256*T]

Same constructor argument, same parameter names (`conv_pre.weight_g/_v`, `ups.i.*`, `resblocks.n.convs{1,2}.j.*`, `conv_post.*`,
and the plain `.weight` names after `remove_weight_norm()`), so the reference checkpoint loads with `strict=True`.  The modules
below are parameter containers only: `forward` runs in libsbk.so (`sbk_vocoder_forward`: dilated Conv1d and the transposed
convs on wgmma, see csrc/sbk_vocoder.cu).  There is no CPU or eager-PyTorch path: calling `forward` with CPU tensors raises.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn
from torch.nn.utils import remove_weight_norm, weight_norm

from .binding import _check, _ptr, load_library


class SbkVocoderConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("num_mels", C.c_int32), ("upsample_initial_channel", C.c_int32), ("n_ups", C.c_int32),
                ("upsample_rates", C.c_int32 * 4), ("upsample_kernel_sizes", C.c_int32 * 4), ("n_kernels", C.c_int32),
                ("resblock_kernel_sizes", C.c_int32 * 3), ("resblock_dilations", (C.c_int32 * 3) * 3)]


def _get(h, k, default=None):
    return h.get(k, default) if isinstance(h, dict) else getattr(h, k, default)


def _padding(k, d=1):
    return (k * d - d) // 2                                   # xutils.get_padding


class _ResBlock1(nn.Module):                                   # reference name: ResBlock1 (models.py:13-49)
    def __init__(self, ch, k, dilations):
        super().__init__()
        self.convs1 = nn.ModuleList([weight_norm(nn.Conv1d(ch, ch, k, 1, dilation=d, padding=_padding(k, d))) for d in dilations])
        self.convs2 = nn.ModuleList([weight_norm(nn.Conv1d(ch, ch, k, 1, dilation=1, padding=_padding(k, 1))) for _ in dilations])

    def remove_weight_norm(self):
        for l in list(self.convs1) + list(self.convs2):
            remove_weight_norm(l)


class VocoderEngine:
    """One sbk_vocoder handle (device + packed weights + workspace)."""

    def __init__(self, h, device):
        self.lib = load_library()
        P, I = C.c_void_p, C.c_int
        self.lib.sbk_vocoder_create.argtypes = [C.POINTER(SbkVocoderConfig), C.POINTER(P)]
        self.lib.sbk_vocoder_destroy.argtypes = [P]
        self.lib.sbk_vocoder_destroy.restype = None
        self.lib.sbk_vocoder_num_weights.argtypes = [P]
        self.lib.sbk_vocoder_weight_name.argtypes = [P, I]
        self.lib.sbk_vocoder_weight_name.restype = C.c_char_p
        self.lib.sbk_vocoder_set_weight.argtypes = [P, C.c_char_p, P, C.POINTER(C.c_int64), I]
        self.lib.sbk_vocoder_pack.argtypes = [P]
        self.lib.sbk_vocoder_workspace_bytes.argtypes = [P, I, I]
        self.lib.sbk_vocoder_workspace_bytes.restype = C.c_size_t
        self.lib.sbk_vocoder_forward.argtypes = [P, P, P, I, I, P]
        self.lib.sbk_vocoder_last_launch_count.argtypes = [P]
        self.lib.sbk_vocoder_last_launch_count.restype = C.c_int64
        self.lib.sbk_vocoder_debug_capture.argtypes = [P, I]
        self.lib.sbk_vocoder_debug_num.argtypes = [P]
        self.lib.sbk_vocoder_debug_name.argtypes = [P, I]
        self.lib.sbk_vocoder_debug_name.restype = C.c_char_p
        self.lib.sbk_vocoder_debug_read.argtypes = [P, C.c_char_p, P, C.POINTER(C.c_int64)]
        rates, ks = list(_get(h, "upsample_rates")), list(_get(h, "upsample_kernel_sizes"))
        rk, rd = list(_get(h, "resblock_kernel_sizes")), [list(d) for d in _get(h, "resblock_dilation_sizes")]
        if str(_get(h, "resblock", "1")) != "1":
            raise RuntimeError("only ResBlock1 generators (HiFi-GAN V1/V2 configs, resblock='1') are supported")
        if len(rates) > 4 or len(rk) != 3 or any(len(d) != 3 for d in rd):
            raise RuntimeError("unsupported HiFi-GAN configuration (need <= 4 upsample stages, 3 resblock kernels x 3 dilations)")
        cfg = SbkVocoderConfig()
        cfg.device, cfg.num_mels = device, int(_get(h, "num_mels", 80))
        cfg.upsample_initial_channel, cfg.n_ups, cfg.n_kernels = int(_get(h, "upsample_initial_channel")), len(rates), len(rk)
        for i, (u, k) in enumerate(zip(rates, ks)):
            cfg.upsample_rates[i], cfg.upsample_kernel_sizes[i] = u, k
        for j in range(3):
            cfg.resblock_kernel_sizes[j] = rk[j]
            for d in range(3):
                cfg.resblock_dilations[j][d] = rd[j][d]
        self.h = C.c_void_p()
        _check(self.lib.sbk_vocoder_create(C.byref(cfg), C.byref(self.h)), "sbk_vocoder_create")
        self.device = device
        self.num_mels = cfg.num_mels
        self.rates = rates
        self.hop = 1
        for u in rates:
            self.hop *= u
        self._last_bt = None

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.sbk_vocoder_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def weight_names(self):
        return [self.lib.sbk_vocoder_weight_name(self.h, i).decode() for i in range(self.lib.sbk_vocoder_num_weights(self.h))]

    def load_state_dict(self, sd):
        """`sd`: effective weights (after remove_weight_norm), reference names."""
        for name in self.weight_names():
            if name not in sd:
                raise RuntimeError(f"missing key '{name}' in the vocoder state_dict (strict)")
            t = sd[name].detach().to(torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _check(self.lib.sbk_vocoder_set_weight(self.h, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                   f"sbk_vocoder_set_weight({name})")
        _check(self.lib.sbk_vocoder_pack(self.h), "sbk_vocoder_pack")

    def workspace_bytes(self, B, T):
        return int(self.lib.sbk_vocoder_workspace_bytes(self.h, B, T))

    def forward(self, mel):
        if not mel.is_cuda or mel.device.index != self.device:
            raise RuntimeError(f"mel lives on {mel.device}; the vocoder runs only on cuda:{self.device} (no CPU path)")
        if mel.dim() != 3 or mel.shape[1] != self.num_mels:
            raise RuntimeError(f"mel shape {tuple(mel.shape)}: expected [B, {self.num_mels}, T]")
        if mel.dtype != torch.float32:
            raise RuntimeError(f"mel: expected float32, got {mel.dtype}")
        mel = mel.contiguous()
        B, _, T = mel.shape
        wav = torch.empty((B, 1, T * self.hop), dtype=torch.float32, device=mel.device)
        with torch.cuda.device(mel.device):
            stream = C.c_void_p(torch.cuda.current_stream(mel.device).cuda_stream)
            rc = self.lib.sbk_vocoder_forward(self.h, _ptr(mel), _ptr(wav), B, T, stream)
            if rc != 0 and b"out of memory" in self.lib.sbk_last_error():
                torch.cuda.empty_cache()
                rc = self.lib.sbk_vocoder_forward(self.h, _ptr(mel), _ptr(wav), B, T, stream)
            _check(rc, "sbk_vocoder_forward")
        self._last_bt = (B, T)
        return wav

    def last_launch_count(self):
        return int(self.lib.sbk_vocoder_last_launch_count(self.h))

    # ---- test hooks: the intermediates of the last forward run with capture on (sbk_vocoder_debug_*)
    def debug_capture(self, on=True):
        _check(self.lib.sbk_vocoder_debug_capture(self.h, 1 if on else 0), "sbk_vocoder_debug_capture")

    def debug_names(self):
        return [self.lib.sbk_vocoder_debug_name(self.h, i).decode() for i in range(self.lib.sbk_vocoder_debug_num(self.h))]

    def _debug_len(self, name):
        """signal length of a captured tensor: T before the first transposed conv, times each rate after it"""
        B, T = self._last_bt
        parts = name.split(".")
        if parts[0] in ("mel_in", "conv_pre"):
            return T
        if parts[0] == "wav":
            return T * self.hop
        stage = int(parts[1]) // 3 if parts[0] == "resblocks" else int(parts[1])
        done = stage if (parts[0] == "ups" and parts[2] == "z") else stage + 1
        L = T
        for u in self.rates[:done]:
            L *= u
        return L

    def debug_read(self, name):
        """captured tensor `name` as a [B, C, L] fp32 CUDA tensor (wav: [B, 1, L])"""
        n = C.c_int64(0)
        _check(self.lib.sbk_vocoder_debug_read(self.h, name.encode(), None, C.byref(n)), "sbk_vocoder_debug_read")
        flat = torch.empty(n.value, dtype=torch.float32, device=f"cuda:{self.device}")
        _check(self.lib.sbk_vocoder_debug_read(self.h, name.encode(), _ptr(flat), C.byref(n)), "sbk_vocoder_debug_read")
        B, L = self._last_bt[0], self._debug_len(name)
        if name == "wav":
            return flat.view(B, 1, L)
        Ch = n.value // (B * L)
        return flat.view(B, Ch // 4, L, 4).permute(0, 1, 3, 2).reshape(B, Ch, L)


class Generator(nn.Module):
    """HiFi-GAN generator (models.py:77-128): parameter tree of the reference, forward in libsbk."""

    def __init__(self, h):
        super().__init__()
        self.h = h
        rates, ks = list(_get(h, "upsample_rates")), list(_get(h, "upsample_kernel_sizes"))
        rk, rd = list(_get(h, "resblock_kernel_sizes")), [list(d) for d in _get(h, "resblock_dilation_sizes")]
        c0 = int(_get(h, "upsample_initial_channel"))
        self.num_kernels, self.num_upsamples = len(rk), len(rates)
        self.conv_pre = weight_norm(nn.Conv1d(int(_get(h, "num_mels", 80)), c0, 7, 1, padding=3))
        self.ups = nn.ModuleList([weight_norm(nn.ConvTranspose1d(c0 // 2 ** i, c0 // 2 ** (i + 1), k, u, padding=(k - u) // 2))
                                  for i, (u, k) in enumerate(zip(rates, ks))])
        self.resblocks = nn.ModuleList()
        ch = c0
        for i in range(len(rates)):
            ch = c0 // 2 ** (i + 1)
            for k, d in zip(rk, rd):
                self.resblocks.append(_ResBlock1(ch, k, d))
        self.conv_post = weight_norm(nn.Conv1d(ch, 1, 7, 1, padding=3))
        self._engine = None
        self._engine_sig = None

    def remove_weight_norm(self):
        print('Removing weight norm...')
        for l in self.ups:
            remove_weight_norm(l)
        for l in self.resblocks:
            l.remove_weight_norm()
        remove_weight_norm(self.conv_pre)
        remove_weight_norm(self.conv_post)

    def effective_state_dict(self):
        """Reference names of the plain conv weights; with weight norm still attached w = g * v / ||v|| (dim 0)."""
        sd = self.state_dict()
        out = {}
        for k, v in sd.items():
            if k.endswith(".weight_v"):
                g = sd[k[:-2] + "_g"]
                norm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(g.shape)
                out[k[:-9] + ".weight"] = v * (g / norm)
            elif not k.endswith(".weight_g"):
                out[k] = v
        return out

    def engine(self) -> VocoderEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the HiFi-GAN generator runs only on a CUDA device (sm_90a); move the module with .cuda() "
                               "first - there is no CPU fallback")
        sig = (dev.index,) + tuple((n, p.data_ptr(), p._version) for n, p in self.named_parameters())
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = VocoderEngine(self.h, dev.index)
            self._engine_sig = None
        if sig != self._engine_sig:
            with torch.cuda.device(dev):
                self._engine.load_state_dict(self.effective_state_dict())
            self._engine_sig = sig
        return self._engine

    @torch.no_grad()
    def forward(self, x):
        return self.engine().forward(x)
