"""Drop-in `PostNet` for DiffVC (replaces DiffVC/model/postnet.py:40-53, built at DiffVC/model/vc.py:34).

Same constructor `PostNet(dim, groups=8)`, the same submodule tree (`init_conv`, `res_block.block{1,2}.block.{0,1}`,
`res_block.res`, `final_conv`: 14 tensors, 1,623,297 parameters at dim = 128), so `FwdDiffusion` / `DiffVC` checkpoints load
unchanged, and the same `forward(x, mask)` -> [B, n_feats, T].  The modules below are parameter containers; `forward` runs in
libsbk.so (`sbk_postnet_forward`: the two 7x7 convs on wgmma, csrc/sbk_postnet.cu).  Inference only: there is no CPU path
and no autograd through this module.

`precision`: "fp32x3" (default; "fp32" maps to it) runs the fp32-class tf32 + fp16-correction split, "tf32" ("bf16" maps to
it) plain tf32 operands.  The mapping lives in the library (sbk_postnet.cu)."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from .binding import PREC, _check, _check_precision, _NativeHandle, _ptr
from .gradtts import BaseModule, Mish


_SBK_ERR_UNSUPPORTED = 4


class SbkPostNetConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("device", "dim", "groups", "precision")]


class _Block(BaseModule):                        # reference name: Block (postnet.py:15-23)
    def __init__(self, dim, groups=8):
        super().__init__()
        self.block = nn.Sequential(nn.Conv2d(dim, dim, 7, padding=3), nn.GroupNorm(groups, dim), Mish())


class _ResnetBlock(BaseModule):                  # reference name: ResnetBlock (:26-37)
    def __init__(self, dim, groups=8):
        super().__init__()
        self.block1 = _Block(dim, groups=groups)
        self.block2 = _Block(dim, groups=groups)
        self.res = nn.Conv2d(dim, dim, 1)


class PostNetEngine(_NativeHandle):
    """One sbk_postnet handle.  Creating it is host logic (no GPU work): the weight inventory can be queried anywhere."""
    PREFIX = "sbk_postnet"
    STATE_DICT = "the PostNet state_dict"

    def __init__(self, dim, groups=8, device=0, precision="fp32x3"):
        super().__init__()
        P, I = C.c_void_p, C.c_int
        self.lib.sbk_postnet_workspace_bytes.argtypes = [P, I, I, I]
        self.lib.sbk_postnet_workspace_bytes.restype = C.c_size_t
        self.lib.sbk_postnet_forward.argtypes = [P, P, P, P, I, I, I, P]
        rc = self._create(SbkPostNetConfig(device, dim, groups, PREC[precision]))
        if rc == _SBK_ERR_UNSUPPORTED:
            raise ValueError(self.lib.sbk_last_error().decode())
        _check(rc, "sbk_postnet_create")
        self.device, self.dim = device, dim

    def forward(self, x, mask):
        for n, v in (("x", x), ("mask", mask)):
            if not v.is_cuda or v.device.index != self.device:
                raise RuntimeError(f"{n} lives on {v.device}; the PostNet runs only on cuda:{self.device} (no CPU path)")
        if x.dim() != 3 or x.dtype != torch.float32:
            raise RuntimeError(f"expected x [B,n_feats,T] float32, got {tuple(x.shape)} {x.dtype}")
        B, Fm, T = x.shape
        if tuple(mask.shape) != (B, 1, T):
            raise RuntimeError(f"expected mask [B,1,T] = {(B, 1, T)}, got {tuple(mask.shape)}")
        x, mask = x.contiguous(), mask.to(torch.float32).contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            self._call(self.lib.sbk_postnet_forward, "sbk_postnet_forward", self.h, _ptr(x), _ptr(mask), _ptr(out), B, Fm, T,
                       self._stream())
        return out


class PostNet(BaseModule):
    def __init__(self, dim, groups=8, *, precision="fp32x3"):
        super().__init__()
        _check_precision(precision)
        PostNetEngine(dim, groups, precision=precision).close()     # the library's config check (host logic): ValueError
        self.dim, self.groups, self.precision = dim, groups, precision
        self.init_conv = nn.Conv2d(1, dim, 1)
        self.res_block = _ResnetBlock(dim, groups=groups)
        self.final_conv = nn.Conv2d(dim, 1, 1)
        self._engine = None
        self._engine_sig = None

    def engine(self) -> PostNetEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("the PostNet runs only on a CUDA device (sm_90a); move the module with .cuda() first - "
                               "there is no CPU fallback")
        sig = (dev.index,) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = PostNetEngine(self.dim, self.groups, dev.index, self.precision)
            self._engine_sig = None
        if sig != self._engine_sig:
            with torch.cuda.device(dev):
                self._engine.load_state_dict(self.state_dict())
            self._engine_sig = sig
        return self._engine

    @torch.no_grad()
    def forward(self, x, mask):
        return self.engine().forward(x, mask)
