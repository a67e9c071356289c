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

from .binding import PREC, _check, _ptr, load_library
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


def _bind(lib):
    P, I = C.c_void_p, C.c_int
    lib.sbk_postnet_create.argtypes = [C.POINTER(SbkPostNetConfig), C.POINTER(P)]
    lib.sbk_postnet_destroy.argtypes = [P]
    lib.sbk_postnet_destroy.restype = None
    lib.sbk_postnet_num_weights.argtypes = [P]
    lib.sbk_postnet_weight_name.argtypes = [P, I]
    lib.sbk_postnet_weight_name.restype = C.c_char_p
    lib.sbk_postnet_set_weight.argtypes = [P, C.c_char_p, P, C.POINTER(C.c_int64), I]
    lib.sbk_postnet_pack.argtypes = [P]
    lib.sbk_postnet_workspace_bytes.argtypes = [P, I, I, I]
    lib.sbk_postnet_workspace_bytes.restype = C.c_size_t
    lib.sbk_postnet_forward.argtypes = [P, P, P, P, I, I, I, P]
    lib.sbk_postnet_last_launch_count.argtypes = [P]
    lib.sbk_postnet_last_launch_count.restype = C.c_int64
    return lib


class PostNetEngine:
    """One sbk_postnet handle.  Creating it is host logic (no GPU work): the weight inventory can be queried anywhere."""

    def __init__(self, dim, groups=8, device=0, precision="fp32x3"):
        self.lib = _bind(load_library())
        cfg = SbkPostNetConfig(device, dim, groups, PREC[precision])
        self.h = C.c_void_p()
        rc = self.lib.sbk_postnet_create(C.byref(cfg), C.byref(self.h))
        if rc == _SBK_ERR_UNSUPPORTED:
            raise ValueError(self.lib.sbk_last_error().decode())
        _check(rc, "sbk_postnet_create")
        self.device, self.dim = device, dim

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.lib.sbk_postnet_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def weight_names(self):
        return [self.lib.sbk_postnet_weight_name(self.h, i).decode() for i in range(self.lib.sbk_postnet_num_weights(self.h))]

    def load_state_dict(self, sd):
        for name in self.weight_names():
            if name not in sd:
                raise RuntimeError(f"missing key '{name}' in the PostNet state_dict (strict)")
            t = sd[name].detach().to(torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _check(self.lib.sbk_postnet_set_weight(self.h, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                   f"sbk_postnet_set_weight({name})")
        _check(self.lib.sbk_postnet_pack(self.h), "sbk_postnet_pack")

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
            stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
            args = (self.h, _ptr(x), _ptr(mask), _ptr(out), B, Fm, T, stream)
            rc = self.lib.sbk_postnet_forward(*args)
            if rc != 0 and b"out of memory" in self.lib.sbk_last_error():
                torch.cuda.empty_cache()          # the workspace is raw cudaMalloc, outside torch's caching allocator
                rc = self.lib.sbk_postnet_forward(*args)
            _check(rc, "sbk_postnet_forward")
        return out

    def last_launch_count(self):
        return int(self.lib.sbk_postnet_last_launch_count(self.h))


class PostNet(BaseModule):
    def __init__(self, dim, groups=8, *, precision="fp32x3"):
        super().__init__()
        if precision not in PREC:
            raise ValueError(f"precision must be one of {sorted(PREC)}, got {precision!r}")
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
