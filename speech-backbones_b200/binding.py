"""ctypes binding of libsbk.so (include/sbk.h).  No CPU fallback: if the library is missing or
the call fails, a RuntimeError is raised."""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsbk.so")

PREC = {"fp32": 0, "tf32": 1, "bf16": 2, "fp32x3": 3}
MODEL = {"gradtts": 0, "diffvc": 1}

EXPORTS = [
    "sbk_create", "sbk_destroy", "sbk_set_weight", "sbk_pack", "sbk_num_weights", "sbk_weight_name",
    "sbk_workspace_bytes", "sbk_estimator", "sbk_reverse_diffusion", "sbk_reverse_steps",
    "sbk_reverse_diffusion_host", "sbk_last_launch_count", "sbk_debug_read", "sbk_debug_num",
    "sbk_debug_name", "sbk_last_error", "sbk_version", "sbk_profile_ops", "sbk_debug_capture", "sbk_debug_layout", "sbk_debug_op_layout", "sbk_vc_estimator", "sbk_vc_reverse_diffusion", "sbk_vc_conditioning",
    "sbk_prior_expand", "sbk_last_host_launches", "sbk_workspace_bytes_n",
    "sbk_vc_cond_debug_num", "sbk_vc_cond_debug_name", "sbk_vc_cond_debug_op_layout", "sbk_vc_cond_debug_read",
]


class SbkConfig(C.Structure):
    _fields_ = [("model", C.c_int32), ("n_feats", C.c_int32), ("dim", C.c_int32), ("n_spks", C.c_int32),
                ("spk_emb_dim", C.c_int32), ("beta_min", C.c_float), ("beta_max", C.c_float),
                ("pe_scale", C.c_float), ("device", C.c_int32), ("precision", C.c_int32),
                ("use_graph", C.c_int32), ("dim_cond", C.c_int32), ("use_ref_t", C.c_int32)]


_lib = None


def load_library() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
                           "There is no CPU fallback for the sampler.")
    lib = C.CDLL(LIB_PATH)
    P, I, F = C.c_void_p, C.c_int, C.c_void_p
    lib.sbk_workspace_bytes.argtypes = [P, I, I]
    lib.sbk_workspace_bytes.restype = C.c_size_t
    lib.sbk_workspace_bytes_n.argtypes = [P, I, I, I]
    lib.sbk_workspace_bytes_n.restype = C.c_size_t
    lib.sbk_estimator.argtypes = [P, F, F, F, F, F, F, I, I, P]
    lib.sbk_reverse_diffusion.argtypes = [P, F, F, F, F, F, F, I, I, I, I, P]
    lib.sbk_vc_estimator.argtypes = [P, F, F, F, F, F, F, I, I, P]
    lib.sbk_vc_reverse_diffusion.argtypes = [P, F, F, F, F, F, F, I, I, I, I, P]
    lib.sbk_vc_conditioning.argtypes = [P, F, F, F, F, F, I, I, I, P]
    lib.sbk_reverse_steps.argtypes = [P, F, F, F, F, F, I, I, I, I, I, I, P]
    lib.sbk_reverse_diffusion_host.argtypes = [P, F, F, F, F, F, F, I, I, I, I]
    lib.sbk_prior_expand.argtypes = [F, F, F, F, F, C.c_float, I, I, I, I, F, F, F, F, P]
    lib.sbk_last_host_launches.argtypes = [P]
    lib.sbk_debug_read.argtypes = [P, C.c_char_p, F, C.POINTER(C.c_int64)]
    lib.sbk_debug_num.argtypes = [P]
    lib.sbk_debug_capture.argtypes = [P, I]
    lib.sbk_debug_layout.argtypes = [P]
    lib.sbk_debug_op_layout.argtypes = [P, C.c_char_p]
    lib.sbk_debug_name.argtypes = [P, I]
    lib.sbk_debug_name.restype = C.c_char_p
    lib.sbk_vc_cond_debug_num.argtypes = [P]
    lib.sbk_vc_cond_debug_name.argtypes = [P, I]
    lib.sbk_vc_cond_debug_name.restype = C.c_char_p
    lib.sbk_vc_cond_debug_op_layout.argtypes = [P, C.c_char_p]
    lib.sbk_vc_cond_debug_read.argtypes = [P, C.c_char_p, F, C.POINTER(C.c_int64)]
    lib.sbk_profile_ops.argtypes = [P, F, F, F, I, C.POINTER(C.c_int)]
    lib.sbk_last_error.restype = C.c_char_p
    lib.sbk_version.restype = C.c_char_p
    _lib = lib
    return lib


def _check(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"{what} failed (code {rc}): {load_library().sbk_last_error().decode()}")


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _check_precision(precision):
    if precision not in PREC:
        raise ValueError(f"precision must be one of {sorted(PREC)}, got {precision!r}")
    return precision


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name}: expected float32, got {t.dtype}")
    return t.contiguous()


def prior_expand(mu_x, w_ceil, x_mask, y_lengths, Ty, noise_tf=None, temperature=1.0, want_attn=True):
    """sbk_prior_expand (GradTTS.forward, tts.py:82-94): alignment path, aligned prior mu_y, terminal sample z, y_mask.
    mu_x [B,F,Tx], w_ceil / x_mask [B,Tx] fp32, y_lengths [B] int64, noise_tf [B,Ty,F] or None; all CUDA tensors.
    Returns (mu_y [B,F,Ty], z [B,F,Ty], y_mask [B,1,Ty], attn [B,1,Tx,Ty] or None)."""
    lib = load_library()
    for n, t in (("mu_x", mu_x), ("w_ceil", w_ceil), ("x_mask", x_mask), ("y_lengths", y_lengths)):
        if not t.is_cuda:
            raise RuntimeError(f"{n} must be a CUDA tensor: the glue kernel has no CPU path")
    B, Fm, Tx = mu_x.shape
    mu_x, w_ceil, x_mask = _f32c(mu_x, "mu_x"), _f32c(w_ceil, "w_ceil"), _f32c(x_mask, "x_mask")
    if tuple(w_ceil.shape) != (B, Tx) or tuple(x_mask.shape) != (B, Tx) or tuple(y_lengths.shape) != (B,):
        raise RuntimeError(f"shape mismatch: mu_x {tuple(mu_x.shape)}, w_ceil {tuple(w_ceil.shape)}, x_mask {tuple(x_mask.shape)}, "
                           f"y_lengths {tuple(y_lengths.shape)}")
    if y_lengths.dtype != torch.int64:
        raise RuntimeError(f"y_lengths: expected int64, got {y_lengths.dtype}")
    y_lengths = y_lengths.contiguous()
    if noise_tf is not None:
        noise_tf = _f32c(noise_tf, "noise_tf")
        if tuple(noise_tf.shape) != (B, Ty, Fm):
            raise RuntimeError(f"noise_tf shape {tuple(noise_tf.shape)} != {(B, Ty, Fm)} (memory order of randn_like(mu_y))")
    dev = mu_x.device
    mu_y = torch.empty((B, Fm, Ty), dtype=torch.float32, device=dev)
    z = torch.empty_like(mu_y)
    y_mask = torch.empty((B, 1, Ty), dtype=torch.float32, device=dev)
    attn = torch.empty((B, 1, Tx, Ty), dtype=torch.float32, device=dev) if want_attn else None
    with torch.cuda.device(dev):
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _check(lib.sbk_prior_expand(_ptr(mu_x), _ptr(w_ceil), _ptr(x_mask), _ptr(y_lengths), _ptr(noise_tf),
                                    C.c_float(float(temperature)), B, Fm, Tx, int(Ty), _ptr(mu_y), _ptr(z), _ptr(y_mask),
                                    _ptr(attn), stream), "sbk_prior_expand")
    return mu_y, z, y_mask, attn


class _NativeHandle:
    """One libsbk handle of the C prefix PREFIX ("sbk", "sbk_vocoder", "sbk_postnet", "sbk_textenc"): the entry points every
    engine shares - create / destroy, the strict weight inventory and loader, the launch count - declared once here."""
    PREFIX = "sbk"
    STATE_DICT = "state_dict"           # how load_state_dict's missing-key error names the state dict

    def __init__(self):
        self.lib = load_library()
        P, I = C.c_void_p, C.c_int
        self._fn("destroy").argtypes = [P]
        self._fn("destroy").restype = None
        self._fn("num_weights").argtypes = [P]
        self._fn("weight_name").argtypes = [P, I]
        self._fn("weight_name").restype = C.c_char_p
        self._fn("set_weight").argtypes = [P, C.c_char_p, P, C.POINTER(C.c_int64), I]
        self._fn("pack").argtypes = [P]
        self._fn("last_launch_count").argtypes = [P]
        self._fn("last_launch_count").restype = C.c_int64
        self.h = C.c_void_p()

    def _fn(self, name):
        return getattr(self.lib, f"{self.PREFIX}_{name}")

    def _create(self, cfg):
        """<prefix>_create(&cfg, &h); returns its status code"""
        create = self._fn("create")
        create.argtypes = [C.POINTER(type(cfg)), C.POINTER(C.c_void_p)]
        return create(C.byref(cfg), C.byref(self.h))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self._fn("destroy")(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def weight_names(self):
        return [self._fn("weight_name")(self.h, i).decode() for i in range(self._fn("num_weights")(self.h))]

    def load_state_dict(self, sd, prefix=""):
        """`sd` maps reference names (optionally under `prefix`, e.g. 'decoder.') to tensors (CPU or CUDA)."""
        for name in self.weight_names():
            key = prefix + name
            if key not in sd:
                raise RuntimeError(f"missing key '{key}' in {self.STATE_DICT} (strict)")
            t = sd[key].detach().to(torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _check(self._fn("set_weight")(self.h, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                   f"{self.PREFIX}_set_weight({name})")
        _check(self._fn("pack")(self.h), f"{self.PREFIX}_pack")

    def _call(self, fn, what, *args):
        """One libsbk call; if its workspace allocation ran out of memory while torch holds cached blocks (the workspace
        is raw cudaMalloc, outside torch's caching allocator), release them and retry once."""
        rc = fn(*args)
        if rc != 0 and b"out of memory" in self.lib.sbk_last_error():
            torch.cuda.empty_cache()
            rc = fn(*args)
        _check(rc, what)

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def last_launch_count(self):
        return int(self._fn("last_launch_count")(self.h))


class Engine(_NativeHandle):
    """One sbk_handle: a (device, configuration) pair owning packed weights, workspace and graphs.  load_state_dict is the
    strict loading of Grad-TTS/inference.py:53."""

    def __init__(self, n_feats=80, dim=64, n_spks=1, spk_emb_dim=64, beta_min=0.05, beta_max=20.0,
                 pe_scale=1000.0, device=0, precision="fp32x3", use_graph=True, model="gradtts", dim_cond=0,
                 use_ref_t=True):
        super().__init__()
        self.cfg = SbkConfig(MODEL[model], n_feats, dim, n_spks, spk_emb_dim, beta_min, beta_max, pe_scale,
                             device, PREC[precision], 1 if use_graph else 0, dim_cond, 1 if use_ref_t else 0)
        self.model = model
        self.dim_cond = dim_cond
        _check(self._create(self.cfg), "sbk_create")
        self.device = device
        self.n_feats = n_feats
        self.n_spks = n_spks
        self.spk_emb_dim = spk_emb_dim

    def workspace_bytes(self, B, T, n_timesteps=1024):
        return int(self.lib.sbk_workspace_bytes_n(self.h, B, T, int(n_timesteps)))

    def _check_inputs(self, x, mask, mu, spk, t=None):
        for n, v in (("x", x), ("mask", mask), ("mu", mu)):
            if not v.is_cuda:
                raise RuntimeError(f"{n} must be a CUDA tensor: the sampler has no CPU path")
        B, F, T = x.shape
        if F != self.n_feats or mu.shape != x.shape or mask.shape != (B, 1, T):
            raise RuntimeError(f"shape mismatch: x {tuple(x.shape)}, mu {tuple(mu.shape)}, mask {tuple(mask.shape)}")
        if self.n_spks > 1 and spk is None:
            raise RuntimeError("spk embedding required for a multi-speaker model")
        # libsbk reads raw pointers on ITS device and stream: a short t / spk would be an out-of-bounds device read and a
        # tensor on another GPU would be consumed through a peer pointer - the reference raises on both, so does this
        for n, v in (("x", x), ("mask", mask), ("mu", mu), ("spk", spk), ("t", t)):
            if v is not None and (not v.is_cuda or v.device.index != self.device):
                raise RuntimeError(f"{n} lives on {v.device}, this engine on cuda:{self.device}")
        if t is not None and tuple(t.shape) != (B,):
            raise RuntimeError(f"t shape {tuple(t.shape)} != {(B,)}")
        if self.n_spks > 1 and tuple(spk.shape) != (B, self.spk_emb_dim):
            raise RuntimeError(f"spk shape {tuple(spk.shape)} != {(B, self.spk_emb_dim)}")
        return B, T

    def estimator(self, x, mask, mu, t, spk=None):
        B, T = self._check_inputs(x, mask, mu, spk, t)
        x, mask, mu, t = _f32c(x, "x"), _f32c(mask, "mask"), _f32c(mu, "mu"), _f32c(t, "t")
        spk = _f32c(spk, "spk") if (spk is not None and self.n_spks > 1) else None
        out = torch.empty_like(x)
        self._call(self.lib.sbk_estimator, "sbk_estimator", self.h, _ptr(x), _ptr(mask), _ptr(mu), _ptr(t), _ptr(spk), _ptr(out),
                   B, T, self._stream())
        return out

    # ---- oversize batches: utterances are independent, so a batch whose workspace would not fit is run in slices
    max_workspace_bytes = None      # default: 60 % of the device memory

    def batch_slices(self, B, T, n_timesteps=1024):
        limit = self.max_workspace_bytes
        if limit is None:
            limit = 0.6 * torch.cuda.get_device_properties(self.device).total_memory
        need = self.workspace_bytes(B, T, n_timesteps)
        if need <= limit or B == 1:
            return [(0, B)]
        per = need / B
        chunk = max(1, int(limit // per))
        return [(lo, min(B, lo + chunk)) for lo in range(0, B, chunk)]

    def reverse_diffusion(self, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None):
        B, T = self._check_inputs(z, mask, mu, spk)
        sl = self.batch_slices(B, T, n_timesteps)
        if len(sl) > 1:
            outs = [self.reverse_diffusion(z[a:b], mask[a:b], mu[a:b], n_timesteps, stoc,
                                           None if spk is None else spk[a:b],
                                           None if noise is None else noise[:, a:b].contiguous()) for a, b in sl]
            return torch.cat(outs, 0)
        z, mask, mu = _f32c(z, "z"), _f32c(mask, "mask"), _f32c(mu, "mu")
        spk = _f32c(spk, "spk") if (spk is not None and self.n_spks > 1) else None
        if stoc:
            if noise is None:
                raise RuntimeError("stoc=True needs pre-drawn noise [N,B,n_feats,T]")
            noise = _f32c(noise, "noise")
            if tuple(noise.shape) != (n_timesteps, B, self.n_feats, T):
                raise RuntimeError(f"noise shape {tuple(noise.shape)} != {(n_timesteps, B, self.n_feats, T)}")
        out = torch.empty_like(z)
        self._call(self.lib.sbk_reverse_diffusion, "sbk_reverse_diffusion", self.h, _ptr(z), _ptr(mask), _ptr(mu), _ptr(spk),
                   _ptr(noise) if stoc else None, _ptr(out), B, T, int(n_timesteps), 1 if stoc else 0, self._stream())
        return out

    def reverse_steps(self, xt, mask, mu, n_timesteps, step_begin, step_end, stoc=False, spk=None, noise=None):
        B, T = self._check_inputs(xt, mask, mu, spk)
        assert xt.is_contiguous() and xt.dtype == torch.float32
        mask, mu = _f32c(mask, "mask"), _f32c(mu, "mu")
        spk = _f32c(spk, "spk") if (spk is not None and self.n_spks > 1) else None
        noise = _f32c(noise, "noise") if stoc else None
        _check(self.lib.sbk_reverse_steps(self.h, _ptr(xt), _ptr(mask), _ptr(mu), _ptr(spk), _ptr(noise), B, T,
                                          int(n_timesteps), int(step_begin), int(step_end), 1 if stoc else 0,
                                          self._stream()), "sbk_reverse_steps")
        return xt

    # ---- DiffVC (model="diffvc")
    VC_MODES = {"pf": 0, "em": 1, "ml": 2}

    def vc_estimator(self, x, mask, mean, cond, t):
        B, T = self._check_inputs(x, mask, mean, None, t)
        x, mask, mean, cond, t = (_f32c(v, n) for v, n in ((x, "x"), (mask, "mask"), (mean, "mean"), (cond, "cond"), (t, "t")))
        if tuple(cond.shape) != (B, self.dim_cond):
            raise RuntimeError(f"cond shape {tuple(cond.shape)} != {(B, self.dim_cond)}")
        out = torch.empty_like(x)
        _check(self.lib.sbk_vc_estimator(self.h, _ptr(x), _ptr(mask), _ptr(mean), _ptr(cond), _ptr(t), _ptr(out), B, T,
                                         self._stream()), "sbk_vc_estimator")
        return out

    def vc_conditioning(self, ref, ref_mask, mean_ref, c, n_timesteps):
        """Native hoisted conditioning branch (tensor-core modes): cond [N, B, dim_cond] for t_i = 1 - i/N."""
        for n, t in (("ref", ref), ("ref_mask", ref_mask), ("mean_ref", mean_ref), ("c", c)):
            if not t.is_cuda:
                raise RuntimeError(f"{n} must be a CUDA tensor: the sampler has no CPU path")
        B, Fm, Tr = ref.shape
        ref, ref_mask, mean_ref, c = _f32c(ref, "ref"), _f32c(ref_mask, "ref_mask"), _f32c(mean_ref, "mean_ref"), _f32c(c, "c")
        if Fm != self.n_feats or mean_ref.shape != ref.shape or ref_mask.shape != (B, 1, Tr) or tuple(c.shape) != (B, 256):
            raise RuntimeError("shape mismatch in vc_conditioning inputs")
        out = torch.empty((n_timesteps, B, self.dim_cond), dtype=torch.float32, device=ref.device)
        _check(self.lib.sbk_vc_conditioning(self.h, _ptr(ref), _ptr(ref_mask), _ptr(mean_ref), _ptr(c), _ptr(out), B, Tr,
                                            int(n_timesteps), self._stream()), "sbk_vc_conditioning")
        self._vc_shape = (B, Tr)
        return out

    def vc_cond_debug_names(self):
        """Tensors the last vc_conditioning call captured (debug_capture on), in launch order; they hold its last step."""
        return [self.lib.sbk_vc_cond_debug_name(self.h, i).decode() for i in range(self.lib.sbk_vc_cond_debug_num(self.h))]

    def vc_cond_debug_read(self, name):
        """One captured RefBlock tensor as a CPU float64 tensor: conv-shaped ones ([B][H][C/4][Tr][4] in the kernels) as NCHW
        [B, C, H, Tr]; xt_ref as [B, H, Tr]; stats / ysum as [B, C, 2]; tb as the flat row."""
        fmt = int(self.lib.sbk_vc_cond_debug_op_layout(self.h, name.encode()))
        if fmt < 0:
            raise RuntimeError(f"vc_cond_debug_read: no captured tensor named '{name}'")
        n = C.c_int64(0)
        _check(self.lib.sbk_vc_cond_debug_read(self.h, name.encode(), None, C.byref(n)), "sbk_vc_cond_debug_read")
        out = torch.empty(n.value, dtype=torch.float64 if fmt == 3 else torch.float32)
        _check(self.lib.sbk_vc_cond_debug_read(self.h, name.encode(), C.c_void_p(out.data_ptr()), C.byref(n)),
               "sbk_vc_cond_debug_read")
        B, Tr = self._vc_shape
        H = self.n_feats
        if fmt == 1:                                       # [B][H][C/4][Tr][4] -> [B, C, H, Tr]
            Cc = n.value // (B * H * Tr)
            out = out.view(B, H, Cc // 4, Tr, 4).permute(0, 2, 4, 1, 3).reshape(B, Cc, H, Tr)
        elif fmt == 3:
            out = out.view(B, -1, 2)
        elif name.endswith(".xt_ref"):
            out = out.view(B, H, Tr)
        return out.double().contiguous()

    def vc_reverse_diffusion(self, z, mask, mean, cond, n_timesteps, mode, noise=None):
        B, T = self._check_inputs(z, mask, mean, None)
        sl = self.batch_slices(B, T, n_timesteps)
        if len(sl) > 1:
            outs = [self.vc_reverse_diffusion(z[a:b], mask[a:b], mean[a:b], cond[:, a:b].contiguous(), n_timesteps, mode,
                                              None if noise is None else noise[:, a:b].contiguous()) for a, b in sl]
            return torch.cat(outs, 0)
        z, mask, mean, cond = _f32c(z, "z"), _f32c(mask, "mask"), _f32c(mean, "mean"), _f32c(cond, "cond")
        if tuple(cond.shape) != (n_timesteps, B, self.dim_cond):
            raise RuntimeError(f"cond shape {tuple(cond.shape)} != {(n_timesteps, B, self.dim_cond)}")
        if mode != "pf":
            if noise is None:
                raise RuntimeError("modes 'em'/'ml' need pre-drawn noise [N,B,n_feats,T]")
            noise = _f32c(noise, "noise")
        out = torch.empty_like(z)
        self._call(self.lib.sbk_vc_reverse_diffusion, "sbk_vc_reverse_diffusion", self.h, _ptr(z), _ptr(mask), _ptr(mean),
                   _ptr(cond), _ptr(noise) if mode != "pf" else None, _ptr(out), B, T, int(n_timesteps),
                   self.VC_MODES[mode], self._stream())
        return out

    def reverse_diffusion_host(self, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None, out=None):
        """Host-buffer entry point: CPU (ideally pinned) tensors in, CPU tensor out; copies are inside the call."""
        for n, t in (("z", z), ("mask", mask), ("mu", mu)):
            if t.is_cuda:
                raise RuntimeError(f"{n}: reverse_diffusion_host takes host tensors")
        B, _, T = z.shape
        z, mask, mu = _f32c(z, "z"), _f32c(mask, "mask"), _f32c(mu, "mu")
        spk = _f32c(spk, "spk") if (spk is not None and self.n_spks > 1) else None
        noise = _f32c(noise, "noise") if stoc else None
        if out is None:
            out = torch.empty_like(z, pin_memory=z.is_pinned())
        _check(self.lib.sbk_reverse_diffusion_host(self.h, _ptr(z), _ptr(mask), _ptr(mu), _ptr(spk), _ptr(noise),
                                                   _ptr(out), B, T, int(n_timesteps), 1 if stoc else 0),
               "sbk_reverse_diffusion_host")
        return out

    def last_host_launches(self):
        """Host launches the Euler loop of the last sampler call took (1 = the whole loop ran as one CUDA graph)."""
        return int(self.lib.sbk_last_host_launches(self.h))

    def profile_ops(self):
        """[(name, ms, flops, bytes)] for one step of the current plan, one CUDA event pair per launch."""
        cap = 512
        ms, fl, by, n = (C.c_float * cap)(), (C.c_double * cap)(), (C.c_double * cap)(), C.c_int(0)
        _check(self.lib.sbk_profile_ops(self.h, ms, fl, by, cap, C.byref(n)), "sbk_profile_ops")
        names = self.debug_names()
        return [(names[i], ms[i], fl[i], by[i]) for i in range(n.value)]

    # ---- test hooks
    def debug_capture(self, on=True):
        _check(self.lib.sbk_debug_capture(self.h, 1 if on else 0), "sbk_debug_capture")

    def debug_layout(self, name=None):
        """0: [B][H][W][C]; 1: [B][H][C/4][W][4]; 2: [B][H][C/8][W][8] (bf16 operand tensor, widened to fp32 by debug_read)."""
        if name is not None:
            return int(self.lib.sbk_debug_op_layout(self.h, name.encode()))
        return int(self.lib.sbk_debug_layout(self.h))

    def debug_names(self):
        return [self.lib.sbk_debug_name(self.h, i).decode() for i in range(self.lib.sbk_debug_num(self.h))]

    def debug_read(self, name):
        n = C.c_int64(0)
        _check(self.lib.sbk_debug_read(self.h, name.encode(), None, C.byref(n)), "sbk_debug_read")
        if n.value == 0:
            return None
        out = torch.empty(n.value, dtype=torch.float32)
        _check(self.lib.sbk_debug_read(self.h, name.encode(), C.c_void_p(out.data_ptr()), C.byref(n)), "sbk_debug_read")
        return out
