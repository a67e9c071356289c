"""Drop-in `Diffusion` for Grad-TTS (replaces Grad-TTS/model/diffusion.py:227-294).

Same constructor, same parameter names/shapes under `estimator.*` (so
`GradTTS.load_state_dict(strict=True)`, inference.py:53, keeps working) and the same
`forward(z, mask, mu, n_timesteps, stoc=False, spk=None)` surface called from
`GradTTS.forward` (tts.py:96).  Sampling runs in libsbk.so (hand-written sm_90a CUDA,
CUDA-graph replay of the Euler loop); there is NO CPU or eager-PyTorch sampling path -
calling `forward` with CPU tensors raises.  The training-time methods
(`forward_diffusion`, `loss_t`, `compute_loss`; diffusion.py:244-252,281-294) stay plain
PyTorch over the same parameters, as in the reference; they need autograd and are not on
the accelerated path.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .binding import Engine, check_lengths, prior_expand


class BaseModule(nn.Module):
    """Grad-TTS/model/base.py:13-37 surface (`nparams`, `relocate_input`)."""

    @property
    def nparams(self):
        return int(sum(np.prod(p.shape) for p in self.parameters() if p.requires_grad))

    def relocate_input(self, x: list):
        dev = next(self.parameters()).device
        return [v.to(dev) if isinstance(v, torch.Tensor) and v.device != dev else v for v in x]


# ---------------------------------------------------------------------------------------------
# parameter containers.  Attribute names are dictated by the reference checkpoint format.
# Their torch forwards exist for the autograd (training) methods only.
# ---------------------------------------------------------------------------------------------
class Mish(BaseModule):
    def forward(self, x):
        return F.mish(x)


class _ConvGNMish(BaseModule):           # reference name: Block
    def __init__(self, cin, cout, groups=8):
        super().__init__()
        self.block = nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1), nn.GroupNorm(groups, cout), Mish())

    def forward(self, x, mask):
        return self.block(x * mask) * mask


class _TimeResBlock(BaseModule):         # reference name: ResnetBlock
    def __init__(self, cin, cout, time_dim, groups=8):
        super().__init__()
        self.mlp = nn.Sequential(Mish(), nn.Linear(time_dim, cout))
        self.block1 = _ConvGNMish(cin, cout, groups)
        self.block2 = _ConvGNMish(cout, cout, groups)
        self.res_conv = nn.Conv2d(cin, cout, 1) if cin != cout else nn.Identity()

    def forward(self, x, mask, temb):
        h = self.block1(x, mask) + self.mlp(temb)[:, :, None, None]
        return self.block2(h, mask) + self.res_conv(x * mask)


class _LinAttn(BaseModule):              # reference name: LinearAttention
    def __init__(self, c, heads=4, dim_head=32):
        super().__init__()
        self.heads = heads
        self.to_qkv = nn.Conv2d(c, heads * dim_head * 3, 1, bias=False)
        self.to_out = nn.Conv2d(heads * dim_head, c, 1)

    def forward(self, x):
        b, _, h, w = x.shape
        q, k, v = self.to_qkv(x).view(b, 3, self.heads, -1, h * w).unbind(1)
        ctx = torch.einsum("bhdn,bhen->bhde", k.softmax(-1), v)
        return self.to_out(torch.einsum("bhde,bhdn->bhen", ctx, q).reshape(b, -1, h, w))


class _Gate(BaseModule):                 # reference name: Rezero
    def __init__(self, fn):
        super().__init__()
        self.fn = fn
        self.g = nn.Parameter(torch.zeros(1))

    def forward(self, x):
        return self.fn(x) * self.g


class _Skip(BaseModule):                 # reference name: Residual
    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def forward(self, x):
        return self.fn(x) + x


class _Resample(BaseModule):             # reference names: Downsample / Upsample
    def __init__(self, c, up):
        super().__init__()
        self.conv = nn.ConvTranspose2d(c, c, 4, 2, 1) if up else nn.Conv2d(c, c, 3, 2, 1)

    def forward(self, x):
        return self.conv(x)


class SinusoidalPosEmb(BaseModule):
    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def forward(self, x, scale=1000):
        half = self.dim // 2
        freqs = torch.exp(torch.arange(half, device=x.device).float() * -(math.log(10000) / (half - 1)))
        ang = scale * x[:, None] * freqs[None, :]
        return torch.cat((ang.sin(), ang.cos()), dim=-1)


class GradLogPEstimator2d(BaseModule):
    """Parameter tree of the score U-Net (names as in diffusion.py:128-172)."""

    def __init__(self, dim, dim_mults=(1, 2, 4), groups=8, n_spks=None, spk_emb_dim=64, n_feats=80, pe_scale=1000):
        super().__init__()
        if tuple(dim_mults) != (1, 2, 4) or groups != 8:
            raise ValueError("the sm_90a engine is built for dim_mults=(1,2,4), groups=8 (the reference defaults)")
        self.dim, self.dim_mults, self.groups = dim, dim_mults, groups
        self.n_spks = 1 if n_spks is None else n_spks
        self.spk_emb_dim, self.pe_scale, self.n_feats = spk_emb_dim, pe_scale, n_feats
        if self.n_spks > 1:
            self.spk_mlp = nn.Sequential(nn.Linear(spk_emb_dim, spk_emb_dim * 4), Mish(),
                                         nn.Linear(spk_emb_dim * 4, n_feats))
        self.time_pos_emb = SinusoidalPosEmb(dim)
        self.mlp = nn.Sequential(nn.Linear(dim, dim * 4), Mish(), nn.Linear(dim * 4, dim))
        chans = [2 + (1 if self.n_spks > 1 else 0)] + [dim * m for m in dim_mults]
        pairs = list(zip(chans[:-1], chans[1:]))
        self.downs = nn.ModuleList()
        for i, (ci, co) in enumerate(pairs):
            last = i == len(pairs) - 1
            self.downs.append(nn.ModuleList([_TimeResBlock(ci, co, dim), _TimeResBlock(co, co, dim),
                                             _Skip(_Gate(_LinAttn(co))),
                                             nn.Identity() if last else _Resample(co, up=False)]))
        mid = chans[-1]
        self.mid_block1 = _TimeResBlock(mid, mid, dim)
        self.mid_attn = _Skip(_Gate(_LinAttn(mid)))
        self.mid_block2 = _TimeResBlock(mid, mid, dim)
        self.ups = nn.ModuleList()
        for ci, co in reversed(pairs[1:]):
            self.ups.append(nn.ModuleList([_TimeResBlock(co * 2, ci, dim), _TimeResBlock(ci, ci, dim),
                                           _Skip(_Gate(_LinAttn(ci))), _Resample(ci, up=True)]))
        self.final_block = _ConvGNMish(dim, dim)
        self.final_conv = nn.Conv2d(dim, 1, 1)

    def forward(self, x, mask, mu, t, spk=None):
        """Autograd path for training (Diffusion.loss_t).  Inference never calls this."""
        temb = self.mlp(self.time_pos_emb(t, scale=self.pe_scale))
        planes = [mu, x]
        if self.n_spks > 1:
            planes.append(self.spk_mlp(spk)[:, :, None].expand(-1, -1, x.shape[-1]))
        h = torch.stack(planes, 1)
        m = mask[:, None]
        pyramid, skips = [m], []
        for r1, r2, att, down in self.downs:
            mk = pyramid[-1]
            h = att(r2(r1(h, mk, temb), mk, temb))
            skips.append(h)
            h = down(h * mk)
            pyramid.append(mk[..., ::2])
        pyramid.pop()
        mk = pyramid[-1]
        h = self.mid_block2(self.mid_attn(self.mid_block1(h, mk, temb)), mk, temb)
        for r1, r2, att, up in self.ups:
            mk = pyramid.pop()
            h = r1(torch.cat((h, skips.pop()), 1), mk, temb)
            h = up(att(r2(h, mk, temb)) * mk)
        h = self.final_block(h, m)
        return (self.final_conv(h * m) * m).squeeze(1)


def get_noise(t, beta_init, beta_term, cumulative=False):
    """diffusion.py:219-224."""
    if cumulative:
        return beta_init * t + 0.5 * (beta_term - beta_init) * (t ** 2)
    return beta_init + (beta_term - beta_init) * t


class Diffusion(BaseModule):
    """Score-based decoder.  `precision`/`use_graph` are extra, keyword-only engine knobs.  The default precision
    "fp32x3" is fp32-class arithmetic on the tensor cores (tf32 main product + one fp16 correction product per MAC, exact fp32 everywhere else): it matches
    the reference's fp32 path to ~1e-6 per estimator call.  "tf32" is what PyTorch's own GPU convs compute by default
    (~1.5e-3 per call), "bf16" is config 3's arithmetic, "fp16" runs bf16's operand bytes and MMA rate with fp16 operands
    (tf32-class error; operands saturate at +-65504), "fp32" the CUDA-core FFMA path."""

    def __init__(self, n_feats, dim, n_spks=1, spk_emb_dim=64, beta_min=0.05, beta_max=20, pe_scale=1000,
                 *, precision="fp32x3", use_graph=True):
        super().__init__()
        self.n_feats, self.dim, self.n_spks, self.spk_emb_dim = n_feats, dim, n_spks, spk_emb_dim
        self.beta_min, self.beta_max, self.pe_scale = beta_min, beta_max, pe_scale
        self.precision, self.use_graph = precision, use_graph
        self.estimator = GradLogPEstimator2d(dim, n_spks=n_spks, spk_emb_dim=spk_emb_dim, n_feats=n_feats,
                                             pe_scale=pe_scale)
        self._engine = None
        self._engine_sig = None

    # ---- engine management -------------------------------------------------------------------
    def _weights_signature(self, device):
        return (device.index,) + tuple((p.data_ptr(), p._version) for p in self.estimator.parameters())

    def engine(self) -> Engine:
        """The libsbk handle for the module's current device/weights (re-packed when weights change)."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("Diffusion sampling runs only on a CUDA device (sm_90a); move the module with "
                               ".cuda() first - there is no CPU fallback")
        sig = self._weights_signature(dev)
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = Engine(self.n_feats, self.dim, self.n_spks, self.spk_emb_dim, self.beta_min,
                                  self.beta_max, self.pe_scale, device=dev.index, precision=self.precision,
                                  use_graph=self.use_graph)
            self._engine_sig = None
        if sig != self._engine_sig:
            sd = {"estimator." + k: v for k, v in self.estimator.state_dict().items()}
            with torch.cuda.device(dev):
                self._engine.load_state_dict(sd)
            self._engine_sig = sig
        return self._engine

    # ---- sampling (diffusion.py:254-279) -----------------------------------------------------
    @torch.no_grad()
    def reverse_diffusion(self, z, mask, mu, n_timesteps, stoc=False, spk=None, *, lengths=None):
        """lengths: optional int64 [B] valid frames per utterance (e.g. y_lengths): utterance b is then sampled on its own
        fix_len_compatibility(lengths[b]) frames, as a call on its slices alone would be, and its frames past them are 0
        (Engine.estimator).  None keeps the padded-batch semantics of the reference's batched call."""
        eng = self.engine()
        # The sampler state (xt, mu, noise, Euler update) is fp32 in every precision mode; reduced-precision callers
        # (config 3: bf16 tensors in / out) are widened here and the result is cast back to the caller's dtype.
        io_dtype = z.dtype
        if io_dtype != torch.float32:
            z, mask, mu = z.float(), mask.float(), mu.float()
            spk = None if spk is None else spk.float()
        with torch.cuda.device(z.device):
            if lengths is not None:     # checked before any launch or noise draw
                lengths = check_lengths(lengths, z.shape[0], z.shape[2], z.device, "z")
            if not stoc:
                out = eng.reverse_diffusion(z, mask, mu, n_timesteps, False, spk, None, lengths)
            else:
                out = self._stochastic(eng, z, mask, mu, n_timesteps, spk, lengths)
        return out if io_dtype == torch.float32 else out.to(io_dtype)

    # bytes of pre-drawn Euler-Maruyama noise resident at once (config 3: N=1000 x B=128 would be 21 GB if materialised)
    noise_window_bytes = 256 << 20

    def _stochastic(self, eng, z, mask, mu, n_timesteps, spk, lengths=None):
        """stoc=True: the reference draws torch.randn(z.shape) once per step, in step order (:267).  The same draws, in the
        same order, are made here a window of steps at a time and streamed through `sbk_reverse_steps`, so the noise
        resident at any moment is bounded by `noise_window_bytes` instead of growing with N."""
        per_step = z.numel() * 4
        window = max(1, min(n_timesteps, self.noise_window_bytes // per_step))
        draw = lambda n: torch.stack([torch.randn(z.shape, dtype=z.dtype, device=z.device) for _ in range(n)])
        if window >= n_timesteps or len(eng.batch_slices(z.shape[0], z.shape[2])) > 1:
            return eng.reverse_diffusion(z, mask, mu, n_timesteps, True, spk, draw(n_timesteps), lengths)
        xt = (z * mask).contiguous()                                                # :256
        for s0 in range(0, n_timesteps, window):
            s1 = min(n_timesteps, s0 + window)
            eng.reverse_steps(xt, mask, mu, n_timesteps, s0, s1, True, spk, draw(s1 - s0), lengths)
        return xt

    @torch.no_grad()
    def forward(self, z, mask, mu, n_timesteps, stoc=False, spk=None, *, lengths=None):
        return self.reverse_diffusion(z, mask, mu, n_timesteps, stoc, spk, lengths=lengths)

    def rolling(self, capacity, max_frames):
        """A RollingSampler (rolling.py) of `capacity` slots at up to `max_frames` frames with this module's configuration,
        precision and current weights: utterances join and leave a running batch at any step, each mel equal to its own
        `forward` call.  The slot plan is a native plan of its own, so the sampler holds an engine of its own and this
        module's `forward` calls stay usable alongside it; weights changed later are not seen by the sampler."""
        from .rolling import RollingSampler
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("Diffusion sampling runs only on a CUDA device (sm_90a); move the module with "
                               ".cuda() first - there is no CPU fallback")
        eng = Engine(self.n_feats, self.dim, self.n_spks, self.spk_emb_dim, self.beta_min, self.beta_max, self.pe_scale,
                     device=dev.index, precision=self.precision, use_graph=self.use_graph)
        with torch.cuda.device(dev):
            eng.load_state_dict({"estimator." + k: v for k, v in self.estimator.state_dict().items()})
            return RollingSampler(eng, capacity, max_frames)

    @torch.no_grad()
    def forward_host(self, z, mask, mu, n_timesteps, stoc=False, spk=None):
        """Same call for HOST tensors (pinned for async copies): H2D, loop, D2H inside libsbk."""
        eng = self.engine()
        noise = torch.randn((n_timesteps,) + tuple(z.shape), dtype=z.dtype) if stoc else None
        return eng.reverse_diffusion_host(z, mask, mu, n_timesteps, stoc, spk, noise)

    # ---- training-time methods: plain PyTorch (diffusion.py:244-252, 281-294) -----------------
    def forward_diffusion(self, x0, mask, mu, t):
        cum = get_noise(t[:, None, None], self.beta_min, self.beta_max, cumulative=True)
        decay = torch.exp(-0.5 * cum)
        z = torch.randn(x0.shape, dtype=x0.dtype, device=x0.device, requires_grad=False)
        xt = x0 * decay + mu * (1.0 - decay) + z * torch.sqrt(1.0 - torch.exp(-cum))
        return xt * mask, z * mask

    def loss_t(self, x0, mask, mu, t, spk=None):
        xt, z = self.forward_diffusion(x0, mask, mu, t)
        cum = get_noise(t[:, None, None], self.beta_min, self.beta_max, cumulative=True)
        score = self.estimator(xt, mask, mu, t, spk) * torch.sqrt(1.0 - torch.exp(-cum))
        return torch.sum((score + z) ** 2) / (torch.sum(mask) * self.n_feats), xt

    def compute_loss(self, x0, mask, mu, spk=None, offset=1e-5):
        t = torch.rand(x0.shape[0], dtype=x0.dtype, device=x0.device, requires_grad=False)
        return self.loss_t(x0, mask, mu, torch.clamp(t, offset, 1.0 - offset), spk)


# ---- the step before the path: GradTTS.forward between the text encoder and the decoder (tts.py:77-99) ----------------
def fix_len_compatibility(length, num_downsamplings_in_unet=2):
    """Grad-TTS/model/utils.py:13-17."""
    while length % (2 ** num_downsamplings_in_unet) != 0:
        length += 1
    return length


def reference_order_noise(B, n_feats, Ty, dtype, device):
    """The draws of the reference's `torch.randn_like(mu_y)` (tts.py:94) as a contiguous [B,Ty,n_feats] tensor.
    There mu_y is `matmul(...).transpose(1, 2)`, a [B,n_feats,Ty] VIEW with strides (Ty*n_feats, 1, n_feats); randn_like
    keeps those strides and torch's generators fill strided tensors differently from contiguous ones, so the only way to
    get the same numbers from the same generator state is to make the same call on a tensor with the same strides."""
    proto = torch.empty((B, Ty, n_feats), dtype=dtype, device=device).transpose(1, 2)
    noise = torch.randn_like(proto)
    return noise.transpose(1, 2)            # the same memory, now a contiguous [B,Ty,n_feats] tensor


@torch.no_grad()
def synthesize_from_encoder(decoder, mu_x, logw, x_mask, n_timesteps, temperature=1.0, stoc=False, spk=None,
                            length_scale=1.0, want_attn=True, noise_tf=None, *, ragged=False):
    """Drop-in for Grad-TTS/model/tts.py:77-99 - everything `GradTTS.forward` does after `self.encoder(...)`:

        mu_x, logw, x_mask = self.encoder(x, x_lengths, spk)
        return synthesize_from_encoder(self.decoder, mu_x, logw, x_mask, n_timesteps, temperature, stoc, spk, length_scale)

    The durations and output lengths (tts.py:77-81) are the reference's own four tiny ops on [B,1,Tx] tensors; the ONE
    host synchronisation (`int(y_lengths.max())`) is kept because it fixes the SHAPE of what the method returns.
    Everything sized [B,Tx,Ty] or [B,F,Ty] - generate_path, the 0/1 matmul, the terminal sample - is one libsbk kernel
    (`sbk_prior_expand`) that writes mu_y / z / y_mask in the layout the sampler reads.  The noise is drawn by torch with
    the reference's own call on a tensor with the reference's strides (`reference_order_noise`), so with the same
    generator state z equals the reference's z bit for bit.  Returns (encoder_outputs, decoder_outputs, attn) like the reference.

    ragged=True samples each utterance on its own fix_len_compatibility(y_lengths[b]) frames (the decoder gets
    lengths=y_lengths), as the reference's B = 1 call on that utterance would, instead of the padded batch; its frames past
    them come out 0.  Follow it with the vocoder's `lengths=y_lengths` for per-utterance waveforms."""
    if not mu_x.is_cuda:
        raise RuntimeError("synthesize_from_encoder runs only on a CUDA device (sm_90a); there is no CPU fallback")
    B, Fm, Tx = mu_x.shape
    w = torch.exp(logw) * x_mask                                                   # :77
    w_ceil = torch.ceil(w) * length_scale                                          # :78
    y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()               # :79
    y_max_length = int(y_lengths.max())                                            # :80 (host sync: output shape)
    y_max_length_ = fix_len_compatibility(y_max_length)                            # :81
    if noise_tf is None:                                                           # (tests may inject pre-drawn noise [B,Ty,F])
        noise_tf = reference_order_noise(B, Fm, y_max_length_, mu_x.dtype, mu_x.device)  # :94, the reference's draws
    mu_y, z, y_mask, attn = prior_expand(mu_x, w_ceil.reshape(B, Tx), x_mask.reshape(B, Tx).to(torch.float32), y_lengths,
                                         y_max_length_, noise_tf, temperature, want_attn)
    if ragged:
        decoder_outputs = decoder(z, y_mask, mu_y, n_timesteps, stoc, spk, lengths=y_lengths)
    else:
        decoder_outputs = decoder(z, y_mask, mu_y, n_timesteps, stoc, spk)         # :96
    # (the reference slices attn's dim 2 - the token axis - with the frame count, tts.py:99; kept as is)
    return (mu_y[:, :, :y_max_length], decoder_outputs[:, :, :y_max_length],
            None if attn is None else attn[:, :, :y_max_length])
