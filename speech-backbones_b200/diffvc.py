"""Drop-in `Diffusion`, `FwdDiffusion` and `DiffVC` for DiffVC (replace DiffVC/model/diffusion.py:109-222 and
DiffVC/model/vc.py:19-144; `DiffVC` and `FwdDiffusion` are at the end of this file).

`Diffusion` has the same constructor `(n_feats, dim_unet, dim_spk, use_ref_t, beta_min, beta_max)`, the same 206 parameter
names/shapes under `estimator.*` (so `DiffVC.load_state_dict` / `vc_*.pt` checkpoints load unchanged) and the same
`forward(z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode)` surface called from `DiffVC.forward`
(DiffVC/model/vc.py:125), including the reference's behaviour for an invalid mode (prints and returns `z`, :201-203).

Split of the work.  Everything in the conditioning branch of `GradLogPEstimator.forward` (:62-71: time sinusoid,
RefBlock on the diffused reference, speaker embedding, cond_block) depends on t, ref and c only - never on xt - so it
is hoisted out of the loop and evaluated once for all N steps (`conditioning_table`): natively in libsbk.so in the
tensor-core mode, with PyTorch ops in the exact-fp32 mode.  The U-Net (downs/mid/ups/final), the three samplers
pf / em / ml and the fold of the conditioning vector into the first ResnetBlock always run in libsbk.so.  There is no
CPU path: CPU tensors raise.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .binding import Engine
from .gradtts import (BaseModule, Mish, SinusoidalPosEmb, _ConvGNMish, _Gate, _LinAttn, _Resample, _Skip, _TimeResBlock)
from .postnet import PostNet
from .rolling import VcRollingSampler
from .text_encoder import MelEncoder


class RefBlock(BaseModule):
    """Parameter container + PyTorch forward of DiffVC/model/modules.py:128-166."""

    def __init__(self, out_dim, time_emb_dim):
        super().__init__()
        b = out_dim // 4
        self.mlp1 = nn.Sequential(Mish(), nn.Linear(time_emb_dim, b))
        self.mlp2 = nn.Sequential(Mish(), nn.Linear(time_emb_dim, 2 * b))

        def cig(ci, co):
            return nn.Sequential(nn.Conv2d(ci, co, 3, 1, 1), nn.InstanceNorm2d(co, affine=True), nn.GLU(dim=1))
        self.block11, self.block12 = cig(1, 2 * b), cig(b, 2 * b)
        self.block21, self.block22 = cig(b, 4 * b), cig(2 * b, 4 * b)
        self.block31, self.block32 = cig(2 * b, 8 * b), cig(4 * b, 8 * b)
        self.final_conv = nn.Conv2d(4 * b, out_dim, 1)

    def forward(self, x, mask, temb):
        y = self.block12(self.block11(x * mask) * mask) + self.mlp1(temb)[:, :, None, None]
        y = self.block22(self.block21(y * mask) * mask) + self.mlp2(temb)[:, :, None, None]
        y = self.final_conv(self.block32(self.block31(y * mask) * mask) * mask)
        return (y * mask).sum((2, 3)) / (mask.sum((2, 3)) * x.shape[2])


class GradLogPEstimator(BaseModule):
    """Parameter tree of DiffVC's score U-Net (names as in DiffVC/model/diffusion.py:17-59)."""

    def __init__(self, dim_base, dim_cond, use_ref_t, dim_mults=(1, 2, 4)):
        super().__init__()
        if tuple(dim_mults) != (1, 2, 4):
            raise ValueError("the sm_90a engine is built for dim_mults=(1,2,4)")
        self.use_ref_t, self.dim_base, self.dim_cond = use_ref_t, dim_base, dim_cond
        chans = [2 + dim_cond] + [dim_base * m for m in dim_mults]
        pairs = list(zip(chans[:-1], chans[1:]))
        self.time_pos_emb = SinusoidalPosEmb(dim_base)
        self.mlp = nn.Sequential(nn.Linear(dim_base, dim_base * 4), Mish(), nn.Linear(dim_base * 4, dim_base))
        cond_total = dim_base + 256
        if use_ref_t:
            self.ref_block = RefBlock(out_dim=dim_cond, time_emb_dim=dim_base)
            cond_total += dim_cond
        self.cond_block = nn.Sequential(nn.Linear(cond_total, 4 * dim_cond), Mish(), nn.Linear(4 * dim_cond, dim_cond))
        self.downs = nn.ModuleList()
        for i, (ci, co) in enumerate(pairs):
            last = i == len(pairs) - 1
            self.downs.append(nn.ModuleList([_TimeResBlock(ci, co, dim_base), _TimeResBlock(co, co, dim_base),
                                             _Skip(_Gate(_LinAttn(co))),
                                             nn.Identity() if last else _Resample(co, up=False)]))
        mid = chans[-1]
        self.mid_block1 = _TimeResBlock(mid, mid, dim_base)
        self.mid_attn = _Skip(_Gate(_LinAttn(mid)))
        self.mid_block2 = _TimeResBlock(mid, mid, dim_base)
        self.ups = nn.ModuleList()
        for ci, co in reversed(pairs[1:]):
            self.ups.append(nn.ModuleList([_TimeResBlock(co * 2, ci, dim_base), _TimeResBlock(ci, ci, dim_base),
                                           _Skip(_Gate(_LinAttn(ci))), _Resample(ci, up=True)]))
        self.final_block = _ConvGNMish(dim_base, dim_base)
        self.final_conv = nn.Conv2d(dim_base, 1, 1)

    def conditioning(self, ref, ref_mask, c, t):
        """The xt-independent branch (:62-71): [B] time values -> conditioning vectors [B, dim_cond]."""
        cond = self.time_pos_emb(t, scale=1000)
        if self.use_ref_t:
            cond = torch.cat([cond, self.ref_block(ref, ref_mask[:, None], self.mlp(cond))], 1)
        return self.cond_block(torch.cat([cond, c], 1))

    def forward(self, x, x_mask, mean, ref, ref_mask, c, t):
        """Autograd path for training (Diffusion.loss_t); inference never calls this."""
        temb = self.mlp(self.time_pos_emb(t, scale=1000))
        cond = self.conditioning(ref, ref_mask, c, t)
        h = torch.stack([mean, x], 1)
        m = x_mask[:, None]
        h = torch.cat([h, cond[:, :, None, None].expand(-1, -1, h.shape[2], h.shape[3])], 1)
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


class Diffusion(BaseModule):
    def __init__(self, n_feats, dim_unet, dim_spk, use_ref_t, beta_min, beta_max, *, precision="fp32x3", use_graph=True):
        super().__init__()
        self.estimator = GradLogPEstimator(dim_unet, dim_spk, use_ref_t)
        self.n_feats, self.dim_unet, self.dim_spk, self.use_ref_t = n_feats, dim_unet, dim_spk, use_ref_t
        self.beta_min, self.beta_max = beta_min, beta_max
        self.precision, self.use_graph = precision, use_graph
        self._engine = None
        self._engine_sig = None

    # ---- scalars (diffusion.py:120-155) -------------------------------------------------------
    def get_beta(self, t):
        return self.beta_min + (self.beta_max - self.beta_min) * t

    def get_gamma(self, s, t, p=1.0, use_torch=False):
        bi = self.beta_min + 0.5 * (self.beta_max - self.beta_min) * (t + s)
        bi = bi * (t - s)
        return torch.exp(-0.5 * p * bi)[:, None, None] if use_torch else math.exp(-0.5 * p * bi)

    def compute_diffused_mean(self, x0, mask, mean, t, use_torch=False):
        w = self.get_gamma(0, t, use_torch=use_torch)
        return (x0 * w + mean * (1.0 - w)) * mask

    # ---- engine ------------------------------------------------------------------------------
    def _device(self):
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("DiffVC sampling runs only on a CUDA device (sm_90a); move the module with .cuda() "
                               "first - there is no CPU fallback")
        return dev

    def _new_engine(self, dev) -> Engine:
        return Engine(self.n_feats, self.dim_unet, 1, 64, self.beta_min, self.beta_max, 1000.0, device=dev.index,
                      precision=self.precision, use_graph=self.use_graph, model="diffvc", dim_cond=self.dim_spk,
                      use_ref_t=self.use_ref_t)

    def engine(self) -> Engine:
        dev = self._device()
        sig = (dev.index,) + tuple((p.data_ptr(), p._version) for p in self.estimator.parameters())
        if self._engine is None or self._engine.device != dev.index:
            if self._engine is not None:
                self._engine.close()
            self._engine = self._new_engine(dev)
            self._engine_sig = None
        if sig != self._engine_sig:
            with torch.cuda.device(dev):
                self._engine.load_state_dict({"estimator." + k: v for k, v in self.estimator.state_dict().items()})
            self._engine_sig = sig
        return self._engine

    def rolling(self, capacity, max_frames):
        """A VcRollingSampler (rolling.py) of `capacity` slots at up to `max_frames` frames with this module's configuration,
        precision and current weights: utterances join and leave a running batch at any step.  The slot plan is a native
        plan of its own, so the sampler holds an engine of its own and this module's `forward` calls stay usable alongside
        it; weights changed later are not seen by the sampler."""
        return self._rolling(VcRollingSampler, capacity, max_frames)

    def _rolling(self, sampler, capacity, max_frames, *args):
        dev = self._device()
        eng = self._new_engine(dev)
        with torch.cuda.device(dev):
            eng.load_state_dict({"estimator." + k: v for k, v in self.estimator.state_dict().items()})
            return sampler(*args, eng, capacity, max_frames)

    # ---- sampling (diffusion.py:164-205) ------------------------------------------------------
    @torch.no_grad()
    def conditioning_table(self, ref, ref_mask, mean_ref, c, n_timesteps, *, ref_lengths=None):
        """cond[i] for every step i (t_i = 1 - i/N): the hoisted conditioning branch, native in every precision
        (libsbk `sbk_vc_conditioning`: RefBlock convs on wgmma - tf32 + fp16 correction for the fp32-class modes - plus the
        InstanceNorm / GLU / cond_block kernels).  There is no PyTorch fallback.  ref_lengths (int64 [B], keyword only): each
        sample's rows are computed on exactly its own reference frames, as its B = 1 call."""
        with torch.cuda.device(ref.device):
            return self.engine().vc_conditioning(ref, ref_mask, mean_ref, c, n_timesteps, ref_lengths)

    # lengths (int64 [B] on z's device, e.g. x_lengths; keyword only): a ragged batch for the score U-Net.  Row b is sampled
    # on its own T_b = fix_len_compatibility(lengths[b]) frames, as the call on its [:T_b] slices would be given the same
    # draws noise[:, b, :, :T_b], and is 0 from T_b on (Engine.vc_reverse_diffusion).  The noise is drawn on the batch
    # shapes exactly as without lengths.  ref_lengths (int64 [B], e.g. x_ref_lengths): the conditioning table row by row on
    # each reference's own frames (conditioning_table).
    @torch.no_grad()
    def reverse_diffusion(self, z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode, *, lengths=None, ref_lengths=None):
        eng = self.engine()
        cond = self.conditioning_table(ref, ref_mask, mean_ref, c, n_timesteps, ref_lengths=ref_lengths)
        noise = None
        if mode != "pf":   # the reference draws randn_like(z) once per step, in step order (:194)
            noise = torch.stack([torch.randn_like(z) for _ in range(n_timesteps)])
        with torch.cuda.device(z.device):
            return eng.vc_reverse_diffusion(z, mask, mean, cond, n_timesteps, mode, noise, lengths)

    @torch.no_grad()
    def forward(self, z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode, *, lengths=None, ref_lengths=None):
        if mode not in ["pf", "em", "ml"]:
            print("Inference mode must be one of [pf, em, ml]!")
            return z
        return self.reverse_diffusion(z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode, lengths=lengths,
                                      ref_lengths=ref_lengths)

    # ---- training-time methods: plain PyTorch (diffusion.py:157-162, 207-222) ------------------
    def forward_diffusion(self, x0, mask, mean, t):
        xt_mean = self.compute_diffused_mean(x0, mask, mean, t, use_torch=True)
        variance = 1.0 - self.get_gamma(0, t, p=2.0, use_torch=True)
        z = torch.randn(x0.shape, dtype=x0.dtype, device=x0.device, requires_grad=False)
        return (xt_mean + z * torch.sqrt(variance)) * mask, z * mask

    def loss_t(self, x0, mask, mean, x_ref, mean_ref, c, t):
        xt, z = self.forward_diffusion(x0, mask, mean, t)
        xt_ref = self.compute_diffused_mean(x_ref, mask, mean_ref, t, use_torch=True)[:, None]
        z_est = self.estimator(xt, mask, mean, xt_ref, mask, c, t)
        z_est = z_est * torch.sqrt(1.0 - self.get_gamma(0, t, p=2.0, use_torch=True))
        return torch.sum((z_est + z) ** 2) / (torch.sum(mask) * self.n_feats)

    def compute_loss(self, x0, mask, mean, x_ref, mean_ref, c, offset=1e-5):
        t = torch.rand(x0.shape[0], dtype=x0.dtype, device=x0.device, requires_grad=False)
        return self.loss_t(x0, mask, mean, x_ref, mean_ref, c, torch.clamp(t, offset, 1.0 - offset))


# ---- the step before the path: DiffVC.forward between the encoders and the decoder (DiffVC/model/vc.py:107-127) -------
def fix_len_compatibility(length, num_downsamplings_in_unet=2):
    """DiffVC/model/utils.py (same helper as Grad-TTS/model/utils.py:13-17)."""
    while length % (2 ** num_downsamplings_in_unet) != 0:
        length += 1
    return length


@torch.no_grad()
def decoder_inputs(decoder, x, x_lengths, mean):
    """DiffVC/model/vc.py:104,107,111-123: (mean_x, z, x_mask_new, mean_new, max_length) - the decoder's inputs, with z's
    draw (randn_like of the re-padded mean_x), as convert_from_encoder passes them to the decoder."""
    b, n_feats, t_in = x.shape
    max_length = int(x_lengths.max())                                              # :111 (host sync: output shape)
    if t_in != max_length:                                                         # the reference's x_mask (:104) has max_length frames
        raise RuntimeError(f"x has {t_in} frames but max(x_lengths) = {max_length}: DiffVC.forward expects a batch padded to its longest item")
    max_length_new = fix_len_compatibility(max_length)                             # :112
    frames = torch.arange(max_length_new, device=x.device)
    x_mask_new = (frames.unsqueeze(0) < x_lengths.unsqueeze(1)).unsqueeze(1).to(x.dtype)        # :113
    x_mask = x_mask_new[:, :, :max_length]                                         # :104
    mean_x = decoder.compute_diffused_mean(x, x_mask, mean, 1.0)                   # :107

    def repad(v):                                                                  # :114-120 without the per-sample loop
        out = torch.zeros((b, n_feats, max_length_new), dtype=x.dtype, device=x.device)
        out[:, :, :max_length] = torch.where(x_mask != 0, v, out[:, :, :max_length])
        return out

    mean_new, mean_x_new = repad(mean), repad(mean_x)
    z = mean_x_new
    z += torch.randn_like(mean_x_new, device=mean_x_new.device)                    # :122-123
    return mean_x, z, x_mask_new, mean_new, max_length


@torch.no_grad()
def convert_from_encoder(decoder, x, x_lengths, mean, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode="ml", *,
                         ragged=False, x_ref_lengths=None):
    """Drop-in for DiffVC/model/vc.py:107,110-127 - what `DiffVC.forward` does once `mean = self.encoder(x, x_mask)` and
    `mean_ref = self.encoder(x_ref, x_ref_mask)` exist:

        return convert_from_encoder(self.decoder, x, x_lengths, mean, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode)

    The reference re-pads `mean` and `mean_x` to a length the U-Net accepts with a Python loop over the batch that indexes
    `x_lengths[i]` on the host: 2B slice copies and B device-to-host synchronisations per call (vc.py:118-120).  Here the same
    tensors are one masked pad each (bit-identical: a copy of the valid prefix into zeros), the only synchronisation left is
    `int(x_lengths.max())`, which fixes the SHAPE of the returned tensor, and the noise draw is the reference's own call
    (`randn_like` of a contiguous [B,n_feats,T'] tensor), so the generator stream is unchanged.  Returns (mean_x, y).

    ragged=True (keyword only): the decoder samples row b on its own fix_len_compatibility(x_lengths[b]) frames and runs the
    conditioning branch on its own x_ref_lengths[b] reference frames (the sum of x_ref_mask's row when not given), so each
    row is the reference's B = 1 call on that utterance given the same draws; y is 0 past x_lengths[b]'s U-Net grid."""
    mean_x, z, x_mask_new, mean_new, max_length = decoder_inputs(decoder, x, x_lengths, mean)
    if ragged:
        if x_ref_lengths is None:
            x_ref_lengths = x_ref_mask.sum((1, 2)).round().to(torch.int64)
        y = decoder(z, x_mask_new, mean_new, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode, lengths=x_lengths,
                    ref_lengths=x_ref_lengths)
    else:
        y = decoder(z, x_mask_new, mean_new, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode)     # :125
    return mean_x, y[:, :, :max_length]


# ---- the whole model: DiffVC/model/vc.py:19-144 ------------------------------------------------------------------------------
def sequence_mask(length, max_length=None):
    """DiffVC/model/utils.py (same helper as Grad-TTS/model/utils.py:6-10)."""
    if max_length is None:
        max_length = length.max()
    x = torch.arange(int(max_length), dtype=length.dtype, device=length.device)
    return x.unsqueeze(0) < length.unsqueeze(1)


class FwdDiffusion(BaseModule):
    """Drop-in for DiffVC's "average voice" encoder (vc.py:19-48): `MelEncoder` (text_encoder.py) followed by `PostNet`
    (postnet.py), the reference's constructor and state_dict (`encoder.*`, `postnet.*`: 8,464,529 parameters at
    DiffVC's configuration).  `forward(x, mask)` runs both halves in libsbk; `precision` selects the PostNet's arithmetic
    (the mel encoder is exact fp32 on CUDA cores).  Training (`compute_loss`, :43-48) is not implemented here."""

    def __init__(self, n_feats, channels, filters, heads, layers, kernel, dropout, window_size, dim, *, precision="fp32x3"):
        super().__init__()
        self.n_feats, self.channels, self.filters, self.heads, self.layers = n_feats, channels, filters, heads, layers
        self.kernel, self.dropout, self.window_size, self.dim = kernel, dropout, window_size, dim
        self.encoder = MelEncoder(n_feats, channels, filters, heads, layers, kernel, dropout, window_size)
        self.postnet = PostNet(dim, precision=precision)

    # lengths (int64 [B] or None; keyword only): a ragged batch.  The mel encoder's masked convs and masked softmax already
    # keep each row's valid frames independent of its batch-mates; the PostNet then runs row b on exactly its lengths[b]
    # frames (PostNet.forward), and the row is 0 after them where the padded batch has final_conv.bias.
    @torch.no_grad()
    def forward(self, x, mask, *, lengths=None):                                    # :37-41
        x, mask = self.relocate_input([x, mask])
        z = self.encoder(x, mask)
        return self.postnet(z, mask, lengths=lengths)


class DiffVC(BaseModule):
    """Drop-in for `model.vc.DiffVC` (vc.py:52-144): the same constructor, the same 346-tensor state_dict (`encoder.*` of
    `FwdDiffusion`, `decoder.*` of `Diffusion`; 126,259,128 parameters at the notebook's configuration, so `vc_*.pt`
    checkpoints load strictly) and the same `forward(x, x_lengths, x_ref, x_ref_lengths, c, n_timesteps, mode)` ->
    (mean_x, y).  Encoder, PostNet and decoder run in libsbk; the random draws are the reference's, in its order."""

    def __init__(self, n_feats, channels, filters, heads, layers, kernel, dropout, window_size, enc_dim, spk_dim, use_ref_t,
                 dec_dim, beta_min, beta_max, *, precision="fp32x3"):
        super().__init__()
        self.n_feats, self.channels, self.filters, self.heads, self.layers = n_feats, channels, filters, heads, layers
        self.kernel, self.dropout, self.window_size, self.enc_dim, self.spk_dim = kernel, dropout, window_size, enc_dim, spk_dim
        self.use_ref_t, self.dec_dim, self.beta_min, self.beta_max = use_ref_t, dec_dim, beta_min, beta_max
        self.encoder = FwdDiffusion(n_feats, channels, filters, heads, layers, kernel, dropout, window_size, enc_dim,
                                    precision=precision)
        self.decoder = Diffusion(n_feats, dec_dim, spk_dim, use_ref_t, beta_min, beta_max, precision=precision)

    def load_encoder(self, enc_path):                                               # :77-79
        enc_dict = torch.load(enc_path, map_location=lambda loc, storage: loc)
        self.encoder.load_state_dict(enc_dict, strict=False)

    @torch.no_grad()
    # ragged=True (keyword only): each utterance of the padded batch is converted as the reference's own B = 1 call on it,
    # given the same draws: x_lengths go to the encoder's PostNet and the U-Net, x_ref_lengths to the reference's PostNet
    # and the RefBlock branch.  False: the reference's padded-batch semantics, byte for byte as before.
    def forward(self, x, x_lengths, x_ref, x_ref_lengths, c, n_timesteps, mode="ml", *, ragged=False):   # :82-127
        x, x_lengths = self.relocate_input([x, x_lengths])
        x_ref, x_ref_lengths, c = self.relocate_input([x_ref, x_ref_lengths, c])
        x_mask = sequence_mask(x_lengths).unsqueeze(1).to(x.dtype)
        x_ref_mask = sequence_mask(x_ref_lengths).unsqueeze(1).to(x_ref.dtype)
        if not ragged:
            mean = self.encoder(x, x_mask)
            mean_ref = self.encoder(x_ref, x_ref_mask)
            return convert_from_encoder(self.decoder, x, x_lengths, mean, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode)
        mean = self.encoder(x, x_mask, lengths=x_lengths)
        mean_ref = self.encoder(x_ref, x_ref_mask, lengths=x_ref_lengths)
        return convert_from_encoder(self.decoder, x, x_lengths, mean, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode,
                                    ragged=True, x_ref_lengths=x_ref_lengths)

    def rolling(self, capacity, max_frames):
        """A DiffVCRollingSampler: voice conversion of single utterances through a rolling decoder batch of `capacity` slots
        at up to `max_frames` U-Net frames (a multiple of 4).  submit(x, x_ref, c, n_timesteps, mode="ml") takes one
        utterance's B = 1 `forward` arguments; each result is that call's (mean_x, y)."""
        return self.decoder._rolling(DiffVCRollingSampler, capacity, max_frames, self)

    def compute_loss(self, x, x_lengths, x_ref, c):                                 # :129-144
        x, x_lengths, x_ref, c = self.relocate_input([x, x_lengths, x_ref, c])
        x_mask = sequence_mask(x_lengths).unsqueeze(1).to(x.dtype)
        mean = self.encoder(x, x_mask).detach()
        mean_ref = self.encoder(x_ref, x_mask).detach()                            # the reference uses x_mask here (:142)
        return self.decoder.compute_loss(x, x_mask, mean, x_ref, mean_ref, c)


class DiffVCRollingSampler(VcRollingSampler):
    """`DiffVC.rolling`: one utterance per request through a rolling batch of the model's decoder.

    submit(x [1, n_feats, L], x_ref [1, n_feats, R], c [1, 256], n_timesteps, mode="ml") runs the encoder on x and x_ref
    and forms the decoder's inputs as `DiffVC.forward` does at B = 1 (decoder_inputs: mean_x, the re-padded mean, and z's
    draw), then queues the decoder request, whose step noise is drawn after z, in `forward`'s order.  advance / drain return
    {id: (mean_x [1, n_feats, L], y [1, n_feats, L])}."""

    def __init__(self, model, engine, capacity, max_frames):
        self.model = model
        self._mean_x = {}
        super().__init__(engine, capacity, max_frames)

    def submit(self, x, x_ref, c, n_timesteps, mode="ml") -> int:
        F = self.engine.n_feats
        for name, v in (("x", x), ("x_ref", x_ref)):
            if not isinstance(v, torch.Tensor) or v.dim() != 3 or v.shape[-1] < 1:
                raise ValueError(f"{name}: expected a [1, {F}, frames] tensor, got {getattr(v, 'shape', type(v).__name__)}")
        L, R = x.shape[-1], x_ref.shape[-1]
        x, x_ref = self._tensor("x", x, (1, F, L)), self._tensor("x_ref", x_ref, (1, F, R))
        c = self._tensor("c", c, (1, 256))
        if fix_len_compatibility(L) > self.max_frames:
            raise ValueError(f"x has {L} frames: the decoder runs {fix_len_compatibility(L)} > max_frames = {self.max_frames}")
        self._steps(n_timesteps)
        if mode not in ("pf", "em", "ml"):
            raise ValueError(f"mode must be one of ['pf', 'em', 'ml'], got {mode!r}")
        x_mask, x_ref_mask = torch.ones(1, 1, L, device=self.device), torch.ones(1, 1, R, device=self.device)
        mean = self.model.encoder(x, x_mask)
        mean_ref = self.model.encoder(x_ref, x_ref_mask)
        mean_x, z, x_mask_new, mean_new, _ = decoder_inputs(self.model.decoder, x, torch.tensor([L], device=self.device), mean)
        rid = super().submit(z, x_mask_new, mean_new, x_ref, x_ref_mask, mean_ref, c, n_timesteps, mode)
        self._mean_x[rid] = mean_x
        return rid

    def _result(self, r, mel):
        mean_x = self._mean_x.pop(r.rid)
        return mean_x, mel[:, :, :mean_x.shape[-1]]
