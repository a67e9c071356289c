"""Parameter inventory of the Grad-TTS score U-Net and deterministic synthetic data.

The reference ships no checkpoints (SURVEY.md section 8c), so every parity test,
the smoke test and bench.py run on weights produced by `synthetic_state_dict`:
each tensor is drawn from its own seeded CPU generator, keyed by its
state_dict name, so the values are independent of module construction order
and identical on every machine with the same torch build.

Names/shapes follow Grad-TTS/model/diffusion.py:128-172 (GradLogPEstimator2d.__init__):
`estimator.downs.{l}.{0,1}` ResnetBlock, `.2` Residual(Rezero(LinearAttention)),
`.3` Downsample; `mid_block1/mid_attn/mid_block2`; `ups.{l}.{0..3}`; final_block; final_conv.
"""
from __future__ import annotations

import hashlib
import math
from dataclasses import dataclass

import torch

ATTN_HEADS = 4
ATTN_DIM_HEAD = 32
ATTN_HIDDEN = ATTN_HEADS * ATTN_DIM_HEAD   # 128, diffusion.py:83-86
GN_GROUPS = 8                              # diffusion.py:50


@dataclass(frozen=True)
class UNetConfig:
    """Constructor arguments of Diffusion (Grad-TTS/model/diffusion.py:228-230)."""
    n_feats: int = 80
    dim: int = 64
    n_spks: int = 1
    spk_emb_dim: int = 64
    beta_min: float = 0.05
    beta_max: float = 20.0
    pe_scale: float = 1000.0

    @property
    def in_channels(self) -> int:
        return 2 + (1 if self.n_spks > 1 else 0)

    @property
    def level_dims(self):
        return [self.in_channels, self.dim, self.dim * 2, self.dim * 4]


def resnet_layout(cfg: UNetConfig):
    """Ordered list of (prefix, cin, cout) of the 12 ResnetBlocks, execution order.

    Mirrors the constructor loops at diffusion.py:146-170: three down levels
    (the last without Downsample), two mid blocks, two up levels fed by
    cat(x, skip) (hence cin = 2*cout_of_level).
    """
    d = cfg.level_dims
    out = []
    for l in range(3):
        out.append((f"estimator.downs.{l}.0", d[l], d[l + 1]))
        out.append((f"estimator.downs.{l}.1", d[l + 1], d[l + 1]))
    out.append(("estimator.mid_block1", d[3], d[3]))
    out.append(("estimator.mid_block2", d[3], d[3]))
    # reversed(in_out[1:]) = [(d2, d3), (d1, d2)]
    for j, (cin, cout) in enumerate([(d[2], d[3]), (d[1], d[2])]):
        out.append((f"estimator.ups.{j}.0", cout * 2, cin))
        out.append((f"estimator.ups.{j}.1", cin, cin))
    return out


def attention_layout(cfg: UNetConfig):
    """Ordered list of (prefix, channels) of the 6 LinearAttention blocks."""
    d = cfg.level_dims
    return [("estimator.downs.0.2", d[1]), ("estimator.downs.1.2", d[2]),
            ("estimator.downs.2.2", d[3]), ("estimator.mid_attn", d[3]),
            ("estimator.ups.0.2", d[2]), ("estimator.ups.1.2", d[1])]


def estimator_param_spec(cfg: UNetConfig):
    """Ordered {name: shape} for every tensor under `estimator.` (172 for n_spks=1)."""
    dim = cfg.dim
    spec: dict[str, tuple] = {}
    if cfg.n_spks > 1:
        spec["estimator.spk_mlp.0.weight"] = (cfg.spk_emb_dim * 4, cfg.spk_emb_dim)
        spec["estimator.spk_mlp.0.bias"] = (cfg.spk_emb_dim * 4,)
        spec["estimator.spk_mlp.2.weight"] = (cfg.n_feats, cfg.spk_emb_dim * 4)
        spec["estimator.spk_mlp.2.bias"] = (cfg.n_feats,)
    spec["estimator.mlp.0.weight"] = (dim * 4, dim)
    spec["estimator.mlp.0.bias"] = (dim * 4,)
    spec["estimator.mlp.2.weight"] = (dim, dim * 4)
    spec["estimator.mlp.2.bias"] = (dim,)

    def resnet(prefix, cin, cout):
        spec[f"{prefix}.mlp.1.weight"] = (cout, dim)
        spec[f"{prefix}.mlp.1.bias"] = (cout,)
        for blk, ci in (("block1", cin), ("block2", cout)):
            spec[f"{prefix}.{blk}.block.0.weight"] = (cout, ci, 3, 3)
            spec[f"{prefix}.{blk}.block.0.bias"] = (cout,)
            spec[f"{prefix}.{blk}.block.1.weight"] = (cout,)
            spec[f"{prefix}.{blk}.block.1.bias"] = (cout,)
        if cin != cout:
            spec[f"{prefix}.res_conv.weight"] = (cout, cin, 1, 1)
            spec[f"{prefix}.res_conv.bias"] = (cout,)

    def attn(prefix, c):
        spec[f"{prefix}.fn.g"] = (1,)
        spec[f"{prefix}.fn.fn.to_qkv.weight"] = (ATTN_HIDDEN * 3, c, 1, 1)
        spec[f"{prefix}.fn.fn.to_out.weight"] = (c, ATTN_HIDDEN, 1, 1)
        spec[f"{prefix}.fn.fn.to_out.bias"] = (c,)

    rl = {p: (ci, co) for p, ci, co in resnet_layout(cfg)}
    al = dict(attention_layout(cfg))
    d = cfg.level_dims
    for l in range(3):
        for k in (0, 1):
            p = f"estimator.downs.{l}.{k}"
            resnet(p, *rl[p])
        attn(f"estimator.downs.{l}.2", al[f"estimator.downs.{l}.2"])
        if l < 2:
            spec[f"estimator.downs.{l}.3.conv.weight"] = (d[l + 1], d[l + 1], 3, 3)
            spec[f"estimator.downs.{l}.3.conv.bias"] = (d[l + 1],)
    resnet("estimator.mid_block1", *rl["estimator.mid_block1"])
    attn("estimator.mid_attn", al["estimator.mid_attn"])
    resnet("estimator.mid_block2", *rl["estimator.mid_block2"])
    for j in range(2):
        for k in (0, 1):
            p = f"estimator.ups.{j}.{k}"
            resnet(p, *rl[p])
        c = al[f"estimator.ups.{j}.2"]
        attn(f"estimator.ups.{j}.2", c)
        spec[f"estimator.ups.{j}.3.conv.weight"] = (c, c, 4, 4)   # ConvTranspose2d: [Cin, Cout, 4, 4]
        spec[f"estimator.ups.{j}.3.conv.bias"] = (c,)
    spec["estimator.final_block.block.0.weight"] = (dim, dim, 3, 3)
    spec["estimator.final_block.block.0.bias"] = (dim,)
    spec["estimator.final_block.block.1.weight"] = (dim,)
    spec["estimator.final_block.block.1.bias"] = (dim,)
    spec["estimator.final_conv.weight"] = (1, dim, 1, 1)
    spec["estimator.final_conv.bias"] = (1,)
    return spec


def _key_seed(seed: int, name: str) -> int:
    h = hashlib.sha256(f"{seed}:{name}".encode()).digest()
    return int.from_bytes(h[:7], "little")


def synthetic_tensor(seed: int, name: str, shape, kind: str = "normal") -> torch.Tensor:
    g = torch.Generator(device="cpu")
    g.manual_seed(_key_seed(seed, name))
    if kind == "normal":
        return torch.randn(*shape, generator=g, dtype=torch.float32)
    if kind == "uniform":
        return torch.rand(*shape, generator=g, dtype=torch.float32) * 2.0 - 1.0
    raise ValueError(kind)


def synthetic_state_dict(cfg: UNetConfig, seed: int = 1234, rezero_g: float = 0.02,
                         spec=None) -> dict[str, torch.Tensor]:
    """Seeded weights with PyTorch-default-like scales (uniform +-1/sqrt(fan_in)).

    `Rezero.g` is set to `rezero_g` (not the reference's 0 init, diffusion.py:43):
    a zero gate would leave all six LinearAttention blocks untested (SURVEY.md 8c).
    GroupNorm affine is perturbed away from (1, 0) so gamma/beta handling is exercised.
    """
    sd = {}
    for name, shape in (spec or estimator_param_spec(cfg)).items():
        if name.endswith(".fn.g") or name.endswith(".g") and len(shape) == 1 and shape[0] == 1:
            sd[name] = torch.full(shape, float(rezero_g), dtype=torch.float32)
        elif ".block.1." in name or ".norm." in name or (".ref_block.block" in name and ".1." in name):   # GroupNorm / InstanceNorm affine
            base = 1.0 if name.endswith("weight") else 0.0
            sd[name] = base + 0.1 * synthetic_tensor(seed, name, shape)
        elif name.endswith("bias"):
            sd[name] = 0.05 * synthetic_tensor(seed, name, shape, "uniform")
        else:
            if len(shape) == 4 and ".3.conv." in name and shape[2] == 4:
                fan_in = shape[0] * 4      # ConvTranspose2d 4x4 s2: 4 taps reach each output
            else:
                fan_in = int(math.prod(shape[1:]))
            sd[name] = synthetic_tensor(seed, name, shape, "uniform") / math.sqrt(fan_in)
    return sd


def synthetic_inputs(B: int, T: int, n_feats: int = 80, seed: int = 1234, ragged: bool = False,
                     n_spks: int = 1, spk_emb_dim: int = 64):
    """(z, mask, mu, spk, lengths) as GradTTS.forward builds them (tts.py:84-94):
    mu = N(0,1), z = mu + N(0,1)/1.5, mask = prefix-ones [B,1,T].  `ragged` draws
    lengths from U{T/2..T} (parity runs); otherwise full masks (throughput runs)."""
    mu = synthetic_tensor(seed, f"mu:{B}x{T}", (B, n_feats, T))
    z = mu + synthetic_tensor(seed, f"eps:{B}x{T}", (B, n_feats, T)) / 1.5
    if ragged:
        g = torch.Generator(device="cpu")
        g.manual_seed(_key_seed(seed, f"len:{B}x{T}"))
        lengths = torch.randint(max(1, T // 2), T + 1, (B,), generator=g)
        lengths[0] = T
    else:
        lengths = torch.full((B,), T, dtype=torch.long)
    mask = (torch.arange(T)[None, :] < lengths[:, None]).to(torch.float32)[:, None, :]
    spk = None
    if n_spks > 1:
        spk = synthetic_tensor(seed, f"spk:{B}", (B, spk_emb_dim))
    return z, mask, mu, spk, lengths


def synthetic_encoder_outputs(B: int, Tx: int, x_lengths, dur_mean: float = 1.0, n_feats: int = 80, seed: int = 1234):
    """Seeded stand-ins for the text encoder's outputs (Grad-TTS/model/tts.py:75): mu_x [B,n_feats,Tx],
    logw [B,1,Tx] (log durations ~ N(dur_mean, 0.5)), x_mask [B,1,Tx] from `x_lengths`; masked positions are zeroed the
    way the encoder leaves them."""
    g = torch.Generator().manual_seed(_key_seed(seed, f"encoder_outputs/{B}/{Tx}"))
    lengths = torch.tensor(list(x_lengths), dtype=torch.long)
    x_mask = (torch.arange(Tx)[None, :] < lengths[:, None]).to(torch.float32)[:, None, :]
    mu_x = torch.randn(B, n_feats, Tx, generator=g) * x_mask
    logw = (torch.randn(B, 1, Tx, generator=g) * 0.5 + dur_mean) * x_mask
    return mu_x, logw, x_mask


HIFIGAN_V1 = dict(upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=512,
                  resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]], num_mels=80)


def hifigan_param_spec(h=None):
    """[(name, shape)] of the HiFi-GAN V1 generator's state_dict after remove_weight_norm
    (Grad-TTS/hifi-gan/models.py:77-101, Grad-TTS/checkpts/hifigan-config.json; inference.py:60-63)."""
    h = h or HIFIGAN_V1
    c0 = h["upsample_initial_channel"]
    spec = [("conv_pre.weight", (c0, h["num_mels"], 7)), ("conv_pre.bias", (c0,))]
    for i, k in enumerate(h["upsample_kernel_sizes"]):
        spec += [(f"ups.{i}.weight", (c0 // 2 ** i, c0 // 2 ** (i + 1), k)), (f"ups.{i}.bias", (c0 // 2 ** (i + 1),))]
    n, ch = 0, c0
    for i in range(len(h["upsample_rates"])):
        ch = c0 // 2 ** (i + 1)
        for k, d in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
            for grp in ("convs1", "convs2"):
                for j in range(len(d)):
                    spec += [(f"resblocks.{n}.{grp}.{j}.weight", (ch, ch, k)), (f"resblocks.{n}.{grp}.{j}.bias", (ch,))]
            n += 1
    return spec + [("conv_post.weight", (1, ch, 7)), ("conv_post.bias", (1,))]


def synthetic_hifigan_state_dict(seed: int = 1234, h=None):
    """Seeded weights for a HiFi-GAN generator (`h`, default V1) after remove_weight_norm: the reference ships no vocoder
    checkpoint.  He-style scales (std = 1/sqrt(fan_in)) keep the activations O(1) through the 15-conv-deep residual stacks,
    so the tanh output is neither saturated nor vanishing."""
    import math
    sd = {}
    for name, shape in hifigan_param_spec(h):
        g = torch.Generator().manual_seed(_key_seed(seed, "hifigan/" + name))
        if name.endswith(".bias"):
            sd[name] = torch.randn(shape, generator=g) * 0.02
        else:
            fan_in = shape[1] * shape[2] if not name.startswith("ups.") else shape[0] * shape[2] / 4.0
            sd[name] = torch.randn(shape, generator=g) / math.sqrt(fan_in)
    return sd


def synthetic_noise(N: int, B: int, T: int, n_feats: int = 80, seed: int = 1234) -> torch.Tensor:
    """Pre-drawn per-step noise [N,B,n_feats,T] for the stochastic sampler (diffusion.py:267)."""
    return synthetic_tensor(seed, f"noise:{N}x{B}x{T}", (N, B, n_feats, T))


# ---------------------------------------------------------------------------------------------
# DiffVC decoder (DiffVC/model/diffusion.py:17-59, DiffVC/model/modules.py:128-154)
# ---------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class DiffVCConfig:
    """Constructor arguments of DiffVC's Diffusion (DiffVC/model/diffusion.py:110; params.py:26-28)."""
    n_feats: int = 80
    dim_unet: int = 256
    dim_spk: int = 128
    use_ref_t: bool = True
    beta_min: float = 0.05
    beta_max: float = 20.0

    @property
    def level_dims(self):
        return [2 + self.dim_spk, self.dim_unet, self.dim_unet * 2, self.dim_unet * 4]


def diffvc_param_spec(cfg: DiffVCConfig):
    """Ordered {name: shape} of the 206 tensors under `estimator.` of DiffVC's decoder."""
    dim, dc = cfg.dim_unet, cfg.dim_spk
    spec: dict[str, tuple] = {}
    spec["estimator.mlp.0.weight"] = (dim * 4, dim)
    spec["estimator.mlp.0.bias"] = (dim * 4,)
    spec["estimator.mlp.2.weight"] = (dim, dim * 4)
    spec["estimator.mlp.2.bias"] = (dim,)
    cond_total = dim + 256
    if cfg.use_ref_t:
        base = dc // 4
        spec["estimator.ref_block.mlp1.1.weight"] = (base, dim)
        spec["estimator.ref_block.mlp1.1.bias"] = (base,)
        spec["estimator.ref_block.mlp2.1.weight"] = (2 * base, dim)
        spec["estimator.ref_block.mlp2.1.bias"] = (2 * base,)
        for name, ci, co in (("block11", 1, 2 * base), ("block12", base, 2 * base), ("block21", base, 4 * base),
                             ("block22", 2 * base, 4 * base), ("block31", 2 * base, 8 * base),
                             ("block32", 4 * base, 8 * base)):
            spec[f"estimator.ref_block.{name}.0.weight"] = (co, ci, 3, 3)
            spec[f"estimator.ref_block.{name}.0.bias"] = (co,)
            spec[f"estimator.ref_block.{name}.1.weight"] = (co,)
            spec[f"estimator.ref_block.{name}.1.bias"] = (co,)
        spec["estimator.ref_block.final_conv.weight"] = (dc, 4 * base, 1, 1)
        spec["estimator.ref_block.final_conv.bias"] = (dc,)
        cond_total += dc
    spec["estimator.cond_block.0.weight"] = (4 * dc, cond_total)
    spec["estimator.cond_block.0.bias"] = (4 * dc,)
    spec["estimator.cond_block.2.weight"] = (dc, 4 * dc)
    spec["estimator.cond_block.2.bias"] = (dc,)
    d = cfg.level_dims

    def resnet(prefix, cin, cout):
        spec[f"{prefix}.mlp.1.weight"] = (cout, dim)
        spec[f"{prefix}.mlp.1.bias"] = (cout,)
        for blk, ci in (("block1", cin), ("block2", cout)):
            spec[f"{prefix}.{blk}.block.0.weight"] = (cout, ci, 3, 3)
            spec[f"{prefix}.{blk}.block.0.bias"] = (cout,)
            spec[f"{prefix}.{blk}.block.1.weight"] = (cout,)
            spec[f"{prefix}.{blk}.block.1.bias"] = (cout,)
        if cin != cout:
            spec[f"{prefix}.res_conv.weight"] = (cout, cin, 1, 1)
            spec[f"{prefix}.res_conv.bias"] = (cout,)

    def attn(prefix, c):
        spec[f"{prefix}.fn.g"] = (1,)
        spec[f"{prefix}.fn.fn.to_qkv.weight"] = (ATTN_HIDDEN * 3, c, 1, 1)
        spec[f"{prefix}.fn.fn.to_out.weight"] = (c, ATTN_HIDDEN, 1, 1)
        spec[f"{prefix}.fn.fn.to_out.bias"] = (c,)

    for l in range(3):
        resnet(f"estimator.downs.{l}.0", d[l], d[l + 1])
        resnet(f"estimator.downs.{l}.1", d[l + 1], d[l + 1])
        attn(f"estimator.downs.{l}.2", d[l + 1])
        if l < 2:
            spec[f"estimator.downs.{l}.3.conv.weight"] = (d[l + 1], d[l + 1], 3, 3)
            spec[f"estimator.downs.{l}.3.conv.bias"] = (d[l + 1],)
    resnet("estimator.mid_block1", d[3], d[3])
    attn("estimator.mid_attn", d[3])
    resnet("estimator.mid_block2", d[3], d[3])
    for j, (cin, cout) in enumerate([(d[2], d[3]), (d[1], d[2])]):
        resnet(f"estimator.ups.{j}.0", cout * 2, cin)
        resnet(f"estimator.ups.{j}.1", cin, cin)
        attn(f"estimator.ups.{j}.2", cin)
        spec[f"estimator.ups.{j}.3.conv.weight"] = (cin, cin, 4, 4)
        spec[f"estimator.ups.{j}.3.conv.bias"] = (cin,)
    spec["estimator.final_block.block.0.weight"] = (dim, dim, 3, 3)
    spec["estimator.final_block.block.0.bias"] = (dim,)
    spec["estimator.final_block.block.1.weight"] = (dim,)
    spec["estimator.final_block.block.1.bias"] = (dim,)
    spec["estimator.final_conv.weight"] = (1, dim, 1, 1)
    spec["estimator.final_conv.bias"] = (1,)
    return spec


def synthetic_diffvc_inputs(B: int, T: int, T_ref: int, n_feats: int = 80, seed: int = 1234, ragged: bool = False):
    """(z, mask, mean, ref, ref_mask, mean_ref, c) as DiffVC.forward builds them (DiffVC/model/vc.py:104-125):
    z = mean + N(0,1); c = L2-normalised 256-d speaker embedding."""
    mean = synthetic_tensor(seed, f"vc_mean:{B}x{T}", (B, n_feats, T))
    z = mean + synthetic_tensor(seed, f"vc_eps:{B}x{T}", (B, n_feats, T))
    ref = synthetic_tensor(seed, f"vc_ref:{B}x{T_ref}", (B, n_feats, T_ref))
    mean_ref = synthetic_tensor(seed, f"vc_mean_ref:{B}x{T_ref}", (B, n_feats, T_ref))
    c = synthetic_tensor(seed, f"vc_c:{B}", (B, 256))
    c = c / c.norm(dim=1, keepdim=True)

    def lens(tag, n):
        if not ragged:
            return torch.full((B,), n, dtype=torch.long)
        g = torch.Generator(device="cpu")
        g.manual_seed(_key_seed(seed, f"{tag}:{B}x{n}"))
        l = torch.randint(max(1, n // 2), n + 1, (B,), generator=g)
        l[0] = n
        return l
    mask = (torch.arange(T)[None, :] < lens("vc_len", T)[:, None]).to(torch.float32)[:, None, :]
    ref_mask = (torch.arange(T_ref)[None, :] < lens("vc_reflen", T_ref)[:, None]).to(torch.float32)[:, None, :]
    return z, mask, mean, ref, ref_mask, mean_ref, c


# ---------------------------------------------------------------------------------------------
# DiffVC encoder side: FwdDiffusion = MelEncoder + PostNet (DiffVC/model/vc.py:19-48, postnet.py:15-53)
# ---------------------------------------------------------------------------------------------
def postnet_param_spec(dim: int = 128, prefix: str = ""):
    """Ordered {name: shape} of PostNet(dim).state_dict() (DiffVC/model/postnet.py:40-45): 14 tensors."""
    spec = {f"{prefix}init_conv.weight": (dim, 1, 1, 1), f"{prefix}init_conv.bias": (dim,)}
    for blk in ("block1", "block2"):
        q = f"{prefix}res_block.{blk}.block"
        spec.update({f"{q}.0.weight": (dim, dim, 7, 7), f"{q}.0.bias": (dim,), f"{q}.1.weight": (dim,), f"{q}.1.bias": (dim,)})
    spec.update({f"{prefix}res_block.res.weight": (dim, dim, 1, 1), f"{prefix}res_block.res.bias": (dim,),
                 f"{prefix}final_conv.weight": (1, dim, 1, 1), f"{prefix}final_conv.bias": (1,)})
    return spec


def synthetic_postnet_state_dict(dim: int = 128, seed: int = 1234, prefix: str = ""):
    """Seeded PostNet weights at PyTorch's default init scale (conv weights and biases uniform +-1/sqrt(fan_in)); the
    GroupNorm affine is perturbed away from (1, 0) so that gamma / beta handling is exercised."""
    sd = {}
    for name, shape in postnet_param_spec(dim, prefix).items():
        if ".block.1." in name:
            sd[name] = (1.0 if name.endswith("weight") else 0.0) + 0.1 * synthetic_tensor(seed, "postnet/" + name, shape)
        else:
            wshape = postnet_param_spec(dim, prefix)[name[:-len("bias")] + "weight"] if name.endswith("bias") else shape
            fan_in = int(math.prod(wshape[1:]))
            sd[name] = synthetic_tensor(seed, "postnet/" + name, shape, "uniform") / math.sqrt(fan_in)
    return sd


DIFFVC_MODEL_ARGS = (80, 192, 768, 2, 6, 3, 0.1, 4, 128, 128, True, 256, 0.05, 20.0)   # DiffVC/inference.ipynb, params.py


def mel_encoder_param_spec(n_feats=80, ch=192, filt=768, n_heads=2, n_layers=6, kernel=3, window=4, prefix=""):
    """Ordered {name: shape} of DiffVC's MelEncoder.state_dict() (DiffVC/model/encoder.py:258-277)."""
    s = {f"{prefix}init_proj.weight": (ch, n_feats, 1), f"{prefix}init_proj.bias": (ch,)}
    for i in range(3):
        q = f"{prefix}prenet"
        s.update({f"{q}.conv_layers.{i}.weight": (ch, ch, 5), f"{q}.conv_layers.{i}.bias": (ch,),
                  f"{q}.norm_layers.{i}.gamma": (ch,), f"{q}.norm_layers.{i}.beta": (ch,)})
    s.update({f"{prefix}prenet.proj.weight": (ch, ch, 1), f"{prefix}prenet.proj.bias": (ch,)})
    for i in range(n_layers):
        a = f"{prefix}encoder.attn_layers.{i}"
        s.update({f"{a}.emb_rel_k": (1, 2 * window + 1, ch // n_heads), f"{a}.emb_rel_v": (1, 2 * window + 1, ch // n_heads)})
        for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
            s.update({f"{a}.{c}.weight": (ch, ch, 1), f"{a}.{c}.bias": (ch,)})
        e = f"{prefix}encoder"
        s.update({f"{e}.norm_layers_1.{i}.gamma": (ch,), f"{e}.norm_layers_1.{i}.beta": (ch,),
                  f"{e}.ffn_layers.{i}.conv_1.weight": (filt, ch, kernel), f"{e}.ffn_layers.{i}.conv_1.bias": (filt,),
                  f"{e}.ffn_layers.{i}.conv_2.weight": (ch, filt, kernel), f"{e}.ffn_layers.{i}.conv_2.bias": (ch,),
                  f"{e}.norm_layers_2.{i}.gamma": (ch,), f"{e}.norm_layers_2.{i}.beta": (ch,)})
    s.update({f"{prefix}term_proj.weight": (n_feats, ch, 1), f"{prefix}term_proj.bias": (n_feats,)})
    return s


def diffvc_model_param_spec(args=DIFFVC_MODEL_ARGS):
    """Ordered {name: shape} of the whole DiffVC(*args).state_dict() (DiffVC/model/vc.py:52-75): `encoder.encoder.*`
    (MelEncoder), `encoder.postnet.*` (PostNet), `decoder.estimator.*` - 346 tensors, 126,259,128 parameters."""
    n_feats, ch, filt, heads, layers, kernel, _, window, enc_dim, spk_dim, use_ref_t, dec_dim, bmin, bmax = args
    spec = mel_encoder_param_spec(n_feats, ch, filt, heads, layers, kernel, window, prefix="encoder.encoder.")
    spec.update(postnet_param_spec(enc_dim, prefix="encoder.postnet."))
    dec = diffvc_param_spec(DiffVCConfig(n_feats, dec_dim, spk_dim, use_ref_t, bmin, bmax))
    spec.update({"decoder." + k: v for k, v in dec.items()})
    return spec
