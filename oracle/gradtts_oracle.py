"""CPU ORACLE (test infrastructure, not product) for the Grad-TTS reverse-diffusion sampler.

A functional, state_dict-driven restatement of the reference algorithm in plain
PyTorch CPU fp32 ops.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this file; the product path
(speech-backbones_b200/) never does.

Pinned: `scripts/make_golden.py` runs THIS file and the unmodified reference
modules (imported from /root/reference) on identical weights/inputs and asserts
agreement before writing tests/golden/*.pt; tests/test_oracle.py re-checks the
oracle against those committed reference outputs on every run.  The reference
itself holds no golden vectors for this path (SURVEY.md 8c), so the imported
reference module is the anchor.

Every function cites the reference lines it restates (paths relative to
/root/reference/Grad-TTS/).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

HEADS = 4          # model/diffusion.py:83
GROUPS = 8         # model/diffusion.py:50


def mish(x):
    """model/diffusion.py:16-18: x * tanh(softplus(x))."""
    return x * torch.tanh(F.softplus(x))


def _tap(taps, name, value):
    """test hook: record an intermediate (NCHW) under the name libsbk's debug reader uses"""
    if taps is not None:
        taps[name] = value.detach().clone()


def conv_gn_mish(p, pre, x, mask, taps=None):
    """Block.forward, model/diffusion.py:56-58: Mish(GN8(Conv3x3(x*mask)))*mask."""
    y = F.conv2d(x * mask, p[f"{pre}.block.0.weight"], p[f"{pre}.block.0.bias"], padding=1)
    _tap(taps, f"{pre}.raw", y)
    y = F.group_norm(y, GROUPS, p[f"{pre}.block.1.weight"], p[f"{pre}.block.1.bias"], eps=1e-5)
    return mish(y) * mask


def resnet(p, pre, x, mask, temb, taps=None):
    """ResnetBlock.forward, model/diffusion.py:74-79.  The time projection is added
    AFTER block1's output mask (so padded columns become non-zero)."""
    h = conv_gn_mish(p, f"{pre}.block1", x, mask, taps)
    h = h + F.linear(mish(temb), p[f"{pre}.mlp.1.weight"], p[f"{pre}.mlp.1.bias"])[:, :, None, None]
    h = conv_gn_mish(p, f"{pre}.block2", h, mask, taps)
    wname = f"{pre}.res_conv.weight"
    xm = x * mask
    res = F.conv2d(xm, p[wname], p[f"{pre}.res_conv.bias"]) if wname in p else xm
    _tap(taps, f"{pre}.out", h + res)
    return h + res


def rezero_linear_attention(p, pre, x, taps=None):
    """Residual(Rezero(LinearAttention)), model/diffusion.py:39-46,82-110.
    softmax over ALL H*W positions of k (no mask); context = k v^T; out = context^T q."""
    b, c, h, w = x.shape
    qkv = F.conv2d(x, p[f"{pre}.fn.fn.to_qkv.weight"])
    qkv = qkv.reshape(b, 3, HEADS, -1, h * w)            # 'b (qkv heads c) h w -> qkv b heads c (h w)'
    q, k, v = qkv[:, 0], qkv[:, 1], qkv[:, 2]
    k = k.softmax(dim=-1)
    ctx = torch.einsum("bhdn,bhen->bhde", k, v)
    _tap(taps, f"{pre}.ctx", ctx)
    out = torch.einsum("bhde,bhdn->bhen", ctx, q).reshape(b, -1, h, w)
    out = F.conv2d(out, p[f"{pre}.fn.fn.to_out.weight"], p[f"{pre}.fn.fn.to_out.bias"])
    _tap(taps, f"{pre}.out", out * p[f"{pre}.fn.g"] + x)
    return out * p[f"{pre}.fn.g"] + x


def sinusoid(t, dim, scale):
    """SinusoidalPosEmb.forward, model/diffusion.py:118-125."""
    half = dim // 2
    f = math.log(10000) / (half - 1)
    # the fp32 frequency table and the fp32 argument are evaluated on the CPU whatever t's device and dtype: at scale 1000 the
    # argument reaches ~1000 rad, where one ulp of a frequency (a GPU expf may differ from the CPU's) or a float64 argument
    # moves it by ~3e-5 (bit-identical to before for fp32 CPU t)
    f = torch.exp(torch.arange(half).float() * -f)
    e = ((scale * t.detach().cpu().float())[:, None] * f[None, :]).to(t.device, t.dtype)
    return torch.cat((e.sin(), e.cos()), dim=-1)


def estimator(p, cfg, x, mask, mu, t, spk=None, taps=None):
    """GradLogPEstimator2d.forward, model/diffusion.py:174-216.
    x, mu: [B,80,T]; mask: [B,1,T]; t: [B]; spk: None or [B,spk_emb_dim] -> [B,80,T]."""
    pre = "estimator"
    temb = sinusoid(t, cfg.dim, cfg.pe_scale)
    temb = F.linear(temb, p[f"{pre}.mlp.0.weight"], p[f"{pre}.mlp.0.bias"])
    temb = F.linear(mish(temb), p[f"{pre}.mlp.2.weight"], p[f"{pre}.mlp.2.bias"])
    if cfg.n_spks < 2:
        h = torch.stack([mu, x], 1)
    else:
        s = F.linear(spk, p[f"{pre}.spk_mlp.0.weight"], p[f"{pre}.spk_mlp.0.bias"])
        s = F.linear(mish(s), p[f"{pre}.spk_mlp.2.weight"], p[f"{pre}.spk_mlp.2.bias"])
        h = torch.stack([mu, x, s[:, :, None].repeat(1, 1, x.shape[-1])], 1)
    m = mask[:, None]                                       # [B,1,1,T]
    skips, masks = [], [m]
    for l in range(3):
        mk = masks[-1]
        h = resnet(p, f"{pre}.downs.{l}.0", h, mk, temb, taps)
        h = resnet(p, f"{pre}.downs.{l}.1", h, mk, temb, taps)
        h = rezero_linear_attention(p, f"{pre}.downs.{l}.2", h, taps)
        skips.append(h)
        if l < 2:
            h = F.conv2d(h * mk, p[f"{pre}.downs.{l}.3.conv.weight"],
                         p[f"{pre}.downs.{l}.3.conv.bias"], stride=2, padding=1)
            _tap(taps, f"{pre}.downs.{l}.3.out", h)
        else:
            h = h * mk                                      # Identity()(x * mask_down), :196
        masks.append(mk[:, :, :, ::2])
    masks = masks[:-1]
    mk = masks[-1]
    h = resnet(p, f"{pre}.mid_block1", h, mk, temb, taps)
    h = rezero_linear_attention(p, f"{pre}.mid_attn", h, taps)
    h = resnet(p, f"{pre}.mid_block2", h, mk, temb, taps)
    for j in range(2):
        mk = masks.pop()
        h = torch.cat((h, skips.pop()), dim=1)
        h = resnet(p, f"{pre}.ups.{j}.0", h, mk, temb, taps)
        h = resnet(p, f"{pre}.ups.{j}.1", h, mk, temb, taps)
        h = rezero_linear_attention(p, f"{pre}.ups.{j}.2", h, taps)
        h = F.conv_transpose2d(h * mk, p[f"{pre}.ups.{j}.3.conv.weight"],
                               p[f"{pre}.ups.{j}.3.conv.bias"], stride=2, padding=1)
        _tap(taps, f"{pre}.ups.{j}.3.out", h)
    h = conv_gn_mish(p, f"{pre}.final_block", h, m, taps)
    out = F.conv2d(h * m, p[f"{pre}.final_conv.weight"], p[f"{pre}.final_conv.bias"])
    return (out * m).squeeze(1)


def beta_t(t, beta_min, beta_max):
    """get_noise(cumulative=False), model/diffusion.py:219-224."""
    return beta_min + (beta_max - beta_min) * t


@torch.no_grad()
def reverse_diffusion(p, cfg, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None):
    """Diffusion.reverse_diffusion, model/diffusion.py:254-275.

    stoc=False: xt <- (xt - 0.5*(mu - xt - est)*beta*h)*mask
    stoc=True : xt <- (xt - ((0.5*(mu - xt) - est)*beta*h + eps*sqrt(beta*h)))*mask
                (est is NOT halved on this branch, :265).
    `noise` [N,B,80,T] supplies eps per step; if None it is drawn with torch.randn
    from the global generator in the reference's order (:267)."""
    h = 1.0 / n_timesteps
    xt = z * mask
    for i in range(n_timesteps):
        t = (1.0 - (i + 0.5) * h) * torch.ones(z.shape[0], dtype=z.dtype, device=z.device)
        bt = beta_t(t[:, None, None], cfg.beta_min, cfg.beta_max)
        est = estimator(p, cfg, xt, mask, mu, t, spk)
        if stoc:
            det = (0.5 * (mu - xt) - est) * bt * h
            eps = noise[i] if noise is not None else torch.randn(z.shape, dtype=z.dtype, device=z.device)
            dxt = det + eps * torch.sqrt(bt * h)
        else:
            dxt = 0.5 * (mu - xt - est) * bt * h
        xt = (xt - dxt) * mask
    return xt


# ---------------------------------------------------------------------------------------------------------------
# The step before the path (SURVEY.md 8f rank 2): GradTTS.forward between the text encoder and the decoder
# ---------------------------------------------------------------------------------------------------------------
def sequence_mask(length, max_length=None):
    """model/utils.py:6-10."""
    if max_length is None:
        max_length = length.max()
    x = torch.arange(int(max_length), dtype=length.dtype, device=length.device)
    return x.unsqueeze(0) < length.unsqueeze(1)


def fix_len_compatibility(length, num_downsamplings_in_unet=2):
    """model/utils.py:13-17."""
    while length % (2 ** num_downsamplings_in_unet) != 0:
        length += 1
    return length


def generate_path(duration, mask):
    """model/utils.py:26-39: path[b,i,t] = [t < cum_i] - [t < cum_(i-1)], times mask."""
    b, t_x, t_y = mask.shape
    cum_duration = torch.cumsum(duration, 1)
    path = sequence_mask(cum_duration.view(b * t_x), t_y).to(mask.dtype).view(b, t_x, t_y)
    path = path - F.pad(path, [0, 0, 1, 0, 0, 0])[:, :-1]
    return path * mask


def prior_expand(mu_x, logw, x_mask, length_scale=1.0, temperature=1.0, noise_tf=None):
    """model/tts.py:77-94.  mu_x [B,F,Tx], logw / x_mask [B,1,Tx]; noise_tf [B,Ty,F] = the draws of `randn_like(mu_y)`
    in the memory order of the reference's transposed mu_y (drawn from the global generator when None).
    Returns dict(y_lengths, y_max_length, y_mask [B,1,Ty], attn [B,1,Tx,Ty], mu_y [B,F,Ty], z [B,F,Ty])."""
    w = torch.exp(logw) * x_mask                                            # :77
    w_ceil = torch.ceil(w) * length_scale                                   # :78
    y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()        # :79
    y_max_length = int(y_lengths.max())                                     # :80
    y_max_length_ = fix_len_compatibility(y_max_length)                     # :81
    y_mask = sequence_mask(y_lengths, y_max_length_).unsqueeze(1).to(x_mask.dtype)              # :83
    attn_mask = x_mask.unsqueeze(-1) * y_mask.unsqueeze(2)                                      # :84
    attn = generate_path(w_ceil.squeeze(1), attn_mask.squeeze(1)).unsqueeze(1)                  # :85
    mu_y = torch.matmul(attn.squeeze(1).transpose(1, 2), mu_x.transpose(1, 2)).transpose(1, 2)  # :88-89
    if noise_tf is None:
        noise = torch.randn_like(mu_y)                                      # :94 (fills mu_y's transposed memory order)
    else:
        noise = noise_tf.transpose(1, 2)
    z = mu_y + noise / temperature                                          # :94
    return dict(w_ceil=w_ceil, y_lengths=y_lengths, y_max_length=y_max_length, y_mask=y_mask, attn=attn,
                mu_y=mu_y.contiguous(), z=z.contiguous())
