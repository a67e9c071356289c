"""CPU ORACLE (test infrastructure, not product) for the DiffVC reverse-diffusion sampler.

Functional, state_dict-driven restatement of DiffVC/model/diffusion.py + modules.py in plain PyTorch CPU
fp32 ops; the U-Net blocks are shared with the Grad-TTS oracle (the reference's modules.py:16-116 is the same
code as Grad-TTS/model/diffusion.py:16-110).  Pinned by scripts/make_golden_diffvc.py against the UNMODIFIED
reference imported from /root/reference/DiffVC, plus the reference's one known answer: the decoder holds
117,794,599 parameters (SURVEY.md 8c).  Paths below are relative to /root/reference/DiffVC/.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from .gradtts_oracle import conv_gn_mish, mish, resnet, rezero_linear_attention, sinusoid


def ref_block(p, pre, x, mask, temb):
    """RefBlock.forward, model/modules.py:156-166: 6 x (Conv3x3 -> InstanceNorm2d(affine) -> GLU), two time
    biases, 1x1 conv, masked mean over (mel, frames)."""
    def cig(name, y):
        y = F.conv2d(y * mask, p[f"{pre}.{name}.0.weight"], p[f"{pre}.{name}.0.bias"], padding=1)
        y = F.instance_norm(y, weight=p[f"{pre}.{name}.1.weight"], bias=p[f"{pre}.{name}.1.bias"], eps=1e-5)
        return F.glu(y, dim=1)
    y = cig("block11", x)
    y = cig("block12", y)
    y = y + F.linear(mish(temb), p[f"{pre}.mlp1.1.weight"], p[f"{pre}.mlp1.1.bias"])[:, :, None, None]
    y = cig("block21", y)
    y = cig("block22", y)
    y = y + F.linear(mish(temb), p[f"{pre}.mlp2.1.weight"], p[f"{pre}.mlp2.1.bias"])[:, :, None, None]
    y = cig("block31", y)
    y = cig("block32", y)
    y = F.conv2d(y * mask, p[f"{pre}.final_conv.weight"], p[f"{pre}.final_conv.bias"])
    return (y * mask).sum((2, 3)) / (mask.sum((2, 3)) * x.shape[2])


def conditioning(p, cfg, ref, ref_mask, c, t):
    """The xt-independent half of GradLogPEstimator.forward, model/diffusion.py:62-71: returns (temb [B,dim], cond [B,dim_spk])."""
    pre = "estimator"
    cond = sinusoid(t, cfg.dim_unet, 1000.0)                     # SinusoidalPosEmb hard-codes x1000, modules.py:123
    temb = F.linear(cond, p[f"{pre}.mlp.0.weight"], p[f"{pre}.mlp.0.bias"])
    temb = F.linear(mish(temb), p[f"{pre}.mlp.2.weight"], p[f"{pre}.mlp.2.bias"])
    if cfg.use_ref_t:
        cond = torch.cat([cond, ref_block(p, f"{pre}.ref_block", ref, ref_mask[:, None], temb)], 1)
    cond = torch.cat([cond, c], 1)
    cond = F.linear(cond, p[f"{pre}.cond_block.0.weight"], p[f"{pre}.cond_block.0.bias"])
    cond = F.linear(mish(cond), p[f"{pre}.cond_block.2.weight"], p[f"{pre}.cond_block.2.bias"])
    return temb, cond


def estimator(p, cfg, x, x_mask, mean, ref, ref_mask, c, t, taps=None):
    """GradLogPEstimator.forward, model/diffusion.py:61-106.  x, mean [B,80,T]; x_mask [B,1,T]; ref [B,1,80,Tr]
    (the stacked diffused reference); ref_mask [B,1,Tr]; c [B,256]; t [B]."""
    pre = "estimator"
    temb, cond = conditioning(p, cfg, ref, ref_mask, c, t)
    h = torch.stack([mean, x], 1)
    m = x_mask[:, None]
    h = torch.cat([h, cond[:, :, None, None].expand(-1, -1, h.shape[2], h.shape[3])], 1)
    skips, masks = [], [m]
    for l in range(3):
        mk = masks[-1]
        h = resnet(p, f"{pre}.downs.{l}.0", h, mk, temb, taps)
        h = resnet(p, f"{pre}.downs.{l}.1", h, mk, temb, taps)
        h = rezero_linear_attention(p, f"{pre}.downs.{l}.2", h, taps)
        skips.append(h)
        if l < 2:
            h = F.conv2d(h * mk, p[f"{pre}.downs.{l}.3.conv.weight"], p[f"{pre}.downs.{l}.3.conv.bias"], stride=2, padding=1)
        else:
            h = h * mk
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
        h = F.conv_transpose2d(h * mk, p[f"{pre}.ups.{j}.3.conv.weight"], p[f"{pre}.ups.{j}.3.conv.bias"], stride=2, padding=1)
    h = conv_gn_mish(p, f"{pre}.final_block", h, m, taps)
    out = F.conv2d(h * m, p[f"{pre}.final_conv.weight"], p[f"{pre}.final_conv.bias"])
    return (out * m).squeeze(1)


def _gamma(cfg, s, t, p=1.0):
    """get_gamma, model/diffusion.py:124-131 (host scalars)."""
    bi = cfg.beta_min + 0.5 * (cfg.beta_max - cfg.beta_min) * (t + s)
    bi *= (t - s)
    return math.exp(-0.5 * p * bi)


def step_coefficients(cfg, n_timesteps, i, mode):
    """Host scalars of step i, model/diffusion.py:169-193: returns (t, A, Bc, sigma, gamma0t) such that
    dxt = (mean - xt)*A - est*Bc + eps*sigma, and the diffused reference uses weight gamma(0,t)."""
    h = 1.0 / n_timesteps
    t = 1.0 - i * h
    beta_t = cfg.beta_min + (cfg.beta_max - cfg.beta_min) * t
    if mode == "pf":
        return t, 0.5 * beta_t * h, 0.5 * beta_t * h, 0.0, _gamma(cfg, 0, t)
    if mode == "ml":
        kappa = _gamma(cfg, 0, t - h) * (1.0 - _gamma(cfg, t - h, t, p=2.0))
        kappa /= (_gamma(cfg, 0, t) * beta_t * h)
        kappa -= 1.0
        ct = 1.0 - _gamma(cfg, 0, t, p=2.0)
        nu = _gamma(cfg, 0, t - h) * (1.0 - _gamma(cfg, t - h, t, p=2.0)) / ct
        mu = _gamma(cfg, t - h, t) * (1.0 - _gamma(cfg, 0, t - h, p=2.0)) / ct
        omega = nu / _gamma(cfg, 0, t)
        omega += mu
        omega -= (0.5 * beta_t * h + 1.0)
        sigma = math.sqrt((1.0 - _gamma(cfg, 0, t - h, p=2.0)) * (1.0 - _gamma(cfg, t - h, t, p=2.0)) / ct)
    else:
        kappa, omega, sigma = 0.0, 0.0, math.sqrt(beta_t * h)
    return t, 0.5 * beta_t * h + omega, (1.0 + kappa) * (beta_t * h), sigma, _gamma(cfg, 0, t)


@torch.no_grad()
def reverse_diffusion(p, cfg, z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode, noise=None):
    """Diffusion.reverse_diffusion, model/diffusion.py:164-196 (modes pf / em / ml; t_i = 1 - i/N).
    `noise` [N,B,80,T] supplies the per-step randn_like(z) of em/ml; None draws from the global generator."""
    xt = z * mask
    for i in range(n_timesteps):
        t, A, Bc, sigma, g0t = step_coefficients(cfg, n_timesteps, i, mode)
        time = t * torch.ones(z.shape[0], dtype=z.dtype, device=z.device)
        xt_ref = ((ref * g0t + mean_ref * (1.0 - g0t)) * ref_mask)[:, None]          # compute_diffused_mean, :151-155
        est = estimator(p, cfg, xt, mask, mean, xt_ref, ref_mask, c, time)
        if mode == "pf":
            dxt = 0.5 * (mean - xt - est) * (2.0 * A)
        else:
            dxt = (mean - xt) * A
            dxt = dxt - est * Bc
            eps = noise[i] if noise is not None else torch.randn_like(z)
            dxt = dxt + eps * sigma
        xt = (xt - dxt) * mask
    return xt


# ---------------------------------------------------------------------------------------------------------------
# The step before the path (SURVEY.md 8f rank 2, DiffVC): DiffVC.forward between the encoders and the decoder
# ---------------------------------------------------------------------------------------------------------------
def prepare_decoder_inputs(cfg, x, x_lengths, mean, noise=None):
    """DiffVC/model/vc.py:104,107,110-123 as written there (the per-sample copy loop included).
    Returns dict(x_mask, mean_x, max_length, x_mask_new, mean_new, z)."""
    def sequence_mask(length, max_length=None):                  # DiffVC/model/utils.py
        if max_length is None:
            max_length = length.max()
        r = torch.arange(int(max_length), dtype=length.dtype, device=length.device)
        return r.unsqueeze(0) < length.unsqueeze(1)

    x_mask = sequence_mask(x_lengths).unsqueeze(1).to(x.dtype)                                   # :104
    g = _gamma(cfg, 0, 1.0)
    mean_x = (x * g + mean * (1.0 - g)) * x_mask                                                 # :107, diffusion.py:151-155
    b = x.shape[0]
    max_length = int(x_lengths.max())
    max_length_new = max_length
    while max_length_new % 4 != 0:
        max_length_new += 1
    x_mask_new = sequence_mask(x_lengths, max_length_new).unsqueeze(1).to(x.dtype)
    mean_new = torch.zeros((b, x.shape[1], max_length_new), dtype=x.dtype)
    mean_x_new = torch.zeros((b, x.shape[1], max_length_new), dtype=x.dtype)
    for i in range(b):
        mean_new[i, :, :x_lengths[i]] = mean[i, :, :x_lengths[i]]
        mean_x_new[i, :, :x_lengths[i]] = mean_x[i, :, :x_lengths[i]]
    z = mean_x_new + (torch.randn_like(mean_x_new) if noise is None else noise)
    return dict(x_mask=x_mask, mean_x=mean_x, max_length=max_length, x_mask_new=x_mask_new, mean_new=mean_new, z=z)
