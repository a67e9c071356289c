"""CPU ORACLE (test infrastructure, not product) for the Grad-TTS text encoder (SURVEY.md 8f rank 4; the module whose outputs
feed the glue in front of the hot path): Grad-TTS/model/text_encoder.py:281-326 (TextEncoder) with its ConvReluNorm prenet
(:32-64), the 6-layer relative-position transformer (:96-278) and the duration predictor (:67-93), eval mode (no dropout).

Functional, state_dict-driven, plain PyTorch CPU fp32.  The windowed relative-position attention is restated DIRECTLY -
    scores[i,j] += q_i . E_k[j-i+w] / sqrt(d)   and   out_i += sum_j p[i,j] E_v[j-i+w]     for |j-i| <= w
- instead of through the reference's pad / reshape skewing tricks (:186-207), so agreement with the reference also checks
that reading of them.  Only tests/ may import this file; no product kernel exists for this row.
Pinned by scripts/make_golden_text_encoder.py against the UNMODIFIED reference TextEncoder (strict load of the seeded weights)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def param_spec(n_vocab=149, n_feats=80, ch=192, filt=768, filt_dp=256, n_layers=6, kernel=3, window=4, n_heads=2, spk_extra=0):
    """[(name, shape)] of TextEncoder.state_dict() (text_encoder.py:281-310); spk_extra = spk_emb_dim when n_spks > 1 (the
    encoder, proj_m and proj_w then run on n_channels + spk_emb_dim channels, :305-310)."""
    s = [("emb.weight", (n_vocab, ch))]
    for i in range(3):
        s += [(f"prenet.conv_layers.{i}.weight", (ch, ch, 5)), (f"prenet.conv_layers.{i}.bias", (ch,)),
              (f"prenet.norm_layers.{i}.gamma", (ch,)), (f"prenet.norm_layers.{i}.beta", (ch,))]
    s += [("prenet.proj.weight", (ch, ch, 1)), ("prenet.proj.bias", (ch,))]
    ch = ch + spk_extra
    for i in range(n_layers):
        a = f"encoder.attn_layers.{i}"
        s += [(f"{a}.emb_rel_k", (1, 2 * window + 1, ch // n_heads)), (f"{a}.emb_rel_v", (1, 2 * window + 1, ch // n_heads))]
        for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
            s += [(f"{a}.{c}.weight", (ch, ch, 1)), (f"{a}.{c}.bias", (ch,))]
        s += [(f"encoder.norm_layers_1.{i}.gamma", (ch,)), (f"encoder.norm_layers_1.{i}.beta", (ch,)),
              (f"encoder.ffn_layers.{i}.conv_1.weight", (filt, ch, kernel)), (f"encoder.ffn_layers.{i}.conv_1.bias", (filt,)),
              (f"encoder.ffn_layers.{i}.conv_2.weight", (ch, filt, kernel)), (f"encoder.ffn_layers.{i}.conv_2.bias", (ch,)),
              (f"encoder.norm_layers_2.{i}.gamma", (ch,)), (f"encoder.norm_layers_2.{i}.beta", (ch,))]
    s += [("proj_m.weight", (n_feats, ch, 1)), ("proj_m.bias", (n_feats,)),
          ("proj_w.conv_1.weight", (filt_dp, ch, kernel)), ("proj_w.conv_1.bias", (filt_dp,)),
          ("proj_w.norm_1.gamma", (filt_dp,)), ("proj_w.norm_1.beta", (filt_dp,)),
          ("proj_w.conv_2.weight", (filt_dp, filt_dp, kernel)), ("proj_w.conv_2.bias", (filt_dp,)),
          ("proj_w.norm_2.gamma", (filt_dp,)), ("proj_w.norm_2.beta", (filt_dp,)),
          ("proj_w.proj.weight", (1, filt_dp, 1)), ("proj_w.proj.bias", (1,))]
    return s


def synthetic_weights(seed, spk_extra=0, **config):
    """Seeded stand-in weights (the reference ships no Grad-TTS checkpoint): 1/sqrt(fan_in) scales, LayerNorm gains near 1.
    `config`: param_spec's shape arguments (n_heads, kernel, window, filt, ...); each tensor depends only on the seed, its
    name and its shape, so the defaults give Grad-TTS's tensors."""
    from speech_backbones_b200.spec import synthetic_tensor
    sd = {}
    for name, shape in param_spec(spk_extra=spk_extra, **config):
        if name.endswith(".gamma"):
            sd[name] = 1.0 + 0.1 * synthetic_tensor(seed, "textenc/" + name, shape)
        elif name.endswith((".beta", ".bias")):
            sd[name] = 0.05 * synthetic_tensor(seed, "textenc/" + name, shape)
        else:
            conv = not name.startswith("emb") and "emb_rel" not in name
            fan_in = shape[1] * (shape[2] if len(shape) > 2 else 1) if conv else shape[-1]
            sd[name] = synthetic_tensor(seed, "textenc/" + name, shape) / fan_in ** 0.5
    return sd


def layer_norm(x, gamma, beta, eps=1e-4):
    """:11-29: normalise over the channel axis (dim 1), biased variance, eps 1e-4."""
    m = x.mean(1, keepdim=True)
    v = ((x - m) ** 2).mean(1, keepdim=True)
    return (x - m) * torch.rsqrt(v + eps) * gamma[None, :, None] + beta[None, :, None]


def rel_attention(p, pre, x, mask, n_heads, window):
    """MultiHeadAttention.forward for self-attention (:133-171), eval mode, in x's dtype and on x's device."""
    b, ch, t = x.shape
    d = ch // n_heads
    q = F.conv1d(x, p[f"{pre}.conv_q.weight"], p[f"{pre}.conv_q.bias"]).view(b, n_heads, d, t).transpose(2, 3)   # [b,h,t,d]
    k = F.conv1d(x, p[f"{pre}.conv_k.weight"], p[f"{pre}.conv_k.bias"]).view(b, n_heads, d, t).transpose(2, 3)
    v = F.conv1d(x, p[f"{pre}.conv_v.weight"], p[f"{pre}.conv_v.bias"]).view(b, n_heads, d, t).transpose(2, 3)
    scores = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(d)
    ek, ev = p[f"{pre}.emb_rel_k"][0], p[f"{pre}.emb_rel_v"][0]                   # [2w+1, d], shared by the heads
    idx = torch.arange(t, device=x.device)
    zero = torch.zeros((), dtype=x.dtype, device=x.device)
    rel = idx[None, :] - idx[:, None]                                              # j - i
    band = rel.abs() <= window
    slot = (rel + window).clamp(0, 2 * window)
    qe = torch.matmul(q, ek.t())                                                   # [b,h,t,2w+1]: q_i . E_k[r]
    scores = scores + torch.where(band, qe.gather(-1, slot.expand(b, n_heads, t, t)), zero) / math.sqrt(d)
    scores = scores.masked_fill(mask == 0, -1e4)
    pa = F.softmax(scores, dim=-1)
    out = torch.matmul(pa, v)
    # sum_j p[i,j] E_v[j-i+w] over the band = (band weights scattered by relative offset) @ E_v
    wrel = torch.zeros(b, n_heads, t, 2 * window + 1, dtype=x.dtype, device=x.device)
    wrel.scatter_add_(-1, slot.expand(b, n_heads, t, t), torch.where(band, pa, zero))
    out = out + torch.matmul(wrel, ev)
    out = out.transpose(2, 3).contiguous().view(b, ch, t)
    return F.conv1d(out, p[f"{pre}.conv_o.weight"], p[f"{pre}.conv_o.bias"])


def text_encoder(p, x, x_lengths, n_heads=2, n_layers=6, kernel=3, window=4, spk=None):
    """TextEncoder.forward (:312-326): token ids [B,Tx] -> (mu_x [B,80,Tx], logw [B,1,Tx], x_mask [B,1,Tx]).  spk [B,E] for a
    multi-speaker model: concatenated to every token after the prenet (:317-318).  Runs in the weights' dtype (float32, or
    float64 for a high-precision reference) on the tensors' device."""
    ch = p["emb.weight"].shape[1]
    h = (F.embedding(x, p["emb.weight"]) * math.sqrt(ch)).transpose(1, -1)
    t = h.shape[2]
    x_mask = (torch.arange(t, device=h.device)[None, :] < x_lengths[:, None]).unsqueeze(1).to(h.dtype)
    # prenet: ConvReluNorm (:57-64)
    org = h
    for i in range(3):
        h = F.conv1d(h * x_mask, p[f"prenet.conv_layers.{i}.weight"], p[f"prenet.conv_layers.{i}.bias"], padding=2)
        h = torch.relu(layer_norm(h, p[f"prenet.norm_layers.{i}.gamma"], p[f"prenet.norm_layers.{i}.beta"]))
    h = (org + F.conv1d(h, p["prenet.proj.weight"], p["prenet.proj.bias"])) * x_mask
    if spk is not None:
        h = torch.cat([h, spk.unsqueeze(-1).repeat(1, 1, h.shape[-1])], dim=1)
    # encoder (:267-278)
    attn_mask = x_mask.unsqueeze(2) * x_mask.unsqueeze(-1)
    for i in range(n_layers):
        h = h * x_mask
        y = rel_attention(p, f"encoder.attn_layers.{i}", h, attn_mask, n_heads, window)
        h = layer_norm(h + y, p[f"encoder.norm_layers_1.{i}.gamma"], p[f"encoder.norm_layers_1.{i}.beta"])
        y = F.conv1d(h * x_mask, p[f"encoder.ffn_layers.{i}.conv_1.weight"], p[f"encoder.ffn_layers.{i}.conv_1.bias"], padding=kernel // 2)
        y = F.conv1d(torch.relu(y) * x_mask, p[f"encoder.ffn_layers.{i}.conv_2.weight"], p[f"encoder.ffn_layers.{i}.conv_2.bias"],
                     padding=kernel // 2) * x_mask
        h = layer_norm(h + y, p[f"encoder.norm_layers_2.{i}.gamma"], p[f"encoder.norm_layers_2.{i}.beta"])
    h = h * x_mask
    mu = F.conv1d(h, p["proj_m.weight"], p["proj_m.bias"]) * x_mask
    # duration predictor (:83-93)
    d = F.conv1d(h * x_mask, p["proj_w.conv_1.weight"], p["proj_w.conv_1.bias"], padding=kernel // 2)
    d = layer_norm(torch.relu(d), p["proj_w.norm_1.gamma"], p["proj_w.norm_1.beta"])
    d = F.conv1d(d * x_mask, p["proj_w.conv_2.weight"], p["proj_w.conv_2.bias"], padding=kernel // 2)
    d = layer_norm(torch.relu(d), p["proj_w.norm_2.gamma"], p["proj_w.norm_2.beta"])
    logw = F.conv1d(d * x_mask, p["proj_w.proj.weight"], p["proj_w.proj.bias"]) * x_mask
    return mu, logw, x_mask


# ---- DiffVC "average voice" mel encoder (DiffVC/model/encoder.py:257-284): the same prenet and encoder blocks around 1x1 projections
def mel_param_spec(n_feats=80, ch=192, filt=768, n_layers=6, kernel=3, window=4, n_heads=2):
    """[(name, shape)] of MelEncoder.state_dict() (DiffVC/model/encoder.py:258-277; DiffVC/params.py:16-22)."""
    s = [("init_proj.weight", (ch, n_feats, 1)), ("init_proj.bias", (ch,))]
    for i in range(3):
        s += [(f"prenet.conv_layers.{i}.weight", (ch, ch, 5)), (f"prenet.conv_layers.{i}.bias", (ch,)),
              (f"prenet.norm_layers.{i}.gamma", (ch,)), (f"prenet.norm_layers.{i}.beta", (ch,))]
    s += [("prenet.proj.weight", (ch, ch, 1)), ("prenet.proj.bias", (ch,))]
    for i in range(n_layers):
        a = f"encoder.attn_layers.{i}"
        s += [(f"{a}.emb_rel_k", (1, 2 * window + 1, ch // n_heads)), (f"{a}.emb_rel_v", (1, 2 * window + 1, ch // n_heads))]
        for c in ("conv_q", "conv_k", "conv_v", "conv_o"):
            s += [(f"{a}.{c}.weight", (ch, ch, 1)), (f"{a}.{c}.bias", (ch,))]
        s += [(f"encoder.norm_layers_1.{i}.gamma", (ch,)), (f"encoder.norm_layers_1.{i}.beta", (ch,)),
              (f"encoder.ffn_layers.{i}.conv_1.weight", (filt, ch, kernel)), (f"encoder.ffn_layers.{i}.conv_1.bias", (filt,)),
              (f"encoder.ffn_layers.{i}.conv_2.weight", (ch, filt, kernel)), (f"encoder.ffn_layers.{i}.conv_2.bias", (ch,)),
              (f"encoder.norm_layers_2.{i}.gamma", (ch,)), (f"encoder.norm_layers_2.{i}.beta", (ch,))]
    s += [("term_proj.weight", (n_feats, ch, 1)), ("term_proj.bias", (n_feats,))]
    return s


def mel_synthetic_weights(seed, **config):
    """As synthetic_weights, for MelEncoder; `config`: mel_param_spec's shape arguments (defaults: DiffVC's)."""
    from speech_backbones_b200.spec import synthetic_tensor
    sd = {}
    for name, shape in mel_param_spec(**config):
        if name.endswith(".gamma"):
            sd[name] = 1.0 + 0.1 * synthetic_tensor(seed, "melenc/" + name, shape)
        elif name.endswith((".beta", ".bias")):
            sd[name] = 0.05 * synthetic_tensor(seed, "melenc/" + name, shape)
        else:
            fan_in = shape[1] * (shape[2] if len(shape) > 2 else 1) if "emb_rel" not in name else shape[-1]
            sd[name] = synthetic_tensor(seed, "melenc/" + name, shape) / fan_in ** 0.5
    return sd


def mel_encoder(p, x, x_mask, n_heads=2, n_layers=6, kernel=3, window=4):
    """MelEncoder.forward (DiffVC/model/encoder.py:279-284): mel [B,80,T], x_mask [B,1,T] -> "average voice" mel [B,80,T]."""
    h = F.conv1d(x * x_mask, p["init_proj.weight"], p["init_proj.bias"])
    org = h
    for i in range(3):                                                          # ConvReluNorm (:62-69)
        h = F.conv1d(h * x_mask, p[f"prenet.conv_layers.{i}.weight"], p[f"prenet.conv_layers.{i}.bias"], padding=2)
        h = torch.relu(layer_norm(h, p[f"prenet.norm_layers.{i}.gamma"], p[f"prenet.norm_layers.{i}.beta"]))
    h = (org + F.conv1d(h, p["prenet.proj.weight"], p["prenet.proj.bias"])) * x_mask
    attn_mask = x_mask.unsqueeze(2) * x_mask.unsqueeze(-1)
    for i in range(n_layers):                                                   # Encoder (:243-254)
        h = h * x_mask
        y = rel_attention(p, f"encoder.attn_layers.{i}", h, attn_mask, n_heads, window)
        h = layer_norm(h + y, p[f"encoder.norm_layers_1.{i}.gamma"], p[f"encoder.norm_layers_1.{i}.beta"])
        y = F.conv1d(h * x_mask, p[f"encoder.ffn_layers.{i}.conv_1.weight"], p[f"encoder.ffn_layers.{i}.conv_1.bias"], padding=kernel // 2)
        y = F.conv1d(torch.relu(y) * x_mask, p[f"encoder.ffn_layers.{i}.conv_2.weight"], p[f"encoder.ffn_layers.{i}.conv_2.bias"],
                     padding=kernel // 2) * x_mask
        h = layer_norm(h + y, p[f"encoder.norm_layers_2.{i}.gamma"], p[f"encoder.norm_layers_2.{i}.beta"])
    h = h * x_mask
    return F.conv1d(h * x_mask, p["term_proj.weight"], p["term_proj.bias"])
