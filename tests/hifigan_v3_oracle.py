"""CPU oracle (test infrastructure, not product) for HiFi-GAN generators with ResBlock2 blocks, the HiFi-GAN V3 config.

oracle/hifigan_oracle.py restates Grad-TTS/hifi-gan/models.py:77-128 with ResBlock1 (:13-49).  This module adds ResBlock2
(:53-74) and the Generator's choice between the two (:84: ResBlock1 for resblock == '1', ResBlock2 otherwise), in the same
plain PyTorch CPU fp32 ops over the effective weights (after remove_weight_norm).  A config without a ResBlock2 goes to
oracle/hifigan_oracle.py unchanged, so V1 results are the same tensors.

Pinned: scripts/make_golden_hifigan_v3.py builds the UNMODIFIED reference Generator from the V3 values below with seeded
weights, removes weight norm, and asserts this file reproduces its output (max abs diff 0) before writing
tests/golden/hifigan_v3_golden.pt; tests/test_hifigan_v3.py re-checks on every CPU run.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import hifigan_oracle as H

LRELU_SLOPE = H.LRELU_SLOPE

# the public HiFi-GAN config_v3.json (not in the reference tree; its Generator accepts these values unchanged)
V3 = dict(resblock="2", upsample_rates=[8, 8, 4], upsample_kernel_sizes=[16, 16, 8], upsample_initial_channel=256,
          resblock_kernel_sizes=[3, 5, 7], resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]], num_mels=80)


def is_rb2(h):
    """models.py:84: ResBlock2 unless resblock == '1' (V1's config in this project has no key: ResBlock1)"""
    return str(h.get("resblock", "1")) != "1"


def param_spec(h=V3):
    """[(name, shape)] of the generator's state_dict after remove_weight_norm: ResBlock2 has two convs per block,
    resblocks.n.convs.{0,1}, at the first two dilations (models.py:53-62)."""
    if not is_rb2(h):
        return H.param_spec(h)
    c0 = h["upsample_initial_channel"]
    spec = [("conv_pre.weight", (c0, h["num_mels"], 7)), ("conv_pre.bias", (c0,))]
    for i, k in enumerate(h["upsample_kernel_sizes"]):
        spec += [(f"ups.{i}.weight", (c0 // 2 ** i, c0 // 2 ** (i + 1), k)), (f"ups.{i}.bias", (c0 // 2 ** (i + 1),))]
    n, ch = 0, c0
    for i in range(len(h["upsample_rates"])):
        ch = c0 // 2 ** (i + 1)
        for k in h["resblock_kernel_sizes"]:
            for j in range(2):
                spec += [(f"resblocks.{n}.convs.{j}.weight", (ch, ch, k)), (f"resblocks.{n}.convs.{j}.bias", (ch,))]
            n += 1
    return spec + [("conv_post.weight", (1, ch, 7)), ("conv_post.bias", (1,))]


def resblock2(p, pre, x, k, dilations):
    """models.py:64-69: x = conv_d(lrelu(x)) + x for the block's two convs (dilations[0], dilations[1])."""
    for j, d in enumerate(dilations[:2]):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = F.conv1d(xt, p[f"{pre}.convs.{j}.weight"], p[f"{pre}.convs.{j}.bias"], padding=H.get_padding(k, d), dilation=d)
        x = xt + x
    return x


def generator(p, x, h=V3):
    """models.py:104-119 with the config's block: mel [B,80,T] -> waveform [B,1,T*prod(upsample_rates)]."""
    if not is_rb2(h):
        return H.generator(p, x, h)
    nk = len(h["resblock_kernel_sizes"])
    x = F.conv1d(x, p["conv_pre.weight"], p["conv_pre.bias"], padding=3)
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        x = F.leaky_relu(x, LRELU_SLOPE)
        x = F.conv_transpose1d(x, p[f"ups.{i}.weight"], p[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        xs = None
        for j in range(nk):
            r = resblock2(p, f"resblocks.{i * nk + j}", x, h["resblock_kernel_sizes"][j], h["resblock_dilation_sizes"][j])
            xs = r if xs is None else xs + r
        x = xs / nk
    x = F.leaky_relu(x)                       # models.py:115: default slope 0.01 here, not LRELU_SLOPE
    x = F.conv1d(x, p["conv_post.weight"], p["conv_post.bias"], padding=3)
    return torch.tanh(x)


def macs_per_mel_frame(h=V3):
    """Algorithmic multiply-accumulates per input mel frame (oracle/hifigan_oracle.py's count, with 2 convs per ResBlock2
    instead of 2 * len(dilations) per ResBlock1)."""
    if not is_rb2(h):
        return H.macs_per_mel_frame(h)
    total = h["upsample_initial_channel"] * h["num_mels"] * 7
    rate = 1
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        cin, cout = h["upsample_initial_channel"] // 2 ** i, h["upsample_initial_channel"] // 2 ** (i + 1)
        total += cin * cout * k * rate
        rate *= u
        for kk in h["resblock_kernel_sizes"]:
            total += 2 * cout * cout * kk * rate
    total += cout * 7 * rate
    return total
