"""CPU ORACLE (test infrastructure, not product) for DiffVC's encoder side: PostNet and FwdDiffusion.

Functional, state_dict-driven restatement of DiffVC/model/postnet.py and the FwdDiffusion forward of DiffVC/model/vc.py in
plain PyTorch CPU fp32 ops, plus the seeded weights of FwdDiffusion and of the whole DiffVC model.  Pinned by
scripts/make_golden_fwd_diffusion.py and scripts/make_golden_diffvc_e2e.py against the UNMODIFIED reference imported from
/root/reference/DiffVC.  Paths below are relative to /root/reference/DiffVC/.
"""
from __future__ import annotations

import torch.nn.functional as F

from .gradtts_oracle import mish


# ---------------------------------------------------------------------------------------------------------------
# The encoder side of DiffVC.forward: FwdDiffusion = MelEncoder + PostNet (DiffVC/model/vc.py:19-48)
# ---------------------------------------------------------------------------------------------------------------
def postnet(p, x, mask, pre="", groups=8):
    """PostNet.forward, model/postnet.py:47-53 (Block :21-23, ResnetBlock :33-37).  x [B,80,T], mask [B,1,T] -> [B,80,T]
    (not masked: a padded column is final_conv.bias)."""
    x, m = x.unsqueeze(1), mask.unsqueeze(1)
    h0 = F.conv2d(x * m, p[f"{pre}init_conv.weight"], p[f"{pre}init_conv.bias"])

    def block(name, y):
        q = f"{pre}res_block.{name}.block"
        y = F.conv2d(y * m, p[f"{q}.0.weight"], p[f"{q}.0.bias"], padding=3)
        y = F.group_norm(y, groups, p[f"{q}.1.weight"], p[f"{q}.1.bias"], eps=1e-5)
        return mish(y) * m
    h = block("block2", block("block1", h0))
    out = F.conv2d(h0 * m, p[f"{pre}res_block.res.weight"], p[f"{pre}res_block.res.bias"]) + h
    return F.conv2d(out * m, p[f"{pre}final_conv.weight"], p[f"{pre}final_conv.bias"]).squeeze(1)


def fwd_diffusion(p, x, mask):
    """FwdDiffusion.forward, model/vc.py:37-41: the mel encoder (text_encoder_oracle.mel_encoder) then the PostNet.
    `p` holds FwdDiffusion.state_dict() (`encoder.*`, `postnet.*`)."""
    from .text_encoder_oracle import mel_encoder
    z = mel_encoder({k[len("encoder."):]: v for k, v in p.items() if k.startswith("encoder.")}, x, mask)
    return postnet(p, z, mask, pre="postnet.")


def fwd_synthetic_weights(seed):
    """Seeded weights for FwdDiffusion(80, 192, 768, 2, 6, 3, 0.1, 4, 128).state_dict(): the mel encoder's
    (text_encoder_oracle.mel_synthetic_weights) under `encoder.`, the PostNet's (spec.py) under `postnet.`."""
    from speech_backbones_b200.spec import synthetic_postnet_state_dict
    from .text_encoder_oracle import mel_synthetic_weights
    sd = {"encoder." + k: v for k, v in mel_synthetic_weights(seed).items()}
    sd.update(synthetic_postnet_state_dict(128, seed, prefix="postnet."))
    return sd


def model_synthetic_weights(seed):
    """Seeded weights for the whole DiffVC(*DIFFVC_MODEL_ARGS).state_dict(), 346 tensors: FwdDiffusion's under `encoder.`
    and the decoder's (spec.py) under `decoder.`."""
    from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_state_dict
    sd = {"encoder." + k: v for k, v in fwd_synthetic_weights(seed).items()}
    cfg = DiffVCConfig()
    sd.update({"decoder." + k: v for k, v in synthetic_state_dict(cfg, seed, spec=diffvc_param_spec(cfg)).items()})
    return sd
