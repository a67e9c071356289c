"""Generate tests/golden/fwd_diffusion_golden.pt from the UNMODIFIED DiffVC PostNet and FwdDiffusion (container only: needs
/root/reference or the bytecode oracle/build_ref.py compiled from it).

Builds `PostNet(128)` (DiffVC/model/postnet.py:40-53) and `FwdDiffusion(80, 192, 768, 2, 6, 3, 0.1, 4, 128)`
(DiffVC/model/vc.py:19-41, DiffVC/params.py) from the reference tree, loads seeded weights strictly, asserts that
oracle/postnet_oracle.py:postnet / fwd_diffusion reproduce them (<= 1e-5 max abs), and stores ONLY the reference outputs;
tests rebuild weights and inputs from the seeds.  Ragged batches: B = 3 with a length-1 item, T = 5 (smaller than the 7x7
kernel), T = 128 (one pixel tile) and T = 203 (a partial second tile).

    python scripts/make_golden_fwd_diffusion.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import postnet_oracle as O, ref_import  # noqa: E402
from speech_backbones_b200.spec import postnet_param_spec, synthetic_postnet_state_dict  # noqa: E402

CASES = [dict(B=3, T=5, lengths=[5, 1, 3]), dict(B=2, T=128, lengths=[128, 77]), dict(B=3, T=203, lengths=[203, 1, 150])]
SEED = 8642


def case_inputs(seed, c):
    """x [B,80,T] (standard normal, padded columns included) and the prefix mask [B,1,T] of a case."""
    x = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(seed + c["T"]))
    mask = (torch.arange(c["T"])[None, :] < torch.tensor(c["lengths"])[:, None]).float()[:, None]
    return x, mask


def main():
    ref_import.import_model("diffvc")
    import model.postnet as rpn
    import model.vc as rvc
    pn = rpn.PostNet(128).eval()
    psd = synthetic_postnet_state_dict(128, SEED)
    assert {k: tuple(v.shape) for k, v in pn.state_dict().items()} == postnet_param_spec(128)
    pn.load_state_dict(psd, strict=True)
    fwd = rvc.FwdDiffusion(80, 192, 768, 2, 6, 3, 0.1, 4, 128).eval()
    fsd = O.fwd_synthetic_weights(SEED)
    fwd.load_state_dict(fsd, strict=True)
    out = {"seed": SEED, "torch": torch.__version__, "nparams_postnet": sum(v.numel() for v in psd.values()),
           "nparams_fwd": sum(v.numel() for v in fsd.values()), "postnet": [], "fwd": []}
    for c in CASES:
        x, mask = case_inputs(SEED, c)
        with torch.no_grad():
            y, yo = pn(x, mask), O.postnet(psd, x, mask)
            z, zo = fwd(x, mask), O.fwd_diffusion(fsd, x, mask)
        e1, e2 = (y - yo).abs().max().item(), (z - zo).abs().max().item()
        print(c, "oracle vs reference max abs: postnet %.2e, fwd_diffusion %.2e" % (e1, e2))
        assert e1 <= 1e-5 and e2 <= 1e-5
        out["postnet"].append(dict(c, out=y))
        out["fwd"].append(dict(c, out=z))
    torch.save(out, os.path.join(ROOT, "tests", "golden", "fwd_diffusion_golden.pt"))
    print("wrote tests/golden/fwd_diffusion_golden.pt", out["nparams_postnet"], out["nparams_fwd"])


if __name__ == "__main__":
    main()
