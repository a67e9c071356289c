"""Generate tests/golden/diffvc_e2e_golden.pt from the UNMODIFIED DiffVC model (container only: needs /root/reference or the
bytecode oracle/build_ref.py compiled from it).

Builds `DiffVC(80, 192, 768, 2, 6, 3, 0.1, 4, 128, 128, True, 256, 0.05, 20.0)` (DiffVC/inference.ipynb) from the reference
tree, loads the seeded 346-tensor state_dict strictly (oracle/postnet_oracle.py:model_synthetic_weights) and records
`DiffVC.forward` (DiffVC/model/vc.py:82-127) at B = 2, ragged T = 64 / T_ref = 48, N = 3, in 'pf' and 'ml' modes.  Stored:
the outputs (mean_x, y), the encoder outputs mean and mean_ref, and the tensors the reference's randn_like drew (re-drawn
after re-seeding; the script checks that replaying them reproduces y bit for bit).  Weights and inputs are rebuilt from the
seeds by the tests.

    python scripts/make_golden_diffvc_e2e.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import postnet_oracle as O, ref_import  # noqa: E402
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS  # noqa: E402

SEED, NOISE_SEED = 5151, 77
B, T, TR, N = 2, 64, 48, 3
LENGTHS, REF_LENGTHS = [64, 41], [48, 30]


def inputs(seed):
    """x [B,80,T], x_lengths, x_ref [B,80,T_ref], x_ref_lengths, c [B,256] (L2-normalised speaker embedding)."""
    g = torch.Generator().manual_seed(seed)
    x, x_ref, c = torch.randn(B, 80, T, generator=g), torch.randn(B, 80, TR, generator=g), torch.randn(B, 256, generator=g)
    return x, torch.tensor(LENGTHS), x_ref, torch.tensor(REF_LENGTHS), c / c.norm(dim=1, keepdim=True)


def main():
    ref_import.import_model("diffvc")
    import model.vc as rvc
    model = rvc.DiffVC(*DIFFVC_MODEL_ARGS)
    model.load_state_dict(O.model_synthetic_weights(SEED), strict=True)
    model.eval()
    assert model.nparams == 126_259_128
    x, xl, xr, xrl, c = inputs(SEED)
    out = {"seed": SEED, "noise_seed": NOISE_SEED, "torch": torch.__version__, "B": B, "T": T, "T_ref": TR, "N": N,
           "lengths": LENGTHS, "ref_lengths": REF_LENGTHS, "cases": []}
    with torch.no_grad():
        x_mask = (torch.arange(T)[None, :] < xl[:, None]).float()[:, None]
        xr_mask = (torch.arange(TR)[None, :] < xrl[:, None]).float()[:, None]
        mean, mean_ref = model.encoder(x, x_mask), model.encoder(xr, xr_mask)
        for mode in ("pf", "ml"):
            torch.manual_seed(NOISE_SEED)
            mean_x, y = model(x, xl, xr, xrl, c, N, mode=mode)
            # the draws: randn_like(mean_x_new) (vc.py:123), then randn_like(z) once per step in 'ml' (diffusion.py:194)
            t_new = T + (-T) % 4
            torch.manual_seed(NOISE_SEED)
            noise = [torch.randn(B, 80, t_new) for _ in range(1 + (N if mode != "pf" else 0))]
            it = iter(noise)
            orig = torch.randn_like
            torch.randn_like = lambda t, **kw: next(it).clone()
            try:
                mx2, y2 = model(x, xl, xr, xrl, c, N, mode=mode)
            finally:
                torch.randn_like = orig
            assert next(it, None) is None and torch.equal(mx2, mean_x) and torch.equal(y2, y)
            print(mode, "mean_x", tuple(mean_x.shape), "y", tuple(y.shape), "draws", len(noise))
            out["cases"].append(dict(mode=mode, mean_x=mean_x, y=y, noise=torch.stack(noise)))
    out["mean"], out["mean_ref"] = mean, mean_ref
    torch.save(out, os.path.join(ROOT, "tests", "golden", "diffvc_e2e_golden.pt"))
    print("wrote tests/golden/diffvc_e2e_golden.pt")


if __name__ == "__main__":
    main()
