"""Generate tests/golden/diffvc_ragged_golden.pt from the UNMODIFIED DiffVC model (container only: needs /root/reference or
the bytecode oracle/build_ref.py compiled from it).

A ragged DiffVC batch converted per utterance: the reference's DiffVC (DiffVC/model/vc.py, imported, not copied) runs each
utterance ALONE, at B = 1 - the call DiffVC/inference.ipynb makes - on the slices x[b, :, :L_b], x_ref[b, :, :R_b] of a
B = 4 batch with x_lengths {160, 131, 61, 1} (T = 160) and x_ref_lengths {97, 144, 130, 1} (T_ref = 144): the 128-pixel
seam, a level-0 edge inside the second tile, a length that is not a multiple of 4 and one-frame utterances.  N = 3 in 'pf'
and 'ml'.  The batch's draws are recorded (torch.manual_seed(NOISE_SEED), then randn [B, 80, T'] for the re-padded mean and
once per step), and utterance b replays their slices [b:b+1, :, :T'_b] - the draws a ragged batch row sees.  For contrast
the script also runs the reference's padded-batch DiffVC.forward on the whole batch with those draws.

Stored, as in make_golden_ragged_decoder.py, are digests rather than tensors: per output (mean_x, y) the SHA-256 of its fp32
bytes, its shape and its float64 L2 norm.  Weights (oracle/postnet_oracle.py: model_synthetic_weights) and inputs come back
from the seeds.  The script asserts that the oracle (oracle/postnet_oracle.py fwd_diffusion + oracle/diffvc_oracle.py
prepare_decoder_inputs / reverse_diffusion) reproduces every B = 1 mean_x bit for bit and every y bit for bit or within
rel-L2 1e-6, and records which (`oracle_bitwise`, `oracle_rel_l2`), so tests/test_vc_ragged.py can check the oracle against
the digests and the GPU tests compare the engine with the oracle's outputs.

    python scripts/make_golden_diffvc_ragged.py
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import diffvc_oracle as D, postnet_oracle as O, ref_import  # noqa: E402
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS, DiffVCConfig  # noqa: E402

SEED, NOISE_SEED = 6262, 91
B, T, TR, N = 4, 160, 144, 3
LENGTHS, REF_LENGTHS = [160, 131, 61, 1], [97, 144, 130, 1]
MODES = ("pf", "ml")


def fix_len(n):
    return n + (-n) % 4


def inputs():
    """x [B,80,T], x_ref [B,80,T_ref], c [B,256] (L2-normalised); every frame random, the padded ones too"""
    g = torch.Generator().manual_seed(SEED)
    x, x_ref, c = torch.randn(B, 80, T, generator=g), torch.randn(B, 80, TR, generator=g), torch.randn(B, 256, generator=g)
    return x, x_ref, c / c.norm(dim=1, keepdim=True)


def draws(mode):
    """the batch's draws: randn_like(mean_x_new) (vc.py:123), then randn_like(z) once per step in 'ml' (diffusion.py:194)"""
    torch.manual_seed(NOISE_SEED)
    return [torch.randn(B, 80, fix_len(T)) for _ in range(1 + (N if mode != "pf" else 0))]


def utterance(b, x, x_ref, c, noise):
    """utterance b's B = 1 inputs and draws: x[b, :, :L_b], x_ref[b, :, :R_b], noise[k][b:b+1, :, :T'_b]"""
    L, R = LENGTHS[b], REF_LENGTHS[b]
    return (x[b:b + 1, :, :L].contiguous(), torch.tensor([L]), x_ref[b:b + 1, :, :R].contiguous(), torch.tensor([R]),
            c[b:b + 1], [d[b:b + 1, :, :fix_len(L)].contiguous() for d in noise])


def oracle_forward(p, x, xl, xr, xrl, c, mode, noise):
    """DiffVC.forward (vc.py:82-127) restated with the oracle: (mean_x, y)"""
    cfg = DiffVCConfig()
    enc = {k[len("encoder."):]: v for k, v in p.items() if k.startswith("encoder.")}
    dec = {k[len("decoder."):]: v for k, v in p.items() if k.startswith("decoder.")}
    x_mask = (torch.arange(x.shape[2])[None, :] < xl[:, None]).to(x.dtype)[:, None]
    xr_mask = (torch.arange(xr.shape[2])[None, :] < xrl[:, None]).to(xr.dtype)[:, None]
    mean, mean_ref = O.fwd_diffusion(enc, x, x_mask), O.fwd_diffusion(enc, xr, xr_mask)
    d = D.prepare_decoder_inputs(cfg, x, xl, mean, noise[0])
    steps = torch.stack(noise[1:]) if len(noise) > 1 else None
    y = D.reverse_diffusion(dec, cfg, d["z"], d["x_mask_new"], d["mean_new"], xr, xr_mask, mean_ref, c, N, mode, steps)
    return d["mean_x"], y[:, :, :d["max_length"]]


def pin(t):
    t = t.detach().to(torch.float32).contiguous()
    return {"sha256": hashlib.sha256(t.numpy().tobytes()).hexdigest(), "shape": list(t.shape),
            "norm": float(t.double().norm())}


def run_reference(model, x, xl, xr, xrl, c, mode, noise):
    it = iter(noise)
    orig = torch.randn_like
    torch.randn_like = lambda t, **kw: next(it).clone()
    try:
        out = model(x, xl, xr, xrl, c, N, mode=mode)
    finally:
        torch.randn_like = orig
    assert next(it, None) is None
    return out


def main():
    ref_import.import_model("diffvc")
    import model.vc as rvc
    model = rvc.DiffVC(*DIFFVC_MODEL_ARGS)
    sd = O.model_synthetic_weights(SEED)
    model.load_state_dict(sd, strict=True)
    model.eval()
    x, x_ref, c = inputs()
    out = {"seed": SEED, "noise_seed": NOISE_SEED, "torch": torch.__version__, "B": B, "T": T, "T_ref": TR, "N": N,
           "lengths": LENGTHS, "ref_lengths": REF_LENGTHS, "cases": []}
    with torch.no_grad():
        for mode in MODES:
            noise = draws(mode)
            rows = []
            for b in range(B):
                args = utterance(b, x, x_ref, c, noise)
                mean_x, y = run_reference(model, *args[:5], mode, args[5])
                om, oy = oracle_forward(sd, *args[:5], mode, args[5])
                assert torch.equal(om, mean_x), f"oracle mean_x differs from the reference: {mode} row {b}"
                exact = torch.equal(oy, y)
                err = ((oy.double() - y.double()).norm() / y.double().norm()).item()
                assert exact or err <= 1e-6, f"oracle y differs from the reference: {mode} row {b}: rel-L2 {err:.3e}"
                rows.append({"mean_x": pin(mean_x), "y": pin(y), "oracle_bitwise": exact, "oracle_rel_l2": err})
                print(mode, "row", b, "y", tuple(y.shape), "oracle bit for bit" if exact else f"oracle rel-L2 {err:.3e}")
            pm, py = run_reference(model, x, torch.tensor(LENGTHS), x_ref, torch.tensor(REF_LENGTHS), c, mode, noise)
            out["cases"].append({"mode": mode, "rows": rows, "padded": {"mean_x": pin(pm), "y": pin(py)}})
    torch.save(out, os.path.join(ROOT, "tests", "golden", "diffvc_ragged_golden.pt"))
    print("wrote tests/golden/diffvc_ragged_golden.pt")


if __name__ == "__main__":
    main()
