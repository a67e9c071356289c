"""Generate tests/golden/gradtts_ragged_golden.pt from the UNMODIFIED reference (container only).

A ragged batch computed per utterance: the reference's Diffusion (/root/reference/Grad-TTS/model/diffusion.py, imported,
not copied) runs each utterance ALONE, at B = 1 and T_b = fix_len_compatibility(lengths[b]) frames - the call
Grad-TTS/inference.py:72-81 makes - on the [:T_b] slices of a B = 5, T = 512 batch with lengths {512, 301, 260, 130, 1}.
Cases: one estimator call with a different t per row; an N = 10 trajectory (stoc=False); an N = 5 trajectory with
stoc=True, utterance b drawing its noise after torch.manual_seed(NOISE_SEED + b) (so the batch's noise[:, b, :, :T_b] is
known: `utterance_noise`); an n_spks = 4 estimator call.  For contrast the script also runs the reference's padded-batch
estimator call (B = 5 at T = 512, the padded columns live).

The outputs themselves are not stored - 1.8 MB of fp32 would be most of the golden directory - but pinned: per output the
SHA-256 of its fp32 bytes, its shape and its float64 L2 norm, with the case descriptions; weights and inputs come back from
the seeds in speech_backbones_b200.spec.  The script asserts that oracle/gradtts_oracle.py reproduces every output bit for
bit, so the oracle's outputs ARE the reference's: tests/test_ragged_decoder.py checks the oracle against the digests, and
the GPU tests compare the engine with those oracle outputs.

    python scripts/make_golden_ragged_decoder.py
"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.gradtts import fix_len_compatibility  # noqa: E402
from oracle import gradtts_oracle as O  # noqa: E402
from _ref_import import import_gradtts  # noqa: E402

SEED, NOISE_SEED = 1234, 7
B, T = 5, 512
LENGTHS = [512, 301, 260, 130, 1]
T_EST = [0.9, 0.5, 0.3, 0.7, 0.1]
CASES = [dict(kind="est", n_spks=1), dict(kind="traj", n_spks=1, N=10, stoc=False),
         dict(kind="traj", n_spks=1, N=5, stoc=True), dict(kind="est", n_spks=4)]


def batch_inputs(n_spks):
    """z, mask, mu, spk of the batch: z / mu random on every frame (the padded ones too), mask from LENGTHS"""
    z, _, mu, spk, _ = synthetic_inputs(B, T, seed=SEED, n_spks=n_spks)
    L = torch.tensor(LENGTHS, dtype=torch.int64)
    mask = (torch.arange(T)[None, :] < L[:, None]).to(torch.float32)[:, None, :]
    return z, mask, mu, spk


def utterance_noise(b, N):
    """the noise utterance b's stoc call draws: torch.manual_seed(NOISE_SEED + b), then randn([1, 80, T_b]) per step"""
    torch.manual_seed(NOISE_SEED + b)
    Tb = fix_len_compatibility(LENGTHS[b])
    return torch.stack([torch.randn(1, 80, Tb) for _ in range(N)])


def pin(t):
    """what the golden keeps of an fp32 output: SHA-256 of its bytes, shape, float64 L2 norm"""
    t = t.detach().to(torch.float32).contiguous()
    return {"sha256": hashlib.sha256(t.numpy().tobytes()).hexdigest(), "shape": list(t.shape),
            "norm": t.double().norm().item()}


def main():
    md = import_gradtts()
    out = {"seed": SEED, "noise_seed": NOISE_SEED, "B": B, "T": T, "lengths": LENGTHS, "t": T_EST, "cases": [],
           "torch": torch.__version__}
    for case in CASES:
        cfg = UNetConfig(n_spks=case["n_spks"])
        sd = synthetic_state_dict(cfg, SEED)
        ref = md.Diffusion(cfg.n_feats, cfg.dim, n_spks=cfg.n_spks, spk_emb_dim=cfg.spk_emb_dim, beta_min=cfg.beta_min,
                           beta_max=cfg.beta_max, pe_scale=cfg.pe_scale).eval()
        ref.load_state_dict(sd, strict=True)
        z, mask, mu, spk = batch_inputs(case["n_spks"])
        t = torch.tensor(T_EST)
        rows = []
        with torch.no_grad():
            for b in range(B):
                Tb = fix_len_compatibility(LENGTHS[b])
                zb, mb, mub = z[b:b + 1, :, :Tb], mask[b:b + 1, :, :Tb], mu[b:b + 1, :, :Tb]
                sb = None if spk is None else spk[b:b + 1]
                if case["kind"] == "est":
                    y = ref.estimator(zb * mb, mb, mub, t[b:b + 1], sb)
                    y_orc = O.estimator(sd, cfg, zb * mb, mb, mub, t[b:b + 1], sb)
                else:
                    torch.manual_seed(NOISE_SEED + b)
                    y = ref(zb, mb, mub, case["N"], case["stoc"], sb)
                    noise = utterance_noise(b, case["N"]) if case["stoc"] else None
                    y_orc = O.reverse_diffusion(sd, cfg, zb, mb, mub, case["N"], case["stoc"], sb, noise)
                assert torch.isfinite(y).all(), (case, b)
                assert torch.equal(y, y_orc), (case, b, (y - y_orc).abs().max().item())
                rows.append(pin(y[0]))
            entry = dict(case, rows=rows)
            if case["kind"] == "est" and case["n_spks"] == 1:
                padded = ref.estimator(z * mask, mask, mu, t, spk)
                assert torch.equal(padded, O.estimator(sd, cfg, z * mask, mask, mu, t, spk))
                entry["padded"] = pin(padded)
        print(case, "row norms", [round(r["norm"], 3) for r in rows])
        out["cases"].append(entry)
    path = os.path.join(ROOT, "tests", "golden", "gradtts_ragged_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
