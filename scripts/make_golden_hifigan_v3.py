"""Generate tests/golden/hifigan_v3_golden.pt from the UNMODIFIED reference HiFi-GAN generator with the V3 config
(container only).

The recipe of make_golden_hifigan.py: imports Grad-TTS/hifi-gan/models.py from /root/reference (matplotlib stubbed), builds
Generator(h) from an AttrDict of the public HiFi-GAN config_v3.json values (ResBlock2; the reference tree ships no V3
config), loads seeded weights (spec.synthetic_hifigan_state_dict, which replaces init_weights' std 0.01), calls
remove_weight_norm() as inference.py:63 does, and stores ONLY the reference outputs; tests rebuild weights and inputs from
the seeds.  Asserts that tests/hifigan_v3_oracle.py reproduces the reference exactly on every case, that the parameter
inventories (oracle, spec, reference state_dict) agree, and the V3 sizes: 1,462,273 parameters, 22,482,944 MAC per mel frame.

    python scripts/make_golden_hifigan_v3.py
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from hifigan_v3_oracle import V3, generator, macs_per_mel_frame, param_spec  # noqa: E402
from make_golden_hifigan import import_reference_generator  # noqa: E402
from speech_backbones_b200.spec import HIFIGAN_V3, hifigan_param_spec, synthetic_hifigan_state_dict  # noqa: E402

CASES = [dict(B=1, T=32), dict(B=2, T=20), dict(B=1, T=5)]
SEED = 2468
NPARAMS, MACS = 1_462_273, 22_482_944


def main():
    Generator, _ = import_reference_generator()
    from env import AttrDict                              # on the path import_reference_generator set up
    assert HIFIGAN_V3 == V3
    ref = Generator(AttrDict(V3)).eval()
    ref.remove_weight_norm()
    sd = synthetic_hifigan_state_dict(SEED, V3)
    ref_shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    assert ref_shapes == dict(param_spec(V3)) == dict(hifigan_param_spec(V3)), "parameter inventory differs from the reference's state_dict"
    ref.load_state_dict(sd, strict=True)
    out = {"seed": SEED, "torch": torch.__version__, "config": dict(V3), "cases": [],
           "nparams": sum(v.numel() for v in sd.values()), "macs_per_mel_frame": macs_per_mel_frame(V3)}
    assert out["nparams"] == NPARAMS and len(sd) == 46, (out["nparams"], len(sd))
    assert out["macs_per_mel_frame"] == MACS, out["macs_per_mel_frame"]
    for c in CASES:
        g = torch.Generator().manual_seed(SEED + c["T"])
        mel = torch.randn(c["B"], 80, c["T"], generator=g)
        with torch.no_grad():
            y = ref(mel)
            yo = generator(sd, mel, V3)
        assert y.shape == (c["B"], 1, c["T"] * 256)
        err = (yo - y).abs().max().item()
        assert err == 0.0, err
        out["cases"].append(dict(c, out=y.clone()))
        print(f"B={c['B']} T={c['T']}: |y|max={y.abs().max():.3f}, oracle == reference (max abs diff {err})")
    path = os.path.join(ROOT, "tests", "golden", "hifigan_v3_golden.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path), "bytes; params", out["nparams"], "MAC/frame", out["macs_per_mel_frame"])


if __name__ == "__main__":
    main()
