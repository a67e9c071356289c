"""Same results at the shipped U-Net widths: this tree against another built source tree (e.g. the parent commit, built in
place with `python __graft_entry__.py`), on the same seeded inputs and the same GPU.

    python scripts/gpu_gn_partials_ab.py OTHER_ROOT

A change to how the convs attribute and flush their GroupNorm partials must leave Grad-TTS dim = 64 and DiffVC
dim_unet = 256 (cpg 8 / 16 / 32k, group-aligned tiles) exactly as they were.  One worker process per tree imports the
package of ITS tree only and runs, in every precision mode, one estimator call and a 3-step reverse diffusion: Grad-TTS at
n_spks = 1 (deterministic) and n_spks = 4 (stochastic), DiffVC in the pf and ml modes.  The outputs are compared with
torch.equal; exit status 1 if any differs."""
import os
import subprocess
import sys
import tempfile

MODES = ("fp32x3", "tf32", "bf16", "fp32")
B, T, N = 2, 260, 3


def worker(root, path):
    sys.path.insert(0, root)
    import torch
    from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
    from speech_backbones_b200.binding import Engine
    from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs
    res = {}
    t = torch.linspace(0.9, 0.2, B, device="cuda")
    g = torch.Generator().manual_seed(7)
    noise = torch.randn(N, B, 80, T, generator=g).cuda()
    for n_spks in (1, 4):
        sd = synthetic_state_dict(UNetConfig(n_spks=n_spks))
        z, mask, mu, spk, _ = (None if v is None else v.cuda() for v in synthetic_inputs(B, T, ragged=True, n_spks=n_spks))
        for m in MODES:
            e = Engine(n_spks=n_spks, precision=m)
            e.load_state_dict(sd)
            res[f"gradtts/spk{n_spks}/{m}/estimator"] = e.estimator(z * mask, mask, mu, t, spk).cpu()
            res[f"gradtts/spk{n_spks}/{m}/reverse"] = e.reverse_diffusion(z, mask, mu, N, n_spks > 1, spk,
                                                                          noise if n_spks > 1 else None).cpu()
            e.close()
    cfg = DiffVCConfig()
    sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    z, mask, mean = (v.cuda() for v in synthetic_diffvc_inputs(B, T, 100, ragged=True)[:3])
    cond = (torch.randn(N, B, cfg.dim_spk, generator=g) * 0.5).cuda()
    for m in MODES:
        e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=m)
        e.load_state_dict(sd)
        res[f"diffvc/{m}/estimator"] = e.vc_estimator(z * mask, mask, mean, cond[0], t).cpu()
        for mode in ("pf", "ml"):
            res[f"diffvc/{m}/reverse-{mode}"] = e.vc_reverse_diffusion(z, mask, mean, cond, N, mode,
                                                                       None if mode == "pf" else noise).cpu()
        e.close()
    torch.save(res, path)


def main():
    if len(sys.argv) == 4 and sys.argv[1] == "--worker":
        return worker(sys.argv[2], sys.argv[3])
    import torch
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    other = os.path.abspath(sys.argv[1])
    with tempfile.TemporaryDirectory() as tmp:
        out = {}
        for tag, root in (("this", here), ("other", other)):
            path = os.path.join(tmp, f"{tag}.pt")
            subprocess.check_call([sys.executable, os.path.abspath(__file__), "--worker", root, path])
            out[tag] = torch.load(path)
    bad = 0
    for k, v in out["this"].items():
        same = torch.equal(v, out["other"][k])
        bad += not same
        print(f"{k:36s} {'equal' if same else 'DIFFERENT, max |diff| %.3e' % (v - out['other'][k]).abs().max().item()}")
    print(f"{len(out['this']) - bad} of {len(out['this'])} outputs equal")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
