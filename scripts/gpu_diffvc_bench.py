"""BASELINE config 4: DiffVC decoder fast-ML sampler, B=64, T=T_ref=256, N in {6, 30}, mode 'ml', one GPU.
Reports mel-frames/s for the whole `Diffusion.forward` (hoisted PyTorch conditioning + libsbk loop) and for the loop alone."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

ge.build()
from speech_backbones_b200.diffvc import Diffusion  # noqa: E402
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs, synthetic_state_dict  # noqa: E402

precision = sys.argv[1] if len(sys.argv) > 1 else "tf32"
B, T, Tr = (int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[3])) if len(sys.argv) > 3 else (64, 256, 256)
cfg = DiffVCConfig()
dec = Diffusion(80, 256, 128, True, 0.05, 20.0, precision=precision).eval()
dec.load_state_dict(synthetic_state_dict(cfg, spec=diffvc_param_spec(cfg)))
dec = dec.cuda()
args = [v.cuda() for v in synthetic_diffvc_inputs(B, T, Tr)]
z, mask, mean, ref, ref_mask, mean_ref, c = args
eng = dec.engine()
for N in (6, 30):
    dec(*args, n_timesteps=N, mode="ml")
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    cond = dec.conditioning_table(ref, ref_mask, mean_ref, c, N)
    noise = torch.stack([torch.randn_like(z) for _ in range(N)])
    e[1].record()
    y = eng.vc_reverse_diffusion(z, mask, mean, cond, N, "ml", noise)
    e[2].record()
    torch.cuda.synchronize()
    t_cond, t_loop = e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])
    print(json.dumps({"case": f"DiffVC ml N={N}", "precision": precision, "B": B, "T": T, "T_ref": Tr,
                      "ms_conditioning": t_cond, "ms_loop_libsbk": t_loop, "ms_per_step": t_loop / N,
                      "mel_frames_per_s": B * T / ((t_cond + t_loop) * 1e-3), "mel_frames_per_s_loop_only": B * T / (t_loop * 1e-3),
                      "tflops_loop": 2013.7e6 * B * T * N / (t_loop * 1e-3) / 1e12, "finite": bool(torch.isfinite(y).all())}), flush=True)
rows = eng.profile_ops()
tot = sum(r[1] for r in rows)
print(f"# per-launch profile, one step: {tot:.3f} ms")
for n, ms, fl, by in rows:
    print(f"{n:44s} {ms:8.4f} ms  {fl / ms / 1e9 if ms else 0:8.1f} TFLOP/s  {by / ms / 1e6 if ms else 0:8.1f} GB/s")
