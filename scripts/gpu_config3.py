"""BASELINE config 3: Grad-TTS batch=128, T=512, N=1000 long-horizon sampler, bf16, one GPU.
The drop-in module in precision="bf16" is called with bf16 tensors (z, mask, mu) and returns a bf16 tensor; the whole
N=1000 call is CUDA-event timed after a short warm-up call (plan + graph already built).  Size-independent checks at
the full size: finite output, padded frames exactly zero, batch entries independent (a 2-utterance slice re-run alone
reproduces its rows).  The tf32 engine at the same shape (N=50) is timed beside it.
usage: python scripts/gpu_config3.py [N=1000] [B=128]"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

ge.build()
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.gradtts import Diffusion  # noqa: E402

N = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
B = int(sys.argv[2]) if len(sys.argv) > 2 else 128
T = 512
cfg = UNetConfig()
sd = synthetic_state_dict(cfg)
z, mask, mu, _, lengths = synthetic_inputs(B, T, ragged=True)


def timed(dec, args, n):
    dec(*args, 3)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    y = dec(*args, n)
    e1.record()
    torch.cuda.synchronize()
    return y, e0.elapsed_time(e1)


dec = Diffusion(80, 64, precision="bf16").eval()
dec.load_state_dict(sd)
dec = dec.cuda()
args16 = (z.cuda().bfloat16(), mask.cuda().bfloat16(), mu.cuda().bfloat16())
y, ms = timed(dec, args16, N)
valid = float(mask.sum())
pad = (y.float().cpu() * (1 - mask)).abs().max().item()
# batch independence at the full size: rows 5..6 alone, same padded T
y2 = dec(args16[0][5:7], args16[1][5:7], args16[2][5:7], N)
dep = ((y2.float() - y[5:7].float()).norm() / y[5:7].float().norm()).item()
out = {"case": "config3: Grad-TTS B=%d T=%d N=%d bf16 (module, bf16 tensors in/out, ragged lengths)" % (B, T, N),
       "precision": "bf16", "B": B, "T": T, "N": N, "ms_per_call": ms, "ms_per_sampler_step": ms / N,
       "mel_frames_per_s": B * T / (ms * 1e-3), "valid_mel_frames_per_s": valid / (ms * 1e-3),
       "frame_steps_per_s": B * T * N / (ms * 1e-3), "out_dtype": str(y.dtype), "finite": bool(torch.isfinite(y.float()).all()),
       "padded_frames_max_abs": pad, "rows_5_6_alone_vs_in_batch_rel_l2": dep,
       "workspace_GB": dec.engine().workspace_bytes(B, T) / 1e9}
print(json.dumps(out), flush=True)
del dec
dec32 = Diffusion(80, 64, precision="tf32").eval()
dec32.load_state_dict(sd)
dec32 = dec32.cuda()
args32 = (z.cuda(), mask.cuda(), mu.cuda())
y32, ms32 = timed(dec32, args32, 50)
dec16 = Diffusion(80, 64, precision="bf16").eval()
dec16.load_state_dict(sd)
dec16 = dec16.cuda()
y16, ms16 = timed(dec16, args32, 50)
print(json.dumps({"case": "same shape, N=50, fp32 tensors: tf32 vs bf16 engines", "B": B, "T": T, "N": 50,
                  "tf32_ms_per_step": ms32 / 50, "bf16_ms_per_step": ms16 / 50,
                  "tf32_mel_frames_per_s": B * T / (ms32 * 1e-3), "bf16_mel_frames_per_s": B * T / (ms16 * 1e-3),
                  "bf16_vs_tf32_rel_l2": ((y16 - y32).norm() / y32.norm()).item()}), flush=True)
