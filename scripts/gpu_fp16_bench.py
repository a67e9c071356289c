"""The fp16 sampler mode against bf16 and tf32 at the BASELINE shapes: config 2 (Grad-TTS, B 32, T 512, N 50) and config 4
(DiffVC fast-ML, B 64, T = T_ref = 256, N 6: native conditioning table + sampler loop).  The three modes alternate, one timed
call each in turn, so the clock drift of a power-limited card is shared; reported per mode and shape: the median and the
spread of REPS calls (CUDA events), mel-frames/s at the median, and fp16's rate over bf16's and tf32's.  The card's name,
power limit and SM clocks are read in the same run.  Prints one JSON line per (shape, mode) and one per shape comparison.
usage: python scripts/gpu_fp16_bench.py [reps]"""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402

ge.build()
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.binding import Engine  # noqa: E402
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs  # noqa: E402
from speech_backbones_b200.spec import synthetic_state_dict as vc_state_dict  # noqa: E402

REPS = int(sys.argv[1]) if len(sys.argv) > 1 else 7
MODES = ("fp16", "bf16", "tf32")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    return q


def gradtts_case():
    B, T, N = 32, 512, 50
    sd = synthetic_state_dict(UNetConfig())
    z, mask, mu, _, _ = (v.cuda() if v is not None else None for v in synthetic_inputs(B, T))
    engines = {}
    for m in MODES:
        engines[m] = Engine(precision=m)
        engines[m].load_state_dict(sd)
    run = {m: (lambda e=engines[m]: e.reverse_diffusion(z, mask, mu, N)) for m in MODES}
    return "gradtts config 2", B * T, run, engines


def diffvc_case():
    B, T, N = 64, 256, 6
    cfg = DiffVCConfig()
    sd = vc_state_dict(cfg, spec=diffvc_param_spec(cfg))
    z, mask, mean, ref, ref_mask, mean_ref, c = (v.cuda() for v in synthetic_diffvc_inputs(B, T, T))
    noise = torch.randn(N, B, 80, T, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    engines = {}
    for m in MODES:
        engines[m] = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=m)
        engines[m].load_state_dict(sd)

    def call(e):
        cond = e.vc_conditioning(ref, ref_mask, mean_ref, c, N)
        return e.vc_reverse_diffusion(z, mask, mean, cond, N, "ml", noise)
    run = {m: (lambda e=engines[m]: call(e)) for m in MODES}
    return "diffvc config 4 (ml, N 6)", B * T, run, engines


def measure(name, frames, run):
    for m in MODES:                                     # warm-up: plans, graphs, module loads
        for _ in range(2):
            run[m]()
    torch.cuda.synchronize()
    ms = {m: [] for m in MODES}
    for _ in range(REPS):
        for m in MODES:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = run[m]()
            e1.record()
            torch.cuda.synchronize()
            ms[m].append(e0.elapsed_time(e1))
            assert bool(torch.isfinite(y).all()), (name, m)
    med = {m: statistics.median(v) for m, v in ms.items()}
    for m in MODES:
        print(json.dumps({"case": name, "precision": m, "reps": REPS, "ms_median": round(med[m], 3),
                          "ms_min": round(min(ms[m]), 3), "ms_max": round(max(ms[m]), 3),
                          "mel_frames_per_s": round(frames / (med[m] * 1e-3), 1), "card": card()}), flush=True)
    print(json.dumps({"case": name, "fp16_rate_over_bf16": round(med["bf16"] / med["fp16"], 4),
                      "fp16_rate_over_tf32": round(med["tf32"] / med["fp16"], 4)}), flush=True)


print("# card (name, power limit, SM clock, max SM clock):", card(), flush=True)
for make in (gradtts_case, diffvc_case):
    name, frames, run, engines = make()
    measure(name, frames, run)
    for e in engines.values():
        e.close()
    torch.cuda.empty_cache()
