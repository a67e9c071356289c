"""The HiFi-GAN V1 vocoder (sbk_vocoder_forward) in its three precision modes, one GPU.

    python scripts/gpu_vocoder_bench.py [--iters 20] [--warmup 5] [--T 512]

Two shapes: B = 32 (the pipeline batch) and B = 1 (latency), T = 512 mel frames each.  Per (shape, mode) one JSON line with
the card's name and power limit read in the same run:
  * ms per call: the median of `--iters` CUDA-event-timed calls after `--warmup` calls;
  * mel-frames/s and the achieved algorithmic TFLOP/s (2 x 307,052,544 MAC per mel frame,
    oracle/hifigan_oracle.py:macs_per_mel_frame);
  * rel-L2 and max-abs of the mode's waveform against the tf32 waveform of the same (timed) input.
The modes run interleaved, one timed call of each in turn, so clock drift of a power-limited card is shared among them.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from speech_backbones_b200.hifigan import Generator  # noqa: E402
from speech_backbones_b200.spec import HIFIGAN_V1, synthetic_hifigan_state_dict  # noqa: E402

MAC_PER_FRAME = 307_052_544            # HiFi-GAN V1 (hifigan_golden.pt["macs_per_mel_frame"])
MODES = ("tf32", "fp32x3", "bf16")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--T", type=int, default=512)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    info = card()
    sd = synthetic_hifigan_state_dict(2468)
    gens = {}
    for mode in MODES:
        g = Generator(HIFIGAN_V1, precision=mode).eval()
        g.remove_weight_norm()
        g.load_state_dict(sd, strict=True)
        gens[mode] = g.cuda()
    for B in (32, 1):
        mel = torch.randn(B, 80, a.T, generator=torch.Generator().manual_seed(B)).cuda()
        outs, times = {}, {m: [] for m in MODES}
        for m in MODES:
            for _ in range(a.warmup):
                outs[m] = gens[m](mel)
        torch.cuda.synchronize()
        for _ in range(a.iters):
            for m in MODES:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                gens[m](mel)
                e1.record()
                torch.cuda.synchronize()
                times[m].append(e0.elapsed_time(e1))
        ref = outs["tf32"].double()
        for m in MODES:
            ms = statistics.median(times[m])
            d = outs[m].double() - ref
            print(json.dumps({"case": "HiFi-GAN V1 vocoder", "precision": m, "B": B, "T": a.T, "ms": round(ms, 4),
                              "ms_min": round(min(times[m]), 4), "ms_max": round(max(times[m]), 4),
                              "mel_frames_per_s": B * a.T / (ms * 1e-3),
                              "tflops_algorithmic": 2.0 * MAC_PER_FRAME * B * a.T / (ms * 1e-3) / 1e12,
                              "rel_l2_vs_tf32": (d.norm() / ref.norm()).item(), "max_abs_vs_tf32": d.abs().max().item(),
                              "launches": gens[m].engine().last_launch_count(), **info}), flush=True)


if __name__ == "__main__":
    main()
