"""Ragged vs padded Grad-TTS decoding at BASELINE config 2's shape (B = 32, T = 512, N = 50), on one GPU.

The batch's lengths come from spec.synthetic_inputs(32, 512, ragged=True) (U{256..512}, 12,461 of 16,384 frames valid).
For each of fp32x3, tf32 and bf16 the same batch runs as a padded call (no lengths) and as a ragged call (lengths=): the
two alternate, one timed call of each in turn, so clock drift of a power-limited card is shared.  Reported per mode: ms per
call (median, min, max over the runs) and mel-frames/s over the sum of the lengths, with the card's name and power limit
read in the same run.  The padded U-Net work a ragged call skips, from counting tiles and pixels: 14 % / 2 % / 0 % of the
128-pixel 3x3 tiles at levels 0 / 1 / 2, and 24 % of the pixels of the element-wise passes.

    python scripts/gpu_ragged_bench.py [--runs 5] [--warmup 2]
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

from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.binding import Engine  # noqa: E402

B, T, N = 32, 512, 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    z, mask, mu, _, lengths = synthetic_inputs(B, T, ragged=True)
    z, mask, mu, L = z.cuda(), mask.cuda(), mu.cuda(), lengths.cuda()
    frames = int(lengths.sum())
    sd = synthetic_state_dict(UNetConfig())
    res = {"shape": {"B": B, "T": T, "N": N, "valid_frames": frames, "padded_frames": B * T}, **card(), "modes": {}}
    for precision in ("fp32x3", "tf32", "bf16"):
        eng = Engine(precision=precision)
        eng.load_state_dict(sd)
        calls = {"padded": lambda: eng.reverse_diffusion(z, mask, mu, N),
                 "ragged": lambda: eng.reverse_diffusion(z, mask, mu, N, lengths=L)}
        for _ in range(args.warmup):
            for f in calls.values():
                f()
        ms = {k: [] for k in calls}
        for _ in range(args.runs):
            for k, f in calls.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                ms[k].append(e0.elapsed_time(e1))
        row = {}
        for k, v in ms.items():
            med = statistics.median(v)
            row[k] = {"ms_median": round(med, 2), "ms_min": round(min(v), 2), "ms_max": round(max(v), 2),
                      "mel_frames_per_s": round(frames / (med / 1e3))}
        row["ragged_over_padded"] = round(row["ragged"]["ms_median"] / row["padded"]["ms_median"], 3)
        res["modes"][precision] = row
        print(precision, json.dumps(row), flush=True)
        eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
