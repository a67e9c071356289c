"""DiffVC's inference front end on one GPU: `LogMel` and `mel_spectral_subtraction` on B = 64 utterances of seeded lengths
2 - 10 s (22050 Hz), against the same batch through the float64 CPU restatement (oracle/frontend_oracle.py).

Prints one JSON line per measurement, each with the card's name and power limit read in the same run:
  * LogMel (ragged batch): median CUDA-event ms per call over `--iters` timed calls (each timed alone), frames/s;
  * the DFT GEMM alone (torch.profiler, its k_conv_tc kernel): ms and achieved TFLOP/s from the columns it computes
    (2 x 1024 x 768 per frame, the 744 columns of bins 0 - 371 padded to the 128-wide N tile) and from the 744 used ones;
  * mel_spectral_subtraction (ragged, the notebook's call: the same mel as both arguments, smoothing_window=1): median ms;
  * the CPU restatement of both on the same batch: seconds, once.

    python scripts/gpu_frontend_bench.py [--iters 20] [--warmup 3] [--out results/frontend_bench.jsonl]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import frontend_oracle as O  # noqa: E402
from speech_backbones_b200.frontend import LogMel, mel_spectral_subtraction  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    info = card()
    rng = np.random.default_rng(a.seed)
    lengths = rng.integers(2 * 22050, 10 * 22050 + 1, size=a.B)
    L = int(lengths.max())
    wav = torch.from_numpy((0.1 * rng.standard_normal((a.B, L))).astype(np.float32))
    for b, n in enumerate(lengths):
        wav[b, n:] = 0
    wav_d, len_d = wav.cuda(), torch.from_numpy(lengths).cuda()
    frames = int((lengths // 256).sum())
    lm = LogMel()
    mel, ml = lm(wav_d, len_d)
    T = mel.shape[-1]
    lines = []

    def emit(d):
        d.update(info)
        lines.append(json.dumps(d))
        print(lines[-1], flush=True)

    ms = median_ms(lambda: lm(wav_d, len_d), a.iters, a.warmup)
    emit({"what": "LogMel", "B": a.B, "T": T, "frames": frames, "ms": ms, "frames_per_s": frames / (ms * 1e-3)})

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            lm(wav_d, len_d)
        torch.cuda.synchronize()
    gemm = [e for e in prof.key_averages() if "k_conv_tc" in e.key]
    if gemm:
        g_ms = sum(e.device_time_total for e in gemm) / sum(e.count for e in gemm) / 1e3
        computed = 2.0 * a.B * T * 1024 * 768
        emit({"what": "LogMel DFT GEMM (k_conv_tc<G_PW>, fp32x3)", "ms": g_ms, "rows": a.B * T,
              "tflops_computed_cols": computed / (g_ms * 1e-3) / 1e12,
              "tflops_used_cols": computed * 744 / 768 / (g_ms * 1e-3) / 1e12,
              "share_of_call": g_ms / ms})

    ms = median_ms(lambda: mel_spectral_subtraction(mel, mel, smoothing_window=1, lengths=ml), a.iters, a.warmup)
    emit({"what": "mel_spectral_subtraction", "B": a.B, "T": T, "frames": frames, "ms": ms, "frames_per_s": frames / (ms * 1e-3)})

    t0 = time.perf_counter()
    mels = [O.get_mel(wav[b, :n].numpy()) for b, n in enumerate(lengths)]
    t1 = time.perf_counter()
    for m in mels:
        O.mel_spectral_subtraction(m, m, smoothing_window=1)
    t2 = time.perf_counter()
    emit({"what": "CPU float64 restatement (oracle/frontend_oracle.py), one process", "get_mel_s": t1 - t0,
          "spectral_subtraction_s": t2 - t1, "cpu_count": os.cpu_count()})
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
