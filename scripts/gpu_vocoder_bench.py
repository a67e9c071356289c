"""The HiFi-GAN vocoder (sbk_vocoder_forward) in its three precision modes, one GPU.

    python scripts/gpu_vocoder_bench.py [--config v1|v3] [--iters 20] [--warmup 5] [--T 512]

--config v1 (the default): Grad-TTS's shipped config; v3: the public HiFi-GAN V3 config (ResBlock2, spec.HIFIGAN_V3).

Two shapes: B = 32 (the pipeline batch) and B = 1 (latency), T = 512 mel frames each.  Per (shape, mode) one JSON line with
the card's name and power limit read in the same run:
  * ms per call: the median of `--iters` CUDA-event-timed calls after `--warmup` calls;
  * mel-frames/s and the achieved algorithmic TFLOP/s (2 x MAC per mel frame: V1 307,052,544, V3 22,482,944,
    macs_per_mel_frame);
  * rel-L2 and max-abs of the mode's waveform against the tf32 waveform of the same (timed) input.
  * v3 only: the activation bytes a call must move through HBM (model below) and the time that takes at the card's
    3.35 TB/s peak, next to the achieved rate - V3's last stage (32 channels, 256 samples per frame) has ~1 MAC per byte.
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
from speech_backbones_b200.spec import HIFIGAN_V1, HIFIGAN_V3, synthetic_hifigan_state_dict  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
from hifigan_v3_oracle import macs_per_mel_frame  # noqa: E402

CONFIGS = {"v1": ("HiFi-GAN V1 vocoder", HIFIGAN_V1), "v3": ("HiFi-GAN V3 vocoder", HIFIGAN_V3)}
MODES = ("tf32", "fp32x3", "bf16")
HBM_PEAK = 3.35e12                     # H100 SXM5 HBM3, bytes/s


def hbm_bytes_per_frame(h, mode):
    """Activation bytes per mel frame one call reads and writes in HBM if every launch reads each input element once
    (strip halos and GEMM A re-reads hit L2) and writes each output once; weights are not counted.  A conv input (operand)
    takes 4 bytes per element in tf32 and fp32x3 (its correction chunks are derived in shared memory), 2 in bf16; the
    residual stream, the GEMM output and the MRF inputs are fp32."""
    ob = {"tf32": 4, "bf16": 2, "fp32x3": 4}[mode]
    rb2 = str(h.get("resblock", "1")) != "1"
    c, nm = h["upsample_initial_channel"], h["num_mels"]
    total = 4 * nm + ob * nm                                  # mel_in
    total += ob * nm + ob * c                                 # conv_pre -> SA
    rate, nu = 1, len(h["upsample_rates"])
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        co = c // 2
        total += ob * c * rate + 4 * k * co * rate            # GEMM: SA -> Z
        total += 4 * k * co * rate + (4 + ob) * co * rate * u   # fold: Z -> X0, A0
        rate *= u
        n = co * rate                                         # elements of one stage tensor per frame
        # ResBlock2: conv0 reads A0 + X0, writes X1 + A1; conv1 reads A1 + X1, writes R
        # ResBlock1, per dilation: conv1 reads A, writes Hb; conv2 reads Hb + x, writes x' (+ A but the last)
        per_block = (3 * ob + 16) if rb2 else (3 * (3 * ob + 8) + 2 * ob)
        total += 3 * per_block * n
        total += 12 * n + (4 if i + 1 == nu else ob) * n       # MRF
        c = co
    return total + 4 * c * rate + 4 * rate                    # conv_post + tanh


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--T", type=int, default=512)
    ap.add_argument("--config", choices=sorted(CONFIGS), default="v1")
    a = ap.parse_args()
    case, h = CONFIGS[a.config]
    mac_per_frame = macs_per_mel_frame(h)
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    info = card()
    sd = synthetic_hifigan_state_dict(2468, h)
    gens = {}
    for mode in MODES:
        g = Generator(h, precision=mode).eval()
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
            row = {"case": case, "precision": m, "B": B, "T": a.T, "ms": round(ms, 4),
                   "ms_min": round(min(times[m]), 4), "ms_max": round(max(times[m]), 4),
                   "mel_frames_per_s": B * a.T / (ms * 1e-3),
                   "tflops_algorithmic": 2.0 * mac_per_frame * B * a.T / (ms * 1e-3) / 1e12,
                   "rel_l2_vs_tf32": (d.norm() / ref.norm()).item(), "max_abs_vs_tf32": d.abs().max().item(),
                   "launches": gens[m].engine().last_launch_count()}
            if a.config != "v1":
                nbytes = hbm_bytes_per_frame(h, m) * B * a.T
                row.update({"hbm_bytes_model": nbytes, "hbm_gbytes_per_s_model": nbytes / (ms * 1e-3) / 1e9,
                            "ms_at_hbm_peak": round(nbytes / HBM_PEAK * 1e3, 4)})
            print(json.dumps({**row, **info}), flush=True)


if __name__ == "__main__":
    main()
