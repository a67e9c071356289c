"""The whole of inference.py's GPU work in libsbk: text encoder -> durations / alignment / prior (sbk_prior_expand) -> N-step
sampler -> HiFi-GAN vocoder, timed stage by stage with CUDA events (median of 5 after 2 warm-ups).  The vocoder runs in the
decoder's precision (fp32x3, tf32 or bf16); the bf16 rows hand it the mel as bfloat16, as a pipeline that keeps its tensors
in bf16 would.

    python scripts/gpu_pipeline_bench.py            # config 1's shape (B=1, 221 tokens, N=10) and a batch (B=32, N=50)

Prints one JSON line per configuration (with the card's name and power limit): ms per stage, kernel launches per stage, mel-frames/s of the sampler and the vocoder,
the vocoder's achieved TFLOP/s (307.3 MMAC per mel frame, oracle/hifigan_oracle.py:macs_per_mel_frame) against the measured
tf32 tensor rate, and the real-time factor at 22.05 kHz (hop 256)."""
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
from oracle import hifigan_oracle as H, text_encoder_oracle as T  # noqa: E402  (weights + MAC counts only)
from speech_backbones_b200 import UNetConfig, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.gradtts import Diffusion, synthesize_from_encoder  # noqa: E402
from speech_backbones_b200.hifigan import Generator  # noqa: E402
from speech_backbones_b200.spec import HIFIGAN_V1, synthetic_hifigan_state_dict  # noqa: E402
from speech_backbones_b200.text_encoder import TextEncoder  # noqa: E402

dev = torch.device("cuda", 0)
enc = TextEncoder(149, 80, 192, 768, 256, 2, 6, 3, 0.1, window_size=4).eval()
enc.load_state_dict(T.synthetic_weights(1234), strict=True)
enc = enc.to(dev)
decs, vocs = {}, {}
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                   capture_output=True, text=True)
CARD = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip()}


def vocoder(precision):
    if precision not in vocs:
        v = Generator(HIFIGAN_V1, precision=precision).eval()
        v.remove_weight_norm()
        v.load_state_dict(synthetic_hifigan_state_dict(2468), strict=True)
        vocs[precision] = v.to(dev)
    return vocs[precision]


def decoder(precision):
    if precision not in decs:
        d = Diffusion(80, 64, precision=precision).eval()
        d.load_state_dict(synthetic_state_dict(UNetConfig()))
        decs[precision] = d.to(dev)
    return decs[precision]


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        out = fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts), out


def run(B, Tx, N, precision):
    g = torch.Generator().manual_seed(7)
    x = torch.randint(0, 148, (B, Tx), generator=g).to(dev)
    x_lengths = torch.full((B,), Tx, dtype=torch.long, device=dev)
    dec = decoder(precision)
    voc = vocoder(precision)
    ms_enc, (mu_x, logw, x_mask) = timed(lambda: enc(x, x_lengths))
    # synthetic durations with the reference's scale: the random-weight duration predictor is not trained, so logw is replaced
    # by log(2.3 frames per token) to give config 1's utterance length (221 tokens -> ~512 frames)
    logw = torch.full_like(logw, 0.834)
    ms_all, (mu_y, y, attn) = timed(lambda: synthesize_from_encoder(dec, mu_x, logw, x_mask, N, temperature=1.5, length_scale=0.91, want_attn=False))
    T_y = y.shape[-1]
    z, mask, muy = torch.randn_like(y), torch.ones((B, 1, T_y), device=dev), y.clone()
    T4 = (T_y + 3) // 4 * 4
    if T4 != T_y:
        z, mask, muy = (torch.nn.functional.pad(v, (0, T4 - T_y)) for v in (z, mask, muy))
    ms_dec, _ = timed(lambda: dec(z.contiguous(), mask.contiguous(), muy.contiguous(), N))
    mel = y.contiguous().to(torch.bfloat16 if precision == "bf16" else torch.float32)
    ms_voc, wav = timed(lambda: voc(mel))
    frames = B * T_y
    voc_flops = 2.0 * H.macs_per_mel_frame() * frames
    out = {"case": f"B={B} tokens={Tx} N={N} decoder and vocoder precision {precision}", "frames_per_utterance": T_y, **CARD,
           "ms": {"text_encoder": round(ms_enc, 3), "glue+sampler": round(ms_all, 3), "sampler_alone": round(ms_dec, 3),
                  "vocoder": round(ms_voc, 3), "total": round(ms_enc + ms_all + ms_voc, 3)},
           "launches": {"text_encoder": enc.engine().last_launch_count(), "sampler": dec.engine().last_launch_count(),
                        "sampler_host_launches": dec.engine().last_host_launches(), "vocoder": voc.engine().last_launch_count()},
           "sampler_mel_frames_per_s": frames / (ms_dec * 1e-3), "vocoder_mel_frames_per_s": frames / (ms_voc * 1e-3),
           "vocoder_tflops": voc_flops / (ms_voc * 1e-3) / 1e12,
           "audio_seconds": frames * 256 / 22050.0, "rtf_total": (ms_enc + ms_all + ms_voc) * 1e-3 / (frames * 256 / 22050.0),
           "wav_finite": bool(torch.isfinite(wav).all())}
    print(json.dumps(out), flush=True)


for B, Tx, N, prec in ((1, 221, 10, "fp32x3"), (1, 221, 10, "tf32"), (1, 221, 10, "bf16"),
                       (32, 221, 50, "fp32x3"), (32, 221, 50, "tf32"), (32, 221, 50, "bf16")):
    run(B, Tx, N, prec)
