"""DiffVC's PostNet and DiffVC.forward at BASELINE config 4 shapes (B = 64, T = T_ref = 256), one GPU.

Prints one JSON line per measurement, each carrying the card's name and power limit read in the same run:
  * the native PostNet (sbk_postnet_forward) in fp32x3 and tf32: ms per call and algorithmic TFLOP/s
    (2 x 129,781,760 MAC per frame x B x T / time);
  * the cuDNN baseline: the oracle's PyTorch restatement of the PostNet (oracle/postnet_oracle.py:postnet) on the same card,
    cudnn.benchmark on, allow_tf32 False and True;
  * DiffVC.forward at N = 6 'ml', split into the encoder (two FwdDiffusion calls) and the decoder (convert_from_encoder).
Times are CUDA-event times over `--iters` calls after `--warmup` calls.

    python scripts/gpu_postnet_bench.py [--iters 10] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import postnet_oracle as O  # noqa: E402
from speech_backbones_b200.diffvc import DiffVC, convert_from_encoder  # noqa: E402
from speech_backbones_b200.postnet import PostNet  # noqa: E402
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS, synthetic_postnet_state_dict  # noqa: E402

MAC_PER_FRAME = 129_781_760          # PostNet(128) on 80 mel bins: 80 x (2 x 128 x 128 x 49 + 128 x 128 + 2 x 128)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=256)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    info = card()
    B, T = a.B, a.T
    tflop = 2.0 * MAC_PER_FRAME * B * T / 1e12

    def emit(**kw):
        print(json.dumps({**kw, "B": B, "T": T, **info}), flush=True)

    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, 80, T, generator=g).cuda()
    lengths = torch.randint(T // 2, T + 1, (B,), generator=g)
    lengths[0] = T
    mask = (torch.arange(T)[None, :] < lengths[:, None]).float()[:, None].cuda()
    sd = synthetic_postnet_state_dict(128, 1234)
    outs = {}
    for precision in ("fp32x3", "tf32"):
        m = PostNet(128, precision=precision).eval()
        m.load_state_dict(sd)
        m = m.cuda()
        ms = timed(lambda: m(x, mask), a.iters, a.warmup)
        outs[precision] = m(x, mask)
        emit(case="PostNet native", precision=precision, ms=ms, tflops_algorithmic=tflop / (ms * 1e-3),
             launches=m.engine().last_launch_count())
        del m
    sdc = {k: v.cuda() for k, v in sd.items()}
    torch.backends.cudnn.benchmark = True
    for tf32 in (False, True):
        torch.backends.cudnn.allow_tf32 = tf32
        with torch.no_grad():
            ms = timed(lambda: O.postnet(sdc, x, mask), a.iters, a.warmup)
            y = O.postnet(sdc, x, mask)
        emit(case="PostNet cuDNN (PyTorch restatement)", allow_tf32=tf32, ms=ms, tflops_algorithmic=tflop / (ms * 1e-3),
             rel_l2_native_fp32x3_vs_this=((outs["fp32x3"] - y).norm() / y.norm()).item())
    torch.backends.cudnn.allow_tf32 = True
    del outs, sdc

    # DiffVC.forward, N = 6 'ml': encoder (MelEncoder + PostNet, twice) and decoder
    for precision in ("fp32x3", "tf32"):
        model = DiffVC(*DIFFVC_MODEL_ARGS, precision=precision).cuda()
        model.load_state_dict(O.model_synthetic_weights(1234), strict=True)
        model.eval()
        x_ref = torch.randn(B, 80, T, generator=g).cuda()
        c = torch.randn(B, 256, generator=g)
        c = (c / c.norm(dim=1, keepdim=True)).cuda()
        xl, xrl = lengths.cuda(), lengths.flip(0).cuda()
        xr_mask = (torch.arange(T)[None, :] < lengths.flip(0)[:, None]).float()[:, None].cuda()
        with torch.no_grad():
            t_enc = timed(lambda: (model.encoder(x, mask), model.encoder(x_ref, xr_mask)), a.iters, a.warmup)
            mean, mean_ref = model.encoder(x, mask), model.encoder(x_ref, xr_mask)
            t_dec = timed(lambda: convert_from_encoder(model.decoder, x, xl, mean, x_ref, xr_mask, mean_ref, c, 6, "ml"),
                          max(1, a.iters // 2), 1)
            t_all = timed(lambda: model(x, xl, x_ref, xrl, c, n_timesteps=6, mode="ml"), max(1, a.iters // 2), 1)
        emit(case="DiffVC.forward N=6 ml", precision=precision, ms_total=t_all, ms_encoder_two_calls=t_enc, ms_decoder=t_dec,
             mel_frames_per_s=B * T / (t_all * 1e-3))
        del model


if __name__ == "__main__":
    main()
