"""Ragged vs padded DiffVC at BASELINE config 4's shape (B = 64, T = T_ref = 256, mode ml, N = 6), on one GPU.

Source and reference lengths are seeded draws from U{128..256}.  The stages of DiffVC.forward are timed on their own:
  * FwdDiffusion (mel encoder + PostNet), run once on the source mels and once on the reference mels;
  * the conditioning table (`Engine.vc_conditioning`, the RefBlock branch, N steps) on the reference;
  * the sampler, `Engine.vc_reverse_diffusion` (the score U-Net, N steps), on T' = fix_len_compatibility(256) = 256.
Each stage runs three ways on the same inputs: padded (no lengths), ragged (lengths=) and a loop of B single-utterance
calls, each on its own frames.  fp32x3 and tf32 alternate, and within a mode the three ways alternate, one timed call of each
in turn, so clock drift of a power-limited card is shared.  Reported per mode and stage: ms per call (median, min, max over
the runs), with the card's name and power limit, and its SM clock and active throttle reasons read right after the timed
runs.

    python scripts/gpu_vc_ragged_bench.py [--runs 5] [--warmup 2]
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

from speech_backbones_b200.binding import Engine  # noqa: E402
from speech_backbones_b200.diffvc import fix_len_compatibility  # noqa: E402
from speech_backbones_b200.diffvc import FwdDiffusion  # noqa: E402
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS, DiffVCConfig, diffvc_param_spec, synthetic_state_dict  # noqa: E402
from oracle.postnet_oracle import fwd_synthetic_weights  # noqa: E402

B, T, N, MODE = 64, 256, 6, "ml"


def card(fields="name,power.limit,clocks.max.sm"):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def timed(f):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    f()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    g = torch.Generator().manual_seed(4)
    src_len = torch.randint(128, T + 1, (B,), generator=g)
    ref_len = torch.randint(128, T + 1, (B,), generator=g)
    x = torch.randn(B, 80, T, generator=g).cuda()
    x_ref = torch.randn(B, 80, T, generator=g).cuda()
    mean = torch.randn(B, 80, T, generator=g).cuda()
    z = mean + torch.randn(B, 80, T, generator=g).cuda()
    cfg = DiffVCConfig()
    cond = (torch.randn(N, B, cfg.dim_spk, generator=g) * 0.5).cuda()
    mean_ref = torch.randn(B, 80, T, generator=g).cuda()
    spk = torch.randn(B, 256, generator=g)
    spk = (spk / spk.norm(dim=1, keepdim=True)).cuda()
    noise = torch.randn(N, B, 80, T, generator=g).cuda()

    def mask_of(lengths, t):
        return (torch.arange(t)[None, :] < lengths[:, None]).float()[:, None].cuda()
    m_src, m_ref = mask_of(src_len, T), mask_of(ref_len, T)
    Ls, Lr = src_len.cuda(), ref_len.cuda()
    tp = [fix_len_compatibility(int(v)) for v in src_len]
    pn_sd = fwd_synthetic_weights(1234)
    vc_sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    res = {"shape": {"B": B, "T": T, "T_ref": T, "N": N, "mode": MODE, "src_frames": int(src_len.sum()),
                     "ref_frames": int(ref_len.sum()), "padded_frames": B * T}, **card(), "modes": {}}
    nets = {}
    for precision in ("fp32x3", "tf32"):
        pn = FwdDiffusion(*DIFFVC_MODEL_ARGS[:8], 128, precision=precision).eval()
        pn.load_state_dict(pn_sd, strict=True)
        eng = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision)
        eng.load_state_dict(vc_sd)
        nets[precision] = (pn.cuda(), eng)
    ones = {L: torch.ones(1, 1, L, device="cuda") for L in set(src_len.tolist()) | set(ref_len.tolist())}

    def stages(precision):
        pn, eng = nets[precision]

        def pn_loop(v, lengths):
            for b, L in enumerate(lengths.tolist()):
                pn(v[b:b + 1, :, :L], ones[L])

        def vc_loop():
            for b in range(B):
                Tb = tp[b]
                eng.vc_reverse_diffusion(z[b:b + 1, :, :Tb], m_src[b:b + 1, :, :Tb], mean[b:b + 1, :, :Tb], cond[:, b:b + 1],
                                         N, MODE, noise[:, b:b + 1, :, :Tb])
        def cond_loop():
            for b, R in enumerate(ref_len.tolist()):
                eng.vc_conditioning(x_ref[b:b + 1, :, :R], ones[R], mean_ref[b:b + 1, :, :R], spk[b:b + 1], N)
        return {
            "fwd_diffusion_src": {"padded": lambda: pn(x, m_src), "ragged": lambda: pn(x, m_src, lengths=Ls),
                                  "b1_loop": lambda: pn_loop(x, src_len)},
            "fwd_diffusion_ref": {"padded": lambda: pn(x_ref, m_ref), "ragged": lambda: pn(x_ref, m_ref, lengths=Lr),
                                  "b1_loop": lambda: pn_loop(x_ref, ref_len)},
            "conditioning": {"padded": lambda: eng.vc_conditioning(x_ref, m_ref, mean_ref, spk, N),
                             "ragged": lambda: eng.vc_conditioning(x_ref, m_ref, mean_ref, spk, N, ref_lengths=Lr),
                             "b1_loop": cond_loop},
            "sampler": {"padded": lambda: eng.vc_reverse_diffusion(z, m_src, mean, cond, N, MODE, noise),
                        "ragged": lambda: eng.vc_reverse_diffusion(z, m_src, mean, cond, N, MODE, noise, lengths=Ls),
                        "b1_loop": vc_loop},
        }
    calls = {p: stages(p) for p in nets}
    for _ in range(args.warmup):
        for p in calls:
            for st in calls[p].values():
                for f in st.values():
                    f()
    ms = {p: {s: {k: [] for k in st} for s, st in calls[p].items()} for p in calls}
    for _ in range(args.runs):
        for p in calls:
            for s, st in calls[p].items():
                for k, f in st.items():
                    ms[p][s][k].append(timed(f))
    res["after_runs"] = card("clocks.sm,clocks_throttle_reasons.active,temperature.gpu,power.draw")["nvidia_smi"]
    for p in calls:
        row = {}
        for s, st in ms[p].items():
            row[s] = {k: {"ms_median": round(statistics.median(v), 3), "ms_min": round(min(v), 3), "ms_max": round(max(v), 3)}
                      for k, v in st.items()}
            row[s]["ragged_over_padded"] = round(row[s]["ragged"]["ms_median"] / row[s]["padded"]["ms_median"], 3)
        res["modes"][p] = row
        print(p, json.dumps(row), flush=True)
    for pn, eng in nets.values():
        eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
