"""Rolling vs static batching of a DiffVC decode service on one GPU, replaying a seeded arrival trace.

BASELINE config 4's decoder (dim_unet 256, dim_cond 128, 'ml', N = 6) at capacity 64, max_frames 256: 128 requests,
L ~ U{128..256} (T_b = fix_len_compatibility(L)), reference R ~ U{128..256}, arriving as a Poisson process at 0.9x the static
batch's measured throughput.  Two schedulers serve the same trace:
  (a) static: when the GPU is free, take up to 64 queued requests: one `vc_conditioning(..., ref_lengths=)` over their
      references, then one `vc_reverse_diffusion(..., lengths=)` at T = 256 (rows padded to 64 with 4-frame fillers);
  (b) rolling: `Diffusion.rolling(64, 256)`; a request's conditioning runs at its submission (B = 1), and each epoch runs to
      the next completion or - while slots are free and a request is due - to the step boundary nearest its arrival.
Time is virtual: the GPU time of each call (host clock around work that ends in a synchronise), the conditioning at
submission included, is added to the clock, and when nothing is queued the clock jumps to the next arrival.  Reported per
mode: valid mel-frames/s over the busy-or-waiting span, p50 / p95 latency (arrival to mel) in ms and in sampler steps, and
  - the per-step time at full occupancy (64 busy slots, the trace's lengths) against a `vc_reverse_diffusion(lengths=)` step
    at the same (B, T) and rows, the two alternating;
  - the cost of idle slots: a step with 32 of 64 slots busy against a `lengths=` step at B = 32.
The card's name, power limit and SM clock are read in the same run.

    python scripts/gpu_vc_rolling_bench.py [--modes tf32,bf16] [--requests 128] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gpu_rolling_bench import StepClock, card, summary, timed  # noqa: E402
from speech_backbones_b200.diffvc import Diffusion, fix_len_compatibility  # noqa: E402
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_state_dict  # noqa: E402

CAP, T, TR, N, MODE = 64, 256, 256, 6, "ml"


def make_trace(n, seed=11):
    """per request: (z, mask, mean [1,80,T_b], ref, ref_mask, mean_ref [1,80,R], c [1,256], noise [N,1,80,T_b], T_b)"""
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n):
        L = int(torch.randint(128, 257, (1,), generator=g))
        R = int(torch.randint(128, 257, (1,), generator=g))
        Tb = fix_len_compatibility(L)
        mask = (torch.arange(Tb) < L).float()[None, None]
        mean = torch.randn(1, 80, Tb, generator=g) * mask
        z = mean + torch.randn(1, 80, Tb, generator=g)
        ref = torch.randn(1, 80, R, generator=g)
        c = torch.randn(1, 256, generator=g)
        noise = torch.randn(N, 1, 80, Tb, generator=g)
        reqs.append([t.cuda() for t in (z, mask, mean, ref, torch.ones(1, 1, R), ref * 0.5, c / c.norm(), noise)] + [Tb])
    gaps = torch.empty(n).exponential_(1.0, generator=g)
    return reqs, gaps


def pack(reqs, B=CAP):
    """rows padded to B with 4-frame fillers: decoder inputs at (B, T), references at (B, TR), noise [N, B, 80, T]"""
    z = torch.zeros(B, 80, T, device="cuda"); mean = torch.zeros_like(z); mask = torch.zeros(B, 1, T, device="cuda")
    ref = torch.zeros(B, 80, TR, device="cuda"); rmask = torch.zeros(B, 1, TR, device="cuda")
    c = torch.zeros(B, 256, device="cuda"); c[:, 0] = 1.0
    noise = torch.zeros(N, B, 80, T, device="cuda")
    L = torch.full((B,), 4, dtype=torch.int64); RL = torch.ones(B, dtype=torch.int64)
    for b, (zb, mb, meanb, refb, rmb, _, cb, nb, Tb) in enumerate(reqs):
        R = refb.shape[-1]
        z[b, :, :Tb], mean[b, :, :Tb], mask[b, :, :Tb], L[b] = zb[0], meanb[0], mb[0], Tb
        ref[b, :, :R], rmask[b, :, :R], c[b], RL[b] = refb[0], rmb[0], cb[0], R
        noise[:, b, :, :Tb] = nb[:, 0]
    rmask[RL == 1, :, 0] = 1.0
    return z, mask, mean, ref, rmask, ref * 0.5, c, noise, L.cuda(), RL.cuda()


def static_call(eng, z, mask, mean, ref, rmask, mref, c, noise, L, RL):
    cond = eng.vc_conditioning(ref, rmask, mref, c, N, ref_lengths=RL)
    return eng.vc_reverse_diffusion(z, mask, mean, cond, N, MODE, noise, lengths=L)


def static_run(eng, reqs, arrive):
    now, i, n = 0.0, 0, len(reqs)
    clock, done, queue = StepClock(), {}, []
    while len(done) < n:
        while i < n and arrive[i] <= now:
            queue.append(i); i += 1
        if not queue:
            now = arrive[i]
            continue
        take, queue = queue[:CAP], queue[CAP:]
        packed = pack([reqs[j] for j in take])
        _, ms = timed(lambda: static_call(eng, *packed))
        clock.run(now, ms, N)
        now += ms
        for j in take:
            done[j] = now
    lat = [done[j] - arrive[j] for j in range(n)]
    steps = [clock.steps_at(done[j]) - clock.steps_at(arrive[j]) for j in range(n)]
    return lat, steps, max(done.values()) - arrive[0]


def rolling_run(rs, reqs, arrive, step_ms):
    now, i, n = 0.0, 0, len(reqs)
    clock, done, rid_of = StepClock(), {}, {}
    while len(done) < n:
        while i < n and arrive[i] <= now:
            r = reqs[i]
            rid, ms = timed(lambda: rs.submit(*r[:7], N, MODE, r[7]))     # its conditioning is GPU time too
            clock.run(now, ms, 0)
            now += ms
            rid_of[rid] = i
            i += 1
        if rs.busy == 0:
            now = arrive[i]
            continue
        cap = None
        if rs.busy < CAP and i < n:
            cap = max(1, int(round((arrive[i] - now) / step_ms)))
        k = min(rs.next_completion(), cap) if cap else rs.next_completion()
        out, ms = timed(lambda: rs.advance(max_steps=k))
        step_ms = ms / k
        clock.run(now, ms, k)
        now += ms
        for rid in out:
            done[rid_of[rid]] = now
    lat = [done[j] - arrive[j] for j in range(n)]
    steps = [clock.steps_at(done[j]) - clock.steps_at(arrive[j]) for j in range(n)]
    return lat, steps, max(done.values()) - arrive[0]


def per_step(dec, eng, reqs, busy, reps):
    """per-step ms of a rolling step with `busy` of CAP slots running vs a lengths= step at (busy, T) on the same rows,
    alternating.  The slots run requests of more steps than the window advances, so none finishes inside it."""
    rows = reqs[:busy]
    z, mask, mean, ref, rmask, mref, c, noise, L, RL = pack(rows, busy)
    cond = eng.vc_conditioning(ref, rmask, mref, c, N, ref_lengths=RL)
    long_n = N * (reps + 2)
    rs = dec.rolling(CAP, T)
    for r in rows:
        rs.submit(*r[:7], long_n, MODE, torch.randn(long_n, 1, 80, r[8], device="cuda"))
    rs.advance(max_steps=N)
    eng.vc_reverse_diffusion(z, mask, mean, cond, N, MODE, noise, lengths=L)
    roll, batch = [], []
    for _ in range(reps):
        _, ms = timed(lambda: rs.advance(max_steps=N))
        roll.append(ms / N)
        _, ms = timed(lambda: eng.vc_reverse_diffusion(z, mask, mean, cond, N, MODE, noise, lengths=L))
        batch.append(ms / N)
    r, b = statistics.median(roll), statistics.median(batch)
    return {"busy_slots": busy, "rolling_step_ms": r, "lengths_step_ms": b, "rolling_over_lengths": r / b,
            "rolling_runs": roll, "lengths_runs": batch}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="tf32,bf16")
    ap.add_argument("--requests", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    reqs, gaps = make_trace(args.requests)
    frames = sum(r[1].sum().item() for r in reqs)
    res = {"trace": {"requests": args.requests, "N": N, "mode": MODE, "capacity": CAP, "T": T, "valid_frames": frames},
           **card(), "modes": {}}
    cfg = DiffVCConfig()
    sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    for precision in args.modes.split(","):
        dec = Diffusion(80, cfg.dim_unet, cfg.dim_spk, True, cfg.beta_min, cfg.beta_max, precision=precision).eval()
        dec.load_state_dict(sd, strict=True)
        dec = dec.cuda()
        eng = dec.engine()
        packed = pack(reqs[:CAP])
        static_call(eng, *packed)                                           # warm-up: plan, graph
        _, batch_ms = timed(lambda: static_call(eng, *packed))
        rate = 0.9 * CAP / batch_ms                                          # requests per ms
        arrive = torch.cumsum(gaps / rate, 0).tolist()
        arrive = [a - arrive[0] for a in arrive]
        lat, steps, span = static_run(eng, reqs, arrive)
        st = summary(lat, steps, frames, span)
        rs = dec.rolling(CAP, T)
        rs.submit(*reqs[0][:7], 2, MODE)                                     # warm-up: slot plan, graph
        rs.drain()
        lat, steps, span = rolling_run(rs, reqs, arrive, batch_ms / N)
        ro = summary(lat, steps, frames, span)
        del rs
        occ = [per_step(dec, eng, reqs, b, args.reps) for b in (CAP, CAP // 2)]
        res["modes"][precision] = {"static_batch_ms": batch_ms, "arrival_rate_per_s": rate * 1e3, "static": st, "rolling": ro,
                                   "per_step": occ}
        print(json.dumps({precision: res["modes"][precision]}), flush=True)
    res["card_after"] = card()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
