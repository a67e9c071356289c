"""Rolling vs static batching of a Grad-TTS decode service on one GPU, replaying a seeded arrival trace.

256 requests, T_b = fix_len_compatibility(U{256..512}), N = 50, arriving as a Poisson process at 0.9x the static batch's
measured throughput (so neither scheduler is idle for long nor swamped).  Two schedulers serve the same trace:
  (a) static: when the GPU is free, take up to 32 queued requests and run them as one `reverse_diffusion(..., lengths=)`
      at T = 512 (rows padded to 32 with 4-frame fillers when fewer are queued: one plan, one graph);
  (b) rolling: `Diffusion.rolling(32, 512)`; each epoch runs to the next completion, or - while slots are free and a request
      is due - to the step boundary nearest its arrival.
Time is virtual: the GPU time of each call (host clock around work that ends in a synchronise) is added to the clock, and
when nothing is queued the clock jumps to the next arrival.  Reported per mode: valid mel-frames/s over the busy-or-waiting
span, p50 / p95 latency (arrival to mel) in ms and in sampler steps (the steps the GPU ran in that interval; a partial epoch
counts its share), and
  - per-step time at full occupancy (32 busy slots, the trace's lengths) against a `reverse_diffusion(lengths=)` step at the
    same (B, T) and rows, the two alternating;
  - the cost of idle slots: a step with 16 of 32 slots busy against a `lengths=` step at B = 16.
The card's name, power limit and SM clock are read in the same run.

    python scripts/gpu_rolling_bench.py [--modes fp32x3,tf32,bf16,fp32] [--requests 256] [--reps 5] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from speech_backbones_b200 import UNetConfig, synthetic_state_dict  # noqa: E402
from speech_backbones_b200.gradtts import Diffusion, fix_len_compatibility  # noqa: E402

CAP, T, N = 32, 512, 50


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(), "nvidia_smi(name, power.limit, clocks.sm, clocks.max.sm)": q.stdout.strip()}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, (time.perf_counter() - t0) * 1e3


def make_trace(n, seed=7):
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for i in range(n):
        y = int(torch.randint(256, 513, (1,), generator=g))
        Tb = fix_len_compatibility(y)
        mu = torch.randn(1, 80, Tb, generator=g)
        z = mu + torch.randn(1, 80, Tb, generator=g) / 1.5
        mask = (torch.arange(Tb) < y).to(torch.float32)[None, None]
        reqs.append((z.cuda(), mask.cuda(), mu.cuda(), Tb))
    gaps = torch.empty(n).exponential_(1.0, generator=g)       # unit-rate gaps, scaled by the arrival rate later
    return reqs, gaps


def pack(reqs):
    """rows padded to CAP with 4-frame fillers: (z, mask, mu, lengths) at (CAP, T)"""
    z = torch.zeros(CAP, 80, T, device="cuda"); mu = torch.zeros_like(z); mask = torch.zeros(CAP, 1, T, device="cuda")
    L = torch.full((CAP,), 4, dtype=torch.int64)
    for b, (zb, mb, mub, Tb) in enumerate(reqs):
        z[b, :, :Tb], mu[b, :, :Tb], mask[b, :, :Tb], L[b] = zb[0], mub[0], mb[0], Tb
    return z, mask, mu, L.cuda()


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def summary(lat_ms, lat_steps, frames, span_ms):
    return {"mel_frames_per_s": frames / (span_ms / 1e3), "p50_ms": pct(lat_ms, .5), "p95_ms": pct(lat_ms, .95),
            "p50_steps": pct(lat_steps, .5), "p95_steps": pct(lat_steps, .95), "span_ms": span_ms}


class StepClock:
    """virtual time and the sampler's step count at each epoch edge, to express a latency in steps"""

    def __init__(self):
        self.edges = [(0.0, 0.0)]              # (ms, steps)

    def run(self, t0, ms, steps):
        self.edges.append((t0, self.edges[-1][1]))
        self.edges.append((t0 + ms, self.edges[-1][1] + steps))

    def steps_at(self, t):
        for (ta, sa), (tb, sb) in zip(self.edges, self.edges[1:]):
            if ta <= t <= tb:
                return sa if tb == ta else sa + (sb - sa) * (t - ta) / (tb - ta)
        return self.edges[-1][1]


def static_run(eng, reqs, arrive):
    now, i, n = 0.0, 0, len(reqs)
    clock, done = StepClock(), {}
    queue = []
    while len(done) < n:
        while i < n and arrive[i] <= now:
            queue.append(i); i += 1
        if not queue:
            now = arrive[i]
            continue
        take, queue = queue[:CAP], queue[CAP:]
        z, mask, mu, L = pack([reqs[j] for j in take])
        _, ms = timed(lambda: eng.reverse_diffusion(z, mask, mu, N, lengths=L))
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
            z, mask, mu, _ = reqs[i]
            rid_of[rs.submit(z, mask, mu, N)] = i
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


def full_occupancy(dec, eng, reqs, busy, reps):
    """per-step ms of a rolling step with `busy` of CAP slots running vs a lengths= step at (busy, T), alternating"""
    rows = reqs[:busy]
    z, mask, mu, L = pack(rows)
    z, mask, mu, L = z[:busy].contiguous(), mask[:busy].contiguous(), mu[:busy].contiguous(), L[:busy].contiguous()
    rs = dec.rolling(CAP, T)
    for zb, mb, mub, _ in rows:
        rs.submit(zb, mb, mub, 100000)
    steps = 50
    rs.advance(max_steps=steps)
    eng.reverse_diffusion(z, mask, mu, steps, lengths=L)
    roll, batch = [], []
    for _ in range(reps):
        _, ms = timed(lambda: rs.advance(max_steps=steps))
        roll.append(ms / steps)
        _, ms = timed(lambda: eng.reverse_diffusion(z, mask, mu, steps, lengths=L))
        batch.append(ms / steps)
    return {"busy_slots": busy, "rolling_step_ms": statistics.median(roll), "lengths_step_ms": statistics.median(batch),
            "rolling_over_lengths": statistics.median(roll) / statistics.median(batch),
            "rolling_runs": roll, "lengths_runs": batch}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--modes", default="fp32x3,tf32,bf16,fp32")
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    reqs, gaps = make_trace(args.requests)
    frames = sum(r[3] for r in reqs)
    res = {"trace": {"requests": args.requests, "N": N, "capacity": CAP, "T": T, "valid_frames": frames}, **card(), "modes": {}}
    sd = synthetic_state_dict(UNetConfig())
    for precision in args.modes.split(","):
        dec = Diffusion(80, 64, precision=precision).eval()
        dec.load_state_dict(sd)
        dec = dec.cuda()
        eng = dec.engine()
        z, mask, mu, L = pack(reqs[:CAP])
        eng.reverse_diffusion(z, mask, mu, N, lengths=L)                     # warm-up: plan, graph
        _, batch_ms = timed(lambda: eng.reverse_diffusion(z, mask, mu, N, lengths=L))
        rate = 0.9 * CAP / batch_ms                                          # requests per ms
        arrive = torch.cumsum(gaps / rate, 0).tolist()
        arrive = [a - arrive[0] for a in arrive]
        lat, steps, span = static_run(eng, reqs, arrive)
        st = summary(lat, steps, frames, span)
        rs = dec.rolling(CAP, T)
        warm = rs.submit(*reqs[0][:3], 2)
        rs.drain()
        lat, steps, span = rolling_run(rs, reqs, arrive, batch_ms / N)
        ro = summary(lat, steps, frames, span)
        del rs, warm
        occ = [full_occupancy(dec, eng, reqs, b, args.reps) for b in (CAP, CAP // 2)]
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
