"""Per-launch A/B of two builds of the tensor-core convs: this tree and another source tree (e.g. the parent commit, built
in place with `python __graft_entry__.py`), both on the same GPU in one session.

    python scripts/gpu_conv_inflight.py OTHER_ROOT [--reps=5] [--T=512]

Each rep runs one worker process per tree, alternating, so both builds see the same clocks and neighbours; a worker
imports the package of ITS tree only and, for B = 32 and B = 1 and each of fp32x3 / tf32 / bf16, plans the engine, runs
two warm-up reverse steps and records one `sbk_profile_ops` profile (one CUDA-event pair per launch).  The report is the
median over the reps of the per-launch ms, summed per launch kind: 3x3 Block convs (`.raw`), ResnetBlock 1x1 tails,
attention output (the per-sample 1x1 mix), Downsample, Upsample, the GroupNorm / Mish activation passes (`.act`), the
attention k|v kernel (`.kvpart`); and the sum over every launch of the step."""
import json
import os
import statistics
import subprocess
import sys

KINDS = ("conv3x3", "tail1x1", "attn_out", "down", "up", "act", "kvpart", "other")


def kind(name):
    if name.endswith(".raw"):
        return "conv3x3"
    if name.endswith(".act") or name.endswith(".kvpart"):
        return name.rsplit(".", 1)[1]
    if name.endswith(".3.out"):
        return "down" if ".downs." in name else "up"
    if name.endswith(".out") and (".2." in name or "mid_attn" in name):
        return "attn_out"
    if name.endswith(".out") and name != "estimator.out":
        return "tail1x1"
    return "other"


def worker(root, T):
    sys.path.insert(0, root)
    import torch
    import __graft_entry__ as ge
    ge.build()
    from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
    from speech_backbones_b200.binding import Engine
    sd = synthetic_state_dict(UNetConfig())
    out = {}
    for B in (32, 1):
        z, mask, mu, _, _ = synthetic_inputs(B, T)
        zd, md, mud = z.cuda(), mask.cuda(), mu.cuda()
        for prec in ("fp32x3", "tf32", "bf16"):
            e = Engine(precision=prec)
            e.load_state_dict(sd)
            e.reverse_diffusion(zd, md, mud, 2)
            torch.cuda.synchronize()
            out[f"{B}/{prec}"] = [(n, t) for n, t, _, _ in e.profile_ops()]
            e.close()
    print("RESULT " + json.dumps(out), flush=True)


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    opt = dict(a[2:].split("=", 1) for a in sys.argv[1:] if a.startswith("--") and "=" in a)
    T = int(opt.get("T", 512))
    if len(args) != 1:
        sys.exit(__doc__)
    if "--worker" in sys.argv:
        return worker(os.path.abspath(args[0]), T)
    reps = int(opt.get("reps", 5))
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    roots = {"this": here, "other": os.path.abspath(args[0])}
    print("#", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip())
    runs = {k: [] for k in roots}
    for _ in range(reps):
        for k, root in roots.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), root, "--worker", f"--T={T}"],
                               capture_output=True, text=True, cwd=root)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
            if p.returncode != 0 or not line:
                sys.exit(f"worker for {root} failed ({p.returncode}):\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            runs[k].append(json.loads(line[0][len("RESULT "):]))
    print(f"# per-launch ms, median of {reps} profiles per build, T = {T}; this = {roots['this']}, other = {roots['other']}")
    print(f"{'B/mode':10s} {'kind':9s} {'launches':>8s} {'other ms':>9s} {'this ms':>9s} {'other/this':>10s}")
    for case in runs["this"][0]:
        med = {}
        for k in roots:
            per = {}
            for r in runs[k]:
                for n, t in r[case]:
                    per.setdefault(n, []).append(t)
            med[k] = {n: statistics.median(v) for n, v in per.items()}
        for kd in KINDS + ("step",):
            names = [n for n in med["this"] if kd == "step" or kind(n) == kd]
            a = sum(med["other"].get(n, 0.0) for n in names)
            b = sum(med["this"][n] for n in names)
            print(f"{case:10s} {kd:9s} {len(names):8d} {a:9.3f} {b:9.3f} {a / b if b else 0:10.3f}x")


if __name__ == "__main__":
    main()
