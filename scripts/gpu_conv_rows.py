"""One- vs two-row tiles of the tensor-core 3x3 convs: L2 operand bytes per launch counted from shapes, and, on a GPU,
per-launch ms (sbk_profile_ops, one CUDA-event pair per launch) with SBK_CONV3_ROWS=1 and =2 alternated in one process.

    python scripts/gpu_conv_rows.py [B] [T] [precision ...] [--bytes-only]

L2 -> SM bytes of one launch = tiles x K sub-stages x (A halo tile + weight stage), sbk_conv_tc.cu: a tile is R rows x
128 pixels x NT channels, the halo tile 2 chunks x (R + 2) rows x 130 pixels x 16 B, the weight stage 9 taps x 2 chunks x NT
x 16 B; fp32x3 runs two sub-stages per K stage (correction + main).  Out-of-image rows and columns come from the zero page
and are counted like image bytes."""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# the tensor-core 3x3 convs of one Grad-TTS estimator call in plan order (sbk_api.cu build_plan): (name, cin, cout, level);
# downs.0.0.block1 (2 input channels) runs on CUDA cores
RESNETS = [("downs.0.0", 2, 64, 0), ("downs.0.1", 64, 64, 0), ("downs.1.0", 64, 128, 1), ("downs.1.1", 128, 128, 1),
           ("downs.2.0", 128, 256, 2), ("downs.2.1", 256, 256, 2), ("mid_block1", 256, 256, 2), ("mid_block2", 256, 256, 2),
           ("ups.0.0", 512, 128, 2), ("ups.0.1", 128, 128, 2), ("ups.1.0", 256, 64, 1), ("ups.1.1", 64, 64, 1)]
CONVS = [(f"estimator.{p}.block{k}.raw", cin if k == 1 else cout, cout, lvl)
         for p, cin, cout, lvl in RESNETS for k in (1, 2) if (p, k) != ("downs.0.0", 1)]
CONVS.append(("estimator.final_block.raw", 64, 64, 0))


def l2_bytes(B, T, cin, cout, lvl, rows, nt, precision, H0=80):
    H, W = H0 >> lvl, T >> lvl
    tiles = B * math.ceil(W / 128) * math.ceil(H / rows) * (cout // nt)
    sub = cin // (16 if precision == "bf16" else 8) * (2 if precision == "fp32x3" else 1)
    return tiles * sub * (2 * (rows + 2) * 130 * 16 + 9 * 2 * nt * 16)


def plan_tile(B, T, cout, lvl, rows, num_sms, H0=80):
    """(rows, NT) of sbk_api.cu tc_conv for a forced row count."""
    H, W = H0 >> lvl, T >> lvl
    if rows == 2:
        return 2, 64
    if cout % 128 == 0 and B * math.ceil(W / 128) * H * (cout // 128) * 2 > num_sms:
        return 1, 128
    return 1, 64


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    B = int(args[0]) if len(args) > 0 else 32
    T = int(args[1]) if len(args) > 1 else 512
    precs = args[2:] or ["fp32x3", "tf32", "bf16"]
    bytes_only = "--bytes-only" in sys.argv
    num_sms = 132
    for prec in precs:
        tot = {k: sum(l2_bytes(B, T, ci, co, lv, r, nt(co), prec) for _, ci, co, lv in CONVS)
               for k, r, nt in (("1 row x 128", 1, lambda c: 128 if c % 128 == 0 else 64), ("2 rows x 64", 2, lambda c: 64),
                                ("2 rows x 128", 2, lambda c: 128 if c % 128 == 0 else 64))}
        print(f"# B={B} T={T} {prec}: L2 operand bytes per step of {len(CONVS)} 3x3 launches: " +
              ", ".join(f"{k} {v / 1e9:.1f} GB" for k, v in tot.items()))
    if bytes_only:
        return

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: run with --bytes-only for the byte count")
    import __graft_entry__ as ge
    ge.build()
    from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
    from speech_backbones_b200.binding import Engine
    import subprocess
    print("#", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip())
    num_sms = torch.cuda.get_device_properties(0).multi_processor_count
    cfg = UNetConfig()
    sd = synthetic_state_dict(cfg)
    z, mask, mu, _, _ = synthetic_inputs(B, T)
    zd, md, mud = z.cuda(), mask.cuda(), mu.cuda()
    REPS = 5
    for prec in precs:
        engs = {}
        for rows in (1, 2):
            os.environ["SBK_CONV3_ROWS"] = str(rows)          # read when the engine plans (B, T)
            e = Engine(precision=prec)
            e.load_state_dict(sd)
            e.reverse_diffusion(zd, md, mud, 2)
            engs[rows] = e
        os.environ.pop("SBK_CONV3_ROWS")
        ms = {1: {}, 2: {}}
        for _ in range(REPS):                                 # alternated: both see the same clocks and neighbours
            for rows, e in engs.items():
                for n, t, _, _ in e.profile_ops():
                    ms[rows].setdefault(n, []).append(t)
        med = {r: {n: sorted(v)[len(v) // 2] for n, v in d.items()} for r, d in ms.items()}
        print(f"\n## {prec}: median of {REPS} per-launch profiles per row count; GB/s = L2 operand bytes / ms")
        print(f"{'conv':36s} {'cin':>4s} {'cout':>4s} {'lvl':>3s} | {'1-row ms':>8s} {'GB':>6s} {'GB/s':>6s} | "
              f"{'2-row ms':>8s} {'GB':>6s} {'GB/s':>6s} | speed-up")
        sums = {1: [0.0, 0.0], 2: [0.0, 0.0]}
        for n, ci, co, lv in CONVS:
            cells = []
            for rows in (1, 2):
                r, nt = plan_tile(B, T, co, lv, rows, num_sms)
                by = l2_bytes(B, T, ci, co, lv, r, nt, prec)
                t = med[rows][n]
                sums[rows][0] += t
                sums[rows][1] += by
                cells.append(f"{t:8.3f} {by / 1e9:6.2f} {by / t / 1e6:6.0f}")
            print(f"{n[len('estimator.'):]:36s} {ci:4d} {co:4d} {lv:3d} | {cells[0]} | {cells[1]} | "
                  f"{med[1][n] / med[2][n]:.2f}x")
        print(f"{'all 3x3 convs':52s} | {sums[1][0]:8.3f} {sums[1][1] / 1e9:6.1f} {sums[1][1] / sums[1][0] / 1e6:6.0f} | "
              f"{sums[2][0]:8.3f} {sums[2][1] / 1e9:6.1f} {sums[2][1] / sums[2][0] / 1e6:6.0f} | {sums[1][0] / sums[2][0]:.2f}x")
        step = {r: sum(med[r].values()) for r in (1, 2)}
        print(f"whole step (sum of per-launch ms): 1-row {step[1]:.3f} ms, 2-row {step[2]:.3f} ms, {step[1] / step[2]:.3f}x")
        for e in engs.values():
            e.close()


if __name__ == "__main__":
    main()
