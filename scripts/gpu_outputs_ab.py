"""Bit-identity A/B of two builds: this tree and another built source tree (e.g. the parent commit, built in place with
`python __graft_entry__.py`), on the same GPU.

    python scripts/gpu_outputs_ab.py OTHER_ROOT

One worker process per tree imports the package of ITS tree only and runs, in every precision mode the engine has, the
U-Net's `reverse_diffusion` (B = 32 and 1, T = 512, 4 steps; at B = 1 also one captured estimator call: at B = 32 its
captures would be tens of GB per mode), the HiFi-GAN vocoder V1 and V3 with capture on (B = 32, T = 512 and B = 3,
T = 301), the PostNet (B = 64, T = 256, ragged mask) and the RefBlock conditioning branch (`sbk_vc_conditioning`,
N = 6, with capture).  It reports a digest of every output and capture (sha) and
each call's launch count; the report says per (engine, mode, shape) whether the outputs, every capture and the launch
counts of the two trees are equal.  Exit status 1 if anything differs."""
import hashlib
import json
import os
import subprocess
import sys

MODES = ("fp32x3", "tf32", "bf16", "fp32")


def sha(t):
    """SHA-256 of a CPU tensor's bytes; a CUDA tensor (float32) is reduced on the device to a position-weighted sum of its
    bit patterns mod 2^64 first (a copy of every vocoder capture to the host would dominate the run)"""
    if t is None:
        return None
    t = t.detach().contiguous()
    if t.is_cuda:
        import torch
        v = t.view(-1).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
        w = (torch.arange(v.numel(), device=v.device, dtype=torch.int64) * 0x9E3779B1 + 0x7F4A7C15) & 0xFFFFFFFF
        return f"{v.numel()}:{int((v * w).sum())}:{int(v.sum())}"
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()


def worker(root):
    sys.path.insert(0, root)
    import torch
    from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
    from speech_backbones_b200.binding import Engine
    from speech_backbones_b200.hifigan import VocoderEngine
    from speech_backbones_b200.postnet import PostNetEngine
    from speech_backbones_b200.spec import (HIFIGAN_V1, HIFIGAN_V3, DiffVCConfig, diffvc_param_spec,
                                            synthetic_hifigan_state_dict, synthetic_postnet_state_dict)
    res = {}                                  # "engine/mode/shape" -> {"out": sha, "launches": n, "cap:<name>": sha}
    sd = synthetic_state_dict(UNetConfig())
    for B in (32, 1):
        z, mask, mu, _, _ = synthetic_inputs(B, 512, ragged=True)
        z, mask, mu = z.cuda(), mask.cuda(), mu.cuda()
        for m in MODES:
            e = Engine(precision=m)
            e.load_state_dict(sd)
            r = {"out": sha(e.reverse_diffusion(z, mask, mu, 4)), "launches": e.last_launch_count()}
            if B == 1:
                e.debug_capture(True)
                r["est"] = sha(e.estimator(z, mask, mu, torch.linspace(0.9, 0.2, B, device="cuda")))
                r["est_launches"] = e.last_launch_count()
                r.update({f"cap:{n}": sha(e.debug_read(n)) for n in e.debug_names()})
            e.close()
            res[f"unet/{m}/B{B}"] = r
            print(f"{root}: unet {m} B={B} done", file=sys.stderr, flush=True)
    for vname, h in (("v1", HIFIGAN_V1), ("v3", HIFIGAN_V3)):
        vsd = synthetic_hifigan_state_dict(1234, h)
        for B, T in ((32, 512), (3, 301)):
            mel = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(B * T)).cuda()
            for m in MODES:
                e = VocoderEngine(h, 0, m)
                e.load_state_dict(vsd)
                e.debug_capture(True)
                r = {"out": sha(e.forward(mel)), "launches": e.last_launch_count()}
                r.update({f"cap:{n}": sha(e.debug_read(n)) for n in e.debug_names()})
                e.close()
                res[f"vocoder-{vname}/{m}/B{B}T{T}"] = r
                print(f"{root}: vocoder {vname} {m} B={B} done", file=sys.stderr, flush=True)
    psd = synthetic_postnet_state_dict(128, 7)
    x = torch.randn(64, 80, 256, generator=torch.Generator().manual_seed(64)).cuda()
    pmask = (torch.arange(256)[None, :] < torch.randint(1, 257, (64,), generator=torch.Generator().manual_seed(1))[:, None])
    pmask = pmask.float()[:, None].cuda()
    for m in MODES:
        e = PostNetEngine(128, precision=m)
        e.load_state_dict(psd)
        res[f"postnet/{m}/B64T256"] = {"out": sha(e.forward(x, pmask)), "launches": e.last_launch_count()}
        e.close()
    cfg = DiffVCConfig()
    vcsd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    gen = torch.Generator().manual_seed(257)
    ref, mean_ref, c = torch.randn(2, 80, 257, generator=gen), torch.randn(2, 80, 257, generator=gen), torch.randn(2, 256, generator=gen)
    rmask = (torch.arange(257)[None, :] < torch.tensor([257, 129])[:, None]).float()[:, None]
    ref, mean_ref, c, rmask = ref.cuda(), mean_ref.cuda(), (c / c.norm(dim=1, keepdim=True)).cuda(), rmask.cuda()
    for m in MODES:
        e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=m, use_ref_t=cfg.use_ref_t)
        e.load_state_dict(vcsd)
        e.debug_capture(True)
        r = {"out": sha(e.vc_conditioning(ref, rmask, mean_ref, c, 6)), "launches": e.last_launch_count()}
        r.update({f"cap:{n}": sha(e.vc_cond_debug_read(n)) for n in e.vc_cond_debug_names()})
        e.close()
        res[f"refblock/{m}/B2Tr257N6"] = r
    print("RESULT " + json.dumps(res), flush=True)


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    if len(args) != 1:
        sys.exit(__doc__)
    if "--worker" in sys.argv:
        return worker(os.path.abspath(args[0]))
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    roots = {"this": here, "other": os.path.abspath(args[0])}
    print("#", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip())
    got = {}
    for k, root in roots.items():
        p = subprocess.run([sys.executable, os.path.abspath(__file__), root, "--worker"], stdout=subprocess.PIPE, text=True, cwd=root)
        line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
        if p.returncode != 0 or not line:
            sys.exit(f"worker for {root} failed ({p.returncode}):\n{p.stdout[-2000:]}")
        got[k] = json.loads(line[0][len("RESULT "):])
    bad = 0
    print(f"{'engine/mode/shape':32s} {'outputs':8s} {'captures':>12s} {'launches':>16s}")
    for case in sorted(set(got["this"]) | set(got["other"])):
        a, b = got["other"].get(case, {}), got["this"].get(case, {})
        caps = sorted(n for n in set(a) | set(b) if n.startswith("cap:"))
        outs = [n for n in ("out", "est") if n in a or n in b]
        launches = [n for n in ("launches", "est_launches") if n in a or n in b]
        ok_out = all(a.get(n) == b.get(n) for n in outs)
        ok_cap = sum(a.get(n) == b.get(n) for n in caps)
        ok_l = all(a.get(n) == b.get(n) for n in launches)
        bad += (not ok_out) + (ok_cap != len(caps)) + (not ok_l)
        lc = "/".join(str(b.get(n)) for n in launches)
        print(f"{case:32s} {'equal' if ok_out else 'DIFFER':8s} {ok_cap:5d}/{len(caps):<5d}  {'equal' if ok_l else 'DIFFER':6s} {lc:>9s}")
        for n in caps:
            if a.get(n) != b.get(n):
                print(f"    capture differs: {n[4:]}")
    print("ALL BITWISE EQUAL" if bad == 0 else f"{bad} DIFFERENCES")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
