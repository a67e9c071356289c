"""How much of the GPU's reduced-precision error is the SAME error the operand-rounding model makes?  For every golden
estimator case: rel-L2 of the GPU output vs the fp32 reference, vs the model's output (oracle/precision_model.py, CPU), and
of the model vs the reference; the trajectory cases and the fp32x3 mode print GPU-vs-reference only.  If the kernels round exactly where the model does, GPU-vs-model is well below GPU-vs-reference
(what is left is accumulation order amplified through rounding flips).  Diagnostic for the next round; not part of the suite.
usage: python scripts/gpu_vs_precision_model.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as ge  # noqa: E402

ge.build()
from helpers import case_id, case_inputs, rel_l2, stoc_noise  # noqa: E402
from oracle import gradtts_oracle as O  # noqa: E402
from precision_model_fp16 import operand_rounding  # noqa: E402  (oracle/precision_model.py + the fp16 mode)
from speech_backbones_b200.binding import Engine  # noqa: E402

golden = torch.load(os.path.join(ROOT, "tests", "golden", "gradtts_golden.pt"), weights_only=False)
for mode in ("tf32", "bf16", "fp16", "fp32x3"):
    eng = None
    for c in golden["cases"]:
        if c["n_spks"] != 1 or (c["kind"] == "traj" and mode == "fp32x3"):
            continue
        cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
        if eng is None:
            eng = Engine(precision=mode)
            eng.load_state_dict(sd)
        if c["kind"] == "traj":
            noise = stoc_noise(golden, c).cuda() if c["stoc"] else None
            y_gpu = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), c["N"], c["stoc"], None, noise).cpu()
            print(f"{mode} {case_id(c)}: GPU-vs-ref {rel_l2(y_gpu, c['out']):.3e}", flush=True)
            continue
        xt, t = z * mask * c["scale"], torch.tensor(c["t"])
        y_gpu = eng.estimator(xt.cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
        if mode == "fp32x3":
            print(f"{mode} {case_id(c)}: GPU-vs-ref {rel_l2(y_gpu, c['out']):.3e}", flush=True)
            continue
        with operand_rounding(mode, sd), torch.no_grad():
            y_model = O.estimator(sd, cfg, xt, mask, mu, t, spk)
        print(f"{mode} {case_id(c)}: GPU-vs-ref {rel_l2(y_gpu, c['out']):.3e}  model-vs-ref {rel_l2(y_model, c['out']):.3e}  "
              f"GPU-vs-model {rel_l2(y_gpu, y_model):.3e}", flush=True)
    eng.close()
