"""GPU parity at the shapes, precisions and horizons BASELINE.json's configs are benchmarked on (VERDICT r1 item 2).

The CPU oracle is the checker; each case is sized so that the oracle finishes in under a minute on the GPU box's host cores:

* config 3 (bf16, N = 1000): one utterance (B=1, T=64) run to N = 1000 on the GPU in bf16 AND on the CPU oracle in fp32 - the
  claim "operand-rounding errors do not grow with the number of steps" measured, not modelled;
* config 4 (DiffVC, fast-ML sampler N = 6, T = T_ref = 256): one sample against the oracle, conditioning branch native;
* config 2 / config 3 batches: an utterance alone reproduces its rows inside the batch exactly in every mode
  (the property batch sharding across GPUs rests on), at T = 512.
(config 2's B=32 x T=512 estimator check in all tensor-core modes lives in tests/test_fp32x3_gpu.py.)
"""
import pytest
import torch

from helpers import rel_l2
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
from oracle import diffvc_oracle as OV
from oracle import gradtts_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def n1000_case():
    """B=1, T=64, N=1000 on the CPU oracle - computed once (about a minute on the GPU box's host cores) for both modes."""
    cfg = UNetConfig()
    sd = synthetic_state_dict(cfg)
    z, mask, mu, _, _ = synthetic_inputs(1, 64)
    with torch.no_grad():
        ref = O.reverse_diffusion(sd, cfg, z, mask, mu, 1000)
    return sd, z, mask, mu, ref


@pytest.mark.parametrize("precision,tol", [("bf16", 1e-2), ("fp32x3", 2e-4)])
def test_config3_long_horizon_n1000_vs_oracle(sbk_lib, n1000_case, precision, tol):
    """N = 1000 Euler steps, B=1, T=64: the GPU trajectory against the fp32 CPU oracle run to the same N."""
    from speech_backbones_b200.binding import Engine
    sd, z, mask, mu, ref = n1000_case
    N = 1000
    eng = Engine(precision=precision)
    eng.load_state_dict(sd)
    y = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), N).cpu()
    assert eng.last_host_launches() == 1                      # the whole 1000-step loop is ONE graph launch
    eng.close()
    err = rel_l2(y, ref)
    print(precision, "N=1000 B=1 T=64 rel_l2 vs oracle %.3e" % err)
    assert torch.isfinite(y).all()
    assert err <= tol


def test_config4_diffvc_ml_n6_t256_vs_oracle(sbk_lib):
    """DiffVC fast maximum-likelihood sampler, N = 6, T = T_ref = 256, one sample, default (fp32-class) precision, the
    hoisted RefBlock / cond_block branch evaluated natively (sbk_vc_conditioning)."""
    from speech_backbones_b200.diffvc import Diffusion
    from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs
    cfg = DiffVCConfig()
    sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    z, mask, mean, ref, ref_mask, mean_ref, c = synthetic_diffvc_inputs(1, 256, 256, seed=1234, ragged=False)
    N = 6
    torch.manual_seed(77)
    noise = torch.stack([torch.randn_like(z) for _ in range(N)])
    with torch.no_grad():
        want = OV.reverse_diffusion(sd, cfg, z, mask, mean, ref, ref_mask, mean_ref, c, N, "ml", noise=noise)
    for precision, tol in (("fp32x3", 2e-4), ("bf16", 4e-2)):
        dec = Diffusion(80, cfg.dim_unet, cfg.dim_spk, True, cfg.beta_min, cfg.beta_max, precision=precision).eval()
        dec.load_state_dict(sd, strict=True)
        dec = dec.cuda()
        eng = dec.engine()
        cond = dec.conditioning_table(ref.cuda(), ref_mask.cuda(), mean_ref.cuda(), c.cuda(), N)
        y = eng.vc_reverse_diffusion(z.cuda(), mask.cuda(), mean.cuda(), cond, N, "ml", noise.cuda()).cpu()
        err = rel_l2(y, want)
        print("DiffVC ml N=6 T=256", precision, "rel_l2 vs oracle %.3e" % err)
        assert err <= tol
        eng.close()


@pytest.mark.parametrize("precision", ["fp32x3", "tf32", "bf16"])
def test_alone_vs_in_batch_at_config_shapes(sbk_lib, precision):
    """scripts/gpu_config3.py's probe as a test: rows 5..6 of a B=8, T=512 ragged batch re-run alone (same padded T) for
    N = 20 steps reproduce their rows: bit for bit in the tf32 / bf16 modes (fp64 GroupNorm statistics, one
    accumulation run per output whatever the tiling), to fp32 rounding in the fp32x3 mode (a 2-utterance batch takes the
    64-wide N tiles: same sums, different fp32 rounding points)."""
    from speech_backbones_b200.binding import Engine
    cfg = UNetConfig()
    eng = Engine(precision=precision)
    eng.load_state_dict(synthetic_state_dict(cfg))
    z, mask, mu, _, _ = synthetic_inputs(8, 512, ragged=True)
    zd, md, mud = z.cuda(), mask.cuda(), mu.cuda()
    full = eng.reverse_diffusion(zd, md, mud, 20).cpu()
    part = eng.reverse_diffusion(zd[5:7].contiguous(), md[5:7].contiguous(), mud[5:7].contiguous(), 20).cpu()
    dep = rel_l2(part, full[5:7])
    print(precision, "rows 5..6 alone vs in batch", dep)
    assert dep == 0.0 if precision != "fp32x3" else dep < 1e-6
    eng.close()
