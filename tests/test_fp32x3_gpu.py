"""GPU parity of the fp32-class tensor-core mode (precision="fp32x3", the drop-in modules' default).

Every dense contraction runs on wgmma as x_hi*w_hi (tf32) + (x_lo*w + x*w_lo) (one f16 MMA over packed fp16
correction chunks), fp32 accumulation in registers with the runs folded in round-to-nearest fp32;
GroupNorm, Mish, softmax, the attention context and the Euler update are exact fp32.  The reference computes in fp32
(Grad-TTS/model/diffusion.py:174-216,254-275 on the CPU), so this mode is held to an fp32-class bound against the
committed outputs of the unmodified reference:

    per estimator call / per intermediate  rel-L2 <= 1e-5      (the CUDA-core fp32 mode measures 0.6-2.6e-6)
    trajectories (N <= 50)                 rel-L2 <= 2e-4      (the random-weight reverse SDE is expansive, SURVEY 8c)

and, at the benchmarked shape (B=32, T=512), against the CPU oracle on two samples of the batch (padded T kept).
"""
import pytest
import torch

from helpers import case_id, case_inputs, rel_l2, stoc_noise
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
from oracle import gradtts_oracle as O
from test_parity_gpu import _golden_cases, stagewise_errors

pytestmark = pytest.mark.gpu

X3_EST_TOL = 1e-5
X3_STRESS_TOL = 3e-5       # |xt| x100: attention logits of O(100), exp() amplifies the 2^-22 operand residual
X3_TRAJ_TOL = 2e-4


@pytest.fixture(scope="module")
def x3_engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache = {}

    def get(n_spks=1, precision="fp32x3"):
        key = (n_spks, precision)
        if key not in cache:
            cfg = UNetConfig(n_spks=n_spks)
            e = Engine(n_spks=n_spks, precision=precision)
            e.load_state_dict(synthetic_state_dict(cfg, 1234))
            cache[key] = e
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("B,T,n_spks", [(2, 32, 1), (3, 100, 1), (1, 256, 1), (1, 4, 1), (2, 32, 4)])
def test_x3_stagewise(x3_engines, B, T, n_spks):
    cfg = UNetConfig(n_spks=n_spks)
    sd = synthetic_state_dict(cfg)
    z, mask, mu, spk, _ = synthetic_inputs(B, T, ragged=True, n_spks=n_spks)
    t = torch.linspace(0.9, 0.2, B)
    rows = stagewise_errors(x3_engines(n_spks), cfg, sd, z * mask, mask, mu, t, spk, masked_storage=True)
    report = "\n".join(f"{n:48s} rel_l2={e:.3e} |ref|max={m:.3g}" for n, e, m in rows)
    print(report)
    bad = [r for r in rows if not (r[1] <= X3_EST_TOL)]
    assert not bad, "first divergent stage: %s\n%s" % (bad[0][0], report)


def test_x3_vs_reference_golden(x3_engines, golden):
    """All 13 committed reference cases: single estimator calls and trajectories, 1 and 4 speakers."""
    worst = {}
    for idx, c in _golden_cases("est") + _golden_cases("traj"):
        eng = x3_engines(c["n_spks"])
        cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
        spk_d = None if spk is None else spk.cuda()
        if c["kind"] == "est":
            y = eng.estimator((z * mask * c["scale"]).cuda(), mask.cuda(), mu.cuda(), torch.tensor(c["t"]).cuda(), spk_d).cpu()
            tol = X3_EST_TOL if c["scale"] == 1.0 else X3_STRESS_TOL
        else:
            noise = stoc_noise(golden, c).cuda() if c["stoc"] else None
            y = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), c["N"], c["stoc"], spk_d, noise).cpu()
            tol = X3_TRAJ_TOL
        err = rel_l2(y, c["out"])
        print("fp32x3", case_id(c), "rel_l2 %.3e" % err)
        worst[case_id(c)] = (err, tol)
        assert (y * (1 - mask)).abs().max().item() == 0.0
    bad = {k: v for k, v in worst.items() if not v[0] <= v[1]}
    assert not bad, bad


@pytest.mark.parametrize("precision,tol", [("fp32x3", X3_EST_TOL), ("tf32", 4e-3), ("bf16", 2e-2)])
def test_benchmarked_shape_vs_oracle(x3_engines, precision, tol):
    """The bench shape (config 2: B=32, T=512, ragged lengths, padded T kept) in every tensor-core mode: two samples of the
    batch against the CPU oracle, padded frames exactly zero."""
    eng = x3_engines(1, precision)
    B, T = 32, 512
    z, mask, mu, _, _ = synthetic_inputs(B, T, ragged=True)
    t = torch.full((B,), 0.5)
    y = eng.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
    assert torch.isfinite(y).all()
    assert (y * (1 - mask)).abs().max().item() == 0.0
    cfg = UNetConfig()
    sd = synthetic_state_dict(cfg)
    for b in (5, 30):
        ref = O.estimator(sd, cfg, (z * mask)[b:b + 1], mask[b:b + 1], mu[b:b + 1], t[b:b + 1])
        err = rel_l2(y[b:b + 1], ref)
        print(precision, "B=32 T=512 sample", b, "rel_l2 %.3e" % err)
        assert err <= tol


def test_x3_reproducible_and_batch_independent(x3_engines):
    z, mask, mu, _, _ = synthetic_inputs(3, 512, ragged=True)
    t = torch.tensor([0.9, 0.5, 0.1])
    eng = x3_engines(1)
    xt = (z * mask).cuda()
    a = eng.estimator(xt, mask.cuda(), mu.cuda(), t.cuda()).cpu()
    b = eng.estimator(xt, mask.cuda(), mu.cuda(), t.cuda()).cpu()
    one = eng.estimator(xt[1:2], mask[1:2].cuda(), mu[1:2].cuda(), t[1:2].cuda()).cpu()
    print("fp32x3 run-to-run", rel_l2(b, a), "alone vs in batch", rel_l2(one, a[1:2]))
    assert rel_l2(b, a) < 1e-6
    assert rel_l2(one, a[1:2]) < 1e-6


def test_default_module_is_fp32_class(golden):
    """`Diffusion(80, 64)` - the documented one-line drop-in - runs the fp32-class mode."""
    from speech_backbones_b200.gradtts import Diffusion
    idx, c = next((i, c) for i, c in _golden_cases("traj") if c["N"] == 10 and c["B"] == 2)
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    dec = Diffusion(80, 64).eval()
    assert dec.precision == "fp32x3"
    dec.load_state_dict(sd, strict=True)
    dec = dec.cuda()
    y = dec(z.cuda(), mask.cuda(), mu.cuda(), n_timesteps=10).cpu()
    assert rel_l2(y, c["out"]) <= X3_TRAJ_TOL
