"""GPU parity tests: the sm_90a path (through the C ABI / the drop-in module) vs the CPU oracle and the
committed reference goldens.  Tolerances (fp32 CUDA-core path): rel-L2 <= 1e-4 per estimator call and per
intermediate, <= 2e-3 on trajectories (the random-weight reverse SDE is expansive, SURVEY.md 8c)."""
import pytest
import torch

from helpers import case_id, case_inputs, nhwc_to_nchw, rel_l2, stoc_noise
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_noise, synthetic_state_dict
from oracle import gradtts_oracle as O

pytestmark = pytest.mark.gpu

EST_TOL = 1e-4
TRAJ_TOL = 2e-3


@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache = {}

    def get(n_spks=1, use_graph=True, seed=1234, precision="fp32"):
        key = (n_spks, use_graph, seed, precision)
        if key not in cache:
            cfg = UNetConfig(n_spks=n_spks)
            e = Engine(n_spks=n_spks, use_graph=use_graph, precision=precision)
            e.load_state_dict(synthetic_state_dict(cfg, seed))
            cache[key] = e
        return cache[key]
    yield get
    for e in cache.values():
        e.close()


# tensors that feed LinearAttention keep their padded columns (attention reads the unmasked x, diffusion.py:192);
# in the tensor-core modes every other activation is stored already multiplied by its level's mask
ATTN_INPUTS = {"estimator.downs.0.1.out", "estimator.downs.1.1.out", "estimator.downs.2.1.out",
               "estimator.mid_block1.out", "estimator.ups.0.1.out", "estimator.ups.1.1.out"}


def stagewise_errors(eng, cfg, sd, xt, mask, mu, t, spk, masked_storage=False):
    """Run one estimator call on the GPU and compare every named intermediate with the oracle's."""
    dev = "cuda"
    eng.debug_capture(True)
    y = eng.estimator(xt.to(dev), mask.to(dev), mu.to(dev), t.to(dev), None if spk is None else spk.to(dev))
    torch.cuda.synchronize()
    eng.debug_capture(False)
    taps = {}
    y_ref = O.estimator(sd, cfg, xt, mask, mu, t, spk, taps=taps)
    rows = []
    for name in eng.debug_names():
        if name not in taps:
            continue
        ref = taps[name]
        got = eng.debug_read(name)
        if got is None:
            continue
        if name.endswith(".ctx"):
            got = got.view(ref.shape)
        else:
            B, C, H, W = ref.shape
            got = nhwc_to_nchw(got, B, H, W, C, eng.debug_layout(name))
            if masked_storage and not name.endswith(".raw") and name not in ATTN_INPUTS:
                mk = mask[:, None, :, ::mask.shape[-1] // W]          # this level's mask [B,1,1,W]
                ref = ref * mk
        rows.append((name, rel_l2(got, ref), ref.abs().max().item()))
    rows.append(("estimator.out", rel_l2(y.cpu(), y_ref), y_ref.abs().max().item()))
    return rows


@pytest.mark.parametrize("B,T,n_spks", [(2, 32, 1), (3, 100, 1), (1, 4, 1), (2, 32, 4)])
def test_stagewise_intermediates(engines, B, T, n_spks):
    cfg = UNetConfig(n_spks=n_spks)
    sd = synthetic_state_dict(cfg)
    z, mask, mu, spk, _ = synthetic_inputs(B, T, ragged=True, n_spks=n_spks)
    t = torch.linspace(0.9, 0.2, B)
    rows = stagewise_errors(engines(n_spks), cfg, sd, z * mask, mask, mu, t, spk)
    report = "\n".join(f"{n:48s} rel_l2={e:.3e} |ref|max={m:.3g}" for n, e, m in rows)
    print(report)
    bad = [r for r in rows if not (r[1] <= EST_TOL)]
    assert not bad, "first divergent stage: %s\n%s" % (bad[0][0], report)


def _golden_cases(kind):
    import os
    path = os.path.join(os.path.dirname(__file__), "golden", "gradtts_golden.pt")
    g = torch.load(path, weights_only=False)
    return [(i, c) for i, c in enumerate(g["cases"]) if c["kind"] == kind]


@pytest.mark.parametrize("idx,c", _golden_cases("est"), ids=[case_id(c) for _, c in _golden_cases("est")])
def test_estimator_vs_reference_golden(engines, golden, idx, c):
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    eng = engines(c["n_spks"])
    xt = z * mask * c["scale"]
    y = eng.estimator(xt.cuda(), mask.cuda(), mu.cuda(), torch.tensor(c["t"]).cuda(),
                      None if spk is None else spk.cuda()).cpu()
    err = rel_l2(y, golden["cases"][idx]["out"])
    print(case_id(c), "rel_l2", err)
    assert err <= EST_TOL
    assert (y * (1 - mask)).abs().max().item() == 0.0        # padded frames are exactly zero


@pytest.mark.parametrize("idx,c", _golden_cases("traj"), ids=[case_id(c) for _, c in _golden_cases("traj")])
def test_trajectory_vs_reference_golden(engines, golden, idx, c):
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    eng = engines(c["n_spks"])
    noise = stoc_noise(golden, c).cuda() if c["stoc"] else None
    y = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), c["N"], c["stoc"],
                              None if spk is None else spk.cuda(), noise).cpu()
    ref = golden["cases"][idx]["out"]
    err = rel_l2(y, ref)
    print(case_id(c), "rel_l2", err)
    assert err <= TRAJ_TOL
    assert (y * (1 - mask)).abs().max().item() == 0.0


def test_dropin_module_forward_matches_golden(golden):
    """Diffusion(...).load_state_dict(strict) -> .cuda() -> forward(z, mask, mu, N): the call tts.py:96 makes."""
    from speech_backbones_b200.gradtts import Diffusion
    idx, c = next((i, c) for i, c in _golden_cases("traj") if c["N"] == 10 and c["B"] == 2)
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    dec = Diffusion(80, 64).eval()
    dec.load_state_dict(sd, strict=True)
    dec = dec.cuda()
    y = dec(z.cuda(), mask.cuda(), mu.cuda(), n_timesteps=10, stoc=False, spk=None)
    assert y.shape == z.shape and y.is_cuda and y.dtype == torch.float32
    assert rel_l2(y.cpu(), c["out"]) <= TRAJ_TOL
    # weights changed in place -> engine re-packs
    with torch.no_grad():
        dec.estimator.final_conv.bias.add_(1.0)
    y2 = dec(z.cuda(), mask.cuda(), mu.cuda(), n_timesteps=10)
    assert rel_l2(y2.cpu(), c["out"]) > 1e-3
    # stochastic branch runs and is finite (its RNG stream is torch's CUDA generator, not comparable to CPU)
    y3 = dec(z.cuda(), mask.cuda(), mu.cuda(), n_timesteps=3, stoc=True)
    assert torch.isfinite(y3).all()
    assert dec.engine().last_launch_count() > 0


def test_graph_replay_equals_eager_launches(engines):
    z, mask, mu, _, _ = synthetic_inputs(2, 64, ragged=True)
    a = engines(1, True).reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 6)
    b = engines(1, False).reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 6)
    # GN statistics are accumulated with fp64 atomics, so run-to-run differences are at the 1e-7 level
    assert rel_l2(a.cpu(), b.cpu()) < 1e-5
    # second replay of the instantiated graph, different N (time table is rebuilt, graph reused)
    c = engines(1, True).reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 6)
    assert rel_l2(c.cpu(), a.cpu()) < 1e-5


def test_sliced_steps_equal_one_shot(engines):
    eng = engines(1, True)
    B, T, N = 2, 32, 8
    z, mask, mu, _, _ = synthetic_inputs(B, T, ragged=True)
    noise = synthetic_noise(N, B, T).cuda()
    for stoc in (False, True):
        full = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), N, stoc, None, noise if stoc else None)
        xt = (z * mask).cuda().contiguous()
        for s0, s1 in ((0, 3), (3, 4), (4, 8)):
            eng.reverse_steps(xt, mask.cuda(), mu.cuda(), N, s0, s1, stoc, None, noise[s0:s1] if stoc else None)
        assert rel_l2(xt.cpu(), full.cpu()) < 1e-5


def test_host_buffer_entry_point(engines):
    eng = engines(1, True)
    z, mask, mu, _, _ = synthetic_inputs(2, 32, ragged=True)
    dev = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 5).cpu()
    host = eng.reverse_diffusion_host(z.pin_memory(), mask.pin_memory(), mu.pin_memory(), 5)
    assert not host.is_cuda
    assert rel_l2(host, dev) < 1e-5


def test_batch_independence_and_padding(engines):
    """Utterances never mix (the property that lets batches shard across GPUs, SURVEY.md 8e):
    sample b alone at the same padded T gives the same result as inside the batch."""
    eng = engines(1, True)
    z, mask, mu, _, _ = synthetic_inputs(4, 64, ragged=True)
    t = torch.full((4,), 0.4)
    full = eng.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
    for b in (1, 3):
        one = eng.estimator((z * mask)[b:b + 1].cuda(), mask[b:b + 1].cuda(), mu[b:b + 1].cuda(), t[b:b + 1].cuda()).cpu()
        assert rel_l2(one, full[b:b + 1]) < 1e-5


def test_config2_shape_properties(engines):
    """BASELINE config 2 (B=32, T=512): too big for the oracle in a test, so check size-independent properties
    plus the oracle on one sample (padding is live, so the sample keeps the batch's padded T)."""
    eng = engines(1, True)
    B, T = 32, 512
    z, mask, mu, _, _ = synthetic_inputs(B, T, ragged=True)
    t = torch.full((B,), 0.5)
    y = eng.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
    assert torch.isfinite(y).all()
    assert (y * (1 - mask)).abs().max().item() == 0.0
    cfg = UNetConfig()
    sd = synthetic_state_dict(cfg)
    b = 5
    ref = O.estimator(sd, cfg, (z * mask)[b:b + 1], mask[b:b + 1], mu[b:b + 1], t[b:b + 1])
    assert rel_l2(y[b:b + 1], ref) <= EST_TOL
    out = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 2).cpu()
    assert torch.isfinite(out).all() and (out * (1 - mask)).abs().max().item() == 0.0


# ---- tensor-core precision modes (wgmma tf32 / bf16 operands, fp32 accumulate in registers) ----
# Tolerances follow the operand rounding (SURVEY.md 8c, measured by emulation on the reference):
# tf32 (10-bit mantissa) ~1e-3 per estimator call, bf16 (8-bit) ~9e-3; GN/softmax/Mish/Euler stay fp32.
# bf16 mode: conv inputs AND the residual stream are stored as bf16 (8-bit mantissa, 2^-9 relative rounding per store),
# accumulation / GN statistics / raw conv outputs / sampler state fp32 (SURVEY 8c predicted 9e-3 per call, 3-5e-3 on
# trajectories).
TC_TOL = {"tf32": (4e-3, 8e-3), "bf16": (2e-2, 1e-2)}       # (per estimator call / stage, trajectory)
# The |xt| x100 stress case drives the attention logits k to O(100): softmax turns the tf32 operand rounding of the
# k projection (|k| * 2^-11 absolute) into a relative error of the same size in p = exp(k - max), so this one case
# gets a wider bound (measured 4.7e-3; the reference's own TF32 GPU path has the same sensitivity).
TC_TOL_STRESS = {"tf32": 1e-2, "bf16": 6e-2}


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
@pytest.mark.parametrize("B,T", [(2, 32), (3, 100), (1, 256), (1, 4)])
def test_tensor_core_stagewise(engines, precision, B, T):
    cfg = UNetConfig()
    sd = synthetic_state_dict(cfg)
    z, mask, mu, spk, _ = synthetic_inputs(B, T, ragged=True)
    t = torch.linspace(0.9, 0.2, B)
    rows = stagewise_errors(engines(1, True, 1234, precision), cfg, sd, z * mask, mask, mu, t, spk, masked_storage=True)
    report = "\n".join(f"{n:48s} rel_l2={e:.3e} |ref|max={m:.3g}" for n, e, m in rows)
    print(report)
    bad = [r for r in rows if not (r[1] <= TC_TOL[precision][0])]
    assert not bad, "first divergent stage: %s\n%s" % (bad[0][0], report)


@pytest.mark.parametrize("precision", ["tf32", "bf16"])
def test_tensor_core_vs_reference_golden(engines, golden, precision):
    eng = engines(1, True, 1234, precision)
    for idx, c in _golden_cases("est") + _golden_cases("traj"):
        if c["n_spks"] != 1:
            continue
        cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
        if c["kind"] == "est":
            y = eng.estimator((z * mask * c["scale"]).cuda(), mask.cuda(), mu.cuda(), torch.tensor(c["t"]).cuda()).cpu()
            tol = TC_TOL[precision][0] if c["scale"] == 1.0 else TC_TOL_STRESS[precision]
        else:
            noise = stoc_noise(golden, c).cuda() if c["stoc"] else None
            y = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), c["N"], c["stoc"], None, noise).cpu()
            tol = TC_TOL[precision][1]
        err = rel_l2(y, c["out"])
        print(precision, case_id(c), "rel_l2", err)
        assert err <= tol, case_id(c)
        assert (y * (1 - mask)).abs().max().item() == 0.0


def test_tf32_multispeaker_and_module(golden):
    from speech_backbones_b200.gradtts import Diffusion
    idx, c = next((i, c) for i, c in _golden_cases("traj") if c["n_spks"] == 4)
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    dec = Diffusion(80, 64, n_spks=4, precision="tf32").eval()
    dec.load_state_dict(sd, strict=True)
    dec = dec.cuda()
    y = dec(z.cuda(), mask.cuda(), mu.cuda(), c["N"], False, spk.cuda()).cpu()
    assert rel_l2(y, c["out"]) <= TC_TOL["tf32"][1]


def test_bf16_multispeaker_module_and_bf16_io(golden):
    """Config 3's calling convention: the module in bf16 mode, bf16 tensors in -> bf16 tensor out (state stays fp32)."""
    from speech_backbones_b200.gradtts import Diffusion
    idx, c = next((i, c) for i, c in _golden_cases("traj") if c["n_spks"] == 4)
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    dec = Diffusion(80, 64, n_spks=4, precision="bf16").eval()
    dec.load_state_dict(sd, strict=True)
    dec = dec.cuda()
    y = dec(z.cuda(), mask.cuda(), mu.cuda(), c["N"], False, spk.cuda()).cpu()
    assert y.dtype == torch.float32 and rel_l2(y, c["out"]) <= TC_TOL["bf16"][1]
    yb = dec(z.cuda().bfloat16(), mask.cuda().bfloat16(), mu.cuda().bfloat16(), c["N"], False, spk.cuda().bfloat16())
    assert yb.dtype == torch.bfloat16 and yb.shape == z.shape
    assert rel_l2(yb.float().cpu(), c["out"]) <= TC_TOL["bf16"][1] + 1.5e-2        # + bf16 rounding of z / mu / the result


def test_bf16_tracks_tf32_at_config_shapes(engines):
    """bf16 vs tf32 engines on the same inputs at config 2's width (T=512): the two tensor-core modes must agree to bf16
    rounding and padded frames must be exactly zero."""
    z, mask, mu, _, _ = synthetic_inputs(3, 512, ragged=True)
    t = torch.tensor([0.9, 0.5, 0.1])
    e16, e32 = engines(1, True, 1234, "bf16"), engines(1, True, 1234, "tf32")
    y16 = e16.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
    y32 = e32.estimator((z * mask).cuda(), mask.cuda(), mu.cuda(), t.cuda()).cpu()
    assert rel_l2(y16, y32) <= TC_TOL["bf16"][0]
    assert (y16 * (1 - mask)).abs().max().item() == 0.0


@pytest.mark.parametrize("precision", ["fp32", "tf32", "bf16"])
def test_reproducible_and_batch_independent(engines, precision):
    """Same call twice -> same result; an utterance alone -> the same rows as inside a batch.  GroupNorm statistics are
    accumulated in fp64 (smem + global atomics), so the summation order cannot move the fp32 mean / rstd (1e-8 of order noise would be amplified by
    operand-rounding flips through this random-weight U-Net to visible per-call differences)."""
    z, mask, mu, _, _ = synthetic_inputs(3, 512, ragged=True)
    t = torch.tensor([0.9, 0.5, 0.1])
    eng = engines(1, True, 1234, precision)
    xt = (z * mask).cuda()
    a = eng.estimator(xt, mask.cuda(), mu.cuda(), t.cuda()).cpu()
    b = eng.estimator(xt, mask.cuda(), mu.cuda(), t.cuda()).cpu()
    one = eng.estimator(xt[1:2], mask[1:2].cuda(), mu[1:2].cuda(), t[1:2].cuda()).cpu()
    print(precision, "run-to-run", rel_l2(b, a), "alone vs in batch", rel_l2(one, a[1:2]))
    assert rel_l2(b, a) < 1e-6
    assert rel_l2(one, a[1:2]) < 1e-6
    n1 = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 10).cpu()
    n2 = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 10).cpu()
    assert rel_l2(n2, n1) < 1e-6


def test_oversize_batch_is_sliced(engines):
    """A batch whose workspace exceeds the limit is processed in independent slices with identical results."""
    eng = engines(1, True)
    z, mask, mu, _, _ = synthetic_inputs(5, 32, ragged=True)
    full = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 3).cpu()
    eng.max_workspace_bytes = eng.workspace_bytes(2, 32)
    try:
        assert len(eng.batch_slices(5, 32)) == 3
        sliced = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 3).cpu()
    finally:
        eng.max_workspace_bytes = None
    assert rel_l2(sliced, full) < 1e-5


def test_error_paths_raise(engines):
    eng = engines(1, True)
    z, mask, mu, _, _ = synthetic_inputs(1, 8)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        eng.reverse_diffusion(z, mask, mu, 2)
    with pytest.raises(RuntimeError, match="multiple of 4"):
        eng.reverse_diffusion(z[..., :6].contiguous().cuda(), mask[..., :6].contiguous().cuda(), mu[..., :6].contiguous().cuda(), 2)
    with pytest.raises(RuntimeError, match="noise"):
        eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 2, stoc=True)
