"""The fp16 sampler mode on the GPU (sbk.h SBK_PREC_F16): the bf16 mode's operand layout, tiling and launches with fp16
elements, which keep tf32's 11 significant bits.

  * Accuracy: the Grad-TTS golden estimator calls and trajectories, and the DiffVC golden calls, within the tf32 mode's
    bounds (test_parity_gpu.py TC_TOL / TC_TOL_STRESS, test_diffvc_gpu.py TOL): fp16's operand rounding is tf32-class
    (tests/precision_model_fp16.py; the measured figures are pinned next to the model in
    test_precision_model_fp16.py).
  * The ragged and rolling machinery: a ragged row is bit for bit its own B = 1 call, with NaN past every edge of the
    batch's inputs (Grad-TTS; DiffVC at a pinned 3x3 tile layout, as test_vc_ragged_gpu.py pins it), and a rolling trace's
    mels are bit for bit the rows of a `lengths=` call - as in the tf32 and bf16 modes.
  * Run-to-run bitwise reproducibility, and the drop-in module's half-precision calling convention."""
import pytest
import torch

import test_ragged_decoder_gpu as RG
import test_rolling_gpu as RO
import test_vc_ragged_gpu as VR
import test_vc_rolling_gpu as VRO
from helpers import case_id, case_inputs, rel_l2, stoc_noise
from oracle import diffvc_oracle as DO
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_noise, synthetic_state_dict
from speech_backbones_b200.gradtts import fix_len_compatibility
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs
from speech_backbones_b200.spec import synthetic_state_dict as vc_state_dict
from test_diffvc_gpu import TOL as VC_TOL
from test_parity_gpu import TC_TOL, TC_TOL_STRESS

pytestmark = pytest.mark.gpu

EST_TOL, TRAJ_TOL, STRESS_TOL = TC_TOL["tf32"][0], TC_TOL["tf32"][1], TC_TOL_STRESS["tf32"]


@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache = {}

    def get(n_spks=1, seed=1234):
        if (n_spks, seed) not in cache:
            e = Engine(n_spks=n_spks, precision="fp16")
            e.load_state_dict(synthetic_state_dict(UNetConfig(n_spks=n_spks), seed))
            cache[(n_spks, seed)] = e
        return cache[(n_spks, seed)]
    yield get
    for e in cache.values():
        e.close()


# ---- accuracy: the reference goldens within the tf32 bounds ---------------------------------------------------------------
def test_gradtts_golden_within_tf32_bounds(engines, golden):
    """Every golden case, single- and multi-speaker: estimator calls within the tf32 per-call bound (the |xt| x100 stress
    case within tf32's stress bound), trajectories - deterministic and stochastic - within the tf32 trajectory bound."""
    seen = {"est": 0, "traj": 0, "stoc": 0, "spk": 0}
    for c in golden["cases"]:
        cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
        eng = engines(c["n_spks"], golden["seed"])
        s = None if spk is None else spk.cuda()
        if c["kind"] == "est":
            y = eng.estimator((z * mask * c["scale"]).cuda(), mask.cuda(), mu.cuda(), torch.tensor(c["t"]).cuda(), s).cpu()
            tol = EST_TOL if c["scale"] == 1.0 else STRESS_TOL
        else:
            noise = stoc_noise(golden, c).cuda() if c["stoc"] else None
            y = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), c["N"], c["stoc"], s, noise).cpu()
            tol = TRAJ_TOL
            seen["stoc"] += c["stoc"]
        err = rel_l2(y, c["out"])
        print(f"fp16 {case_id(c)}: rel-L2 {err:.3e} (bound {tol})")
        assert err <= tol, case_id(c)
        assert (y * (1 - mask)).abs().max().item() == 0.0
        seen[c["kind"]] += 1
        seen["spk"] += c["n_spks"] > 1
    assert seen["est"] and seen["traj"] and seen["stoc"] and seen["spk"], seen


@pytest.fixture(scope="module")
def vc_golden():
    import os
    return torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "diffvc_golden.pt"), weights_only=False)


def test_diffvc_golden_within_tf32_bounds(sbk_lib, vc_golden):
    """DiffVC's golden estimator calls and pf / em / ml trajectories (conditioning from the CPU oracle, as
    test_diffvc_gpu.py feeds it) within the tf32 mode's DiffVC bounds, and the native conditioning branch - which runs tf32
    operands in an fp16 handle, as in a bf16 one - feeding the ml sampler."""
    from speech_backbones_b200.binding import Engine
    cfg = DiffVCConfig()
    sd = vc_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    eng = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision="fp16")
    try:
        eng.load_state_dict(sd)
        for c in vc_golden["cases"]:
            z, mask, mean, r, rmask, mean_ref, spk = synthetic_diffvc_inputs(c["B"], c["T"], c["Tr"], seed=vc_golden["seed"],
                                                                             ragged=c["ragged"])
            if c["kind"] == "est":
                t = torch.tensor(c["t"])
                g = DO._gamma(cfg, 0, 0.5)
                _, cond = DO.conditioning(sd, cfg, ((r * g + mean_ref * (1.0 - g)) * rmask)[:, None], rmask, spk, t)
                y = eng.vc_estimator((z * mask).cuda(), mask.cuda(), mean.cuda(), cond.cuda(), t.cuda()).cpu()
                tol = VC_TOL["tf32"][0]
            else:
                N, mode = c["N"], c["mode"]
                rows = []
                for i in range(N):
                    t, _, _, _, g0t = DO.step_coefficients(cfg, N, i, mode)
                    xt_ref = ((r * g0t + mean_ref * (1.0 - g0t)) * rmask)[:, None]
                    rows.append(DO.conditioning(sd, cfg, xt_ref, rmask, spk, t * torch.ones(c["B"]))[1])
                noise = None
                if mode != "pf":
                    torch.manual_seed(vc_golden["noise_seed"])
                    noise = torch.stack([torch.randn_like(z) for _ in range(N)]).cuda()
                y = eng.vc_reverse_diffusion(z.cuda(), mask.cuda(), mean.cuda(), torch.stack(rows).cuda(), N, mode, noise).cpu()
                tol = VC_TOL["tf32"][1]
                if mode == "ml":
                    native = eng.vc_conditioning(r.cuda(), rmask.cuda(), mean_ref.cuda(), spk.cuda(), N)
                    yn = eng.vc_reverse_diffusion(z.cuda(), mask.cuda(), mean.cuda(), native, N, mode, noise).cpu()
                    assert rel_l2(yn, c["out"]) <= tol
            err = rel_l2(y, c["out"])
            print(f"fp16 diffvc {c['kind']} B{c['B']} T{c['T']} {c.get('mode', '')}: rel-L2 {err:.3e} (bound {tol})")
            assert err <= tol
            assert (y * (1 - mask)).abs().max().item() == 0.0
    finally:
        eng.close()


# ---- ragged batches: each row bit for bit its own call --------------------------------------------------------------------
def _rows_equal(out, single, tb):
    out = out.cpu()
    for b, Tb in enumerate(tb):
        row = out[b:b + 1, :, :Tb]
        one = single(b, Tb).cpu()
        assert bool(torch.isfinite(row).all()), (b, Tb)
        assert torch.equal(row, one), (b, Tb, (row - one).abs().max().item())
        assert torch.count_nonzero(out[b, :, Tb:]) == 0, b


@pytest.mark.parametrize("stoc", [False, True], ids=["det", "stoc"])
def test_gradtts_ragged_rows_with_nan_past_every_edge(engines, stoc):
    """B = 9, T = 516 (test_ragged_decoder_gpu.py's tile-edge batch): z, mask, mu - and the stochastic noise - NaN from every
    T_b on.  The estimator's and the sampler's rows are bit for bit the B = 1 calls on [:T_b] and 0 past T_b."""
    eng = engines()
    z, mask, mu, L = RG._nan_inputs()
    sl = RG._sl
    t = torch.linspace(0.9, 0.1, RG.NB, device="cuda")
    x = z * mask
    est = eng.estimator(x, mask, mu, t, lengths=L)
    _rows_equal(est, lambda b, Tb: eng.estimator(sl(x, b, Tb), sl(mask, b, Tb), sl(mu, b, Tb), t[b:b + 1]), RG.NTB)
    noise = RG._nan_past_edges(synthetic_noise(3, RG.NB, RG.NT)).cuda() if stoc else None
    out = eng.reverse_diffusion(z, mask, mu, 3, stoc, None, noise, lengths=L)
    _rows_equal(out, lambda b, Tb: eng.reverse_diffusion(sl(z, b, Tb), sl(mask, b, Tb), sl(mu, b, Tb), 3, stoc, None,
                                                         noise[:, b:b + 1, :, :Tb].contiguous() if stoc else None), RG.NTB)


@pytest.mark.parametrize("layout", ["rows1", "rows2"])
def test_diffvc_ragged_rows_at_a_pinned_layout(sbk_lib, layout, monkeypatch):
    """DiffVC's U-Net at T = 160, lengths {160, 131, 61, 1}, inputs NaN past every T'_b, the 3x3 tile layout pinned
    (SBK_CONV3_ROWS): the estimator's rows and the ml sampler's rows are bit for bit the B = 1 calls."""
    from speech_backbones_b200.binding import Engine
    monkeypatch.setenv("SBK_CONV3_ROWS", layout[-1])
    cfg = DiffVCConfig()
    eng = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision="fp16")
    try:
        eng.load_state_dict(vc_state_dict(cfg, VR.SEED, spec=diffvc_param_spec(cfg)))
        T, lengths, N = VR.T_VC, VR.LEN_VC, 3
        B = len(lengths)
        z, mean, cond = VR._vc_inputs(lengths, T, cfg.dim_spk, VR.SEED)
        mask = VR._mask(lengths, T)
        tp = [fix_len_compatibility(n) for n in lengths]
        L = torch.tensor(lengths).cuda()
        t = torch.tensor([0.9, 0.5, 0.3, 0.7])
        y = eng.vc_estimator(VR._poison(z * mask, tp).cuda(), mask.cuda(), VR._poison(mean, tp).cuda(), cond.cuda(), t.cuda(),
                             lengths=L)
        sl = lambda v, b, Tb: v[b:b + 1, :, :Tb].contiguous().cuda()             # noqa: E731
        _rows_equal(y, lambda b, Tb: eng.vc_estimator(sl(z * mask, b, Tb), sl(mask, b, Tb), sl(mean, b, Tb),
                                                      cond[b:b + 1].cuda(), t[b:b + 1].cuda()), tp)
        condn = torch.randn(N, B, cfg.dim_spk, generator=torch.Generator().manual_seed(VR.SEED)) * 0.5
        noise = torch.randn(N, B, 80, T, generator=torch.Generator().manual_seed(VR.SEED + 1))
        y = eng.vc_reverse_diffusion(VR._poison(z, tp).cuda(), mask.cuda(), VR._poison(mean, tp).cuda(), condn.cuda(), N, "ml",
                                     VR._poison(noise.transpose(0, 1), tp).transpose(0, 1).cuda(), lengths=L)
        _rows_equal(y, lambda b, Tb: eng.vc_reverse_diffusion(sl(z, b, Tb), sl(mask, b, Tb), sl(mean, b, Tb),
                                                              condn[:, b:b + 1].contiguous().cuda(), N, "ml",
                                                              noise[:, b:b + 1, :, :Tb].contiguous().cuda()), tp)
    finally:
        eng.close()


# ---- rolling batches: every finished mel is its row of a lengths= call ------------------------------------------------------
def test_gradtts_rolling_trace_equals_ragged_rows(sbk_lib):
    """test_rolling_gpu.py's 12-request trace (capacity 4, max_frames 512, N in {1, 3, 10, 50}) in fp16: each finished mel is
    bit for bit its row of an engine reverse_diffusion(..., lengths=) call and its own B = 1 forward."""
    dec = RO.Diffusion(80, 64, precision="fp16").eval()
    dec.load_state_dict(synthetic_state_dict(UNetConfig()))
    dec = dec.cuda()
    out, index, single = RO._run_trace(dec)[:3]
    RO._check("tf32", dec, out, index, single)            # "tf32": _check's bit-for-bit class, which fp16 belongs to


def test_diffvc_rolling_trace_equals_ragged_rows(sbk_lib, monkeypatch):
    """test_vc_rolling_gpu.py's trace in fp16 with the 3x3 layout pinned: each finished mel is bit for bit its row of a
    vc_reverse_diffusion(..., lengths=) call."""
    monkeypatch.setenv("SBK_CONV3_ROWS", "1")
    cfg = DiffVCConfig()
    dec = VRO._decoder(vc_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg)), "fp16")
    out, index, single = VRO._run_trace(dec)[:3]
    VRO._check_ragged_rows(dec, out, index)


# ---- reproducibility and the drop-in module -------------------------------------------------------------------------------
def test_run_to_run_bitwise(engines):
    z, mask, mu, _, _ = synthetic_inputs(3, 512, ragged=True)
    t = torch.tensor([0.9, 0.5, 0.1]).cuda()
    eng = engines()
    xt = (z * mask).cuda()
    a = eng.estimator(xt, mask.cuda(), mu.cuda(), t)
    assert torch.equal(a, eng.estimator(xt, mask.cuda(), mu.cuda(), t))
    n1 = eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 10)
    assert torch.equal(n1, eng.reverse_diffusion(z.cuda(), mask.cuda(), mu.cuda(), 10))


def test_module_half_in_half_out(golden):
    """The call a `model.half()` user makes: Diffusion(..., precision="fp16") fed torch.half tensors returns torch.half (the
    sampler state stays fp32 inside), within the tf32 trajectory bound plus the fp16 rounding of z / mu / the result."""
    from speech_backbones_b200.gradtts import Diffusion
    c = next(c for c in golden["cases"] if c["kind"] == "traj" and c["n_spks"] == 4)
    cfg, sd, z, mask, mu, spk = case_inputs(golden, c)
    dec = Diffusion(80, 64, n_spks=4, precision="fp16").eval()
    dec.load_state_dict(sd, strict=True)
    dec = dec.cuda()
    y = dec(z.cuda(), mask.cuda(), mu.cuda(), c["N"], False, spk.cuda())
    assert y.dtype == torch.float32 and rel_l2(y.cpu(), c["out"]) <= TRAJ_TOL
    yh = dec(z.cuda().half(), mask.cuda().half(), mu.cuda().half(), c["N"], False, spk.cuda().half())
    assert yh.dtype == torch.half and yh.shape == z.shape
    err = rel_l2(yh.float().cpu(), c["out"])
    print(f"fp16 module, half tensors in and out: rel-L2 {err:.3e}")
    assert err <= TRAJ_TOL + 2e-3
