"""Rolling DiffVC batches on the GPU (`diffvc.Diffusion.rolling`, `DiffVC.rolling`, sbk.h: sbk_vc_rolling_*).

A seeded trace of 10 requests runs through a sampler of capacity 4 at max_frames 160: L in {1, 61, 131, 160, ...} (so T_b =
fix_len_compatibility(L) and a mask shorter than T_b), reference lengths R from 3 to 150, pf / em / ml with N in {1, 3, 6},
some requests submitted between advances into freed slots.  Every finished mel equals
  1. bit for bit in every mode, its row of an engine `vc_reverse_diffusion(..., lengths=)` call at (4, 160) with the same
     N, mode, conditioning rows and draws, the other rows other requests;
  2. with the 3x3 tile layout pinned (SBK_CONV3_ROWS = 1 or 2), the module's own B = 1 `forward`: bit for bit in tf32 and
     bf16, rel-L2 <= 1e-6 in fp32x3 and fp32 (the bound of test_vc_ragged_gpu.py);
  3. at the default layout, that call within the trajectory bound TOL[precision][1] of test_diffvc_gpu.py (the slot plan's
     tile count picks two-row tiles where the B = 1 plan picks one-row tiles), with the gap printed.
The module's own `forward` calls run between the sampler's steps: the sampler's slot plan is its own."""
import os

import pytest
import torch

from helpers import rel_l2
from test_diffvc_gpu import TOL
from speech_backbones_b200.diffvc import Diffusion, fix_len_compatibility
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_state_dict

pytestmark = pytest.mark.gpu

MODES = ("fp32x3", "tf32", "bf16", "fp32")
BITWISE = {"tf32", "bf16"}
CAP, TMAX = 4, 160
LENGTHS = [160, 61, 131, 1, 97, 160, 44, 131, 8, 61]
REFS = [97, 150, 3, 64, 128, 31, 150, 77, 12, 129]
STEPS = [6, 3, 1, 6, 3, 1, 6, 3, 6, 1]
SAMPLERS = ["ml", "pf", "em", "em", "ml", "pf", "pf", "ml", "em", "ml"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def state_dict():
    cfg = DiffVCConfig()
    return synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))


def _decoder(sd, precision):
    dec = Diffusion(80, 256, 128, True, 0.05, 20.0, precision=precision).eval()
    dec.load_state_dict(sd, strict=True)
    return dec.cuda()


def _pin(monkeypatch, layout):
    if layout != "auto":
        monkeypatch.setenv("SBK_CONV3_ROWS", layout[-1])


def _request(i):
    """(z, mask, mean, ref, ref_mask, mean_ref, c) of trace request i: the decoder's inputs at T_b = fix_len(L), mask 1 on L
    frames, mean 0 past them (as DiffVC.forward re-pads it), a reference of R frames"""
    L, R = LENGTHS[i], REFS[i]
    Tb = fix_len_compatibility(L)
    g = torch.Generator().manual_seed(300 + i)
    mask = (torch.arange(Tb) < L).float()[None, None]
    mean = torch.randn(1, 80, Tb, generator=g) * mask
    z = mean + torch.randn(1, 80, Tb, generator=g)
    ref = torch.randn(1, 80, R, generator=g)
    mean_ref = ref * 0.5 + torch.randn(1, 80, R, generator=g) * 0.1
    c = torch.randn(1, 256, generator=g)
    c = c / c.norm()
    return [t.cuda() for t in (z, mask, mean, ref, torch.ones(1, 1, R), mean_ref, c)]


def _noise(i):
    """the step draws of forward / submit after torch.manual_seed(700 + i) (None for pf)"""
    if SAMPLERS[i] == "pf":
        return None
    torch.manual_seed(700 + i)
    z = _request(i)[0]
    return torch.stack([torch.randn_like(z) for _ in range(STEPS[i])])


def _run_trace(dec):
    rs = dec.rolling(CAP, TMAX)
    out, index, single, launches = {}, {}, {}, []

    def submit(i):
        args = _request(i)
        torch.manual_seed(700 + i)
        rid = rs.submit(*args, STEPS[i], SAMPLERS[i])           # em / ml: draws its noise here
        index[rid] = i
        torch.manual_seed(700 + i)
        single[rid] = dec(*args, STEPS[i], SAMPLERS[i])        # the module's own call, between the sampler's steps

    def advance(**kw):
        out.update(rs.advance(**kw))
        launches.append(rs.engine.last_host_launches())

    for i in range(6):
        submit(i)
    advance(max_steps=2)
    submit(6)
    advance()
    advance(max_steps=1)
    for i in range(7, 10):
        submit(i)
    while rs.busy or rs.pending:
        advance()
    assert rs.steps_run < sum(STEPS)
    return out, index, single, launches


def _check_ragged_rows(dec, out, index):
    """contract 1: each request's mel is its row of a lengths= call at the sampler's shape, bit for bit"""
    eng = dec.engine()
    for i in range(len(LENGTHS)):
        rows = [i] + [j for j in range(len(LENGTHS)) if j != i][:CAP - 1]
        rows = rows[CAP - i % CAP:] + rows[:CAP - i % CAP]
        b = rows.index(i)
        N, mode = STEPS[i], SAMPLERS[i]
        z = torch.randn(CAP, 80, TMAX, device="cuda")
        mean = torch.randn(CAP, 80, TMAX, device="cuda")
        mask = torch.zeros(CAP, 1, TMAX, device="cuda")
        cond = torch.randn(N, CAP, 128, device="cuda") * 0.5
        for k, j in enumerate(rows):
            zj, mj, meanj = _request(j)[:3]
            Tj = zj.shape[-1]
            z[k, :, :Tj], mean[k, :, :Tj], mask[k, :, :Tj] = zj[0], meanj[0], mj[0]
        zi, mi, meani, ref, rmask, mref, c = _request(i)
        Tb = zi.shape[-1]
        cond[:, b] = eng.vc_conditioning(ref, rmask, mref, c, N)[:, 0]
        noise = None
        if mode != "pf":
            noise = torch.randn(N, CAP, 80, TMAX, device="cuda")
            noise[:, b, :, :Tb] = _noise(i)[:, 0]
        L = torch.tensor([fix_len_compatibility(LENGTHS[j]) for j in rows], device="cuda")
        y = eng.vc_reverse_diffusion(z, mask, mean, cond, N, mode, noise, lengths=L)
        rid = next(r for r, k in index.items() if k == i)
        assert torch.equal(out[rid], y[b:b + 1, :, :Tb]), (i, mode, N, rel_l2(out[rid], y[b:b + 1, :, :Tb]))


@pytest.mark.parametrize("layout", ["auto", "rows1", "rows2"])
@pytest.mark.parametrize("precision", MODES)
def test_trace_equals_ragged_and_single_calls(state_dict, precision, layout, monkeypatch):
    _pin(monkeypatch, layout)
    dec = _decoder(state_dict, precision)
    out, index, single, launches = _run_trace(dec)
    assert all(n == 1 for n in launches), launches
    assert sorted(out) == list(range(len(LENGTHS)))
    gaps = []
    for rid, y in out.items():
        i = index[rid]
        assert y.shape == (1, 80, fix_len_compatibility(LENGTHS[i]))
        assert bool(torch.isfinite(y).all()), rid
        err = rel_l2(y, single[rid])
        gaps.append(err)
        if layout == "auto":
            assert err <= TOL[precision][1], (precision, i, err)
        elif precision in BITWISE:
            assert torch.equal(y, single[rid]), (precision, layout, i, err)
        else:
            assert err <= 1e-6, (precision, layout, i, err)
    print(f"rolling DiffVC {precision} {layout}: vs own B = 1 forward, rel-L2 max {max(gaps):.2e} "
          + " ".join(f"{g:.1e}" for g in gaps))
    _check_ragged_rows(dec, out, index)


def test_alone_equals_full_and_released_slots_stay_finite(state_dict):
    dec = _decoder(state_dict, "tf32")
    rs = dec.rolling(CAP, TMAX)
    args = _request(4)
    torch.manual_seed(1)
    rid = rs.submit(*args, 3, "ml")
    alone = rs.drain()[rid]
    assert rs.engine.last_host_launches() == 1
    for i in (0, 1, 3):                          # three other requests, then the same one again, into used slots
        torch.manual_seed(2 + i)
        rs.submit(*_request(i), STEPS[i], SAMPLERS[i])
    torch.manual_seed(1)
    rid = rs.submit(*args, 3, "ml")
    full = rs.drain()
    assert all(bool(torch.isfinite(y).all()) for y in full.values())
    assert torch.equal(full[rid], alone)
    # every slot released: one more request alone in the cleared plan is still the same
    torch.manual_seed(1)
    rid = rs.submit(*args, 3, "ml")
    assert torch.equal(rs.drain()[rid], alone)


def test_vc_conditioning_between_advances_leaves_the_slots_intact(state_dict):
    dec = _decoder(state_dict, "tf32")
    results = []
    for interfere in (False, True):
        rs = dec.rolling(2, TMAX)
        ids = []
        for i in (0, 4):
            torch.manual_seed(50 + i)
            ids.append(rs.submit(*_request(i), STEPS[i], SAMPLERS[i]))
        out = rs.advance(max_steps=1)
        if interfere:
            g = torch.Generator().manual_seed(9)
            ref = torch.randn(3, 80, 200, generator=g).cuda()
            rs.engine.vc_conditioning(ref, torch.ones(3, 1, 200).cuda(), ref, torch.randn(3, 256, generator=g).cuda(), 5)
        out.update(rs.drain())
        results.append([out[r] for r in ids])
    assert all(torch.equal(a, b) for a, b in zip(*results))


def test_native_refusals(state_dict):
    from speech_backbones_b200.binding import Engine
    dec = _decoder(state_dict, "tf32")
    rs = dec.rolling(2, 64)
    eng = rs.engine
    z, mask, mean, ref, rmask, mref, c = _request(1)            # T_b = 64
    cond = eng.vc_conditioning(ref, rmask, mref, c, 3)
    noise = torch.randn(3, 1, 80, 64, device="cuda")
    for args in ((2, z, mask, mean, cond, 3, "pf"), (0, z, mask, mean, cond, 0, "pf")):
        with pytest.raises(RuntimeError):
            eng.vc_rolling_admit(*args)                         # slot out of range, N = 0
    with pytest.raises(RuntimeError):
        eng.vc_rolling_admit(0, z, mask, mean, cond, 3, "ml", None)     # ml without noise
    with pytest.raises(RuntimeError):
        eng.rolling_admit(0, z, mask, mean, 3)                  # a DiffVC handle through the Grad-TTS admission
    eng.vc_rolling_admit(0, z, mask, mean, cond, 3, "em", noise)
    with pytest.raises(RuntimeError):
        eng.vc_rolling_admit(0, z, mask, mean, cond, 3, "pf")   # busy
    eng.rolling_advance(3)
    assert torch.isfinite(eng.rolling_read(0, 64)).all()
    eng.vc_reverse_diffusion(z, mask, mean, cond, 3, "pf")      # another call replaces the slot plan
    with pytest.raises(RuntimeError, match="no slot plan"):
        eng.rolling_advance(1)
    with pytest.raises(RuntimeError):
        eng.rolling_reserve(2, 64)                              # still Grad-TTS only
    tts = Engine(n_feats=80, dim=64, precision="tf32")
    with pytest.raises(RuntimeError):
        tts.vc_rolling_reserve(2, 64)
    with pytest.raises(RuntimeError):
        tts.vc_rolling_admit(0, z, mask, mean, cond, 3, "pf")
    tts.close()


# ---- DiffVC.rolling on the reference golden --------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["auto", "rows1"])
@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_reference_golden_through_diffvc_rolling(monkeypatch, precision, layout):
    """The cases of tests/golden/diffvc_ragged_golden.pt (x_lengths {160, 131, 61, 1}, x_ref_lengths {97, 144, 130, 1}, N = 3,
    pf and ml), one utterance per request of DiffVC.rolling(2, 160), the recorded draws replayed as
    test_vc_ragged_gpu.py replays them: mean_x bit for bit the B = 1 DiffVC.forward's; y that call's bit for bit (tf32) or
    within 1e-6 (fp32x3) with the layout pinned, within the trajectory bound at the default layout, and within ENC_TOL /
    TRAJ_TOL of the reference's B = 1 outputs."""
    from speech_backbones_b200.diffvc import DiffVC
    from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS
    from oracle import postnet_oracle as O
    from test_postnet_gpu import ENC_TOL, TRAJ_TOL
    from test_vc_ragged_gpu import _golden_script, _replay
    G = _golden_script()
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_ragged_golden.pt"), weights_only=False)
    _pin(monkeypatch, layout)
    sd = O.model_synthetic_weights(G.SEED)
    model = DiffVC(*DIFFVC_MODEL_ARGS, precision=precision).eval()
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    x, x_ref, c = G.inputs()
    for case in golden["cases"]:
        mode = case["mode"]
        noise = G.draws(mode)
        rs = model.rolling(2, G.T)
        ids = []
        for b in range(G.B):
            args = G.utterance(b, x, x_ref, c, noise)
            it = _replay(monkeypatch, args[5])
            ids.append(rs.submit(args[0].cuda(), args[2].cuda(), args[4].cuda(), G.N, mode))
            assert next(it, None) is None
        out = rs.drain()
        for b, rid in enumerate(ids):
            args = G.utterance(b, x, x_ref, c, noise)
            L = G.LENGTHS[b]
            mean_x, y = (t.cpu() for t in out[rid])
            _replay(monkeypatch, args[5])
            m1, y1 = (t.cpu() for t in model(*(a.cuda() for a in args[:5]), G.N, mode))
            assert mean_x.shape == (1, 80, L) and y.shape == (1, 80, L)
            assert torch.equal(mean_x, m1), f"{mode} mean_x utterance {b}"
            err = rel_l2(y, y1)
            if layout == "auto":
                assert err <= TOL[precision][1], (mode, b, err)
                om, oy = G.oracle_forward(sd, *args[:5], mode, args[5])
                e1, e2 = rel_l2(mean_x, om), rel_l2(y, oy)
                print(f"DiffVC.rolling {precision} {mode} utterance {b} (L={L}, R={G.REF_LENGTHS[b]}): vs own call {err:.2e}, "
                      f"vs the reference's B = 1 call mean_x {e1:.2e} y {e2:.2e}")
                assert e1 <= ENC_TOL[precision] and e2 <= TRAJ_TOL[precision]
            elif precision == "tf32":
                assert torch.equal(y, y1), (mode, b, err)
            else:
                assert err <= 1e-6, (mode, b, err)
