"""Rolling DiffVC batches without a GPU: the C ABI's new entry points, VcRollingSampler's argument refusals and draws, its
reuse of RollingSampler's scheduler (FIFO admission, epochs that end at the next completion, slot reuse), and the order of
DiffVC.rolling's draws - against a fake engine that records the slot operations."""
import types

import pytest
import torch

from speech_backbones_b200.diffvc import Diffusion, DiffVCRollingSampler, fix_len_compatibility
from speech_backbones_b200.rolling import VcRollingSampler
from test_rolling import FakeEngine

F, DC = 80, 128


class FakeVcEngine(FakeEngine):
    """The DiffVC engine surface VcRollingSampler uses; a slot's result is mean * (steps it ran)"""

    def __init__(self):
        super().__init__()
        self.dim_cond = DC
        self.admitted = {}                  # slot -> (z, cond, mode, noise) of its last admission

    def vc_rolling_reserve(self, capacity, max_frames):
        self.log.append(("reserve", capacity, max_frames))

    def vc_conditioning(self, ref, ref_mask, mean_ref, c, n_timesteps, ref_lengths=None):
        assert ref.shape[0] == 1 and ref_lengths is None
        self.log.append(("cond", ref.shape[-1], n_timesteps))
        return torch.full((n_timesteps, 1, DC), float(ref.shape[-1]))

    def vc_rolling_admit(self, slot, z, mask, mean, cond, n_timesteps, mode, noise=None):
        assert slot not in self.slots and cond.shape == (n_timesteps, 1, DC)
        self.log.append(("admit", slot, z.shape[-1], n_timesteps, mode))
        self.slots[slot] = [mean.clone(), n_timesteps, 0]
        self.admitted[slot] = (z.clone(), cond.clone(), mode, noise)


def _req(Tb, R=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(1, F, Tb, generator=g)
    ref = torch.randn(1, F, R, generator=g)
    c = torch.randn(1, 256, generator=g)
    return mean + torch.randn(1, F, Tb, generator=g), torch.ones(1, 1, Tb), mean, ref, torch.ones(1, 1, R), ref * 0.5, c


def test_new_symbols_are_exported(sbk_lib):
    from speech_backbones_b200.binding import EXPORTS
    for name in ("sbk_vc_rolling_reserve", "sbk_vc_rolling_admit"):
        assert name in EXPORTS
        getattr(sbk_lib, name)


def test_null_handle_is_refused(sbk_lib):
    SBK_ERR_ARG = 1
    assert sbk_lib.sbk_vc_rolling_reserve(None, 4, 512, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_vc_rolling_admit(None, 0, None, None, None, None, None, 4, 1, 0, None) == SBK_ERR_ARG


def test_fifo_admission_epochs_and_slot_reuse():
    eng = FakeVcEngine()
    rs = VcRollingSampler(eng, 2, 64)
    Ns, modes = [5, 2, 3, 1, 4], ["pf", "ml", "em", "pf", "ml"]
    reqs = [_req(4 * (i + 1), 8 + i, i) for i in range(5)]
    ids = [rs.submit(*reqs[i], Ns[i], modes[i]) for i in range(5)]
    assert ids == [0, 1, 2, 3, 4]
    assert rs.busy == 2 and rs.pending == 3 and rs.next_completion() == 2
    out = rs.advance()
    assert list(out) == [1] and rs.slots[1].rid == 2 and rs.next_completion() == 3
    out.update(rs.advance())
    assert [r.rid for r in rs.slots] == [3, 4]
    out.update(rs.drain())
    assert sorted(out) == [0, 1, 2, 3, 4]
    assert [e[1] for e in eng.log if e[0] == "advance"] == [2, 3, 1, 3]
    admits = [e[1:] for e in eng.log if e[0] == "admit"]
    assert admits == [(0, 4, 5, "pf"), (1, 8, 2, "ml"), (1, 12, 3, "em"), (0, 16, 1, "pf"), (1, 20, 4, "ml")]
    # each request's conditioning table: computed at submission, on its own reference, with its own N
    assert [e[1:] for e in eng.log if e[0] == "cond"] == [(8 + i, Ns[i]) for i in range(5)]
    assert torch.equal(out[4], reqs[4][2] * 4)
    assert rs.busy == 0 and rs.pending == 0 and rs.advance() == {}


def test_argument_refusals_before_any_launch():
    eng = FakeVcEngine()
    rs = VcRollingSampler(eng, 2, 16)
    z, mask, mean, ref, rmask, mref, c = _req(8)
    good = [z, mask, mean, ref, rmask, mref, c, 2, "ml", None]

    def with_(**kw):
        names = ["z", "mask", "mean", "ref", "ref_mask", "mean_ref", "c", "n_timesteps", "mode", "noise"]
        return [kw.get(n, v) for n, v in zip(names, good)]
    bad = {
        "frames not a multiple of 4": with_(z=z[..., :6], mask=mask[..., :6], mean=mean[..., :6]),
        "frames past max_frames": with_(z=torch.zeros(1, F, 20), mask=torch.ones(1, 1, 20), mean=torch.zeros(1, F, 20)),
        "float64": with_(z=z.double()),
        "mask shape": with_(mask=mask[:, :, :4]),
        "mean shape": with_(mean=mean[:, :40]),
        "batch of two": with_(z=z.repeat(2, 1, 1), mask=mask.repeat(2, 1, 1), mean=mean.repeat(2, 1, 1)),
        "ref not 3-d": with_(ref=ref[0]),
        "ref_mask shape": with_(ref_mask=rmask[:, :, :5]),
        "mean_ref shape": with_(mean_ref=mref[:, :, :5]),
        "ref float64": with_(ref=ref.double()),
        "c shape": with_(c=c[:, :128]),
        "c on another device": with_(c=c.to("meta")),
        "N = 0": with_(n_timesteps=0),
        "N not an int": with_(n_timesteps=2.0),
        "mode": with_(mode="sde"),
        "noise shape": with_(noise=torch.zeros(3, 1, F, 8)),
        "not a tensor": with_(z=z.tolist()),
    }
    for name, args in bad.items():
        with pytest.raises(ValueError):
            rs.submit(*args)
        assert eng.log == [("reserve", 2, 16)], name
    with pytest.raises(ValueError):
        VcRollingSampler(FakeVcEngine(), 2, 18)


@pytest.mark.parametrize("mode", ["em", "ml"])
def test_noise_is_drawn_at_submit_in_reverse_diffusions_order(mode):
    eng = FakeVcEngine()
    rs = VcRollingSampler(eng, 1, 8)
    z, *rest = _req(8)
    torch.manual_seed(5)
    rs.submit(z, *rest, 3, mode)
    torch.manual_seed(5)
    want = torch.stack([torch.randn_like(z) for _ in range(3)])
    assert torch.equal(rs.slots[0].noise, want) and torch.equal(eng.admitted[0][3], want)
    rs.submit(z, *rest, 2, "pf")                    # pf: no draws, no noise
    assert rs.queue[0].noise is None


def test_diffvc_rolling_draws_z_before_the_step_noise():
    """DiffVCRollingSampler.submit: the encoder on x and x_ref, then z = re-padded mean_x + randn_like (decoder_inputs),
    then the N step draws, as DiffVC.forward at B = 1 draws them"""
    dec = Diffusion(F, 8, DC, True, 0.05, 20.0)
    model = types.SimpleNamespace(encoder=lambda x, mask: (x * 0.5 + 1.0) * mask, decoder=dec)
    eng = FakeVcEngine()
    rs = DiffVCRollingSampler(model, eng, 2, 16)
    L, R, N = 13, 9, 3
    g = torch.Generator().manual_seed(1)
    x, x_ref, c = torch.randn(1, F, L, generator=g), torch.randn(1, F, R, generator=g), torch.randn(1, 256, generator=g)
    torch.manual_seed(7)
    rid = rs.submit(x, x_ref, c, N, "ml")
    Tp = fix_len_compatibility(L)
    torch.manual_seed(7)
    zdraw = torch.randn(1, F, Tp)
    steps = torch.stack([torch.randn(1, F, Tp) for _ in range(N)])
    mean = (x * 0.5 + 1.0)
    mean_x = dec.compute_diffused_mean(x, torch.ones(1, 1, L), mean, 1.0)
    want_z = torch.zeros(1, F, Tp)
    want_z[:, :, :L] = mean_x
    z, cond, mode, noise = eng.admitted[0]
    assert torch.equal(z, want_z + zdraw) and torch.equal(noise, steps) and mode == "ml"
    assert ("cond", R, N) in eng.log
    out = rs.drain()
    got_mean_x, y = out[rid]
    assert torch.equal(got_mean_x, mean_x) and y.shape == (1, F, L)
    with pytest.raises(ValueError):
        rs.submit(torch.randn(1, F, 17), x_ref, c, N)      # 20 U-Net frames > max_frames
    with pytest.raises(ValueError):
        rs.submit(x, x_ref, c, N, "sde")
