"""Rolling Grad-TTS batches without a GPU: the C ABI's new entry points, RollingSampler's argument refusals, and its
scheduler - FIFO admission, epochs that end at the next completion, slot reuse, drain - against a fake engine that records
the slot operations and computes a recognisable "mel" per request."""
import pytest
import torch

from speech_backbones_b200.rolling import RollingSampler

F = 80


class FakeEngine:
    """The engine surface RollingSampler uses.  A slot's result is mu * (steps it ran): wrong step counts show."""

    def __init__(self, n_spks=1, spk_emb_dim=64):
        self.n_feats, self.n_spks, self.spk_emb_dim = F, n_spks, spk_emb_dim
        self.torch_device = torch.device("cpu")
        self.log = []                       # ("admit", slot, T_b, N) | ("advance", k) | ("read", slot) | ("release", slot)
        self.slots = {}                     # slot -> [mu, N, steps run]

    def rolling_reserve(self, capacity, max_frames):
        self.log.append(("reserve", capacity, max_frames))

    def rolling_admit(self, slot, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None):
        assert slot not in self.slots
        self.log.append(("admit", slot, z.shape[-1], n_timesteps))
        self.slots[slot] = [mu.clone(), n_timesteps, 0]

    def rolling_advance(self, steps):
        self.log.append(("advance", steps))
        for s in self.slots.values():
            s[2] = min(s[1], s[2] + steps)

    def rolling_read(self, slot, frames):
        mu, n, done = self.slots[slot]
        assert done == n and mu.shape[-1] == frames
        self.log.append(("read", slot))
        return mu * done

    def rolling_release(self, slot):
        self.log.append(("release", slot))
        del self.slots[slot]


def _req(Tb, seed=0):
    g = torch.Generator().manual_seed(seed)
    mu = torch.randn(1, F, Tb, generator=g)
    return mu + torch.randn(1, F, Tb, generator=g), torch.ones(1, 1, Tb), mu


def test_new_symbols_are_exported(sbk_lib):
    from speech_backbones_b200.binding import EXPORTS
    for name in ("sbk_rolling_reserve", "sbk_rolling_admit", "sbk_rolling_advance", "sbk_rolling_read", "sbk_rolling_release"):
        assert name in EXPORTS
        getattr(sbk_lib, name)


def test_null_handle_is_refused(sbk_lib):
    SBK_ERR_ARG = 1
    assert sbk_lib.sbk_rolling_reserve(None, 4, 512, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_rolling_admit(None, 0, None, None, None, None, None, 4, 1, 0, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_rolling_advance(None, 1, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_rolling_read(None, 0, None, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_rolling_release(None, 0, None) == SBK_ERR_ARG


def test_fifo_admission_epochs_and_slot_reuse():
    eng = FakeEngine()
    rs = RollingSampler(eng, 2, 64)
    Ns = [5, 2, 3, 1, 4]
    reqs = [_req(4 * (i + 1), i) for i in range(5)]
    ids = [rs.submit(*reqs[i], Ns[i]) for i in range(5)]
    assert ids == [0, 1, 2, 3, 4]
    assert rs.busy == 2 and rs.pending == 3
    # slots 0, 1 run requests 0 (N=5) and 1 (N=2): the first epoch ends when request 1 finishes
    assert rs.next_completion() == 2
    out = rs.advance()
    assert list(out) == [1]
    # request 2 (N=3) takes slot 1; request 0 has 3 steps left
    assert rs.slots[1].rid == 2 and rs.next_completion() == 3
    out = rs.advance()
    assert sorted(out) == [0, 2]
    assert [r.rid for r in rs.slots] == [3, 4]
    out.update(rs.drain())
    assert sorted(out) == [0, 2, 3, 4]
    epochs = [e[1] for e in eng.log if e[0] == "advance"]
    # epoch lengths: min(N_b - i_b) over busy slots - 2 (req 1), 3 (req 0 and 2), 1 (req 3), 3 (req 4's rest)
    assert epochs == [2, 3, 1, 3]
    assert rs.steps_run == sum(epochs)
    admits = [e for e in eng.log if e[0] == "admit"]
    assert [(a[1], a[2], a[3]) for a in admits] == [(0, 4, 5), (1, 8, 2), (1, 12, 3), (0, 16, 1), (1, 20, 4)]
    # each mel ran exactly its own N steps
    assert torch.equal(out[4], reqs[4][2] * 4)
    assert rs.busy == 0 and rs.pending == 0 and rs.advance() == {}


def test_drain_returns_every_id_exactly_once():
    eng = FakeEngine()
    rs = RollingSampler(eng, 3, 32)
    g = torch.Generator().manual_seed(3)
    seen, Ns = [], {}
    for i in range(20):
        N = int(torch.randint(1, 7, (1,), generator=g))
        Ns[rs.submit(*_req(4 * int(torch.randint(1, 9, (1,), generator=g)), i), N)] = N
        if i % 4 == 3:
            seen += list(rs.advance(max_steps=2))
    seen += list(rs.drain())
    assert sorted(seen) == list(range(20))
    assert eng.slots == {}
    assert [e for e in eng.log if e[0] == "read"] and all(k <= 6 for k in (e[1] for e in eng.log if e[0] == "advance"))


def test_max_steps_caps_an_epoch():
    eng = FakeEngine()
    rs = RollingSampler(eng, 1, 8)
    rid = rs.submit(*_req(8), 5)
    assert rs.advance(max_steps=2) == {} and rs.advance(max_steps=2) == {}
    out = rs.advance(max_steps=2)
    assert list(out) == [rid]
    assert [e[1] for e in eng.log if e[0] == "advance"] == [2, 2, 1]


def test_argument_refusals_before_any_launch():
    eng = FakeEngine(n_spks=4)
    rs = RollingSampler(eng, 2, 16)
    z, mask, mu = _req(8)
    spk = torch.zeros(1, 64)
    bad = {
        "frames not a multiple of 4": (z[..., :6], mask[..., :6], mu[..., :6], 2, False, spk, None),
        "frames past max_frames": (torch.zeros(1, F, 20), torch.ones(1, 1, 20), torch.zeros(1, F, 20), 2, False, spk, None),
        "float64": (z.double(), mask, mu, 2, False, spk, None),
        "mask shape": (z, mask[:, :, :4], mu, 2, False, spk, None),
        "mu shape": (z, mask, mu[:, :40], 2, False, spk, None),
        "batch of two": (z.repeat(2, 1, 1), mask.repeat(2, 1, 1), mu.repeat(2, 1, 1), 2, False, spk, None),
        "N = 0": (z, mask, mu, 0, False, spk, None),
        "N not an int": (z, mask, mu, 2.0, False, spk, None),
        "no spk": (z, mask, mu, 2, False, None, None),
        "spk shape": (z, mask, mu, 2, False, torch.zeros(1, 32), None),
        "noise shape": (z, mask, mu, 2, True, spk, torch.zeros(3, 1, F, 8)),
        "not a tensor": (z.tolist(), mask, mu, 2, False, spk, None),
    }
    for name, args in bad.items():
        with pytest.raises(ValueError):
            rs.submit(*args)
        assert eng.log == [("reserve", 2, 16)], name
    with pytest.raises(ValueError):
        rs.advance(max_steps=0)
    with pytest.raises(ValueError):
        RollingSampler(FakeEngine(), 0, 16)
    with pytest.raises(ValueError):
        RollingSampler(FakeEngine(), 2, 18)


def test_stochastic_request_draws_its_noise_in_step_order():
    eng = FakeEngine()
    rs = RollingSampler(eng, 1, 8)
    z, mask, mu = _req(8)
    torch.manual_seed(5)
    rs.submit(z, mask, mu, 3, stoc=True)
    torch.manual_seed(5)
    want = torch.stack([torch.randn(z.shape) for _ in range(3)])
    assert torch.equal(rs.slots[0].noise, want)
