"""Rolling Grad-TTS batches on the GPU (`Diffusion.rolling`, sbk.h: sbk_rolling_*).

A seeded trace of 12 requests runs through a sampler of capacity 4 at max_frames 512: T_b in {4, 132, 508, 512, ...},
N in {1, 3, 10, 50}, admitted at different steps, most of them into a slot another request has left.  Every finished mel
equals
  - the module's own B = 1 `forward` on that utterance: bit for bit in tf32 and bf16, rel-L2 < 1e-6 in fp32x3 and fp32
    (the ragged batch's bound, test_ragged_decoder_gpu.py), and
  - bit for bit in every mode, its row of an engine `reverse_diffusion(..., lengths=)` call at (4, 512) with N_b steps.
The module's `forward` calls are interleaved with the sampler's steps: the sampler's slot plan is its own."""
import pytest
import torch

from helpers import rel_l2
from speech_backbones_b200 import UNetConfig, synthetic_state_dict
from speech_backbones_b200.gradtts import Diffusion, fix_len_compatibility

pytestmark = pytest.mark.gpu

MODES = ("fp32x3", "tf32", "bf16", "fp32")
CAP, TMAX = 4, 512
FRAMES = [4, 132, 508, 512, 260, 64, 388, 200, 452, 16, 320, 96]
STEPS = [50, 3, 10, 1, 50, 10, 3, 1, 10, 50, 1, 3]


def _same(precision, got, want):
    if precision in ("tf32", "bf16"):
        return torch.equal(got, want)
    return rel_l2(got, want) < 1e-6


@pytest.fixture(scope="module")
def decoders(sbk_lib):
    cache = {}

    def get(precision, n_spks=1):
        if (precision, n_spks) not in cache:
            dec = Diffusion(80, 64, n_spks=n_spks, precision=precision).eval()
            dec.load_state_dict(synthetic_state_dict(UNetConfig(n_spks=n_spks)))
            cache[(precision, n_spks)] = dec.cuda()
        return cache[(precision, n_spks)]
    return get


def _request(i, n_spks=1):
    """(z, mask, mu, spk) of trace request i: z and mu random on all T_b frames, mask 1 on the first T_b - (i % 3) frames"""
    Tb = FRAMES[i]
    g = torch.Generator().manual_seed(100 + i)
    mu = torch.randn(1, 80, Tb, generator=g)
    z = mu + torch.randn(1, 80, Tb, generator=g) / 1.5
    mask = (torch.arange(Tb) < max(1, Tb - i % 3)).to(torch.float32)[None, None]
    spk = torch.randn(1, 64, generator=g) if n_spks > 1 else None
    return z.cuda(), mask.cuda(), mu.cuda(), None if spk is None else spk.cuda()


def _noise(i):
    """the draws of Diffusion.forward(..., stoc=True) after torch.manual_seed(500 + i)"""
    torch.manual_seed(500 + i)
    return torch.stack([torch.randn((1, 80, FRAMES[i]), device="cuda") for _ in range(STEPS[i])])


def _run_trace(dec, n_spks=1, stoc_of=lambda i: False):
    """The trace: 6 requests up front (2 queue), then more between steps.  Returns ({id: mel}, {id: trace index},
    {id: B = 1 forward}, host launches of every advance)."""
    rs = dec.rolling(CAP, TMAX)
    out, index, single, launches = {}, {}, {}, []

    def submit(i):
        z, mask, mu, spk = _request(i, n_spks)
        stoc = stoc_of(i)
        noise = _noise(i) if stoc else None
        rid = rs.submit(z, mask, mu, STEPS[i], stoc, spk, noise)
        index[rid] = i
        if stoc:
            torch.manual_seed(500 + i)
        single[rid] = dec(z, mask, mu, STEPS[i], stoc, spk)       # the module's own call, between the sampler's steps

    def advance(**kw):
        out.update(rs.advance(**kw))
        launches.append(rs.engine.last_host_launches())

    for i in range(6):
        submit(i)
    advance(max_steps=2)
    for i in range(6, 9):
        submit(i)
    advance()
    advance(max_steps=5)
    for i in range(9, 12):
        submit(i)
    while rs.busy or rs.pending:
        advance()
    assert rs.steps_run < sum(STEPS)
    return out, index, single, launches, rs


def _check(precision, dec, out, index, single, n_spks=1, stoc_of=lambda i: False):
    assert sorted(out) == list(range(12))
    eng = dec.engine()
    for rid, y in out.items():
        i = index[rid]
        Tb = FRAMES[i]
        assert y.shape == (1, 80, Tb)
        assert bool(torch.isfinite(y).all()), rid
        assert _same(precision, y, single[rid]), (precision, rid, Tb, STEPS[i], rel_l2(y, single[rid]))
    # against the ragged batch at the sampler's shape: each request in row i % 4 of a (4, 512) call with its N, the other
    # rows other requests of the trace
    for i in range(12):
        rows = [i] + [j for j in range(12) if j != i][:CAP - 1]
        rows = rows[CAP - i % CAP:] + rows[:CAP - i % CAP]
        z = torch.randn(CAP, 80, TMAX, device="cuda")
        mu = torch.randn(CAP, 80, TMAX, device="cuda")
        mask = torch.zeros(CAP, 1, TMAX, device="cuda")
        spk = torch.zeros(CAP, 64, device="cuda") if n_spks > 1 else None
        noise = torch.randn(STEPS[i], CAP, 80, TMAX, device="cuda") if stoc_of(i) else None
        for b, j in enumerate(rows):
            zj, mj, muj, sj = _request(j, n_spks)
            Tj = FRAMES[j]
            z[b, :, :Tj], mu[b, :, :Tj], mask[b, :, :Tj] = zj[0], muj[0], mj[0]
            if spk is not None:
                spk[b] = sj[0]
        b = rows.index(i)
        if noise is not None:
            noise[:, b, :, :FRAMES[i]] = _noise(i)[:, 0]
        L = torch.tensor([FRAMES[j] for j in rows], dtype=torch.int64, device="cuda")
        y = eng.reverse_diffusion(z, mask, mu, STEPS[i], noise is not None, spk, noise, lengths=L)
        rid = next(r for r, k in index.items() if k == i)
        assert torch.equal(out[rid], y[b:b + 1, :, :FRAMES[i]]), (precision, i, rel_l2(out[rid], y[b:b + 1, :, :FRAMES[i]]))


@pytest.mark.parametrize("precision", MODES)
def test_trace_equals_single_and_ragged_calls(decoders, precision):
    dec = decoders(precision)
    out, index, single, launches, _ = _run_trace(dec)
    assert all(n == 1 for n in launches), launches
    _check(precision, dec, out, index, single)


@pytest.mark.parametrize("precision", MODES)
def test_multi_speaker_stochastic_trace(decoders, precision):
    """n_spks = 4, and every other request stochastic with the draws of a reseeded generator"""
    dec = decoders(precision, 4)
    stoc_of = lambda i: i % 2 == 1                  # noqa: E731
    out, index, single, _, _ = _run_trace(dec, 4, stoc_of)
    _check(precision, dec, out, index, single, 4, stoc_of)


def test_unpinned_noise_matches_forward(decoders):
    """stoc=True without noise: the sampler draws what forward draws from the same generator state"""
    dec = decoders("tf32")
    rs = dec.rolling(2, 64)
    z, mask, mu, _ = _request(5)
    torch.manual_seed(9)
    rid = rs.submit(z, mask, mu, 4, stoc=True)
    out = rs.drain()
    torch.manual_seed(9)
    assert torch.equal(out[rid], dec(z, mask, mu, 4, stoc=True))


@pytest.mark.parametrize("precision", MODES)
def test_idle_slots(decoders, precision):
    """One request in 4 slots, then two: the idle slots leave only finite values in the live rows, every epoch is one host
    launch, and the mels are still their single calls"""
    dec = decoders(precision)
    rs = dec.rolling(CAP, TMAX)
    for i in (0, 2):
        z, mask, mu, _ = _request(i)
        rid = rs.submit(z, mask, mu, 7)
        got = rs.drain()
        assert rs.engine.last_host_launches() == 1
        assert bool(torch.isfinite(got[rid]).all())
        assert _same(precision, got[rid], dec(z, mask, mu, 7))
    reqs = [_request(i) for i in (1, 3)]
    ids = [rs.submit(z, mask, mu, n) for (z, mask, mu, _), n in zip(reqs, (3, 6))]
    first = rs.advance()
    assert list(first) == [ids[0]] and rs.engine.last_host_launches() == 1
    second = rs.advance()
    assert list(second) == [ids[1]] and rs.engine.last_host_launches() == 1
    for (z, mask, mu, _), n, y in zip(reqs, (3, 6), (first[ids[0]], second[ids[1]])):
        assert bool(torch.isfinite(y).all())
        assert _same(precision, y, dec(z, mask, mu, n))


def test_native_refusals(decoders):
    from speech_backbones_b200.binding import Engine
    dec = decoders("tf32")
    rs = dec.rolling(2, 64)
    eng = rs.engine
    z, mask, mu, _ = _request(5)                   # T_b = 64
    for args in ((2, z, mask, mu, 3), (0, z, mask, mu, 0)):
        with pytest.raises(RuntimeError):
            eng.rolling_admit(*args)
    with pytest.raises(RuntimeError):
        eng.rolling_admit(0, z, mask, mu, 3, True, None, None)          # stoc without noise
    with pytest.raises(RuntimeError):
        eng.rolling_read(0, 64)                                          # nothing finished there
    eng.rolling_admit(0, z, mask, mu, 3)
    with pytest.raises(RuntimeError):
        eng.rolling_admit(0, z, mask, mu, 3)                             # busy
    eng.reverse_diffusion(z, mask, mu, 2)                                # another call replaces the slot plan
    with pytest.raises(RuntimeError):
        eng.rolling_advance(1)
    vc = Engine(n_feats=80, dim=64, model="diffvc", dim_cond=128, precision="tf32")
    with pytest.raises(RuntimeError):
        vc.rolling_reserve(2, 64)
    vc.close()


# rel-L2 bounds of a trajectory against the reference, those of test_ragged_decoder_gpu.py
REF_TOL = {"fp32x3": 2e-4, "tf32": 8e-3, "bf16": 1e-2, "fp32": 2e-3}


@pytest.mark.parametrize("precision", MODES)
def test_reference_golden_through_the_sampler(decoders, precision):
    """The sampling cases of tests/golden/gradtts_ragged_golden.pt, each utterance a request, against the unmodified
    reference run on that utterance alone (the CPU oracle reproduces the golden bit for bit, test_ragged_decoder.py)"""
    from test_ragged_decoder import golden_inputs, load_golden, oracle_outputs, utterance_noise
    g = load_golden()
    for idx, c in enumerate(g["cases"]):
        if c["kind"] == "est":
            continue
        ref_rows = oracle_outputs(g, idx)[0]
        dec = Diffusion(80, 64, n_spks=c["n_spks"], precision=precision).eval()
        dec.load_state_dict(synthetic_state_dict(UNetConfig(n_spks=c["n_spks"]), g["seed"]))
        dec = dec.cuda()
        z, mask, mu, spk, _ = golden_inputs(g, c["n_spks"])
        rs = dec.rolling(2, g["T"])                 # fewer slots than utterances: most of them wait and reuse a slot
        ids = []
        for b, n in enumerate(g["lengths"]):
            Tb = fix_len_compatibility(n)
            noise = utterance_noise(g, b, c["N"]).cuda() if c["stoc"] else None
            ids.append(rs.submit(z[b:b + 1, :, :Tb].cuda().contiguous(), mask[b:b + 1, :, :Tb].cuda().contiguous(),
                                 mu[b:b + 1, :, :Tb].cuda().contiguous(), c["N"], c["stoc"],
                                 None if spk is None else spk[b:b + 1].cuda(), noise))
        out = rs.drain()
        for b, rid in enumerate(ids):
            err = rel_l2(out[rid][0].cpu(), ref_rows[b])
            print(precision, c.get("N"), c.get("stoc"), c["n_spks"], "utterance", b, "rel-L2", err)
            assert err <= REF_TOL[precision], (precision, c, b, err)
