"""Ragged Grad-TTS batches on the GPU: `lengths=` in `Engine.estimator / reverse_diffusion / reverse_steps` and in the
drop-in `Diffusion`.

The reference synthesizes one utterance per call (Grad-TTS/inference.py:72-81: B = 1 at T = fix_len_compatibility(y_len)).
With `lengths`, each row of a padded batch is that call: out[b, :, :T_b] equals the engine's own B = 1 call on the [:T_b]
slices of its inputs (T_b = fix_len_compatibility(lengths[b])), and out[b, :, T_b:] is 0.  tf32 and bf16 rows are bit for
bit their single calls; fp32x3 and fp32 rows agree with them to fp32 rounding (rel-L2 < 1e-6, the bound of the existing
batch-independence tests: fp32x3 picks its N-tile width from the tile count, which moves fp32 rounding points).

B = 5, T = 512, lengths {512, 301, 260, 130, 1}: T_b = 512, 304, 260, 132, 4 - level-0 tile tails, a level-1 width of 130
(crossing a 128-pixel tile), odd level-2 widths 65 and 33, and a level-2 width of 1.  The padded frames of z and mu hold
random values, not zeros, so any read of them into a valid frame would show."""
import pytest
import torch

from helpers import rel_l2
from op_replay import Replay
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_noise, synthetic_state_dict
from speech_backbones_b200.gradtts import fix_len_compatibility

pytestmark = pytest.mark.gpu

MODES = ("fp32x3", "tf32", "bf16", "fp32")
B, T = 5, 512
LENGTHS = [512, 301, 260, 130, 1]
TB = [fix_len_compatibility(n) for n in LENGTHS]


@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache = {}

    def get(precision, n_spks=1):
        if (precision, n_spks) not in cache:
            e = Engine(n_spks=n_spks, precision=precision)
            e.load_state_dict(synthetic_state_dict(UNetConfig(n_spks=n_spks)))
            cache[(precision, n_spks)] = e
        return cache[(precision, n_spks)]
    yield get
    for e in cache.values():
        e.close()


def _inputs(lengths=LENGTHS, n_spks=1):
    z, _, mu, spk, _ = synthetic_inputs(B, T, n_spks=n_spks)
    L = torch.tensor(lengths, dtype=torch.int64)
    mask = (torch.arange(T)[None, :] < L[:, None]).to(torch.float32)[:, None, :]
    return z.cuda(), mask.cuda(), mu.cuda(), None if spk is None else spk.cuda(), L.cuda()


def _same(precision, got, want):
    if precision in ("tf32", "bf16"):
        return torch.equal(got, want)
    return rel_l2(got, want) < 1e-6


def _check_rows(precision, out, single, lengths=LENGTHS):
    """single(b, Tb) -> the engine's B = 1 call on utterance b at T_b frames"""
    out = out.cpu()
    for b, n in enumerate(lengths):
        Tb = fix_len_compatibility(n)
        one = single(b, Tb).cpu()
        assert _same(precision, out[b:b + 1, :, :Tb], one), (precision, b, Tb, rel_l2(out[b:b + 1, :, :Tb], one))
        assert torch.count_nonzero(out[b, :, Tb:]) == 0, (precision, b)


def _sl(x, b, Tb):
    return x[b:b + 1, ..., :Tb].contiguous()


@pytest.mark.parametrize("precision", MODES)
def test_rows_equal_single_utterance_calls(engines, precision):
    eng = engines(precision)
    z, mask, mu, _, L = _inputs()
    t = torch.tensor([0.9, 0.5, 0.3, 0.7, 0.1], device="cuda")
    xt = z * mask
    est = eng.estimator(xt, mask, mu, t, lengths=L)
    _check_rows(precision, est, lambda b, Tb: eng.estimator(_sl(xt, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), t[b:b + 1]))
    traj = eng.reverse_diffusion(z, mask, mu, 10, lengths=L)
    _check_rows(precision, traj, lambda b, Tb: eng.reverse_diffusion(_sl(z, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), 10))
    noise = synthetic_noise(5, B, T).cuda()
    stoc = eng.reverse_diffusion(z, mask, mu, 5, True, None, noise, lengths=L)
    _check_rows(precision, stoc, lambda b, Tb: eng.reverse_diffusion(_sl(z, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), 5, True,
                                                                     None, noise[:, b:b + 1, :, :Tb].contiguous()))


@pytest.mark.parametrize("precision", MODES)
def test_full_lengths_equal_the_dense_call(engines, precision):
    eng = engines(precision)
    z, _, mu, _, _ = _inputs()
    mask = torch.ones(B, 1, T, device="cuda")
    L = torch.full((B,), T, dtype=torch.int64, device="cuda")
    t = torch.linspace(0.9, 0.1, B, device="cuda")
    assert torch.equal(eng.estimator(z, mask, mu, t, lengths=L), eng.estimator(z, mask, mu, t))
    assert torch.equal(eng.reverse_diffusion(z, mask, mu, 4, lengths=L), eng.reverse_diffusion(z, mask, mu, 4))


@pytest.mark.parametrize("precision", MODES)
def test_graph_replay_with_new_lengths(engines, precision):
    """Two ragged loops in a row at the same (B, T, N) replay the same graph: the second reads its own lengths (the plan's
    copy), and each loop is one host launch."""
    eng = engines(precision)
    for lengths in ([130, 512, 1, 301, 260], [4, 64, 500, 129, 256]):
        z, mask, mu, _, L = _inputs(lengths)
        out = eng.reverse_diffusion(z, mask, mu, 6, lengths=L)
        assert eng.last_host_launches() == 1
        _check_rows(precision, out, lambda b, Tb: eng.reverse_diffusion(_sl(z, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), 6),
                    lengths)


@pytest.mark.parametrize("precision", MODES)
def test_drop_in_module(engines, precision):
    from speech_backbones_b200.gradtts import Diffusion
    dec = Diffusion(80, 64, precision=precision).eval()
    dec.load_state_dict(synthetic_state_dict(UNetConfig()))
    dec = dec.cuda()
    z, mask, mu, _, L = _inputs()
    y = dec(z, mask, mu, 6, lengths=L)
    assert torch.equal(y, dec.engine().reverse_diffusion(z, mask, mu, 6, lengths=L))
    torch.manual_seed(7)
    one = dec(z, mask, mu, 6, stoc=True, lengths=L)
    dec.noise_window_bytes = z.numel() * 4 * 2          # windows of 2 steps through reverse_steps
    torch.manual_seed(7)
    win = dec(z, mask, mu, 6, stoc=True, lengths=L)
    assert _same(precision, win, one), rel_l2(win, one)
    for b, Tb in enumerate(TB):
        assert torch.count_nonzero(win[b, :, Tb:]) == 0


def test_oversize_batch_with_lengths(engines):
    eng = engines("tf32")
    z, mask, mu, _, L = _inputs()
    full = eng.reverse_diffusion(z, mask, mu, 3, lengths=L)
    eng.max_workspace_bytes = eng.workspace_bytes(2, T, 3)
    try:
        assert len(eng.batch_slices(B, T, 3)) > 1
        sliced = eng.reverse_diffusion(z, mask, mu, 3, lengths=L)
    finally:
        eng.max_workspace_bytes = None
    assert torch.equal(sliced, full)


@pytest.mark.parametrize("precision", MODES)
def test_multi_speaker_rows(engines, precision):
    eng = engines(precision, n_spks=4)
    z, mask, mu, spk, L = _inputs(n_spks=4)
    t = torch.tensor([0.9, 0.5, 0.3, 0.7, 0.1], device="cuda")
    xt = z * mask
    est = eng.estimator(xt, mask, mu, t, spk, lengths=L)
    _check_rows(precision, est, lambda b, Tb: eng.estimator(_sl(xt, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), t[b:b + 1],
                                                            spk[b:b + 1].contiguous()))


def test_bad_lengths_raise_before_any_launch(engines):
    from speech_backbones_b200.gradtts import Diffusion
    eng = engines("tf32")
    z, mask, mu, _, L = _inputs()
    t = torch.full((B,), 0.5, device="cuda")
    bad = {"int32": L.to(torch.int32), "shape": L[:4], "cpu": L.cpu(), "zero": torch.where(L == 1, 0, L),
           "over": torch.where(L == 512, 513, L)}
    dec = Diffusion(80, 64, precision="tf32").eval()
    dec.load_state_dict(synthetic_state_dict(UNetConfig()))
    dec = dec.cuda()
    for name, lengths in bad.items():
        n0 = eng.last_launch_count()
        with pytest.raises(ValueError):
            eng.estimator(z, mask, mu, t, lengths=lengths)
        with pytest.raises(ValueError):
            eng.reverse_diffusion(z, mask, mu, 2, lengths=lengths)
        with pytest.raises(ValueError):
            eng.reverse_steps(z.clone(), mask, mu, 2, 0, 2, lengths=lengths)
        with pytest.raises(ValueError):
            dec(z, mask, mu, 2, stoc=True, lengths=lengths)
        assert eng.last_launch_count() == n0, name


def test_synthesize_from_encoder_ragged(engines):
    from speech_backbones_b200 import gradtts as G
    from speech_backbones_b200.spec import synthetic_encoder_outputs
    dec = G.Diffusion(80, 64, precision="tf32").eval()
    dec.load_state_dict(synthetic_state_dict(UNetConfig()))
    dec = dec.cuda()
    mu_x, logw, x_mask = [v.cuda() for v in synthetic_encoder_outputs(3, 40, [40, 17, 3], 1.2, seed=5)]
    w_ceil = torch.ceil(torch.exp(logw) * x_mask)
    y_lengths = torch.clamp_min(torch.sum(w_ceil, [1, 2]), 1).long()
    Ty = fix_len_compatibility(int(y_lengths.max()))
    noise_tf = torch.randn(3, Ty, 80, generator=torch.Generator().manual_seed(3)).cuda()
    mu_y, y, _ = G.synthesize_from_encoder(dec, mu_x, logw, x_mask, 5, 1.5, noise_tf=noise_tf, ragged=True)
    for b in range(3):
        n = int(y_lengths[b])
        _, y1, _ = G.synthesize_from_encoder(dec, mu_x[b:b + 1, :, :int(x_mask[b].sum())].contiguous(),
                                             logw[b:b + 1, :, :int(x_mask[b].sum())].contiguous(),
                                             x_mask[b:b + 1, :, :int(x_mask[b].sum())].contiguous(), 5, 1.5,
                                             noise_tf=noise_tf[b:b + 1, :fix_len_compatibility(n)].contiguous())
        assert torch.equal(y[b:b + 1, :, :n], y1[:, :, :n]), b


# rel-L2 bounds against the reference, those of the existing parity tests: (per estimator call, trajectory)
REF_TOL = {"fp32x3": (1e-5, 2e-4), "tf32": (4e-3, 8e-3), "bf16": (2e-2, 1e-2), "fp32": (1e-4, 2e-3)}


@pytest.fixture(scope="module")
def ref_golden():
    """(golden, [oracle outputs per case]), the oracle run once for every mode"""
    from test_ragged_decoder import load_golden, oracle_outputs
    g = load_golden()
    return g, [oracle_outputs(g, i) for i in range(len(g["cases"]))]


@pytest.mark.parametrize("precision", MODES)
def test_rows_match_the_reference_golden(engines, ref_golden, precision):
    """Each ragged row against the unmodified reference run on that utterance alone: tests/golden/gradtts_ragged_golden.pt
    pins the reference's outputs by digest, and the CPU oracle reproduces them bit for bit (test_ragged_decoder.py), so
    the rows are compared with the oracle's outputs."""
    from test_ragged_decoder import batch_noise, golden_inputs
    g = ref_golden[0]
    for idx, c in enumerate(g["cases"]):
        ref_rows = ref_golden[1][idx][0]
        eng = engines(precision, c["n_spks"])
        z, mask, mu, spk, L = [None if v is None else v.cuda() for v in golden_inputs(g, c["n_spks"])]
        if c["kind"] == "est":
            y = eng.estimator(z * mask, mask, mu, torch.tensor(g["t"], device="cuda"), spk, lengths=L).cpu()
            tol = REF_TOL[precision][0]
        else:
            noise = batch_noise(g, c["N"]).cuda() if c["stoc"] else None
            y = eng.reverse_diffusion(z, mask, mu, c["N"], c["stoc"], spk, noise, lengths=L).cpu()
            tol = REF_TOL[precision][1]
        for b, n in enumerate(g["lengths"]):
            Tb = fix_len_compatibility(n)
            err = rel_l2(y[b, :, :Tb], ref_rows[b])
            print(precision, c["kind"], c.get("N"), c.get("stoc"), c["n_spks"], "utterance", b, "rel-L2", err)
            assert err <= tol, (precision, c, b, err)
            assert torch.count_nonzero(y[b, :, Tb:]) == 0


# ---- a batch at the tile edges, with NaN wherever the call must not read ----------------------------------------------------
# B = 9, T = 516 (test_op_isolation_gpu.py's first ragged case): T_b = 4, 516, 128, 132, 256, 260, 508, 388, 4 - the dense
# grid ends in a partial tile at every level, edges on, past and short of tile seams, 4-frame utterances first and last.
NB, NT = 9, 516
NLENGTHS = [1, 516, 128, 129, 253, 257, 505, 385, 2]
NTB = [fix_len_compatibility(n) for n in NLENGTHS]


def _nan_past_edges(v, lengths=NLENGTHS):
    """v [..., B, C, T] with NaN at every frame >= T_b of row b"""
    TB = torch.tensor([fix_len_compatibility(n) for n in lengths], device=v.device)
    past = torch.arange(v.shape[-1], device=v.device)[None, :] >= TB[:, None]
    return torch.where(past[:, None], float("nan"), v)


def _nan_inputs():
    """(z, mask, mu, L): mask 1 below lengths[b], 0 on [lengths[b], T_b); z, mask and mu NaN from T_b on"""
    z, _, mu, _, _ = synthetic_inputs(NB, NT)
    L = torch.tensor(NLENGTHS, dtype=torch.int64)
    mask = (torch.arange(NT)[None, :] < L[:, None]).to(torch.float32)[:, None, :]
    return (_nan_past_edges(z).cuda(), _nan_past_edges(mask).cuda(), _nan_past_edges(mu).cuda(), L.cuda())


@pytest.mark.parametrize("precision", ("tf32", "bf16"))
def test_every_captured_op_equals_the_single_call(engines, precision):
    """The ops of a ragged call, each cropped to utterance b's widths (T_b >> level), equal the captures of the engine's own
    B = 1 call on [:T_b] bit for bit: a divergence is placed at the first op where it appears, not in the final mel."""
    eng = engines(precision)
    sd = synthetic_state_dict(UNetConfig())
    z, mask, mu, L = _nan_inputs()
    t = torch.linspace(0.9, 0.1, NB)
    x = z * mask
    rp = Replay(eng, sd, precision, "gradtts", x, mask, mu, t, lengths=NLENGTHS).hold()
    judged = rp.judged_names()
    for b, Tb in enumerate(NTB):
        one = Replay(eng, sd, precision, "gradtts", _sl(x, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), t[b:b + 1])
        assert one.names == rp.names, b
        rp.select((b, Tb))
        for n in judged:
            got, want = rp.capture(n), one.capture(n)
            assert got.shape == want.shape, (n, b, tuple(got.shape), tuple(want.shape))
            assert torch.equal(got, want), f"{n}{rp.tag}: differs from the B = 1 call, max |diff| " \
                                           f"{(got - want).abs().nan_to_num(float('inf')).max().item():.3g}"
        assert torch.equal(rp.y, one.y), b


@pytest.mark.parametrize("stoc", [False, True], ids=["det", "stoc"])
@pytest.mark.parametrize("precision", MODES)
def test_poisoned_loop_rows_equal_single_calls(engines, precision, stoc):
    """reverse_diffusion (N = 3) on a batch whose inputs - and, stochastic, noise - are NaN past every T_b, right after a
    dense NaN loop of the same kind at the same (B, T, N) has left NaN in the plan's buffers and in the graph's.  Every row
    is finite and equals its single call, and is 0 past T_b."""
    eng = engines(precision)
    z, mask, mu, L = _nan_inputs()
    noise = _nan_past_edges(synthetic_noise(3, NB, NT)).cuda() if stoc else None
    # the single calls first: each builds a plan of its own shape, which would replace the poisoned one
    single = [eng.reverse_diffusion(_sl(z, b, Tb), _sl(mask, b, Tb), _sl(mu, b, Tb), 3, stoc, None,
                                    noise[:, b:b + 1, :, :Tb].contiguous() if stoc else None).cpu()
              for b, Tb in enumerate(NTB)]
    nan = torch.full_like(z, float("nan"))
    dense = eng.reverse_diffusion(nan, torch.ones_like(mask), nan, 3, stoc, None, torch.full_like(noise, float("nan"))
                                  if stoc else None)
    assert bool(torch.isnan(dense).all())
    out = eng.reverse_diffusion(z, mask, mu, 3, stoc, None, noise, lengths=L).cpu()
    for b, Tb in enumerate(NTB):
        row = out[b:b + 1, :, :Tb]
        assert bool(torch.isfinite(row).all()), (precision, b, Tb)
        assert _same(precision, row, single[b]), (precision, b, Tb, rel_l2(row, single[b]))
        assert torch.count_nonzero(out[b, :, Tb:]) == 0, (precision, b)
