"""Op isolation for the text encoder and DiffVC's mel encoder (csrc/sbk_textenc.cu) on the GPU: every captured op, per
utterance on its own tokens, against its float64 replay from the GPU's own captured inputs (tests/textenc_replay.py), then
bit-level independence of the utterances of a batch, NaN in the workspace, the sequence-length limit, and the end-to-end
outputs against the float64 oracle per utterance.

Shapes:
  * Grad-TTS's text encoder (192 channels, 2 heads of 96, kernel 3, window 4): Tx = 1 (one key; the conv halo on both
    sides), 5 and 9 (shorter than, and equal to, the 2w + 1 = 9 band), 33 (one key past a warp), and B = 8 at Tx = 221 with
    lengths 221, 1, 4, 5, 9, 130, 64, 217: mask edges at every t % 8 phase of k_te_conv's tile and inside the band.
  * The multi-speaker text encoder: 192 + 64 = 256 channels, so q|k|v fills all three 256-channel slots, d = 128.
  * A non-default accepted config: 8 heads (d = 24: lanes idle in the p.V pass), kernel 9 (a halo of 4 on an 8-token tile),
    window 15 (31 of 32 lanes build q.E_k).
  * The mel encoder at DiffVC's config with a ragged caller mask, at T = 1409 (k_te_attn above the 48 KB shared-memory
    default) and T = 6272 (the longest accepted sequence at d = 96: 200 KB); T = 6273 is refused before any launch.

Run with -s for every op's check 1 (|err| / bound) and check 2 (max / median group ratio) and one WORST line per case."""
import math

import pytest
import torch

from helpers import rel_l2
from oracle import text_encoder_oracle as T
from speech_backbones_b200.binding import _ptr
from speech_backbones_b200.text_encoder import MelEncoder, TextEncoder
from textenc_replay import R_UNIFORM, TextEncReplay

pytestmark = pytest.mark.gpu

GRADTTS = dict(n_vocab=149, n_feats=80, n_channels=192, filter_channels=768, filter_channels_dp=256, n_heads=2, n_layers=6,
               kernel_size=3, p_dropout=0.1, window_size=4)
SBK_ERR_UNSUPPORTED = 4
MAX_T = 6272                  # 8 warps x (96 + 6272 + 32) floats = 200 KB of k_te_attn shared memory
NAN = float("nan")
# End to end against the float64 oracle, per utterance: the fp32 tolerance the suite holds the whole batch to
# (test_text_encoder.TE_TOL), now for each utterance alone, on mu / the mel encoder's output (rel-L2) and on every logw
# element relative to the utterance's largest |logw|.
E2E_TOL = 2e-5


def _text_encoder(seed, spk_extra=0, n_spks=1, **over):
    a = dict(GRADTTS, **over)
    sd = T.synthetic_weights(seed, spk_extra=spk_extra, filt=a["filter_channels"], filt_dp=a["filter_channels_dp"],
                             n_layers=a["n_layers"], kernel=a["kernel_size"], window=a["window_size"], n_heads=a["n_heads"])
    m = TextEncoder(**a, spk_emb_dim=spk_extra or 64, n_spks=n_spks).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd, a


def _mel_encoder(seed):
    sd = T.mel_synthetic_weights(seed)
    m = MelEncoder(80, 192, 768, 2, 6, 3, 0.1, window_size=4).eval()
    m.load_state_dict(sd, strict=True)
    return m.cuda(), sd


def _ids(B, Tx, seed):
    return torch.randint(0, 148, (B, Tx), generator=torch.Generator().manual_seed(seed))


def _mel_inputs(lengths, Tn, seed):
    x = torch.randn(len(lengths), 80, Tn, generator=torch.Generator().manual_seed(seed))
    mask = (torch.arange(Tn)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]
    return x, mask


def _report_and_assert(tag, rp):
    rows = rp.rows
    for name, elem, unif, where in rows:
        print(f"{tag} {name:18s} |err|/bound {elem:.3e}  max/median {unif:6.2f} {where}")
    we, wu = max(rows, key=lambda r: r[1]), max(rows, key=lambda r: r[2])
    print(f"WORST {tag}: |err|/bound {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    assert not rp.nonfinite, "NaN / Inf inside an utterance: " + ", ".join(rp.nonfinite)
    bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)


# ---- every op against its float64 replay -----------------------------------------------------------------------------
TE_CASES = [("gradtts", [1]), ("gradtts", [5]), ("gradtts", [9]), ("gradtts", [33]),
            ("gradtts", [221, 1, 4, 5, 9, 130, 64, 217]), ("multispeaker", [45, 13]), ("h8-k9-w15", [70, 23, 9])]
TE_CONFIGS = {"gradtts": dict(), "multispeaker": dict(spk_extra=64, n_spks=4),
              "h8-k9-w15": dict(n_heads=8, kernel_size=9, window_size=15)}


@pytest.mark.parametrize("config,lengths", TE_CASES, ids=[f"{c}-" + "x".join(map(str, l)) for c, l in TE_CASES])
def test_text_encoder_ops_in_isolation(sbk_lib, config, lengths):
    m, sd, a = _text_encoder(21, **TE_CONFIGS[config])
    B, Tx = len(lengths), max(lengths)
    spk = torch.randn(B, 64, generator=torch.Generator().manual_seed(3)) if config == "multispeaker" else None
    rp = TextEncReplay(m.engine(), sd, a["n_heads"], a["window_size"], lengths, ids=_ids(B, Tx, Tx), spk=spk)
    rp.run()
    _report_and_assert(f"textenc {config} B={B} Tx={Tx}", rp)


MEL_CASES = [[1409, 700], [MAX_T, 3001]]


@pytest.mark.parametrize("lengths", MEL_CASES, ids=["x".join(map(str, l)) for l in MEL_CASES])
def test_mel_encoder_ops_in_isolation(sbk_lib, lengths):
    m, sd = _mel_encoder(8)
    x, mask = _mel_inputs(lengths, max(lengths), 5)
    rp = TextEncReplay(m.engine(), sd, 2, 4, lengths, mel=x, mel_mask=mask)
    rp.run()
    _report_and_assert(f"melenc B={len(lengths)} T={max(lengths)}", rp)


# ---- the capture hook ------------------------------------------------------------------------------------------------
def test_textenc_capture_is_transparent(sbk_lib):
    """Capture on changes neither the outputs (bitwise) nor the launch count, and names every tensor in launch order."""
    m, _, _ = _text_encoder(21, spk_extra=64, n_spks=4)
    eng = m.engine()
    x, L = _ids(2, 40, 1).cuda(), torch.tensor([40, 17]).cuda()
    spk = torch.randn(2, 64, generator=torch.Generator().manual_seed(2)).cuda()
    off = eng.forward(x, L, spk)
    n_off = eng.last_launch_count()
    eng.debug_capture(True)
    try:
        on = eng.forward(x, L, spk)
        n_on = eng.last_launch_count()
    finally:
        eng.debug_capture(False)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(on, off)) and n_on == n_off
    enc = [f"enc.{i}.{s}" for i in range(6) for s in ("qkv", "attn", "ln1", "ffn1", "ln2")]
    assert eng.debug_names() == ["mask", "embed", "prenet.0", "prenet.1", "prenet.2", "prenet.proj", "spk_concat", *enc,
                                 "mu", "dp.1", "dp.2", "logw"]
    assert torch.equal(eng.debug_read("mu"), on[0].cpu()) and torch.equal(eng.debug_read("logw"), on[1].cpu())
    mel, _ = _mel_encoder(8)
    me = mel.engine()
    xm, mk = _mel_inputs([50, 31], 50, 1)
    off = me.forward_mel(xm.cuda(), mk.cuda())
    n_off = me.last_launch_count()
    me.debug_capture(True)
    try:
        on = me.forward_mel(xm.cuda(), mk.cuda())
        n_on = me.last_launch_count()
    finally:
        me.debug_capture(False)
    assert torch.equal(on, off) and n_on == n_off
    assert me.debug_names() == ["init_proj", "prenet.0", "prenet.1", "prenet.2", "prenet.proj", *enc, "out"]


# ---- the sequence-length limit ---------------------------------------------------------------------------------------
def test_too_long_sequence_is_refused_before_any_launch(sbk_lib):
    """Tx = 6273 exceeds k_te_attn's 200 KB of shared memory at d = 96: both forwards return SBK_ERR_UNSUPPORTED and leave
    every output as it was (x_mask is the text encoder's first launch, the mel encoder's output its last)."""
    Tx = MAX_T + 1
    m, _, _ = _text_encoder(21)
    eng = m.engine()
    x, L = _ids(1, Tx, 0).cuda(), torch.tensor([Tx]).cuda()
    mu, logw, mask = (torch.full(s, -7.0, device="cuda") for s in ((1, 80, Tx), (1, 1, Tx), (1, 1, Tx)))
    torch.cuda.synchronize()
    rc = eng.lib.sbk_textenc_forward(eng.h, _ptr(x), _ptr(L), None, _ptr(mu), _ptr(logw), _ptr(mask), 1, Tx, eng._stream())
    torch.cuda.synchronize()
    assert rc == SBK_ERR_UNSUPPORTED, eng.lib.sbk_last_error()
    assert b"shared-memory" in eng.lib.sbk_last_error()
    for t in (mu, logw, mask):
        assert bool((t == -7.0).all()), "a refused call wrote to its outputs"
    mel, _ = _mel_encoder(8)
    me = mel.engine()
    xm, mk = torch.zeros(1, 80, Tx, device="cuda"), torch.ones(1, 1, Tx, device="cuda")
    out = torch.full((1, 80, Tx), -7.0, device="cuda")
    rc = me.lib.sbk_melenc_forward(me.h, _ptr(xm), _ptr(mk), _ptr(out), 1, Tx, me._stream())
    torch.cuda.synchronize()
    assert rc == SBK_ERR_UNSUPPORTED and bool((out == -7.0).all())


# ---- independence of the utterances of a batch -----------------------------------------------------------------------
RAGGED = [221, 1, 4, 5, 9, 130, 64, 217]


def test_text_encoder_rows_equal_their_own_calls(sbk_lib):
    """Each row of a ragged batch is bit for bit its own B = 1 call at Tx = L_b, and token ids past L_b (random, or outside
    the vocabulary) do not change a bit."""
    m, _, _ = _text_encoder(21)
    eng = m.engine()
    B, Tx = len(RAGGED), max(RAGGED)
    x, L = _ids(B, Tx, 77), torch.tensor(RAGGED)
    mu, logw, mask = (t.cpu() for t in eng.forward(x.cuda(), L.cuda()))
    for b, Lb in enumerate(RAGGED):
        m1, w1, k1 = (t.cpu() for t in eng.forward(x[b:b + 1, :Lb].contiguous().cuda(), L[b:b + 1].cuda()))
        assert torch.equal(mu[b:b + 1, :, :Lb], m1) and torch.equal(logw[b:b + 1, :, :Lb], w1), f"row {b} (L={Lb})"
        assert torch.equal(mask[b:b + 1, :, :Lb], k1)
    past = torch.arange(Tx)[None, :] >= L[:, None]
    for fill in (torch.randint(0, 149, (B, Tx), generator=torch.Generator().manual_seed(5)),
                 torch.where(torch.arange(Tx)[None, :] % 2 == 0, 10 ** 9, -3).expand(B, Tx)):
        x2 = torch.where(past, fill, x)
        out = [t.cpu() for t in eng.forward(x2.cuda(), L.cuda())]
        assert all(torch.equal(a, b) for a, b in zip(out, (mu, logw, mask))), "ids past L_b changed the output"


def _not_nan(eng, names, skip=()):
    left = []
    for n in names:
        v = eng.debug_read(n)
        if n not in skip and not bool(torch.isnan(v).all()):
            left.append(f"{n} ({int((~torch.isnan(v)).sum())} of {v.numel()} not NaN)")
    return left


@pytest.mark.parametrize("kind", ["text", "mel"])
def test_nan_workspace_changes_nothing(sbk_lib, kind):
    """A larger call on NaN weights (emb.weight / init_proj.weight) leaves NaN in every captured tensor that no ReLU
    writes; after the real weights are reloaded (the workspace survives a reload) a smaller call gives the bits of a fresh
    handle.  The ReLU outputs (prenet.i, enc.i.ffn1, and the duration predictor behind its ReLU) hold 0 instead: fmaxf(NaN,
    0) is 0, so the kernels' ReLU stops a NaN where torch.relu passes it on."""
    if kind == "text":
        m, sd, _ = _text_encoder(21)
        fresh, _, _ = _text_encoder(21)
        key = "emb.weight"
        big = (_ids(3, 300, 1), torch.tensor([300, 200, 17]))
        small = (_ids(2, 150, 2), torch.tensor([150, 61]))
        run = lambda e, a: [t.cpu() for t in e.forward(a[0].cuda(), a[1].cuda())]
    else:
        m, sd = _mel_encoder(8)
        fresh, _ = _mel_encoder(8)
        key = "init_proj.weight"
        big = _mel_inputs([300, 200, 17], 300, 1)
        small = _mel_inputs([150, 61], 150, 2)
        run = lambda e, a: [e.forward_mel(a[0].cuda(), a[1].cuda()).cpu()]
    eng = m.engine()
    bad = dict(sd)
    bad[key] = torch.full_like(sd[key], NAN)
    eng.load_state_dict(bad)
    eng.debug_capture(True)
    try:
        run(eng, big)
        torch.cuda.synchronize()
        relu = ("mask", "prenet.0", "prenet.1", "prenet.2", "dp.1", "dp.2", "logw") + tuple(f"enc.{i}.ffn1" for i in range(6))
        left = _not_nan(eng, eng.debug_names(), skip=relu)
    finally:
        eng.debug_capture(False)
    assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
    eng.load_state_dict(sd)
    got, want = run(eng, small), run(fresh.engine(), small)
    assert all(torch.equal(a, b) for a, b in zip(got, want)), "NaN left in the workspace reached a later call"


# ---- end to end against float64, per utterance -----------------------------------------------------------------------
def _sd64(sd):
    return {k: v.double().cuda() for k, v in sd.items()}


def test_text_encoder_vs_float64_per_utterance(sbk_lib):
    """mu within E2E_TOL rel-L2 of the float64 oracle for every utterance alone, every logw element within E2E_TOL of the
    utterance's largest |logw|, and the durations ceil(exp(logw)) equal to float64's wherever float64's exp(logw) is
    farther than that bound from an integer."""
    m, sd, _ = _text_encoder(21)
    B, Tx = len(RAGGED), max(RAGGED)
    x, L = _ids(B, Tx, 91), torch.tensor(RAGGED)
    mu, logw, _ = (t.double() for t in m.engine().forward(x.cuda(), L.cuda()))
    with torch.no_grad():
        mu64, logw64, _ = T.text_encoder(_sd64(sd), x.cuda(), L.cuda())
    for b, Lb in enumerate(RAGGED):
        e_mu = rel_l2(mu[b, :, :Lb], mu64[b, :, :Lb])
        lw, lw64 = logw[b, 0, :Lb], logw64[b, 0, :Lb]
        tol = E2E_TOL * max(1.0, lw64.abs().max().item())
        e_w = (lw - lw64).abs().max().item()
        w64 = lw64.exp()
        clear = (w64 - w64.round()).abs() > w64 * math.expm1(tol)
        same = torch.equal(torch.ceil(lw.exp())[clear], torch.ceil(w64)[clear])
        print(f"textenc e2e b={b} L={Lb}: mu rel-L2 {e_mu:.2e}  logw max|err| {e_w:.2e} (bound {tol:.2e})  "
              f"durations compared at {int(clear.sum())} of {Lb} tokens")
        assert e_mu <= E2E_TOL and e_w <= tol and same, (b, e_mu, e_w)


def test_mel_encoder_vs_float64_per_utterance(sbk_lib):
    m, sd = _mel_encoder(8)
    lengths = [1409, 700, 33]
    x, mask = _mel_inputs(lengths, max(lengths), 12)
    y = m(x.cuda(), mask.cuda()).double()
    with torch.no_grad():
        y64 = T.mel_encoder(_sd64(sd), x.double().cuda(), mask.double().cuda())
    for b, Lb in enumerate(lengths):
        e = rel_l2(y[b, :, :Lb], y64[b, :, :Lb])
        print(f"melenc e2e b={b} L={Lb}: rel-L2 {e:.2e}")
        assert e <= E2E_TOL, (b, e)
