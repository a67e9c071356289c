"""Op isolation for ragged DiffVC batches on the GPU: every op of the score U-Net (`vc_estimator(..., lengths=)`), the
RefBlock conditioning branch (`vc_conditioning(..., ref_lengths=)`) and the PostNet (`forward(..., lengths=)`), per
utterance, on that utterance's own frames against its float64 replay from the GPU's own captured inputs (tests/op_replay.py
Replay, RefBlockReplay, PostNetReplay).

Every ragged call here follows a dense call at the same shape on all-NaN inputs, which leaves NaN in every workspace buffer
a capture sees (asserted), and its inputs AND mask are NaN past each utterance's edge: T'_b = fix_len_compatibility(L_b)
for the U-Net, R_b for the RefBlock, L_b for the PostNet.  A ragged kernel must read nothing at or past an edge, so a load
where a zero fill belongs, a statistic that runs one column long, or a mask applied by multiplication (NaN * 0 = NaN)
instead of by selection puts a NaN or a wrong value into the utterance's own frames, which check 1 (|err| <= kappa A) and
check 2 (max / median group ratio <= R_UNIFORM) then see.  Outputs the API defines past an edge must be exactly 0.

Shapes:
  * U-Net: B = 6, T = 516, lengths {1, 516, 128, 129, 257, 509} (T'_b = 4, 516, 128, 132, 260, 512): edges on the 128-pixel
    seam at every level, 4 columns past a seam, a 4-frame utterance first, a full-length row ending in a partial tile; in all
    four modes with the 3x3 layout pinned to one- and two-row tiles (the fp32 mode runs no wgmma 3x3 conv).
  * RefBlock: Tr = 300, R = {300, 257, 256, 129, 128, 1} (either side of k_first_conv's 256 seam and the wgmma 128 seam, a
    one-frame reference), the same at log-mel level (-5, where InstanceNorm's E[x^2] - E[x]^2 cancels), and dim_spk = 256
    at Tr = 257, R = {257, 129, 3}; N = 1 and 4, all four handle precisions.
  * PostNet: test_vc_ragged_gpu.PN_CASES, lengths 2 and 6 (shorter than the 7x7 halo on both sides: the three zero columns
    cover the whole image), and dense calls (all-ones and 0/1 masks); all four handle precisions.

Run with -s for every op's check 1 and check 2 and one WORST line per utterance and per call."""
import pytest
import torch

from helpers import rel_l2
from op_replay import R_UNIFORM, PostNetReplay, RefBlockReplay, Replay
from speech_backbones_b200.diffvc import fix_len_compatibility
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_postnet_state_dict, synthetic_state_dict
from test_conv_rows_gpu import conv3_rows_of
from test_diffvc_gpu import COND_TOL
from test_refblock_isolation_gpu import LOG_MEL_SHIFT, oracle_table
from test_vc_ragged_gpu import PN_CASES

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32x3", "tf32", "bf16", "fp32"]
SEED = 4421
NAN = float("nan")


def _worst(tag, rows):
    we, wu = max(rows, key=lambda r: r[1]), max(rows, key=lambda r: r[2])
    print(f"WORST {tag}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")


def _report_and_assert(tag, rows, nonfinite):
    for name, elem, unif, where in rows:
        print(f"{tag} {name:44s} |err|/(kA) {elem:.3e}  max/median {unif:6.2f} {where}")
    utts = {}
    for r in rows:
        if " b=" in r[0]:
            utts.setdefault(r[0][r[0].index(" b="):], []).append(r)
    for utt, urows in utts.items():
        _worst(tag + utt, urows)
    _worst(tag, rows)
    assert not nonfinite, "NaN / Inf inside an utterance: " + ", ".join(nonfinite)
    bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)


def _not_nan(read, names, skip=()):
    """names whose capture (read(name); None: the op keeps no copy) is not all NaN"""
    left = []
    for n in names:
        v = read(n)
        if v is not None and n not in skip and not bool(torch.isnan(v).all()):
            left.append(f"{n} ({int((~torch.isnan(v)).sum())} of {v.numel()} not NaN)")
    return left


def _ragged_mask(lengths, edges, T):
    """[B, 1, T]: 1 below L_b, 0 from L_b to the edge, NaN at and past the edge"""
    f = torch.arange(T)[None, :]
    L, E = torch.tensor(lengths)[:, None], torch.tensor(edges)[:, None]
    return torch.where(f >= E, NAN, (f < L).float())[:, None]


def _past(x, edges):
    """x with every frame at or past edges[b] set to NaN (a copy)"""
    x = x.clone()
    for b, e in enumerate(edges):
        x[b, ..., e:] = NAN
    return x


# ---- the score U-Net ---------------------------------------------------------------------------------------------------
UNET_CASES = [(516, [1, 516, 128, 129, 257, 509])]
UNET_RUNS = [(p, l) for p in PRECISIONS for l in (("rows1", "rows2") if p != "fp32" else ("rows1",))]


@pytest.fixture(scope="module")
def vc_engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cfg = DiffVCConfig()
    sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    cache = {}

    def get(precision, layout):
        # one handle per 3x3 tile layout: a plan keeps the layout it was built with
        if (precision, layout) not in cache:
            e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision)
            e.load_state_dict(sd)
            cache[precision, layout] = e
        return cache[precision, layout], cfg, sd
    yield get
    for e in cache.values():
        e.close()


def _poison_unet(eng, B, T, cond, t):
    """A dense vc_estimator call at (B, T) on x = mean = NaN (mask all ones), capture on: every buffer a captured op writes
    in this plan's workspace then holds NaN.  Returns the names whose capture is not all NaN (there should be none)."""
    nan = torch.full((B, 80, T), NAN, device="cuda")
    eng.debug_capture(True)
    try:
        eng.vc_estimator(nan, torch.ones(B, 1, T, device="cuda"), nan, cond.cuda(), t.cuda())
        torch.cuda.synchronize()
        return _not_nan(eng.debug_read, eng.debug_names())
    finally:
        eng.debug_capture(False)


def _vc_inputs(B, T, dc, seed):
    g = torch.Generator().manual_seed(seed)
    mean = torch.randn(B, 80, T, generator=g)
    z = mean + torch.randn(B, 80, T, generator=g)
    cond = torch.randn(B, dc, generator=g) * 0.5
    return z, mean, cond


@pytest.mark.parametrize("precision,layout", UNET_RUNS, ids=[f"{p}-{l}" for p, l in UNET_RUNS])
@pytest.mark.parametrize("T,lengths", UNET_CASES, ids=[f"B{len(l)}-T{t}" for t, l in UNET_CASES])
def test_vc_unet_ragged_ops_in_isolation(vc_engines, monkeypatch, precision, layout, T, lengths):
    monkeypatch.setenv("SBK_CONV3_ROWS", layout[-1])
    eng, cfg, sd = vc_engines(precision, layout)
    B = len(lengths)
    z, mean, cond = _vc_inputs(B, T, cfg.dim_spk, SEED + T)
    t = torch.linspace(0.9, 0.2, B)
    tp = [fix_len_compatibility(n) for n in lengths]
    mask = _ragged_mask(lengths, tp, T)
    x, mu = _past(z * mask, tp), _past(mean, tp)
    L = torch.tensor(lengths).cuda()
    args = [v.cuda() for v in (x, mask, mu, cond, t)]
    rows3 = conv3_rows_of(lambda: eng.vc_estimator(*args, lengths=L))
    assert rows3 == (set() if precision == "fp32" else {int(layout[-1])}), f"3x3 tile rows launched: {rows3}"
    left = _poison_unet(eng, B, T, cond, t)
    assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
    rp = Replay(eng, sd, precision, "diffvc", x, mask, mu, t, cond=cond, dim=cfg.dim_unet, lengths=lengths)
    rows = rp.run()
    for b, Tb in enumerate(tp):
        assert torch.count_nonzero(rp.full["y"][b, :, Tb:]) == 0, f"utterance {b}: output not 0 past T'_b = {Tb}"
    _report_and_assert(f"diffvc ragged {precision} {layout} B={B} T={T}", rows, rp.nonfinite)


@pytest.mark.parametrize("mode", ["pf", "ml"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_vc_reverse_diffusion_rows_after_nan_workspace(vc_engines, monkeypatch, precision, mode):
    """vc_reverse_diffusion(..., lengths=) at N = 3 right after a dense loop at the same (B, T, N) on NaN inputs: each row
    equals its own B = 1 call - bit for bit in tf32 / bf16, rel-L2 <= 1e-6 in fp32x3 / fp32 (test_vc_ragged_gpu._same, one-row
    3x3 tiles pinned) - and is exactly 0 past T'_b; z, mean, noise and mask are NaN there."""
    monkeypatch.setenv("SBK_CONV3_ROWS", "1")
    eng, cfg, _ = vc_engines(precision, "rows1")
    T, lengths, N = 160, [160, 131, 61, 1], 3
    B = len(lengths)
    z, mean, _ = _vc_inputs(B, T, cfg.dim_spk, SEED + 7)
    cond = torch.randn(N, B, cfg.dim_spk, generator=torch.Generator().manual_seed(SEED)) * 0.5
    noise = None if mode == "pf" else torch.randn(N, B, 80, T, generator=torch.Generator().manual_seed(SEED + 1))
    nan = torch.full((B, 80, T), NAN, device="cuda")
    eng.vc_reverse_diffusion(nan, torch.ones(B, 1, T, device="cuda"), nan, cond.cuda(), N, mode,
                             None if noise is None else torch.full_like(noise, NAN).cuda())
    torch.cuda.synchronize()
    tp = [fix_len_compatibility(n) for n in lengths]
    mask = _ragged_mask(lengths, tp, T)
    y = eng.vc_reverse_diffusion(_past(z, tp).cuda(), mask.cuda(), _past(mean, tp).cuda(), cond.cuda(), N, mode,
                                 None if noise is None else _past(noise.transpose(0, 1), tp).transpose(0, 1).cuda(),
                                 lengths=torch.tensor(lengths).cuda()).cpu()
    for b, Tb in enumerate(tp):
        one = eng.vc_reverse_diffusion(z[b:b + 1, :, :Tb].contiguous().cuda(), mask[b:b + 1, :, :Tb].contiguous().cuda(),
                                       mean[b:b + 1, :, :Tb].contiguous().cuda(), cond[:, b:b + 1].contiguous().cuda(), N,
                                       mode, None if noise is None else noise[:, b:b + 1, :, :Tb].contiguous().cuda()).cpu()
        got = y[b:b + 1, :, :Tb]
        err = rel_l2(got, one)
        print(f"vc_reverse_diffusion after NaN {precision} {mode} row {b} (T'={Tb}): rel-L2 vs own call {err:.2e}")
        if precision in ("tf32", "bf16"):
            assert torch.equal(got, one), f"row {b}: max |diff| {(got - one).abs().max().item():.3e}"
        else:
            assert err <= 1e-6, f"row {b}: rel-L2 {err:.3e}"
        assert torch.count_nonzero(y[b, :, Tb:]) == 0


# ---- the RefBlock conditioning branch ----------------------------------------------------------------------------------
RB_CONFIGS = {"spk128": DiffVCConfig(), "spk256": DiffVCConfig(dim_spk=256)}
RB_CASES = [("spk128", 300, [300, 257, 256, 129, 128, 1], 0.0), ("spk128", 300, [300, 257, 256, 129, 128, 1], LOG_MEL_SHIFT),
            ("spk256", 257, [257, 129, 3], 0.0)]
RB_IDS = [f"{c}-Tr{t}-" + "x".join(map(str, l)) + ("-logmel" if s else "") for c, t, l, s in RB_CASES]


@pytest.fixture(scope="module")
def rb_engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache, sds = {}, {}

    def get(config, precision):
        cfg = RB_CONFIGS[config]
        if config not in sds:
            sds[config] = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
        if (config, precision) not in cache:
            e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision)
            e.load_state_dict(sds[config])
            cache[config, precision] = e
        return cache[config, precision], cfg, sds[config]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("N", [1, 4])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("config,Tr,ref_lengths,shift", RB_CASES, ids=RB_IDS)
def test_refblock_ragged_ops_in_isolation(rb_engines, config, Tr, ref_lengths, shift, precision, N):
    """Every op of the last step of vc_conditioning(..., ref_lengths=) per reference on its own R_b frames, after a dense
    NaN call at the same (B, Tr, N); ref, mean_ref and the mask NaN past R_b.  Each reference's cond rows also equal its own
    B = 1 call bit for bit, and meet COND_TOL against the float64 oracle on ref[b:b+1, :, :R_b]."""
    eng, cfg, sd = rb_engines(config, precision)
    B = len(ref_lengths)
    gen = torch.Generator().manual_seed(7919 * Tr + B)
    ref = torch.randn(B, 80, Tr, generator=gen) + shift
    mean_ref = torch.randn(B, 80, Tr, generator=gen) + shift
    c = torch.randn(B, 256, generator=gen)
    c = c / c.norm(dim=1, keepdim=True)
    nan = torch.full((B, 80, Tr), NAN, device="cuda")
    eng.debug_capture(True)
    try:
        eng.vc_conditioning(nan, torch.ones(B, 1, Tr, device="cuda"), nan, c.cuda(), N)
        torch.cuda.synchronize()
        # tb depends on t alone: it is the step's time-bias row, not a function of the reference
        left = _not_nan(eng.vc_cond_debug_read, eng.vc_cond_debug_names(), skip=("ref_block.tb",))
    finally:
        eng.debug_capture(False)
    assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
    rmask = _ragged_mask(ref_lengths, ref_lengths, Tr)
    rp = RefBlockReplay(eng, sd, precision, cfg, _past(ref, ref_lengths), rmask, _past(mean_ref, ref_lengths), c, N,
                        ref_lengths=ref_lengths)
    tag = f"refblock ragged {config} Tr={Tr}{' logmel' if shift else ''} {precision} N={N}"
    rows = rp.run()
    print(f"{tag} InstanceNorm variance rel. error: " + ", ".join(f"{b} {v:.2e}" for b, v in rp.var_err.items()))
    _report_and_assert(tag, rows, rp.nonfinite)
    table = rp.table.cpu()
    for b, R in enumerate(ref_lengths):
        one_args = (ref[b:b + 1, :, :R].contiguous(), torch.ones(1, 1, R), mean_ref[b:b + 1, :, :R].contiguous(), c[b:b + 1])
        one = eng.vc_conditioning(*(v.cuda() for v in one_args), N).cpu()
        assert torch.equal(table[:, b:b + 1], one), f"reference {b} (R={R}): not its own call bit for bit"
        want = oracle_table(sd, cfg, *one_args, N)
        errs = [rel_l2(rp.table[i, b:b + 1], want[i]) for i in range(N)]
        print(f"{tag} b={b} R={R} cond rel-L2 vs float64 oracle per step: " + ", ".join(f"{e:.2e}" for e in errs))
        assert max(errs) <= COND_TOL[precision], (b, errs)


# ---- the PostNet -------------------------------------------------------------------------------------------------------
PN_RAGGED = PN_CASES + [(64, [64, 6, 2])]
PN_DENSE = [(160, [160, 160]), (263, [263, 129, 1])]       # (T, mask lengths): all-ones, then a 0/1 mask


@pytest.fixture(scope="module")
def postnets(sbk_lib):
    from speech_backbones_b200.postnet import PostNetEngine
    sd = synthetic_postnet_state_dict(128, SEED)
    cache = {}

    def get(precision):
        if precision not in cache:
            e = PostNetEngine(128, precision=precision)
            e.load_state_dict(sd)
            cache[precision] = e
        return cache[precision], sd
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("T,lengths", PN_RAGGED, ids=[f"T{t}-" + "x".join(map(str, l)) for t, l in PN_RAGGED])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_postnet_ragged_ops_in_isolation(postnets, precision, T, lengths):
    """Every PostNet op of a ragged call per utterance on its own L_b frames, after a dense NaN call at the same (B, T); x
    and the mask NaN past L_b.  Each row also equals its own B = 1 call bit for bit and is exactly 0 past L_b."""
    eng, sd = postnets(precision)
    B = len(lengths)
    nan = torch.full((B, 80, T), NAN, device="cuda")
    eng.debug_capture(True)
    try:
        eng.forward(nan, torch.ones(B, 1, T, device="cuda"))
        torch.cuda.synchronize()
        left = _not_nan(eng.debug_read, eng.debug_names())
    finally:
        eng.debug_capture(False)
    assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
    x = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(SEED + T))
    rp = PostNetReplay(eng, sd, precision, _past(x, lengths), _ragged_mask(lengths, lengths, T), lengths=lengths)
    _report_and_assert(f"postnet ragged {precision} T={T}", rp.run(), rp.nonfinite)
    y = rp.full["y"]
    for b, Lb in enumerate(lengths):
        assert torch.count_nonzero(y[b, :, Lb:]) == 0, f"utterance {b}: output not 0 past L_b = {Lb}"
        one = eng.forward(x[b:b + 1, :, :Lb].contiguous().cuda(), torch.ones(1, 1, Lb, device="cuda"))
        assert torch.equal(y[b:b + 1, :, :Lb].float(), one), f"row {b} (L={Lb}): not its own call bit for bit"


@pytest.mark.parametrize("T,mask_lengths", PN_DENSE, ids=[f"T{t}-" + "x".join(map(str, l)) for t, l in PN_DENSE])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_postnet_ops_in_isolation(postnets, precision, T, mask_lengths):
    """Every PostNet op of a dense call against its float64 replay; with a 0/1 mask the GroupNorm statistics cover the whole
    grid, padded columns included, as the reference's do."""
    eng, sd = postnets(precision)
    B = len(mask_lengths)
    x = torch.randn(B, 80, T, generator=torch.Generator().manual_seed(SEED + 2 * T))
    mask = (torch.arange(T)[None, :] < torch.tensor(mask_lengths)[:, None]).float()[:, None]
    rp = PostNetReplay(eng, sd, precision, x, mask)
    _report_and_assert(f"postnet dense {precision} T={T}", rp.run(), rp.nonfinite)


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_postnet_capture_is_transparent(postnets, precision):
    """Capture on changes neither the output (bitwise) nor the launch count, dense or ragged, and names every captured
    tensor in launch order."""
    eng, _ = postnets(precision)
    T, lengths = 300, [300, 129, 3]
    x = torch.randn(3, 80, T, generator=torch.Generator().manual_seed(SEED)).cuda()
    mask = (torch.arange(T)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None].cuda()
    for L in (None, torch.tensor(lengths).cuda()):
        off = eng.forward(x, mask, L)
        n_off = eng.last_launch_count()
        eng.debug_capture(True)
        try:
            on = eng.forward(x, mask, L)
            n_on = eng.last_launch_count()
        finally:
            eng.debug_capture(False)
        torch.cuda.synchronize()
        assert torch.equal(on, off)
        assert n_on == n_off
        assert eng.debug_names() == ["a0", "block1.raw", "block1.stats", "block1.act", "block2.raw", "block2.stats", "res"]
