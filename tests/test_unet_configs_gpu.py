"""The score U-Net at the widths its constructors accept beyond those of the shipped checkpoints (Grad-TTS dim = 64,
n_feats = 80, spk_emb_dim = 64; DiffVC dim_unet = 256, dim_spk = 128): every captured op of one estimator call against its
float64 replay (tests/op_replay.py Replay, judged as in test_op_isolation_gpu.py: check 1 |err| / (kappa A) <= 1, check 2
max / median <= R_UNIFORM), in all four precision modes, and one trajectory per drop-in module at non-default
hyper-parameters against the float64 oracle.

GroupNorm(8, C) runs at C / 8 = cpg channels per group, and three kernels write its partial sums tile by tile: the planar
first conv (64-channel tiles), the CUDA-core convs of the fp32 mode (64) and the wgmma convs (64 or 128, conv_tc_ntile and
the planner).  At dim = 64 / 128 / 256 / 512 every tile starts on a group boundary and cpg is 8, 16 or a multiple of 32.
The widths below also run cpg an odd multiple of 8 (24) or of 16 (48), tiles that start inside a group (cpg 40, 80, 96)
and groups wider than a tile (cpg 96 / 160 / 192): a partial credited to the wrong group, or a group a tile touches but
does not flush, gives a wrong mean / rstd to every consumer of that GroupNorm, which check 1 sees at once.
test_gn_tile_kinds_covered says which of these kinds the cases run, under the planner's N-tile rule.

Run with -s for every op's checks and one WORST line per case (and per utterance of a ragged call)."""
import pytest
import torch

from helpers import rel_l2
from op_replay import RESNETS, Replay
from test_diffvc_gpu import TOL as VC_TOL
from test_op_isolation_gpu import MODES, _mask, _report_and_assert
from test_rolling_gpu import REF_TOL
from speech_backbones_b200.gradtts import fix_len_compatibility
from speech_backbones_b200.spec import (DiffVCConfig, UNetConfig, diffvc_param_spec, estimator_param_spec,
                                        synthetic_diffvc_inputs, synthetic_inputs, synthetic_state_dict)

gpu = pytest.mark.gpu
NAN = float("nan")

# Grad-TTS: (id, UNetConfig fields, B, T, lengths); level widths T, T/2, T/4, level heights n_feats, /2, /4
GRADTTS_CASES = [
    ("dim128", dict(dim=128), 2, 260, [260, 131]),                 # cpg 16 / 32 / 64
    ("dim192", dict(dim=192), 2, 132, [132, 67]),                  # cpg 24 / 48 / 96
    ("dim320", dict(dim=320), 1, 132, [132]),                      # cpg 40 / 80 / 160: 128-wide tiles start mid-group
    ("dim384", dict(dim=384), 1, 68, [68]),                        # cpg 48 / 96 / 192 >= the N tile (~275 M weights)
    ("feats4", dict(n_feats=4), 2, 132, [132, 61]),                # heights 4 / 2 / 1
    ("feats8", dict(n_feats=8), 2, 132, [132, 61]),                # 8 / 4 / 2
    ("feats100", dict(n_feats=100), 2, 132, [132, 61]),            # 100 / 50 / 25 (odd)
    ("feats128", dict(n_feats=128), 2, 132, [132, 61]),            # 128 / 64 / 32
    # k_spk's MLP at another width, the planar first conv's third input, the time table at another scale
    ("spk3-emb16-pe500", dict(n_spks=3, spk_emb_dim=16, pe_scale=500.0), 2, 132, [132, 61]),
    ("spk3-emb256", dict(n_spks=3, spk_emb_dim=256), 2, 132, [132, 61]),
]
# ragged calls (lengths=) after a NaN call at the same (B, T), as test_gradtts_ragged_ops_in_isolation
GRADTTS_RAGGED = [
    ("dim192", dict(dim=192), 3, 260, [260, 131, 1]),
    ("feats100", dict(n_feats=100), 2, 132, [132, 61]),
]
# DiffVC: (id, DiffVCConfig fields, B, T); a mask edge off the tile grid on every row after the first
DIFFVC_CASES = [
    ("unet128", dict(dim_unet=128), 2, 132),
    ("unet192", dict(dim_unet=192), 2, 132),
    ("spk256", dict(dim_spk=256), 2, 132),
    ("noref-spk36", dict(use_ref_t=False, dim_spk=36), 2, 132),    # a multiple of 4, not of 8
    ("noref-spk64", dict(use_ref_t=False, dim_spk=64), 2, 132),
    ("feats100", dict(n_feats=100), 2, 132),
]
DIFFVC_RAGGED = [("unet192", dict(dim_unet=192), 3, 260, [260, 131, 1])]
T_REF = 100

_SD = {}


def _state_dict(cfg):
    """synthetic weights of a config (seed 1234), made once per module run"""
    key = repr(cfg)
    if key not in _SD:
        spec = diffvc_param_spec(cfg) if isinstance(cfg, DiffVCConfig) else None
        _SD[key] = synthetic_state_dict(cfg, 1234, spec=spec)
    return _SD[key]


def _engine(cfg, precision):
    from speech_backbones_b200.binding import Engine
    if isinstance(cfg, DiffVCConfig):
        e = Engine(cfg.n_feats, cfg.dim_unet, beta_min=cfg.beta_min, beta_max=cfg.beta_max, precision=precision,
                   model="diffvc", dim_cond=cfg.dim_spk, use_ref_t=cfg.use_ref_t)
    else:
        e = Engine(cfg.n_feats, cfg.dim, cfg.n_spks, cfg.spk_emb_dim, cfg.beta_min, cfg.beta_max, cfg.pe_scale,
                   precision=precision)
    e.load_state_dict(_state_dict(cfg))
    return e


def _poison(eng, call, B, n_feats, T):
    """A dense call at (B, T) on x = mu = NaN (mask all ones), capture on: every buffer a captured op writes in the plan's
    workspace, which the ragged call at (B, T) then reuses, holds NaN.  Returns the names whose capture is not all NaN."""
    nan = torch.full((B, n_feats, T), NAN, device="cuda")
    eng.debug_capture(True)
    try:
        call(nan, torch.ones(B, 1, T, device="cuda"), nan)
        torch.cuda.synchronize()
        left = []
        for name in eng.debug_names():
            v = eng.debug_read(name)
            if v is not None and not bool(torch.isnan(v).all()):
                left.append(f"{name} ({int((~torch.isnan(v)).sum())} of {v.numel()} not NaN)")
        return left
    finally:
        eng.debug_capture(False)


def _ragged_inputs(x, mask, mu, lengths):
    """NaN at and past every utterance's edge T_b = fix_len_compatibility(L_b) in x, mask and mu; mask 0 on [L_b, T_b)"""
    B, _, T = x.shape
    TB = torch.tensor([fix_len_compatibility(n) for n in lengths])
    past = (torch.arange(T)[None, :] >= TB[:, None])[:, None]
    mask = torch.where(past, NAN, mask)
    return torch.where(past, NAN, x * mask), mask, torch.where(past, NAN, mu), TB


def _judge_ragged(tag, rp, TB):
    rows = rp.run()
    assert not rp.nonfinite, "NaN / Inf inside an utterance: " + ", ".join(rp.nonfinite)
    for b, Tb in enumerate(TB.tolist()):
        assert torch.count_nonzero(rp.full["y"][b, :, Tb:]) == 0, f"utterance {b}: output not 0 past T_b = {Tb}"
    _report_and_assert(tag, rows)


def _vc_cond(cfg, sd, B, T, t):
    """DiffVC's estimator inputs and its conditioning rows from the CPU oracle at the config"""
    from oracle import diffvc_oracle as D
    z, _, mean, r, rmask, mean_ref, spk = synthetic_diffvc_inputs(B, T, T_REF, n_feats=cfg.n_feats, ragged=True)
    g = D._gamma(cfg, 0, 0.5)
    xt_ref = ((r * g + mean_ref * (1.0 - g)) * rmask)[:, None]
    _, cond = D.conditioning(sd, cfg, xt_ref, rmask, spk, t)
    return z, mean, cond


# ---- op isolation ------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", GRADTTS_CASES, ids=[c[0] for c in GRADTTS_CASES])
def test_gradtts_config_ops_in_isolation(sbk_lib, case, precision):
    name, kw, B, T, lengths = case
    cfg = UNetConfig(**kw)
    sd = _state_dict(cfg)
    eng = _engine(cfg, precision)
    try:
        z, _, mu, spk, _ = synthetic_inputs(B, T, n_feats=cfg.n_feats, n_spks=cfg.n_spks, spk_emb_dim=cfg.spk_emb_dim)
        mask = _mask(B, T, lengths)
        t = torch.linspace(0.9, 0.2, B)
        rows = Replay(eng, sd, precision, "gradtts", z * mask, mask, mu, t, spk=spk, dim=cfg.dim,
                      pe_scale=cfg.pe_scale).run()
        _report_and_assert(f"gradtts {name} {precision} B={B} T={T}", rows)
    finally:
        eng.close()


@gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", GRADTTS_RAGGED, ids=[c[0] for c in GRADTTS_RAGGED])
def test_gradtts_config_ragged_ops_in_isolation(sbk_lib, case, precision):
    name, kw, B, T, lengths = case
    cfg = UNetConfig(**kw)
    sd = _state_dict(cfg)
    eng = _engine(cfg, precision)
    try:
        z, _, mu, spk, _ = synthetic_inputs(B, T, n_feats=cfg.n_feats, n_spks=cfg.n_spks, spk_emb_dim=cfg.spk_emb_dim)
        t = torch.linspace(0.9, 0.2, B)
        left = _poison(eng, lambda x, m, u: eng.estimator(x, m, u, t.cuda()), B, cfg.n_feats, T)
        assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
        x, mask, mu, TB = _ragged_inputs(z, _mask(B, T, lengths), mu, lengths)
        rp = Replay(eng, sd, precision, "gradtts", x, mask, mu, t, spk=spk, dim=cfg.dim, pe_scale=cfg.pe_scale,
                    lengths=lengths)
        _judge_ragged(f"gradtts ragged {name} {precision} B={B} T={T}", rp, TB)
    finally:
        eng.close()


@gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", DIFFVC_CASES, ids=[c[0] for c in DIFFVC_CASES])
def test_diffvc_config_ops_in_isolation(sbk_lib, case, precision):
    name, kw, B, T = case
    cfg = DiffVCConfig(**kw)
    sd = _state_dict(cfg)
    eng = _engine(cfg, precision)
    try:
        t = torch.linspace(0.8, 0.3, B)
        z, mean, cond = _vc_cond(cfg, sd, B, T, t)
        mask = _mask(B, T, [T] + [T // 2 + 3] * (B - 1))
        rows = Replay(eng, sd, precision, "diffvc", z * mask, mask, mean, t, cond=cond, dim=cfg.dim_unet).run()
        _report_and_assert(f"diffvc {name} {precision} B={B} T={T}", rows)
    finally:
        eng.close()


@gpu
@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("case", DIFFVC_RAGGED, ids=[c[0] for c in DIFFVC_RAGGED])
def test_diffvc_config_ragged_ops_in_isolation(sbk_lib, case, precision):
    name, kw, B, T, lengths = case
    cfg = DiffVCConfig(**kw)
    sd = _state_dict(cfg)
    eng = _engine(cfg, precision)
    try:
        t = torch.linspace(0.9, 0.2, B)
        z, mean, cond = _vc_cond(cfg, sd, B, T, t)
        left = _poison(eng, lambda x, m, u: eng.vc_estimator(x, m, u, cond.cuda(), t.cuda()), B, cfg.n_feats, T)
        assert not left, "captures not poisoned by the NaN call: " + ", ".join(left)
        x, mask, mu, TB = _ragged_inputs(z, _mask(B, T, lengths), mean, lengths)
        rp = Replay(eng, sd, precision, "diffvc", x, mask, mu, t, cond=cond, dim=cfg.dim_unet, lengths=lengths)
        _judge_ragged(f"diffvc ragged {name} {precision} B={B} T={T}", rp, TB)
    finally:
        eng.close()


# ---- which GroupNorm tilings the cases run -------------------------------------------------------------------------------
H100_SMS = 132          # the H100 SXM's SM count, which the planner's N-tile choice reads


def gn_tilings(spec, B, H0, T, sms=H100_SMS):
    """{(Cout, N tile)} of the convs that write GroupNorm partials, as the planner tiles them (sbk_api.cu tc_conv): the
    planar first conv and every conv of the fp32 mode in 64-channel tiles; in the tensor-core modes the 3x3 convs in 128-wide
    tiles when Cout % 128 == 0, unless two-row tiles (from 4 waves of them on) or too few one-row tiles to fill half the SMs
    make them 64 wide."""
    Hs, Ws = (H0, H0 // 2, H0 // 4), (T, T // 2, T // 4)
    convs = [(lvl, spec[f"estimator.{pre}.block1.block.0.weight"][0]) for pre, (lvl, _) in RESNETS.items()]
    convs.append((0, spec["estimator.final_block.block.0.weight"][0]))
    out = set()
    for lvl, cout in convs:
        out.add((cout, 64))
        wt = (Ws[lvl] + 127) // 128
        two = B * wt * ((Hs[lvl] + 1) // 2) * (cout // 64) >= 4 * sms
        if cout % 128 == 0 and not two and B * wt * Hs[lvl] * (cout // 128) * 2 > sms:
            out.add((cout, 128))
    return out


KINDS = ("cpg an odd multiple of 8 (> 8)", "cpg an odd multiple of 16 (> 16)",
         "cpg a multiple of 32, a tile starting inside a group and ending in the next",
         "cpg >= the N tile, not a multiple of it")


def _tile_kinds(cout, nt):
    """the kinds of GroupNorm tiling (KINDS) a conv of Cout channels in nt-wide N tiles runs; the widths of dim = 64
    (cpg 8, 16, 32 and 64, 128 in group-aligned tiles) run none of them"""
    cpg = cout // 8
    kinds = set()
    if cpg % 16 == 8 and cpg > 8:
        kinds.add(KINDS[0])
    if cpg % 32 == 16 and cpg > 16:
        kinds.add(KINDS[1])
    if cpg % 32 == 0 and any(n0 % cpg and (n0 + nt - 1) // cpg != n0 // cpg for n0 in range(0, cout, nt)):
        kinds.add(KINDS[2])
    if cpg >= nt and cpg % nt:
        kinds.add(KINDS[3])
    return kinds


def _groups_per_tile(cout, nt):
    cpg = cout // 8
    return max((n0 + nt - 1) // cpg - n0 // cpg + 1 for n0 in range(0, cout, nt))


def test_gn_tile_kinds_covered():
    """Across the cases above, the planner's tilings include each kind of GroupNorm tiling that the shipped widths do not
    run; if the tables are trimmed, this says which kind was lost."""
    tilings = set()
    for case in GRADTTS_CASES + GRADTTS_RAGGED:
        cfg, B, T = UNetConfig(**case[1]), case[2], case[3]
        tilings |= gn_tilings(estimator_param_spec(cfg), B, cfg.n_feats, T)
    for case in DIFFVC_CASES + DIFFVC_RAGGED:
        cfg, B, T = DiffVCConfig(**case[1]), case[2], case[3]
        tilings |= gn_tilings(diffvc_param_spec(cfg), B, cfg.n_feats, T)
    kinds = set().union(*(_tile_kinds(c, nt) for c, nt in tilings))
    assert kinds == set(KINDS), f"not covered: {sorted(set(KINDS) - kinds)} (tilings {sorted(tilings)})"
    shipped = gn_tilings(estimator_param_spec(UNetConfig()), 1, 80, 132) | gn_tilings(
        diffvc_param_spec(DiffVCConfig()), 1, 80, 132)
    assert not set().union(*(_tile_kinds(c, nt) for c, nt in shipped)), "the shipped widths run one of KINDS"


def test_gn_tiles_fit_the_slot_rows():
    """The GroupNorm epilogues keep 8 partial slots per warp (sbk_conv_tc.cu s_st; 8 groups in k_igemm and k_first_conv):
    at every dim the constructor accepts up to 4096, no tile the planner can choose touches more than 8 groups."""
    for dim in range(64, 4097, 64):
        for cout in (dim, 2 * dim, 4 * dim):
            for nt in (64, 128) if cout % 128 == 0 else (64,):
                assert _groups_per_tile(cout, nt) <= 8, (dim, cout, nt)


# ---- trajectories through the drop-in modules at non-default hyper-parameters ------------------------------------------
N_TRAJ = 4
NOISE_SEED = 913


@gpu
@pytest.mark.parametrize("precision", MODES)
def test_gradtts_dropin_nondefault_trajectory(sbk_lib, precision):
    """Diffusion(100, 192, n_spks=3, spk_emb_dim=16, beta_min=0.1, beta_max=40, pe_scale=500): step_coefs and the time
    table at values no other test uses, both samplers, against oracle.gradtts_oracle.reverse_diffusion in float64 with
    the module's own draws."""
    from oracle import gradtts_oracle as O
    from speech_backbones_b200.gradtts import Diffusion
    cfg = UNetConfig(n_feats=100, dim=192, n_spks=3, spk_emb_dim=16, beta_min=0.1, beta_max=40.0, pe_scale=500.0)
    sd = _state_dict(cfg)
    dec = Diffusion(100, 192, n_spks=3, spk_emb_dim=16, beta_min=0.1, beta_max=40, pe_scale=500, precision=precision)
    dec.load_state_dict(sd, strict=True)
    dec = dec.eval().cuda()
    z, mask, mu, spk, _ = (v.cuda() for v in synthetic_inputs(2, 132, n_feats=100, ragged=True, n_spks=3, spk_emb_dim=16))
    p64 = {k: v.cuda().double() for k, v in sd.items()}
    for stoc in (False, True):
        torch.manual_seed(NOISE_SEED)
        noise = torch.stack([torch.randn(z.shape, device="cuda") for _ in range(N_TRAJ)]) if stoc else None
        torch.manual_seed(NOISE_SEED)
        y = dec(z, mask, mu, N_TRAJ, stoc, spk)
        ref = O.reverse_diffusion(p64, cfg, z.double(), mask.double(), mu.double(), N_TRAJ, stoc, spk.double(),
                                  None if noise is None else noise.double())
        err = rel_l2(y, ref)
        print(f"gradtts Diffusion(100, 192, 3, 16, 0.1, 40, 500) {precision} stoc={stoc} N={N_TRAJ} rel-L2 {err:.3e}")
        assert err <= REF_TOL[precision], (stoc, err)
        assert (y * (1 - mask)).abs().max().item() == 0.0


@gpu
@pytest.mark.parametrize("precision", MODES)
def test_diffvc_dropin_nondefault_trajectory(sbk_lib, precision):
    """DiffVC's Diffusion(80, 192, 64, False, 0.1, 30): vc_step_coefs at other betas, without the RefBlock, in every
    sampler mode, against oracle.diffvc_oracle.reverse_diffusion in float64 with the module's own draws."""
    from oracle import diffvc_oracle as D
    from speech_backbones_b200.diffvc import Diffusion
    cfg = DiffVCConfig(n_feats=80, dim_unet=192, dim_spk=64, use_ref_t=False, beta_min=0.1, beta_max=30.0)
    sd = _state_dict(cfg)
    dec = Diffusion(80, 192, 64, False, 0.1, 30, precision=precision)
    dec.load_state_dict(sd, strict=True)
    dec = dec.eval().cuda()
    args = [v.cuda() for v in synthetic_diffvc_inputs(2, 132, T_REF, ragged=True)]
    z, mask = args[0], args[1]
    p64 = {k: v.cuda().double() for k, v in sd.items()}
    for mode in ("pf", "em", "ml"):
        torch.manual_seed(NOISE_SEED)
        noise = torch.stack([torch.randn_like(z) for _ in range(3)]) if mode != "pf" else None
        torch.manual_seed(NOISE_SEED)
        y = dec(*args, n_timesteps=3, mode=mode)
        ref = D.reverse_diffusion(p64, cfg, *(v.double() for v in args), 3, mode,
                                  None if noise is None else noise.double())
        err = rel_l2(y, ref)
        print(f"diffvc Diffusion(80, 192, 64, False, 0.1, 30) {precision} {mode} N=3 rel-L2 {err:.3e}")
        assert err <= VC_TOL[precision][1], (mode, err)
        assert (y * (1 - mask)).abs().max().item() == 0.0
