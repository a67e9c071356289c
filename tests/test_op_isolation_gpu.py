"""Op isolation on the GPU: every captured op of one estimator call against its float64 replay (tests/op_replay.py), in all
four precision modes, at shapes where the 128-pixel row tiles of the wgmma conv break: every level runs a ragged tile after
full ones, mask edges fall next to tile seams, and the grids hold more tiles than SMs, so CTAs move between tiles with
different border patterns.  Plus the PostNet at every dim its handle accepts, end to end against the float64 oracle.

Run with -s to see, per case and op, the worst |err| / (kappa A) (check 1, must be <= 1) and the worst group ratio
max / median (check 2, must be <= R_UNIFORM)."""
import pytest
import torch

from helpers import rel_l2
from op_replay import MIN_GROUP, R_UNIFORM, Replay, ntile_widths, uniformity
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict

pytestmark = pytest.mark.gpu
MODES = ["fp32", "fp32x3", "tf32", "bf16"]

# (B, T, lengths, n_spks): level widths T, T/2, T/4
GRADTTS_CASES = [
    (1, 132, [132], 1),                 # 132 / 66 / 33: a 4-column tile after a full one at level 0
    (2, 516, [516, 257], 1),            # 516 / 258 / 129: remainder tiles of 4, 2 and 1 columns; mask edge at 257
    (3, 508, [508, 129, 128], 1),       # 508 / 254 / 127: tiles 4, 2 and 1 columns short; mask edges at the seam
    (2, 260, [260, 131], 4),            # multi-speaker first Block (3 planar input channels)
]
DIFFVC_CASES = [(1, 260), (2, 132)]     # DiffVC U-Net, dim 256, ragged masks


def _mask(B, T, lengths):
    return (torch.arange(T)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]


@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache = {}

    def get(model, precision, n_spks=1):
        key = (model, precision, n_spks)
        if key not in cache:
            if model == "diffvc":
                from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec
                cfg = DiffVCConfig()
                sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
                e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision)
            else:
                cfg = UNetConfig(n_spks=n_spks)
                sd = synthetic_state_dict(cfg, 1234)
                e = Engine(n_spks=n_spks, precision=precision)
            e.load_state_dict(sd)
            cache[key] = (e, cfg, sd)
        return cache[key]
    yield get
    for e, _, _ in cache.values():
        e.close()


def _report_and_assert(tag, rows):
    for name, elem, unif, where in rows:
        print(f"{tag} {name:44s} |err|/(kA) {elem:.3e}  max/median {unif:6.2f} {where}")
    we = max(rows, key=lambda r: r[1])
    wu = max(rows, key=lambda r: r[2])
    print(f"WORST {tag}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("B,T,lengths,n_spks", GRADTTS_CASES, ids=[f"B{c[0]}-T{c[1]}-spk{c[3]}" for c in GRADTTS_CASES])
def test_gradtts_ops_in_isolation(engines, precision, B, T, lengths, n_spks):
    eng, cfg, sd = engines("gradtts", precision, n_spks)
    z, _, mu, spk, _ = synthetic_inputs(B, T, n_spks=n_spks)
    mask = _mask(B, T, lengths)
    t = torch.linspace(0.9, 0.2, B)
    rows = Replay(eng, sd, precision, "gradtts", z * mask, mask, mu, t, spk=spk, dim=cfg.dim,
                  pe_scale=cfg.pe_scale).run()
    _report_and_assert(f"gradtts {precision} B={B} T={T} spk={n_spks}", rows)


@pytest.mark.parametrize("precision", MODES)
@pytest.mark.parametrize("B,T", DIFFVC_CASES)
def test_diffvc_ops_in_isolation(engines, precision, B, T):
    from oracle import diffvc_oracle as D
    from speech_backbones_b200.spec import synthetic_diffvc_inputs
    eng, cfg, sd = engines("diffvc", precision)
    z, mask, mean, r, rmask, mean_ref, spk = synthetic_diffvc_inputs(B, T, 100, ragged=True)
    if B > 1:
        mask = _mask(B, T, [T] + [T // 2 + 3] * (B - 1))         # a mask edge off the tile grid
    t = torch.linspace(0.8, 0.3, B)
    g = D._gamma(cfg, 0, 0.5)
    xt_ref = ((r * g + mean_ref * (1.0 - g)) * rmask)[:, None]
    _, cond = D.conditioning(sd, cfg, xt_ref, rmask, spk, t)
    rows = Replay(eng, sd, precision, "diffvc", z * mask, mask, mean, t, cond=cond, dim=cfg.dim_unet).run()
    _report_and_assert(f"diffvc {precision} B={B} T={T}", rows)


def test_conv3x3_runs_both_ntile_widths():
    """The planner picks 64- or 128-wide N tiles for a 3x3 conv with Cout % 128 == 0 from B, W and the SM count; across the
    Grad-TTS cases above (run in every tensor-core mode) both widths must occur, or the cases no longer cover both."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sd = synthetic_state_dict(UNetConfig(), 1234)
    for precision in ("fp32x3", "tf32", "bf16"):
        widths = set()
        for B, T, _, _ in GRADTTS_CASES:
            widths |= ntile_widths(sd, B, 80, T, sms)
        assert widths == {64, 128}, f"{precision}: N-tile widths {widths} on {sms} SMs"


# ---- PostNet: the dims its handle accepts, both precisions, against the float64 oracle ----------------------------------
POSTNET_TOL = {"fp32x3": 2e-5, "tf32": 4e-3}          # test_postnet_gpu.py's per-call bounds
ALIAS = {"fp32x3": "fp32", "tf32": "bf16"}
# (n_feats, B, T, lengths): ragged tiles, n_feats < 7 (kernel rows that read only the zero page), odd n_feats, T = 1
POSTNET_CASES = [(80, 3, 263, [263, 129, 1]), (3, 2, 129, [129, 64]), (81, 1, 127, [127]), (80, 1, 1, [1])]


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
@pytest.mark.parametrize("dim", [64, 128, 256, 512])
def test_postnet_accepted_dims(sbk_lib, dim, precision):
    from oracle import postnet_oracle as P
    from speech_backbones_b200.postnet import PostNetEngine
    from speech_backbones_b200.spec import synthetic_postnet_state_dict
    sd = synthetic_postnet_state_dict(dim, 1234)
    e, alias = PostNetEngine(dim, precision=precision), PostNetEngine(dim, precision=ALIAS[precision])
    try:
        e.load_state_dict(sd)
        alias.load_state_dict(sd)
        sd64 = {k: v.cuda().double() for k, v in sd.items()}
        for n_feats, B, T, lengths in POSTNET_CASES:
            x = torch.randn(B, n_feats, T, generator=torch.Generator().manual_seed(dim + n_feats + T)).cuda()
            mask = _mask(B, T, lengths).cuda()
            y = e.forward(x, mask)
            ref = P.postnet(sd64, x.double(), mask.double())
            err = rel_l2(y, ref)
            # uniformity of the output over its columns (b, t) and rows (b, h), valid frames only: e_g = RMS error.
            # Utterances shorter than the 7-wide kernel are left out: every column of theirs sees a different set of taps.
            long_enough = (torch.tensor(lengths) >= 7).float().cuda()[:, None, None, None]
            cnt = (mask[:, None] * long_enough).expand(B, 1, n_feats, T).double()
            d = (y.double() - ref)[:, None] * cnt
            unif, where = uniformity(d, cnt, cnt, min_group=MIN_GROUP, valid=cnt)
            print(f"postnet dim={dim} {precision} n_feats={n_feats} B={B} T={T} rel_l2 {err:.3e} "
                  f"max/median {unif:.2f} {where}")
            assert err <= POSTNET_TOL[precision]
            assert unif <= R_UNIFORM, where
            bias = sd["final_conv.bias"].item()
            pad = mask.expand_as(y) == 0
            assert bool((y[pad] == bias).all()), "a padded column must equal final_conv.bias exactly"
            assert torch.equal(alias.forward(x, mask), y), f"a {ALIAS[precision]} handle must run the {precision} path"
    finally:
        e.close()
        alias.close()
