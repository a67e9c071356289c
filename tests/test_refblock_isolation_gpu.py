"""Op isolation for DiffVC's hoisted conditioning branch (sbk_vc_conditioning) on the GPU: every op of the last step of one
call against its float64 replay from the GPU's own captured inputs (tests/op_replay.py RefBlockReplay), at reference lengths
where the branch's tiles break:

  * Tr = 24, B = 2: the golden trajectory case, one partial tile everywhere;
  * Tr = 300, B = 1: wgmma tiles 128 | 128 | 44 per row and k_first_conv tiles 256 | 44;
  * Tr = 257, B = 2, lengths [257, 129]: a 1-pixel last wgmma tile, a 1-frame k_first_conv tail, and a mask edge one column
    past the 128-pixel seam;
  * Tr = 131, B = 3, lengths [131, 128, 1]: Tr not a multiple of 4, a mask edge exactly at the seam, a one-frame reference;
  * Tr = 300 at the level of real log-mels (ref and mean_ref around -5): the conv outputs' mean dwarfs their spread, the
    regime where InstanceNorm's E[x^2] - E[x]^2 cancels;
  * dim_spk = 256 (base 64: a 128-channel first conv, convs up to 512 output channels) at Tr = 257;
  * use_ref_t = False, where only k_vc_cond runs.

Each case runs in all four handle precisions (the branch itself is tf32 on tf32 / bf16 handles and fp32x3 on fp32x3 / fp32
handles), at N = 1 (t = 1) and at the last step of N = 4 (t = 0.25).  Every step's cond is also held to COND_TOL against the
oracle's conditioning evaluated in float64.

Run with -s to see, per case and op, the worst |err| / (kappa A) (check 1, must be <= 1), the worst group ratio max / median
(check 2, must be <= R_UNIFORM; 0 where op_replay.RB_NO_UNIFORMITY says why it has no groups) and the relative error of the
variance k_in_glu derives from each block's captured sums."""
import os

import pytest
import torch

from helpers import rel_l2
from op_replay import FIRST_CONV_TILE, R_UNIFORM, TC_TILE, RefBlockReplay
from oracle import diffvc_oracle as O
from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs, synthetic_state_dict
from test_diffvc_gpu import COND_TOL

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRECISIONS = ["fp32", "fp32x3", "tf32", "bf16"]
CONFIGS = {"spk128": DiffVCConfig(), "spk256": DiffVCConfig(dim_spk=256), "noref": DiffVCConfig(use_ref_t=False)}
LOG_MEL_SHIFT = -5.0
# (config, Tr, reference lengths or None for the golden case, shift of ref and mean_ref)
CASES = [("spk128", 24, None, 0.0), ("spk128", 300, [300], 0.0), ("spk128", 257, [257, 129], 0.0),
         ("spk128", 131, [131, 128, 1], 0.0), ("spk128", 300, [300], LOG_MEL_SHIFT), ("spk256", 257, [257, 129], 0.0),
         ("noref", 24, None, 0.0)]
CASE_IDS = [f"{c}-Tr{t}-" + ("golden" if l is None else "x".join(map(str, l))) + ("-logmel" if s else "")
            for c, t, l, s in CASES]


@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cache, sds = {}, {}

    def get(config, precision):
        cfg = CONFIGS[config]
        if config not in sds:
            sds[config] = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
        if (config, precision) not in cache:
            e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision, use_ref_t=cfg.use_ref_t)
            e.load_state_dict(sds[config])
            cache[config, precision] = e
        return cache[config, precision], cfg, sds[config]
    yield get
    for e in cache.values():
        e.close()


def case_inputs(Tr, lengths, shift):
    """(ref, ref_mask, mean_ref, c) on the CPU: the golden trajectory case, or seeded N(0, 1) mels (+ shift) with the given
    reference lengths"""
    if lengths is None:
        g = torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_golden.pt"), weights_only=False)
        c = next(c for c in g["cases"] if c["kind"] == "traj" and c["mode"] == "ml" and c["B"] == 2)
        assert c["Tr"] == Tr
        _, _, _, ref, rmask, mean_ref, spk = synthetic_diffvc_inputs(c["B"], c["T"], c["Tr"], seed=g["seed"], ragged=c["ragged"])
        return ref, rmask, mean_ref, spk
    B = len(lengths)
    gen = torch.Generator().manual_seed(7919 * Tr + B)
    ref = torch.randn(B, 80, Tr, generator=gen) + shift
    mean_ref = torch.randn(B, 80, Tr, generator=gen) + shift
    c = torch.randn(B, 256, generator=gen)
    c = c / c.norm(dim=1, keepdim=True)
    rmask = (torch.arange(Tr)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]
    return ref, rmask, mean_ref, c


def oracle_table(sd, cfg, ref, rmask, mean_ref, c, N, dev="cuda"):
    """O.conditioning for every step of an N-step call, in float64 (weights and inputs)"""
    d = torch.float64
    p = {k: v.to(dev, d) for k, v in sd.items()}
    ref, rmask, mean_ref, c = (v.to(dev, d) for v in (ref, rmask, mean_ref, c))
    rows = []
    for i in range(N):
        t, _, _, _, g0t = O.step_coefficients(cfg, N, i, "ml")
        xt_ref = ((ref * g0t + mean_ref * (1.0 - g0t)) * rmask)[:, None]
        rows.append(O.conditioning(p, cfg, xt_ref, rmask, c, t * torch.ones(ref.shape[0], dtype=d, device=dev))[1])
    return torch.stack(rows)


def _report_and_assert(tag, rows, var_err):
    for name, elem, unif, where in rows:
        print(f"{tag} {name:14s} |err|/(kA) {elem:.3e}  max/median {unif:6.2f} {where}")
    if var_err:
        print(f"{tag} InstanceNorm variance rel. error: " + ", ".join(f"{b} {v:.2e}" for b, v in var_err.items()))
    we, wu = max(rows, key=lambda r: r[1]), max(rows, key=lambda r: r[2])
    print(f"WORST {tag}: |err|/(kA) {we[1]:.3e} ({we[0]})  max/median {wu[2]:.2f} ({wu[0]} {wu[3]})")
    bad = [r for r in rows if not (r[1] <= 1.0 and r[2] <= R_UNIFORM)]
    assert not bad, "ops out of bounds: " + ", ".join(f"{n} ({e:.3g}, {u:.3g} {w})" for n, e, u, w in bad)


@pytest.mark.parametrize("N", [1, 4])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("config,Tr,lengths,shift", CASES, ids=CASE_IDS)
def test_refblock_ops_in_isolation(engines, config, Tr, lengths, shift, precision, N):
    eng, cfg, sd = engines(config, precision)
    ref, rmask, mean_ref, c = case_inputs(Tr, lengths, shift)
    rp = RefBlockReplay(eng, sd, precision, cfg, ref, rmask, mean_ref, c, N)
    tag = f"{config} Tr={Tr} {lengths or 'golden'}{' logmel' if shift else ''} {precision} N={N}"
    # the chain: every step's cond against the float64 oracle
    want = oracle_table(sd, cfg, ref, rmask, mean_ref, c, N)
    errs = [rel_l2(rp.table[i], want[i]) for i in range(N)]
    print(f"{tag} cond rel-L2 vs float64 oracle per step: " + ", ".join(f"{e:.2e}" for e in errs))
    _report_and_assert(tag, rp.run(), rp.var_err)
    assert max(errs) <= COND_TOL[precision], errs


def test_refblock_aliases_compute_the_same_table(engines):
    """bf16 handles run the branch as tf32 handles do, fp32 handles as fp32x3 handles do: bit for bit."""
    ref, rmask, mean_ref, c = (v.cuda() for v in case_inputs(257, [257, 129], 0.0))
    tab = {p: engines("spk128", p)[0].vc_conditioning(ref, rmask, mean_ref, c, 4) for p in PRECISIONS}
    assert torch.equal(tab["bf16"], tab["tf32"])
    assert torch.equal(tab["fp32"], tab["fp32x3"])


def _expected_names():
    names = ["ref_block.xt_ref", "ref_block.tb"]
    for b in ("block11", "block12", "block21", "block22", "block31", "block32"):
        names += [f"ref_block.{b}.raw", f"ref_block.{b}.stats", f"ref_block.{b}.act"]
    return names + ["ref_block.ysum"]


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_refblock_capture_is_transparent(engines, precision):
    """Capture on changes neither the table (bitwise) nor the launch count, and names every written tensor in launch order."""
    eng, _, _ = engines("spk128", precision)
    ref, rmask, mean_ref, c = (v.cuda() for v in case_inputs(257, [257, 129], 0.0))
    off = eng.vc_conditioning(ref, rmask, mean_ref, c, 4)
    n_off = eng.last_launch_count()
    eng.debug_capture(True)
    try:
        on = eng.vc_conditioning(ref, rmask, mean_ref, c, 4)
        n_on = eng.last_launch_count()
    finally:
        eng.debug_capture(False)
    torch.cuda.synchronize()
    assert torch.equal(on, off)
    assert n_on == n_off
    assert eng.vc_cond_debug_names() == _expected_names()
    # the estimator's own capture list is untouched by the branch
    assert not any(n.startswith("ref_block.") for n in eng.debug_names())


def test_refblock_cases_reach_the_edges():
    """The case list keeps a ragged wgmma tile after a full one, the k_first_conv seam, a Tr that is not a multiple of 4, a
    one-frame reference and a mask edge at a tile seam."""
    trs = [Tr for _, Tr, _, _ in CASES]
    lens = [l for _, _, ls, _ in CASES if ls for l in ls]
    assert any(Tr > TC_TILE and Tr % TC_TILE for Tr in trs)
    assert any(Tr > FIRST_CONV_TILE for Tr in trs)
    assert any(Tr % 4 for Tr in trs)
    assert 1 in lens
    assert any(l % TC_TILE == 0 and l < Tr for _, Tr, ls, _ in CASES if ls for l in ls)
    assert any(s for *_, s in CASES)
