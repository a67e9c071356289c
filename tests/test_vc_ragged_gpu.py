"""Ragged DiffVC batches on the GPU: the PostNet (`PostNet.forward(x, mask, lengths=)`, so `FwdDiffusion.forward(...,
lengths=)`) and the score U-Net (`Engine.vc_estimator / vc_reverse_diffusion(..., lengths=)`).

The reference converts one utterance per call (DiffVC/inference.ipynb, B = 1).  For utterance b of a padded batch with
L_b = lengths[b], that call runs:
  * the PostNet on exactly L_b frames - its GroupNorm statistics and 7x7 borders see no padding, and there is no rounding
    of the length;
  * the U-Net on T'_b = fix_len_compatibility(L_b) frames with the mask valid for L_b of them (the Grad-TTS rule).
With `lengths`, row b must equal that call on its valid frames, and be exactly 0 past them.  The inputs past every edge are
NaN here, so any read of them into a valid output would show.

Bounds.  The PostNet packs its N tile once per handle and every one of its ops is per pixel or cut at the edge exactly as
the B = 1 call cuts it, so its rows are bit for bit the single calls in every mode.

The U-Net's 3x3 convs pick one- or two-row tiles from the launch's tile count (sbk_api.cu: two-row tiles from 4 waves on,
SBK_CONV3_ROWS overrides the choice).  At DiffVC's widths (256 / 512 / 1024 channels) the two layouts round the raw conv
outputs differently in the last bit, so a dense padded batch's full-length row already differs from its B = 1 call when the
two shapes pick different layouts (first at downs.1.0.block2.raw, |diff| ~2e-6 in tf32).  Grad-TTS's 64-channel U-Net does
not show this.  So the ragged machinery is held bit for bit (tf32, bf16) or within rel-L2 1e-6 (fp32x3, fp32: their N tile
depends on the tile count) with the layout pinned to either one, and the default layout within the per-call and trajectory
bounds of test_diffvc_gpu.py, with the measured gap printed.

Lengths {160, 131, 61, 1} at T = 160 (the 128-pixel seam, a level-0 edge inside the second tile, a length that is not a
multiple of 4, one frame), and {300, 129, 128, 127, 3} at T = 300 for the PostNet (edges one column either side of the
seam and a tile that ends past the image)."""
import os

import pytest
import torch

from helpers import rel_l2
from oracle import postnet_oracle as O
from test_diffvc_gpu import TOL
from speech_backbones_b200.diffvc import fix_len_compatibility
from speech_backbones_b200.spec import (DIFFVC_MODEL_ARGS, DiffVCConfig, diffvc_param_spec, synthetic_postnet_state_dict,
                                        synthetic_state_dict)

pytestmark = pytest.mark.gpu

PRECISIONS = ["fp32x3", "tf32", "bf16", "fp32"]
BITWISE_UNET = {"tf32", "bf16"}
PN_CASES = [(160, [160, 131, 61, 1]), (300, [300, 129, 128, 127, 3])]
T_VC, LEN_VC = 160, [160, 131, 61, 1]
SEED = 2718
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mask(lengths, T):
    return (torch.arange(T)[None, :] < torch.tensor(lengths)[:, None]).float()[:, None]


def _poison(x, lengths):
    """x with every frame at or past lengths[b] set to NaN (a copy)"""
    x = x.clone()
    for b, L in enumerate(lengths):
        x[b, ..., L:] = float("nan")
    return x


def _same(a, b, precision, layout, bound):
    """a U-Net row against its single call: pinned 3x3 layout - bit for bit (tf32, bf16) or rel-L2 1e-6; default layout -
    rel-L2 `bound`.  Returns the rel-L2 gap."""
    err = rel_l2(a, b)
    if layout == "auto":
        assert err <= bound, f"{precision}: rel-L2 {err:.3e} > {bound}"
    elif precision in BITWISE_UNET:
        assert torch.equal(a, b), f"{precision}: max |diff| {(a - b).abs().max().item():.3e}"
    else:
        assert err <= 1e-6, f"{precision}: rel-L2 {err:.3e}"
    return err


LAYOUTS = ["auto", "rows1", "rows2"]


def _pin(monkeypatch, layout):
    """pin the 3x3 convs' tile layout for every plan this test builds (read when a plan is built)"""
    if layout != "auto":
        monkeypatch.setenv("SBK_CONV3_ROWS", layout[-1])


# ---- PostNet ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def postnets():
    from speech_backbones_b200.postnet import PostNet
    sd = synthetic_postnet_state_dict(128, SEED)
    cache = {}

    def get(precision):
        if precision not in cache:
            m = PostNet(128, precision=precision).eval()
            m.load_state_dict(sd, strict=True)
            cache[precision] = m.cuda()
        return cache[precision]
    return get


@pytest.mark.parametrize("T,lengths", PN_CASES, ids=[f"T{t}" for t, _ in PN_CASES])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_postnet_rows_equal_single_calls(postnets, precision, T, lengths):
    m = postnets(precision)
    x = torch.randn(len(lengths), 80, T, generator=torch.Generator().manual_seed(SEED + T)).cuda()
    mask = _mask(lengths, T).cuda()
    L = torch.tensor(lengths).cuda()
    y = m(_poison(x, lengths), mask, lengths=L)
    assert not torch.isnan(y).any()
    padded = m(x, mask)
    gaps = []
    for b, Lb in enumerate(lengths):
        one = m(x[b:b + 1, :, :Lb].contiguous(), torch.ones(1, 1, Lb, device="cuda"))
        assert torch.equal(y[b:b + 1, :, :Lb], one), f"row {b} (L={Lb}): max |diff| {(y[b, :, :Lb] - one[0]).abs().max().item():.3e}"
        if Lb < T:
            assert y[b, :, Lb:].abs().max().item() == 0.0
        gaps.append(rel_l2(padded[b:b + 1, :, :Lb].cpu(), one.cpu()))
    print(f"postnet {precision} T={T}: padded-batch rows vs their own calls, rel-L2 " + " ".join(f"{g:.2e}" for g in gaps))
    # the padded batch is the reference's padded semantics, not the single calls: its short rows differ
    assert max(gaps[1:]) > 1e-4


@pytest.mark.parametrize("precision", PRECISIONS)
def test_postnet_full_lengths_equal_dense(postnets, precision):
    m = postnets(precision)
    T = 160
    x = torch.randn(3, 80, T, generator=torch.Generator().manual_seed(SEED)).cuda()
    mask = torch.ones(3, 1, T, device="cuda")
    assert torch.equal(m(x, mask, lengths=torch.full((3,), T, device="cuda")), m(x, mask))


def test_postnet_vs_oracle_per_utterance():
    """Row b of a ragged batch against the CPU oracle of the utterance's own call (the fp32x3 bound of test_postnet_gpu.py)"""
    from speech_backbones_b200.postnet import PostNet
    sd = synthetic_postnet_state_dict(128, SEED)
    m = PostNet(128, precision="fp32x3").eval()
    m.load_state_dict(sd, strict=True)
    m = m.cuda()
    T, lengths = PN_CASES[0]
    x = torch.randn(len(lengths), 80, T, generator=torch.Generator().manual_seed(SEED + T))
    y = m(_poison(x, lengths).cuda(), _mask(lengths, T).cuda(), lengths=torch.tensor(lengths).cuda()).cpu()
    for b, Lb in enumerate(lengths):
        ref = O.postnet(sd, x[b:b + 1, :, :Lb], torch.ones(1, 1, Lb))
        assert rel_l2(y[b:b + 1, :, :Lb], ref) <= 2e-5


def test_postnet_bad_lengths_raise_before_launch(postnets):
    m = postnets("tf32")
    T = 32
    x, mask = torch.randn(2, 80, T).cuda(), torch.ones(2, 1, T).cuda()
    m(x, mask)
    n = m.engine().last_launch_count()
    for bad in (torch.tensor([32, 3], dtype=torch.int32).cuda(), torch.tensor([32]).cuda(), torch.tensor([32, 3]),
                torch.tensor([32, 0]).cuda(), torch.tensor([33, 3]).cuda()):
        with pytest.raises(ValueError):
            m(x, mask, lengths=bad)
    assert m.engine().last_launch_count() == n


def test_fwd_diffusion_rows_equal_single_calls():
    """FwdDiffusion = MelEncoder + PostNet: the mel encoder's masked convs and -1e4 masked softmax keep a row's valid frames
    independent of its batch-mates (unchanged), and the ragged PostNet runs each row on its own frames."""
    from speech_backbones_b200.diffvc import FwdDiffusion
    torch.manual_seed(SEED)
    m = FwdDiffusion(*DIFFVC_MODEL_ARGS[:8], 128, precision="tf32").eval()
    m.load_state_dict(O.fwd_synthetic_weights(SEED), strict=True)
    m = m.cuda()
    T, lengths = T_VC, LEN_VC
    x = torch.randn(len(lengths), 80, T, generator=torch.Generator().manual_seed(SEED)).cuda()
    x = x * _mask(lengths, T).cuda() + (1 - _mask(lengths, T).cuda()) * 3.0     # finite padding: the encoder masks it
    mask = _mask(lengths, T).cuda()
    enc = m.encoder(x, mask)
    y = m(x, mask, lengths=torch.tensor(lengths).cuda())
    for b, Lb in enumerate(lengths):
        one_mask = torch.ones(1, 1, Lb, device="cuda")
        xb = x[b:b + 1, :, :Lb].contiguous()
        enc_one = m.encoder(xb, one_mask)
        print(f"mel encoder row {b} (L={Lb}): rel-L2 vs its own call {rel_l2(enc[b:b + 1, :, :Lb].cpu(), enc_one.cpu()):.3e}")
        assert torch.equal(enc[b:b + 1, :, :Lb], enc_one), f"mel encoder row {b}"
        assert torch.equal(y[b:b + 1, :, :Lb], m(xb, one_mask)), f"FwdDiffusion row {b}"
        if Lb < T:
            assert y[b, :, Lb:].abs().max().item() == 0.0


# ---- the score U-Net ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def engines(sbk_lib):
    from speech_backbones_b200.binding import Engine
    cfg = DiffVCConfig()
    sd = synthetic_state_dict(cfg, 1234, spec=diffvc_param_spec(cfg))
    cache = {}

    def get(precision, layout="auto"):
        # one handle per 3x3 tile layout: a plan keeps the layout it was built with (_pin)
        if (precision, layout) not in cache:
            e = Engine(80, cfg.dim_unet, model="diffvc", dim_cond=cfg.dim_spk, precision=precision)
            e.load_state_dict(sd)
            cache[precision, layout] = e
        return cache[precision, layout], cfg
    yield get
    for e in cache.values():
        e.close()


def _vc_inputs(lengths, T, dc, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(lengths)
    mean = torch.randn(B, 80, T, generator=g)
    z = mean + torch.randn(B, 80, T, generator=g)
    cond = torch.randn(B, dc, generator=g) * 0.5
    return z, mean, cond


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_vc_estimator_rows_equal_single_calls(engines, precision, layout, monkeypatch):
    _pin(monkeypatch, layout)
    eng, cfg = engines(precision, layout)
    T, lengths = T_VC, LEN_VC
    B = len(lengths)
    z, mean, cond = _vc_inputs(lengths, T, cfg.dim_spk, SEED)
    mask = _mask(lengths, T)
    t = torch.tensor([0.9, 0.5, 0.3, 0.7])
    tp = [fix_len_compatibility(L) for L in lengths]
    L = torch.tensor(lengths).cuda()
    y = eng.vc_estimator(_poison(z * mask, tp).cuda(), mask.cuda(), _poison(mean, tp).cuda(), cond.cuda(), t.cuda(),
                         lengths=L).cpu()
    assert not torch.isnan(y).any()
    padded = eng.vc_estimator((z * mask).cuda(), mask.cuda(), mean.cuda(), cond.cuda(), t.cuda()).cpu()
    gaps, errs = [], []
    for b in range(B):
        Tb = tp[b]
        one = eng.vc_estimator((z * mask)[b:b + 1, :, :Tb].contiguous().cuda(), mask[b:b + 1, :, :Tb].contiguous().cuda(),
                               mean[b:b + 1, :, :Tb].contiguous().cuda(), cond[b:b + 1].cuda(), t[b:b + 1].cuda()).cpu()
        errs.append(_same(y[b:b + 1, :, :Tb], one, precision, layout, TOL[precision][0]))
        if Tb < T:
            assert y[b, :, Tb:].abs().max().item() == 0.0
        gaps.append(rel_l2(padded[b:b + 1, :, :Tb], one))
    print(f"vc_estimator {precision} {layout}: ragged rows vs their own calls, rel-L2 " + " ".join(f"{g:.2e}" for g in errs))
    print(f"vc_estimator {precision} {layout}: padded-batch rows vs their own calls, rel-L2 " + " ".join(f"{g:.2e}" for g in gaps))
    assert max(gaps[1:]) > 1e-3
    full = eng.vc_estimator((z * mask).cuda(), mask.cuda(), mean.cuda(), cond.cuda(), t.cuda(),
                            lengths=torch.full((B,), T).cuda()).cpu()
    assert torch.equal(full, padded), "full lengths must be the dense call bit for bit"


@pytest.mark.parametrize("layout", ["auto", "rows1"])
@pytest.mark.parametrize("mode", ["pf", "em", "ml"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_vc_reverse_diffusion_rows_equal_single_calls(engines, precision, mode, layout, monkeypatch):
    _pin(monkeypatch, layout)
    eng, cfg = engines(precision, layout)
    T, N = T_VC, 3
    tp_all = {}
    # two ragged calls at the same (B, T, N) with different lengths: both replay the ragged loop graph, both right
    for lengths in (LEN_VC, [97, 160, 4, 130]):
        B = len(lengths)
        z, mean, _ = _vc_inputs(lengths, T, cfg.dim_spk, SEED + sum(lengths))
        mask = _mask(lengths, T)
        cond = torch.randn(N, B, cfg.dim_spk, generator=torch.Generator().manual_seed(SEED)) * 0.5
        noise = None if mode == "pf" else torch.randn(N, B, 80, T, generator=torch.Generator().manual_seed(SEED + 1))
        tp = [fix_len_compatibility(L) for L in lengths]
        tp_all[tuple(lengths)] = tp
        y = eng.vc_reverse_diffusion(_poison(z, tp).cuda(), mask.cuda(), _poison(mean, tp).cuda(), cond.cuda(), N, mode,
                                     None if noise is None else _poison(noise.transpose(0, 1), tp).transpose(0, 1).cuda(),
                                     lengths=torch.tensor(lengths).cuda()).cpu()
        assert not torch.isnan(y).any()
        assert eng.last_host_launches() <= N
        for b in range(B):
            Tb = tp[b]
            one = eng.vc_reverse_diffusion(z[b:b + 1, :, :Tb].contiguous().cuda(), mask[b:b + 1, :, :Tb].contiguous().cuda(),
                                           mean[b:b + 1, :, :Tb].contiguous().cuda(), cond[:, b:b + 1].contiguous().cuda(), N,
                                           mode, None if noise is None else noise[:, b:b + 1, :, :Tb].contiguous().cuda()).cpu()
            err = _same(y[b:b + 1, :, :Tb], one, precision, layout, TOL[precision][1])
            print(f"vc_reverse_diffusion {precision} {mode} {layout} lengths {lengths} row {b}: rel-L2 {err:.2e}")
            if Tb < T:
                assert y[b, :, Tb:].abs().max().item() == 0.0


def test_vc_full_lengths_loop_equals_dense(engines):
    eng, cfg = engines("tf32")
    T, N, B = T_VC, 3, 2
    z, mean, _ = _vc_inputs([T, T], T, cfg.dim_spk, SEED)
    mask = torch.ones(B, 1, T)
    cond = torch.randn(N, B, cfg.dim_spk, generator=torch.Generator().manual_seed(SEED)) * 0.5
    noise = torch.randn(N, B, 80, T, generator=torch.Generator().manual_seed(SEED + 2))
    args = (z.cuda(), mask.cuda(), mean.cuda(), cond.cuda(), N, "ml", noise.cuda())
    assert torch.equal(eng.vc_reverse_diffusion(*args, lengths=torch.full((B,), T).cuda()), eng.vc_reverse_diffusion(*args))


def test_vc_bad_lengths_raise_before_launch(engines):
    eng, cfg = engines("tf32")
    T, B = 32, 2
    x, mean = torch.randn(B, 80, T).cuda(), torch.randn(B, 80, T).cuda()
    mask, cond, t = torch.ones(B, 1, T).cuda(), torch.randn(B, cfg.dim_spk).cuda(), torch.rand(B).cuda()
    eng.vc_estimator(x, mask, mean, cond, t)
    n = eng.last_launch_count()
    for bad in (torch.tensor([32, 3], dtype=torch.int32).cuda(), torch.tensor([32]).cuda(), torch.tensor([32, 3]),
                torch.tensor([32, 0]).cuda(), torch.tensor([33, 3]).cuda()):
        with pytest.raises(ValueError):
            eng.vc_estimator(x, mask, mean, cond, t, lengths=bad)
        with pytest.raises(ValueError):
            eng.vc_reverse_diffusion(x, mask, mean, cond[None], 1, "pf", lengths=bad)
    assert eng.last_launch_count() == n


def test_dense_unet_rows_depend_on_the_3x3_tile_layout(engines, monkeypatch):
    """The finding behind the default-layout bounds above: in a DENSE call, a full-length row of a padded batch differs in
    the last bits from its own B = 1 call (tf32) because the two shapes pick different 3x3 tile layouts at DiffVC's
    widths; with the layout pinned they are equal."""
    T, B = T_VC, 4
    z, mean, cond = _vc_inputs([T] * B, T, DiffVCConfig().dim_spk, SEED)
    mask, t = torch.ones(B, 1, T), torch.tensor([0.9, 0.5, 0.3, 0.7])
    gaps = {}
    for layout in ("auto", "rows1"):
        _pin(monkeypatch, layout)
        eng, _ = engines("tf32", layout)
        y = eng.vc_estimator(z.cuda(), mask.cuda(), mean.cuda(), cond.cuda(), t.cuda()).cpu()
        one = eng.vc_estimator(z[:1].cuda(), mask[:1].cuda(), mean[:1].cuda(), cond[:1].cuda(), t[:1].cuda()).cpu()
        gaps[layout] = rel_l2(y[:1], one)
        monkeypatch.delenv("SBK_CONV3_ROWS", raising=False)
    print(f"dense tf32 full-length row 0 vs its own call: rel-L2 {gaps['auto']:.2e} (default layout), "
          f"{gaps['rows1']:.2e} (one-row tiles)")
    assert gaps["rows1"] == 0.0
    assert 0.0 < gaps["auto"] <= TOL["tf32"][0]


# ---- the RefBlock conditioning branch ----------------------------------------------------------------------------------
REF_CASES = [(160, [97, 144, 130, 1]), (257, [257, 129, 128, 3])]


@pytest.mark.parametrize("Tr,ref_lengths", REF_CASES, ids=[f"Tr{t}" for t, _ in REF_CASES])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_vc_conditioning_rows_equal_single_calls(engines, precision, Tr, ref_lengths):
    """vc_conditioning(..., ref_lengths=) against B = 1 calls on ref[b, :, :R_b] with an all-ones mask: bit for bit in
    every mode (the branch's convs keep one tile layout and its reductions cut each reference's frames as its own call
    does), with ref and mean_ref NaN past every R_b.  Full lengths equal the dense call bit for bit."""
    eng, cfg = engines(precision)
    B, N = len(ref_lengths), 3
    g = torch.Generator().manual_seed(SEED + Tr)
    ref, mean_ref = torch.randn(B, 80, Tr, generator=g), torch.randn(B, 80, Tr, generator=g)
    c = torch.randn(B, 256, generator=g)
    c = c / c.norm(dim=1, keepdim=True)
    rmask = _mask(ref_lengths, Tr)
    cond = eng.vc_conditioning(_poison(ref, ref_lengths).cuda(), rmask.cuda(), _poison(mean_ref, ref_lengths).cuda(),
                               c.cuda(), N, ref_lengths=torch.tensor(ref_lengths).cuda()).cpu()
    assert not torch.isnan(cond).any()
    padded = eng.vc_conditioning(ref.cuda(), rmask.cuda(), mean_ref.cuda(), c.cuda(), N).cpu()
    gaps = []
    for b, Rb in enumerate(ref_lengths):
        one = eng.vc_conditioning(ref[b:b + 1, :, :Rb].contiguous().cuda(), torch.ones(1, 1, Rb).cuda(),
                                  mean_ref[b:b + 1, :, :Rb].contiguous().cuda(), c[b:b + 1].cuda(), N).cpu()
        assert torch.equal(cond[:, b:b + 1], one), f"row {b} (R={Rb}): max |diff| {(cond[:, b:b + 1] - one).abs().max().item():.3e}"
        gaps.append(rel_l2(padded[:, b:b + 1], one))
    print(f"vc_conditioning {precision} Tr={Tr}: padded-batch rows vs their own calls, rel-L2 " + " ".join(f"{v:.2e}" for v in gaps))
    full = eng.vc_conditioning(ref.cuda(), torch.ones(B, 1, Tr).cuda(), mean_ref.cuda(), c.cuda(), N,
                               ref_lengths=torch.full((B,), Tr).cuda()).cpu()
    dense = eng.vc_conditioning(ref.cuda(), torch.ones(B, 1, Tr).cuda(), mean_ref.cuda(), c.cuda(), N).cpu()
    assert torch.equal(full, dense)


def test_vc_conditioning_bad_ref_lengths_raise(engines):
    eng, cfg = engines("tf32")
    B, Tr = 2, 24
    ref, m, c = torch.randn(B, 80, Tr).cuda(), torch.ones(B, 1, Tr).cuda(), torch.randn(B, 256).cuda()
    for bad in (torch.tensor([24, 3], dtype=torch.int32).cuda(), torch.tensor([24, 0]).cuda(), torch.tensor([25, 3]).cuda(),
                torch.tensor([24, 3])):
        with pytest.raises(ValueError):
            eng.vc_conditioning(ref, m, ref, c, 2, ref_lengths=bad)


# ---- DiffVC.forward(..., ragged=True) ----------------------------------------------------------------------------------
def _golden_script():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "make_golden_diffvc_ragged.py")
    spec = importlib.util.spec_from_file_location("make_golden_diffvc_ragged", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _replay(monkeypatch, draws):
    it = iter(draws)
    monkeypatch.setattr(torch, "randn_like", lambda t, **kw: next(it).to(t.device))
    return it


@pytest.mark.parametrize("layout", ["auto", "rows1"])
@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_diffvc_forward_ragged_rows_equal_single_calls(monkeypatch, precision, layout):
    """DiffVC.forward(..., ragged=True) on the batch of tests/golden/diffvc_ragged_golden.pt (x_lengths {160, 131, 61, 1},
    x_ref_lengths {97, 144, 130, 1}, N = 3, pf and ml, the recorded draws replayed), against
      * the per-utterance B = 1 DiffVC.forward on each row's slices, given the same draws: pinned 3x3 layout bit for bit in
        tf32 and within rel-L2 1e-6 in fp32x3, default layout within the trajectory bound;
      * the oracle's B = 1 outputs, which reproduce the unmodified reference's digests (checked here too): ENC_TOL on
        mean_x and TRAJ_TOL on y, the bounds of test_postnet_gpu.py.
    The padding of x and x_ref is finite random, as the torch glue multiplies it by the mask."""
    import hashlib
    from speech_backbones_b200.diffvc import DiffVC
    from test_postnet_gpu import ENC_TOL, TRAJ_TOL
    G = _golden_script()
    golden = torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_ragged_golden.pt"), weights_only=False)
    _pin(monkeypatch, layout)
    sd = O.model_synthetic_weights(G.SEED)
    model = DiffVC(*DIFFVC_MODEL_ARGS, precision=precision).eval()
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    x, x_ref, c = G.inputs()
    xl, rl = torch.tensor(G.LENGTHS), torch.tensor(G.REF_LENGTHS)
    for case in golden["cases"]:
        mode = case["mode"]
        noise = G.draws(mode)
        it = _replay(monkeypatch, noise)
        mean_x, y = model(x.cuda(), xl.cuda(), x_ref.cuda(), rl.cuda(), c.cuda(), G.N, mode, ragged=True)
        assert next(it, None) is None
        mean_x, y = mean_x.cpu(), y.cpu()
        assert not torch.isnan(y).any()
        for b in range(G.B):
            args = G.utterance(b, x, x_ref, c, noise)
            L = G.LENGTHS[b]
            _replay(monkeypatch, args[5])
            m1, y1 = model(*(a.cuda() for a in args[:5]), G.N, mode)
            m1, y1 = m1.cpu(), y1.cpu()
            assert torch.equal(mean_x[b:b + 1, :, :L], m1), f"{mode} mean_x row {b}"
            err = rel_l2(y[b:b + 1, :, :L], y1)
            if layout == "auto":
                assert err <= TOL[precision][1], (mode, b, err)
            elif precision == "tf32":
                assert torch.equal(y[b:b + 1, :, :L], y1), (mode, b, err)
            else:
                assert err <= 1e-6, (mode, b, err)
            if layout == "auto":
                om, oy = G.oracle_forward(sd, *args[:5], mode, args[5])
                if case["rows"][b]["oracle_bitwise"]:
                    assert hashlib.sha256(oy.contiguous().numpy().tobytes()).hexdigest() == case["rows"][b]["y"]["sha256"]
                e1, e2 = rel_l2(mean_x[b:b + 1, :, :L], om), rel_l2(y[b:b + 1, :, :L], oy)
                print(f"DiffVC.forward ragged {precision} {mode} row {b} (L={L}, R={G.REF_LENGTHS[b]}): vs own call {err:.2e}, "
                      f"vs the reference's B = 1 call mean_x {e1:.2e} y {e2:.2e}")
                assert e1 <= ENC_TOL[precision] and e2 <= TRAJ_TOL[precision]
