"""GPU tests of DiffVC's encoder side: the native PostNet (sbk_postnet_forward: two 7x7 convs on wgmma), FwdDiffusion
(MelEncoder + PostNet) and the whole drop-in DiffVC.forward, against the committed outputs of the UNMODIFIED reference
(tests/golden/fwd_diffusion_golden.pt, diffvc_e2e_golden.pt; scripts/make_golden_*.py).

Bounds (rel-L2): the DiffVC per-call bounds of test_diffvc_gpu.py - fp32x3 2e-5, tf32 4e-3 per encoder call; the sampler
trajectory bounds fp32x3 2e-4, tf32 1e-2 on the decoder output.  An fp32 handle must take exactly the fp32x3 path and a bf16
handle exactly the tf32 path (bitwise-equal outputs)."""
import os

import pytest
import torch

from helpers import rel_l2
from oracle import postnet_oracle as O
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS, synthetic_postnet_state_dict

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENC_TOL = {"fp32x3": 2e-5, "tf32": 4e-3}
TRAJ_TOL = {"fp32x3": 2e-4, "tf32": 1e-2}
ALIAS = {"fp32x3": "fp32", "tf32": "bf16"}       # the handle maps the second precision onto the first


@pytest.fixture(scope="module")
def fg():
    return torch.load(os.path.join(ROOT, "tests", "golden", "fwd_diffusion_golden.pt"), weights_only=False)


@pytest.fixture(scope="module")
def e2e():
    return torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_e2e_golden.pt"), weights_only=False)


def _inputs(seed, c):
    x = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(seed + c["T"]))
    mask = (torch.arange(c["T"])[None, :] < torch.tensor(c["lengths"])[:, None]).float()[:, None]
    return x.cuda(), mask.cuda()


def _postnet(seed, precision):
    from speech_backbones_b200.postnet import PostNet
    m = PostNet(128, precision=precision).eval()
    m.load_state_dict(synthetic_postnet_state_dict(128, seed), strict=True)
    return m.cuda()


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_postnet_vs_reference_golden(fg, precision):
    m, alias = _postnet(fg["seed"], precision), _postnet(fg["seed"], ALIAS[precision])
    for c in fg["postnet"]:
        x, mask = _inputs(fg["seed"], c)
        y = m(x, mask)
        err = rel_l2(y.cpu(), c["out"])
        print(f"postnet {precision} B={c['B']} T={c['T']} rel_l2 {err:.3e} launches {m.engine().last_launch_count()}")
        assert err <= ENC_TOL[precision]
        assert torch.equal(alias(x, mask), y), f"a {ALIAS[precision]} handle must run the {precision} path"


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_postnet_padding_and_determinism(fg, precision):
    m = _postnet(fg["seed"], precision)
    bias = m.final_conv.bias.detach().item()
    c = fg["postnet"][2]                                  # B = 3, T = 203, lengths [203, 1, 150]
    x, mask = _inputs(fg["seed"], c)
    y = m(x, mask)
    pad = (mask.expand_as(y) == 0)
    assert pad.any() and bool((y[pad] == bias).all()), "a padded column must equal final_conv.bias exactly"
    assert torch.equal(m(x, mask), y), "two identical calls must be bitwise equal"
    for i in range(3):
        yi = m(x[i:i + 1].contiguous(), mask[i:i + 1].contiguous())
        assert torch.equal(yi, y[i:i + 1]), f"utterance {i} alone differs from its row in the batch"


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_fwd_diffusion_vs_reference_golden(fg, precision):
    from speech_backbones_b200.diffvc import FwdDiffusion
    m = FwdDiffusion(*DIFFVC_MODEL_ARGS[:8], 128, precision=precision).eval()
    m.load_state_dict(O.fwd_synthetic_weights(fg["seed"]), strict=True)
    m = m.cuda()
    for c in fg["fwd"]:
        x, mask = _inputs(fg["seed"], c)
        err = rel_l2(m(x, mask).cpu(), c["out"])
        print(f"fwd_diffusion {precision} B={c['B']} T={c['T']} rel_l2 {err:.3e}")
        assert err <= ENC_TOL[precision]


def _model(e2e, precision):
    from speech_backbones_b200.diffvc import DiffVC
    model = DiffVC(*DIFFVC_MODEL_ARGS, precision=precision)        # the notebook's sequence (DiffVC/inference.ipynb)
    model = model.cuda()
    model.load_state_dict(O.model_synthetic_weights(e2e["seed"]), strict=True)
    model.eval()
    assert model.nparams == 126_259_128
    gen = torch.Generator().manual_seed(e2e["seed"])
    x, x_ref = torch.randn(e2e["B"], 80, e2e["T"], generator=gen), torch.randn(e2e["B"], 80, e2e["T_ref"], generator=gen)
    c = torch.randn(e2e["B"], 256, generator=gen)
    args = (x.cuda(), torch.tensor(e2e["lengths"]).cuda(), x_ref.cuda(), torch.tensor(e2e["ref_lengths"]).cuda(),
            (c / c.norm(dim=1, keepdim=True)).cuda())
    return model, args


def _replay(monkeypatch, noise):
    """The reference's randn_like draws, in order (a GPU cannot reproduce a CPU generator's stream)."""
    it = iter(noise)
    monkeypatch.setattr(torch, "randn_like", lambda t, **kw: next(it).to(t.device))
    return it


@pytest.mark.parametrize("precision", ["fp32x3", "tf32"])
def test_diffvc_forward_end_to_end(e2e, monkeypatch, precision):
    model, args = _model(e2e, precision)
    for case in e2e["cases"]:
        it = _replay(monkeypatch, case["noise"])
        mean_x, y = model(*args, n_timesteps=e2e["N"], mode=case["mode"])
        assert next(it, None) is None, "the forward drew a different number of noise tensors than the reference"
        e1, e2 = rel_l2(mean_x.cpu(), case["mean_x"]), rel_l2(y.cpu(), case["y"])
        print(f"DiffVC.forward {precision} mode={case['mode']} mean_x rel_l2 {e1:.3e} y rel_l2 {e2:.3e}")
        assert e1 <= ENC_TOL[precision] and e2 <= TRAJ_TOL[precision]


def test_diffvc_invalid_mode_prints_and_returns_z(e2e, monkeypatch, capsys):
    model, args = _model(e2e, "fp32x3")
    noise = e2e["cases"][0]["noise"]
    _replay(monkeypatch, noise)
    mean_x, y = model(*args, n_timesteps=e2e["N"], mode="sde")
    assert "Inference mode must be one of [pf, em, ml]!" in capsys.readouterr().out
    T = e2e["T"]
    mask = (torch.arange(T)[None, :] < torch.tensor(e2e["lengths"])[:, None]).float()[:, None].cuda()
    assert torch.equal(y, torch.where(mask != 0, mean_x, torch.zeros_like(mean_x)) + noise[0][:, :, :T].cuda())
