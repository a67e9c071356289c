"""Ragged DiffVC batches, host side (no GPU): the C ABI declares and the library exports the new entry points, and the
Python surfaces take the lengths by keyword only, so every existing positional call keeps its meaning."""
import inspect
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["sbk_postnet_forward_lengths", "sbk_vc_estimator_lengths", "sbk_vc_reverse_diffusion_lengths",
       "sbk_vc_conditioning_lengths"]


def test_header_declares_the_entry_points():
    with open(os.path.join(ROOT, "include", "sbk.h")) as f:
        h = f.read()
    for name in NEW:
        assert re.search(rf"\bint {name}\(", h), name


def test_library_exports_the_entry_points(sbk_lib):
    from speech_backbones_b200.binding import EXPORTS
    for name in NEW:
        assert hasattr(sbk_lib, name), name
    for name in NEW[1:]:
        assert name in EXPORTS


def _kwonly(fn, name):
    p = inspect.signature(fn).parameters[name]
    return p.kind == inspect.Parameter.KEYWORD_ONLY and p.default is None


def test_lengths_are_keyword_only():
    from speech_backbones_b200.diffvc import Diffusion, FwdDiffusion
    from speech_backbones_b200.postnet import PostNet
    assert _kwonly(PostNet.forward, "lengths")
    assert _kwonly(FwdDiffusion.forward, "lengths")
    assert _kwonly(Diffusion.forward, "lengths")
    assert _kwonly(Diffusion.reverse_diffusion, "lengths")
    assert _kwonly(Diffusion.reverse_diffusion, "ref_lengths")
    assert _kwonly(Diffusion.conditioning_table, "ref_lengths")
    from speech_backbones_b200.diffvc import DiffVC, convert_from_encoder
    for fn in (DiffVC.forward, convert_from_encoder):
        p = inspect.signature(fn).parameters["ragged"]
        assert p.kind == inspect.Parameter.KEYWORD_ONLY and p.default is False


def test_engine_methods_default_to_the_padded_batch():
    from speech_backbones_b200.binding import Engine
    for m in (Engine.vc_estimator, Engine.vc_reverse_diffusion):
        assert inspect.signature(m).parameters["lengths"].default is None
    assert inspect.signature(Engine.vc_conditioning).parameters["ref_lengths"].default is None


# ---- the oracle against the unmodified reference's digests (tests/golden/diffvc_ragged_golden.pt) ------------------------
def _golden_script():
    import importlib.util
    path = os.path.join(ROOT, "scripts", "make_golden_diffvc_ragged.py")
    spec = importlib.util.spec_from_file_location("make_golden_diffvc_ragged", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _sha(t):
    import hashlib
    return hashlib.sha256(t.detach().to(torch.float32).contiguous().numpy().tobytes()).hexdigest()


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_ragged_golden.pt"), weights_only=False)


@pytest.mark.parametrize("mode", ["pf", "ml"])
def test_oracle_reproduces_the_per_utterance_reference(golden, mode):
    """Each utterance's B = 1 DiffVC.forward, restated by the oracle, has the digest the unmodified reference recorded"""
    from oracle import postnet_oracle as O
    G = _golden_script()
    case = next(c for c in golden["cases"] if c["mode"] == mode)
    sd = O.model_synthetic_weights(golden["seed"])
    x, x_ref, c = G.inputs()
    noise = G.draws(mode)
    with torch.no_grad():
        for b in range(golden["B"]):
            args = G.utterance(b, x, x_ref, c, noise)
            mean_x, y = G.oracle_forward(sd, *args[:5], mode, args[5])
            row = case["rows"][b]
            for name, t in (("mean_x", mean_x), ("y", y)):
                want = row[name]
                assert list(t.shape) == want["shape"], (mode, b, name)
                if name == "mean_x" or row["oracle_bitwise"]:
                    assert _sha(t) == want["sha256"], (mode, b, name)
                else:       # the generator recorded the oracle's rel-L2 to the reference; the norms must agree to it
                    assert abs(float(t.double().norm()) - want["norm"]) <= 1e-6 * want["norm"], (mode, b, name)


def test_padded_batch_is_not_the_per_utterance_call(golden):
    """Per stage, the reference's padded-batch semantics against each utterance's own call (the oracle): the PostNet, the
    RefBlock conditioning and one U-Net estimator call.  The gaps are printed (-s); the short rows must differ."""
    from oracle import diffvc_oracle as D, postnet_oracle as O
    from speech_backbones_b200.spec import DiffVCConfig
    G = _golden_script()
    sd = O.model_synthetic_weights(golden["seed"])
    enc = {k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}
    dec = {k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")}
    cfg = DiffVCConfig()
    x, x_ref, c = G.inputs()
    L, R = torch.tensor(G.LENGTHS), torch.tensor(G.REF_LENGTHS)

    def mask(l, t):
        return (torch.arange(t)[None, :] < l[:, None]).float()[:, None]

    def gap(a, b):
        return ((a.double() - b.double()).norm() / b.double().norm()).item()
    with torch.no_grad():
        pn = O.postnet(enc, x, mask(L, G.T), pre="postnet.")
        cond = D.conditioning(dec, cfg, x_ref[:, None] * mask(R, G.TR)[:, None], mask(R, G.TR), c, torch.full((G.B,), 0.5))[1]
        xe = x * mask(L, G.T)
        est = D.estimator(dec, cfg, xe, mask(L, G.T), x, x_ref[:, None] * mask(R, G.TR)[:, None], mask(R, G.TR), c,
                          torch.full((G.B,), 0.5))
        gaps = {"postnet": [], "conditioning": [], "estimator": []}
        for b in range(G.B):
            l, r = G.LENGTHS[b], G.REF_LENGTHS[b]
            one = O.postnet(enc, x[b:b + 1, :, :l], torch.ones(1, 1, l), pre="postnet.")
            gaps["postnet"].append(gap(pn[b:b + 1, :, :l], one))
            cr = x_ref[b:b + 1, :, :r][:, None]
            gaps["conditioning"].append(gap(cond[b:b + 1], D.conditioning(dec, cfg, cr, torch.ones(1, 1, r), c[b:b + 1],
                                                                           torch.full((1,), 0.5))[1]))
            # the same conditioning input for both (the padded batch's reference), so the gap is the U-Net's own
            tb = G.fix_len(l)
            xb = torch.zeros(1, 80, tb)
            xb[:, :, :l] = xe[b:b + 1, :, :l]
            mb = mask(torch.tensor([l]), tb)
            mnb = torch.zeros(1, 80, tb)
            mnb[:, :, :l] = x[b:b + 1, :, :l]
            e1 = D.estimator(dec, cfg, xb, mb, mnb, x_ref[b:b + 1, None] * mask(R[b:b + 1], G.TR)[:, None],
                             mask(R[b:b + 1], G.TR), c[b:b + 1], torch.full((1,), 0.5))
            gaps["estimator"].append(gap(est[b:b + 1, :, :l], e1[:, :, :l]))
    for k, v in gaps.items():
        print(f"padded batch vs own call, {k}: rel-L2 " + " ".join(f"{g:.2e}" for g in v))
        assert max(v[1:]) > 1e-4, k
