"""DiffVC's encoder side on the CPU: PostNet (DiffVC/model/postnet.py:40-53), FwdDiffusion (vc.py:19-41) and the whole DiffVC
model (vc.py:52-144).  The oracle against the committed outputs of the UNMODIFIED reference (tests/golden/
fwd_diffusion_golden.pt, diffvc_e2e_golden.pt); the drop-in modules' parameter trees and the reference's one known answer
(DiffVC/inference.ipynb: 126,259,128 parameters); the PostNet handle's C-ABI weight inventory (host logic); rejections."""
import os

import pytest
import torch

from oracle import postnet_oracle as O
from speech_backbones_b200.spec import DIFFVC_MODEL_ARGS, diffvc_model_param_spec, postnet_param_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fg():
    return torch.load(os.path.join(ROOT, "tests", "golden", "fwd_diffusion_golden.pt"), weights_only=False)


def _inputs(seed, c):
    x = torch.randn(c["B"], 80, c["T"], generator=torch.Generator().manual_seed(seed + c["T"]))
    mask = (torch.arange(c["T"])[None, :] < torch.tensor(c["lengths"])[:, None]).float()[:, None]
    return x, mask


def test_postnet_oracle_matches_reference_golden(fg):
    from speech_backbones_b200.spec import synthetic_postnet_state_dict
    sd = synthetic_postnet_state_dict(128, fg["seed"])
    for c in fg["postnet"]:
        x, mask = _inputs(fg["seed"], c)
        with torch.no_grad():
            assert (O.postnet(sd, x, mask) - c["out"]).abs().max().item() <= 1e-5


def test_fwd_diffusion_oracle_matches_reference_golden(fg):
    sd = O.fwd_synthetic_weights(fg["seed"])
    for c in fg["fwd"]:
        x, mask = _inputs(fg["seed"], c)
        with torch.no_grad():
            assert (O.fwd_diffusion(sd, x, mask) - c["out"]).abs().max().item() <= 1e-5


def test_encoder_outputs_of_the_e2e_golden_are_fwd_diffusion():
    g = torch.load(os.path.join(ROOT, "tests", "golden", "diffvc_e2e_golden.pt"), weights_only=False)
    sd = {k[len("encoder."):]: v for k, v in O.model_synthetic_weights(g["seed"]).items() if k.startswith("encoder.")}
    gen = torch.Generator().manual_seed(g["seed"])
    x, x_ref = torch.randn(g["B"], 80, g["T"], generator=gen), torch.randn(g["B"], 80, g["T_ref"], generator=gen)
    mask = (torch.arange(g["T"])[None, :] < torch.tensor(g["lengths"])[:, None]).float()[:, None]
    rmask = (torch.arange(g["T_ref"])[None, :] < torch.tensor(g["ref_lengths"])[:, None]).float()[:, None]
    with torch.no_grad():
        assert (O.fwd_diffusion(sd, x, mask) - g["mean"]).abs().max().item() <= 1e-5
        assert (O.fwd_diffusion(sd, x_ref, rmask) - g["mean_ref"]).abs().max().item() <= 1e-5


def test_module_trees_and_reference_parameter_counts():
    from speech_backbones_b200.diffvc import DiffVC, FwdDiffusion
    from speech_backbones_b200.postnet import PostNet
    pn = PostNet(128)
    assert {k: tuple(v.shape) for k, v in pn.state_dict().items()} == postnet_param_spec(128)
    assert pn.nparams == 1_623_297 and len(pn.state_dict()) == 14
    fwd = FwdDiffusion(*DIFFVC_MODEL_ARGS[:8], 128)
    assert fwd.nparams == 8_464_529
    model = DiffVC(*DIFFVC_MODEL_ARGS)
    spec = diffvc_model_param_spec()
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == spec and len(spec) == 346
    assert model.nparams == 126_259_128                     # DiffVC/inference.ipynb, BASELINE.md
    model.load_state_dict(O.model_synthetic_weights(3), strict=True)
    from oracle import text_encoder_oracle as T
    assert {k[len("encoder.encoder."):]: v for k, v in spec.items() if k.startswith("encoder.encoder.")} == dict(T.mel_param_spec())


def test_postnet_handle_weight_inventory_is_the_modules(sbk_lib):
    from speech_backbones_b200.postnet import PostNet, PostNetEngine
    for sym in ("sbk_postnet_create", "sbk_postnet_destroy", "sbk_postnet_num_weights", "sbk_postnet_weight_name",
                "sbk_postnet_set_weight", "sbk_postnet_pack", "sbk_postnet_workspace_bytes", "sbk_postnet_forward",
                "sbk_postnet_last_launch_count"):
        assert hasattr(sbk_lib, sym), sym
    for dim in (64, 128, 256):
        e = PostNetEngine(dim)
        assert e.weight_names() == list(PostNet(dim).state_dict().keys())
        e.close()


@pytest.mark.parametrize("dim,groups", [(100, 8), (192, 8), (32, 8), (128, 4), (128, 16)])
def test_unsupported_postnet_configs_are_rejected(sbk_lib, dim, groups):
    from speech_backbones_b200.postnet import PostNet
    with pytest.raises(ValueError, match="sbk_postnet_create"):
        PostNet(dim, groups)


@pytest.mark.parametrize("dim", [64, 128, 256, 512])
def test_supported_postnet_dims_are_accepted(sbk_lib, dim):
    """dim 64, 128 or a multiple of 256 (8 GroupNorm groups of 8, 16 or a multiple of 32 channels) creates a handle."""
    from speech_backbones_b200.postnet import PostNet
    assert PostNet(dim).dim == dim


def test_postnet_workspace_same_for_fp32x3_and_tf32(sbk_lib):
    """fp32x3 stores the tf32 mode's tensors: its convs derive the correction operand in shared memory (host-only)."""
    from speech_backbones_b200.postnet import PostNetEngine
    ws = {}
    for precision in ("fp32x3", "tf32", "fp32"):
        e = PostNetEngine(128, precision=precision)
        try:
            ws[precision] = [int(e.lib.sbk_postnet_workspace_bytes(e.h, B, 80, T)) for B, T in ((1, 1), (2, 17), (64, 256))]
        finally:
            e.close()
    assert ws["fp32x3"] == ws["tf32"] == ws["fp32"] and min(ws["tf32"]) > 0, ws


def test_cpu_tensors_raise(sbk_lib):
    from speech_backbones_b200.diffvc import FwdDiffusion
    from speech_backbones_b200.postnet import PostNet
    with pytest.raises(RuntimeError, match="CUDA"):
        PostNet(128)(torch.zeros(1, 80, 8), torch.ones(1, 1, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        FwdDiffusion(*DIFFVC_MODEL_ARGS[:8], 128)(torch.zeros(1, 80, 8), torch.ones(1, 1, 8))
