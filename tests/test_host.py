"""CPU: host-side logic - parameter inventory, strict loading errors, the C-ABI surface, the drop-in module."""
import ctypes as C
import os
import re

import pytest
import torch

from speech_backbones_b200 import UNetConfig, estimator_param_spec, synthetic_inputs, synthetic_state_dict
from oracle import gradtts_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_param_counts_match_survey_anchors():
    # SURVEY.md 8(c): decoder 7,634,887 params in 172 tensors (n_spks=1); 176 tensors multi-speaker
    spec = estimator_param_spec(UNetConfig())
    assert len(spec) == 172
    assert sum(torch.Size(s).numel() for s in spec.values()) == 7_634_887
    assert len(estimator_param_spec(UNetConfig(n_spks=4))) == 176


def test_header_symbols_all_exported(sbk_lib):
    hdr = open(os.path.join(ROOT, "include", "sbk.h")).read()
    names = set(re.findall(r"\b(sbk_[a-z_]+)\s*\(", hdr))
    names -= {"sbk_handle", "sbk_config"}
    assert len(names) >= 17
    for n in sorted(names):
        assert hasattr(sbk_lib, n), f"libsbk.so does not export {n}"
    assert b"sm_90a" in sbk_lib.sbk_version()


@pytest.mark.parametrize("n_spks", [1, 4])
def test_c_abi_weight_inventory_matches_python_spec(sbk_lib, n_spks):
    from speech_backbones_b200.binding import Engine
    eng = Engine(n_spks=n_spks)          # host-only: no CUDA call until set_weight
    assert eng.weight_names() == list(estimator_param_spec(UNetConfig(n_spks=n_spks)).keys())
    assert eng.workspace_bytes(2, 32) > 0
    assert eng.workspace_bytes(2, 30) == 0      # T % 4 != 0 is rejected (fix_len_compatibility)
    eng.close()


def test_c_abi_argument_errors(sbk_lib):
    from speech_backbones_b200.binding import Engine, SbkConfig
    h = C.c_void_p()
    bad = SbkConfig(0, 80, 48, 1, 64, 0.05, 20.0, 1000.0, 0, 0, 1)      # dim not a multiple of 64
    assert sbk_lib.sbk_create(C.byref(bad), C.byref(h)) != 0
    assert b"dim" in sbk_lib.sbk_last_error()
    eng = Engine()
    shape = (C.c_int64 * 2)(3, 3)
    buf = (C.c_float * 9)()
    rc = sbk_lib.sbk_set_weight(eng.h, b"estimator.not_a_key", buf, shape, 2)
    assert rc != 0 and b"unexpected key" in sbk_lib.sbk_last_error()
    rc = sbk_lib.sbk_set_weight(eng.h, b"estimator.mlp.0.weight", buf, shape, 2)
    assert rc != 0 and b"expected" in sbk_lib.sbk_last_error()
    assert sbk_lib.sbk_pack(eng.h) != 0 and b"missing key" in sbk_lib.sbk_last_error()
    eng.close()


def test_prior_expand_argument_errors(sbk_lib):
    """sbk_prior_expand validates its arguments before touching the GPU (return code + sbk_last_error, no exceptions)."""
    buf = (C.c_float * 16)()
    lens = (C.c_int64 * 1)(4)
    f = sbk_lib.sbk_prior_expand
    assert f(None, buf, buf, lens, None, C.c_float(1.0), 1, 1, 4, 4, buf, buf, buf, None, None) != 0
    assert b"null" in sbk_lib.sbk_last_error()
    assert f(buf, buf, buf, lens, None, C.c_float(1.0), 1, 1, 0, 4, buf, buf, buf, None, None) != 0
    assert b"bad sizes" in sbk_lib.sbk_last_error()
    assert f(buf, buf, buf, lens, None, C.c_float(1.0), 1, 1, 20000, 4, buf, buf, buf, None, None) != 0
    assert b"12000" in sbk_lib.sbk_last_error()
    assert f(buf, buf, buf, lens, buf, C.c_float(0.0), 1, 1, 4, 4, buf, buf, buf, None, None) != 0
    assert b"temperature" in sbk_lib.sbk_last_error()


def test_module_state_dict_is_reference_compatible():
    from speech_backbones_b200.gradtts import Diffusion
    for n_spks in (1, 4):
        cfg = UNetConfig(n_spks=n_spks)
        m = Diffusion(80, 64, n_spks=n_spks)
        spec = estimator_param_spec(cfg)
        got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
        assert got == {k: tuple(v) for k, v in spec.items()}
        m.load_state_dict(synthetic_state_dict(cfg), strict=True)
    assert Diffusion(80, 64).nparams == 7_634_887


def test_module_sampling_refuses_cpu():
    from speech_backbones_b200.gradtts import Diffusion
    m = Diffusion(80, 64)
    z, mask, mu, _, _ = synthetic_inputs(1, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(z, mask, mu, 2)


def test_module_training_forward_matches_oracle():
    """The autograd (training) estimator path over the same parameters equals the oracle."""
    from speech_backbones_b200.gradtts import Diffusion
    for n_spks in (1, 4):
        cfg = UNetConfig(n_spks=n_spks)
        sd = synthetic_state_dict(cfg)
        m = Diffusion(80, 64, n_spks=n_spks).eval()
        m.load_state_dict(sd)
        z, mask, mu, spk, _ = synthetic_inputs(2, 16, ragged=True, n_spks=n_spks)
        t = torch.tensor([0.3, 0.8])
        with torch.no_grad():
            a = m.estimator(z * mask, mask, mu, t, spk)
            b = O.estimator(sd, cfg, z * mask, mask, mu, t, spk)
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5)
    loss, _ = m.compute_loss(z, mask, mu, spk)
    loss.backward()
    assert torch.isfinite(loss)


def test_sinusoid_frequency_table_matches_torch():
    """libsbk computes exp(fp32(j) * fp32(-ln(1e4)/(half-1))) with glibc expf (correctly rounded) on the host.
    torch's vectorised fp32 exp (SinusoidalPosEmb, diffusion.py:121-122) may differ by 1 ulp on a few entries;
    the sin/cos argument error that induces is pe_scale * t * f * 2^-24 <= 6e-5 * f, so the high-frequency
    entries (f near 1) must agree exactly and no entry may be off by more than 1 ulp."""
    import math
    import numpy as np
    half = 32
    neg = np.float32(-(math.log(10000.0) / (half - 1)))
    libm = C.CDLL("libm.so.6")
    libm.expf.restype = C.c_float
    libm.expf.argtypes = [C.c_float]
    mine = np.array([libm.expf(float(np.float32(j) * neg)) for j in range(half)], dtype=np.float32)
    ref = torch.exp(torch.arange(half).float() * -(math.log(10000) / (half - 1))).numpy()
    ulp = np.abs(mine.view(np.int32) - ref.view(np.int32))
    assert ulp.max() <= 1
    assert np.array_equal(mine[:8], ref[:8])
    assert (1000.0 * np.abs(mine.astype(np.float64) - ref.astype(np.float64))).max() < 1e-6


def test_diffvc_module_and_c_abi_inventory():
    """DiffVC drop-in: 206 reference names/shapes, 117,794,599 parameters, same inventory through the C ABI."""
    from speech_backbones_b200.binding import Engine
    from speech_backbones_b200.diffvc import Diffusion
    from speech_backbones_b200.spec import DiffVCConfig, diffvc_param_spec, synthetic_diffvc_inputs
    cfg = DiffVCConfig()
    spec = diffvc_param_spec(cfg)
    m = Diffusion(80, 256, 128, True, 0.05, 20.0)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v) for k, v in spec.items()}
    assert m.nparams == 117_794_599
    e = Engine(80, 256, model="diffvc", dim_cond=128)
    assert e.weight_names() == list(spec)
    e.close()
    args = synthetic_diffvc_inputs(1, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(*args, n_timesteps=2, mode="pf")
    assert m(*args, n_timesteps=2, mode="nope") is args[0]
