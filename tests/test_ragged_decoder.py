"""Ragged Grad-TTS batches without a GPU: the per-utterance reference golden, the C ABI's new entry points, and the host-side
refusals.

tests/golden/gradtts_ragged_golden.pt (scripts/make_golden_ragged_decoder.py) pins the unmodified reference's outputs for
each utterance of a B = 5, T = 512 batch with lengths {512, 301, 260, 130, 1}, computed ALONE at B = 1 and
T_b = fix_len_compatibility(lengths[b]) - what Grad-TTS/inference.py does - plus the reference's padded-batch estimator
output for the same inputs, each pinned by the SHA-256 of its fp32 bytes (and its shape and norm).  The oracle reproduces
every one of them bit for bit (test_oracle_reproduces_each_utterance), so its outputs stand for the reference's: the GPU
side (test_ragged_decoder_gpu.py) compares the engine's ragged rows with `oracle_outputs`."""
import hashlib
import os

import pytest
import torch

from helpers import rel_l2
from speech_backbones_b200 import UNetConfig, synthetic_inputs, synthetic_state_dict
from speech_backbones_b200.gradtts import fix_len_compatibility
from oracle import gradtts_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "gradtts_ragged_golden.pt"), weights_only=False)


def golden_inputs(g, n_spks):
    """the batch's z, mask, mu, spk: z / mu random on every frame (the padded ones too), mask from the lengths"""
    z, _, mu, spk, _ = synthetic_inputs(g["B"], g["T"], seed=g["seed"], n_spks=n_spks)
    L = torch.tensor(g["lengths"], dtype=torch.int64)
    mask = (torch.arange(g["T"])[None, :] < L[:, None]).to(torch.float32)[:, None, :]
    return z, mask, mu, spk, L


def utterance_noise(g, b, N):
    """the noise utterance b's stoc=True call drew: torch.manual_seed(noise_seed + b), then randn([1, 80, T_b]) per step"""
    torch.manual_seed(g["noise_seed"] + b)
    Tb = fix_len_compatibility(g["lengths"][b])
    return torch.stack([torch.randn(1, 80, Tb) for _ in range(N)])


def batch_noise(g, N):
    """[N, B, 80, T] whose [:, b, :, :T_b] is utterance b's noise; random past T_b (never read)"""
    noise = torch.randn(N, g["B"], 80, g["T"], generator=torch.Generator().manual_seed(11))
    for b in range(g["B"]):
        Tb = fix_len_compatibility(g["lengths"][b])
        noise[:, b, :, :Tb] = utterance_noise(g, b, N)[:, 0]
    return noise


def oracle_outputs(g, idx):
    """the oracle's outputs for golden case idx: each utterance alone ([80, T_b] per row), and for the padded-batch case
    also the batch call [B, 80, T] (None otherwise)"""
    c = g["cases"][idx]
    cfg = UNetConfig(n_spks=c["n_spks"])
    sd = synthetic_state_dict(cfg, g["seed"])
    z, mask, mu, spk, _ = golden_inputs(g, c["n_spks"])
    t = torch.tensor(g["t"])
    rows = []
    for b, n in enumerate(g["lengths"]):
        Tb = fix_len_compatibility(n)
        zb, mb, mub = z[b:b + 1, :, :Tb], mask[b:b + 1, :, :Tb], mu[b:b + 1, :, :Tb]
        sb = None if spk is None else spk[b:b + 1]
        if c["kind"] == "est":
            y = O.estimator(sd, cfg, zb * mb, mb, mub, t[b:b + 1], sb)
        else:
            noise = utterance_noise(g, b, c["N"]) if c["stoc"] else None
            y = O.reverse_diffusion(sd, cfg, zb, mb, mub, c["N"], c["stoc"], sb, noise)
        rows.append(y[0])
    padded = O.estimator(sd, cfg, z * mask, mask, mu, t, spk) if "padded" in c else None
    return rows, padded


def matches(t, pin):
    """t is bit for bit the output the golden pinned (SHA-256 of the fp32 bytes)"""
    t = t.detach().to(torch.float32).contiguous()
    return list(t.shape) == pin["shape"] and hashlib.sha256(t.numpy().tobytes()).hexdigest() == pin["sha256"]


@pytest.fixture(scope="module")
def golden():
    return load_golden()


@pytest.fixture(scope="module")
def oracle(golden):
    return [oracle_outputs(golden, i) for i in range(len(golden["cases"]))]


@pytest.mark.parametrize("idx", range(4))
def test_oracle_reproduces_each_utterance(golden, oracle, idx):
    c = golden["cases"][idx]
    rows, padded = oracle[idx]
    for b, (y, pin) in enumerate(zip(rows, c["rows"])):
        assert matches(y, pin), (idx, b, "norm", y.double().norm().item(), "golden", pin["norm"])
    if padded is not None:
        assert matches(padded, c["padded"]), (idx, "padded")


def test_padded_batch_is_not_the_per_utterance_call(golden, oracle):
    """Why lengths exist: in the padded batch the short utterances' GroupNorm statistics, attention softmax and conv borders
    see the padded frames, so their rows are not what the reference computes for them alone."""
    c = golden["cases"][0]
    assert c["kind"] == "est" and "padded" in c
    rows, padded = oracle[0]
    assert matches(padded, c["padded"])
    for b in range(1, golden["B"]):
        Tb = fix_len_compatibility(golden["lengths"][b])
        err = rel_l2(padded[b, :, :Tb], rows[b])
        print("utterance", b, "padded batch vs alone: rel-L2", err)
        assert err > 1e-2, b


def test_new_symbols_are_exported(sbk_lib):
    from speech_backbones_b200.binding import EXPORTS
    for name in ("sbk_estimator_lengths", "sbk_reverse_diffusion_lengths", "sbk_reverse_steps_lengths"):
        assert name in EXPORTS
        getattr(sbk_lib, name)


def test_null_handle_is_refused(sbk_lib):
    SBK_ERR_ARG = 1
    assert sbk_lib.sbk_estimator_lengths(None, None, None, None, None, None, None, None, 1, 4, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_reverse_diffusion_lengths(None, None, None, None, None, None, None, None, 1, 4, 1, 0, None) == SBK_ERR_ARG
    assert sbk_lib.sbk_reverse_steps_lengths(None, None, None, None, None, None, None, 1, 4, 1, 0, 1, 0, None) == SBK_ERR_ARG


def test_lengths_check_refuses_bad_input():
    """the shared check (binding.check_lengths, also the vocoder's) runs on the host before any launch"""
    from speech_backbones_b200.binding import check_lengths
    L = torch.tensor([4, 1, 3])
    assert torch.equal(check_lengths(L, 3, 4, L.device, "z"), L)
    for bad in (L.to(torch.int32), L[:2], torch.tensor([4, 0, 3]), torch.tensor([5, 1, 3]), [4, 1, 3]):
        with pytest.raises(ValueError):
            check_lengths(bad, 3, 4, L.device, "z")
