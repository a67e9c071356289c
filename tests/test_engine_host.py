"""CPU: the strict weight loader every native engine shares (the U-Net for Grad-TTS and DiffVC, the HiFi-GAN vocoder, DiffVC's
PostNet, the text and mel encoders).  Name, rank and shape are checked before any CUDA call, and each error names the
engine's own C entry point."""
import ctypes as C
import re

import pytest


def _engine(kind):
    from speech_backbones_b200.binding import Engine
    from speech_backbones_b200.hifigan import VocoderEngine
    from speech_backbones_b200.postnet import PostNetEngine
    from speech_backbones_b200.spec import HIFIGAN_V1
    from speech_backbones_b200.text_encoder import MelEncoder, TextEncEngine, TextEncoder
    if kind == "gradtts":
        return Engine()
    if kind == "diffvc":
        return Engine(80, 256, model="diffvc", dim_cond=128)
    if kind == "vocoder":
        return VocoderEngine(HIFIGAN_V1, 0)
    if kind == "postnet":
        return PostNetEngine(128)
    if kind == "text":
        return TextEncEngine(TextEncoder(149, 80, 192, 768, 256, 2, 6, 3, 0.1, window_size=4), 0)
    return TextEncEngine(MelEncoder(80, 192, 768, 2, 6, 3, 0.1, window_size=4), 0, kind=1)


KINDS = ["gradtts", "diffvc", "vocoder", "postnet", "text", "mel"]


@pytest.fixture(params=KINDS)
def engine(request, sbk_lib):
    eng = _engine(request.param)
    yield eng
    eng.close()


def _set_weight(eng, name, shape):
    """<prefix>_set_weight with a one-float buffer: every call here is refused before the data is read"""
    dims = (C.c_int64 * len(shape))(*shape)
    rc = eng._fn("set_weight")(eng.h, name.encode(), (C.c_float * 1)(), dims, len(shape))
    return rc, eng.lib.sbk_last_error().decode()


def test_unexpected_key(engine):
    rc, msg = _set_weight(engine, "not_a_weight.weight", (3, 3))
    assert rc != 0
    assert msg.startswith(f"{engine.PREFIX}_set_weight: ") and "unexpected key 'not_a_weight.weight'" in msg


def test_wrong_rank_and_wrong_dim(engine):
    name = engine.weight_names()[0]
    results = [_set_weight(engine, name, (10 ** 9,) * r) for r in range(1, 6)]
    assert all(rc != 0 and msg.startswith(f"{engine.PREFIX}_set_weight: '{name}' ") and "expected" in msg
               for rc, msg in results)
    dims = [msg for _, msg in results if "dim 0 is 1000000000, expected" in msg]
    ranks = [msg for _, msg in results if re.search(r"rank \d, expected \d", msg)]
    assert len(dims) == 1 and len(ranks) == 4          # exactly one of the five ranks is the weight's own


def test_pack_with_a_key_missing(engine):
    rc = engine._fn("pack")(engine.h)
    msg = engine.lib.sbk_last_error().decode()
    assert rc != 0
    assert msg.startswith(f"{engine.PREFIX}_pack: ") and f"missing key '{engine.weight_names()[0]}' (strict)" in msg


def test_load_state_dict_names_the_missing_key(engine):
    name = engine.weight_names()[0]
    with pytest.raises(RuntimeError, match=re.escape(f"missing key '{name}' in {engine.STATE_DICT} (strict)")):
        engine.load_state_dict({})
