"""CPU test helper: the operand-rounding model of the fp16 sampler mode (sbk.h SBK_PREC_F16).

The fp16 mode stores exactly what the bf16 mode stores, at the same points, in the same layout: the weights and every
stored operand tensor (Block activations, ResnetBlock / attention / resample outputs) are 16-bit, the raw conv outputs and
the attention's k, v, P, V fp32.  Only the 16-bit element differs: fp16 rounded to nearest even and saturated to +-65504
(cvt.rn.satfinite on the device; the host packers clamp first).  So its model is oracle/precision_model.py's bf16 model
with round_f16_sat in place of round_bf16, which `fp16_operand_rounding` runs by rebinding that one rounding primitive
for the duration of the context."""
from __future__ import annotations

import contextlib

from oracle import precision_model as P


@contextlib.contextmanager
def fp16_operand_rounding(p):
    """operand_rounding("bf16", p) with every bf16 rounding point rounding to fp16 (round_f16_sat) instead; `p` is the
    state_dict, as for operand_rounding.  The oracle module is restored on exit."""
    r16 = P.round_bf16
    P.round_bf16 = P.round_f16_sat            # read when the context is entered (weights) and at every rounding point
    try:
        with P.operand_rounding("bf16", p):
            yield
    finally:
        P.round_bf16 = r16


@contextlib.contextmanager
def operand_rounding(mode, p):
    """oracle/precision_model.operand_rounding, with the fp16 mode added"""
    with (fp16_operand_rounding(p) if mode == "fp16" else P.operand_rounding(mode, p)):
        yield
