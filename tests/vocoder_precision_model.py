"""CPU operand-rounding MODEL of the HiFi-GAN vocoder's precision modes (test infrastructure, not product).

The vocoder counterpart of oracle/precision_model.py `operand_rounding`, built from its rounding primitives: it runs
oracle/hifigan_oracle.py with every tensor-core operand rounded where libsbk rounds it (csrc/sbk_vocoder.cu) and everything
else in fp32.

  tf32    weights round-to-nearest-away to tf32 (the packer); activations are fp32 in memory and the tensor core's tf32
          datapath truncates them;
  bf16    weights and the conv inputs (the LeakyReLU operands and the mel) round-to-nearest-even to bf16; the residual
          stream x, the transposed convs' GEMM output and the fold stay fp32;
  fp32x3  x*w = trunc_tf32(x) * rna_tf32(w) + f16(x_lo) * f16(w) + f16(x * 2^-12) * f16(w_lo * 2^12) (fp32x3_product: the
          three products are summed in float64, so the model isolates operand rounding from fp32 accumulation).

conv_post runs on CUDA cores in fp32 in every mode (k_voc_post), so it stays exact here.  A ConvTranspose1d's operand
rounding equals that of its GEMM (the fold only adds fp32 GEMM outputs).
"""
from __future__ import annotations

import contextlib

from oracle import hifigan_oracle as H
from oracle.precision_model import _Shim, fp32x3_product, round_bf16, round_tf32_rna, trunc_tf32

MODES = ("tf32", "bf16", "fp32x3")


@contextlib.contextmanager
def vocoder_operand_rounding(mode, p):
    """Patch hifigan_oracle's F.conv1d / F.conv_transpose1d so that generator(p, ...) runs with `mode` operand rounding.
    `p` is the state_dict the generator is called with (its conv_post weight identifies the exact CUDA-core conv)."""
    assert mode in MODES, mode
    F0 = H.F
    exact = id(p["conv_post.weight"])

    def op(f, x, w, b, *a, **k):
        if id(w) == exact:
            return f(x, w, b, *a, **k)
        if mode == "fp32x3":
            y = fp32x3_product(f, x, w, *a, **k)
            return y if b is None else y + b[None, :, None]
        if mode == "tf32":
            return f(trunc_tf32(x), round_tf32_rna(w), b, *a, **k)
        return f(round_bf16(x), round_bf16(w), b, *a, **k)

    H.F = _Shim(F0, conv1d=lambda x, w, b=None, *a, **k: op(F0.conv1d, x, w, b, *a, **k),
                conv_transpose1d=lambda x, w, b=None, *a, **k: op(F0.conv_transpose1d, x, w, b, *a, **k))
    try:
        yield
    finally:
        H.F = F0
