"""CPU ORACLE helper (test infrastructure, not product): an operand-rounding MODEL of the two tensor-core modes.

Runs oracle/gradtts_oracle.py with every tensor-core operand rounded where libsbk rounds it, everything else in fp32:

  tf32  conv / projection weights: round-to-nearest-away to 10 mantissa bits (host packers, cvt.rna);
        Block activations (the second conv's input): cvt.rna in k_gn_act; every other A operand (residual-stream
        tensors, the softmax numerators P and V in the context product) is fp32 in memory and the tensor core's tf32
        datapath drops the low 13 mantissa bits (truncation);
  bf16  weights and every stored operand tensor (Block activations, ResnetBlock / attention / resample outputs = the
        residual stream) round-to-nearest-even to bf16; P and V as in tf32.

  fp32x3  x*w = trunc_tf32(x) * rna_tf32(w)  +  fp16(x_lo) * fp16(w)  +  fp16(x * 2^-12) * fp16(w_lo * 2^12)  with
        x_lo = x - trunc_tf32(x), w_lo = w - rna_tf32(w) (sbk_internal.h: corr_chunk; the three products are summed in
        float64 here, so the model isolates the OPERAND roundings of the mode from fp32 accumulation effects).

It predicts the error of a precision mode from its rounding points alone, so tests can check that the error MEASURED on
the GPU (scripts/gpu_vs_precision_model.py) is explained by operand rounding and by nothing else.  It is a model, not a
bit-exact emulator: accumulation order, the folded attention matrix and the fast Mish are not modelled.
"""
from __future__ import annotations

import contextlib

import torch

from oracle import gradtts_oracle as O


def round_tf32_rna(x):
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32).reshape(x.shape)


def trunc_tf32(x):
    return (x.contiguous().view(torch.int32) & -0x2000).view(torch.float32).reshape(x.shape)


def round_bf16(x):
    return x.bfloat16().float()


def round_f16_sat(x):
    return x.clamp(-65504.0, 65504.0).half().float()


def fp32x3_product(op, x, w, *a, **k):
    """One conv / transposed conv in the fp32x3 mode's operand arithmetic (float64 sums): tf32 main + fp16 correction."""
    xh, wh = trunc_tf32(x), round_tf32_rna(w)
    xl, wl = x - xh, w - wh
    d = torch.float64
    y = (op(xh.to(d), wh.to(d), None, *a, **k)
         + op(round_f16_sat(xl).to(d), round_f16_sat(w).to(d), None, *a, **k)
         + op(round_f16_sat(x * 2.0 ** -12).to(d), round_f16_sat(wl * 2.0 ** 12).to(d), None, *a, **k))
    return y.float()


class _Shim:
    """forwards attribute access to `base` except for the overridden names"""

    def __init__(self, base, **over):
        self._base, self._over = base, over

    def __getattr__(self, name):
        over = object.__getattribute__(self, "_over")
        return over[name] if name in over else getattr(object.__getattribute__(self, "_base"), name)


@contextlib.contextmanager
def operand_rounding(mode, p):
    """Patch the oracle module so that estimator()/reverse_diffusion() run with `mode` ('tf32' | 'bf16') operand rounding.
    `p` is the state_dict (needed to recognise the second conv of each Block and the CUDA-core first conv)."""
    assert mode in ("tf32", "bf16", "fp32x3")
    x3 = mode == "fp32x3"
    rw = round_tf32_rna if mode == "tf32" else round_bf16
    act_ids = {id(v) for k, v in p.items() if k.endswith(".block2.block.0.weight")}
    exact_ids = {id(p["estimator.downs.0.0.block1.block.0.weight"]), id(p["estimator.final_conv.weight"])}
    exact_ids |= {id(v) for k, v in p.items() if k == "estimator.downs.0.0.res_conv.weight"}     # planar inputs: CUDA cores
    F0, T0 = O.F, O.torch

    def ra(x, w):
        if mode == "bf16":
            return round_bf16(x)
        return round_tf32_rna(x) if id(w) in act_ids else trunc_tf32(x)

    def conv2d(x, w, b=None, stride=1, padding=0, *a, **k):
        if id(w) in exact_ids:
            y = F0.conv2d(x, w, b, stride, padding, *a, **k)
        elif x3:
            y = fp32x3_product(F0.conv2d, x, w, stride, padding, *a, **k)
            y = y if b is None else y + b[None, :, None, None]
        else:
            y = F0.conv2d(ra(x, w), rw(w), b, stride, padding, *a, **k)
        return round_bf16(y) if (mode == "bf16" and stride == 2) else y        # Downsample output: a stored operand tensor

    def conv_transpose2d(x, w, b=None, stride=1, padding=0, *a, **k):
        if x3:
            y = fp32x3_product(F0.conv_transpose2d, x, w, stride, padding, *a, **k)
            return y if b is None else y + b[None, :, None, None]
        y = F0.conv_transpose2d(ra(x, w), rw(w), b, stride, padding, *a, **k)
        return round_bf16(y) if mode == "bf16" else y

    def einsum(eq, a, b):
        if eq == "bhdn,bhen->bhde" and x3:                                     # k_attn_kv_wg (fp32x3): P_hi V_hi + [P_lo V + P V_lo], fp16 chunks
            ah, bh = trunc_tf32(a), trunc_tf32(b)                              # scaled by exact powers of two (sbk_attn_x3.cu)
            d = T0.float64
            return (T0.einsum(eq, ah.to(d), bh.to(d))
                    + T0.einsum(eq, round_f16_sat((a - ah) * 256.0).to(d), round_f16_sat(b / 256.0).to(d))
                    + T0.einsum(eq, round_f16_sat(a / 16.0).to(d), round_f16_sat((b - bh) * 16.0).to(d))).float()
        if eq == "bhdn,bhen->bhde":                                            # context = P V^T on the tensor core (tf32, P from shared memory)
            return T0.einsum(eq, trunc_tf32(a), trunc_tf32(b))
        return T0.einsum(eq, a, b)

    res0, att0 = O.resnet, O.rezero_linear_attention

    def resnet(*a, **k):
        y = res0(*a, **k)
        return round_bf16(y) if mode == "bf16" else y

    def attention(*a, **k):
        y = att0(*a, **k)
        return round_bf16(y) if mode == "bf16" else y

    O.F = _Shim(F0, conv2d=conv2d, conv_transpose2d=conv_transpose2d)
    O.torch = _Shim(T0, einsum=einsum)
    O.resnet, O.rezero_linear_attention = resnet, attention
    try:
        yield
    finally:
        O.F, O.torch, O.resnet, O.rezero_linear_attention = F0, T0, res0, att0
