"""The vocoder's op replay (tests/op_replay.py VocoderReplay) in the fp32x3 and bf16 precision modes.

`VocoderModeReplay` runs the same captured call and the same float64 replays as VocoderReplay and changes only what the
mode changes:

  fp32x3  kappa("fp32x3", K) with the Conv1d kernel's accumulation runs: 6 sub-stages of TAPS MMAs each (18, 42, 66
          MMAs; the GEMM's runs, 6 x 4 MMAs, are shorter than op_replay.X3_RUN).  Its Conv1d N tiles are at most 64 wide
          (conv_tc_ntile in FORM_X3), which the uniformity check groups by.
  bf16    the weights are replayed as the packer stores them (bf16, round to nearest even); the conv inputs are bf16 as
          captured (read back through sbk_vocoder_debug_op_layout).  An activated output (conv_pre, convs1) is stored as
          bf16: + EPS_STORE_BF16.  The bitwise ops (mel layout, LeakyReLU second outputs, the MRF mean before the last
          stage) reproduce the kernels' bf16 stores.
The bitwise ops that stay fp32 (the fold, the last MRF mean) and conv_post are judged as in tf32.
"""
from __future__ import annotations

import torch

from op_replay import EPS_ADD, VOC_SLOPE, VocoderReplay, _bitwise, kappa, lrelu_f32
from oracle.precision_model import round_bf16


def x3_run(taps):
    """MMAs per fp32x3 accumulation run of a Conv1d with `taps` taps (FLUSH = 6 sub-stages of one MMA per tap)"""
    return 6 * taps


class VocoderModeReplay(VocoderReplay):
    """VocoderReplay of an engine in precision `mode` ("fp32x3", "bf16"; "fp32" runs fp32x3, "tf32" is VocoderReplay)."""

    def __init__(self, eng, sd, h, mel, mode, dev="cuda"):
        super().__init__(eng, sd, h, mel, dev)
        self.mode = "fp32x3" if mode == "fp32" else mode
        assert self.mode in ("tf32", "fp32x3", "bf16"), mode
        if self.mode == "bf16":
            for k, v in sd.items():
                if k.endswith(".weight") and not k.startswith("conv_post"):
                    self.p[k] = round_bf16(v.float()).to(dev, torch.float64)

    def operand(self, t):
        """an operand tensor as its producer stores it in this mode"""
        return round_bf16(t.float()) if self.mode == "bf16" else t

    def conv_op(self, name):
        got, ref, A, _, floor, Alin, pad, nt = super().conv_op(name)
        if name == "conv_pre":
            w, act, addin = self.p["conv_pre.weight"], True, False
        else:
            _, n, grp, d = name.split(".")[:4]
            w, act, addin = self.p[f"resblocks.{n}.{grp}.{d}.weight"], grp == "convs1", grp == "convs2"
        # as VocoderReplay: bias add (+ residual add) + LeakyReLU's product, one fp32 rounding each
        k = kappa(self.mode, w.shape[1] * w.shape[2], extra=EPS_ADD * (1 + addin + act),
                  store_bf16=act and self.mode == "bf16", run=x3_run(w.shape[2]))
        return got, ref, A, k, floor, Alin, pad, (min(nt, 64) if self.mode == "fp32x3" else nt)

    def gemm_op(self, i):
        got, ref, A, _, floor, Alin, pad, nt = super().gemm_op(i)
        return got, ref, A, kappa(self.mode, self.p[f"ups.{i}.weight"].shape[0]), floor, Alin, pad, nt

    def fold_vs_convt(self, i):
        got, ref, A, _, floor, Alin, pad, nt = super().fold_vs_convt(i)
        return got, ref, A, kappa(self.mode, self.p[f"ups.{i}.weight"].shape[0], extra=2 * EPS_ADD), floor, Alin, pad, nt

    def _operand_ref(self, name):
        """the bit-exact reference of a bitwise op whose output is a conv operand, or None"""
        nu = len(self.h["upsample_rates"])
        parts = name.split(".")
        if name == "mel_in":
            return self.mel
        if parts[0] == "ups" and parts[2:] == ["a"]:
            return lrelu_f32(self.got(f"ups.{parts[1]}.x"), VOC_SLOPE)
        if parts[0] == "resblocks" and parts[2] == "convs2" and parts[4:] == ["a"]:
            return lrelu_f32(self.got(name[:-2] + ".x"), VOC_SLOPE)
        if parts[0] == "mrf" and int(parts[1]) + 1 < nu:
            i = int(parts[1])
            r = [self.got(f"resblocks.{3 * i + j}.convs2.2.x").float() for j in range(3)]
            inv = torch.tensor(1.0 / 3.0, dtype=torch.float32, device=r[0].device)
            return lrelu_f32(((r[0] + r[1]) + r[2]) * inv, VOC_SLOPE)
        return None

    def run(self):
        rows = super().run()
        if self.mode != "bf16":
            return rows
        out = []
        for row in rows:
            ref = self._operand_ref(row[0])
            out.append(row if ref is None else (row[0],) + _bitwise(self.got(row[0]), self.operand(ref)))
        return out
