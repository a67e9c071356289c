"""Float64 op replay of one captured text-encoder or mel-encoder call (csrc/sbk_textenc.cu, sbk_textenc_debug_capture).

Every captured op is recomputed in float64 from the GPU's OWN captured inputs (never from the oracle's chain), with the
semantics of oracle/text_encoder_oracle.py, so each kernel is judged alone.  Each op gets a per-element bound B (absolute)
derived from the kernel's fp32 arithmetic, u = 2^-24 (round to nearest; the library builds without fast math: sqrtf and
`/` are correctly rounded, expf is within 2 ulp), first order in u throughout:

k_te_mask, k_te_embed, k_te_concat_spk: exact.  mask is (t < L_b); embed is one fp32 product emb[id] * fp32(sqrt C); the
  speaker concat copies.  All three must match bit for bit.

k_te_conv, the conv: acc = bias, then K*Ci FFMAs (zero taps included).  Each FFMA rounds once, its result bounded by the
  companion A = |b| + sum |x||w|, so |err| <= (K*Ci + 1) u A.  The inputs' x_mask multiply is exact (0 / 1).
  Epilogue: ReLU and the mask multiplies are exact (and 1-Lipschitz); the residual add rounds once more on |acc| + |r|:
  with A <- A + |r|, kappa = (K*Ci + 2) u.
  LayerNorm (eps 1e-4, biased variance, C channels) of y with an incoming error bound delta_c = kappa A_c:
    z_c = g_c r (y_c - m) + b_c,  r = (var + eps)^-1/2,  yh = (y - m) r
    propagated:  |dz_c| <= |g_c| r (delta_c + mean(delta) + |yh_c| mean(|yh| delta))     (d z / d y of the LayerNorm)
    own arithmetic, n = ceil(C/32) + 5 (a lane's sequential sum, then 5 shuffle adds):
      mean:  e_m <= (n + 1) u mean|y|;   variance: the e_m term cancels (sum (y - m) = 0), sum of squares (n + 2) u, / C,
      + eps: rel. (n + 4) u;  r = 1 / sqrtf(.): rho_r = (n + 4) u / 2 + 2 u  (+ |1e-4f - 1e-4| / (2 (var + eps)))
      (y - e_m - m) * r * g + b:  |g| r e_m + |g yh| (rho_r + 3 u) + u |z|.
  ReLU after the LayerNorm is 1-Lipschitz.

k_te_attn, per (utterance, head, query i), scale = 1/sqrt(d), w the window:
  scores s_ij = scale (q_i.k_j + [|j-i| <= w] q_i.E_k[j-i+w]), masked -> -1e4 (exact).  q.k runs as 4 FFMA chains of
  d/4 plus two adds, q.E_k as one chain of d, each then times fp32(1/sqrtf(d)) (2 u from the exact scale, 1 u rounding),
  and one add: |ds_ij| <= (d + 4) u S_ij with the companion S_ij = scale (|q_i|.|k_j| + [band] |q_i|.|E_k|).
  softmax: e_j = expf(s_j - mx), mx the fp32 max (a shift common to every e_j: it cancels); the subtraction rounds
  (u |s_j - mx|) and expf is within 2 ulp (4 u): e_j's relative error rho_j = |ds_ij| + u |s_j - mx| + 4 u.  Through the
  normalisation p_ij = e_j / Z this gives |dp_ij| <= p_ij (rho_j + sum_k p_ik rho_k).
  The sums: Z over T terms (ceil(T/32) - 1 + 5 adds of positives) and 1/Z (1 u); a = sum_j e_j v_j over T FFMAs and
  r = sum_band e_j E_v over at most 2w + 1, (a + r) and * (1/Z) one rounding each.  With PV_ic = sum_j p_ij |V_ijc|
  (V = v_j + [band] E_v[j-i+w]):
    |err_ic| <= sum_j p_ij rho_j |V_ijc| + (sum_k p_ik rho_k) PV_ic + (ceil(T/32) + 6 + T + 2w + 3) u PV_ic.
  The float64 replay runs over chunks of queries so T = 6272 fits in memory.

Check 1: max |got - ref| / B <= 1 over each utterance's own tokens (t < L_b).  Check 2 (op_replay.R_UNIFORM): the error
grouped as e_g = ||err_g|| / ||B_g||, and the largest e_g over the median of the other groups, for groups that match how the
kernels tile the work: each token (b, t) over its channels, the token phase t % 8 (k_te_conv's TE_TOK-token register
tile), the output-channel slot c // 256 (TE_MAXCO: a thread's three channels), and for attention also each head, the query
class (within w of either edge of the utterance, or interior) and the 32-channel lane pass of the p.V loop.  Tokens within
K // 2 of an utterance edge see zero taps (a different mix of rounding sources) and are left out of the token and phase
groups: check 1 judges them.  Rounding noise is spread evenly over these groups, so a defect in one phase of the tile, one
channel slot, one lane pass or the band edge stands out.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from op_replay import MIN_GROUP, R_UNIFORM, _max_over_median

U = 2.0 ** -24
LN_EPS = 1e-4
LN_EPS_F32 = float(np.float32(1e-4))
TE_TOK = 8                   # k_te_conv: tokens per CTA
TE_SLOT = 256                # k_te_conv: output channels c, c + 256, c + 512 per thread
LANES = 32                   # k_te_attn: channels of one p.V lane pass
ATTN_CHUNK = 1 << 22         # float64 elements of one [H, queries, T] score block


# ---- the ops in float64 ----------------------------------------------------------------------------------------------
def conv_tm(x, w, b):
    """Conv1d on token-major x [B, T, Ci] (zero padding K // 2) -> (ref, A) [B, T, Co]."""
    K = w.shape[2]
    xp = x.transpose(1, 2)
    ref = F.conv1d(xp, w, b, padding=K // 2).transpose(1, 2)
    A = (F.conv1d(xp.abs(), w.abs(), padding=K // 2) + b.abs()[:, None]).transpose(1, 2)
    return ref, A


def layer_norm_bound(y, delta, g, be):
    """LayerNorm over the last axis of the exact pre-LN values y, whose GPU value is within delta -> (z, bound)."""
    C = y.shape[-1]
    m = y.mean(-1, keepdim=True)
    dv = y - m
    ve = dv.pow(2).mean(-1, keepdim=True) + LN_EPS
    r = ve.rsqrt()
    yh = dv * r
    z = yh * g + be
    ag = g.abs()
    prop = ag * r * (delta + delta.mean(-1, keepdim=True) + yh.abs() * (yh.abs() * delta).mean(-1, keepdim=True))
    n = math.ceil(C / 32) + 5
    e_m = (n + 1) * U * y.abs().mean(-1, keepdim=True)
    rho_r = (n + 4) * U / 2 + 2 * U + abs(LN_EPS_F32 - LN_EPS) / (2 * ve)
    own = ag * r * e_m + (ag * yh.abs()) * (rho_r + 3 * U) + U * z.abs()
    return z, prop + own


def conv_op(x, w, b, mask, in_mask=False, relu1=False, mask1=False, res=None, res_mask=False, ln=None, relu2=False,
            mask2=False):
    """k_te_conv's fused op on its captured input (token-major float64) -> (ref, bound)."""
    m = mask[..., None]
    if in_mask:
        x = x * m
    ref, A = conv_tm(x, w, b)
    n_round = w.shape[1] * w.shape[2] + 1
    if relu1:
        ref = ref.clamp_min(0)
    if mask1:
        ref, A = ref * m, A * m
    if res is not None:
        r = res * m if res_mask else res
        ref, A = ref + r, A + r.abs()
        n_round += 1
    bound = n_round * U * A
    if ln is not None:
        ref, bound = layer_norm_bound(ref, bound, *ln)
    if relu2:
        ref = ref.clamp_min(0)
    if mask2:
        ref, bound = ref * m, bound * m
    return ref, bound


def _band(i0, i1, T, w, dev):
    """(band [n, T] bool, slot [n, T]) of queries i0..i1-1: |j - i| <= w and the E index j - i + w"""
    rel = torch.arange(T, device=dev)[None, :] - torch.arange(i0, i1, device=dev)[:, None]
    return rel.abs() <= w, (rel + w).clamp(0, 2 * w)


def _rel_sum(pw, slot, band, E):
    """sum_j pw[..., i, j] E[j - i + w] over the band: pw [H, n, T] -> [H, n, d]"""
    H, n, T = pw.shape
    wrel = torch.zeros(H, n, E.shape[0], dtype=pw.dtype, device=pw.device)
    wrel.scatter_add_(-1, slot.expand(H, n, T), torch.where(band, pw, torch.zeros((), dtype=pw.dtype, device=pw.device)))
    return wrel @ E


def attn_op(qkv, mask, ek, ev, H, w):
    """k_te_attn on its captured q|k|v (token-major float64 [B, T, 3C]) -> (ref, bound, PV) [B, T, C]."""
    B, T, C3 = qkv.shape
    C = C3 // 3
    d = C // H
    scale = 1.0 / math.sqrt(d)
    ref = torch.zeros(B, T, C, dtype=qkv.dtype, device=qkv.device)
    bound, pvs = torch.zeros_like(ref), torch.zeros_like(ref)
    n_sum = math.ceil(T / 32) + 6 + T + 2 * w + 3
    chunk = max(1, ATTN_CHUNK // (H * T))
    for b in range(B):
        q, k, v = (qkv[b, :, s * C:(s + 1) * C].reshape(T, H, d).transpose(0, 1) for s in range(3))    # [H, T, d]
        mk = mask[b]
        for i0 in range(0, T, chunk):
            i1 = min(T, i0 + chunk)
            qc = q[:, i0:i1]
            band, slot = _band(i0, i1, T, w, qkv.device)
            sl = slot.expand(H, i1 - i0, T)
            s = (qc @ k.transpose(1, 2) + torch.where(band, (qc @ ek.t()).gather(-1, sl), 0.0)) * scale
            S = (qc.abs() @ k.abs().transpose(1, 2) + torch.where(band, (qc.abs() @ ek.abs().t()).gather(-1, sl), 0.0)) * scale
            keep = (mk[i0:i1, None] * mk[None, :]) != 0
            s = torch.where(keep, s, torch.full((), -1e4, dtype=s.dtype, device=s.device))
            S = torch.where(keep, S, torch.zeros((), dtype=S.dtype, device=S.device))
            p = torch.softmax(s, -1)
            mx = s.amax(-1, keepdim=True)
            rho = (d + 4) * U * S + U * (s - mx).abs() + 4 * U
            out = p @ v + _rel_sum(p, slot, band, ev)
            pv = p @ v.abs() + _rel_sum(p, slot, band, ev.abs())
            prho = p * rho
            bd = prho @ v.abs() + _rel_sum(prho, slot, band, ev.abs()) + (prho.sum(-1, keepdim=True) + n_sum * U) * pv
            ref[b, i0:i1] = out.transpose(0, 1).reshape(i1 - i0, C)
            bound[b, i0:i1] = bd.transpose(0, 1).reshape(i1 - i0, C)
            pvs[b, i0:i1] = pv.transpose(0, 1).reshape(i1 - i0, C)
    return ref, bound, pvs


# ---- check 2 ---------------------------------------------------------------------------------------------------------
def token_groups(L, C, pad, head_dim=None, w=None):
    """{name: [L, C] integer group label, -1 = left out} for one utterance of L tokens and C channels"""
    t = torch.arange(L)[:, None].expand(L, C)
    c = torch.arange(C)[None, :].expand(L, C)
    inner = (t >= pad) & (t < L - pad)
    none = torch.full((L, C), -1, dtype=torch.long)
    g = {"tok": torch.where(inner, t, none), "phase": torch.where(inner, t % TE_TOK, none)}
    if C > TE_SLOT:
        g["slot"] = c // TE_SLOT
    if head_dim is not None:
        g["head"] = c // head_dim
        g["qclass"] = ((t < w) | (t >= L - w)).long()
        if head_dim > LANES:
            g["lane"] = (c % head_dim) // LANES
    return g


def uniformity_tok(err, B, groups, min_group=MIN_GROUP):
    """max over the groupings of  max_g e_g / median of the other groups' e_g,  e_g = ||err_g|| / ||B_g||"""
    worst, where = 0.0, ""
    e2, b2 = err.pow(2).flatten().cpu(), B.pow(2).flatten().cpu()
    for name, lab in groups.items():
        lab = lab.flatten()
        ok = lab >= 0
        if ok.sum() == 0:
            continue
        n = int(lab.max()) + 1
        cnt = torch.bincount(lab[ok], minlength=n)
        en = torch.bincount(lab[ok], e2[ok], minlength=n).sqrt()
        bn = torch.bincount(lab[ok], b2[ok], minlength=n).sqrt()
        use = (cnt >= min_group) & (bn > 0)
        if use.sum() < 2:
            continue
        r, i = _max_over_median(en[use] / bn[use])
        if r > worst:
            worst, where = r, f"{name}[{int(use.nonzero()[i])}]"
    return worst, where


# ---- the replay ------------------------------------------------------------------------------------------------------
def _bitwise(got, ref):
    return 0.0 if torch.equal(got, ref) else math.inf


class TextEncReplay:
    """Runs one text-encoder call (ids, lengths[, spk]) or mel-encoder call (mel, mel_mask, lengths = the mask's lengths)
    on `eng` (a TextEncEngine) with capture on, then replays every captured op in float64 on `dev`.  `run()` -> rows
    (name, elem, unif, where), one per op and utterance; `nonfinite` names captures with NaN / Inf inside an utterance."""

    def __init__(self, eng, sd, n_heads, window, lengths, ids=None, spk=None, mel=None, mel_mask=None, dev="cuda"):
        self.H, self.w, self.lengths, self.dev = n_heads, window, list(lengths), dev
        self.mel = mel is not None
        eng.debug_capture(True)
        try:
            if self.mel:
                self.out = eng.forward_mel(mel.cuda(), mel_mask.cuda())
            else:
                self.out = eng.forward(ids.cuda(), torch.as_tensor(lengths, dtype=torch.int64).cuda(),
                                       None if spk is None else spk.cuda())
            torch.cuda.synchronize()
        finally:
            eng.debug_capture(False)
        self.names = eng.debug_names()
        self.cap = {n: eng.debug_read(n) for n in self.names}
        self.p = {k: v.to(dev, torch.float64) for k, v in sd.items()}
        self.ids, self.spk, self.x_mel = ids, spk, mel
        B = len(self.lengths)
        T = self.cap["prenet.proj"].shape[1]
        self.B, self.T = B, T
        if self.mel:
            self.mask = mel_mask[:, 0].to(dev, torch.float64)
        else:
            self.mask = (torch.arange(T)[None, :] < torch.tensor(self.lengths)[:, None]).to(dev, torch.float64)
        self.nonfinite = []
        self.rows = []

    def g(self, name):
        return self.cap[name].to(self.dev, torch.float64)

    def _judge(self, name, got, ref, bound, pad=0, head_dim=None):
        """per utterance: check 1 and check 2 on its own tokens (token-major [B, T, C] tensors)"""
        err = (got - ref).abs()
        for b, L in enumerate(self.lengths):
            e, bd, gb = err[b, :L], bound[b, :L], got[b, :L]
            if not bool(torch.isfinite(gb).all()):
                self.nonfinite.append(f"{name} b={b}")
            elem = (e / (bd + torch.finfo(torch.float32).tiny)).max().item()
            unif, where = uniformity_tok(e, bd, token_groups(L, e.shape[1], pad, head_dim, self.w))
            self.rows.append((f"{name} b={b}", elem, unif, where))

    def _exact(self, name, got, ref):
        for b, L in enumerate(self.lengths):
            self.rows.append((f"{name} b={b}", _bitwise(got[b, :L], ref[b, :L]), 0.0, ""))

    def conv(self, name, x, wkey, bkey, **kw):
        ref, bound = conv_op(x, self.p[wkey], self.p[bkey], self.mask, **kw)
        K = self.p[wkey].shape[2]
        return ref, bound, K // 2

    def run(self):
        p, B, T = self.p, self.B, self.T
        if self.mel:
            x = self.x_mel.to(self.dev, torch.float64).transpose(1, 2)
            ref, bd, pad = self.conv("init_proj", x, "init_proj.weight", "init_proj.bias", in_mask=True)
            self._judge("init_proj", self.g("init_proj"), ref, bd, pad)
            h0 = self.g("init_proj")
        else:
            mask = self.cap["mask"][..., 0]
            want = (torch.arange(T)[None, :] < torch.tensor(self.lengths)[:, None]).float()
            self.rows.append(("mask", _bitwise(mask, want), 0.0, ""))
            emb = self.cap_weights_f32("emb.weight")
            C = emb.shape[1]
            ids = self.ids.clamp(0, emb.shape[0] - 1)
            want = emb[ids] * torch.tensor(math.sqrt(C), dtype=torch.float32)
            got = self.cap["embed"]
            self.rows.append(("embed", _bitwise(got, want), 0.0, ""))    # every token, padded ones included
            h0 = self.g("embed")
        cur = h0
        for i in range(3):
            ref, bd, pad = self.conv(f"prenet.{i}", cur, f"prenet.conv_layers.{i}.weight", f"prenet.conv_layers.{i}.bias",
                                     in_mask=True, ln=self.ln(f"prenet.norm_layers.{i}"), relu2=True)
            self._judge(f"prenet.{i}", self.g(f"prenet.{i}"), ref, bd, pad)
            cur = self.g(f"prenet.{i}")
        ref, bd, pad = self.conv("prenet.proj", cur, "prenet.proj.weight", "prenet.proj.bias", res=h0, mask2=True)
        self._judge("prenet.proj", self.g("prenet.proj"), ref, bd, pad)
        h = self.g("prenet.proj")
        if "spk_concat" in self.cap:
            got = self.cap["spk_concat"]
            want = torch.cat([self.cap["prenet.proj"], self.spk.float()[:, None, :].expand(B, T, -1)], -1)
            self._exact("spk_concat", got, want)
            h = self.g("spk_concat")
        Ce = h.shape[-1]
        li = 0
        while f"enc.{li}.qkv" in self.cap:
            a, q = f"encoder.attn_layers.{li}", f"enc.{li}"
            wqkv = torch.cat([p[f"{a}.conv_{s}.weight"] for s in "qkv"])
            bqkv = torch.cat([p[f"{a}.conv_{s}.bias"] for s in "qkv"])
            ref, bd = conv_op(h, wqkv, bqkv, self.mask, in_mask=True)
            self._judge(f"{q}.qkv", self.g(f"{q}.qkv"), ref, bd)
            ref, bd, _ = attn_op(self.g(f"{q}.qkv"), self.mask, p[f"{a}.emb_rel_k"][0], p[f"{a}.emb_rel_v"][0], self.H, self.w)
            self._judge(f"{q}.attn", self.g(f"{q}.attn"), ref, bd, head_dim=Ce // self.H)
            ref, bd, pad = self.conv(f"{q}.ln1", self.g(f"{q}.attn"), f"{a}.conv_o.weight", f"{a}.conv_o.bias", res=h,
                                     res_mask=True, ln=self.ln(f"encoder.norm_layers_1.{li}"))
            self._judge(f"{q}.ln1", self.g(f"{q}.ln1"), ref, bd, pad)
            f = f"encoder.ffn_layers.{li}"
            ln1 = self.g(f"{q}.ln1")
            ref, bd, pad = self.conv(f"{q}.ffn1", ln1, f"{f}.conv_1.weight", f"{f}.conv_1.bias", in_mask=True, relu1=True,
                                     mask1=True)
            self._judge(f"{q}.ffn1", self.g(f"{q}.ffn1"), ref, bd, pad)
            ref, bd, pad = self.conv(f"{q}.ln2", self.g(f"{q}.ffn1"), f"{f}.conv_2.weight", f"{f}.conv_2.bias", mask1=True,
                                     res=ln1, ln=self.ln(f"encoder.norm_layers_2.{li}"))
            self._judge(f"{q}.ln2", self.g(f"{q}.ln2"), ref, bd, pad)
            h = self.g(f"{q}.ln2")
            li += 1
        if self.mel:
            ref, bd, _ = self.conv("out", h, "term_proj.weight", "term_proj.bias", in_mask=True)
            self._judge("out", self.g("out").transpose(1, 2), ref, bd)
            return self.rows
        ref, bd, _ = self.conv("mu", h, "proj_m.weight", "proj_m.bias", in_mask=True, mask2=True)
        self._judge("mu", self.g("mu").transpose(1, 2), ref, bd)
        ref, bd, pad = self.conv("dp.1", h, "proj_w.conv_1.weight", "proj_w.conv_1.bias", in_mask=True, relu1=True,
                                 ln=self.ln("proj_w.norm_1"))
        self._judge("dp.1", self.g("dp.1"), ref, bd, pad)
        ref, bd, pad = self.conv("dp.2", self.g("dp.1"), "proj_w.conv_2.weight", "proj_w.conv_2.bias", in_mask=True,
                                 relu1=True, ln=self.ln("proj_w.norm_2"))
        self._judge("dp.2", self.g("dp.2"), ref, bd, pad)
        ref, bd, _ = self.conv("logw", self.g("dp.2"), "proj_w.proj.weight", "proj_w.proj.bias", in_mask=True, mask2=True)
        self._judge("logw", self.g("logw").transpose(1, 2), ref, bd)
        return self.rows

    def ln(self, pre):
        return self.p[f"{pre}.gamma"], self.p[f"{pre}.beta"]

    def cap_weights_f32(self, name):
        return self.p[name].float().cpu()


def passes(row):
    return row[1] <= 1.0 and row[2] <= R_UNIFORM
