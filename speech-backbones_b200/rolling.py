"""Rolling Grad-TTS and DiffVC batches: a fixed batch of slots keeps sampling while utterances join and leave it.

Each slot holds one request - the arguments of one B = 1 `Diffusion.forward` call - at its own step of its own
n_timesteps.  When a request finishes, its mel is read out and its slot freed, and the next queued request takes the slot
at the next step boundary.  A finished mel equals `Diffusion.forward` on that utterance alone (bit for bit in tf32,
bf16 and fp16, within fp32 rounding in fp32x3 and fp32), whatever the other slots hold and whenever it was admitted (sbk.h:
sbk_rolling_*).

The queue and the schedule live here, in Python.  The schedule is deterministic, so the host knows when each slot finishes
without reading the device: `advance` runs up to the next completion as one native call (one graph launch) and reads the
finished rows with stream-ordered copies.  The slot operations go through an engine object (binding.Engine; tests inject a
fake) with `rolling_reserve / rolling_admit / rolling_advance / rolling_read / rolling_release`, `n_feats`, `n_spks`,
`spk_emb_dim` and `torch_device`.

`VcRollingSampler` is the same queue and schedule over a DiffVC engine (sbk.h: sbk_vc_rolling_*): a request is the arguments
of one B = 1 DiffVC `Diffusion.forward`, its conditioning table is computed at submission (`vc_conditioning` at B = 1, on
the request's own reference frames) and the slot folds row i_b of it at every step.  It overrides only what differs: the
request's checks, the reserve and the admission call.
"""
from __future__ import annotations

from collections import deque
from dataclasses import dataclass

import torch


@dataclass
class _Request:
    rid: int
    z: torch.Tensor
    mask: torch.Tensor
    mu: torch.Tensor
    n_timesteps: int
    stoc: bool
    spk: torch.Tensor | None
    noise: torch.Tensor | None      # kept alive here until the request's mel is read: the slot reads it every step
    frames: int                     # T_b
    done: int = 0                   # steps run


class RollingSampler:
    """A rolling batch of `capacity` slots at up to `max_frames` frames (a multiple of 4) on one Grad-TTS engine.

    submit(...) -> request id (queued while every slot is busy); advance(max_steps=None) -> {id: mel [1, n_feats, T_b]} of
    the requests that finished; drain() -> every remaining result.  Ids are 0, 1, 2, ... in submission order."""

    def __init__(self, engine, capacity: int, max_frames: int):
        if not isinstance(capacity, int) or capacity < 1:
            raise ValueError(f"capacity must be a positive int, got {capacity!r}")
        if not isinstance(max_frames, int) or max_frames < 4 or max_frames % 4 != 0:
            raise ValueError(f"max_frames must be a positive multiple of 4 (fix_len_compatibility), got {max_frames!r}")
        self.engine = engine
        self.capacity, self.max_frames = capacity, max_frames
        self.device = engine.torch_device
        self.slots: list[_Request | None] = [None] * capacity
        self.queue: deque[_Request] = deque()
        self.steps_run = 0                      # steps advanced since the sampler was made
        self._next_id = 0
        self._reserve()

    # ---- what a model's sampler overrides ---------------------------------------------------------------------------
    def _reserve(self):
        self.engine.rolling_reserve(self.capacity, self.max_frames)

    def _admit_into(self, b, r):
        self.engine.rolling_admit(b, r.z, r.mask, r.mu, r.n_timesteps, r.stoc, r.spk, r.noise)
        r.z = r.mask = r.mu = r.spk = None      # copied into the slot on the stream

    def _result(self, r, mel):
        """what advance() returns for a finished request"""
        return mel

    # ---- requests ---------------------------------------------------------------------------------------------------
    def _tensor(self, name, v, shape):
        if not isinstance(v, torch.Tensor):
            raise ValueError(f"{name}: expected a tensor, got {type(v).__name__}")
        if v.dtype != torch.float32:
            raise ValueError(f"{name}: expected float32, got {v.dtype}")
        if v.device != self.device:
            raise ValueError(f"{name} lives on {v.device}; the sampler runs on {self.device}")
        if tuple(v.shape) != shape:
            raise ValueError(f"{name} shape {tuple(v.shape)}: expected {list(shape)}")
        return v.contiguous()

    def _frames(self, z):
        """T_b of a request's z [1, n_feats, T_b]"""
        if not isinstance(z, torch.Tensor) or z.dim() != 3:
            raise ValueError(f"z: expected a [1, n_feats, T_b] tensor, got {getattr(z, 'shape', type(z).__name__)}")
        Tb = z.shape[-1]
        if Tb < 4 or Tb % 4 != 0 or Tb > self.max_frames:
            raise ValueError(f"T_b = {Tb}: must be a multiple of 4 in [4, {self.max_frames}] (fix_len_compatibility)")
        return Tb

    @staticmethod
    def _steps(n_timesteps):
        if isinstance(n_timesteps, bool) or not isinstance(n_timesteps, int) or n_timesteps < 1:
            raise ValueError(f"n_timesteps must be an int >= 1, got {n_timesteps!r}")
        return n_timesteps

    def _enqueue(self, req) -> int:
        self._next_id += 1
        self.queue.append(req)
        self._admit()
        return req.rid

    def submit(self, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None) -> int:
        """Queue one utterance: the arguments of `Diffusion.forward(z, mask, mu, n_timesteps, stoc, spk)` at B = 1, with
        z, mu [1, n_feats, T_b] and mask [1, 1, T_b] (T_b a multiple of 4, at most max_frames).  stoc=True takes the
        per-step draws noise [n_timesteps, 1, n_feats, T_b]; None draws them here as `Diffusion.forward` would
        (torch.randn(z.shape) once per step, in step order).  Every argument is checked before anything is launched."""
        Tb = self._frames(z)
        F = self.engine.n_feats
        z = self._tensor("z", z, (1, F, Tb))
        mask = self._tensor("mask", mask, (1, 1, Tb))
        mu = self._tensor("mu", mu, (1, F, Tb))
        self._steps(n_timesteps)
        if self.engine.n_spks > 1:
            if spk is None:
                raise ValueError("spk [1, spk_emb_dim] is required for a multi-speaker model")
            spk = self._tensor("spk", spk, (1, self.engine.spk_emb_dim))
        else:
            spk = None
        if stoc:
            if noise is None:
                noise = torch.stack([torch.randn(z.shape, dtype=z.dtype, device=z.device) for _ in range(n_timesteps)])
            noise = self._tensor("noise", noise, (n_timesteps, 1, F, Tb))
        else:
            noise = None
        return self._enqueue(_Request(self._next_id, z, mask, mu, n_timesteps, bool(stoc), spk, noise, Tb))

    def _admit(self):
        """FIFO: queued requests take the free slots, lowest slot first"""
        for b in range(self.capacity):
            if not self.queue:
                return
            if self.slots[b] is None:
                r = self.queue.popleft()
                self._admit_into(b, r)
                self.slots[b] = r

    # ---- running ----------------------------------------------------------------------------------------------------
    @property
    def busy(self) -> int:
        return sum(r is not None for r in self.slots)

    @property
    def pending(self) -> int:
        return len(self.queue)

    def next_completion(self) -> int:
        """Steps until the next busy slot finishes (0 when no slot is busy): the minimum of N_b - i_b"""
        left = [r.n_timesteps - r.done for r in self.slots if r is not None]
        return min(left) if left else 0

    def advance(self, max_steps: int | None = None) -> dict:
        """Run up to the next completion, or at most max_steps steps, in one native call; return {id: mel} of the
        requests that finished (their slots take queued requests before this returns)."""
        if max_steps is not None and (isinstance(max_steps, bool) or not isinstance(max_steps, int) or max_steps < 1):
            raise ValueError(f"max_steps must be an int >= 1 or None, got {max_steps!r}")
        self._admit()
        k = self.next_completion()
        if k == 0:
            return {}
        if max_steps is not None:
            k = min(k, max_steps)
        self.engine.rolling_advance(k)
        self.steps_run += k
        out = {}
        for b, r in enumerate(self.slots):
            if r is None:
                continue
            r.done += k
            if r.done == r.n_timesteps:
                out[r.rid] = self._result(r, self.engine.rolling_read(b, r.frames))
                self.engine.rolling_release(b)
                self.slots[b] = None
        self._admit()
        return out

    def drain(self) -> dict:
        """Advance until every submitted request has finished; {id: mel} of all of them not returned before"""
        out = {}
        while self.busy or self.queue:
            out.update(self.advance())
        return out


VC_MODES = ("pf", "em", "ml")


@dataclass
class _VcRequest:
    rid: int
    z: torch.Tensor
    mask: torch.Tensor
    mean: torch.Tensor
    cond: torch.Tensor              # [n_timesteps, 1, dim_cond]: copied into the slot's table at admission
    n_timesteps: int
    mode: str
    noise: torch.Tensor | None      # em / ml: kept alive here until the request's mel is read
    frames: int                     # T_b
    done: int = 0


class VcRollingSampler(RollingSampler):
    """A rolling batch of `capacity` slots at up to `max_frames` frames on one DiffVC engine (reached as
    `diffvc.Diffusion.rolling`).  The queue, schedule, `advance`, `drain`, `busy`, `pending` and `next_completion` are
    RollingSampler's.  A finished mel equals its row of an `Engine.vc_reverse_diffusion(..., lengths=)` call at (capacity,
    max_frames) bit for bit in every mode, and its own B = 1 `Diffusion.forward` where the two plans pick the same 3x3 tile
    layout (sbk.h: sbk_vc_rolling_*).  The engine also provides `vc_conditioning`, `vc_rolling_reserve / vc_rolling_admit`
    and `dim_cond`."""

    def _reserve(self):
        self.engine.vc_rolling_reserve(self.capacity, self.max_frames)

    def _admit_into(self, b, r):
        self.engine.vc_rolling_admit(b, r.z, r.mask, r.mean, r.cond, r.n_timesteps, r.mode, r.noise)
        r.z = r.mask = r.mean = r.cond = None   # copied into the slot on the stream

    def submit(self, z, mask, mean, ref, ref_mask, mean_ref, c, n_timesteps, mode, noise=None) -> int:
        """Queue one utterance: the arguments of DiffVC's `Diffusion.forward(z, mask, mean, ref, ref_mask, mean_ref, c,
        n_timesteps, mode)` at B = 1: z, mean [1, n_feats, T_b], mask [1, 1, T_b] (T_b a multiple of 4, at most max_frames),
        ref, mean_ref [1, n_feats, R], ref_mask [1, 1, R], c [1, 256], mode 'pf', 'em' or 'ml'.  For em / ml, noise
        [n_timesteps, 1, n_feats, T_b] holds the per-step draws; None draws them here as `Diffusion.forward` would
        (randn_like(z) once per step, in step order).  Every argument is checked before anything is launched; then the
        request's conditioning table is computed on its own reference frames (no draws)."""
        Tb = self._frames(z)
        F = self.engine.n_feats
        z = self._tensor("z", z, (1, F, Tb))
        mask = self._tensor("mask", mask, (1, 1, Tb))
        mean = self._tensor("mean", mean, (1, F, Tb))
        if not isinstance(ref, torch.Tensor) or ref.dim() != 3 or ref.shape[-1] < 1:
            raise ValueError(f"ref: expected a [1, n_feats, R] tensor, got {getattr(ref, 'shape', type(ref).__name__)}")
        R = ref.shape[-1]
        ref = self._tensor("ref", ref, (1, F, R))
        ref_mask = self._tensor("ref_mask", ref_mask, (1, 1, R))
        mean_ref = self._tensor("mean_ref", mean_ref, (1, F, R))
        c = self._tensor("c", c, (1, 256))
        N = self._steps(n_timesteps)
        if mode not in VC_MODES:
            raise ValueError(f"mode must be one of {list(VC_MODES)}, got {mode!r}")
        if mode != "pf" and noise is not None:
            noise = self._tensor("noise", noise, (N, 1, F, Tb))
        cond = self.engine.vc_conditioning(ref, ref_mask, mean_ref, c, N)
        if tuple(cond.shape) != (N, 1, self.engine.dim_cond):
            raise ValueError(f"cond shape {tuple(cond.shape)}: expected {[N, 1, self.engine.dim_cond]}")
        if mode == "pf":
            noise = None
        elif noise is None:             # the reference draws randn_like(z) once per step, in step order
            noise = torch.stack([torch.randn_like(z) for _ in range(N)])
        return self._enqueue(_VcRequest(self._next_id, z, mask, mean, cond, N, mode, noise, Tb))
