"""Rolling Grad-TTS batches: a fixed batch of slots keeps sampling while utterances join and leave it.

Each slot holds one request - the arguments of one B = 1 `Diffusion.forward` call - at its own step of its own
n_timesteps.  When a request finishes, its mel is read out and its slot freed, and the next queued request takes the slot
at the next step boundary.  A finished mel equals `Diffusion.forward` on that utterance alone (bit for bit in tf32 and
bf16, within fp32 rounding in fp32x3 and fp32), whatever the other slots hold and whenever it was admitted (sbk.h:
sbk_rolling_*).

The queue and the schedule live here, in Python.  The schedule is deterministic, so the host knows when each slot finishes
without reading the device: `advance` runs up to the next completion as one native call (one graph launch) and reads the
finished rows with stream-ordered copies.  The slot operations go through an engine object (binding.Engine; tests inject a
fake) with `rolling_reserve / rolling_admit / rolling_advance / rolling_read / rolling_release`, `n_feats`, `n_spks`,
`spk_emb_dim` and `torch_device`.
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
        engine.rolling_reserve(capacity, max_frames)

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

    def submit(self, z, mask, mu, n_timesteps, stoc=False, spk=None, noise=None) -> int:
        """Queue one utterance: the arguments of `Diffusion.forward(z, mask, mu, n_timesteps, stoc, spk)` at B = 1, with
        z, mu [1, n_feats, T_b] and mask [1, 1, T_b] (T_b a multiple of 4, at most max_frames).  stoc=True takes the
        per-step draws noise [n_timesteps, 1, n_feats, T_b]; None draws them here as `Diffusion.forward` would
        (torch.randn(z.shape) once per step, in step order).  Every argument is checked before anything is launched."""
        if not isinstance(z, torch.Tensor) or z.dim() != 3:
            raise ValueError(f"z: expected a [1, n_feats, T_b] tensor, got {getattr(z, 'shape', type(z).__name__)}")
        Tb = z.shape[-1]
        if Tb < 4 or Tb % 4 != 0 or Tb > self.max_frames:
            raise ValueError(f"T_b = {Tb}: must be a multiple of 4 in [4, {self.max_frames}] (fix_len_compatibility)")
        F = self.engine.n_feats
        z = self._tensor("z", z, (1, F, Tb))
        mask = self._tensor("mask", mask, (1, 1, Tb))
        mu = self._tensor("mu", mu, (1, F, Tb))
        if isinstance(n_timesteps, bool) or not isinstance(n_timesteps, int) or n_timesteps < 1:
            raise ValueError(f"n_timesteps must be an int >= 1, got {n_timesteps!r}")
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
        req = _Request(self._next_id, z, mask, mu, n_timesteps, bool(stoc), spk, noise, Tb)
        self._next_id += 1
        self.queue.append(req)
        self._admit()
        return req.rid

    def _admit(self):
        """FIFO: queued requests take the free slots, lowest slot first"""
        for b in range(self.capacity):
            if not self.queue:
                return
            if self.slots[b] is None:
                r = self.queue.popleft()
                self.engine.rolling_admit(b, r.z, r.mask, r.mu, r.n_timesteps, r.stoc, r.spk, r.noise)
                r.z = r.mask = r.mu = r.spk = None      # copied into the slot on the stream
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
                out[r.rid] = self.engine.rolling_read(b, r.frames)
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
