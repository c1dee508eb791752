"""Continuous batching of the sampler: requests join a running batch at any step and leave when their own steps are done.

`ContinuousDecoder` keeps up to `max_batch` images in device state buffers.  Every `step()` admits waiting requests into free
slots (FIFO), runs ONE `Engine.decode_step` in which each image sits at its own schedule row, and retires the images that
finished.  Images are independent and the step entry is batch-invariant, so a request's result is bitwise what
`Engine.decode` / `Engine.decode_cfg` gives for it alone, whoever shares its steps.  One host thread drives a decoder.
"""
from __future__ import annotations

from collections import deque
from typing import Callable, List, Optional, Tuple

import numpy as np
import torch


class ContinuousDecoder:
    """Step-level batching over `engine` (a `capi.Engine`, or anything with its `dims`, `steps`, `device`, `tables.k` and
    `decode_step`).  guided: every request runs the guided sampler with its own `cfg_scale` (a decoder is all plain or all
    guided).  postprocess: applied to the stacked latents [n, C, l, l] retiring in one step (e.g. latents -> pixels)."""

    def __init__(self, engine, max_batch: int, *, guided: bool = False, postprocess: Optional[Callable] = None):
        if int(max_batch) < 1:
            raise ValueError(f"max_batch must be >= 1, got {max_batch}")
        d = engine.dims
        self.engine = engine
        self.max_batch = int(max_batch)
        self.guided = bool(guided)
        self.postprocess = postprocess
        self._lat = (d.in_channels, d.latent, d.latent)
        self._k = np.asarray(engine.tables.k, dtype=np.int64).reshape(-1)
        dev = torch.device(engine.device)
        self._tokens = torch.empty(self.max_batch, d.K, dtype=torch.int64, device=dev)
        self._x = torch.empty(self.max_batch, *self._lat, dtype=torch.float32, device=dev)
        self._step = np.zeros(self.max_batch, np.int32)       # next schedule row of every slot
        self._n = np.zeros(self.max_batch, np.int32)          # steps the slot's request runs
        self._range = np.zeros((self.max_batch, 2), np.int32)
        self._scale = np.zeros(self.max_batch, np.float32)
        self._rid: List[Optional[int]] = [None] * self.max_batch
        self._active = 0
        self._queue: deque = deque()
        self._next_id = 0

    @property
    def pending(self) -> int:
        """Requests submitted and not yet admitted."""
        return len(self._queue)

    @property
    def active(self) -> int:
        """Requests in the running batch."""
        return self._active

    def submit(self, ids, noise: Optional[torch.Tensor] = None, *, token_range=None, cfg_scale: Optional[float] = None,
               steps: Optional[int] = None) -> int:
        """Queue one image: ids [K] host int64; noise [1, C, l, l] (default: torch.randn on the CPU global generator, drawn
        now, as `decoding()` draws for one image); token_range (lo, hi) as in `Engine.decode`; steps = the first n schedule
        rows (default: all).  Raises ValueError for a bad request; nothing reaches the running batch then.  -> request id."""
        d = self.engine.dims
        ids = torch.as_tensor(ids)
        if ids.is_cuda or ids.shape != (d.K,) or ids.dtype not in (torch.int64, torch.int32):
            raise ValueError(f"submit: ids must be a host integer tensor [{d.K}], got {ids.dtype} {tuple(ids.shape)} "
                             f"on {ids.device}")
        n = int(self.engine.steps if steps is None else steps)
        if not 1 <= n <= self.engine.steps:
            raise ValueError(f"submit: steps must be in [1, {self.engine.steps}], got {n}")
        lo, hi = (0, d.K) if token_range is None else (int(v) for v in token_range)
        if not 0 <= lo < hi <= d.K:
            raise ValueError(f"submit: token_range ({lo}, {hi}) is not a window 0 <= lo < hi <= K = {d.K}")
        if self.guided:
            if cfg_scale is None:
                raise ValueError("submit: a guided decoder needs cfg_scale")
            k_last = int(self._k[:n].min())
            if lo > k_last:
                raise ValueError(f"submit: token_range ({lo}, {hi}) has no visible token at the last step (the guided sampler "
                                 f"needs lo <= k = {k_last})")
        elif cfg_scale is not None:
            raise ValueError("submit: cfg_scale on a plain decoder (build it with guided=True)")
        win = ids[lo:hi]
        if int(win.min()) < 0 or int(win.max()) >= d.codebook_size:
            raise ValueError(f"submit: token id outside [0, {d.codebook_size}) inside the window: min {int(win.min())}, "
                             f"max {int(win.max())}")
        if noise is None:
            noise = torch.randn(1, *self._lat)
        if tuple(noise.shape) not in ((1, *self._lat), self._lat):
            raise ValueError(f"submit: noise must be [1, {self._lat[0]}, {self._lat[1]}, {self._lat[2]}], got {tuple(noise.shape)}")
        rid = self._next_id
        self._next_id += 1
        self._queue.append((rid, ids.to(torch.int64), noise.reshape(self._lat).to(torch.float32), lo, hi,
                            0.0 if cfg_scale is None else float(cfg_scale), n))
        return rid

    def step(self) -> List[Tuple[int, torch.Tensor]]:
        """Admit, run one Euler step over the active images, retire -> [(request id, output [1, ...])] of the finished ones."""
        while self._queue and self._active < self.max_batch:
            rid, ids, noise, lo, hi, scale, n = self._queue.popleft()
            b = self._active
            self._tokens[b].copy_(ids)
            self._x[b].copy_(noise)
            self._step[b], self._n[b], self._range[b], self._scale[b], self._rid[b] = 0, n, (lo, hi), scale, rid
            self._active += 1
        a = self._active
        if a == 0:
            return []
        x = self._x[:a]
        self.engine.decode_step(self._tokens[:a], x, self._step[:a], token_range=self._range[:a],
                                cfg_scale=self._scale[:a] if self.guided else None, out=x)
        self._step[:a] += 1
        done = np.nonzero(self._step[:a] >= self._n[:a])[0]
        if done.size == 0:
            return []
        sel = torch.as_tensor(done, device=self._x.device)
        outs = self._x.index_select(0, sel)                    # a new tensor: the slots are reused below
        rids = [self._rid[i] for i in done]
        for i in done[::-1]:                                   # fill each hole with the last active row
            last = self._active - 1
            if i != last:
                self._tokens[i].copy_(self._tokens[last])
                self._x[i].copy_(self._x[last])
                self._step[i], self._n[i], self._range[i], self._scale[i] = (self._step[last], self._n[last], self._range[last],
                                                                             self._scale[last])
                self._rid[i] = self._rid[last]
            self._rid[last] = None
            self._active -= 1
        if self.postprocess is not None:
            outs = self.postprocess(outs)
        return [(rid, outs[j:j + 1]) for j, rid in enumerate(rids)]

    def drain(self) -> List[Tuple[int, torch.Tensor]]:
        """Step until no request is pending or active -> every result, in retirement order."""
        out: List[Tuple[int, torch.Tensor]] = []
        while self._queue or self._active:
            out += self.step()
        return out
