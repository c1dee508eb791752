"""Static per-step tables of the 50-step rectified-flow sampler.

Everything the reference recomputes on the host every step — and forces B+2 device syncs for
(sd3/rectified_flow.py:199,233) — is a pure function of the step index:

* ``t_i``            fp32 element i of ``torch.linspace(start, 0, steps+1)``     (rectified_flow.py:66-80)
* ``dt_i``           fp32 ``scheduled_t[i] - scheduled_t_prev[i]``               (rectified_flow.py:273-274,303)
* ``t_mapped_i``     ``long(scheduled_t[i] * 1000)`` — fp32 product, truncated   (rectified_flow.py:77,202)
* ``k_i``            ``DiTi_cont.to_indices(t_mapped_i)``                        (diti_utils.py:73-107)
* visible context    tokens ``0..k_i``  (``arange(K) <= k``; models_ours.py:345-353)
* adaLN positions    ``1000 + 8*k``                                              (diti_utils.py:109-110)

The tables are built by evaluating the same torch expressions the reference evaluates (not by
re-deriving constants), so the fp32 truncation quirk (459.99997 -> 459 ...) is reproduced exactly.
"""
from __future__ import annotations

import dataclasses
import math
from typing import Optional, Sequence, Tuple

import torch

TRADITION = 1000  # rectified_flow.py:28


class DiTiCont:
    """Token-index <-> diffusion-time map; restatement of DiTi_cont (diti_utils.py:84-110)."""

    def __init__(self, n_timesteps: int, K: int, stages: Sequence[int], k_per_stage: Sequence[int]):
        self.K = int(K)
        self.k_per_stage = [int(k) for k in k_per_stage]
        self.stages = [0] + [int(s) for s in stages]
        self.segments = []  # (low, slope, base)
        acc = 0
        for i in range(len(self.k_per_stage)):
            slope = float(self.k_per_stage[i]) / (self.stages[i + 1] - self.stages[i])
            self.segments.append((self.stages[i], slope, acc))
            acc += self.k_per_stage[i]

    def to_indices(self, t: torch.Tensor) -> torch.Tensor:
        # Segment.process (diti_utils.py:79-82): y[xp>=0] = (slope*xp).to(y.dtype)[xp>=0] + base
        ind = torch.zeros_like(t)
        for low, slope, base in self.segments:
            xp = t - low
            sel = xp >= 0
            ind[sel] = (slope * xp).to(ind.dtype)[sel] + base
        return ind.to(torch.long).clamp(0, self.K - 1)

    @staticmethod
    def get_position(k):
        return 1000 + (k * 8)


def timestep_embedding(t: torch.Tensor, dim: int = 256, max_period: int = 10000) -> torch.Tensor:
    """Sinusoidal features fed to every TimestepEmbedder MLP (sd3/mmdit.py:155-175, models.py:57-74).
    Evaluated on the host with the reference's own torch expression; the MLPs run on the device."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


@dataclasses.dataclass
class SamplerTables:
    steps: int
    t: torch.Tensor          # [steps] fp32, scheduled_t
    dt: torch.Tensor         # [steps] fp32, scheduled_t - scheduled_t_prev
    t_mapped: torch.Tensor   # [steps] int64
    k: torch.Tensor          # [steps] int64, last visible context index
    t_freq: torch.Tensor     # [steps,256] fp32: timestep_embedding(t*1000) for MMDiT.t_embedder (mmdit.py:1000,1022)
    pos_freq: torch.Tensor   # [K,256]   fp32: timestep_embedding(1000+8k) for pos-indexed adaLN (mmdit.py:446-458; modules.py:311-317)
    t_freq_uncond: Optional[torch.Tensor] = None   # [steps,256]: features of floor(1000 t).int().clamp(0,999) (MMDiT.cfg_inference, mmdit.py:1127)


def make_tables(K: int, stages: Sequence[int], k_per_stage: Sequence[int], steps: int = 50,
                start: float = 1.0) -> SamplerTables:
    base_t = torch.linspace(start, 0, steps + 1)                 # rectified_flow.py:67 ('uniform' schedule)
    scheduled_t = base_t[:-1]
    scheduled_t_prev = base_t[1:]
    timestep_map = scheduled_t * TRADITION                       # rectified_flow.py:77
    t_mapped = timestep_map.long()                               # rectified_flow.py:202 (.long() truncates)
    diti = DiTiCont(1000, K, stages, k_per_stage)
    k = diti.to_indices(t_mapped)
    # shift_t(t, 1.0) == t (rectified_flow.py:82-83,210); MMDiT multiplies by 1000 in fp32 (mmdit.py:1000)
    t_freq = timestep_embedding(scheduled_t * 1000.0)
    # get_position(torch.arange(K)) is int64 -> .float() inside timestep_embedding
    pos_freq = timestep_embedding(DiTiCont.get_position(torch.arange(K)))
    # the unconditional branch of the guided sampler embeds an INTEGER timestep (mmdit.py:1127): floor(t*1000).int().clamp(0,999)
    t_freq_uncond = timestep_embedding(torch.floor(scheduled_t * 1000).int().clamp(0, 999))
    return SamplerTables(steps=steps, t=scheduled_t.clone(), dt=(scheduled_t - scheduled_t_prev),
                         t_mapped=t_mapped, k=k, t_freq=t_freq, pos_freq=pos_freq, t_freq_uncond=t_freq_uncond)


def renderer_t_freq() -> torch.Tensor:
    """MMDiT_Renderer feeds t = 1000.0 straight into t_embedder (no extra *1000; mmdit.py:1523,1542)."""
    return timestep_embedding(torch.ones(1) * 1000.0)


def dense_flops_per_image_step(D: int, S_ctx: int, S_img: int, last_layer: bool) -> float:
    """2*MAC flops of one JointBlock for one image with S_ctx visible context rows (SURVEY 8d formula)."""
    S = S_ctx + S_img
    per_row = 2 * D * 3 * D + 2 * D * D + 16 * D * D            # qkv + proj + mlp (fc1+fc2 = 2*2*D*4D)
    attn = 4 * S * S * D
    f = S * per_row + attn
    if last_layer:                                              # pre_only context block: no proj / mlp
        f -= S_ctx * (2 * D * D + 16 * D * D)
    return float(f)


def decode_flops_per_image(K: int, stages, k_per_stage, steps: int, depth: int, n_img: int,
                           token_range: Optional[Tuple[int, int]] = None) -> Tuple[float, float]:
    """(masked-effective, dense-as-written) FLOPs of one image's `steps`-step decode (joint blocks only).

    token_range (lo, hi): (useful, executed) instead -- useful counts the image's visible tokens [lo, min(hi, k_i + 1)),
    executed the context stream a token-range call runs, [Lo, min(Hi, k_i + 1)) with the window rounded outward to 64 tokens
    (pass the batch's (min lo, max hi) for a mixed batch)."""
    tb = make_tables(K, stages, k_per_stage, steps)
    D = 64 * depth
    if token_range is not None:
        lo, hi = int(token_range[0]), int(token_range[1])
        Lo, Hi = lo // 64 * 64, min(K, (hi + 63) // 64 * 64)
    eff = dense = 0.0
    for i in range(steps):
        kc = int(tb.k[i]) + 1
        if token_range is None:
            rows_a, rows_b = kc, K
        else:
            rows_a, rows_b = max(0, min(hi, kc) - lo), max(0, min(Hi, kc) - Lo)
        for layer in range(depth):
            eff += dense_flops_per_image_step(D, rows_a, n_img, layer == depth - 1)
            dense += dense_flops_per_image_step(D, rows_b, n_img, layer == depth - 1)
    return eff, dense
