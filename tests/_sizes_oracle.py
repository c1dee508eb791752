"""TEST INFRASTRUCTURE ONLY -- the CPU oracle (oracle/selftok_oracle.py) at any latent geometry (h, w).

The oracle reads its positional crop and unpatchify grid from `d.latent` (square); every other step already follows the input
tensor's shape.  Here both take the grid from the input's own (h, w), as the reference does on every call (cropped_pos_embed,
models_ours.py:183-214 and sd3/mmdit.py:877-916,1001; unpatchify(x, hw)).  The oracle module itself is not modified: its two
grid helpers are swapped for the length of one call, the way the precision studies swap its linear.  At h = w = d.latent
the results are the oracle's own, bit for bit.
"""
from __future__ import annotations

import contextlib

import torch

import selftok_oracle as O


@contextlib.contextmanager
def _grid(d, h: int, w: int):
    crop, unpatchify = O._center_crop_pos, O._unpatchify

    def crop_hw(pos, max_size, gh, gw):
        p = d.enc_patch if max_size == d.enc_pos_max else d.dit_patch
        return crop(pos, max_size, h // p, w // p)

    def unpatchify_hw(x, dd):
        p, c = dd.dit_patch, dd.in_channels
        x = x.reshape(x.shape[0], h // p, w // p, p, p, c)
        return torch.einsum("nhwpqc->nchpwq", x).reshape(x.shape[0], c, h, w)

    O._center_crop_pos, O._unpatchify = crop_hw, unpatchify_hw
    try:
        yield
    finally:
        O._center_crop_pos, O._unpatchify = crop, unpatchify


def encode(sd, d, x0: torch.Tensor, tables=None):
    """O.encode at x0's latent geometry -> (outs_q, ids, z)."""
    with _grid(d, x0.shape[2], x0.shape[3]):
        return O.encode(sd, d, x0, tables)


def decode(sd, d, tokens: torch.Tensor, noise: torch.Tensor, steps: int = 50) -> torch.Tensor:
    """O.decode at noise's latent geometry."""
    with _grid(d, noise.shape[2], noise.shape[3]):
        return O.decode(sd, d, tokens, noise, steps=steps)


def decode_cfg(sd, d, tokens: torch.Tensor, noise: torch.Tensor, cfg_scale: float, steps: int = 50) -> torch.Tensor:
    """O.decode_cfg at noise's latent geometry."""
    with _grid(d, noise.shape[2], noise.shape[3]):
        return O.decode_cfg(sd, d, tokens, noise, cfg_scale, steps=steps)
