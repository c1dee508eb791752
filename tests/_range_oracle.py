"""Token-range restatement of the oracle (test infrastructure): the decoder of oracle/selftok_oracle.py with one token window
per image, written the reference's way -- the dense K + N joint sequence and a boolean mask per image.

The reference's hooks this follows: p_sample_loop(..., super_mask=[B, K]) ANDs the window with the per-step `arange(K) <= k_i`
and uses the result as the conditional mask of the guided branch too (sd3/rectified_flow.py:182,227-231,281-288);
MMDiT_Renderer.forward(..., mask=[B, K]) takes the window as it is (sd3/mmdit.py:1529,1562-1614).  Ids outside an image's
window are never read (they are replaced by id 0 before the lookup), so they cannot change a result.
"""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F

import selftok_oracle as O
from selftoktokenizer_b200 import schedule as sched


def windows(ranges, B: int, K: int) -> torch.Tensor:
    """(lo, hi) pair or [B, 2] windows -> bool [B, K] (the reference's super_mask)."""
    r = torch.as_tensor(ranges, dtype=torch.long)
    if r.shape == (2,):
        r = r.expand(B, 2)
    pos = torch.arange(K)
    return (pos[None] >= r[:, :1]) & (pos[None] < r[:, 1:])


def lookup(sd, d, tokens: torch.Tensor, win: torch.Tensor) -> torch.Tensor:
    return O.lookup(sd, d, torch.where(win, tokens.long(), torch.zeros_like(tokens.long())))


def joint_blocks(sd, d, ctx, x, c, pos_freq, vis: torch.Tensor, ctx_sees_x: bool) -> torch.Tensor:
    """forward_core_with_concat (sd3/mmdit.py:918-933) with a per-image mask: vis [B, K] = visible context tokens of each image."""
    B, Kc, D = ctx.shape
    N = x.shape[1]
    key_ok = torch.cat([vis, torch.ones(B, N, dtype=torch.bool)], dim=1)                      # [B, S]
    ctx_row = key_ok.clone()
    if not ctx_sees_x:
        ctx_row[:, Kc:] = False
    mask = torch.cat([ctx_row[:, None].expand(B, Kc, -1), key_ok[:, None].expand(B, N, -1)], dim=1)[:, None]
    csil = F.silu(c)
    for j in range(d.dit_depth):
        last = j == d.dit_depth - 1
        pc, px = f"model.joint_blocks.{j}.context_block.", f"model.joint_blocks.{j}.x_block."
        if not last:
            cm = O._ctx_adaln(sd, pc, pos_freq)
            c_shift_msa, c_scale_msa, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = cm.chunk(6, dim=1)
            cin = O._ln(ctx) * (1 + c_scale_msa.unsqueeze(0)) + c_shift_msa.unsqueeze(0)
        else:
            c_shift, c_scale = O._lin(sd, pc + "adaLN_modulation.1", csil).chunk(2, dim=1)
            cin = O._ln(ctx) * (1 + c_scale.unsqueeze(1)) + c_shift.unsqueeze(1)
        xm = O._lin(sd, px + "adaLN_modulation.1", csil)
        x_shift_msa, x_scale_msa, x_gate_msa, x_shift_mlp, x_scale_mlp, x_gate_mlp = xm.chunk(6, dim=1)
        xin = O._ln(x) * (1 + x_scale_msa.unsqueeze(1)) + x_shift_msa.unsqueeze(1)
        cq, ck, cv = O._lin(sd, pc + "attn.qkv", cin).reshape(B, Kc, 3, D).unbind(2)
        xq, xk, xv = O._lin(sd, px + "attn.qkv", xin).reshape(B, N, 3, D).unbind(2)
        a = O._attention(torch.cat([cq, xq], 1), torch.cat([ck, xk], 1), torch.cat([cv, xv], 1), d.dit_heads, mask)
        c_attn, x_attn = a[:, :Kc], a[:, Kc:]
        if not last:
            ctx = ctx + c_gate_msa.unsqueeze(0) * O._lin(sd, pc + "attn.proj", c_attn)
            h = O._ln(ctx) * (1 + c_scale_mlp.unsqueeze(0)) + c_shift_mlp.unsqueeze(0)
            ctx = ctx + c_gate_mlp.unsqueeze(0) * O._lin(sd, pc + "mlp.fc2", O._gelu_tanh(O._lin(sd, pc + "mlp.fc1", h)))
        x = x + x_gate_msa.unsqueeze(1) * O._lin(sd, px + "attn.proj", x_attn)
        h = O._ln(x) * (1 + x_scale_mlp.unsqueeze(1)) + x_shift_mlp.unsqueeze(1)
        x = x + x_gate_mlp.unsqueeze(1) * O._lin(sd, px + "mlp.fc2", O._gelu_tanh(O._lin(sd, px + "mlp.fc1", h)))
    shift, scale = O._lin(sd, "model.final_layer.adaLN_modulation.1", csil).chunk(2, dim=1)
    x = O._ln(x) * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1)
    return O._lin(sd, "model.final_layer.linear", x)


def _x_embed(sd, d, x_lat):
    D, g = d.dit_hidden, d.latent // d.dit_patch
    w = sd["model.x_embedder.proj.weight"].reshape(D, -1)
    x = O._linear_impl(O._patchify(x_lat.float(), d.dit_patch), w, sd["model.x_embedder.proj.bias"])
    return x + O._center_crop_pos(sd["model.pos_embed"], d.dit_pos_max, g, g)


def decode(sd, d, tokens, noise, ranges, steps: int = 50, cfg_scale: float = 1.0) -> torch.Tensor:
    """p_sample_loop(..., super_mask = the windows), plain (cfg_scale 1) or guided (uncond_scale = cfg_scale)."""
    tb = sched.make_tables(d.K, d.stages, d.k_per_stage, steps)
    B = tokens.shape[0]
    win = windows(ranges, B, d.K)
    ctx0 = O.context_embed(sd, lookup(sd, d, tokens, win))
    x = noise.float().clone()
    for i in range(steps):
        vis = win & (torch.arange(d.K) <= int(tb.k[i]))[None]
        c = O._t_embed(sd, "model.t_embedder", tb.t_freq[i].reshape(1, -1)).expand(B, -1)
        if cfg_scale == 1.0:
            v = O._unpatchify(joint_blocks(sd, d, ctx0, _x_embed(sd, d, x), c, tb.pos_freq, vis, ctx_sees_x=True), d)
        else:
            v_c = O._unpatchify(joint_blocks(sd, d, ctx0, _x_embed(sd, d, x), c, tb.pos_freq, vis, ctx_sees_x=False), d)
            v_u = O.dit_velocity_uncond(sd, d, x, tb.t_freq_uncond[i])
            v = v_u + cfg_scale * (v_c - v_u)
        x = x - tb.dt[i] * v
    return x


def render(sd, d, tokens, ranges) -> torch.Tensor:
    """MMDiT_Renderer.forward(y=None, encoder_hidden_states=outs_q, mask = the windows)."""
    B = tokens.shape[0]
    win = windows(ranges, B, d.K)
    x = (sd["model.mask_token"].expand(B, d.n_img, -1) + sd["model.positional_embedding"]).contiguous()
    c = O._t_embed(sd, "model.t_embedder", sched.renderer_t_freq()).expand(B, -1)
    ctx = O.context_embed(sd, lookup(sd, d, tokens, win))
    pos_freq = sched.make_tables(d.K, d.stages, d.k_per_stage, 1).pos_freq
    return O._unpatchify(joint_blocks(sd, d, ctx, x, c, pos_freq, win, ctx_sees_x=False), d)
