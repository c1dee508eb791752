"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/tiny_range.npz and mid_range.npz by running the UNMODIFIED reference
(imported through oracle/ref_loader.py, driven with the helpers of oracle/gen_golden.py) with its own token-window hooks:

* sampler      RectifiedFlow.p_sample_loop(..., super_mask=[B, K] bool) -- ANDed with the per-step `arange(K) <= k_i` mask
               (sd3/rectified_flow.py:182,227-231); with uncond_scale = 2.5 the same mask is the guided branch's conditional mask
               (:281-288)
* renderer     pipe.model.model(y=None, encoder_hidden_states=outs_q, mask=[B, K]) (MMDiT_Renderer.forward, sd3/mmdit.py:1529,1562-1614)

    python tests/golden/gen_range.py tiny     # 16 s on the CPU (tiny_range.npz: plain, guided and renderer runs)
    python tests/golden/gen_range.py mid      # 6 s on the CPU (mid_range.npz: B = 4, 50 steps)

tiny_range: the tokens / noise of tiny.npz plus a copy of image 0 (B = 4), windows = a prefix, a suffix that goes empty at late
steps, an interior window and [0, K) (plain sampler); windows whose lo <= k of the last step (guided sampler, uncond_scale 2.5);
the renderer on the tiny_renderer.npz tokens (plus a copy of image 0) with the plain sampler's windows.
mid_range: the tokens / noise of mid.npz (MID geometry, K = 128, B = 4), windows straddling the 64-row tiles.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "oracle"))

import gen_golden as G  # noqa: E402
from selftoktokenizer_b200 import config as C  # noqa: E402

TINY_RANGES = np.array([[0, 9], [20, 32], [5, 17], [0, 32]], dtype=np.int32)
TINY_CFG_RANGES = np.array([[0, 9], [1, 32], [0, 32], [1, 12]], dtype=np.int32)    # lo <= k of the last step (1)
MID_RANGES = np.array([[0, 1], [0, 70], [37, 101], [64, 128]], dtype=np.int32)


def _window(ranges, K):
    pos = torch.arange(K)
    r = torch.from_numpy(ranges).long()
    return (pos[None] >= r[:, :1]) & (pos[None] < r[:, 1:])


def ref_sample(pipe, tokens, noise, ranges, uncond_scale=1.0):
    """The reference pipeline's own sampler call (SelftokPipeline.py:241-282) plus super_mask (and uncond_scale)."""
    B = tokens.shape[0]
    outs_q = G.lookup(pipe, tokens)
    k = pipe.diti.to_indices(torch.tensor([pipe.flow.timestep_map[0]] * B).long())
    enc_mask = pipe.model.encoder.get_encoder_mask(tokens, k)
    ehs = outs_q * enc_mask[..., None].expand_as(outs_q)
    model_kwargs = dict(encoder_hidden_states=ehs, mask=enc_mask, context_see_xt=True)
    with torch.no_grad():
        return pipe.flow.p_sample_loop(pipe.model.model, noise.shape, noise.clone(), model_kwargs=model_kwargs, start_t=pipe._steps,
                                       cond_vary=pipe.cond_vary, diti=pipe.diti, encoder=pipe.model.encoder, x_0=noise.float(),
                                       ori_hidden_states=outs_q, uncond_scale=uncond_scale,
                                       super_mask=_window(ranges, tokens.shape[1]))


def gen_tiny():
    t0 = time.time()
    g = np.load(os.path.join(G.GOLD, "tiny.npz"))
    tokens = torch.from_numpy(g["tokens"])
    noise = torch.from_numpy(g["noise"])
    tokens, noise = torch.cat([tokens, tokens[:1]]), torch.cat([noise, noise[:1]])
    pipe, _ = G.build(C.TINY, tag="tinyrange")
    pred = ref_sample(pipe, tokens, noise, TINY_RANGES)
    pred_cfg = ref_sample(pipe, tokens, noise, TINY_CFG_RANGES, uncond_scale=2.5)
    rpipe, _ = G.build(G.TINY_R, tag="tinyrrange")
    rt = torch.from_numpy(np.load(os.path.join(G.GOLD, "tiny_renderer.npz"))["tokens"])
    rt = torch.cat([rt, rt[:1]])
    with torch.no_grad():
        rend, _ = rpipe.model.model(y=None, encoder_hidden_states=G.lookup(rpipe, rt), mask=_window(TINY_RANGES, rt.shape[1]))
    print(f"tiny_range: {time.time() - t0:.1f}s; window vs full-sequence decode of image 0: "
          f"{float((pred[0] - pred[3]).abs().max()):.3f}", flush=True)
    G.save("tiny_range", tokens=tokens, noise=noise, ranges=TINY_RANGES, pred_x0=pred, cfg_ranges=TINY_CFG_RANGES,
           cfg_scale=np.float32(2.5), pred_x0_cfg=pred_cfg, renderer_tokens=rt, renderer_pred_x0=rend)


def gen_mid():
    t0 = time.time()
    g = np.load(os.path.join(G.GOLD, "mid.npz"))
    tokens, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    G.ref_loader.import_reference()
    enc_name, dit_name = G.ref_loader.register_geometry(C.MID, "midrange")
    pipe = G.ref_loader.build_reference_pipeline(G.ref_loader.dims_to_cfg(C.MID, enc_name, dit_name), G.synth.synth_state_dict(C.MID))
    pred = ref_sample(pipe, tokens, noise, MID_RANGES)
    print(f"mid_range: {time.time() - t0:.1f}s", flush=True)
    G.save("mid_range", tokens=tokens, noise=noise, ranges=MID_RANGES, pred_x0=pred)


if __name__ == "__main__":
    for what in sys.argv[1:] or ["tiny", "mid"]:
        {"tiny": gen_tiny, "mid": gen_mid}[what]()
