"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/tiny_sizes.npz by running the UNMODIFIED reference (imported through
oracle/ref_loader.py, driven with the helpers of oracle/gen_golden.py) at several latent sizes on ONE TINY ImageTokenizer: the
reference crops its positional grids from each input's own (h, w) (models_ours.py:183-214, sd3/mmdit.py:877-916,1001).

    python tests/golden/gen_sizes.py      # about 20 s on the CPU

For every size (h, w) of SIZES: two seeded encoder inputs -> ids and top-1 / top-2 margins (encoder + VQ), then
flow.p_sample_loop from seeded noise of that size with those ids (the pipeline's own sampler arguments, 50 steps).  For
GUIDED_SIZE also the guided sampler (uncond_scale = 2.5).  Keys: ids_{h}x{w}, margin_{h}x{w}, noise_{h}x{w},
pred_{h}x{w}, and pred_cfg_{h}x{w} for the guided size; the encoder inputs are regenerated from their synth names.
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
from selftoktokenizer_b200 import config as C, synth  # noqa: E402

# the default 8 x 8, larger squares, a smaller one, and two non-square sizes (20 / 2 = 10 <= the DiT's 12-patch grid)
SIZES = [(8, 8), (12, 12), (16, 16), (4, 4), (16, 8), (6, 20)]
GUIDED_SIZE = (16, 8)
CFG_SCALE = 2.5
B = 2


def tag(hw):
    return f"{hw[0]}x{hw[1]}"


def ref_sample(pipe, tokens, noise, uncond_scale=1.0):
    """The reference pipeline's own sampler call (SelftokPipeline.py:241-282), with uncond_scale for the guided run."""
    outs_q = G.lookup(pipe, tokens)
    k = pipe.diti.to_indices(torch.tensor([pipe.flow.timestep_map[0]] * tokens.shape[0]).long())
    enc_mask = pipe.model.encoder.get_encoder_mask(tokens, k)
    ehs = outs_q * enc_mask[..., None].expand_as(outs_q)
    model_kwargs = dict(encoder_hidden_states=ehs, mask=enc_mask, context_see_xt=True)
    with torch.no_grad():
        return pipe.flow.p_sample_loop(pipe.model.model, noise.shape, noise.clone(), model_kwargs=model_kwargs, start_t=pipe._steps,
                                       cond_vary=pipe.cond_vary, diti=pipe.diti, encoder=pipe.model.encoder, x_0=noise.float(),
                                       ori_hidden_states=outs_q, uncond_scale=uncond_scale)


def main():
    t0 = time.time()
    d = C.TINY
    pipe, _ = G.build(d, tag="tinysizes")
    out = {"sizes": np.array(SIZES, dtype=np.int32), "guided_size": np.array(GUIDED_SIZE, dtype=np.int32),
           "cfg_scale": np.float32(CFG_SCALE)}
    for hw in SIZES:
        x0 = synth.synth_tensor("golden.sizes.x0." + tag(hw), (B, d.in_channels, *hw), "emb", 1.0)
        _, ids, _, margin = G.ref_encode(pipe, x0)
        gen = torch.Generator().manual_seed(4321 + 100 * hw[0] + hw[1])
        noise = torch.randn(B, d.in_channels, *hw, generator=gen)
        out["ids_" + tag(hw)], out["margin_" + tag(hw)] = ids, margin
        out["noise_" + tag(hw)] = noise
        out["pred_" + tag(hw)] = ref_sample(pipe, ids, noise)
        if hw == GUIDED_SIZE:
            out["pred_cfg_" + tag(hw)] = ref_sample(pipe, ids, noise, CFG_SCALE)
        print(f"{tag(hw)}: min margin {float(margin.min()):.2e}", flush=True)
    G.save("tiny_sizes", **out)
    print(f"tiny_sizes: {time.time() - t0:.1f}s", flush=True)


if __name__ == "__main__":
    main()
