"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/vae_odd128.npz by running the UNMODIFIED reference SDVAE (imported through
oracle/ref_loader.py, built and saved with the helpers of oracle/gen_golden.py) off the power-of-two grid:

* encoder   VAEEncoder at ch = 128 on two seeded 72 x 40 images: latent 9 x 5, so every downsampled level is ragged and the
            middle attention runs over T = 45 tokens
* decoder   VAEDecoder at ch = 128 on two seeded 9 x 5 latents

    python tests/golden/gen_vae_odd.py        # about 25 s on the CPU
"""
from __future__ import annotations

import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "oracle"))

import gen_golden as G  # noqa: E402
from selftoktokenizer_b200 import synth  # noqa: E402


def gen_vae_odd128():
    vae = G.ref_vae(128)
    x = synth.synth_tensor("golden.vae.x72x40", (2, 3, 72, 40), "emb", 0.5)
    z = synth.synth_tensor("golden.vae.z9x5", (2, 16, 9, 5), "emb", 1.0)
    with torch.no_grad():
        mom = vae.encoder(x)
        dec = vae.decoder(z)
    G.save("vae_odd128", dec=dec, moments=mom)


if __name__ == "__main__":
    gen_vae_odd128()
