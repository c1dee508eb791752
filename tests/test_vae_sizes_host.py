"""The VAE restatement (oracle/vae_oracle.py) off the power-of-two grid, against the reference SDVAE (CPU only)."""
import numpy as np
import torch

from selftoktokenizer_b200 import synth


def test_vae_oracle_matches_reference_at_odd_sizes(gold):
    """SDVAE at ch = 128 on 72 x 40 images (latent 9 x 5: every downsampled level is ragged, the middle attention runs over
    T = 45 tokens) and on 9 x 5 latents: tests/golden/gen_vae_odd.py (vae_odd128)."""
    import vae_oracle as V
    g = gold("vae_odd128")
    sd = synth.synth_vae_state_dict(ch=128)
    x = synth.synth_tensor("golden.vae.x72x40", (2, 3, 72, 40), "emb", 0.5)
    z = synth.synth_tensor("golden.vae.z9x5", (2, 16, 9, 5), "emb", 1.0)
    with torch.no_grad():
        mom = V.encode_moments(sd, x).numpy()
        dec = V.decode(sd, z).numpy()
    assert mom.shape == (2, 32, 9, 5) and dec.shape == (2, 3, 72, 40)
    assert np.abs(mom - g["moments"]).max() < 5e-5
    assert np.abs(dec - g["dec"]).max() < 5e-5
