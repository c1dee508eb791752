"""Per-call latent geometry on the CPU: the size-aware oracle (tests/_sizes_oracle.py) against the unmodified reference run at
several sizes on one model (tests/golden/tiny_sizes.npz, written by tests/golden/gen_sizes.py), the ABI surface of
selftok_set_latent_size, and the pipeline's size arithmetic."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sizes_oracle as SO  # noqa: E402
import selftok_oracle as O  # noqa: E402
from selftoktokenizer_b200 import capi, config as C, synth  # noqa: E402
from selftoktokenizer_b200.pipeline import latent_size  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sizes(g):
    return [tuple(int(v) for v in hw) for hw in g["sizes"]]


def _tag(hw):
    return f"{hw[0]}x{hw[1]}"


def test_size_oracle_pinned_to_reference(gold):
    g = gold("tiny_sizes")
    d, sd = C.TINY, synth.synth_state_dict(C.TINY)
    assert len(_sizes(g)) == 6 and (8, 8) in _sizes(g) and (6, 20) in _sizes(g)
    for hw in _sizes(g):
        x0 = synth.synth_tensor("golden.sizes.x0." + _tag(hw), (2, d.in_channels, *hw), "emb", 1.0)
        _, ids, _ = SO.encode(sd, d, x0)
        assert torch.equal(ids, torch.from_numpy(g["ids_" + _tag(hw)])), hw
        noise = torch.from_numpy(g["noise_" + _tag(hw)])
        err = float((SO.decode(sd, d, ids, noise) - torch.from_numpy(g["pred_" + _tag(hw)])).abs().max())
        assert err < 2e-5, (hw, err)
    hw = tuple(int(v) for v in g["guided_size"])
    ids = torch.from_numpy(g["ids_" + _tag(hw)])
    got = SO.decode_cfg(sd, d, ids, torch.from_numpy(g["noise_" + _tag(hw)]), float(g["cfg_scale"]))
    err = float((got - torch.from_numpy(g["pred_cfg_" + _tag(hw)])).abs().max())
    assert err < 2e-5, err


def test_size_oracle_is_the_oracle_at_the_default_size(gold):
    g = gold("tiny")
    d, sd = C.TINY, synth.synth_state_dict(C.TINY)
    tok, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    assert torch.equal(SO.decode(sd, d, tok, noise, steps=4), O.decode(sd, d, tok, noise, steps=4))
    # and the oracle's own grid helpers are back in place afterwards
    assert O._center_crop_pos.__module__ == O.__name__ and O._unpatchify.__module__ == O.__name__


def test_header_and_symbols_declare_the_setter():
    with open(os.path.join(REPO, "include", "selftok_b200.h")) as f:
        header = f.read()
    assert re.search(r"int selftok_set_latent_size\(selftok_handle_t h, int lat_h, int lat_w\);", header)
    assert "selftok_set_latent_size" in capi.SYMBOLS


@pytest.mark.parametrize("size, want", [(256, (32, 32)), ((512, 256), (64, 32)), ((128, 1024), (16, 128)), (16, (2, 2))])
def test_latent_size_of_good_sizes(size, want):
    assert latent_size(size, C.FULL, encode=True) == want


@pytest.mark.parametrize("size", [250, (256, 264), 0, (-16, 32), (1040, 256), "256", (256,), (256.0, 256)])
def test_latent_size_rejects_bad_sizes_on_encode(size):
    with pytest.raises(capi.SelftokError, match="multiples of 16|int or a pair"):
        latent_size(size, C.FULL, encode=True)


def test_latent_size_grids():
    # FULL: the encoder grid holds latents up to 128 (1024 px), the MMDiT's up to 384 (3072 px)
    assert latent_size(3072, C.FULL) == (384, 384)
    with pytest.raises(capi.SelftokError, match="at most 3072"):
        latent_size(3088, C.FULL)
    with pytest.raises(capi.SelftokError, match="at most 1024"):
        latent_size((1040, 512), C.FULL, encode=True)
    # TINY: the DiT's 12-patch grid holds 6 x 20 latents, not 6 x 26
    assert latent_size((48, 160), C.TINY) == (6, 20)
    with pytest.raises(capi.SelftokError, match="at most 192"):
        latent_size((48, 208), C.TINY)


def test_pipeline_noise_must_match_size():
    """SelftokPipeline._latent_hw without an engine or a device."""
    from selftoktokenizer_b200.pipeline import SelftokPipeline
    p = SelftokPipeline.__new__(SelftokPipeline)
    p.datasize, p.dims = 64, C.TINY
    assert p._latent_hw(None, None) == (8, 8)
    assert p._latent_hw((128, 64), torch.zeros(1, 16, 16, 8)) == (16, 8)
    with pytest.raises(capi.SelftokError, match="disagrees"):
        p._latent_hw((128, 64), torch.zeros(1, 16, 8, 16))
    with pytest.raises(capi.SelftokError, match="disagrees"):
        p._latent_hw(None, torch.zeros(1, 16, 12, 12))
    with pytest.raises(capi.SelftokError, match="multiples of 16"):
        p._latent_hw(72, None)
