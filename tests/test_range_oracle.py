"""Token ranges on the CPU: the window oracle (tests/_range_oracle.py) against the plain oracle, its independence of the ids
outside the window, and the FLOP model of token-range calls."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _range_oracle as RO  # noqa: E402
import selftok_oracle as O  # noqa: E402
from selftoktokenizer_b200 import config as C, schedule as S, synth  # noqa: E402


@pytest.fixture(scope="module")
def tiny():
    d = C.TINY
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny.npz"))
    return d, synth.synth_state_dict(d), torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])


def test_full_range_equals_plain_decode(tiny):
    d, sd, tok, noise = tiny
    ref = O.decode(sd, d, tok, noise, steps=50)
    got = RO.decode(sd, d, tok, noise, (0, d.K), steps=50)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-6)


def test_full_range_equals_plain_guided_decode(tiny):
    d, sd, tok, noise = tiny
    ref = O.decode_cfg(sd, d, tok, noise, 2.5, steps=50)
    got = RO.decode(sd, d, tok, noise, (0, d.K), steps=50, cfg_scale=2.5)
    torch.testing.assert_close(got, ref, rtol=0, atol=1e-6)


def test_full_range_equals_plain_render():
    import dataclasses
    d = dataclasses.replace(C.TINY, renderer=True)
    sd = synth.synth_state_dict(d)
    tok = torch.from_numpy(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_renderer.npz"))["tokens"])
    torch.testing.assert_close(RO.render(sd, d, tok, (0, d.K)), O.render(sd, d, tok), rtol=0, atol=1e-6)


def test_ids_outside_window_are_not_read(tiny):
    d, sd, tok, noise = tiny
    ranges = np.array([[0, 9], [20, 32], [5, 17]])
    a = RO.decode(sd, d, tok, noise, ranges, steps=8)
    win = RO.windows(ranges, tok.shape[0], d.K)
    for fill in (torch.full_like(tok, -1), torch.full_like(tok, d.codebook_size + 7), (tok * 7 + 3) % d.codebook_size):
        b = RO.decode(sd, d, torch.where(win, tok, fill), noise, ranges, steps=8)
        assert torch.equal(a, b)


def test_window_changes_the_result(tiny):
    """A strict sub-window is a different decode (the mask is really applied)."""
    d, sd, tok, noise = tiny
    a = RO.decode(sd, d, tok, noise, (0, d.K), steps=8)
    b = RO.decode(sd, d, tok, noise, (0, 4), steps=8)
    assert float((a - b).abs().max()) > 1e-3


def test_flop_model_full_range_unchanged():
    d = C.FULL
    args = (d.K, d.stages, d.k_per_stage, 50, d.dit_depth, d.n_img)
    eff, dense = S.decode_flops_per_image(*args)
    useful, executed = S.decode_flops_per_image(*args, token_range=(0, d.K))
    assert useful == eff and executed == eff and dense > eff
    # a suffix of n tokens computes less; its executed stream is the window rounded outward to 64 tokens
    u, x = S.decode_flops_per_image(*args, token_range=(d.K - 32, d.K))
    u2, x2 = S.decode_flops_per_image(*args, token_range=(d.K - 64, d.K))
    assert u < x == x2 and u < u2 < eff


# ---- pinned to the reference's own window hooks (tests/golden/gen_range.py: p_sample_loop(..., super_mask=...) and
# MMDiT_Renderer.forward(..., mask=...) of the unmodified reference)

def test_window_oracle_pinned_tiny(gold):
    g = gold("tiny_range")
    d, sd = C.TINY, synth.synth_state_dict(C.TINY)
    tok, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    err = float((RO.decode(sd, d, tok, noise, g["ranges"]) - torch.from_numpy(g["pred_x0"])).abs().max())
    assert err < 2e-5, err
    err = float((RO.decode(sd, d, tok, noise, g["cfg_ranges"], cfg_scale=float(g["cfg_scale"])) - torch.from_numpy(g["pred_x0_cfg"])).abs().max())
    assert err < 2e-5, err
    import dataclasses
    dr = dataclasses.replace(C.TINY, renderer=True)
    err = float((RO.render(synth.synth_state_dict(dr), dr, torch.from_numpy(g["renderer_tokens"]), g["ranges"])
                 - torch.from_numpy(g["renderer_pred_x0"])).abs().max())
    assert err < 2e-5, err


def test_window_oracle_pinned_mid(gold):
    g = gold("mid_range")
    d = C.MID
    err = float((RO.decode(synth.synth_state_dict(d), d, torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"]), g["ranges"])
                 - torch.from_numpy(g["pred_x0"])).abs().max())
    assert err < 2e-5, err
