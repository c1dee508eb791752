"""One engine, every image size: per-call latent geometry (selftok_set_latent_size, `latent_hw=`, `size=`) on the device.

* a handle at latent_hw = G is bitwise a handle created at latent = G, on every hot-path entry, with and without graphs;
* interleaved sizes never reuse a stale graph, crop or workspace carve;
* the unmodified reference at several sizes on one model (tests/golden/tiny_sizes.npz);
* the full geometry and the pixel API at sizes other than the engine's own;
* every size error is raised before any launch and leaves the geometry as it was.
"""
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sizes_oracle as SO  # noqa: E402
from selftoktokenizer_b200 import config as C, synth  # noqa: E402
from selftoktokenizer_b200.capi import Engine, SelftokError  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"bf16x3": 1e-3, "fp16": 1e-3}          # tests/test_parity_gpu.py: max-abs on 50-step latents
# tests/test_parity_gpu.py's ragged geometry (K = 40, 6 x 6 image tokens)
RAGGED = dataclasses.replace(C.TINY, K=40, k_per_stage=(14, 10, 8, 5, 3), latent=12, enc_pos_max=24, dit_pos_max=10, enc_depth=1,
                             dit_depth=2, codebook_size=2040)
GEOMS = {"tiny": C.TINY, "mid": C.MID, "ragged": RAGGED}


def _square_sizes(d):
    """Every square latent side both positional grids hold, from a 2 x 2 patch grid up."""
    top = min(d.enc_pos_max * d.enc_patch, d.dit_pos_max * d.dit_patch)
    return list(range(2 * d.dit_patch, top + 1, d.dit_patch))


def _inputs(d, hw, B):
    x0 = synth.synth_tensor(f"sizes.x0.{hw[0]}x{hw[1]}", (B, d.in_channels, *hw), "emb", 1.0).to(DEV)
    noise = synth.synth_tensor(f"sizes.noise.{hw[0]}x{hw[1]}", (B, d.in_channels, *hw), "emb", 1.0).to(DEV)
    return x0, noise


def _all_entries(eng, d, hw, B, latent_hw):
    """Every hot-path entry at latent geometry hw; latent_hw=None for a dedicated engine of that size."""
    x0, noise = _inputs(d, hw, B)
    K = d.K
    ids, outs_q, _ = eng.encode(x0, return_aux=True, latent_hw=latent_hw)
    ranges = np.array([[0, K // 3], [K // 4, K], [0, K], [5, K - 3]][:B], dtype=np.int32)
    steps = np.array([0, 17, 49, 30][:B], dtype=np.int32)
    r = {"ids": ids, "outs_q": outs_q,
         "decode": eng.decode(ids, noise, latent_hw=latent_hw),
         "decode_cfg": eng.decode_cfg(ids, noise, 2.5, latent_hw=latent_hw),
         "decode_range": eng.decode(ids, noise, token_range=ranges, latent_hw=latent_hw),
         "decode_step": eng.decode_step(ids, noise, steps, token_range=ranges, latent_hw=latent_hw),
         "decode_step_cfg": eng.decode_step(ids, noise, steps, cfg_scale=2.5, latent_hw=latent_hw),
         "dit_velocity": eng.dit_velocity(ids, noise, 30, latent_hw=latent_hw)}
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in r.items()}


def _assert_same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), f"{what}: {k} differs"


@pytest.mark.parametrize("geom,precision", [("tiny", "fp16"), ("tiny", "bf16x3"), ("tiny", "fp8"), ("mid", "fp16"), ("mid", "bf16x3"),
                                            ("ragged", "fp16"), ("ragged", "bf16x3")])
def test_one_engine_equals_dedicated_engines(geom, precision):
    d = GEOMS[geom]
    sd = synth.synth_state_dict(d, seed=3)
    B = 3
    one = Engine(d, sd, device=DEV, precision=precision)
    for G in _square_sizes(d):
        own = Engine(dataclasses.replace(d, latent=G), sd, device=DEV, precision=precision)
        for graphs in (True, False):
            one.set_use_graph(graphs)
            own.set_use_graph(graphs)
            want = _all_entries(own, d, (G, G), B, None)
            got = _all_entries(one, d, (G, G), B, (G, G))
            _assert_same(got, want, f"{geom} {precision} latent {G} graphs={graphs}")
        own.close()
    one.close()


def test_interleaved_sizes_reuse_nothing_stale():
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="fp16")
    a, b, c = (8, 8), (16, 16), (4, 6)
    first = _all_entries(eng, d, a, 2, None)
    x0, noise = _inputs(d, a, 2)
    eng.decode(first["ids"], noise)
    launches = eng.last_launch_count
    ws0 = eng.workspace_bytes(2, "decode")
    for hw, B in ((b, 2), (a, 2), (c, 3), (a, 2), (b, 4), (a, 2)):    # b after a, and a larger batch: the workspace regrows
        r = _all_entries(eng, d, hw, B, hw)
        if hw == a:
            _assert_same(r, first, f"size {a} after {eng.latent_hw}")
    assert eng.latent_hw == a
    eng.decode(first["ids"], noise)
    assert eng.last_launch_count == launches
    eng.set_latent_size(*b)
    assert eng.workspace_bytes(2, "decode") > ws0
    eng.set_latent_size(*a)
    assert eng.workspace_bytes(2, "decode") == ws0
    eng.close()


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
def test_sizes_against_reference_fixture(precision, gold):
    g = gold("tiny_sizes")
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision=precision)
    for hw in (tuple(int(v) for v in s) for s in g["sizes"]):
        tag = f"{hw[0]}x{hw[1]}"
        x0 = synth.synth_tensor("golden.sizes.x0." + tag, (2, d.in_channels, *hw), "emb", 1.0)
        ids = eng.encode(x0, latent_hw=hw).cpu()
        assert torch.equal(ids, torch.from_numpy(g["ids_" + tag])), f"{tag}: ids differ from the reference"
        noise = torch.from_numpy(g["noise_" + tag])
        err = float((eng.decode(ids, noise, latent_hw=hw).cpu() - torch.from_numpy(g["pred_" + tag])).abs().max())
        print(f"[{precision}] {tag}: 50-step latents max-abs err vs reference {err:.3e}")
        assert err < TOL[precision], tag
        if "pred_cfg_" + tag in g.files:
            got = eng.decode_cfg(ids, noise, float(g["cfg_scale"]), latent_hw=hw).cpu()
            err = float((got - torch.from_numpy(g["pred_cfg_" + tag])).abs().max())
            print(f"[{precision}] {tag}: guided 50-step latents max-abs err vs reference {err:.3e}")
            assert err < TOL[precision], tag
    eng.close()


def test_full_geometry_one_engine_serves_every_size():
    d = C.FULL
    sd = synth.synth_state_dict(d, device=DEV)
    B = 2
    one = Engine(d, sd, device=DEV, precision="fp16")
    got = {}
    for G in (16, 48, 64):
        x0, noise = _inputs(d, (G, G), B)
        ids = one.encode(x0, latent_hw=(G, G))
        got[G] = (ids, one.decode(ids, noise, latent_hw=(G, G)))
    base = one.device_bytes
    dedicated = 0
    for G in (16, 48, 64):
        own = Engine(dataclasses.replace(d, latent=G), sd, device=DEV, precision="fp16")
        x0, noise = _inputs(d, (G, G), B)
        ids = own.encode(x0)
        assert torch.equal(ids, got[G][0]), f"latent {G}: ids"
        assert torch.equal(own.decode(ids, noise), got[G][1]), f"latent {G}: decode"
        dedicated += own.device_bytes
        own.close()
    print(f"device bytes: one engine serving 256^2 + 128^2, 384^2, 512^2: {base / 2**30:.2f} GiB; "
          f"three dedicated engines: {dedicated / 2**30:.2f} GiB")
    # 512 x 256 pixels (non-square): ids against the oracle's encode at that geometry
    x0 = synth.synth_tensor("sizes.x0.64x32", (1, d.in_channels, 64, 32), "emb", 1.0)
    ids = one.encode(x0, latent_hw=(64, 32)).cpu()
    sd_cpu = {k: v.cpu() for k, v in sd.items()}
    _, ids_ref, _ = SO.encode(sd_cpu, d, x0)
    assert torch.equal(ids, ids_ref)
    one.close()


class _NoFallback:
    def encode(self, *a, **k):
        raise AssertionError("encoder_vae was called: the device VAE should have encoded these images")


def test_pixel_api_at_other_sizes():
    from selftoktokenizer_b200 import SelftokPipeline
    from selftoktokenizer_b200.pipeline import DeviceVAE, SD3LatentFormat
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = C.parse_args_from_yaml(os.path.join(root, "configs/selftok_256_512tok.yml"))
    vae_sd = synth.synth_vae_state_dict(ch=128)
    dvae = DeviceVAE(vae_sd, DEV, encoder_vae=_NoFallback())
    sd = synth.synth_state_dict(C.SelftokDims.from_cfg(cfg, 256), device=DEV)

    def pipeline(ds):
        return SelftokPipeline(cfg=cfg, ckpt_path=None, sd3_path=None, datasize=ds, dtype=torch.float32, device=DEV,
                               state_dict=sd, vae=dvae, precision="fp16")
    p256, p384 = pipeline(256), pipeline(384)
    sq = synth.synth_tensor("sizes.pixels.384", (2, 3, 384, 384), "emb", 0.5).to(DEV)
    tok = p256.encoding(sq, DEV)
    assert torch.equal(tok, p384.encoding(sq, DEV))
    wide = synth.synth_tensor("sizes.pixels.384x640", (2, 3, 384, 640), "emb", 0.5).to(DEV)
    with torch.no_grad():
        exp = p256.engine.encode(SD3LatentFormat().process_in(dvae.decoder.encode(wide)).to(torch.float32), latent_hw=(48, 80))
    assert torch.equal(p256.encoding(wide, DEV), exp)
    idx = tok.cpu().numpy()
    torch.manual_seed(11)
    out = p256.decoding(idx, DEV, size=384)
    torch.manual_seed(11)
    ref = p384.decoding(idx, DEV)
    assert tuple(out.shape) == (2, 3, 384, 384) and torch.equal(out, ref)
    p256.engine.close()
    p384.engine.close()
    dvae.decoder.close()


def test_size_errors_are_raised_before_any_launch():
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="fp16")
    x0, noise = _inputs(d, (8, 8), 2)
    ids = eng.encode(x0)
    ref = eng.decode(ids, noise).clone()
    eng.encode(*_inputs(d, (12, 16), 2)[:1], latent_hw=(12, 16))
    assert eng.latent_hw == (12, 16)
    bad = [
        lambda: eng.encode(torch.zeros(2, 16, 7, 8, device=DEV), latent_hw=(7, 8)),              # odd side
        lambda: eng.decode(ids, torch.zeros(2, 16, 10, 9, device=DEV), latent_hw=(10, 9)),
        lambda: eng.encode(torch.zeros(2, 16, 34, 8, device=DEV), latent_hw=(34, 8)),            # beyond enc_pos_max (16 patches)
        lambda: eng.decode(ids, torch.zeros(2, 16, 26, 8, device=DEV), latent_hw=(26, 8)),       # beyond dit_pos_max (12 patches)
        lambda: eng.dit_velocity(ids, torch.zeros(2, 16, 8, 26, device=DEV), 0, latent_hw=(8, 26)),
        lambda: eng.decode(ids, noise, latent_hw=(8, 12)),                                        # latent_hw disagrees with the tensor
        lambda: eng.decode(ids, torch.zeros(2, 16, 12, 12, device=DEV)),                          # None: the engine's own size only
        lambda: eng.set_latent_size(7, 8),
        lambda: eng.set_latent_size(0, 8),
        lambda: eng.set_latent_size(40, 40),                                                      # beyond both grids
    ]
    for f in bad:
        with pytest.raises(SelftokError):
            f()
        assert eng.latent_hw == (12, 16)
    # the library's own checks, reached without the Python ones: geometry (26, 26) fits the encoder's grid only
    eng.set_latent_size(26, 26)
    lib = eng.lib
    out = torch.empty(2, 16, 26, 26, device=DEV)
    assert lib.selftok_decode(eng.h, ids.data_ptr(), out.data_ptr(), 2, 50, out.data_ptr(), None) == -2
    assert b"MMDiT positional grid" in lib.selftok_last_error()
    assert torch.equal(eng.decode(ids, noise), ref)                     # and back at the default size, bitwise as before
    eng.close()
    dr = dataclasses.replace(C.TINY, renderer=True)
    ren = Engine(dr, synth.synth_state_dict(dr), device=DEV, precision="bf16x3")
    with pytest.raises(SelftokError, match="renderer"):
        ren.set_latent_size(12, 12)
    ren.set_latent_size(8, 8)
    assert ren.latent_hw == (8, 8)
    ren.close()
