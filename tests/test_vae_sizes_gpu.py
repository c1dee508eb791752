"""The SD3 VAE at every image size: convolution tiles that overhang the image edge (`conv_edge`), odd and non-square latents,
and the pipeline at datasizes other than 128 / 256 / 512.

Kernel level, through selftok_k_gemm: the overhanging tiling against fp64 conv2d with the bound of
tests/test_gemm_epilogue_gpu.py (C_TOL), in all three 16-bit precisions and both cluster modes; bitwise against the same
convolution run on a zero-embedded canvas that the exact tiling accepts; and conv_edge = 1 equal to conv_edge = 0 wherever the
exact tiling exists.  VAE level: decode / encode against oracle/vae_oracle.py and the reference fixture vae_odd128, bit
reproducibility, and batch invariance.  Pipeline level: datasize 96 (TINY checkpoint) and 384 (full geometry) through the
device VAE, with no fallback to `encoder_vae`.
"""
import dataclasses
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from selftoktokenizer_b200 import config as C, synth
from test_gemm_epilogue_gpu import C_TOL, CFG_IDS, CFGS, CONVS, SENT32, U22, _dev, _rand, _round_operand, _sent32, _ulp32, gemm, problem

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
UNSUPPORTED = -2            # SELFTOK_ERR_UNSUPPORTED
WG_CFGS, WG_IDS = CFGS[1:], CFG_IDS[1:]

EDGE_CONVS = [  # (C, H, W, stride): H, W = output dims; none of them has an exact 128-pixel box
    (64, 4, 96, 1),
    (64, 3, 64, 1),
    (128, 9, 5, 1),
    (64, 12, 12, 1),
    (64, 1, 3, 1),
    (64, 48, 48, 1),
    (64, 200, 120, 1),
    (64, 8, 8, 2),
    (64, 9, 5, 2),
    (64, 36, 20, 2),
]


def _conv_operands(C_, imgs, H, Wd, stride, N, seed):
    x = _rand((imgs, H * stride, Wd * stride, C_), seed)                        # NHWC input
    w = _rand((N, C_, 3, 3), seed + 1, 1 / math.sqrt(9 * C_))
    b = _rand((N,), seed + 2)
    return x, w, b


def _a_operand(x, stride):
    """The A planes the kernel reads: the NHWC input, or for stride 2 its polyphase planes [img * 4 + py * 2 + px, H, W, C]."""
    if stride == 1:
        return x.contiguous()
    imgs, Hin, Win, C_ = x.shape
    return torch.stack([x[:, py::2, px::2] for py in (0, 1) for px in (0, 1)], 1).reshape(imgs * 4, Hin // 2, Win // 2, C_).contiguous()


def _run_conv(cfg, x, w, b, H, Wd, stride, edge, *, guard=3, pad=8, resid=None):
    """Output [M + guard, N + pad] sentinel buffer with ldo = N + pad; returns (the whole buffer, M, N)."""
    imgs, C_, N = x.shape[0], x.shape[3], w.shape[0]
    M, ldo = imgs * H * Wd, N + pad
    Wmat = w.permute(0, 2, 3, 1).reshape(N, 9 * C_).contiguous()              # K index (ky * 3 + kx) * C + c
    out = _sent32(M + guard, ldo)
    ep = dict(bias=_dev(b), out=out, ldo=ldo)
    if resid is not None:
        ep.update(mode="resid", resid=_dev(resid))
    gemm(cfg, [problem(_dev(_a_operand(x, stride)), _dev(Wmat), M, N, 9 * C_, conv=(C_, H, Wd, stride), conv_edge=edge, **ep)])
    return out.cpu(), M, N


def _assert_sentinels(buf, M, N):
    bits = buf.view(torch.int32)
    assert (bits[M:] == SENT32).all(), "a guard row past M was written"
    assert (bits[:M, N:] == SENT32).all(), "a column past N was written"


@pytest.mark.parametrize("C_,H,Wd,stride", EDGE_CONVS)
@pytest.mark.parametrize("cfg", WG_CFGS, ids=WG_IDS)
def test_edge_conv_vs_fp64(cfg, C_, H, Wd, stride):
    """conv_edge = 1: tiles overhang the right / bottom edge; every real pixel within C_TOL of fp64, nothing else written."""
    ns, N, imgs = cfg[1], 128, 2
    x, w, b = _conv_operands(C_, imgs, H, Wd, stride, N, 300)
    buf, M, _ = _run_conv(cfg, x, w, b, H, Wd, stride, True)
    _assert_sentinels(buf, M, N)
    y = buf[:M, :N]
    xr, wr = _round_operand(_dev(x), ns).permute(0, 3, 1, 2), _round_operand(_dev(w), ns)
    bd = _dev(b).double()
    if stride == 1:
        ref = F.conv2d(xr, wr, bd, padding=1)
        mag = F.conv2d(xr.abs(), wr.abs(), bd.abs(), padding=1)
    else:
        ref = F.conv2d(F.pad(xr, (0, 1, 0, 1)), wr, bd, stride=2)
        mag = F.conv2d(F.pad(xr.abs(), (0, 1, 0, 1)), wr.abs(), bd.abs(), stride=2)
    ref, mag = (t.permute(0, 2, 3, 1).reshape(M, N).cpu() for t in (ref, mag))
    ratio = (y.double() - ref).abs() / (U22 * mag)
    print(f"edge conv ratio {WG_IDS[WG_CFGS.index(cfg)]} C={C_} {H}x{Wd} s{stride}: {ratio.max().item():.4g}")
    assert ratio.max().item() <= C_TOL[ns], ratio.max().item()
    # the VAE's residual epilogue: dropped rows load no residual and store nothing
    r = _rand((M, N), 305)
    buf2, _, _ = _run_conv(cfg, x, w, b, H, Wd, stride, True, resid=torch.nn.functional.pad(r, (0, 8)))
    _assert_sentinels(buf2, M, N)
    exp = y.double() + r.double()
    assert ((buf2[:M, :N].double() - exp).abs() <= _ulp32(exp)).all()


@pytest.mark.parametrize("H,Wd,stride,CH,CW", [(9, 5, 1, 16, 8), (12, 12, 1, 16, 16), (3, 64, 1, 4, 64), (9, 5, 2, 16, 8),
                                                (36, 20, 2, 64, 32)])
@pytest.mark.parametrize("cfg", WG_CFGS, ids=WG_IDS)
def test_edge_conv_equals_cropped_canvas(cfg, H, Wd, stride, CH, CW):
    """The overhanging tiling is bitwise the crop of the same convolution on the input zero-embedded at the top left of a
    CH x CW (output) canvas that the exact tiling accepts: the TMA zero fill supplies exactly the zeros the canvas holds."""
    C_, N, imgs = 64, 128, 2
    x, w, b = _conv_operands(C_, imgs, H, Wd, stride, N, 310)
    canvas = torch.zeros(imgs, CH * stride, CW * stride, C_)
    canvas[:, :H * stride, :Wd * stride] = x
    buf, M, _ = _run_conv(cfg, x, w, b, H, Wd, stride, True)
    big, Mb, _ = _run_conv(cfg, canvas, w, b, CH, CW, stride, False)
    crop = big[:Mb, :N].reshape(imgs, CH, CW, N)[:, :H, :Wd].reshape(M, N)
    assert torch.equal(buf[:M, :N].view(torch.int32), crop.view(torch.int32))


@pytest.mark.parametrize("C_,imgs,H,Wd,stride", CONVS)
@pytest.mark.parametrize("cfg", WG_CFGS, ids=WG_IDS)
def test_edge_conv_keeps_exact_tiling(cfg, C_, imgs, H, Wd, stride):
    """Where an exact 128-pixel box exists, conv_edge = 1 picks it: the result is bitwise that of conv_edge = 0."""
    x, w, b = _conv_operands(C_, imgs, H, Wd, stride, 128, 320)
    r = _rand((imgs * H * Wd, 136), 323)
    for resid in (None, r):
        y0, M, N = _run_conv(cfg, x, w, b, H, Wd, stride, False, resid=resid)
        y1, _, _ = _run_conv(cfg, x, w, b, H, Wd, stride, True, resid=resid)
        assert torch.equal(y0.view(torch.int32), y1.view(torch.int32))


def test_edge_conv_still_rejects_channels():
    """Channels that are not a multiple of 64 stay SELFTOK_ERR_UNSUPPORTED with conv_edge; nothing is written."""
    from selftoktokenizer_b200 import capi
    C_, H, Wd, N = 96, 9, 5, 64
    M = 2 * H * Wd
    A, W, out = torch.zeros(M * C_, device=DEV), torch.zeros(N, 9 * C_, device=DEV), _sent32(M, N)
    st = capi.k_gemm_status(1, 3, [problem(A, W, M, N, 9 * C_, conv=(C_, H, Wd, 1), conv_edge=True, out=out, ldo=N)])
    assert st == -2, st
    assert (out.view(torch.int32) == SENT32).all()


# ---------------------------------------------------------------------------------------------------------- VAE
@pytest.fixture(scope="module")
def vae_sd():
    return synth.synth_vae_state_dict(ch=128)


@pytest.fixture(scope="module")
def vae(vae_sd):
    from selftoktokenizer_b200.capi import VaeDecoder
    v = VaeDecoder(vae_sd, device=DEV)
    yield v
    v.close()


class _NoTF32:
    """The restatement runs in fp32 on the device for speed; TF32 off, so that its convolutions and products are fp32."""

    def __enter__(self):
        self.saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def _sd_dev(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


@pytest.mark.parametrize("h,w", [(1, 3), (6, 10), (9, 5), (12, 12), (24, 24), (40, 24), (48, 48)])
def test_vae_decode_any_size(vae, vae_sd, h, w):
    """Decode at odd, non-square and non-power-of-two latents against the restatement of the reference's SDVAE,
    to the bar of test_device_vae_decoder_against_oracle; norm_ip, bit reproducibility and batch invariance."""
    import vae_oracle as V
    B = 3
    z = synth.synth_tensor(f"vae.sizes.z{h}x{w}", (B, 16, h, w), "emb", 1.0)
    out = vae.decode(z).cpu()
    assert tuple(out.shape) == (B, 3, 8 * h, 8 * w)
    assert torch.equal(out, vae.decode(z).cpu()), "the device VAE must be bit-reproducible"
    assert torch.equal(out[1:2], vae.decode(z[1:2]).cpu()), "an image's result must not depend on its batch"
    with torch.no_grad(), _NoTF32():
        ref = V.decode(_sd_dev(vae_sd), z.to(DEV)).cpu()
    err = float((out.double() - ref).abs().max())
    print(f"device VAE decode latent {h}x{w} B={B}: max-abs err {err:.3e} (|x|max {float(ref.abs().max()):.2f})")
    assert err < 2e-4
    n = vae.decode(z, norm_ip=True).cpu()
    assert float(n.min()) >= 0.0 and float(n.max()) <= 1.0
    assert float((n.double() - (ref.clamp(-1, 1) + 1) / 2).abs().max()) < 1e-4


@pytest.mark.parametrize("H,W", [(72, 40), (96, 96), (200, 120), (384, 384)])
def test_vae_encode_any_size(vae, vae_sd, H, W):
    """Encode at ragged sizes (every downsampled level of 72 x 40 and 200 x 120 is odd somewhere) against the restatement
    (mean and log-variance); bit reproducibility and batch invariance."""
    import vae_oracle as V
    B = 3
    x = synth.synth_tensor(f"vae.sizes.x{H}x{W}", (B, 3, H, W), "emb", 0.5)
    mean, logvar = vae.encode(x, return_logvar=True)
    mean, logvar = mean.cpu(), logvar.cpu()
    assert tuple(mean.shape) == (B, 16, H // 8, W // 8)
    assert torch.equal(mean, vae.encode(x).cpu()), "the device VAE must be bit-reproducible"
    m1, l1 = vae.encode(x[1:2], return_logvar=True)
    assert torch.equal(mean[1:2], m1.cpu()) and torch.equal(logvar[1:2], l1.cpu()), "an image's result must not depend on its batch"
    with torch.no_grad(), _NoTF32():
        mom = V.encode_moments(_sd_dev(vae_sd), x.to(DEV)).cpu()
    e_mean = float((mean.double() - mom[:, :16]).abs().max())
    e_lv = float((logvar.double() - mom[:, 16:]).abs().max())
    print(f"device VAE encode {H}x{W} B={B}: max-abs err mean {e_mean:.3e}, logvar {e_lv:.3e}")
    assert e_mean < 2e-4 and e_lv < 2e-4


def test_vae_against_odd_size_reference_fixture(vae, gold):
    """Both halves against the reference's own SDVAE at 72 x 40 images / 9 x 5 latents (tests/golden/vae_odd128.npz)."""
    g = gold("vae_odd128")
    x = synth.synth_tensor("golden.vae.x72x40", (2, 3, 72, 40), "emb", 0.5)
    z = synth.synth_tensor("golden.vae.z9x5", (2, 16, 9, 5), "emb", 1.0)
    mean, logvar = vae.encode(x, return_logvar=True)
    mom = torch.cat([mean, logvar], dim=1).cpu().numpy()
    dec = vae.decode(z).cpu().numpy()
    e_enc, e_dec = float(np.abs(mom - g["moments"]).max()), float(np.abs(dec - g["dec"]).max())
    print(f"device VAE vs reference at 72x40 / 9x5: encode {e_enc:.3e}, decode {e_dec:.3e}")
    assert e_enc < 2e-4 and e_dec < 2e-4


@pytest.mark.parametrize("what,args", [("decode", (1, 16, 0, 8)), ("decode", (1, 16, 129, 8)), ("encode", (1, 3, 100, 96)),
                                       ("encode", (1, 3, 1032, 1024))])
def test_vae_rejects_sizes_outside_the_range(vae, what, args):
    """Sizes outside the supported ranges are SELFTOK_ERR_UNSUPPORTED before any launch: the output keeps its sentinel."""
    from selftoktokenizer_b200 import capi
    B, Cc, H, W = args
    x = torch.zeros(B, Cc, H, W, device=DEV)
    if what == "decode":
        out = torch.empty(B, 3, 8 * max(H, 1), 8 * W, device=DEV)
        out.view(torch.int32).fill_(SENT32)
        st = vae.lib.selftok_vae_decode(vae.h, x.data_ptr() if x.numel() else out.data_ptr(), B, H, W, out.data_ptr(), 0, None)
    else:
        out = torch.empty(B, 16, H // 8, W // 8, device=DEV)
        out.view(torch.int32).fill_(SENT32)
        st = vae.lib.selftok_vae_encode(vae.h, x.data_ptr(), B, H, W, out.data_ptr(), None, None)
    torch.cuda.synchronize()
    assert st == UNSUPPORTED, st
    assert (out.view(torch.int32) == SENT32).all()
    if what == "encode":
        with pytest.raises(capi.SelftokError, match="status -2"):
            vae.encode(x)
    elif H > 0:
        with pytest.raises(capi.SelftokError, match="status -2"):
            vae.decode(x)


# ---------------------------------------------------------------------------------------------------------- pipeline
class _NoFallback:
    """An `encoder_vae` that must never be called."""

    def encode(self, *a, **k):
        raise AssertionError("encoder_vae was called: the device VAE should have encoded these images")


def _psnr(a, b):
    return 10.0 * np.log10(1.0 / max(float(((a - b) ** 2).mean()), 1e-30))


def _pixel_gate(px, px_ref, gt, what):
    """The pixel bar of tests/test_parity_gpu.py: max-abs <= 1e-3 on [0, 1] images, and PSNR against the same target image
    within 0.01 dB of the reference's reconstruction."""
    err = float(np.abs(px - px_ref).max())
    d_psnr = abs(_psnr(px, gt) - _psnr(px_ref, gt))
    print(f"[{what}] pixels: max-abs err {err:.3e}; PSNR vs target ours {_psnr(px, gt):.4f} dB / reference {_psnr(px_ref, gt):.4f} dB "
          f"(delta {d_psnr:.5f} dB)")
    assert err <= 1e-3, what
    assert d_psnr <= 0.01, what


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
def test_pipeline_datasize96_on_the_device_vae(vae_sd, gold, precision):
    """TINY checkpoint at datasize 96 (latent 12): the reference's tokens and noise through the sampler and the device VAE,
    against the reference's latents through the VAE restatement; encoding() on the device VAE, never on encoder_vae."""
    import vae_oracle as V
    from selftoktokenizer_b200 import SelftokPipeline
    from selftoktokenizer_b200.pipeline import DeviceVAE, SD3LatentFormat
    g = gold("tiny_ds96")
    d = dataclasses.replace(C.TINY, latent=12)
    dvae = DeviceVAE(vae_sd, DEV, encoder_vae=_NoFallback())
    pipe = SelftokPipeline(cfg=None, ckpt_path=None, sd3_path=None, datasize=96, dtype=torch.float32, device=DEV,
                           state_dict=synth.synth_state_dict(C.TINY), dims=d, vae=dvae, precision=precision)
    with torch.no_grad():
        pred_x0 = pipe.decode_latents(g["tokens"], noise=torch.from_numpy(g["noise"]))
        px = pipe._latents_to_pixels(pred_x0).cpu().numpy()
        px_ref = V.images_from_latents(vae_sd, torch.from_numpy(g["pred_x0"])).numpy()
        x0 = synth.synth_tensor("golden.tinyds.x0", (2, d.in_channels, 12, 12), "emb", 1.0)
        gt = V.images_from_latents(vae_sd, x0).numpy()
    assert px.shape == (2, 3, 96, 96)
    _pixel_gate(px, px_ref, gt, f"datasize 96 {precision}")
    images = synth.synth_tensor("vae.sizes.ds96.images", (2, 3, 96, 96), "emb", 0.5).to(DEV)
    tok = pipe.encoding(images, DEV)
    with torch.no_grad():
        exp = pipe.encode_latents(SD3LatentFormat().process_in(dvae.decoder.encode(images)).to(torch.float32))
    assert torch.equal(tok, exp)
    pipe.engine.close()
    dvae.decoder.close()


def test_pipeline_datasize384_full_geometry(vae_sd):
    """Full geometry at datasize 384 (latent 48), synthetic weights, fp16, B = 2: encoding -> decoding and
    decoding_with_renderer, all on the device; each image equals its own B = 1 run bitwise."""
    import os
    from selftoktokenizer_b200 import SelftokPipeline
    from selftoktokenizer_b200.pipeline import DeviceVAE
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dvae = DeviceVAE(vae_sd, DEV, encoder_vae=_NoFallback())
    images = synth.synth_tensor("vae.sizes.ds384.images", (2, 3, 384, 384), "emb", 0.5).to(DEV)
    for yml in ("configs/selftok_256_512tok.yml", "configs/selftok_renderer_512tok.yml"):
        cfg = C.parse_args_from_yaml(os.path.join(root, yml))
        d = C.SelftokDims.from_cfg(cfg, 384)
        pipe = SelftokPipeline(cfg=cfg, ckpt_path=None, sd3_path=None, datasize=384, dtype=torch.float32, device=DEV,
                               state_dict=synth.synth_state_dict(d, device=DEV), vae=dvae, precision="fp16")
        tok = pipe.encoding(images, DEV)
        assert tuple(tok.shape) == (2, d.K)
        for i in range(2):
            assert torch.equal(tok[i:i + 1], pipe.encoding(images[i:i + 1], DEV))
        idx = tok.cpu().numpy()
        if d.renderer:
            out = pipe.decoding_with_renderer(idx, DEV)
            singles = [pipe.decoding_with_renderer(idx[i:i + 1], DEV) for i in range(2)]
        else:
            torch.manual_seed(7)
            noise = torch.randn(2, d.in_channels, 48, 48)
            torch.manual_seed(7)
            out = pipe.decoding(idx, DEV)
            with torch.no_grad():
                singles = [pipe._latents_to_pixels(pipe.decode_latents(idx[i:i + 1], noise=noise[i:i + 1])) for i in range(2)]
        assert tuple(out.shape) == (2, 3, 384, 384)
        assert torch.isfinite(out).all() and float(out.min()) >= 0.0 and float(out.max()) <= 1.0
        for i in range(2):
            assert torch.equal(out[i:i + 1], singles[i]), f"{yml}: image {i} differs from its B = 1 run"
        pipe.engine.close()
    dvae.decoder.close()
