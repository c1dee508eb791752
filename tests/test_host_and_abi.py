"""CPU-side checks: the C-ABI library loads and exports exactly what include/selftok_b200.h declares, the config
surface / state-dict contract, the no-fallback rule, and the world_size-2 token gather over gloo."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from selftoktokenizer_b200 import capi, config as C, schedule as S, synth
from selftoktokenizer_b200 import build as B
from selftoktokenizer_b200.dist import shard_slice

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_loads_and_exports_every_declared_symbol():
    B.build()
    lib = capi.load_library()
    header = open(os.path.join(REPO, "include", "selftok_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(selftok_[a-z0-9_]+)\s*\(", header))
    assert declared == set(capi.SYMBOLS), declared ^ set(capi.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name)
    out = subprocess.run(["nm", "-D", "--defined-only", capi._LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (selftok_\w+)", out))
    assert exported == declared
    assert b"sm_90a" in lib.selftok_version()


def test_sass_contains_hopper_tensor_and_tma_instructions():
    """HGMMA = wgmma.mma_async, UTMALDG = TMA tile load (.MULTICAST: the two-CTA cluster GEMM sharing its weight tile)."""
    B.build()
    cuobjdump = "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", capi._LIB_PATH], capture_output=True, text=True).stdout
    for mnemonic in ("HGMMA", "UTMALDG", "UTMALDG.2D.MULTICAST"):
        assert mnemonic in sass, mnemonic
    # no legacy tensor path left: every tensor-core product of the library is a wgmma (HMMA = mma.sync / wmma)
    assert not re.search(r"\bHMMA", sass), "legacy mma.sync instructions found in the library"


_BASE = 1 << 40          # a 256-byte aligned address; the calls below are rejected before any CUDA call, so nothing is read


def _k_gemm_case(name):
    M, N, K = 64, 64, 64
    a = lambda i: _BASE + i * (1 << 24)
    store = dict(mode="store", out=a(3), ldo=N, bias=a(4))
    resid = dict(mode="resid", out=a(3), ldo=N, resid=a(5), gate=a(6), gate_ld=N)
    split = dict(mode="split", out_hi=a(7), out_lo=a(8), ldo=N)
    ep = {"bias": dict(store, bias=a(4) + 4), "out": dict(store, out=a(3) + 4), "addtab": dict(store, addtab=a(9) + 4, add_ld=N),
          "resid": dict(resid, resid=a(5) + 4), "gate": dict(resid, gate=a(6) + 4), "in_place_out": dict(resid, out=a(5) + 4, resid=a(5) + 4),
          "out_hi": dict(split, out_hi=a(7) + 2), "out_lo": dict(split, out_lo=a(8) + 2), "fp16_out_lo": dict(split, fp16=1),
          "no_out": dict(store, out=0), "no_resid": dict(resid, resid=0), "no_plane": dict(split, out_hi=0),
          "mode": dict(store, mode=3), "gate_period": dict(resid, gate_period=0), "plan_without_rpb": dict(store, plan=a(10))}[name]
    return capi.k_gemm_problem(a(1), a(2), M, N, K, **ep)


@pytest.mark.parametrize("path,nsplit", [(0, 3), (1, 3), (1, 1), (1, 0)])
@pytest.mark.parametrize("case", ["bias", "out", "addtab", "resid", "gate", "in_place_out", "out_hi", "out_lo", "fp16_out_lo",
                                  "no_out", "no_resid", "no_plane", "mode", "gate_period", "plan_without_rpb"])
def test_k_gemm_rejects_bad_epilogue_before_any_cuda_call(case, path, nsplit):
    """Misaligned fp32 bases (the wgmma epilogue moves float2 pairs) and 16-bit plane bases (32-bit pairs), an out_lo plane in the
    fp16 split mode, missing outputs and bad periods are SELFTOK_ERR_BAD_ARG from both GEMM paths, found on the host: the
    addresses here point at nothing, so a call that got as far as the device would fail differently."""
    B.build()
    st = capi.k_gemm_status(path, nsplit, [_k_gemm_case(case)], stream=0)
    assert st == -1, (st, capi.load_library().selftok_last_error())
    assert b"selftok_k_gemm" in capi.load_library().selftok_last_error()


def test_k_gemm_rejects_bad_calls():
    B.build()
    q = _k_gemm_case("bias")
    q.ep.bias = _BASE
    assert capi.k_gemm_status(0, 3, [q, q], stream=0) == -1        # the FFMA path takes one problem
    assert capi.k_gemm_status(1, 2, [q], stream=0) == -1           # nsplit 3 / 1 / 0
    assert capi.k_gemm_status(2, 3, [q], stream=0) == -1
    q.conv_C, q.conv_H, q.conv_W, q.conv_stride = 64, 8, 8, 1
    assert capi.k_gemm_status(0, 3, [q], stream=0) == -1           # no convolution on the FFMA path
    q.conv_C, q.M = 0, 0
    assert capi.k_gemm_status(1, 3, [q], stream=0) == -1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    B.build()
    with pytest.raises(capi.SelftokError):
        capi.Engine(C.TINY, synth.synth_state_dict(C.TINY), device="cuda:0", precision="fp32")


def test_config_surface():
    cfg = C.parse_args_from_yaml(os.path.join(REPO, "configs/selftok_256_512tok.yml"))
    assert cfg.tokenizer.params.k == 512 and cfg.common.is_eval is True
    assert not hasattr(cfg.tokenizer.params, "cut_of_k")
    before = repr(cfg)
    d = C.SelftokDims.from_cfg(cfg)
    assert repr(cfg) == before, "from_cfg must not mutate cfg (the reference does; consciously dropped)"
    assert d == C.FULL and d.dit_hidden == 1536 and d.n_img == 256 and d.enc_n_img == 256
    for yml, K, rend in (("selftok_256_1024tok.yml", 1024, False), ("selftok_renderer_1024tok.yml", 1024, True)):
        dk = C.SelftokDims.from_cfg(C.parse_args_from_yaml(os.path.join(REPO, "configs", yml)))
        assert dk.K == K and dk.renderer is rend and sum(dk.k_per_stage) == K and dk.latent == 32
    r = C.SelftokDims.from_cfg(C.parse_args_from_yaml(os.path.join(REPO, "configs/selftok_renderer_512tok.yml")))
    assert r.renderer and not r.context_see_xt and r.stages == (1000,)
    with pytest.raises(KeyError):
        bad = C.parse_args_from_yaml(os.path.join(REPO, "configs/selftok_256_512tok.yml"))
        bad.tokenizer.params.enc = "Enc-Qformer-Uni-L/2"
        C.SelftokDims.from_cfg(bad)


def test_state_dict_contract_counts():
    assert abs(synth.num_params(C.FULL) / 1e9 - 2.225) < 0.01      # 84 M encoder + codebook + 2.085 B decoder (+ pos tables)
    spec = synth.state_dict_spec(C.FULL)
    assert spec["model.joint_blocks.23.context_block.adaLN_modulation.1.weight"][0] == (3072, 1536)
    assert "model.joint_blocks.23.context_block.attn.proj.weight" not in spec          # pre_only
    assert spec["model.joint_blocks.0.x_block.mlp.fc1.weight"][0] == (6144, 1536)
    assert spec["encoder.quantizer._codebook.embed"][0] == (1, 32768, 16)
    assert spec["model.pos_embed"][0] == (1, 36864, 1536)


def test_flop_model():
    eff, dense = S.decode_flops_per_image(512, C.FULL.stages, C.FULL.k_per_stage, 50, 24, 256)
    assert abs(eff / 1e12 - 43.99) < 0.05 and abs(dense / 1e12 - 55.45) < 0.05   # SURVEY 8a (joint blocks only)


def test_shard_slices_partition():
    for n in (1, 7, 64, 512):
        for w in (1, 2, 3, 8):
            sl = [shard_slice(n, r, w) for r in range(w)]
            assert sl[0][0] == 0 and sl[-1][1] == n
            assert all(sl[i][1] == sl[i + 1][0] for i in range(w - 1))
            assert max(h - l for l, h in sl) - min(h - l for l, h in sl) <= 1


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from selftoktokenizer_b200.dist import shard_slice, gather_tokens
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
n, K = 5, 8
full = torch.arange(n * K, dtype=torch.int64).reshape(n, K)
lo, hi = shard_slice(n, dist.get_rank(), 2)
out = gather_tokens(full[lo:hi].clone(), n)
assert torch.equal(out, full), (dist.get_rank(), out)
dist.destroy_process_group()
print("ok")
"""


def test_token_gather_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), REPO, port, str(r)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for r in range(2)]
    for p in procs:
        out, err = p.communicate(timeout=120)
        assert p.returncode == 0 and "ok" in out, err


_WORKER2 = """
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from selftoktokenizer_b200.dist import shard_slice, gather_rows, host_noise, world
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank, w = world()
n = 5
noise = host_noise(n, (4, 3, 3), seed=11)                       # the same draw on every rank
lo, hi = shard_slice(n, rank, w)
mine = noise[lo:hi] * 2.0                                         # stands for this rank's decode of its slice
full = gather_rows(mine, n)
assert torch.equal(full, noise * 2.0), rank
g = torch.Generator(device="cpu"); g.manual_seed(11)
assert torch.equal(noise, torch.randn(n, 4, 3, 3, generator=g))   # exactly the single-process draw
dist.destroy_process_group()
print("ok")
"""


def test_sharded_noise_and_row_gather_gloo_world2(tmp_path):
    script = tmp_path / "w2.py"
    script.write_text(_WORKER2)
    port = str(31500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), REPO, port, str(r)], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for r in range(2)]
    for p in procs:
        out, err = p.communicate(timeout=120)
        assert p.returncode == 0 and "ok" in out, err


def test_vae_key_mapping_from_diffusers_names():
    """The device VAE takes the in-tree SDVAE key names; a diffusers AutoencoderKL state dict is mapped onto them
    (decoder up_blocks listed lowest resolution first, encoder down_blocks in order, attention projections stored as Linear)."""
    from selftoktokenizer_b200.capi import VaeDecoder
    spec = synth.vae_state_dict_spec(128)

    def to_diffusers(name, shape):                      # the inverse renaming, written independently of the product code
        half = name[:len("decoder.")]
        n = name[len(half):]
        n = n.replace("mid.block_1", "mid_block.resnets.0").replace("mid.block_2", "mid_block.resnets.1")
        n = n.replace("mid.attn_1.norm", "mid_block.attentions.0.group_norm").replace("mid.attn_1.q", "mid_block.attentions.0.to_q")
        n = n.replace("mid.attn_1.k", "mid_block.attentions.0.to_k").replace("mid.attn_1.v", "mid_block.attentions.0.to_v")
        n = n.replace("mid.attn_1.proj_out", "mid_block.attentions.0.to_out.0").replace("nin_shortcut", "conv_shortcut")
        if n.startswith("norm_out"):
            n = "conv_" + n
        m = re.match(r"up\.(\d)\.block\.(\d)\.(.*)", n)
        if m:
            n = f"up_blocks.{3 - int(m.group(1))}.resnets.{m.group(2)}.{m.group(3)}"
        m = re.match(r"up\.(\d)\.upsample\.(.*)", n)
        if m:
            n = f"up_blocks.{3 - int(m.group(1))}.upsamplers.0.{m.group(2)}"
        m = re.match(r"down\.(\d)\.block\.(\d)\.(.*)", n)
        if m:
            n = f"down_blocks.{m.group(1)}.resnets.{m.group(2)}.{m.group(3)}"
        m = re.match(r"down\.(\d)\.downsample\.(.*)", n)
        if m:
            n = f"down_blocks.{m.group(1)}.downsamplers.0.{m.group(2)}"
        if "attentions.0.to_" in n and n.endswith(".weight"):
            shape = shape[:2]                            # Linear [C, C] instead of a 1x1 conv
        return half + n, shape

    fake = {}
    for name, (shape, _, _) in spec.items():
        dn, dshape = to_diffusers(name, tuple(shape))
        fake[dn] = torch.zeros(dshape)
    fake["quant_conv.weight"] = torch.zeros(1)           # neither half: ignored
    back = VaeDecoder.from_diffusers_keys(fake)
    assert set(back) == set(spec)
    for name, (shape, _, _) in spec.items():
        assert tuple(back[name].shape) == tuple(shape), name


def test_host_preprocessing_matches_torchvision():
    """SURVEY 8f4 / the reference's test.py:27-31,45-47: Resize(data_size) + CenterCrop(data_size) + NormalizeToTensor on the way
    in and save_image's quantisation on the way out, PIL-only here, bit-equal to torchvision where that is importable."""
    from PIL import Image
    from selftoktokenizer_b200.preprocess import load_images, resize_center_crop, to_uint8_hwc
    rng = np.random.RandomState(0)
    T = None
    try:
        import torchvision.transforms as T  # noqa: N812
    except Exception:  # pragma: no cover
        pass
    for (w, h) in [(640, 480), (300, 517), (256, 256), (255, 1024), (1000, 256)]:
        img = Image.fromarray(rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
        for size in (128, 256, 512):
            mine = resize_center_crop(img, size)
            assert mine.size == (size, size)
            if T is not None:
                ref = T.Compose([T.Resize(size), T.CenterCrop(size)])(img)
                assert np.array_equal(np.array(ref), np.array(mine)), (w, h, size)
    img = Image.fromarray(rng.randint(0, 256, (70, 90, 3)).astype(np.uint8))
    x = load_images([img, img.convert("L")], 64)                      # grey input is promoted to 3 channels
    assert tuple(x.shape) == (2, 3, 64, 64) and x.dtype == torch.float32 and float(x.min()) >= -1 and float(x.max()) <= 1
    back = to_uint8_hwc((x[0] + 1) / 2)
    assert np.array_equal(back, np.array(resize_center_crop(img, 64)))   # [-1,1] -> [0,1] -> uint8 is the identity on 8-bit pixels
