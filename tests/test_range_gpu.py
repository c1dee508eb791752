"""Token ranges on the GPU: selftok_decode_range / selftok_decode_cfg_range / selftok_render_range through the C ABI.

Checked: [0, K) is bitwise the plain entry; windows match the reference's own window hooks (tests/golden/tiny_range.npz,
mid_range.npz, recorded by tests/golden/gen_range.py) and the window oracle (tests/_range_oracle.py, pinned to those fixtures);
an image's result is the same bit for bit alone, in a mixed-range batch and in a permuted batch; ids outside a window are never
read; graphs keyed by the rounded window bounds never replay a stale plan; SelftokPipeline forwards token_range (sharded entry
included); the kernel-level attention with per-image live context counts; error paths.
"""
import ctypes
import dataclasses
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _range_oracle as RO  # noqa: E402
from selftoktokenizer_b200 import config as C, synth  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = {"fp32": 2e-4, "bf16x3": 1e-3, "fp16": 1e-3, "bf16": 0.35}      # max-abs on latents of O(3) magnitude
PRECS = ["fp32", "bf16x3", "fp16", "bf16"]
# tiny geometry (K = 32; k of the last step is 1): a prefix, a suffix that goes empty at late steps, an interior window, all
TINY_RANGES = np.array([[0, 9], [20, 32], [5, 17]])
TINY_CFG_RANGES = np.array([[0, 9], [1, 32], [0, 32]])               # the guided sampler needs lo <= 1
MID_RANGES = np.array([[0, 1], [0, 70], [37, 101], [64, 128]])


@pytest.fixture(scope="module")
def tiny_sd():
    return synth.synth_state_dict(C.TINY)


@pytest.fixture(scope="module", params=PRECS)
def tiny_engine(request, tiny_sd):
    from selftoktokenizer_b200.capi import Engine
    eng = Engine(C.TINY, tiny_sd, device=DEV, precision=request.param)
    yield eng
    eng.close()


@pytest.fixture(scope="module")
def tiny_rend():
    d = dataclasses.replace(C.TINY, renderer=True)
    return d, synth.synth_state_dict(d)


def _tiny(gold):
    g = gold("tiny")
    return torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])


def test_full_range_is_the_plain_entry(tiny_engine, gold):
    tok, noise = _tiny(gold)
    K = C.TINY.K
    for use_graph in (False, True):
        tiny_engine.set_use_graph(use_graph)
        assert torch.equal(tiny_engine.decode(tok, noise, token_range=(0, K)).cpu(), tiny_engine.decode(tok, noise).cpu())
        assert torch.equal(tiny_engine.decode_cfg(tok, noise, 2.5, token_range=(0, K)).cpu(), tiny_engine.decode_cfg(tok, noise, 2.5).cpu())
    tiny_engine.set_use_graph(True)


@pytest.mark.parametrize("precision", PRECS)
def test_full_range_is_the_plain_render(precision, tiny_rend, gold):
    from selftoktokenizer_b200.capi import Engine
    d, sd = tiny_rend
    tok = torch.from_numpy(gold("tiny_renderer")["tokens"])
    eng = Engine(d, sd, device=DEV, precision=precision)
    try:
        assert torch.equal(eng.render(tok, token_range=(0, d.K)).cpu(), eng.render(tok).cpu())
    finally:
        eng.close()


def test_tiny_against_reference_fixture(tiny_engine, gold):
    """The reference's p_sample_loop(..., super_mask) (plain and uncond_scale = 2.5) recorded in tiny_range.npz."""
    g = gold("tiny_range")
    tok, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    tol = TOL[tiny_engine.precision]
    for use_graph in (False, True):
        tiny_engine.set_use_graph(use_graph)
        err = np.abs(tiny_engine.decode(tok, noise, token_range=g["ranges"]).cpu().numpy() - g["pred_x0"]).max()
        print(f"[{tiny_engine.precision}] range decode vs reference (graph={use_graph}): max-abs err {err:.3e}")
        assert err < tol
    err = np.abs(tiny_engine.decode_cfg(tok, noise, float(g["cfg_scale"]), token_range=g["cfg_ranges"]).cpu().numpy() - g["pred_x0_cfg"]).max()
    print(f"[{tiny_engine.precision}] guided range decode vs reference: max-abs err {err:.3e}")
    assert err < tol


def test_tiny_against_window_oracle(tiny_engine, tiny_sd, gold):
    tok, noise = _tiny(gold)
    d, tol = C.TINY, TOL[tiny_engine.precision]
    ref = RO.decode(tiny_sd, d, tok, noise, TINY_RANGES).numpy()
    for use_graph in (False, True):
        tiny_engine.set_use_graph(use_graph)
        err = np.abs(tiny_engine.decode(tok, noise, token_range=TINY_RANGES).cpu().numpy() - ref).max()
        print(f"[{tiny_engine.precision}] range decode (graph={use_graph}): max-abs err {err:.3e}")
        assert err < tol
    ref = RO.decode(tiny_sd, d, tok, noise, TINY_CFG_RANGES, cfg_scale=2.5).numpy()
    err = np.abs(tiny_engine.decode_cfg(tok, noise, 2.5, token_range=TINY_CFG_RANGES).cpu().numpy() - ref).max()
    print(f"[{tiny_engine.precision}] guided range decode: max-abs err {err:.3e}")
    assert err < tol


@pytest.mark.parametrize("precision", PRECS)
def test_tiny_render_against_reference_fixture(precision, tiny_rend, gold):
    """The reference's MMDiT_Renderer.forward(..., mask=window) recorded in tiny_range.npz."""
    from selftoktokenizer_b200.capi import Engine
    d, sd = tiny_rend
    g = gold("tiny_range")
    eng = Engine(d, sd, device=DEV, precision=precision)
    try:
        err = np.abs(eng.render(torch.from_numpy(g["renderer_tokens"]), token_range=g["ranges"]).cpu().numpy() - g["renderer_pred_x0"]).max()
        print(f"[{precision}] range render vs reference: max-abs err {err:.3e}")
        assert err < TOL[precision]
    finally:
        eng.close()


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
def test_mid_against_reference_fixture(precision, gold):
    """MID geometry (K = 128): windows that straddle the 64-row tiles of the attention and the rounding of the window bounds, against
    the reference's p_sample_loop(..., super_mask) recorded in mid_range.npz."""
    from selftoktokenizer_b200.capi import Engine
    g = gold("mid_range")
    d = C.MID
    tok, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision=precision)
    try:
        err = np.abs(eng.decode(tok, noise, token_range=g["ranges"]).cpu().numpy() - g["pred_x0"]).max()
        print(f"[{precision}] mid range decode: max-abs err {err:.3e}")
        assert err < TOL[precision]
    finally:
        eng.close()


def _invariance(eng, tok, noise, ranges, cfg_scale=None):
    """Mixed-range batch == every image alone == a permuted batch, bitwise (plain sampler, or guided with cfg_scale)."""
    run = (lambda t, n, r: eng.decode(t, n, token_range=r).cpu()) if cfg_scale is None else \
        (lambda t, n, r: eng.decode_cfg(t, n, cfg_scale, token_range=r).cpu())
    B = tok.shape[0]
    full = run(tok, noise, ranges)
    for b in range(B):
        alone = run(tok[b:b + 1], noise[b:b + 1], ranges[b:b + 1])
        assert torch.equal(alone[0], full[b]), f"image {b} {ranges[b].tolist()} differs alone"
    perm = np.random.default_rng(7).permutation(B)
    assert torch.equal(run(tok[perm], noise[perm], ranges[perm]), full[perm])


def test_tiny_batch_composition_invariance(tiny_engine, gold):
    tok, noise = _tiny(gold)
    _invariance(tiny_engine, tok, noise, TINY_RANGES)
    _invariance(tiny_engine, tok, noise, TINY_CFG_RANGES, cfg_scale=2.5)


@pytest.mark.parametrize("precision", ["fp16", "bf16x3"])
def test_full_batch_composition_invariance(precision):
    from selftoktokenizer_b200.capi import Engine
    d = C.FULL
    sd = synth.synth_state_dict(d, device=DEV)
    eng = Engine(d, sd, device=DEV, precision=precision)
    try:
        ranges = np.array([[d.K - n, d.K] for n in (1, 32, 128, 256, 384, 511, 512)] + [[100, 300]])
        tok = (torch.arange(8 * d.K, dtype=torch.int64).reshape(8, d.K) * 2654435761) % d.codebook_size
        noise = synth.synth_tensor("range.full.noise", (8, d.in_channels, d.latent, d.latent), "emb", 1.0)
        _invariance(eng, tok, noise, ranges)
        # guided sampler: every window keeps a visible token at the last step (k = 19 there)
        cfg_ranges = np.array([[0, 512], [0, 1], [19, 512], [5, 300], [10, 64], [0, 200], [19, 20], [3, 511]])
        _invariance(eng, tok, noise, cfg_ranges, cfg_scale=2.5)
    finally:
        eng.close()


def test_ids_outside_window_are_not_read(gold):
    from selftoktokenizer_b200.capi import Engine
    tok, noise = _tiny(gold)
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="fp16")
    try:
        win = RO.windows(TINY_RANGES, 3, d.K)
        base = eng.decode(tok.to(DEV), noise, token_range=TINY_RANGES).cpu()
        assert eng.id_errors() == 0
        for fill in (torch.full_like(tok, -1), torch.full_like(tok, d.codebook_size + 7), (tok * 7 + 3) % d.codebook_size):
            padded = torch.where(win, tok, fill)
            assert torch.equal(eng.decode(padded.to(DEV), noise, token_range=TINY_RANGES).cpu(), base)
            assert eng.id_errors() == 0
            assert torch.equal(eng.decode(padded, noise, token_range=TINY_RANGES).cpu(), base)    # host ids: checked in the window only
        bad = tok.clone()
        bad[1, 25] = d.codebook_size                                           # inside image 1's window [20, 32)
        eng.decode(bad.to(DEV), noise, token_range=TINY_RANGES)
        assert eng.id_errors() == 1
    finally:
        eng.close()


def test_graph_reuse_has_no_stale_plan(gold):
    """Two range sets with the same rounded bounds share one graph: A, B, A each equal their eager result."""
    from selftoktokenizer_b200.capi import Engine
    tok, noise = _tiny(gold)
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="bf16x3")
    try:
        A, B = TINY_RANGES, np.array([[3, 30], [0, 32], [10, 11]])
        eng.set_use_graph(False)
        eager = {k: eng.decode(tok, noise, token_range=r).cpu() for k, r in (("A", A), ("B", B))}
        eng.set_use_graph(True)
        for k, r in (("A", A), ("B", B), ("A", A)):
            assert torch.equal(eng.decode(tok, noise, token_range=r).cpu(), eager[k]), k
    finally:
        eng.close()


def test_caller_workspace(gold):
    from selftoktokenizer_b200.capi import Engine
    tok, noise = _tiny(gold)
    d = C.TINY
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="fp16")
    try:
        lib_ws = eng.decode(tok, noise, token_range=TINY_RANGES).cpu()
        eng.use_torch_workspace(3)
        assert torch.equal(eng.decode(tok, noise, token_range=TINY_RANGES).cpu(), lib_ws)
    finally:
        eng.close()


def _attn_ref(qkv, H, Kc, live, ctx_self):
    """fp32 reference of selftok_k_attention_tc_range: masked SDPA per image; rows with no visible key are 0."""
    B, S = qkv.shape[:2]
    N = S - Kc
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3).double() for i in range(3))
    out = torch.zeros(B, H, S, 64, dtype=torch.float64, device=qkv.device)
    for b in range(B):
        c = int(live[b])
        rows = torch.arange(S, device=qkv.device)
        is_ctx = (rows < c) | (rows >= c + N)
        kmax = torch.where(is_ctx & ctx_self, torch.full_like(rows, c), torch.full_like(rows, c + N))
        mask = torch.arange(S, device=qkv.device)[None] < kmax[:, None]
        s = (q[b] @ k[b].transpose(-1, -2)) / 8.0
        s = s.masked_fill(~mask, float("-inf"))
        p = torch.softmax(s, -1).nan_to_num(0.0)
        out[b] = p @ v[b]
    return out.permute(0, 2, 1, 3).reshape(B, S, H * 64).float()


@pytest.mark.parametrize("ctx_self", [False, True])
def test_k_attention_tc_range(ctx_self):
    from selftoktokenizer_b200 import capi
    H, Kc, N = 2, 70, 100
    live = [0, 1, 63, 64, 65, Kc]
    g = torch.Generator(device="cpu").manual_seed(11)
    qkv = torch.randn(len(live), Kc + N, 3, H, 64, generator=g).to(DEV)
    ref = _attn_ref(qkv, H, Kc, live, ctx_self)
    for ns, tol in ((3, 1e-4), (1, 3e-2), (0, 5e-3)):
        out = capi.k_attention_tc_range(qkv, H, Kc, live, nsplit=ns, ctx_self=ctx_self)
        assert torch.isfinite(out).all()
        err = float((out - ref).abs().max())
        print(f"attention range ns={ns} ctx_self={ctx_self}: max-abs err {err:.3e}")
        assert err < tol
        if ctx_self:                                                           # image 0: its context rows see nothing -> 0
            assert float(out[0, N:].abs().max()) == 0.0


def test_error_paths(tiny_engine, gold):
    from selftoktokenizer_b200 import capi
    tok, noise = _tiny(gold)
    lib, K = tiny_engine.lib, C.TINY.K
    td, nd = tok.to(DEV), noise.to(DEV)
    out = torch.empty_like(nd)
    s = torch.cuda.current_stream().cuda_stream
    cases = [([[0, 9], [-1, 5], [0, K]], False), ([[0, 9], [0, K + 1], [0, K]], False), ([[0, 9], [0, K], [7, 7]], False),
             ([[0, 9], [0, K], [2, K]], True)]                               # guided: lo = 2 > k of the last step (1)
    for rows, guided in cases:
        r = np.ascontiguousarray(rows, dtype=np.int32)
        bad = next(b for b, (lo, hi) in enumerate(rows) if not (0 <= lo < hi <= K) or (guided and lo > 1))
        if guided:
            st = lib.selftok_decode_cfg_range(tiny_engine.h, td.data_ptr(), r.ctypes.data, nd.data_ptr(), 3, 50, ctypes.c_float(2.5),
                                              out.data_ptr(), s)
        else:
            st = lib.selftok_decode_range(tiny_engine.h, td.data_ptr(), r.ctypes.data, nd.data_ptr(), 3, 50, out.data_ptr(), s)
        assert st == -1
        assert f"image {bad}" in lib.selftok_last_error().decode()
    with pytest.raises(capi.SelftokError):
        tiny_engine.decode(tok, noise, token_range=np.zeros((2, 2), dtype=np.int64))   # wrong number of windows
    with pytest.raises(capi.SelftokError):
        tiny_engine.decode(tok[:, :9], noise, token_range=(0, 9))                        # token rows stay [B, K]


def test_pipeline_token_range(tiny_sd, gold, monkeypatch):
    """SelftokPipeline forwards token_range: host ids padded with -1 outside the windows pass the host check, and the sharded
    entry slices the windows per rank (two ranks simulated in one process, gather off)."""
    from selftoktokenizer_b200 import SelftokPipeline, dist as D
    tok, noise = _tiny(gold)
    d = C.TINY
    pipe = SelftokPipeline(cfg=None, ckpt_path=None, sd3_path=None, datasize=d.latent * 8, device=DEV, state_dict=tiny_sd, dims=d,
                           precision="bf16x3")
    win = RO.windows(TINY_RANGES, 3, d.K)
    padded = torch.where(win, tok, torch.full_like(tok, -1)).numpy()
    want = pipe.engine.decode(tok, noise, token_range=TINY_RANGES).cpu()
    assert torch.equal(pipe.decode_latents(padded, noise, token_range=TINY_RANGES).cpu(), want)
    padded_cfg = torch.where(RO.windows(TINY_CFG_RANGES, 3, d.K), tok, torch.full_like(tok, -1)).numpy()
    assert torch.equal(pipe.decode_latents(padded_cfg, noise, cfg_scale=2.5, token_range=TINY_CFG_RANGES).cpu(),
                       pipe.engine.decode_cfg(tok, noise, 2.5, token_range=TINY_CFG_RANGES).cpu())
    with pytest.raises(Exception):
        pipe.decode_latents(padded, noise)                                   # without the windows, -1 is an id error
    parts = []
    for rank in range(2):
        monkeypatch.setattr(D, "world", lambda r=rank: (r, 2))
        parts.append(pipe.decode_latents_sharded(padded, noise, gather=False, token_range=TINY_RANGES).cpu())
    assert torch.equal(torch.cat(parts), want)
    pipe.engine.close()
