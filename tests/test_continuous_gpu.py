"""Step-level batching on the GPU: selftok_decode_step and ContinuousDecoder.

The contract: an image's steps 0..n-1 run through any sequence of step calls, in any batches and interleaved with other images,
are bitwise decode(steps = n) / decode(token_range = its window) / decode_cfg(scale) of that image alone.  Also checked: the
reference fixtures, ids outside the visible rows, aliasing and the caller-owned workspace, the error paths, and the pipeline.
"""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from selftoktokenizer_b200 import config as C, synth  # noqa: E402
from selftoktokenizer_b200.continuous import ContinuousDecoder  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRECS = ["fp32", "bf16x3", "fp16", "bf16"]
TOL = {"fp32": 2e-4, "bf16x3": 1e-3, "fp16": 1e-3, "bf16": 0.35}      # as the range tests: max-abs on latents of O(3)
TINY_RANGES = np.array([[0, 9], [20, 32], [5, 17]])
TINY_CFG_RANGES = np.array([[0, 9], [1, 32], [0, 32]])               # the guided sampler needs lo <= 1 (k of the last step)
ERR_STATE = -3


@pytest.fixture(scope="module")
def tiny_sd():
    return synth.synth_state_dict(C.TINY)


@pytest.fixture(scope="module", params=PRECS)
def tiny_engine(request, tiny_sd):
    from selftoktokenizer_b200.capi import Engine
    eng = Engine(C.TINY, tiny_sd, device=DEV, precision=request.param)
    yield eng
    eng.close()


def _tiny(gold):
    g = gold("tiny")
    return torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])


def _loop(eng, tok, noise, steps=None, **kw):
    """decode_step over the schedule with every image on the same row."""
    x = noise.to(DEV).clone()
    td = tok.to(DEV)
    for i in range(steps or eng.steps):
        eng.decode_step(td, x, i, out=x, **kw)
    return x.cpu()


def test_homogeneous_steps_are_the_decode(tiny_engine, gold):
    tok, noise = _tiny(gold)
    assert torch.equal(_loop(tiny_engine, tok, noise), tiny_engine.decode(tok, noise).cpu())
    assert torch.equal(_loop(tiny_engine, tok, noise, steps=7), tiny_engine.decode(tok, noise, steps=7).cpu())
    assert torch.equal(_loop(tiny_engine, tok, noise, token_range=TINY_RANGES),
                       tiny_engine.decode(tok, noise, token_range=TINY_RANGES).cpu())
    assert torch.equal(_loop(tiny_engine, tok, noise, cfg_scale=2.5), tiny_engine.decode_cfg(tok, noise, 2.5).cpu())
    assert torch.equal(_loop(tiny_engine, tok, noise, token_range=TINY_CFG_RANGES, cfg_scale=2.5),
                       tiny_engine.decode_cfg(tok, noise, 2.5, token_range=TINY_CFG_RANGES).cpu())


def _requests(d, n_req, guided, seed):
    """n_req requests: mixed windows, mixed steps (the full schedule included), mixed scales when guided."""
    rng = np.random.default_rng(seed)
    reqs = []
    for i in range(n_req):
        ids = torch.from_numpy(rng.integers(0, d.codebook_size, d.K)).long()
        noise = synth.synth_tensor(f"cont.noise.{seed}.{i}", (1, d.in_channels, d.latent, d.latent), "emb", 1.0)
        n = 50 if i % 3 == 0 else int(rng.integers(1, 50))
        lo = int(rng.integers(0, d.K - 1)) if i % 2 else 0
        hi = int(rng.integers(lo + 1, d.K + 1)) if i % 4 == 1 else d.K
        reqs.append(dict(ids=ids, noise=noise, steps=n, token_range=(lo, hi), cfg_scale=(1.5 + 0.5 * i) if guided else None))
    return reqs


def _fix_guided(eng, reqs):
    """guided windows keep a visible token at the request's last step"""
    k = eng.tables.k.numpy()
    for r in reqs:
        lo, hi = r["token_range"]
        km = int(k[:r["steps"]].min())
        if lo > km:
            r["token_range"] = (km, max(hi, km + 1))


def _alone(eng, r):
    tok, noise = r["ids"][None], r["noise"]
    if r["cfg_scale"] is None:
        return eng.decode(tok, noise, r["steps"], token_range=r["token_range"]).cpu()
    return eng.decode_cfg(tok, noise, r["cfg_scale"], r["steps"], token_range=r["token_range"]).cpu()


def _staggered(eng, reqs, max_batch, offsets):
    """submit request i before step offsets[i] of the decoder; -> {request id: output}"""
    guided = reqs[0]["cfg_scale"] is not None
    dec = ContinuousDecoder(eng, max_batch, guided=guided)
    out, rid_of = {}, {}
    t, i = 0, 0
    while i < len(reqs) or dec.pending or dec.active:
        while i < len(reqs) and offsets[i] <= t:
            r = reqs[i]
            rid_of[dec.submit(r["ids"], r["noise"], token_range=r["token_range"], cfg_scale=r["cfg_scale"], steps=r["steps"])] = i
            i += 1
        for rid, x in dec.step():
            out[rid_of[rid]] = x.cpu()
        t += 1
    return out


@pytest.mark.parametrize("guided", [False, True])
def test_staggered_requests_are_bitwise_alone(tiny_engine, guided):
    d = C.TINY
    reqs = _requests(d, 8, guided, seed=3 + guided)
    if guided:
        _fix_guided(tiny_engine, reqs)
    offsets = [0, 0, 3, 10, 49, 50, 51, 80]                            # some queue; one joins at the last row of another
    out = _staggered(tiny_engine, reqs, 3, offsets)
    assert sorted(out) == list(range(len(reqs)))
    for i, r in enumerate(reqs):
        assert torch.equal(out[i], _alone(tiny_engine, r)), f"request {i} {r['token_range']} steps={r['steps']}"


@pytest.mark.parametrize("precision", ["fp16", "bf16x3"])
def test_full_staggered_requests_are_bitwise_alone(precision):
    from selftoktokenizer_b200.capi import Engine
    d = C.FULL
    eng = Engine(d, synth.synth_state_dict(d, device=DEV), device=DEV, precision=precision)
    try:
        wins = [(d.K - n, d.K) for n in (1, 32, 128, 256, 384, 511, 512)] + [(100, 300)]
        cfg_wins = [(0, 512), (0, 1), (19, 512), (5, 300), (10, 64), (0, 200), (19, 20), (3, 511)]
        for guided, ws in ((False, wins), (True, cfg_wins)):
            reqs = []
            for i, w in enumerate(ws):
                ids = (torch.arange(d.K, dtype=torch.int64) * 2654435761 + 977 * i) % d.codebook_size
                noise = synth.synth_tensor(f"cont.full.noise.{i}", (1, d.in_channels, d.latent, d.latent), "emb", 1.0)
                reqs.append(dict(ids=ids, noise=noise, steps=50 if i % 2 == 0 else 20 + i, token_range=w,
                                 cfg_scale=(2.5 - 0.25 * i) if guided else None))
            out = _staggered(eng, reqs, 4, [0, 0, 1, 7, 13, 30, 49, 50])
            for i, r in enumerate(reqs):
                assert torch.equal(out[i], _alone(eng, r)), f"guided={guided} request {i} {r['token_range']}"
    finally:
        eng.close()


def test_reference_fixtures(tiny_engine, gold):
    """tiny_range.npz (plain and guided windows), tiny.npz and tiny_cfg.npz through the decoder with staggered admission."""
    tol = TOL[tiny_engine.precision]
    g, gt, gc = gold("tiny_range"), gold("tiny"), gold("tiny_cfg")
    cases = [(g["tokens"], g["noise"], g["ranges"], None, g["pred_x0"]),
             (g["tokens"], g["noise"], g["cfg_ranges"], float(g["cfg_scale"]), g["pred_x0_cfg"]),
             (gt["tokens"], gt["noise"], None, None, gt["pred_x0"]),
             (gt["tokens"], gt["noise"], None, float(gc["cfg_scale"]), gc["pred_x0"])]
    for tok, noise, ranges, scale, want in cases:
        B = tok.shape[0]
        reqs = [dict(ids=torch.from_numpy(tok[b]), noise=torch.from_numpy(noise[b:b + 1]), steps=50,
                     token_range=None if ranges is None else tuple(int(v) for v in ranges[b]), cfg_scale=scale) for b in range(B)]
        out = _staggered(tiny_engine, reqs, 2, [0, 5, 17, 30][:B])
        got = np.concatenate([out[b].numpy() for b in range(B)])
        err = float(np.abs(got - want).max())
        # the guided combination amplifies the per-evaluation error by ~cfg_scale (test_guided_sampler_cfg)
        lim = tol * (2.5 if scale is not None and ranges is None else 1.0)
        print(f"[{tiny_engine.precision}] continuous vs reference (ranges={ranges is not None}, cfg={scale}): max-abs err {err:.3e}")
        assert err < lim


def test_ids_outside_visible_rows_are_not_read(gold):
    from selftoktokenizer_b200.capi import Engine
    d = C.TINY
    tok, noise = _tiny(gold)
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="fp16")
    try:
        k = eng.tables.k.numpy()
        steps = np.array([0, 17, 49], dtype=np.int32)
        base = eng.decode_step(tok.to(DEV), noise, steps, token_range=TINY_RANGES).cpu()
        assert eng.id_errors() == 0
        pos = torch.arange(d.K)[None]
        lo, hi = torch.from_numpy(TINY_RANGES[:, :1]), torch.from_numpy(np.minimum(TINY_RANGES[:, 1:], k[steps][:, None] + 1))
        vis = (pos >= lo) & (pos < hi)
        for fill in (torch.full_like(tok, -1), torch.full_like(tok, d.codebook_size + 7), (tok * 7 + 3) % d.codebook_size):
            padded = torch.where(vis, tok, fill)
            assert torch.equal(eng.decode_step(padded.to(DEV), noise, steps, token_range=TINY_RANGES).cpu(), base)
            assert eng.id_errors() == 0
            assert torch.equal(eng.decode_step(padded, noise, steps, token_range=TINY_RANGES).cpu(), base)    # host check: visible ids only
        bad = tok.clone()
        bad[0, 3] = d.codebook_size                                           # visible for image 0 at step 0
        eng.decode_step(bad.to(DEV), noise, steps, token_range=TINY_RANGES)
        assert eng.id_errors() == 1
    finally:
        eng.close()


def test_aliasing_and_caller_workspace(gold):
    from selftoktokenizer_b200.capi import Engine
    d = C.TINY
    tok, noise = _tiny(gold)
    eng = Engine(d, synth.synth_state_dict(d), device=DEV, precision="bf16x3")
    try:
        steps = np.array([3, 0, 40], dtype=np.int32)
        want = eng.decode_step(tok, noise, steps, token_range=TINY_RANGES, cfg_scale=None).cpu()
        x = noise.to(DEV).clone()
        eng.decode_step(tok, x, steps, token_range=TINY_RANGES, out=x)
        assert torch.equal(x.cpu(), want)
        want_g = eng.decode_step(tok, noise, steps, token_range=TINY_CFG_RANGES, cfg_scale=[2.5, 1.0, 3.0]).cpu()
        eng.use_torch_workspace(3)
        assert torch.equal(eng.decode_step(tok, noise, steps, token_range=TINY_RANGES).cpu(), want)
        assert torch.equal(eng.decode_step(tok, noise, steps, token_range=TINY_CFG_RANGES, cfg_scale=[2.5, 1.0, 3.0]).cpu(), want_g)
    finally:
        eng.close()


def test_error_paths(gold, tiny_sd):
    import dataclasses
    from selftoktokenizer_b200.capi import Engine
    d = C.TINY
    tok, noise = _tiny(gold)
    eng = Engine(d, tiny_sd, device=DEV, precision="fp16")
    lib, K, s = eng.lib, d.K, torch.cuda.current_stream().cuda_stream
    td, nd = tok.to(DEV), noise.to(DEV)
    out = torch.full_like(nd, 12345.0)

    def call(steps, ranges=None, scales=None, h=None, t=td, x=nd, o=out, B=3):
        st = np.ascontiguousarray(steps, dtype=np.int32)
        r = None if ranges is None else np.ascontiguousarray(ranges, dtype=np.int32)
        cs = None if scales is None else np.ascontiguousarray(scales, dtype=np.float32)
        return lib.selftok_decode_step(h or eng.h, None if t is None else t.data_ptr(), None if r is None else r.ctypes.data,
                                       None if st is None else st.ctypes.data, None if cs is None else cs.ctypes.data,
                                       None if x is None else x.data_ptr(), B, None if o is None else o.data_ptr(), s)
    try:
        for steps, ranges, scales, bad in [([0, -1, 3], None, None, 1), ([0, 1, 50], None, None, 2),
                                           ([0, 1, 2], [[0, 9], [-1, 5], [0, K]], None, 1), ([0, 1, 2], [[0, 9], [0, K], [7, 7]], None, 2),
                                           ([0, 1, 2], [[0, K], [0, K + 1], [0, K]], None, 1),
                                           ([0, 49, 0], [[0, 9], [2, K], [0, K]], [2.5, 2.5, 2.5], 1)]:   # k of step 49 is 1
            assert call(steps, ranges, scales) == -1
            assert f"image {bad}" in lib.selftok_last_error().decode()
        assert call([0, 1, 2], B=0) == -1
        assert call([0, 1, 2], t=None) == -1 and call([0, 1, 2], x=None) == -1 and call([0, 1, 2], o=None) == -1
        torch.cuda.synchronize()
        assert bool((out == 12345.0).all()), "a rejected call wrote its output"
        rd = dataclasses.replace(d, renderer=True)
        rend = Engine(rd, synth.synth_state_dict(rd), device=DEV, precision="fp16")
        try:
            assert call([0, 0, 0], h=rend.h) == ERR_STATE
            assert "renderer" in lib.selftok_last_error().decode()
        finally:
            rend.close()
        torch.cuda.synchronize()
        assert bool((out == 12345.0).all())
        with pytest.raises(Exception):
            eng.decode_step(tok, noise, [0, 1])                                  # wrong number of steps
    finally:
        eng.close()


def test_guided_without_cfg_schedule_is_a_state_error(gold, tiny_sd):
    """A handle finalized without selftok_set_cfg_schedule: plain steps work, guided steps are SELFTOK_ERR_STATE."""
    from selftoktokenizer_b200 import capi, schedule as sched
    d = C.TINY
    tok, noise = _tiny(gold)
    eng = capi.Engine(d, tiny_sd, device=DEV, precision="fp16")
    lib = eng.lib
    h = ctypes.c_void_p()
    cfg = capi._Config(K=d.K, latent=d.latent, in_channels=d.in_channels, enc_patch=d.enc_patch, enc_hidden=d.enc_hidden,
                       enc_heads=d.enc_heads, enc_depth=d.enc_depth, enc_qdim=d.enc_qdim, enc_qheads=d.enc_qheads,
                       enc_pos_max=d.enc_pos_max, codebook_size=d.codebook_size, code_dim=d.code_dim, dit_depth=d.dit_depth,
                       dit_patch=d.dit_patch, dit_pos_max=d.dit_pos_max, renderer=0, context_see_xt=int(d.context_see_xt),
                       precision=capi.PREC["fp16"], device=0)
    capi.check(lib.selftok_create(ctypes.byref(cfg), ctypes.byref(h)))
    try:
        for name, t in tiny_sd.items():
            if torch.is_tensor(t) and t.is_floating_point() and (name.startswith("encoder.") or name.startswith("model.")):
                t = t.detach().float().contiguous().cpu()
                capi.check(lib.selftok_load_tensor(h, name.encode(), t.data_ptr(), 0, t.dim(), (ctypes.c_int64 * max(t.dim(), 1))(*t.shape), 0))
        tb = sched.make_tables(d.K, d.stages, d.k_per_stage, 50, 1.0)
        arr = [np.ascontiguousarray(a, dtype=np.float32) for a in (tb.t.numpy(), tb.dt.numpy(), tb.t_freq.numpy(), tb.pos_freq.numpy())]
        k = np.ascontiguousarray(tb.k.numpy(), dtype=np.int32)
        capi.check(lib.selftok_set_schedule(h, 50, arr[0].ctypes.data, arr[1].ctypes.data, k.ctypes.data, arr[2].ctypes.data, arr[3].ctypes.data))
        capi.check(lib.selftok_finalize(h, torch.cuda.current_stream().cuda_stream))
        td, nd = tok.to(DEV), noise.to(DEV)
        out = torch.full_like(nd, 7.0)
        st = np.zeros(3, np.int32)
        cs = np.full(3, 2.5, np.float32)
        s = torch.cuda.current_stream().cuda_stream
        assert lib.selftok_decode_step(h, td.data_ptr(), None, st.ctypes.data, cs.ctypes.data, nd.data_ptr(), 3, out.data_ptr(), s) == ERR_STATE
        assert "cfg" in lib.selftok_last_error().decode()
        torch.cuda.synchronize()
        assert bool((out == 7.0).all())
        assert lib.selftok_decode_step(h, td.data_ptr(), None, st.ctypes.data, None, nd.data_ptr(), 3, out.data_ptr(), s) == 0
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), eng.decode_step(tok, noise, 0).cpu())
    finally:
        lib.selftok_destroy(h)
        eng.close()


class _DeviceVAE:
    """the diffusers decode call shape over the device VAE decoder"""

    def __init__(self, dec):
        self.dec = dec

    def decode(self, z, return_dict=False):
        return (self.dec.decode(z.float()),)


def test_pipeline_continuous_decoder(tiny_sd, gold):
    from selftoktokenizer_b200 import SelftokPipeline
    from selftoktokenizer_b200.capi import VaeDecoder
    d = C.TINY
    g = gold("tiny")
    vae = VaeDecoder(synth.synth_vae_state_dict(ch=128, encoder=False), device=DEV)
    pipe = SelftokPipeline(cfg=None, ckpt_path=None, sd3_path=None, datasize=d.latent * 8, dtype=torch.float32, device=DEV,
                           state_dict=tiny_sd, dims=d, vae=_DeviceVAE(vae), precision="fp16")
    try:
        dec = ContinuousDecoder(pipe.engine, 4)                            # latents: the decoder without the pixel tail
        torch.manual_seed(77)
        dec.submit(torch.from_numpy(g["tokens"][0]))
        torch.manual_seed(77)
        want_lat = pipe.decode_latents(g["tokens"][:1]).cpu()
        (rid, lat), = dec.drain()
        assert torch.equal(lat.cpu(), want_lat)
        # pixels: one request, then two retiring in the same step, each against decoding() of that image alone
        dec = pipe.continuous_decoder(max_batch=4)
        for seeds in ([5], [6, 7]):
            rids = []
            for i, sd_ in enumerate(seeds):
                torch.manual_seed(sd_)
                rids.append(dec.submit(torch.from_numpy(g["tokens"][i])))
            res = dict(dec.drain())
            assert len(res) == len(seeds)
            for i, (rid, sd_) in enumerate(zip(rids, seeds)):
                torch.manual_seed(sd_)
                want = pipe.decoding(g["tokens"][i:i + 1], DEV).cpu()
                got = res[rid].cpu()
                assert got.shape == want.shape
                assert float((got - want).abs().max()) <= 1e-6
    finally:
        pipe.engine.close()
        vae.close()
