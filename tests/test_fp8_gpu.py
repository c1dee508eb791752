"""The fp8 decoder mode (precision "fp8", SELFTOK_PREC_FP8): e4m3 QKV and fc1 GEMMs with per-row scales.

The quantization contract (kernels.h, restated here by quant_e4m3_rows): per row of K fp32 values
  amax = max |x_i| (NaN when the row holds a NaN), inv = 448 / amax, scale = amax / 448 (both correctly rounded; 0 and 0 for
  an all-zero row), code_i = e4m3(x_i * inv) rounded to nearest, saturating to +-448.
Activations are quantized per GEMM row, weights per output channel, and the epilogue computes y = fma(acc, s_a[m] s_w[n], b)
before its mode.

Kernel level: the quantizer bitwise against the restatement, the LN quantizer against the fp32 LN kernel, the e4m3 GEMM
product against fp64 on the dequantized operands, and the epilogue routing, grouping, row-invariance and NaN tests of
test_gemm_epilogue_gpu.py run unchanged on the e4m3 operand type (nsplit 4).
Engine level: the bitwise contracts of the decoder in fp8, and its accuracy against the oracle with the quantization emulated
on the QKV / fc1 linears (the oracle's per-linear call `_lin` is swapped for the duration of a test).
"""
import math

import numpy as np
import pytest
import torch

import selftok_oracle as O
import test_gemm_epilogue_gpu as E
from selftoktokenizer_b200 import config as C, schedule as S, synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E4M3 = 4                                   # selftok_k_gemm nsplit of the e4m3 operand type
CFG8 = [(1, E4M3, 2), (1, E4M3, 1)]
CFG8_IDS = ["e4m3-cta2", "e4m3-cta1"]
# Product bound |y - ref| <= C_ACC * 2^-P_ACC * (sum_k |a_k w_k| + |b|) on the dequantized operands.  The fp8 tensor-core
# accumulator keeps fewer bits than fp32.  Largest ratios on the 2^-13 scale measured by test_e4m3_product_vs_fp64 on an NVIDIA
# H100 80GB HBM3 at a 700 W power limit: 0.14 at K = 64, 2.5 at K = 1536 (M = 257), 3.14 at K = 1536 (M = 1000), 3.50 at
# K = 6144 -- about 1790 on the 2^-22 scale of the 16-bit modes.  A one-row or one-column shift still exceeds the bound on
# most elements, which the test asserts.
P_ACC = 13
C_ACC = 16.0


def _capi():
    from selftoktokenizer_b200 import capi
    return capi


def quant_e4m3_rows(t):
    """The restatement: amax per row (NaN kept), inv = 448 / amax, scale = amax / 448 (0 and 0 for an all-zero row),
    codes = e4m3(x * inv).  The clamp to +-448 stands for satfinite (torch's cast makes 470 a NaN); NaN passes through it.
    Returns (codes as torch.float8_e4m3fn, scales [rows] fp32)."""
    t = t.float()
    amax = t.abs().amax(dim=-1, keepdim=True)
    zero = amax == 0
    inv = torch.where(zero, torch.zeros_like(amax), 448.0 / torch.where(zero, torch.ones_like(amax), amax))
    codes = (t * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return codes, (amax / 448.0).squeeze(-1)


def _codes_bits(c):
    return c.view(torch.uint8)


# ---------------------------------------------------------------------------------------------------------- quantizers
def _quant_rows():
    g = torch.Generator().manual_seed(5)
    K = 1536
    x = torch.randn(9, K, generator=g)
    x[1, 77] = 3e5                                            # one outlier: the rest of the row lands in the subnormal codes
    x[2] = torch.randn(K, generator=g) * 1e-6                 # tiny magnitudes (scale ~ 1e-8)
    x[3] = 0.0                                                # all zero: scale 0, codes 0
    x[4, 5] = float("nan")                                    # NaN row: scale and codes NaN
    x[5] = torch.randn(K, generator=g) * 3e4
    x[6, :] = 1.0
    x[6, 0] = -1.0
    x[7] = torch.linspace(-1, 1, K)
    x[8, 3] = 1e-40                                           # a subnormal fp32 input next to normal ones
    return x


def test_quantizer_bitwise():
    capi = _capi()
    x = _quant_rows()
    codes, scales = capi.k_quant_e4m3(x.to(DEV))
    codes, scales = codes.cpu(), scales.cpu()
    rc, rs = quant_e4m3_rows(x)
    fin = torch.ones(x.shape[0], dtype=torch.bool)
    fin[4] = False
    assert torch.equal(_codes_bits(codes)[fin], _codes_bits(rc)[fin])
    assert torch.equal(scales[fin].view(torch.int32), rs[fin].view(torch.int32))
    assert torch.isnan(scales[4]) and torch.isnan(codes[4].float()).all()
    assert scales[3] == 0 and (_codes_bits(codes[3]) == 0).all()
    assert codes[1].float().abs().max() == 448 and (codes[1].float().abs() < 2 ** -6).float().mean() > 0.5
    # non-multiple-of-16 K still quantizes (only the GEMM needs K % 16)
    c2, s2 = capi.k_quant_e4m3(x[:, :100].contiguous().to(DEV))
    rc2, rs2 = quant_e4m3_rows(x[:, :100])
    assert torch.equal(_codes_bits(c2.cpu())[fin], _codes_bits(rc2)[fin])


def _e4m3_half_step(q):
    """half the e4m3 spacing at code magnitude |q| (subnormal spacing 2^-9 below 2^-6)"""
    e = torch.floor(torch.log2(q.abs().clamp(min=2.0 ** -6)))
    return 0.5 * torch.exp2(e - 3)


@pytest.mark.parametrize("D,M,period", [(192, 37, 1), (1536, 70, 1), (1536, 96, 12), (384, 8, 8)])
def test_ln_quantizer(D, M, period):
    capi = _capi()
    g = torch.Generator().manual_seed(D + M)
    x = (torch.randn(M, D, generator=g) * 2 + 0.5).to(DEV)
    x[3 % M, 11] = float("nan")
    tab = (torch.randn(period, 2 * D, generator=g) * 0.3).to(DEV)
    shift, scale = tab[:, :D], tab[:, D:]
    codes, sc = capi.k_ln_mod_e4m3(x, shift, scale, period)
    ref = capi.k_ln_mod_f32(x, shift, scale, period).cpu().double()
    q, sc = codes.cpu().float().double(), sc.cpu().double()
    ok = torch.ones(M, dtype=torch.bool)
    ok[3 % M] = False
    assert torch.isnan(sc[~ok]).all() and torch.isnan(q[~ok]).all()
    deq = q[ok] * sc[ok, None]
    bound = _e4m3_half_step(ref[ok] / sc[ok, None]) * sc[ok, None] + 1e-6 * ref[ok].abs()
    assert ((deq - ref[ok]).abs() <= bound).all(), ((deq - ref[ok]).abs() / bound).max().item()
    assert (q[ok].abs().amax(1) == 448).all()
    # the row's amax element is the one that maps to +-448
    arg = ref[ok].abs().argmax(1)
    assert (q[ok].gather(1, arg[:, None]).abs() == 448).all()


# ---------------------------------------------------------------------------------------------------------- GEMM product
def _dequant(t):
    c, s = _capi().k_quant_e4m3(t.to(DEV))
    return c.double() * s.double()[:, None]


@pytest.mark.parametrize("M,N,K,ldo", E.PRODUCT_SHAPES + [(257, 292, 6144, 300)])
@pytest.mark.parametrize("cfg", CFG8, ids=CFG8_IDS)
def test_e4m3_product_vs_fp64(cfg, M, N, K, ldo):
    A, W, b = E._rand((M, K), 1), E._rand((N, K), 2, 1 / math.sqrt(K)), E._rand((N,), 3)
    out = E._sent32(M + 3, ldo)
    E.gemm(cfg, [E.problem(E._dev(A), E._dev(W), M, N, K, bias=E._dev(b), out=out, ldo=ldo)])
    out = out.cpu()
    a, w, bd = _dequant(A), _dequant(W), E._dev(b).double()
    ref, mag = (a @ w.t() + bd).cpu(), (a.abs() @ w.abs().t() + bd.abs()).cpu()
    unit = 2.0 ** -P_ACC
    ratio = (out[:M, :N].double() - ref).abs() / (unit * mag)
    print(f"e4m3 product ratio (2^-{P_ACC}) {cfg} M={M} N={N} K={K}: {ratio.max().item():.4g}  "
          f"(at 2^-22: {ratio.max().item() * 2.0 ** (22 - P_ACC):.4g})")
    assert ratio.max().item() <= C_ACC, ratio.max().item()
    bound = C_ACC * unit * mag
    if N > 1:
        assert ((ref[:, 1:] - ref[:, :-1]).abs() > bound[:, 1:]).double().mean() > 0.5
    if M > 1:
        assert ((ref[1:] - ref[:-1]).abs() > bound[1:]).double().mean() > 0.5
    assert (out[:, N:].view(torch.int32) == E.SENT32).all()
    assert (out[M:].view(torch.int32) == E.SENT32).all()


# ---------------------------------------------------------------------------------------------------------- epilogue contract
@pytest.mark.parametrize("mode", E.MODES)
@pytest.mark.parametrize("route", list(E.ROUTES))
@pytest.mark.parametrize("cfg", CFG8, ids=CFG8_IDS)
def test_e4m3_epilogue_routing(cfg, route, mode, monkeypatch):
    monkeypatch.setattr(E, "CFGS", E.CFGS + CFG8)            # its messages name the configuration
    monkeypatch.setattr(E, "CFG_IDS", E.CFG_IDS + CFG8_IDS)
    E.test_epilogue_routing(cfg, route, mode)


@pytest.mark.parametrize("kind", ["resid", "split"])
@pytest.mark.parametrize("cfg", CFG8, ids=CFG8_IDS)
def test_e4m3_grouped_equals_solo(cfg, kind):
    E.test_grouped_equals_solo(cfg, kind)


def test_e4m3_row_invariance():
    E.test_wgmma_row_invariance(E4M3)


@pytest.mark.parametrize("cfg", CFG8, ids=CFG8_IDS)
def test_e4m3_nan_row(cfg):
    E.test_nan_row_stays_nan(cfg)
    # the NaN rows leave every other row bitwise as without them (per-row scales)
    M, N, K = 130, 292, 320
    A, W, b = E._rand((M, K), 94), E._rand((N, K), 95, 1 / math.sqrt(K)), E._rand((N,), 96)
    outs = []
    for poison in (False, True):
        A2 = A.clone()
        if poison:
            A2[[0, 9, 129], [5, 42, 79]] = float("nan")
        out = E._sent32(M, N)
        E.gemm(cfg, [E.problem(E._dev(A2), E._dev(W), M, N, K, bias=E._dev(b), out=out, ldo=N)])
        outs.append(out.cpu())
    keep = [r for r in range(M) if r not in (0, 9, 129)]
    E.assert_bits_equal(outs[1][keep], outs[0][keep], "rows next to NaN rows")


def test_e4m3_host_checks():
    """The convolution mode and K % 16 != 0 are refused before any launch; the output keeps its sentinel."""
    capi = _capi()
    M, N, K, Cc = 256, 64, 9 * 64, 64
    A, W, out = torch.zeros(M * Cc, device=DEV), torch.zeros(N, K, device=DEV), E._sent32(M, N)
    assert capi.k_gemm_status(1, E4M3, [E.problem(A, W, M, N, K, conv=(Cc, 2, 128, 1), out=out, ldo=N)]) == -1
    A = torch.zeros(M, 72, device=DEV)
    assert capi.k_gemm_status(1, E4M3, [E.problem(A, torch.zeros(N, 72, device=DEV), M, N, 72, out=out, ldo=N)]) == -2
    assert (out.view(torch.int32) == E.SENT32).all()


# ---------------------------------------------------------------------------------------------------------- engine contracts
@pytest.fixture(scope="module")
def tiny_sd():
    return synth.synth_state_dict(C.TINY)


@pytest.fixture(scope="module")
def eng8(tiny_sd):
    from selftoktokenizer_b200.capi import Engine
    e = Engine(C.TINY, tiny_sd, device=DEV, precision="fp8")
    yield e
    e.close()


def _tiny(gold):
    g = gold("tiny")
    return torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])


def _contracts(eng, tok, noise, steps):
    # graph == eager
    eng.set_use_graph(False)
    eager = eng.decode(tok, noise, steps).cpu()
    eng.set_use_graph(True)
    graph = eng.decode(tok, noise, steps).cpu()
    assert torch.equal(eager, graph)
    assert torch.isfinite(graph).all()
    # an image alone == the same image in a permuted / mixed batch, plain and guided
    B = tok.shape[0]
    perm = torch.arange(B - 1, -1, -1)
    assert torch.equal(eng.decode(tok[perm], noise[perm], steps).cpu(), graph[perm])
    assert torch.equal(eng.decode(tok[1:2], noise[1:2], steps).cpu(), graph[1:2])
    gd = eng.decode_cfg(tok, noise, 2.5, steps).cpu()
    assert torch.equal(eng.decode_cfg(tok[perm], noise[perm], 2.5, steps).cpu(), gd[perm])
    assert torch.equal(eng.decode_cfg(tok[-1:], noise[-1:], 2.5, steps).cpu(), gd[-1:])
    return graph


def test_fp8_tiny_batch_contracts(eng8, gold):
    tok, noise = _tiny(gold)
    x = _contracts(eng8, tok, noise, None)
    K = C.TINY.K
    # [0, K) == the plain entries
    full = np.array([[0, K]] * tok.shape[0])
    assert torch.equal(eng8.decode(tok, noise, token_range=full).cpu(), x)
    assert torch.equal(eng8.decode_cfg(tok, noise, 2.5, token_range=full).cpu(), eng8.decode_cfg(tok, noise, 2.5).cpu())


def test_fp8_full_geometry_contracts():
    from selftoktokenizer_b200.capi import Engine
    d = C.FULL
    eng = Engine(d, synth.synth_state_dict(d, device=DEV), device=DEV, precision="fp8")
    try:
        noise = synth.synth_tensor("fp8.full.noise", (8, d.in_channels, d.latent, d.latent), "emb", 1.0)
        tok = (torch.arange(8 * d.K, dtype=torch.int64).reshape(8, d.K) * 2654435761) % d.codebook_size
        _contracts(eng, tok, noise, 50)
    finally:
        eng.close()


def test_fp8_decode_step_and_continuous(eng8, gold):
    import test_continuous_gpu as CT
    tok, noise = _tiny(gold)
    assert torch.equal(CT._loop(eng8, tok, noise), eng8.decode(tok, noise).cpu())
    assert torch.equal(CT._loop(eng8, tok, noise, steps=7), eng8.decode(tok, noise, steps=7).cpu())
    assert torch.equal(CT._loop(eng8, tok, noise, cfg_scale=2.5), eng8.decode_cfg(tok, noise, 2.5).cpu())
    reqs = CT._requests(C.TINY, 6, False, 11)
    out = CT._staggered(eng8, reqs, 3, [0, 0, 3, 9, 20, 21])
    for i, r in enumerate(reqs):
        assert torch.equal(out[i], CT._alone(eng8, r)), f"request {i}"


def test_fp8_prepack_workspace_and_bad_ids(tiny_sd, eng8, gold, tmp_path):
    from selftoktokenizer_b200.capi import Engine
    tok, noise = _tiny(gold)
    x = eng8.decode(tok, noise).cpu()
    path = str(tmp_path / "fp8.stkpack")
    e1 = Engine(C.TINY, tiny_sd, device=DEV, precision="fp8", pack_path=path)
    e2 = Engine(C.TINY, None, device=DEV, precision="fp8", pack_path=path)
    try:
        assert e2.restored_from_pack and e2.precision == "fp8"
        assert torch.equal(e1.decode(tok, noise).cpu(), x) and torch.equal(e2.decode(tok, noise).cpu(), x)
        # caller workspace == library workspace (the fp8 row scales are counted in it)
        e2.use_torch_workspace(3)
        assert torch.equal(e2.decode(tok, noise).cpu(), x)
    finally:
        e1.close()
        e2.close()
    # an out-of-range id is counted and poisons its own image.  It also reaches image 0 here -- in fp16 and bf16x3 as well (a
    # defect of the decoder outside this mode) -- so fp8 is held to the fp16 engine's pattern, and image 2 stays bitwise clean.
    bad = tok.clone().to(DEV)
    bad[1, 4] = 10 ** 6
    y = eng8.decode(bad, noise).cpu()
    assert eng8.id_errors() >= 1
    assert torch.isnan(y[1]).all()
    e16 = Engine(C.TINY, tiny_sd, device=DEV, precision="fp16")
    try:
        y16 = e16.decode(bad, noise).cpu()
        e16.id_errors()
    finally:
        e16.close()
    assert [bool(torch.isnan(y[b]).any()) for b in range(3)] == [bool(torch.isnan(y16[b]).any()) for b in range(3)]
    assert torch.equal(y[2], x[2])


def test_fp8_workspace_counts_row_scales(tiny_sd):
    from selftoktokenizer_b200.capi import Engine
    e16 = Engine(C.TINY, tiny_sd, device=DEV, precision="fp16")
    e8 = Engine(C.TINY, tiny_sd, device=DEV, precision="fp8")
    try:
        d, B = C.TINY, 5
        extra = e8.workspace_bytes(B, "decode") - e16.workspace_bytes(B, "decode")
        n_img = (d.latent // d.dit_patch) ** 2
        assert extra >= 4 * B * (d.K + n_img), extra
    finally:
        e16.close()
        e8.close()


# ---------------------------------------------------------------------------------------------------------- accuracy
def _rms(t):
    return float(t.double().pow(2).mean().sqrt())


_EXACT_LIN = O._lin


def _e4m3_lin(sd, prefix, x):
    """the oracle's checkpoint linear with the fp8 mode's quantization on the joint blocks' qkv / fc1: operands quantized per
    row (activations per GEMM row, weights per output channel), the dequantized product accumulated exactly; every other
    linear stays fp32"""
    if not (prefix.startswith("model.joint_blocks.") and prefix.endswith((".attn.qkv", ".mlp.fc1"))):
        return _EXACT_LIN(sd, prefix, x)
    xc, xs = quant_e4m3_rows(x.reshape(-1, x.shape[-1]))
    wc, ws = quant_e4m3_rows(sd[prefix + ".weight"])
    xq = (xc.double() * xs.double()[:, None]).reshape(x.shape)
    wq = wc.double() * ws.double()[:, None]
    return torch.nn.functional.linear(xq, wq).float() + sd[prefix + ".bias"]


def _oracle_velocity(sd, d, tok, x, st, tb, emulate, monkeypatch):
    with monkeypatch.context() as mp:
        mp.setattr(O, "_lin", _e4m3_lin if emulate else _EXACT_LIN)
        with torch.no_grad():
            return O.dit_velocity(sd, d, x, tb.t_freq[st], O.lookup(sd, d, tok), tb.pos_freq, int(tb.k[st]) + 1)


@pytest.mark.parametrize("geom", ["tiny", "mid"])
def test_fp8_velocity_error_is_the_quantization(geom, gold, monkeypatch):
    """RMS(engine - emulating oracle) <= 0.1 RMS(emulating oracle - exact oracle) at the first and last step."""
    from selftoktokenizer_b200.capi import Engine
    d = C.TINY if geom == "tiny" else C.MID
    g = gold(geom)
    sd = synth.synth_state_dict(d)
    tok, x = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    tb = S.make_tables(d.K, d.stages, d.k_per_stage, 50)
    eng = Engine(d, sd, device=DEV, precision="fp8")
    try:
        for st in (0, 49):
            v = eng.dit_velocity(tok, x, st).cpu()
            emu = _oracle_velocity(sd, d, tok, x, st, tb, True, monkeypatch)
            exact = _oracle_velocity(sd, d, tok, x, st, tb, False, monkeypatch)
            r = _rms(v - emu) / _rms(emu - exact)
            print(f"[fp8 {geom}] step {st}: RMS(engine - emulation) / RMS(emulation - exact) = {r:.4f}, "
                  f"RMS(engine - exact) {_rms(v - exact):.3e}")
            assert r <= 0.1, r
    finally:
        eng.close()


def test_fp8_decode_error_against_reference(eng8, gold, monkeypatch):
    """50-step decode: RMS(engine - reference fixture) <= 2 RMS(emulating oracle - reference fixture)."""
    g = gold("tiny")
    d = C.TINY
    tok, noise = torch.from_numpy(g["tokens"]), torch.from_numpy(g["noise"])
    sd = synth.synth_state_dict(d)
    x = eng8.decode(tok, noise).cpu()
    with monkeypatch.context() as mp:
        mp.setattr(O, "_lin", _e4m3_lin)
        with torch.no_grad():
            emu = O.decode(sd, d, tok, noise, steps=50)
    ref = torch.from_numpy(g["pred_x0"])
    r = _rms(x - ref) / _rms(emu - ref)
    print(f"[fp8 tiny] 50-step decode: RMS(engine - ref) {_rms(x - ref):.3e}, RMS(emulation - ref) {_rms(emu - ref):.3e}, ratio {r:.3f}")
    assert r <= 2.0, r
