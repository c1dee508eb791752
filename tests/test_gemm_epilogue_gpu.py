"""Kernel-level tests of the GEMM epilogue contract (kernels.h `Epilogue`) on both GEMM kernels, through selftok_k_gemm:
the fp32 FFMA kernel (path 0) and the wgmma kernel (path 1) in bf16x3 / bf16 / fp16 with one- and two-CTA clusters.

The checks come in two kinds:
- product: EPI_STORE with bias against fp64, with the operands rounded the way the 16-bit planes round them in the
  single-pass modes, to a per-element bound C_TOL * 2^-22 * (sum_k |a_k w_k| + |bias|);
- routing: every other mode against this file's own restatement of the contract, applied to the same kernel's EPI_STORE
  output for the same A, W and bias.  addtab and the 16-bit splits are bitwise, the residual mode within 1 fp32 ulp of
  fma(g, y, r) (the FFMA kernel's r + g * y contracts to one FMA), GELU against fp64 GELU-tanh.
Every output buffer starts as a sentinel, and every element the contract does not address must keep it.

What a +-inf operand gives in bf16x3 is not specified here: its lo plane is inf - inf = NaN, so the product is NaN.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SENT32 = 0x7FA5A5A5          # fp32 sentinel (a NaN bit pattern no kernel produces)
SENT16 = 0x7EA5              # 16-bit plane sentinel
U22 = 2.0 ** -22
# C_TOL = c: the product bound is |y - ref| <= c * 2^-22 * (sum_k |a_k w_k| + |b|) per element.  Largest ratios measured over
# the product and convolution cases on an NVIDIA H100 80GB HBM3 at a 700 W power limit: FFMA 1.71, bf16x3 19.1 (K = 64, where
# the dropped lo * lo terms dominate the accumulation error), bf16 1.65, fp16 2.13.  A one-row or one-column shift of the
# output exceeds these bounds by more than 10x on most elements, which test_product_vs_fp64 asserts.
C_TOL = {"ffma": 4.0, 3: 32.0, 1: 4.0, 0: 4.0}
# GELU-tanh: the FFMA kernel uses tanhf, the wgmma epilogue the MUFU ex2 / rcp form; |err| <= rtol |g| + atol (1 + |y|).
# Largest err / bound measured on the same card with these values: FFMA 0.27, wgmma 0.14.
GELU_TOL = {"ffma": (2.5e-7, 1.25e-7), "wgmma": (1e-6, 1e-7)}

# (path, nsplit, ctas); path 0 ignores nsplit and ctas
CFGS = [(0, 3, 1)] + [(1, ns, ctas) for ns in (3, 1, 0) for ctas in (2, 1)]
_NS_NAME = {3: "x3", 1: "bf16", 0: "fp16"}
CFG_IDS = ["ffma"] + [f"wgmma-{_NS_NAME[ns]}-cta{c}" for ns in (3, 1, 0) for c in (2, 1)]


def _capi():
    from selftoktokenizer_b200 import capi
    return capi


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g, dtype=torch.float64) * scale).float()


def _dev(t):
    return t.to(DEV)


def _i32(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)


def _sent32(rows, ld):
    t = torch.empty(rows, ld, dtype=torch.float32, device=DEV)
    t.view(torch.int32).fill_(SENT32)
    return t


def _sent16(rows, ld):
    return torch.full((rows, ld), SENT16, dtype=torch.int16, device=DEV)


def gemm(cfg, problems):
    capi = _capi()
    path, ns, ctas = cfg
    capi.k_set_gemm_ctas(ctas)
    try:
        capi.k_gemm(path, ns, problems)
    finally:
        capi.k_set_gemm_ctas(2)


def problem(A, W, M, N, K, conv=None, **ep):
    ep = {k: (_i32(v) if isinstance(v, np.ndarray) else v) for k, v in ep.items() if v is not None}
    q = _capi().k_gemm_problem(A, W, M, N, K, conv=conv, **ep)
    q._keep = ep                                          # device index arrays live until the (synchronous) call returns
    return q


def _round_operand(t, nsplit):
    """fp64 copy of an operand as the planes of `nsplit` hold it (bf16x3 and FFMA: the fp32 value itself)."""
    if nsplit == 1:
        return t.to(torch.bfloat16).double()
    if nsplit == 0:
        return t.clamp(-65504, 65504).half().double()
    return t.double()


def _kind(cfg):
    return "ffma" if cfg[0] == 0 else cfg[1]


# ---------------------------------------------------------------------------------------------------------- the restatement
def out_rows(M, rt):
    """Output row of every GEMM row m (kernels.h): row_map, else the token-range plan, else the [image][row] remap, else m."""
    m = np.arange(M)
    if rt.get("row_map") is not None:
        return np.asarray(rt["row_map"], dtype=np.int64)
    rpb_in, rpb_out, row_off = rt.get("rpb_in", 0), rt.get("rpb_out", 0), rt.get("row_off", 0)
    if rt.get("plan") is not None:
        b, r = m // rpb_in, m % rpb_in
        a, c = rt["plan"][b, 0], rt["plan"][b, 1]
        if rt["plan_ctx"]:
            # context stream: an image's slot holds its live rows [a, a + c) first, then its n_img image rows, then its other
            # context rows in stream order
            n_img = rpb_out - rpb_in
            live = (r >= a) & (r < a + c)
            slot = np.where(live, r - a, c + n_img + np.where(r < a, r, r - c))
        else:
            slot = c + r                                  # image stream: after the image's live context rows
        return b * rpb_out + slot
    if rpb_in > 0:
        return (m // rpb_in) * rpb_out + row_off + m % rpb_in
    return m


def table_rows(M, period, tab_rows):
    return np.asarray(tab_rows, dtype=np.int64) if tab_rows is not None else np.arange(M) % period


def bf16_split(y):
    """bf16 hi = rn(y), lo = rn(y - hi) as int16 bit patterns (y fp32, CPU)."""
    hi = y.to(torch.bfloat16)
    lo = (y - hi.float()).to(torch.bfloat16)
    return hi.view(torch.int16), lo.view(torch.int16)


def half_sat(y):
    """IEEE half of y saturated to +-65504 (inf included), NaN kept, as int16 bit patterns."""
    return y.clamp(-65504.0, 65504.0).half().view(torch.int16)


def gelu64(y):
    y = y.double()
    return 0.5 * y * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (y + 0.044715 * y ** 3)))


def _bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def assert_bits_equal(got, exp, what):
    diff = _bits(got) != _bits(exp)
    if diff.any():
        idx = diff.nonzero()[:5].tolist()
        raise AssertionError(f"{what}: {int(diff.sum())} elements differ bitwise, first at {idx}")


# ---------------------------------------------------------------------------------------------------------- product
PRODUCT_SHAPES = [(1, 4, 64, 4), (7, 36, 256, 40), (9, 292, 320, 292), (130, 1536, 64, 1536), (257, 292, 1536, 300),
                  (1000, 36, 320, 36), (1000, 1536, 1536, 1544), (130, 4, 1536, 8)]


def product_ref(A, W, b, nsplit):
    """fp64 reference (on the device) and sum_k |a_k w_k| + |b| of the rounded operands, on the host"""
    a, w, b = _round_operand(_dev(A), nsplit), _round_operand(_dev(W), nsplit), _dev(b).double()
    return (a @ w.t() + b).cpu(), (a.abs() @ w.abs().t() + b.abs()).cpu()


@pytest.mark.parametrize("M,N,K,ldo", PRODUCT_SHAPES)
@pytest.mark.parametrize("cfg", CFGS, ids=CFG_IDS)
def test_product_vs_fp64(cfg, M, N, K, ldo):
    """EPI_STORE + bias: M = 7 / 9 leave row0 + 8 of a thread (or the whole second CTA) invalid, N = 36 / 292 end inside a
    column batch, K = 64 / 256 / 320 / 1536 give 1, 4 (no L2 prefetch point), 5 and 24 k-blocks, ldo > N leaves a pitch gap."""
    A, W, b = _rand((M, K), 1), _rand((N, K), 2, 1 / math.sqrt(K)), _rand((N,), 3)
    out = _sent32(M + 3, ldo)
    gemm(cfg, [problem(_dev(A), _dev(W), M, N, K, bias=_dev(b), out=out, ldo=ldo)])
    out = out.cpu()
    ns = _kind(cfg)
    ref, mag = product_ref(A, W, b, 3 if cfg[0] == 0 else cfg[1])
    ratio = ((out[:M, :N].double() - ref).abs() / (U22 * mag))
    print(f"product ratio {CFG_IDS[CFGS.index(cfg)]} M={M} N={N} K={K}: {ratio.max().item():.4g}")
    assert ratio.max().item() <= C_TOL[ns], (ratio.max().item(), C_TOL[ns])
    # the bound is sharp: a one-column or one-row shift of the output exceeds it by 10x on most elements
    bound = C_TOL[ns] * U22 * mag
    if N > 1:
        assert ((ref[:, 1:] - ref[:, :-1]).abs() / bound[:, 1:]).median() > 10
    if M > 1:
        assert ((ref[1:] - ref[:-1]).abs() / bound[1:]).median() > 10
    assert (out[:, N:].view(torch.int32) == SENT32).all(), "columns [N, ldo) were written"
    assert (out[M:].view(torch.int32) == SENT32).all(), "rows >= M were written"


# ---------------------------------------------------------------------------------------------------------- routing
_PB, _KC, _NI = 5, 70, 33
_S = _KC + _NI
_rng = np.random.default_rng(7)
_a, _c = int(_rng.integers(1, 30)), int(_rng.integers(1, 30))
PLAN = np.array([[0, 0], [0, _KC], [_a, _c], [int(_rng.integers(0, 20)), int(_rng.integers(20, 50))], [_KC - 3, 3]], dtype=np.int64)
_MAP_M = 300
ROUTES = {
    "plain": dict(M=257, N=292, K=320, ldo=296, rows=257 + 2),
    "remap": dict(M=130, N=36, K=64, ldo=40, rows=4 * 45, rpb_in=40, rpb_out=45, row_off=3),
    "plan_ctx": dict(M=_PB * _KC, N=292, K=256, ldo=296, rows=_PB * _S, rpb_in=_KC, rpb_out=_S, row_off=0, plan_ctx=1, plan=PLAN),
    "plan_img": dict(M=_PB * _NI, N=292, K=256, ldo=296, rows=_PB * _S, rpb_in=_NI, rpb_out=_S, row_off=_KC, plan_ctx=0, plan=PLAN),
    "row_map": dict(M=_MAP_M, N=36, K=1536, ldo=36, rows=2 * _MAP_M + 5,
                    row_map=np.random.default_rng(8).permutation(2 * _MAP_M + 5)[:_MAP_M],
                    tab_rows=np.random.default_rng(9).integers(0, 11, _MAP_M)),
}
MODES = ["store", "store_nobias", "store_gelu", "add_p1", "add_p7", "add_tab", "gelu_add", "resid_nogate", "resid_g1",
         "resid_gP", "resid_tab", "resid_inplace", "split_x3", "split_hi", "split_fp16", "split_gelu_x3", "split_gelu_fp16"]
T_ROWS = 11


def _route_ep(rt):
    return {k: rt[k] for k in ("rpb_in", "rpb_out", "row_off", "plan_ctx", "plan", "row_map", "tab_rows") if k in rt}


class _Case:
    def __init__(self, cfg, route, big_bias=False):
        rt = ROUTES[route]
        self.cfg, self.rt = cfg, rt
        self.M, self.N, self.K, self.ldo, self.rows = rt["M"], rt["N"], rt["K"], rt["ldo"], rt["rows"]
        self.A, self.W = _rand((self.M, self.K), 11), _rand((self.N, self.K), 12, 1 / math.sqrt(self.K))
        self.b = _rand((self.N,), 13)
        if big_bias:                                      # drives y past +-65504 in alternate columns
            self.b = self.b + torch.tensor([7e4, -9e4, 0.0, 65500.0] * (self.N // 4))
        self.dA, self.dW, self.db = _dev(self.A), _dev(self.W), _dev(self.b)
        self.orow = out_rows(self.M, rt)
        self._y = {}

    def run(self, **ep):
        gemm(self.cfg, [problem(self.dA, self.dW, self.M, self.N, self.K, ldo=self.ldo, **{**_route_ep(self.rt), **ep})])

    def y(self, act="none", bias=True):
        """the kernel's own EPI_STORE output (plain rows) for this A, W and bias"""
        key = (act, bias)
        if key not in self._y:
            out = _sent32(self.M, self.ldo)
            gemm(self.cfg, [problem(self.dA, self.dW, self.M, self.N, self.K, ldo=self.ldo, act=act, out=out,
                                    bias=self.db if bias else None)])
            self._y[key] = out[:, :self.N].cpu()
        return self._y[key]


def _check_untouched(got, init, rows_written, N, what):
    mask = torch.ones(got.shape[0], dtype=torch.bool)
    mask[torch.from_numpy(np.asarray(rows_written))] = False
    assert torch.equal(_bits(got[mask]), _bits(init[mask])), f"{what}: unaddressed rows written"
    assert torch.equal(_bits(got[:, N:]), _bits(init[:, N:])), f"{what}: columns [N, ldo) written"


def _ulp32(x64):
    x32 = x64.float().abs()
    return torch.from_numpy(np.spacing(x32.numpy())).double()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("route", list(ROUTES))
@pytest.mark.parametrize("cfg", CFGS, ids=CFG_IDS)
def test_epilogue_routing(cfg, route, mode):
    c = _Case(cfg, route, big_bias=mode == "split_fp16")
    M, N, ldo, rows, orow = c.M, c.N, c.ldo, c.rows, c.orow
    rt_tab = c.rt.get("tab_rows")
    kind = "ffma" if cfg[0] == 0 else "wgmma"

    if mode.startswith("store") or mode.startswith("add") or mode == "gelu_add":
        act = "gelu" if "gelu" in mode else "none"
        bias = mode != "store_nobias"
        ep = dict(mode="store", act=act, bias=c.db if bias else None)
        add = tab = None
        if mode.startswith("add") or mode == "gelu_add":
            period = {"add_p1": 1, "add_p7": 7}.get(mode, T_ROWS)
            tab = rt_tab if rt_tab is not None else (np.random.default_rng(3).integers(0, T_ROWS, M) if mode == "add_tab" else None)
            add_ld = N + 4 if mode == "add_p7" else N
            add = _rand((max(period, T_ROWS), add_ld), 21)
            ep.update(addtab=_dev(add), add_ld=add_ld, add_period=period, tab_rows=tab)
            trow = table_rows(M, period, tab)
        out = _sent32(rows, ldo)
        init = out.cpu()
        c.run(out=out, **ep)
        got = out.cpu()
        y = c.y(act, bias)
        _check_untouched(got, init, orow, N, mode)
        if mode == "store_gelu":
            y0 = c.y("none", True)
            g = gelu64(y0)
            rtol, atol = GELU_TOL[kind]
            err = (got[orow, :N].double() - g).abs() / (rtol * g.abs() + atol * (1 + y0.double().abs()))
            print(f"gelu ratio {CFG_IDS[CFGS.index(cfg)]} {route}: {err.max().item():.4g}")
            assert err.max().item() <= 1, err.max().item()
        # the routed output is the plain output, plus one fp32 add of the addtab row
        exp = y if add is None else y + add[torch.from_numpy(trow), :N]
        assert_bits_equal(got[orow, :N], exp, mode)

    elif mode.startswith("resid"):
        y = c.y()
        gate = None
        ep = dict(mode="resid", bias=c.db)
        trow = np.zeros(M, dtype=np.int64)
        if mode != "resid_nogate":
            period = {"resid_g1": 1, "resid_gP": 5}.get(mode, T_ROWS)
            tab = rt_tab if rt_tab is not None else (np.random.default_rng(4).integers(0, T_ROWS, M) if mode == "resid_tab" else None)
            gate_ld = N + 8 if mode in ("resid_gP", "resid_inplace") else N
            gate = _rand((max(period, T_ROWS), gate_ld), 22)
            ep.update(gate=_dev(gate), gate_ld=gate_ld, gate_period=period, tab_rows=tab)
            trow = table_rows(M, period, tab)
        r = _rand((rows, ldo), 23)
        resid = _dev(r)
        out = resid if mode == "resid_inplace" else _sent32(rows, ldo)
        init = out.cpu()
        c.run(out=out, resid=resid, **ep)
        got = out.cpu()
        _check_untouched(got, init, orow, N, mode)
        g = torch.ones(M, N, dtype=torch.float64) if gate is None else gate[torch.from_numpy(trow), :N].double()
        exp = g * y.double() + r[orow, :N].double()                  # fp32 * fp32 is exact in fp64
        err = (got[orow, :N].double() - exp).abs()
        assert (err <= _ulp32(exp)).all(), (err / _ulp32(exp)).max().item()
        if mode == "resid_inplace":                                  # in place == out of place, bitwise
            out2 = _sent32(rows, ldo)
            c.run(out=out2, resid=_dev(r), **ep)
            assert_bits_equal(got[orow, :N], out2.cpu()[orow, :N], "in place vs out of place")

    else:
        gelu = "gelu" in mode
        fp16 = mode.endswith("fp16")
        lo = mode.endswith("x3")
        hi_p, lo_p = _sent16(rows, ldo), (_sent16(rows, ldo) if lo else None)
        c.run(mode="split", act="gelu" if gelu else "none", bias=c.db, out_hi=hi_p, out_lo=lo_p, fp16=int(fp16))
        y = c.y("gelu" if gelu else "none")
        hi_g = hi_p.cpu()
        _check_untouched(hi_g, _sent16(rows, ldo).cpu(), orow, N, mode + " hi")
        if fp16:
            assert_bits_equal(hi_g[orow, :N], half_sat(y), mode)
            if mode == "split_fp16":
                assert (y.abs() > 65504).any() and not torch.isinf(hi_g[orow, :N].view(torch.float16)).any()
        else:
            h, l = bf16_split(y)
            assert_bits_equal(hi_g[orow, :N], h, mode + " hi")
            if lo:
                lo_g = lo_p.cpu()
                _check_untouched(lo_g, _sent16(rows, ldo).cpu(), orow, N, mode + " lo")
                assert_bits_equal(lo_g[orow, :N], l, mode + " lo")


# ---------------------------------------------------------------------------------------------------------- grouped launches
def _grouped_pair(kind, ns):
    """The engine's two pairs: context + image EPI_RESID (gate period Kc / 1, in place), and the QKV SPLIT pair through the
    token-range plan into one joint buffer.  Problem 0 has an odd number of k-blocks, problem 1 an even one, and together
    they have more cluster tiles than the grid has clusters, so CTAs cross from one problem into the other."""
    if kind == "resid":
        Kc, imgs = 125, 8
        specs = [(Kc * imgs, 1536, 320), (4096, 1024, 256)]
        probs = []
        for i, (M, N, K) in enumerate(specs):
            gate_ld = N + 8
            period = Kc if i == 0 else 1
            probs.append(dict(M=M, N=N, K=K, A=_rand((M, K), 30 + i), W=_rand((N, K), 40 + i, 1 / math.sqrt(K)), b=_rand((N,), 50 + i),
                              gate=_rand((period, gate_ld), 60 + i), gate_ld=gate_ld, period=period, r=_rand((M, N + 4), 70 + i)))
        return probs
    B, Kc, NI, N = 16, 128, 256, 1536
    S = Kc + NI
    rng = np.random.default_rng(5)
    plan = np.stack([rng.integers(0, Kc // 2, B), rng.integers(0, Kc // 2, B)], 1)
    plan[0] = (0, Kc)
    plan[1] = (0, 0)
    common = dict(N=N, plan=plan, S=S, B=B, fp16=int(ns == 0), lo=ns == 3)
    return [dict(common, M=B * Kc, K=320, rpb_in=Kc, row_off=0, plan_ctx=1, A=_rand((B * Kc, 320), 31), W=_rand((N, 320), 41, 0.05), b=_rand((N,), 51)),
            dict(common, M=B * NI, K=256, rpb_in=NI, row_off=Kc, plan_ctx=0, A=_rand((B * NI, 256), 32), W=_rand((N, 256), 42, 0.0625), b=_rand((N,), 52))]


def _launch_pair(cfg, kind, probs, grouped):
    if kind == "resid":
        outs = [_dev(p["r"]) for p in probs]
        qs = [problem(_dev(p["A"]), _dev(p["W"]), p["M"], p["N"], p["K"], mode="resid", bias=_dev(p["b"]), out=o, resid=o, ldo=p["N"] + 4,
                      gate=_dev(p["gate"]), gate_ld=p["gate_ld"], gate_period=p["period"]) for p, o in zip(probs, outs)]
    else:
        p0 = probs[0]
        hi = _sent16(p0["B"] * p0["S"], p0["N"])
        lo = _sent16(p0["B"] * p0["S"], p0["N"]) if p0["lo"] else None
        outs = [hi] + ([lo] if lo is not None else [])
        qs = [problem(_dev(p["A"]), _dev(p["W"]), p["M"], p["N"], p["K"], mode="split", bias=_dev(p["b"]), out_hi=hi, out_lo=lo, ldo=p["N"],
                      fp16=p["fp16"], rpb_in=p["rpb_in"], rpb_out=p["S"], row_off=p["row_off"], plan_ctx=p["plan_ctx"], plan=p["plan"])
              for p in probs]
    if grouped:
        gemm(cfg, qs)
    else:
        for q in qs:
            gemm(cfg, [q])
    return [o.cpu() for o in outs]


@pytest.mark.parametrize("kind", ["resid", "split"])
@pytest.mark.parametrize("cfg", CFGS[1:], ids=CFG_IDS[1:])
def test_grouped_equals_solo(cfg, kind):
    probs = _grouped_pair(kind, cfg[1])
    solo = _launch_pair(cfg, kind, probs, grouped=False)
    both = _launch_pair(cfg, kind, probs, grouped=True)
    for s, g in zip(solo, both):
        assert_bits_equal(g, s, f"grouped {kind}")
    if kind == "split":                                   # every slot row is written by exactly one of the two problems
        assert not (solo[0] == SENT16).all(1).any()


# ---------------------------------------------------------------------------------------------------------- row invariance
@pytest.mark.parametrize("ns", [3, 1, 0])
def test_wgmma_row_invariance(ns):
    """A GEMM row's result does not depend on M, the cluster mode or grouping: the first 130 rows, bitwise."""
    R, N, K = 130, 292, 320
    A, W, b = _dev(_rand((4096, K), 80)), _dev(_rand((N, K), 81, 1 / math.sqrt(K))), _dev(_rand((N,), 82))
    results = []
    for M in (R + 1, 1000, 4096):
        for ctas in (2, 1):
            out = _sent32(M, N)
            gemm((1, ns, ctas), [problem(A[:M], W, M, N, K, bias=b, out=out, ldo=N)])
            results.append(out[:R].cpu())
        other = _sent32(2048, 1536)
        out = _sent32(M, N)
        A2, W2 = _dev(_rand((2048, 256), 83)), _dev(_rand((1536, 256), 84, 0.0625))
        gemm((1, ns, 2), [problem(A2, W2, 2048, 1536, 256, out=other, ldo=1536), problem(A[:M], W, M, N, K, bias=b, out=out, ldo=N)])
        results.append(out[:R].cpu())
    for r in results[1:]:
        assert_bits_equal(r, results[0], "row invariance")


def test_ffma_row_invariance():
    """The FFMA kernel sums in a fixed k order, so the 64 x 64 and 128 x 128 tile kernels agree bitwise."""
    K = 320
    A, W, b = _dev(_rand((1000, K), 85)), _dev(_rand((128, K), 86, 1 / math.sqrt(K))), _dev(_rand((128,), 87))
    res = {}
    for M, N in ((64, 128), (65, 128), (1000, 128), (1000, 64), (64, 64)):
        out = _sent32(M, N)
        gemm(CFGS[0], [problem(A[:M], W[:N], M, N, K, bias=b, out=out, ldo=N)])
        res[(M, N)] = out.cpu()
    for key, r in res.items():
        n = key[1]
        assert_bits_equal(r[:64, :n], res[(64, 128)][:, :n], f"FFMA rows at {key}")


# ---------------------------------------------------------------------------------------------------------- implicit convolution
CONVS = [  # (C, images, H, W, stride): H, W = output dims
    (64, 2, 2, 256, 1),      # a 128-pixel tile is part of a row
    (128, 2, 4, 64, 1),      # two whole rows per tile
    (64, 3, 8, 16, 1),       # one whole image per tile
    (128, 3, 8, 8, 1),       # two images per tile (the last tile half past the end)
    (64, 2, 8, 16, 2),
    (64, 2, 64, 64, 2),
]


@pytest.mark.parametrize("C,imgs,H,Wd,stride", CONVS)
@pytest.mark.parametrize("cfg", CFGS[1:], ids=CFG_IDS[1:])
def test_conv_vs_fp64(cfg, C, imgs, H, Wd, stride):
    ns = cfg[1]
    N = 128
    Hin, Win = H * stride, Wd * stride
    x = _rand((imgs, Hin, Win, C), 90)                                        # NHWC input
    w = _rand((N, C, 3, 3), 91, 1 / math.sqrt(9 * C))
    b = _rand((N,), 92)
    Wmat = w.permute(0, 2, 3, 1).reshape(N, 9 * C).contiguous()              # K index (ky * 3 + kx) * C + c
    if stride == 1:
        Aop = x
    else:                                                                     # polyphase planes [img * 4 + py * 2 + px, H, W, C]
        Aop = torch.stack([x[:, py::2, px::2] for py in (0, 1) for px in (0, 1)], 1).reshape(imgs * 4, H, Wd, C)
    M = imgs * H * Wd
    out = _sent32(M, N)
    conv = (C, H, Wd, stride)
    gemm(cfg, [problem(_dev(Aop.contiguous()), _dev(Wmat), M, N, 9 * C, conv=conv, bias=_dev(b), out=out, ldo=N)])
    y = out.cpu()
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
    print(f"conv ratio {CFG_IDS[CFGS.index(cfg)]} C={C} {H}x{Wd} s{stride}: {ratio.max().item():.4g}")
    assert ratio.max().item() <= C_TOL[ns], ratio.max().item()
    # the VAE's residual epilogue on the same convolution
    r = _rand((M, N), 93)
    out2 = _sent32(M, N)
    gemm(cfg, [problem(_dev(Aop.contiguous()), _dev(Wmat), M, N, 9 * C, conv=conv, mode="resid", bias=_dev(b), out=out2,
                       resid=_dev(r), ldo=N)])
    exp = y.double() + r.double()
    assert ((out2.cpu().double() - exp).abs() <= _ulp32(exp)).all()


@pytest.mark.parametrize("C,H,Wd,stride", [(64, 4, 96, 1), (96, 8, 16, 1), (64, 8, 8, 2), (64, 3, 64, 1)])
def test_conv_rejects_untiled_geometry(C, H, Wd, stride):
    """Geometries the 128-pixel tiling does not cover are SELFTOK_ERR_UNSUPPORTED, before any launch."""
    capi = _capi()
    M, N = 2 * H * Wd, 64
    A = torch.zeros(M * C * (4 if stride == 2 else 1), device=DEV)
    W, out = torch.zeros(N, 9 * C, device=DEV), _sent32(M, N)
    st = capi.k_gemm_status(1, 3, [problem(A, W, M, N, 9 * C, conv=(C, H, Wd, stride), out=out, ldo=N)])
    assert st == -2, st
    assert (out.view(torch.int32) == SENT32).all()


# ---------------------------------------------------------------------------------------------------------- conversion edges
@pytest.mark.parametrize("cfg", CFGS, ids=CFG_IDS)
def test_nan_row_stays_nan(cfg):
    """A NaN in one row of A gives a NaN output row in every path and precision (the fp16 A planes used to clamp it to
    -65504), in the fp32 output and in the 16-bit planes."""
    M, N, K = 130, 292, 320
    A, W, b = _rand((M, K), 94), _rand((N, K), 95, 1 / math.sqrt(K)), _rand((N,), 96)
    nan_rows = [0, 9, 129]
    for i, r in enumerate(nan_rows):
        A[r, 37 * i + 5] = float("nan")
    dA, dW, db = _dev(A), _dev(W), _dev(b)
    out = _sent32(M, N)
    gemm(cfg, [problem(dA, dW, M, N, K, bias=db, out=out, ldo=N)])
    y = out.cpu()
    ok = torch.ones(M, dtype=torch.bool)
    ok[nan_rows] = False
    assert torch.isnan(y[nan_rows]).all(), "a NaN row of A came out (partly) finite"
    assert torch.isfinite(y[ok]).all()
    for fp16 in (0, 1):
        hi = _sent16(M, N)
        gemm(cfg, [problem(dA, dW, M, N, K, mode="split", bias=db, out_hi=hi, fp16=fp16, ldo=N)])
        h = hi.cpu().view(torch.float16 if fp16 else torch.bfloat16)
        assert torch.isnan(h[nan_rows]).all() and torch.isfinite(h[ok]).all()


SPECIAL = [7e4, -7e4, float("inf"), float("-inf"), float("nan"), 65504.0, -65504.0, 65519.99, 65520.0, -65520.0, 1e-8, 2.9802322e-08,
           -2.9802322e-08, 5.9604645e-08, 0.0, -0.0, 1.00048828125, 1.00146484375, 6.1035156e-05, -3e38, 3.4028235e38, 0.333333343]


def test_fp16_split_saturates_and_is_the_same_on_both_kernels():
    """y = 0 * W + bias = bias exactly on every path, so the fp16 split planes of the two kernels must be the same bits:
    saturation of +-inf and |y| > 65504 to +-65504, NaN kept, ties and subnormals rounded to nearest even."""
    N = ((len(SPECIAL) + 3) // 4) * 4
    M, K = 9, 64
    b = torch.tensor(SPECIAL + [1.0] * (N - len(SPECIAL)), dtype=torch.float32)
    A, W = torch.zeros(M, K), _rand((N, K), 97)
    planes = {}
    for cfg, cid in zip(CFGS, CFG_IDS):
        hi = _sent16(M, N)
        gemm(cfg, [problem(_dev(A), _dev(W), M, N, K, mode="split", bias=_dev(b), out_hi=hi, fp16=1, ldo=N)])
        planes[cid] = hi.cpu()
    exp = half_sat(b + 0.0).expand(M, N)          # 0 + -0.0 is +0.0
    for cid, p in planes.items():
        fin = ~torch.isnan(b).expand(M, N)
        assert torch.equal(p[fin], exp[fin]), cid
        assert torch.isnan(p.view(torch.float16)[~fin]).all(), cid
        assert torch.equal(p, planes["ffma"]), f"{cid} differs from the FFMA kernel"


@pytest.mark.parametrize("ns", [0, 1])
def test_operand_conversion_saturates(ns):
    """A operands past the half range: the fp16 planes hold +-65504 (inf included), bf16 keeps them."""
    M, N, K = 9, 36, 64
    A, W, b = _rand((M, K), 98), _rand((N, K), 99, 1 / math.sqrt(K)), _rand((N,), 100)
    A[1, 3], A[2, 7], A[3, 11], A[4, 0] = 1e5, -2e5, float("inf"), float("-inf")
    out = _sent32(M, N)
    gemm((1, ns, 2), [problem(_dev(A), _dev(W), M, N, K, bias=_dev(b), out=out, ldo=N)])
    y = out.cpu()
    if ns == 1:
        assert torch.isinf(y[3:5]).all()
        rows = [0, 1, 2, 5, 6, 7, 8]
    else:
        rows = list(range(M))
    ref, mag = product_ref(A[rows], W, b, ns)
    assert ((y[rows].double() - ref).abs() <= C_TOL[ns] * U22 * mag).all()
