"""Kernel-level parity through the C ABI (selftok_k_*): each CUDA kernel against the same op in torch fp64/fp32."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _rand(shape, seed, dev, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dev)


@pytest.mark.parametrize("M,N,K,act", [(300, 192, 64, 0), (1000, 1536, 512, 1), (64, 64, 256, 2), (4096, 64, 1536, 0),
                                        (37, 3072, 512, 0), (512, 16, 512, 0), (130, 130, 16, 0),
                                        (300, 520, 132, 0), (129, 260, 1024, 1)])    # ragged M / N / K on the 128 x 256 tile
def test_linear_f32(dev, M, N, K, act):
    from selftoktokenizer_b200 import capi
    A, W, b = _rand((M, K), 1, dev), _rand((N, K), 2, dev, 1 / math.sqrt(K)), _rand((N,), 3, dev)
    y = capi.k_linear_f32(A, W, b, act)
    ref = A.double() @ W.double().t() + b.double()
    ref = [lambda t: t, lambda t: F.gelu(t, approximate="tanh"), F.silu][act](ref)
    assert (y.double() - ref).abs().max() < 2e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,D,period", [(100, 64, 1), (1000, 1536, 7), (513, 512, 512), (33, 192, 1)])
def test_ln_mod(dev, M, D, period):
    from selftoktokenizer_b200 import capi
    x = _rand((M, D), 4, dev, 3.0) + 0.5
    shift, scale = _rand((period, D), 5, dev), _rand((period, D), 6, dev)
    y = capi.k_ln_mod_f32(x, shift, scale, period)
    idx = torch.arange(M, device=dev) % period
    ref = F.layer_norm(x.double(), (D,), eps=1e-6) * (1 + scale.double()[idx]) + shift.double()[idx]
    assert (y.double() - ref).abs().max() < 2e-5
    y2 = capi.k_ln_mod_f32(x)
    assert (y2.double() - F.layer_norm(x.double(), (D,), eps=1e-6)).abs().max() < 2e-5


@pytest.mark.parametrize("B,Sq,S1,S2,H,hd", [(2, 256, 256, 0, 4, 16), (2, 512, 256, 512, 8, 64), (3, 100, 37, 50, 2, 64),
                                             (1, 768, 768, 0, 3, 64), (2, 16, 16, 0, 4, 16), (2, 32, 16, 32, 2, 64)])
def test_attention_f32(dev, B, Sq, S1, S2, H, hd):
    from selftoktokenizer_b200 import capi
    D = H * hd
    q, k1, v1 = _rand((B, Sq, D), 7, dev), _rand((B, S1, D), 8, dev), _rand((B, S1, D), 9, dev)
    k2 = _rand((B, S2, D), 10, dev) if S2 else None
    v2 = _rand((B, S2, D), 11, dev) if S2 else None
    o = capi.k_attention_f32(q, k1, v1, k2, v2, heads=H)
    k = torch.cat([k1, k2], 1) if S2 else k1
    v = torch.cat([v1, v2], 1) if S2 else v1
    sp = lambda t: t.double().reshape(B, -1, H, hd).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sp(q), sp(k), sp(v)).transpose(1, 2).reshape(B, Sq, D)
    assert (o.double() - ref).abs().max() < 2e-5


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (256, 512, 192), (1000, 576, 192), (4096, 1536, 1536), (48, 192, 768),
                                    (333, 4608, 1536), (2048, 6144, 1536), (1024, 1536, 6144), (129, 260, 128), (257, 256, 64), (1280, 4608, 1536)])
@pytest.mark.parametrize("nsplit", [3, 1, 0])
@pytest.mark.parametrize("ctas", [2, 1])
def test_gemm_tcgen05(dev, M, N, K, nsplit, ctas):
    """Tensor-core GEMM (TMA + wgmma) vs fp64, both with two-CTA clusters sharing the W tile and with one CTA per tile.
    bf16x3 must be fp32-faithful; single-pass bf16 within bf16 rounding."""
    from selftoktokenizer_b200 import capi
    capi.k_set_gemm_ctas(ctas)
    A, W, b = _rand((M, K), 12, dev), _rand((N, K), 13, dev, 1 / math.sqrt(K)), _rand((N,), 14, dev)
    y = capi.k_linear_tc(A, W, b, nsplit)
    torch.cuda.synchronize()
    ref = A.double() @ W.double().t() + b.double()
    err = (y.double() - ref).abs().max().item()
    tol = {3: 2.5e-4, 1: 6e-2, 0: 8e-3}[nsplit]   # bf16x3: ~2^-16 per product, random walk over K; bf16: 2^-9; fp16 (nsplit 0): 2^-12
    assert err < tol, (err, M, N, K, nsplit)
    # and the split really buys precision
    if nsplit == 3 and K >= 192:
        y1 = capi.k_linear_tc(A, W, b, 1)
        assert (y1.double() - ref).abs().max().item() > 30 * err
    capi.k_set_gemm_ctas(2)


@pytest.mark.parametrize("B,S,H,ctx_rows,ctx_keys", [(2, 768, 3, 0, 0), (2, 276, 24, 0, 0), (3, 48, 3, 0, 0), (2, 300, 2, 44, 44),
                                                    (1, 768, 4, 512, 512), (2, 65, 1, 0, 0), (2, 1280, 2, 1024, 1024),
                                                    (3, 640, 5, 384, 384), (2, 700, 3, 300, 300), (5, 129, 2, 0, 0)])
@pytest.mark.parametrize("nsplit", [3, 1, 0])
def test_attention_tensor_core(dev, B, S, H, ctx_rows, ctx_keys, nsplit):
    from selftoktokenizer_b200 import capi
    qkv = _rand((B, S, 3, H, 64), 15, dev)
    o = capi.k_attention_tc(qkv, H, nsplit, ctx_rows, ctx_keys)
    q, k, v = (qkv[:, :, i].double().transpose(1, 2) for i in range(3))
    mask = None
    if ctx_rows:
        mask = torch.ones(S, S, dtype=torch.bool, device=dev)
        mask[:ctx_rows, ctx_keys:] = False
    ref = F.scaled_dot_product_attention(q, k, v, attn_mask=mask).transpose(1, 2).reshape(B, S, H * 64)
    err = (o.double() - ref).abs().max().item()
    # wgmma kernel: 3 = split bf16 (fp32-faithful), 1 = bf16, 0 = IEEE half
    assert err < {3: 3e-5, 1: 2e-2, 0: 3e-3}[nsplit], err
