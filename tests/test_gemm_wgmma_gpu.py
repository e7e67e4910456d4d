"""The wgmma GEMM (gemm_wgmma.cuh) against the fp64 reference of tests/parity.py, per element, at its tile edges:
every tile width x epilogue (staged and direct stores), ragged M / N, K tails, split-K with empty splits, the 3x3
implicit-GEMM conv, and the swap-AB decode GEMM at the Groma-7B weight shapes with every flag the engine can set."""
import math
from types import SimpleNamespace

import pytest
import torch

from tests import parity as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def G():
    from groma_b200 import ops
    return ops


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


def ref_acc(a, w):
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


# (name, kwargs for ops.gemm); residual / gamma / bias tensors are filled in by run_epilogue
EPILOGUES = ["none", "bias", "bias_gelu", "bias_relu", "bias_gamma_residual", "inplace_residual", "bias_swiglu", "f32"]


def run_epilogue(G, a, w, acc, mag, epi, bn, layout, seed=0):
    """Run one epilogue through ops.gemm into a view of a wider buffer and check it against the fp64 reference.
    layout 'staged': row stride a multiple of 8 (shared-memory staged bf16 stores);  'direct': row stride N + 3."""
    M, N = acc.shape
    bias = rnd(N, seed=seed + 1)
    gamma = rnd(N, seed=seed + 2)
    act = {"bias_gelu": G.ACT_GELU, "bias_relu": G.ACT_RELU, "bias_swiglu": G.ACT_SWIGLU}.get(epi, G.ACT_NONE)
    n_out = N // 2 if act == G.ACT_SWIGLU else N
    width = (n_out + 7) // 8 * 8 + 8 if layout == "staged" else n_out + 3
    f32 = epi == "f32"
    buf = torch.full((M, width), 7.0, dtype=torch.float32 if f32 else torch.bfloat16, device="cuda")
    out = buf[:, :n_out]
    kw = dict(block_n=bn, out=out)
    if epi != "none":
        kw["bias"] = bias
    if act != G.ACT_NONE:
        kw["act"] = act
    res_buf = None
    if epi in ("bias_gamma_residual", "inplace_residual"):
        res_buf = rnd(M, width, seed=seed + 3).bfloat16()
        if epi == "bias_gamma_residual":
            kw["gamma"] = gamma
            kw["residual"] = res_buf[:, :n_out]
        else:
            buf = res_buf.clone()
            kw["out"] = kw["residual"] = out = buf[:, :n_out]
    G.gemm(a, w, **kw)
    ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=kw.get("bias"), act=act, gamma=kw.get("gamma"),
                                    residual=res_buf[:, :n_out] if res_buf is not None else None)
    P.check_gemm(out, ref, lmag, out_f32=f32, what=f"M={M} N={N} K={a.shape[1]} block_n={bn} {epi} {layout}")
    pad = buf[:, n_out:]
    if epi == "inplace_residual":
        assert torch.equal(pad, res_buf[:, n_out:]), "columns past N were written"
    else:
        assert (pad == 7.0).all(), "columns past N were written"


# M % 128 in {1, 63, 64, 65, 127}; N % 8 != 0 and N / 2 odd (SwiGLU output tail); K with a partial last k-block
@pytest.mark.parametrize("bn,M,N,K", [
    (16, 129, 50, 592),
    (32, 191, 94, 320),
    (64, 320, 198, 256),
    (128, 449, 394, 200),
    (256, 383, 790, 256),
    (512, 641, 1046, 192),       # two-CTA cluster: 256-row tiles, M % 256 = 129
    (128, 4033, 4094, 256),      # 1024 tiles on ~132 CTAs: every CTA reuses its bias / gamma staging and ring phase
    (256, 4033, 4094, 128),
])
@pytest.mark.parametrize("layout", ["staged", "direct"])
def test_gemm_tile_width_x_epilogue(G, bn, M, N, K, layout):
    a = rnd(M, K, seed=M).bfloat16()
    w = rnd(N, K, seed=N, scale=1.0 / math.sqrt(K)).bfloat16()
    acc, mag = ref_acc(a, w)
    for i, epi in enumerate(EPILOGUES):
        run_epilogue(G, a, w, acc, mag, epi, bn, layout, seed=10 * i)


@pytest.mark.parametrize("K", [8, 16, 40, 72, 592])
@pytest.mark.parametrize("bn", [16, 64, 128, 256, 512])
def test_gemm_k_tails(G, K, bn):
    """K < 64 and K % 64 != 0: the TMA box runs past the row end and must zero-fill."""
    M, N = 257, 300
    a = rnd(M, K, seed=K).bfloat16()
    w = rnd(N, K, seed=K + 1).bfloat16()
    acc, mag = ref_acc(a, w)
    for epi in ("bias_gelu", "f32"):
        run_epilogue(G, a, w, acc, mag, epi, bn, "staged", seed=K)


def test_gemm_splitk_empty_splits(G):
    """K = 256 (4 k-blocks) in 6 splits: two splits get no k-block and must contribute zeros."""
    M, N, K, split = 300, 520, 256, 6
    a = rnd(M, K, seed=1).bfloat16(); w = rnd(N, K, seed=2, scale=1 / 16).bfloat16()
    bias, gamma, res = rnd(N, seed=3), rnd(N, seed=4), rnd(M, N, seed=5).bfloat16()
    acc, mag = ref_acc(a, w)
    ws = torch.full((split, M, N), float("nan"), device="cuda")
    out = G.gemm_splitk(a, w, split, bias=bias, act=G.ACT_GELU, gamma=gamma, residual=res, ws=ws)
    assert (ws[4:] == 0).all()
    ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=bias, act=G.ACT_GELU, gamma=gamma, residual=res)
    P.check_gemm(out, ref, lmag, what="split-K 6 of K=256 gelu+gamma+residual")
    out = G.gemm_splitk(a, w, split, act=G.ACT_SWIGLU, bias=bias)
    ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=bias, act=G.ACT_SWIGLU)
    P.check_gemm(out, ref, lmag, what="split-K 6 of K=256 swiglu")
    out = G.gemm_splitk(a, w, split, out_f32=True)
    P.check_gemm(out, acc, mag, out_f32=True, what="split-K 6 of K=256 fp32")


@pytest.mark.parametrize("B", [1, 3, 16])
def test_gemm_swap_ab_fused_empty_splits(G, B):
    """One-launch split-K (the last CTA of a tile reduces): empty splits, residual, SwiGLU, fp32 out; counters re-armed."""
    N, K, split = 1000, 256, 6
    x = rnd(B, K, seed=B).bfloat16(); w = rnd(N, K, seed=7, scale=1 / 16).bfloat16()
    acc, mag = ref_acc(x, w)
    counters = torch.zeros(64, dtype=torch.int32, device="cuda")
    ws = torch.empty(split * N * B, device="cuda")
    res = rnd(B, N, seed=8).bfloat16()
    for act, residual, dt in ((G.ACT_NONE, res, torch.bfloat16), (G.ACT_SWIGLU, None, torch.bfloat16), (G.ACT_NONE, None, torch.float32)):
        n_out = N // 2 if act == G.ACT_SWIGLU else N
        out = torch.full((B, n_out), 7.0, dtype=dt, device="cuda")
        G.gemm_swap_ab_fused(x, w, ws, counters, split, out, act=act, residual=residual)
        ref, lmag = P.gemm_epilogue_ref(acc, mag, act=act, residual=residual)
        P.check_gemm(out, ref, lmag, out_f32=dt == torch.float32, what=f"swap-AB fused B={B} split 6 act={act} {dt}")
        assert (counters == 0).all(), "tile counters not re-armed"


def test_conv3x3_block_n_256_vs_fp64(G):
    import torch.nn.functional as F
    n_img, H, W, C, Cout, L = 3, 14, 14, 128, 256, 3
    xs = [rnd(n_img, C, H, W, seed=20 + l).bfloat16() for l in range(L)]
    ws = [rnd(Cout, C, 3, 3, seed=30 + l, scale=0.05).bfloat16() for l in range(L)]
    bias = rnd(Cout, seed=40)
    acc = sum(F.conv2d(x.double(), w_.double(), padding=1) for x, w_ in zip(xs, ws)).permute(0, 2, 3, 1).reshape(-1, Cout)
    mag = sum(F.conv2d(x.double().abs(), w_.double().abs(), padding=1) for x, w_ in zip(xs, ws)).permute(0, 2, 3, 1).reshape(-1, Cout)
    ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=bias, act=G.ACT_RELU)
    xpad = torch.zeros((L, n_img, H + 2, W + 2, C), dtype=torch.bfloat16, device="cuda")
    for l in range(L):
        xpad[l, :, 1:-1, 1:-1] = xs[l].permute(0, 2, 3, 1)
    wt = torch.cat([w_.permute(0, 2, 3, 1).reshape(Cout, 9 * C) for w_ in ws], dim=1).contiguous()
    out = G.conv3x3_flat(xpad.reshape(-1, C), wt, n_img, H + 2, W + 2, bias=bias, act=G.ACT_RELU, block_n=256)
    P.check_gemm(out, ref, lmag, what="conv3x3 27 taps block_n=256 bias+relu")


# ------------------------------------------------------------------------------------------------- swap-AB decode GEMM
WEIGHTS = {"qkv": (12288, 4096), "o": (4096, 4096), "gu": (22016, 4096), "down": (4096, 11008), "head": (32114, 4096)}


def engine_splits():
    from groma_b200.config import PathConfig
    from groma_b200.engine import GromaEngine
    stub = SimpleNamespace(cfg=PathConfig(), sms=torch.cuda.get_device_properties(0).multi_processor_count)
    return GromaEngine._decode_splits(stub)


def split_with_empty(K, above):
    """Smallest split factor > above for which some splits receive no 64-deep k-block."""
    kb = (K + 63) // 64
    s = above + 1
    while True:
        per = (kb + s - 1) // s
        if (kb + per - 1) // per < s:
            return s
        s += 1


@pytest.mark.parametrize("name", list(WEIGHTS))
def test_gemm_swap_ab_groma7b_shapes(G, name):
    """ws[split] partials (token-major when transposed) summed over splits == x @ W^T, for every flag combination the
    decode step can use: transposed store, PDL weight prefetch, tile-major weights; batch 1 / 3 / 16 (a full 16-column tile)."""
    N, K = WEIGHTS[name]
    W = rnd(N, K, seed=N + K, scale=1.0 / math.sqrt(K)).bfloat16()
    Wt = G.tile_weight(W)
    W64a = W.double().abs()
    s0 = engine_splits()[name]
    for split in (s0, split_with_empty(K, s0)):
        for B in (1, 3, 16):
            x = rnd(B, K, seed=B).bfloat16()
            ref = x.double() @ W.double().t()
            mag = x.double().abs() @ W64a.t()
            for transposed in (False, True):
                for pdl in (False, True):
                    for tiled in (False, True):
                        shape = (split, B, N) if transposed else (split, N, B)
                        ws = torch.full(shape, float("nan"), device="cuda")
                        if tiled:
                            G.gemm_swap_ab(x, Wt, ws, split_k=split, pdl=pdl, transposed=transposed, tiled=True, n_rows=N)
                        else:
                            G.gemm_swap_ab(x, W, ws, split_k=split, pdl=pdl, transposed=transposed)
                        got = ws.double().sum(0)
                        got = got if transposed else got.t()
                        P.check_gemm(got, ref, mag, out_f32=True,
                                     what=f"swap-AB {name} B={B} split={split} transposed={transposed} pdl={pdl} tiled={tiled}")


def test_gemm_swap_ab_pdl_waits_for_producer(G):
    """A PDL swap-AB GEMM launched right behind splitk_reduce (which releases its dependents at its first instruction) must
    read the activations the reduce writes, not the stale ones: only the weights may be fetched before griddepcontrol.wait."""
    N, K, B, splits = 4096, 4096, 16, 512
    W = rnd(N, K, seed=1, scale=1.0 / 64).bfloat16()
    x_new = rnd(B, K, seed=2).bfloat16()
    x = (-x_new.float() + 3.0).bfloat16()            # stale values
    red = torch.zeros((splits, B, K), device="cuda")  # 128 MB of partials: the reduce runs long enough to overlap
    red[-1] = x_new.float()
    ws = torch.full((1, B, N), float("nan"), device="cuda")
    torch.cuda.synchronize()
    G.splitk_reduce(red, x)
    G.gemm_swap_ab(x, W, ws, split_k=1, pdl=True, transposed=True)
    torch.cuda.synchronize()
    assert torch.equal(x, x_new)
    ref = x_new.double() @ W.double().t()
    mag = x_new.double().abs() @ W.double().abs().t()
    P.check_gemm(ws[0], ref, mag, out_f32=True, what="swap-AB pdl after splitk_reduce")
