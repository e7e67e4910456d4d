"""The per-element comparators of tests/parity.py must accept the kernels' own rounding and reject small, plausible defects.

A CPU model of each kernel's rounding points stands in for the kernel:
  GEMM       bf16 operands, fp32 accumulation one 64-deep k-block at a time (as the wgmma main loop retires them), fp32
             epilogue (bias -> act -> gamma -> residual), bf16 output;
  attention  fp32 scores, online softmax over 128-key tiles (running max, rescale, fp32 row sums of the unrounded
             probabilities), P rounded to bf16 for the PV product, fp32 O, O / l rounded to bf16; the 128-row query tile is
             two 64-row warpgroups.
  decode     split-K partials summed in split order in fp32, then the epilogue of csrc/llama_decode.cu: residual add and
             RMSNorm with its two bf16 rounding points, SwiGLU, or RoPE of bf16-rounded sums with fp32 tables.
The model must pass; each mutation below (one defect the kernels could plausibly have) must fail."""
import math

import pytest
import torch

from tests import parity as P


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def bf16(t):
    return t.bfloat16().float()


# ------------------------------------------------------------------------------------------------- GEMM
M, N, K, BN = 300, 520, 4096, 256


@pytest.fixture(scope="module")
def gemm_case():
    # weights ~ 1/sqrt(K)-ish as in a trained layer: bias and residual are of the accumulator's order
    a, w = bf16(rnd(M, K, seed=1)), bf16(rnd(N, K, seed=2, scale=0.05))
    bias, gamma, res = rnd(N, seed=3), rnd(N, seed=4), bf16(rnd(M, N, seed=5))
    # fp32 accumulators, one 64-deep k-block at a time
    blocks = [a[:, k0:k0 + 64] @ w[:, k0:k0 + 64].t() for k0 in range(0, K, 64)]
    return dict(a=a, w=w, bias=bias, gamma=gamma, res=res, blocks=blocks)


def kernel_gemm_model(c, *, act=P.ACT_NONE, gamma=True, residual=True, skip_block=None, drop_bias_col=None, gamma_first=False):
    acc = torch.zeros(M, N)
    for kb, blk in enumerate(c["blocks"]):
        if skip_block is not None and kb == skip_block[0]:
            blk = blk.clone()
            r, n = skip_block[1], skip_block[2]
            blk[r:r + 128, n:n + BN] = 0          # one k-block missing in one 128 x BN tile
        acc = acc + blk
    bias = c["bias"].clone()
    if drop_bias_col is not None:
        bias[drop_bias_col] = 0
    v = acc + bias
    if act == P.ACT_SWIGLU:
        return bf16(torch.nn.functional.silu(v[:, 0::2]) * v[:, 1::2])
    if gamma and gamma_first:
        v = v * c["gamma"]
    if act == P.ACT_GELU:
        v = torch.nn.functional.gelu(v)
    elif act == P.ACT_RELU:
        v = torch.relu(v)
    if gamma and not gamma_first:
        v = v * c["gamma"]
    if residual:
        v = v + c["res"]
    return bf16(v)


def gemm_reference(c, act, gamma=True, residual=True):
    return P.gemm_ref(c["a"], c["w"], bias=c["bias"], act=act, gamma=c["gamma"] if gamma else None,
                      residual=c["res"] if residual else None)


@pytest.mark.parametrize("act", [P.ACT_NONE, P.ACT_GELU, P.ACT_RELU, P.ACT_SWIGLU])
def test_gemm_model_passes(gemm_case, act):
    epi = dict(gamma=act != P.ACT_SWIGLU, residual=act != P.ACT_SWIGLU)
    ref, lmag = gemm_reference(gemm_case, act, **epi)
    r = P.check_gemm(kernel_gemm_model(gemm_case, act=act, **epi), ref, lmag, what=f"cpu model act={act}")
    assert r > 0.05   # the bound is not vacuous: the model's own rounding uses a visible part of it


def test_gemm_model_fp32_output_passes(gemm_case):
    acc = sum(gemm_case["blocks"], torch.zeros(M, N))
    ref, lmag = P.gemm_ref(gemm_case["a"], gemm_case["w"])
    P.check_gemm(acc, ref, lmag, out_f32=True, what="cpu model fp32 out")


@pytest.mark.parametrize("mutation", ["missing_k_block", "missing_bias_column", "gamma_before_act"])
def test_gemm_mutation_fails(gemm_case, mutation):
    act = P.ACT_GELU if mutation == "gamma_before_act" else P.ACT_NONE
    kw = {"missing_k_block": dict(skip_block=(37, 128, 256)), "missing_bias_column": dict(drop_bias_col=517),
          "gamma_before_act": dict(gamma_first=True)}[mutation]
    got = kernel_gemm_model(gemm_case, act=act, **kw)
    ref, lmag = gemm_reference(gemm_case, act)
    r = P.worst_ratio(got, ref, P.gemm_bound(ref, lmag))
    print(f"[parity] gemm mutation {mutation}: worst err/bound {r:.2f}")
    assert r > 1.5


# ------------------------------------------------------------------------------------------------- attention
S, D, TILE = 966, 128, 128


@pytest.fixture(scope="module")
def attn_case():
    q, k, v = bf16(rnd(1, S, 1, D, seed=11)), bf16(rnd(1, 1, S, D, seed=12)), bf16(rnd(1, 1, S, D, seed=13))
    return dict(q=q, k=k, v=v, scale=1.0 / math.sqrt(D))


def kernel_attention_model(c, *, scale_mul=1.0, drop_key=None, swap_wg_l=False):
    """Causal self-attention, one (batch, head)."""
    q, k, v = c["q"][0, :, 0], c["k"][0, 0], c["v"][0, 0]
    sl2 = torch.tensor(c["scale"] * scale_mul * 1.4426950408889634, dtype=torch.float32)
    rows = torch.arange(S)[:, None]
    m = torch.full((S, 1), float("-inf"))
    l = torch.zeros(S, 1)
    o = torch.zeros(S, D)
    for j0 in range(0, S, TILE):
        keys = torch.arange(j0, min(j0 + TILE, S))[None, :]
        s = q @ k[j0:j0 + TILE].t()
        vis = keys <= rows
        if drop_key is not None:
            key, first_row = drop_key
            vis = vis & ~((keys == key) & (rows >= first_row))
        s = s.masked_fill(~vis, float("-inf"))
        m_new = torch.maximum(m, s.max(1, keepdim=True).values * sl2)
        m_use = torch.where(m_new == float("-inf"), torch.zeros_like(m_new), m_new)
        corr = torch.exp2(m - m_use)
        p = torch.exp2(s * sl2 - m_use)
        l = l * corr + p.sum(1, keepdim=True)
        o = o * corr + bf16(p) @ v[j0:j0 + TILE]
        m = m_new
    if swap_wg_l:
        # rows [64, 128) of every query tile normalised with the l of the matching row of the other warpgroup
        idx = torch.arange(S)
        other = torch.where((idx % 128) >= 64, idx - 64, idx)
        l = l[other]
    return bf16(o / l).reshape(1, S, D)


def test_attention_model_passes(attn_case):
    ref, pv = P.attention_ref(attn_case["q"], attn_case["k"], attn_case["v"], causal=True, scale=attn_case["scale"])
    r = P.check_attention(kernel_attention_model(attn_case), ref, pv, what="cpu model causal S=966 D=128")
    assert r > 0.05


@pytest.mark.parametrize("mutation", ["scale_x1.01", "late_rows_drop_one_key", "warpgroup_l_swapped"])
def test_attention_mutation_fails(attn_case, mutation):
    kw = {"scale_x1.01": dict(scale_mul=1.01), "late_rows_drop_one_key": dict(drop_key=(600, 640)),
          "warpgroup_l_swapped": dict(swap_wg_l=True)}[mutation]
    ref, pv = P.attention_ref(attn_case["q"], attn_case["k"], attn_case["v"], causal=True, scale=attn_case["scale"])
    r = P.worst_ratio(kernel_attention_model(attn_case, **kw), ref, P.attention_bound(ref, pv))
    print(f"[parity] attention mutation {mutation}: worst err/bound {r:.2f}")
    assert r > 1.2


def test_bound_is_per_element():
    """An error of one element in a row of tiny values is caught even when the largest output element is large."""
    ref = torch.tensor([[1000.0, 1e-3, 1.0]], dtype=torch.float64)
    got = ref.clone()
    got[0, 1] += 1e-3
    assert P.worst_ratio(got, ref, P.gemm_bound(ref, torch.zeros_like(ref))) > 1
    assert P.worst_ratio(ref.clone(), ref, P.gemm_bound(ref, torch.zeros_like(ref))) == 0
    got[0, 1] = float("nan")
    assert P.worst_ratio(got, ref, P.gemm_bound(ref, torch.ones_like(ref))) == float("inf")


# ------------------------------------------------------------------------------------------------- decode-step epilogues
# Kernel models: the split-K partials summed in split order in fp32 (splitk_sum4 / splitk_pairs), then the epilogue's own
# rounding points as in csrc/llama_decode.cu.
def splitk_model(ws, drop_last=False):
    acc = torch.zeros(ws.shape[1:])
    for s in range(ws.shape[0] - (1 if drop_last else 0)):
        acc = acc + ws[s]
    return acc


@pytest.fixture(scope="module")
def splitk_case():
    S, B, N = 17, 4, 1000
    ws = rnd(S, B, N, seed=21) * torch.logspace(-2, 1, N)[None, None, :] / math.sqrt(S)
    return ws


@pytest.mark.parametrize("out_bf16", [False, True])
def test_splitk_model_passes(splitk_case, out_bf16):
    ws = splitk_case
    ref, mag = P.splitk_ref(ws)
    got = splitk_model(ws)
    got = bf16(got) if out_bf16 else got
    r = P.check_bound("splitk", got, ref, P.splitk_bound(ref, mag, ws.shape[0], out_bf16), what=f"cpu model bf16={out_bf16}")
    assert r > (0.2 if out_bf16 else 0.01)


@pytest.mark.parametrize("out_bf16", [False, True])
def test_splitk_dropped_split_fails(splitk_case, out_bf16):
    ws = splitk_case
    ref, mag = P.splitk_ref(ws)
    got = splitk_model(ws, drop_last=True)
    got = bf16(got) if out_bf16 else got
    r = P.worst_ratio(got, ref, P.splitk_bound(ref, mag, ws.shape[0], out_bf16))
    print(f"[parity] splitk mutation dropped split (bf16={out_bf16}): worst err/bound {r:.2f}")
    assert r > 1.5


NORM_EPS = 1e-5


@pytest.fixture(scope="module")
def norm_case():
    # residual rows from embedding scale (~1e-2, where eps is a visible part of mean(h^2)) to a grown residual stream
    S, N = 13, 4096
    scale = torch.tensor([1e-2, 2e-2, 0.1, 1.0, 1.0, 6.0])[:, None]
    x = bf16(rnd(6, N, seed=31) * scale)
    ws = rnd(S, 6, N, seed=32) * scale * 0.5 / math.sqrt(S)
    w = 1 + 0.1 * rnd(N, seed=33)
    return ws, x, w


def kernel_norm_model(ws, x, w, *, eps_after_rsqrt=False, residual_after_norm=False):
    acc = splitk_model(ws)
    h = bf16(acc + x)
    src = bf16(acc) if residual_after_norm else h
    ms = (src * src).sum(-1, keepdim=True) / src.shape[-1]
    rs = torch.rsqrt(ms) + NORM_EPS if eps_after_rsqrt else torch.rsqrt(ms + NORM_EPS)
    y = w * bf16(src * rs)
    return h, bf16(y + x if residual_after_norm else y)


def test_reduce_norm_model_passes(norm_case):
    ws, x, w = norm_case
    h, y = kernel_norm_model(ws, x, w)
    P.check_rounded(h, *P.residual_interval(ws, x), what="cpu model residual")
    ref, bound = P.rmsnorm_ref(h, w, NORM_EPS)
    assert P.check_bound("rmsnorm", y, ref, bound, what="cpu model") > 0.2


def test_residual_interval_is_exact_away_from_boundaries(norm_case):
    """Off by one bf16 ulp anywhere but at a rounding boundary is caught: the residual check is not a tolerance."""
    ws, x, w = norm_case
    h, _ = kernel_norm_model(ws, x, w)
    lo, hi = P.residual_interval(ws, x)
    nudged = h.clone()
    nudged[3, 100] = torch.nextafter(h[3, 100].bfloat16(), torch.tensor(float("inf"), dtype=torch.bfloat16)).float()
    assert P.interval_misses(nudged, lo, hi) == 1
    assert int((lo != hi).sum()) < h.numel() // 100    # only a few elements sit at a boundary


@pytest.mark.parametrize("mutation", ["eps_after_rsqrt", "residual_after_norm"])
def test_reduce_norm_mutation_fails(norm_case, mutation):
    ws, x, w = norm_case
    h, y = kernel_norm_model(ws, x, w, **{mutation: True})
    P.check_rounded(h, *P.residual_interval(ws, x), what="cpu model residual")
    ref, bound = P.rmsnorm_ref(h, w, NORM_EPS)
    r = P.worst_ratio(y, ref, bound)
    print(f"[parity] rmsnorm mutation {mutation}: worst err/bound {r:.2f}")
    assert r > 1.5


@pytest.fixture(scope="module")
def swiglu_case():
    S, B, N = 16, 3, 2 * 1500
    return rnd(S, B, N, seed=41) * 2.0 / math.sqrt(S)


def kernel_swiglu_model(ws, swap=False):
    acc = splitk_model(ws)
    g, u = acc[..., 0::2], acc[..., 1::2]
    if swap:
        g, u = u, g
    return bf16(torch.nn.functional.silu(g) * u)


def test_swiglu_model_passes(swiglu_case):
    ref, bound = P.splitk_swiglu_ref(swiglu_case)
    assert P.check_bound("swiglu", kernel_swiglu_model(swiglu_case), ref, bound, what="cpu model") > 0.2


def test_swiglu_swapped_gate_up_fails(swiglu_case):
    ref, bound = P.splitk_swiglu_ref(swiglu_case)
    r = P.worst_ratio(kernel_swiglu_model(swiglu_case, swap=True), ref, bound)
    print(f"[parity] swiglu mutation swapped gate/up: worst err/bound {r:.2f}")
    assert r > 1.5


ROPE_D, ROPE_THETA = 128, 10000.0


def rope_tables(n):
    """fp32 cos / sin tables [n, D/2] as GromaEngine.ensure_rope builds them."""
    inv = 1.0 / (ROPE_THETA ** (torch.arange(0, ROPE_D, 2).float() / ROPE_D))
    fr = torch.outer(torch.arange(n).float(), inv)
    return fr.cos(), fr.sin()


@pytest.fixture(scope="module")
def rope_case():
    S = 17
    ws = rnd(S, 3, 4, ROPE_D, seed=51) * 1.5 / math.sqrt(S)
    return ws, rope_tables(5001)


def kernel_rope_model(ws, tables, pos, *, sin_flip=False, row_off=0):
    x = bf16(splitk_model(ws))
    half = ROPE_D // 2
    c, s = tables[0][pos - row_off], tables[1][pos - row_off]
    if sin_flip:
        s = -s
    x1, x2 = x[..., :half], x[..., half:]
    return torch.cat([bf16(x1 * c - x2 * s), bf16(x2 * c + x1 * s)], -1)


@pytest.mark.parametrize("pos", [0, 1, 257, 4095, 5000])
def test_rope_model_passes(rope_case, pos):
    ws, tables = rope_case
    ref, bound = P.rope_ref(ws, pos, ROPE_THETA)
    r = P.check_bound("rope", kernel_rope_model(ws, tables, pos), ref, bound, what=f"cpu model pos={pos}")
    assert r > 0.1 or pos == 0     # position 0 is the identity: exact


@pytest.mark.parametrize("mutation", ["sin_sign_flipped", "table_row_of_pos_minus_1"])
@pytest.mark.parametrize("pos", [1, 257, 5000])
def test_rope_mutation_fails(rope_case, mutation, pos):
    ws, tables = rope_case
    kw = dict(sin_flip=True) if mutation == "sin_sign_flipped" else dict(row_off=1)
    ref, bound = P.rope_ref(ws, pos, ROPE_THETA)
    r = P.worst_ratio(kernel_rope_model(ws, tables, pos, **kw), ref, bound)
    print(f"[parity] rope mutation {mutation} pos={pos}: worst err/bound {r:.2f}")
    assert r > 1.5
