"""The per-element comparators of tests/parity.py must accept the kernels' own rounding and reject small, plausible defects.

A CPU model of each kernel's rounding points stands in for the kernel:
  GEMM       bf16 operands, fp32 accumulation one 64-deep k-block at a time (as the wgmma main loop retires them), fp32
             epilogue (bias -> act -> gamma -> residual), bf16 output;
  attention  fp32 scores, online softmax over 128-key tiles (running max, rescale, fp32 row sums of the unrounded
             probabilities), P rounded to bf16 for the PV product, fp32 O, O / l rounded to bf16; the 128-row query tile is
             two 64-row warpgroups.
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
