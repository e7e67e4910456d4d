"""fp64 references and per-element error bounds for the tensor-core GEMM and flash-attention kernels.  TEST INFRASTRUCTURE:
imported by the GEMM / attention tests, never by the product.

References are computed in float64 with torch on whatever device the inputs live on (cuBLAS DGEMM / einsum on the GPU for the
large shapes, the CPU for the small ones) -- never with this library.  Every bound is per element, so an error that is small
against the largest element of the output but large against the element it sits in (a dropped key of one row, one k-block
of one tile, one column's bias) is still caught.

GEMM, bf16 output:   |got - ref| <= 2^-7 |ref| + L 2^-16 (|A| |B|^T)
GEMM, fp32 output:   |got - ref| <= 1e-6 |ref| + L 2^-16 (|A| |B|^T)
    The first term is bf16 output rounding (half an ulp: at most 2^-8 relative) plus the fp32 epilogue operations, with a
    factor 2 of room; the second bounds fp32 accumulation of the bf16 products.  L is the gain of the epilogue from the accumulator to the
    output: |gamma|, the largest slope of erf-GELU (1.13), 1 for ReLU / none, and for SwiGLU the partial derivatives
    |silu'(g)| |u| and |silu(g)| applied to the magnitudes of the gate and up columns.
Attention:           |got - ref| <= 2^-7 (P |V|) + 2^-8 |ref|
    P is the exact fp64 softmax.  P |V| bounds the error of P rounded to bf16 before the PV product and of the fp32
    exponentials and sums; 2^-8 |ref| is the bf16 output rounding (half an ulp: at most 2^-8 relative).

Every bound also has an absolute floor of 2^-100: results at the bottom of the fp32 range (silu of a very negative gate is
~1e-40, subnormal, or flushed to 0 by the kernel's fast exponential) carry no relative precision at all.

Each check prints the worst ratio of error to bound it saw (run pytest with -s to see them) and returns it.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

GELU_MAX_SLOPE = 1.13            # max over x of d/dx [x Phi(x)] = 1.1289...
SILU_MAX_SLOPE = 1.1             # max over x of d/dx [x sigmoid(x)] = 1.0998...
ABS_FLOOR = 2.0 ** -100
ACT_NONE, ACT_GELU, ACT_RELU, ACT_SWIGLU = 0, 1, 2, 3   # groma_b200.ops numbering


def _f64(t):
    return None if t is None else t.detach().to(torch.float64)


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def _silu(x):
    return x * torch.sigmoid(x)


def _silu_slope(x):
    s = torch.sigmoid(x)
    return s * (1.0 + x * (1.0 - s))


def gemm_epilogue_ref(acc: torch.Tensor, mag: torch.Tensor, *, bias=None, act: int = ACT_NONE, gamma=None, residual=None):
    """Apply the GEMM epilogue chain (bias -> act -> gamma -> residual; SwiGLU pairs columns (2j, 2j+1) = (gate, up) and
    takes no gamma / residual) to the fp64 accumulator `acc` [M, N] and propagate the accumulation magnitude `mag` =
    |A| |B|^T through it.  Returns (ref, L * mag) in float64; bias / gamma index the last dimension."""
    v = acc + _f64(bias) if bias is not None else acc.clone()
    if act == ACT_SWIGLU:
        g, u = v[..., 0::2], v[..., 1::2]
        gm, um = mag[..., 0::2], mag[..., 1::2]
        return _silu(g) * u, _silu_slope(g).abs() * u.abs() * gm + _silu(g).abs() * um
    gain = torch.ones_like(mag)
    if act == ACT_GELU:
        v, gain = _gelu(v), gain * GELU_MAX_SLOPE
    elif act == ACT_RELU:
        v = torch.relu(v)
    if gamma is not None:
        v = v * _f64(gamma)
        gain = gain * _f64(gamma).abs()
    if residual is not None:
        v = v + _f64(residual)
    return v, gain * mag


def gemm_ref(a: torch.Tensor, w: torch.Tensor, **epi):
    """fp64 reference of epilogue(a[M,K] @ w[N,K]^T) and its L-weighted accumulation magnitude (see gemm_epilogue_ref)."""
    a64, w64 = _f64(a), _f64(w)
    return gemm_epilogue_ref(a64 @ w64.t(), a64.abs() @ w64.abs().t(), **epi)


def gemm_bound(ref: torch.Tensor, lmag: torch.Tensor, out_f32: bool = False) -> torch.Tensor:
    """Per-element GEMM bound: 2^-7 |ref| (1e-6 |ref| for fp32 outputs) + 2^-16 L |A||B|^T."""
    return (1e-6 if out_f32 else 2.0 ** -7) * ref.abs() + 2.0 ** -16 * lmag + ABS_FLOOR


def attention_ref(q, k, v, *, causal: bool, scale: float, q_pos0: int = 0, kv_len: Optional[torch.Tensor] = None,
                  sk: Optional[int] = None):
    """fp64 attention.  q [B,Sq,H,D]; k, v [B,H,>=sk,D] (only the first sk keys take part); key j is visible to query i
    iff j < min(sk, kv_len[b]) and (not causal or j <= q_pos0 + i).  A row without visible keys is 0.
    Returns (ref [B,Sq,H*D], P|V| [B,Sq,H*D]) in float64."""
    B, Sq, H, D = q.shape
    Sk = k.shape[2] if sk is None else sk
    q64, k64, v64 = _f64(q), _f64(k[:, :, :Sk]), _f64(v[:, :, :Sk])
    s = torch.einsum("bqhd,bhkd->bhqk", q64, k64) * scale
    keys = torch.arange(Sk, device=s.device)
    vis = torch.ones(B, 1, Sq, Sk, dtype=torch.bool, device=s.device)
    if causal:
        vis &= (keys[None, :] <= torch.arange(Sq, device=s.device)[:, None] + q_pos0)[None, None]
    if kv_len is not None:
        vis &= (keys[None, :] < kv_len.to(s.device).long()[:, None])[:, None, None, :]
    p = torch.softmax(s.masked_fill(~vis, float("-inf")), -1).nan_to_num(0.0)   # rows without visible keys -> 0
    ref = torch.einsum("bhqk,bhkd->bqhd", p, v64).reshape(B, Sq, H * D)
    pv = torch.einsum("bhqk,bhkd->bqhd", p, v64.abs()).reshape(B, Sq, H * D)
    return ref, pv


def attention_bound(ref: torch.Tensor, pv: torch.Tensor) -> torch.Tensor:
    """Per-element attention bound: 2^-7 P|V| + 2^-8 |ref|."""
    return 2.0 ** -7 * pv + 2.0 ** -8 * ref.abs() + ABS_FLOOR


def worst_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |got - ref| / bound over all elements (inf where got is not finite)."""
    got = got.detach().to(device=ref.device, dtype=torch.float64)
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, float("inf")))
    return ratio.max().item() if ratio.numel() else 0.0


def _report(kind: str, what: str, r: float) -> float:
    print(f"[parity] {kind} {what}: worst err/bound {r:.3f}")
    return r


def check_gemm(got, ref, lmag, *, out_f32: bool = False, what: str = "") -> float:
    """Assert the per-element GEMM bound; return the worst err/bound ratio."""
    r = _report("gemm", what, worst_ratio(got, ref, gemm_bound(ref, lmag, out_f32)))
    assert r <= 1.0, f"{what}: error exceeds the per-element bound by {r:.2f}x"
    return r


def check_attention(got, ref, pv, *, what: str = "") -> float:
    """Assert the per-element attention bound; return the worst err/bound ratio."""
    r = _report("attention", what, worst_ratio(got, ref, attention_bound(ref, pv)))
    assert r <= 1.0, f"{what}: error exceeds the per-element bound by {r:.2f}x"
    return r
