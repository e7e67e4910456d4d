"""fp64 references and per-element error bounds for the tensor-core GEMM and flash-attention kernels and the decode-step
epilogues.  TEST INFRASTRUCTURE: imported by the GEMM / attention / decode tests, never by the product.

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

Decode-step epilogues.  They consume the fp32 split-K partials ws[S, ...] of a swap-AB GEMM, summed in split order in fp32;
the reference is the fp64 sum, and mag = sum_s |ws_s|.  u = 2^-24 (fp32 unit roundoff).
Split-K sum:         |got - ref| <= (S-1) u mag                         (fp32 output; S-1 roundings of a sequential sum)
                     |got - ref| <= (S-1) u mag + 2^-8 (|ref| + (S-1) u mag)               (bf16 output)
Reduce + residual + RMSNorm (h = bf16(sum + x), y = bf16(w * bf16(h * rsqrt(mean(h^2) + eps)))):
    h is bf16_rn of the exact sum, except where sum + x lies within S u (mag + |x|) of a rounding boundary: there either
    neighbour is right.  Both are found by rounding the two ends of that interval (rounding is monotone), so the check is
    exact everywhere else.  y is checked against the fp64 norm of the kernel's own h (its error is h's check): the fp32 sum
    of N squares (N u), the division and eps (2u), rsqrtf (2 ulp), the products (2u) and the two bf16 rounding points
    (2^-8 each) multiply: |got - ref| <= ((1 + 2^-8)^2 (1 + (N/2 + 8) u) - 1) |ref|.
SwiGLU over the summed partials: gemm_epilogue_ref's SwiGLU slopes L with mag as the accumulation magnitude:
                     |got - ref| <= 2^-7 |ref| + (S-1) u L mag
RoPE pair (q, or the appended k) from the fp64 sums s1, s2 of (j, j + D/2): the kernel rounds the sums to bf16 first, so the
    reference rotates bf16_rn(s) -- where s lies within the split-K bound of a rounding boundary the kernel's input may be
    the neighbour (dx below, found as for h).  The angle is pos * theta^(-2j/D) in fp64; the fp32 tables carry ~2 ulp of
    the angle (inverse frequency and product: dth = 2^-22 pos theta^(-2j/D)) plus ~1 ulp of cos / sin (2^-22 absolute):
                     E = |c| dx1 + |s| dx2 + dth |x| + (2^-22 + 2u) (|x1| + |x2|)
                     |got - ref| <= E + 2^-8 (|ref| + E)                   (bf16 output)
    A sign flip of sin or a table row of the wrong position moves the pair by ~|x| theta^(-2j/D): far outside.

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


U32 = 2.0 ** -24   # fp32 unit roundoff


def splitk_ref(ws: torch.Tensor):
    """fp64 sum of the split-K partials ws [S, ...] over the splits, and mag = sum_s |ws_s|."""
    w = _f64(ws)
    return w.sum(0), w.abs().sum(0)


def splitk_bound(ref: torch.Tensor, mag: torch.Tensor, S: int, out_bf16: bool = False) -> torch.Tensor:
    """(S-1) u mag, plus 2^-8 (|ref| + (S-1) u mag) for a bf16 output."""
    e = (S - 1) * U32 * mag
    if out_bf16:
        e = e + 2.0 ** -8 * (ref.abs() + e)
    return e + ABS_FLOOR


def bf16_rn(t: torch.Tensor) -> torch.Tensor:
    """t rounded to bf16 (through fp32: monotone, which is all the interval checks below rely on), as float64."""
    return _f64(t).to(torch.float32).to(torch.bfloat16).to(torch.float64)


def rounding_interval(v: torch.Tensor, e: torch.Tensor):
    """(lo, hi): the smallest and largest bf16 value that rounds some number within e of v."""
    return bf16_rn(v - e), bf16_rn(v + e)


def residual_interval(ws: torch.Tensor, x: torch.Tensor):
    """The bf16 values h = bf16(fp32(sum_s ws_s) + x) may take: (lo, hi), equal except where the fp32 sum lies within its
    error bound S u (mag + |x|) of a rounding boundary.  ws [S, B, N], x [B, N]."""
    acc, mag = splitk_ref(ws)
    x64 = _f64(x).to(acc.device)
    return rounding_interval(acc + x64, ws.shape[0] * U32 * (mag + x64.abs()))


def rmsnorm_ref(h: torch.Tensor, w: torch.Tensor, eps: float):
    """fp64 w * h * rsqrt(mean(h^2) + eps) over the last dimension, and its per-element bound (module docstring)."""
    h64, w64 = _f64(h), _f64(w).to(h.device)
    ref = w64 * h64 * torch.rsqrt(h64.pow(2).mean(-1, keepdim=True) + eps)
    rel = (1 + 2.0 ** -8) ** 2 * (1 + (h.shape[-1] / 2 + 8) * U32) - 1
    return ref, rel * ref.abs() + ABS_FLOOR


def splitk_swiglu_ref(ws: torch.Tensor):
    """fp64 silu(g) * u of the summed partials ws [S, ..., N] with (g, u) = columns (2j, 2j+1), and the bound."""
    acc, mag = splitk_ref(ws)
    ref, lmag = gemm_epilogue_ref(acc, mag, act=ACT_SWIGLU)
    return ref, 2.0 ** -7 * ref.abs() + (ws.shape[0] - 1) * U32 * lmag + ABS_FLOOR


def rope_ref(ws: torch.Tensor, pos: int, theta: float = 10000.0):
    """fp64 rotate-half RoPE at position `pos` of the summed partials ws [S, ..., D] (the kernel: bf16 inputs, fp32 tables,
    bf16 output), and the per-element bound of the module docstring.  Returns (ref, bound), both [..., D]."""
    S = ws.shape[0]
    acc, mag = splitk_ref(ws)
    half = acc.shape[-1] // 2
    x = bf16_rn(acc)
    lo, hi = rounding_interval(acc, (S - 1) * U32 * mag)
    dx = torch.maximum(hi - x, x - lo)
    x1, x2, d1, d2 = x[..., :half], x[..., half:], dx[..., :half], dx[..., half:]
    inv = theta ** (-2.0 * torch.arange(half, dtype=torch.float64, device=acc.device) / (2 * half))
    c, s = torch.cos(pos * inv), torch.sin(pos * inv)
    o1, o2 = x1 * c - x2 * s, x2 * c + x1 * s
    common = 2.0 ** -22 * pos * inv * torch.hypot(x1, x2) + (2.0 ** -22 + 2 * U32) * (x1.abs() + x2.abs())
    e1 = c.abs() * d1 + s.abs() * d2 + common
    e2 = c.abs() * d2 + s.abs() * d1 + common
    ref, e = torch.cat([o1, o2], -1), torch.cat([e1, e2], -1)
    return ref, e + 2.0 ** -8 * (ref.abs() + e) + ABS_FLOOR


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


def check_bound(kind: str, got, ref, bound, *, what: str = "") -> float:
    """Assert |got - ref| <= bound element by element (bound from one of the *_ref / *_bound helpers); return the worst ratio."""
    r = _report(kind, what, worst_ratio(got, ref, bound))
    assert r <= 1.0, f"{kind} {what}: error exceeds the per-element bound by {r:.2f}x"
    return r


def interval_misses(got, lo, hi) -> int:
    """Elements of got outside [lo, hi] (non-finite ones included)."""
    g = got.detach().to(device=lo.device, dtype=torch.float64)
    return int((~((g >= lo) & (g <= hi))).sum().item())


def check_rounded(got, lo, hi, *, what: str = "") -> int:
    """Assert lo <= got <= hi element by element (rounding_interval / residual_interval); print how many elements sat at a
    rounding boundary (lo != hi), where either neighbour is right."""
    miss = interval_misses(got, lo, hi)
    print(f"[parity] rounded {what}: {miss} of {got.numel()} outside, {int((lo != hi).sum())} at a rounding boundary")
    assert miss == 0, f"{what}: {miss} elements are not a rounding of the exact value"
    return miss
