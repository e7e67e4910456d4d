"""The wgmma flash-attention kernel (attention_wgmma.cu, ops.attention_tc) against the fp64 reference of tests/parity.py,
per element, at the edges of its tiling: 128-row query tiles split into two 64-row warpgroups, 128-key tiles in 2-deep
K / V rings, the per-warpgroup causal-mask decision, q_pos0 > 0, ragged kv_len, both operand layouts (KV cache
[B,H,cap,D] with cap % 128 != 0, and fused-qkv activation views), and bit-exact indifference to everything masked."""
import math

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
    return (torch.randn(*shape, generator=g, device="cuda") * scale).bfloat16()


def odd_cap(S):
    """A cache capacity > S that is not a multiple of 128 (the last key tile of a head reads into the next head)."""
    cap = S + 37
    return cap + 1 if cap % 128 == 0 else cap


def cache_case(B, H, Sq, Sk, D, seed=0):
    cap = odd_cap(Sk)
    return rnd(B, Sq, H, D, seed=seed), rnd(B, H, cap, D, seed=seed + 1), rnd(B, H, cap, D, seed=seed + 2)


def qkv_case(B, H, S, D, seed=0):
    x = rnd(B * S, 3 * H * D, seed=seed).reshape(B, S, 3, H, D)
    return x[:, :, 0], x[:, :, 1].permute(0, 2, 1, 3), x[:, :, 2].permute(0, 2, 1, 3)


def check(G, q, k, v, what, *, causal, scale=None, q_pos0=0, kv_len=None, sk=None):
    D = q.shape[3]
    scale = 1.0 / math.sqrt(D) if scale is None else scale
    got = G.attention_tc(q, k, v, causal=causal, scale=scale, q_pos0=q_pos0, kv_len=kv_len, sk=sk)
    ref, pv = P.attention_ref(q, k, v, causal=causal, scale=scale, q_pos0=q_pos0, kv_len=kv_len, sk=sk)
    P.check_attention(got, ref, pv, what=what)
    return got


SQ_EDGES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257]


@pytest.mark.parametrize("layout", ["cache", "qkv"])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("S", SQ_EDGES)
def test_query_geometry(G, S, D, causal, layout):
    """Sq around the 64-row warpgroup split and the 128-row query tile: the second warpgroup partly or wholly past Sq."""
    B, H = 2, 2
    if layout == "cache":
        q, k, v = cache_case(B, H, S, S, D, seed=S)
        check(G, q, k, v, f"Sq=Sk={S} D={D} causal={causal} cache", causal=causal, sk=S)
    else:
        q, k, v = qkv_case(B, H, S, D, seed=S)
        check(G, q, k, v, f"Sq=Sk={S} D={D} causal={causal} qkv", causal=causal)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("r", [0, 1, 64, 127])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6])
def test_key_tile_count(G, n, r, D):
    """n key tiles, the last one holding r keys (r = 0: full): both ring stages wrap their phase more than once."""
    Sk = n * 128 if r == 0 else (n - 1) * 128 + r
    Sq = 129
    q, k, v = cache_case(2, 2, Sq, Sk, D, seed=n * 1000 + r)
    check(G, q, k, v, f"Sq={Sq} Sk={Sk} D={D}", causal=False, sk=Sk)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("Sq,Sk", [(1, 966), (70, 333), (129, 1000)])
def test_causal_q_pos0(G, Sq, Sk, D):
    """Query rows at positions q_pos0 + i with q_pos0 = Sk - Sq: the causal boundary falls inside a warpgroup's rows and
    across the 64-row split ((129, 1000): row limits 871..999, key tiles 6 and 7)."""
    q, k, v = cache_case(2, 3, Sq, Sk, D, seed=Sq)
    check(G, q, k, v, f"causal Sq={Sq} Sk={Sk} q_pos0={Sk - Sq} D={D}", causal=True, q_pos0=Sk - Sq, sk=Sk)


@pytest.mark.parametrize("layout", ["cache", "qkv"])
@pytest.mark.parametrize("D", [64, 128])
def test_causal_ragged_kv_len(G, D, layout):
    """kv_len on tile edges (127, 128, 129), a single key, full length; rows whose causal limit exceeds kv_len."""
    B, H, S = 5, 2, 300
    kv_len = torch.tensor([127, 128, 129, 1, 300], dtype=torch.int32, device="cuda")
    if layout == "cache":
        q, k, v = cache_case(B, H, S, S, D, seed=D)
        check(G, q, k, v, f"causal ragged kv_len D={D} cache", causal=True, kv_len=kv_len, sk=S)
    else:
        q, k, v = qkv_case(B, H, S, D, seed=D)
        check(G, q, k, v, f"causal ragged kv_len D={D} qkv", causal=True, kv_len=kv_len)


def test_engine_vit_call(G):
    """DINOv2 attention as the engine issues it: S = 1025, 16 heads of 64, views into the fused qkv projection."""
    q, k, v = qkv_case(2, 16, 1025, 64, seed=5)
    check(G, q, k, v, "ViT S=1025 H=16 D=64 qkv", causal=False, scale=0.125)


def test_engine_prefill_call(G):
    """LLaMA prefill as the engine issues it: T = 966, 32 heads of 128, B = 2 with right padding, KV cache with headroom."""
    B, H, T, D = 2, 32, 966, 128
    q, k, v = rnd(B, T, H, D, seed=6), rnd(B, H, T + 134, D, seed=7), rnd(B, H, T + 134, D, seed=8)
    kv_len = torch.tensor([966, 613], dtype=torch.int32, device="cuda")
    check(G, q, k, v, "prefill T=966 H=32 D=128 kv_len=[966, 613]", causal=True, kv_len=kv_len, sk=T)


BIG = 1.0e4   # large but finite: the header requires that rows a tile load can touch are finite


def big_like(t, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sign = torch.randint(0, 2, t.shape, generator=g, device="cuda").to(t.dtype) * 2 - 1
    return sign * BIG


@pytest.mark.parametrize("D", [64, 128])
def test_invisible_inputs_have_no_effect(G, D):
    """Overwriting what the kernel must ignore with large finite values leaves the output bit-identical:
    cache rows in [kv_len, cap), keys past the causal limit inside a loaded tile, and the next head's rows that the last
    tile of a head reads."""
    B, H, S = 2, 3, 290
    q, k, v = cache_case(B, H, S, S, D, seed=D + 1)
    cap = k.shape[2]
    kv_len = torch.tensor([290, 150], dtype=torch.int32, device="cuda")
    run = lambda k_, v_: G.attention_tc(q, k_, v_, causal=True, scale=1.0 / math.sqrt(D), kv_len=kv_len, sk=S)
    base = run(k, v)
    ref, pv = P.attention_ref(q, k, v, causal=True, scale=1.0 / math.sqrt(D), kv_len=kv_len, sk=S)
    P.check_attention(base, ref, pv, what=f"invisible-inputs base D={D}")
    # (a) cache rows past kv_len (up to cap) of every head
    k2, v2 = k.clone(), v.clone()
    for b in range(B):
        n = int(kv_len[b])
        k2[b, :, n:] = big_like(k2[b, :, n:], 1); v2[b, :, n:] = big_like(v2[b, :, n:], 2)
    assert torch.equal(run(k2, v2), base)
    # (b) keys past the causal limit of query rows [128, 192) (warpgroup 0 of query tile 1), inside key tile 1
    k2, v2 = k.clone(), v.clone()
    k2[:, :, 192:] = big_like(k2[:, :, 192:], 3); v2[:, :, 192:] = big_like(v2[:, :, 192:], 4)
    assert torch.equal(run(k2, v2)[:, :192], base[:, :192])
    # (c) rows 0..(3*128 - cap) of head 1 are read by head 0's last key tile; head 0 must not see them
    spill = 3 * 128 - cap
    assert spill > 0
    k2, v2 = k.clone(), v.clone()
    k2[:, 1, :spill] = big_like(k2[:, 1, :spill], 5); v2[:, 1, :spill] = big_like(v2[:, 1, :spill], 6)
    assert torch.equal(run(k2, v2)[:, :, :D], base[:, :, :D])


@pytest.mark.parametrize("causal", [False, True])
def test_softmax_stability_rising_max(G, causal):
    """Logits of magnitude ~200 with a trend that makes each row's running max rise in later key tiles, so the running
    output is rescaled (corr) by factors far from 1 many times."""
    B, H, S, D = 1, 2, 600, 64
    g = torch.Generator(device="cuda").manual_seed(9)
    u = torch.zeros(D, device="cuda"); u[0] = 1.0
    q = torch.randn(B, S, H, D, generator=g, device="cuda") * 6 + 24 * u
    k = torch.randn(B, H, odd_cap(S), D, generator=g, device="cuda") * 6
    k[..., 0] += torch.linspace(-50, 50, k.shape[2], device="cuda")
    v = torch.randn(B, H, odd_cap(S), D, generator=g, device="cuda")
    q, k, v = q.bfloat16(), k.bfloat16(), v.bfloat16()
    s = torch.einsum("bqhd,bhkd->bhqk", q.double(), k[:, :, :S].double()) / 8
    assert s.abs().max() > 150
    check(G, q, k, v, f"logits ~{s.abs().max().item():.0f} causal={causal}", causal=causal, sk=S)


def test_kv_len_zero_rows_are_zero(G):
    """A sequence with no visible key produces zeros (finite), the others are unaffected."""
    B, H, S, D = 3, 2, 200, 128
    q, k, v = cache_case(B, H, S, S, D, seed=11)
    kv_len = torch.tensor([0, 100, 0], dtype=torch.int32, device="cuda")
    for causal in (False, True):
        got = check(G, q, k, v, f"kv_len=[0,100,0] causal={causal}", causal=causal, kv_len=kv_len, sk=S)
        assert torch.isfinite(got).all()
        assert (got[0] == 0).all() and (got[2] == 0).all()
