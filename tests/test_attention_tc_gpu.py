"""wgmma flash-attention kernel at LLaMA prefill and DINOv2 shapes, both operand layouts (KV cache [B,H,cap,D] and
fused-qkv activation slices): per element against the fp64 reference of tests/parity.py, and in agreement with the
mma.sync kernel (ops.attention).  The edge cases of the tiling are in tests/test_attention_wgmma_gpu.py."""
import math

import pytest
import torch

from tests import parity as P

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def check(got, q, k, v, what, *, causal, scale, q_pos0=0, kv_len=None):
    ref, pv = P.attention_ref(q.cuda(), k.cuda(), v.cuda(), causal=causal, scale=scale, q_pos0=q_pos0,
                              kv_len=None if kv_len is None else kv_len.cuda())
    P.check_attention(got, ref, pv, what=what)
    return ref


@pytest.mark.parametrize("B,H,S,D,causal", [(1, 1, 128, 128, False), (1, 1, 128, 64, False), (2, 3, 200, 128, True), (2, 2, 1025, 64, False),
                                            (1, 2, 966, 128, True), (3, 2, 70, 64, True),
                                            # S = 1027, 260, 5, 136, 137, 528, 529, 1025: a ragged last key tile of 3, 4, 5, 8, 9, 16,
                                            # 17 or 1 keys and a last query tile of as many rows (warpgroup 1 idle); 1025 causal: 9 tiles
                                            (2, 2, 1027, 128, False), (2, 3, 260, 64, False), (1, 2, 5, 64, False), (2, 1, 136, 128, False),
                                            (1, 2, 137, 64, False), (1, 2, 528, 64, False), (1, 1, 529, 128, False), (2, 2, 1025, 64, True)])
def test_attention_tc_cache_layout(B, H, S, D, causal):
    from groma_b200 import ops as G
    cap = S + 37
    q = rnd(B, S, H, D, seed=1).bfloat16()
    kc = torch.zeros(B, H, cap, D, dtype=torch.bfloat16); vc = torch.zeros_like(kc)
    kc[:, :, :S] = rnd(B, H, S, D, seed=2).bfloat16(); vc[:, :, :S] = rnd(B, H, S, D, seed=3).bfloat16()
    scale = 1.0 / math.sqrt(D)
    got = G.attention_tc(q.cuda(), kc.cuda(), vc.cuda(), causal=causal, scale=scale, sk=S)
    ref = check(got, q, kc[:, :, :S], vc[:, :, :S], f"B={B} H={H} S={S} D={D} causal={causal}", causal=causal, scale=scale)
    # agrees with the mma.sync kernel too
    old = G.attention(q.cuda(), kc.cuda(), vc.cuda(), causal=causal, scale=scale, sk=S)
    assert ((got.double() - old.double()).abs().max() / ref.abs().max()).item() < 1e-2


def test_attention_tc_qkv_layout_and_kvlen():
    from groma_b200 import ops as G
    B, S, H, D = 2, 300, 4, 64
    qkv = rnd(B, S, 3 * H * D, seed=4).bfloat16()
    x = qkv.cuda().reshape(B, S, 3, H, D)
    q, k, v = x[:, :, 0], x[:, :, 1].permute(0, 2, 1, 3), x[:, :, 2].permute(0, 2, 1, 3)
    # one sequence ends inside key tile 0; then one ends 2 keys into key tile 2 (rows 256, 257)
    for lens in ([300, 111], [258, 300]):
        kv_len = torch.tensor(lens, dtype=torch.int32)
        got = G.attention_tc(q, k, v, causal=False, scale=0.125, kv_len=kv_len.cuda())
        check(got, q, k, v, f"qkv layout kv_len={lens}", causal=False, scale=0.125, kv_len=kv_len)
    # causal + kv_len + right-padded rows (LLaMA prefill semantics): rows beyond kv_len still produce finite output
    B, S, H, D = 2, 190, 2, 128
    q = rnd(B, S, H, D, seed=5).bfloat16(); kc = rnd(B, H, 256, D, seed=6).bfloat16(); vc = rnd(B, H, 256, D, seed=7).bfloat16()
    kv_len = torch.tensor([190, 60], dtype=torch.int32)
    got = G.attention_tc(q.cuda(), kc.cuda(), vc.cuda(), causal=True, scale=0.088, kv_len=kv_len.cuda(), sk=S)
    assert torch.isfinite(got).all()
    check(got, q, kc[:, :, :S], vc[:, :, :S], "causal kv_len=[190, 60]", causal=True, scale=0.088, kv_len=kv_len)


def test_attention_tc_query_tail_row_with_ragged_kv():
    """Sq = 4 * 128 + 1, D = 64, non-causal: the last query tile holds one row (warpgroup 1 wholly past Sq).  Ragged kv_len:
    a partly valid last key tile, 2 keys into a tile (258), a length shorter than one tile (7), exactly four tiles (512)."""
    from groma_b200 import ops as G
    B, S, H, D = 4, 513, 2, 64
    q = rnd(B, S, H, D, seed=21).bfloat16(); kc = rnd(B, H, S, D, seed=22).bfloat16(); vc = rnd(B, H, S, D, seed=23).bfloat16()
    for lens in ([513, 130, 258, 7], [513, 513, 512, 385]):
        kv_len = torch.tensor(lens, dtype=torch.int32)
        got = G.attention_tc(q.cuda(), kc.cuda(), vc.cuda(), causal=False, scale=0.125, kv_len=kv_len.cuda(), sk=S)
        assert torch.isfinite(got).all()
        check(got, q, kc, vc, f"Sq=513 kv_len={lens}", causal=False, scale=0.125, kv_len=kv_len)
        check(got[:, -1:], q[:, -1:], kc, vc, f"Sq=513 kv_len={lens} last row", causal=False, scale=0.125, kv_len=kv_len)
