"""two-CTA cluster variant of the wgmma GEMM (block_n=512 selects it): must agree with the single-CTA kernel and torch."""
import pytest
import torch
import torch.nn.functional as F

from tests import parity as P

pytestmark = pytest.mark.gpu


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (256, 256, 256), (512, 512, 1024), (300, 200, 192), (1000, 1024, 1024),
                                   (4096, 4096, 1024), (129, 300, 128), (2048, 1234, 320), (15456, 4096, 4096)])
def test_gemm_2cta_plain(M, N, K):
    from groma_b200 import ops as G
    a = rnd(M, K, seed=1).bfloat16().cuda(); w = rnd(N, K, seed=2).bfloat16().cuda()
    ref = (a.float() @ w.float().t()).cpu()
    o2 = G.gemm(a, w, out_f32=True, block_n=512).cpu()
    assert ((o2 - ref).abs().max() / ref.abs().max()).item() < 2e-5
    o1 = G.gemm(a, w, out_f32=True, block_n=256).cpu()
    assert torch.equal(o1, o2)          # same K order per element -> bit-identical accumulators


def test_gemm_2cta_epilogues_and_conv():
    """256- and 512-wide (two-CTA) epilogues: each per element against fp64 (tests/parity.py), and bit-identical."""
    from groma_b200 import ops as G
    M, N, K = 640, 768, 256
    a = rnd(M, K, seed=3).bfloat16().cuda(); w = rnd(N, K, seed=4, scale=0.1).bfloat16().cuda()
    bias = rnd(N, seed=5).cuda(); gamma = rnd(N, seed=6).cuda(); res = rnd(M, N, seed=7).bfloat16().cuda()
    acc, mag = a.double() @ w.double().t(), a.double().abs() @ w.double().abs().t()
    for act in (G.ACT_NONE, G.ACT_GELU, G.ACT_RELU):
        o1 = G.gemm(a, w, bias=bias, act=act, gamma=gamma, residual=res, block_n=256)
        o2 = G.gemm(a, w, bias=bias, act=act, gamma=gamma, residual=res, block_n=512)
        ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=bias, act=act, gamma=gamma, residual=res)
        P.check_gemm(o1, ref, lmag, what=f"block_n=256 act={act} bias+gamma+residual")
        P.check_gemm(o2, ref, lmag, what=f"block_n=512 act={act} bias+gamma+residual")
        assert torch.equal(o1, o2)
    o1, o2 = G.gemm(a, w, bias=bias, act=G.ACT_SWIGLU, block_n=256), G.gemm(a, w, bias=bias, act=G.ACT_SWIGLU, block_n=512)
    ref, lmag = P.gemm_epilogue_ref(acc, mag, bias=bias, act=G.ACT_SWIGLU)
    P.check_gemm(o1, ref, lmag, what="block_n=256 bias+swiglu")
    P.check_gemm(o2, ref, lmag, what="block_n=512 bias+swiglu")
    assert torch.equal(o1, o2)
    # 3x3 conv over zero-bordered maps, 3 stacked levels (27 taps)
    n_img, H, W, C, Cout, L = 3, 14, 14, 128, 256, 3
    xs = [rnd(n_img, C, H, W, seed=20 + l).bfloat16() for l in range(L)]
    ws = [rnd(Cout, C, 3, 3, seed=30 + l, scale=0.05).bfloat16() for l in range(L)]
    bias = rnd(Cout, seed=40)
    ref = F.relu(sum(F.conv2d(x.float(), w_.float(), padding=1) for x, w_ in zip(xs, ws)) + bias[None, :, None, None]).permute(0, 2, 3, 1).reshape(-1, Cout)
    acc64 = sum(F.conv2d(x.double(), w_.double(), padding=1) for x, w_ in zip(xs, ws)).permute(0, 2, 3, 1).reshape(-1, Cout)
    mag64 = sum(F.conv2d(x.double().abs(), w_.double().abs(), padding=1) for x, w_ in zip(xs, ws)).permute(0, 2, 3, 1).reshape(-1, Cout)
    ref64, lmag = P.gemm_epilogue_ref(acc64, mag64, bias=bias, act=G.ACT_RELU)
    xpad = torch.zeros((L, n_img, H + 2, W + 2, C), dtype=torch.bfloat16)
    for l in range(L):
        xpad[l, :, 1:-1, 1:-1] = xs[l].permute(0, 2, 3, 1)
    wt = torch.cat([w_.permute(0, 2, 3, 1).reshape(Cout, 9 * C) for w_ in ws], dim=1).contiguous()
    out = G.conv3x3_flat(xpad.reshape(-1, C).cuda(), wt.cuda(), n_img, H + 2, W + 2, bias=bias.cuda(), act=G.ACT_RELU, block_n=512)
    assert ((out.float().cpu() - ref).abs().max() / ref.abs().max()).item() < 6e-3
    P.check_gemm(out, ref64, lmag, what="conv3x3 27 taps block_n=512 bias+relu")
