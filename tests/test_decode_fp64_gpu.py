"""The default (bf16-cache) decode step against fp64 at Groma-7B shapes (tests/parity.py has the references and bounds):
  - decode attention, TMA ring and LDG kernels (every GROMA_DEC_UNROLL), 32 heads, context edges at the 16-key chunks and the
    2-CTA split, peaked softmax with the maximum placed where the running-max correction and the cross-CTA merge matter; the
    cache is carved out of a NaN-filled allocation, so a read past a row's keys or into the next head shows up as NaN;
  - the fused qkv reduce + RoPE + KV append (decode_reduce_rope_kv, decode_rope_attention) against an independent fp64 RoPE,
    with tables from GromaEngine.ensure_rope, at split boundaries, cap - 1 and past max_pos;
  - the split-K reduce epilogues (residual + RMSNorm on all three kernels, SwiGLU, head reduce + argmax);
  - one whole step (default, unfused and persistent) of a 2-layer LLaMA at Groma-7B width against the bf16 oracle.
Run with -s to see the worst err/bound ratio of every case."""
import math
import os
import subprocess
import sys

import pytest
import torch

from tests import parity as P
from tests.fullsize import BARS, nrel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 128
SCALE = 1.0 / math.sqrt(D)
NAN = float("nan")


@pytest.fixture(scope="module")
def G():
    from groma_b200 import ops
    return ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _carve(shape, fill=NAN, pad_rows=64):
    """A contiguous bf16 tensor of `shape` at the start of a larger allocation whose tail (pad_rows rows of D) holds `fill`.
    Returns (view, whole allocation)."""
    n = math.prod(shape)
    buf = torch.full((n + pad_rows * D,), fill, dtype=torch.bfloat16, device="cuda")
    return buf[:n].view(shape), buf


def _visible(kv_len, cap):
    """[B, 1, cap, 1] mask of the keys a row attends."""
    return (torch.arange(cap, device=kv_len.device)[None, :] < kv_len.long()[:, None])[:, None, :, None]


def _attention_ref(q, k, v, kv_len):
    """fp64 attention of q [B, H*D] over the first kv_len[b] keys of k, v [B, H, cap, D]; keys past kv_len (NaN here) are
    zeroed first -- they carry no weight, and a kernel that reads them returns NaN."""
    B, H, cap, _ = k.shape
    vis = _visible(kv_len, cap)
    k0 = torch.where(vis, k.double(), 0.0)
    v0 = torch.where(vis, v.double(), 0.0)
    return P.attention_ref(q.reshape(B, 1, H, D), k0, v0, causal=False, scale=SCALE, kv_len=kv_len)


# ------------------------------------------------------------------------------------------------------- decode attention
ATT_CTX = (1, 2, 15, 16, 17, 31, 32, 33, 64, 65, 1030, 4096)
ATT_CASES = [(B, H, ctx) for B in (1, 5, 16) for H in (4, 32) for ctx in ATT_CTX]
PEAKS = ("flat", "last_key", "second_cta_first_key", "partial_last_chunk", "rising")
LDG_UNROLLS = (4, 2, 6, 8)


def _peak_index(kind, n):
    """Key that gets the maximum score in a row of n keys (2-CTA split: CTA 1 holds keys [per, n); 16-key chunks)."""
    per = (n + 1) // 2
    if kind == "last_key":
        return n - 1
    if kind == "second_cta_first_key":
        return per if per < n else n - 1
    lo, cnt = (per, n - per) if n > per else (0, per)
    return lo + 16 * ((cnt - 1) // 16)          # first key of the CTA's last chunk (partial unless cnt % 16 == 0)


def _att_inputs(B, H, ctx):
    """q [B, H*D] bf16; k, v [B, H, cap, D] bf16 views into NaN-padded allocations, NaN at every position >= kv_len[b];
    kv_len int32 [B].  Odd contexts with B > 1 have ragged rows, row 0 always has kv_len = ctx; full rows have cap = ctx + 5.
    Scores ~ N(0, 8^2) (a peaked softmax); per (b, h) one of PEAKS: the maximum (+40) at a chosen key, or a ramp -30 .. +30
    over the key order (every chunk beats the one before: the running-max correction runs at every update)."""
    g = _gen(B * 100003 + H * 1009 + ctx)
    ragged = B > 1 and ctx % 2 == 1
    cap = ctx if ragged else ctx + 5
    kv_len = torch.full((B,), ctx, dtype=torch.int32, device="cuda")
    if ragged:
        kv_len = torch.randint(1, ctx + 1, (B,), generator=g, device="cuda", dtype=torch.int32)
        kv_len[0] = ctx
    q = torch.randn(B, H, D, generator=g, device="cuda") * 8.0
    q = q.bfloat16().float()
    kf = torch.randn(B, H, cap, D, generator=g, device="cuda")
    vf = torch.randn(B, H, cap, D, generator=g, device="cuda")
    qn2 = q.pow(2).sum(-1)                                          # [B, H]
    delta = torch.zeros(B, H, cap, device="cuda")
    rising = torch.zeros(B, H, dtype=torch.bool, device="cuda")
    lens = kv_len.tolist()
    for b in range(B):
        n = lens[b]
        for h in range(H):
            kind = PEAKS[(b * H + h + ctx) % len(PEAKS)]
            if kind == "rising":
                rising[b, h] = True
                delta[b, h, :n] = torch.linspace(-30.0, 30.0, n, device="cuda")
            elif kind != "flat":
                delta[b, h, _peak_index(kind, n)] = 40.0
    # rising rows: drop the random part of the score, so the ramp alone orders the keys
    proj = (kf * q[:, :, None, :]).sum(-1, keepdim=True) / qn2[:, :, None, None] * q[:, :, None, :]
    kf = torch.where(rising[:, :, None, None], kf - proj, kf)
    kf = kf + (delta / SCALE / qn2[:, :, None])[..., None] * q[:, :, None, :]
    k, kbuf = _carve((B, H, cap, D))
    v, vbuf = _carve((B, H, cap, D))
    vis = _visible(kv_len, cap)
    k.copy_(torch.where(vis, kf, NAN))
    v.copy_(torch.where(vis, vf, NAN))
    return q.bfloat16().reshape(B, H * D).contiguous(), k, v, kv_len


def _run_attention_cases(path):
    """Every ATT_CASES output of this process's decode attention kernel, saved to `path` (GROMA_DEC_ATTN_TMA and
    GROMA_DEC_UNROLL pick the kernel; both are read once per process)."""
    from groma_b200 import ops
    outs = {}
    for c in ATT_CASES:
        q, k, v, kv_len = _att_inputs(*c)
        out = torch.empty_like(q)
        ops.decode_attention(q, k, v, kv_len, SCALE, out)
        outs[c] = out.cpu()
    torch.save(outs, path)


@pytest.fixture(scope="module")
def ldg_outputs(tmp_path_factory):
    """{unroll: {case: output}} of the LDG kernel, one process per GROMA_DEC_UNROLL."""
    res = {}
    for u in LDG_UNROLLS:
        path = str(tmp_path_factory.mktemp(f"ldg{u}") / "out.pt")
        code = (f"import sys; sys.path.insert(0, {ROOT!r}); from tests.test_decode_fp64_gpu import _run_attention_cases; "
                f"_run_attention_cases({path!r})")
        env = {**os.environ, "GROMA_DEC_ATTN_TMA": "0", "GROMA_DEC_UNROLL": str(u)}
        subprocess.run([sys.executable, "-c", code], env=env, check=True, cwd=ROOT)
        res[u] = torch.load(path)
    return res


@pytest.mark.parametrize("case", ATT_CASES, ids=lambda c: "B%d-H%d-ctx%d" % c)
def test_decode_attention_tma_and_ldg_vs_fp64(G, ldg_outputs, case):
    """TMA ring kernel within the fp64 attention bound; LDG kernel at unroll 4 bit-identical to it, at unroll 2 / 6 / 8
    within the bound."""
    assert os.environ.get("GROMA_DEC_ATTN_TMA", "1") != "0"
    B = case[0]
    q, k, v, kv_len = _att_inputs(*case)
    out = torch.empty_like(q)
    G.decode_attention(q, k, v, kv_len, SCALE, out)
    ref, pv = _attention_ref(q, k, v, kv_len)
    P.check_attention(out.reshape(B, 1, -1), ref, pv, what=f"decode tma {case}")
    assert torch.equal(ldg_outputs[4][case], out.cpu()), "LDG kernel (unroll 4) differs from the TMA kernel"
    for u in LDG_UNROLLS[1:]:
        P.check_attention(ldg_outputs[u][case].cuda().reshape(B, 1, -1), ref, pv, what=f"decode ldg unroll {u} {case}")


def test_decode_attention_empty_row_is_zero(G):
    """kv_len = 0: the row's output is exactly 0 (its whole cache block is NaN and must not be read)."""
    B, H, cap = 3, 4, 40
    g = _gen(77)
    kv_len = torch.tensor([0, 40, 17], dtype=torch.int32, device="cuda")
    q = torch.randn(B, H * D, generator=g, device="cuda").bfloat16()
    k, _ = _carve((B, H, cap, D))
    v, _ = _carve((B, H, cap, D))
    vis = _visible(kv_len, cap)
    k.copy_(torch.where(vis, torch.randn(B, H, cap, D, generator=g, device="cuda"), NAN))
    v.copy_(torch.where(vis, torch.randn(B, H, cap, D, generator=g, device="cuda"), NAN))
    out = torch.full_like(q, 7.0)
    G.decode_attention(q, k, v, kv_len, SCALE, out)
    assert torch.equal(out[0], torch.zeros_like(out[0]))
    ref, pv = _attention_ref(q, k, v, kv_len)
    P.check_attention(out.reshape(B, 1, -1), ref, pv, what="decode tma kv_len 0 / 40 / 17")


# ------------------------------------------------------------------------------------------------- fused RoPE + KV append
ROPE_S = (1, 3, 16, 17)
ROPE_POS = (0, 15, 16, 257, 1030, 5000)
ROPE_H = 32


@pytest.fixture(scope="module")
def rope_tables():
    """cos / sin tables of a real engine (head_dim 128), rebuilt past max_pos by ensure_rope."""
    from groma_b200.config import tiny_config
    from groma_b200.engine import GromaEngine
    from groma_b200.synth import make_state_dict
    cfg = tiny_config()
    eng = GromaEngine(cfg, make_state_dict(cfg, seed=0))
    assert cfg.head_dim == D and eng.rope_len == cfg.max_pos < 5001
    eng.ensure_rope(5001)
    assert eng.rope_len >= 5001
    return eng.rope_cos, eng.rope_sin, cfg.rope_theta


def _rope_inputs(S, pos):
    """ws [S, B, 3*H*D]; kv_len with the appended position as the last key (row 0), the last key of CTA 0 (row 1), the first
    key of CTA 1 (row 2) and past the row's keys (row 3); the cache with NaN at pos (stale row) and past each kv_len."""
    B, H = 4, ROPE_H
    g = _gen(S * 7919 + pos)
    lens = [pos + 1, 2 * pos + 2, 2 * pos, pos // 2]
    cap = pos + 1 if pos == 1030 else max(lens) + 3         # pos = 1030: the appended row is the last of its (b, h) block
    kv_len = torch.tensor([min(n, cap) for n in lens], dtype=torch.int32, device="cuda")
    ws = torch.randn(S, B, 3 * H * D, generator=g, device="cuda") * (1.5 / math.sqrt(S))
    k, kbuf = _carve((B, H, cap, D))
    v, vbuf = _carve((B, H, cap, D))
    vis = _visible(kv_len, cap)
    k.copy_(torch.where(vis, torch.randn(B, H, cap, D, generator=g, device="cuda"), NAN))
    v.copy_(torch.where(vis, torch.randn(B, H, cap, D, generator=g, device="cuda"), NAN))
    k[:, :, pos] = NAN
    v[:, :, pos] = NAN
    return ws, kv_len, (k, kbuf), (v, vbuf)


def _only_row_changed(buf_after, buf_before, view_after, pos):
    """The allocation holding the cache is unchanged except at position pos of every (b, h) block."""
    a = buf_after.clone()
    a[: view_after.numel()].view(view_after.shape)[:, :, pos] = buf_before[: view_after.numel()].view(view_after.shape)[:, :, pos]
    return torch.equal(a.view(torch.int16), buf_before.view(torch.int16))


@pytest.mark.parametrize("pos", ROPE_POS)
@pytest.mark.parametrize("S", ROPE_S)
def test_rope_append_and_fused_attention_vs_fp64(G, rope_tables, S, pos):
    cos_t, sin_t, theta = rope_tables
    B, H = 4, ROPE_H
    ws, kv_len, (k0, kbuf0), (v0, vbuf0) = _rope_inputs(S, pos)
    pos_t = torch.tensor([pos], dtype=torch.int32, device="cuda")
    wsv = ws.view(S, B, 3, H, D)
    q_ref, q_bound = P.rope_ref(wsv[:, :, 0], pos, theta)
    k_ref, k_bound = P.rope_ref(wsv[:, :, 1], pos, theta)
    v_sum, v_mag = P.splitk_ref(wsv[:, :, 2])
    v_lo, v_hi = P.rounding_interval(v_sum, (S - 1) * P.U32 * v_mag)

    # stand-alone reduce + RoPE + append
    kbuf1, vbuf1 = kbuf0.clone(), vbuf0.clone()
    k1, v1 = kbuf1[: k0.numel()].view(k0.shape), vbuf1[: v0.numel()].view(v0.shape)
    q = torch.empty(B, H * D, dtype=torch.bfloat16, device="cuda")
    G.decode_reduce_rope_kv(ws, q, k1, v1, cos_t, sin_t, pos_t, H, D, pdl=False)
    # fused into the attention launch
    kbuf2, vbuf2 = kbuf0.clone(), vbuf0.clone()
    k2, v2 = kbuf2[: k0.numel()].view(k0.shape), vbuf2[: v0.numel()].view(v0.shape)
    out = torch.empty(B, H * D, dtype=torch.bfloat16, device="cuda")
    G.decode_rope_attention(ws, k2, v2, kv_len, pos_t, cos_t, sin_t, SCALE, out, pdl=False)
    torch.cuda.synchronize()

    tag = f"S={S} pos={pos}"
    P.check_bound("rope", q.view(B, H, D), q_ref, q_bound, what=f"q {tag}")
    for name, kc, vc, kb, vb in (("reduce_rope_kv", k1, v1, kbuf1, vbuf1), ("rope_attention", k2, v2, kbuf2, vbuf2)):
        P.check_bound("rope", kc[:, :, pos], k_ref, k_bound, what=f"appended k {name} {tag}")
        P.check_rounded(vc[:, :, pos], v_lo, v_hi, what=f"appended v {name} {tag}")
        assert _only_row_changed(kb, kbuf0, k0, pos) and _only_row_changed(vb, vbuf0, v0, pos), f"{name}: a row other than pos changed"
    ref, pv = _attention_ref(q, k2, v2, kv_len)
    P.check_attention(out.reshape(B, 1, -1), ref, pv, what=f"fused rope attention {tag}")


# ------------------------------------------------------------------------------------------------- reduce epilogues, head tail
EPI_S = (1, 2, 13, 16, 17)
EPS = 1e-5


@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("S", EPI_S)
@pytest.mark.parametrize("N", [256, 1000, 4096, 5120])   # kernel <1> (1000: a partial warp), the 8-CTA cluster, kernel <4>
def test_reduce_norm_vs_fp64(G, N, S, B):
    g = _gen(N * 31 + S * 7 + B)
    # rows from embedding scale (~1e-2: eps is a visible part of mean(h^2)) to a grown residual stream
    scale = (torch.logspace(-2, 0.8, B, device="cuda") if B > 1 else torch.tensor([0.02], device="cuda"))[:, None]
    ws = torch.randn(S, B, N, generator=g, device="cuda") * scale * (0.5 / math.sqrt(S))
    x0 = (torch.randn(B, N, generator=g, device="cuda") * scale).bfloat16()
    w = 1 + 0.1 * torch.randn(N, generator=g, device="cuda")
    x = x0.clone()
    y = torch.empty_like(x)
    G.decode_reduce_norm(ws, x, w, y, EPS, pdl=False)
    tag = f"N={N} S={S} B={B}"
    P.check_rounded(x, *P.residual_interval(ws, x0), what=f"reduce_norm residual {tag}")
    ref, bound = P.rmsnorm_ref(x, w, EPS)
    P.check_bound("rmsnorm", y, ref, bound, what=f"reduce_norm {tag}")


@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("S", EPI_S)
@pytest.mark.parametrize("N", [512, 2 * 11008])
def test_reduce_swiglu_vs_fp64(G, N, S, B):
    g = _gen(N * 37 + S * 11 + B)
    ws = torch.randn(S, B, N, generator=g, device="cuda") * (2.0 / math.sqrt(S))
    out = torch.empty(B, N // 2, dtype=torch.bfloat16, device="cuda")
    G.decode_reduce_swiglu(ws, out, pdl=False)
    ref, bound = P.splitk_swiglu_ref(ws)
    P.check_bound("swiglu", out, ref, bound, what=f"reduce_swiglu N={N} S={S} B={B}")


def test_head_argmax_vs_fp64(G):
    """V = 32114 (the last 1/8 slice and the last thread pass are ragged), S = 16, B = 16: logits within the split-K bound;
    ids the fp64 argmax except where the fp64 top-2 gap lies inside the bound."""
    S, B, V = 16, 16, 32114
    g = _gen(4242)
    ws = torch.randn(S, B, V, generator=g, device="cuda") * (3.0 / math.sqrt(S))
    ws[:, 3, V - 1] += 30.0 / S                                # maxima in the last column and in rank 7's slice
    ws[:, 4, V - 5000] += 30.0 / S
    logits = torch.empty(B, V, device="cuda")
    ids = torch.full((B,), -1, dtype=torch.int64, device="cuda")
    pos = torch.tensor([41], dtype=torch.int32, device="cuda")
    kvl = torch.arange(B, dtype=torch.int32, device="cuda") + 40
    G.decode_head_argmax(ws, logits, ids, pos, kvl, pdl=False)
    ref, mag = P.splitk_ref(ws)
    bound = P.splitk_bound(ref, mag, S)
    P.check_bound("splitk", logits, ref, bound, what="head logits V=32114 S=16 B=16")
    want = ref.argmax(-1)
    rows = torch.arange(B, device="cuda")
    gap = ref[rows, want] - ref[rows, ids]
    assert bool((gap <= bound[rows, want] + bound[rows, ids]).all()), (ids.tolist(), want.tolist())
    assert torch.equal(ids, logits.argmax(-1))
    assert ids[3].item() == V - 1 and ids[4].item() == V - 5000
    assert pos.item() == 42 and torch.equal(kvl, torch.arange(B, dtype=torch.int32, device="cuda") + 41)


# ------------------------------------------------------------------------------------------------- one step at Groma-7B width
CTX = 1030


@pytest.fixture(scope="module")
def wide():
    """A bare engine with the Groma-7B LLaMA width (4096 / 32 heads / 11008 / 32000 + 114) at depth 2 and a tiny vision side
    (the step never touches it), plus bf16 and fp32 oracles sharing the widened weights."""
    from groma_b200.config import tiny_config
    from groma_b200.engine import GromaEngine
    from groma_b200.synth import make_state_dict
    from oracle.groma_oracle import Oracle
    from tests.fullsize import widen_state_dict
    cfg = tiny_config(llm_hidden=4096, llm_layers=2, llm_heads=32, llm_inter=11008, vocab=32000, max_pos=4096)
    sd = make_state_dict(cfg, seed=0, dtype=torch.bfloat16, device="cuda")
    eng = GromaEngine(cfg, sd)
    sd32 = widen_state_dict(sd)
    del sd
    return dict(cfg=cfg, eng=eng, ob=Oracle(cfg, sd32, "bf16", prerounded=True), of=Oracle(cfg, sd32, "fp32", prerounded=True))


def _oracle_step(o, ids, kv, kv_len, pos):
    """One decode step of oracle o over the GPU's cache kv [L, 2, B, H, >= pos, D]: (logits [B, V], appended k / v rows
    [L, 2, B, H, D])."""
    L = kv.shape[0]
    past = [(kv[i, 0, :, :, :pos].permute(0, 2, 1, 3).float().cpu(), kv[i, 1, :, :, :pos].permute(0, 2, 1, 3).float().cpu())
            for i in range(L)]
    x = o.embed(ids.cpu())[:, None]
    h, new = o.llm(x, kv=past, kv_len=kv_len.cpu().long(), pos0=pos)
    rows = torch.stack([torch.stack([new[i][0][:, pos], new[i][1][:, pos]]) for i in range(L)])
    return o.logits(h)[:, 0], rows


def _bar(floor):
    """tests/fullsize.py's rule: no further from the bf16 oracle than floor_factor x its distance from the fp32 oracle + eps."""
    return BARS["floor_factor"] * floor + BARS["eps"]


@pytest.mark.parametrize("B", [16, 3])
def test_wide_decode_step_vs_oracle(wide, B):
    """Two consecutive steps of the default (fused, PDL, fused rope attention, fused head tail), unfused and persistent
    decode step; logits and the appended K/V rows of both layers within fullsize.BARS of the bf16 oracle (floor: the bf16
    oracle's distance from the fp32 oracle on the same inputs), tokens equal up to a two-sided near-tie.  B = 3: row 1 is
    right-padded -- its kv_len stops at 700 prompt tokens while the step appends at the shared position."""
    cfg, eng, ob, of = wide["cfg"], wide["eng"], wide["ob"], wide["of"]
    V = cfg.vocab + cfg.num_new_token
    g = _gen(1000 + B)
    eng.alloc_kv(B, CTX + 6)
    kv0 = torch.zeros_like(eng.kv)
    kv0[:, :, :, :, :CTX] = torch.randn(kv0[:, :, :, :, :CTX].shape, generator=g, device="cuda").bfloat16()
    ids0 = torch.randint(0, V, (B,), generator=g, device="cuda")
    kvl0 = torch.full((B,), CTX + 1, dtype=torch.int32, device="cuda")
    if B == 3:
        kvl0[1] = 701
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    first = {}
    for mode in ("default", "unfused", "mega"):
        eng.use_megakernel, eng.fused_decode = mode == "mega", mode != "unfused"
        eng.use_pdl = eng.fused_rope_attn = eng.fused_head_tail = True
        eng.kv.copy_(kv0)
        d = eng._decode_buffers(B)
        d["ids"].copy_(ids0)
        d["pos"].fill_(CTX)
        d["kv_len"].copy_(kvl0)
        for step in range(2):
            pos = CTX + step
            ids_in, kvl_in = d["ids"].clone(), d["kv_len"].clone()
            logits = eng.decode_step(B).clone()
            if mode == "mega":
                eng.check_decode_status()
                assert eng._mk["grid"] == sms
            torch.cuda.synchronize()
            got_rows = eng.kv[:, :, :, :, pos].float().cpu()
            assert int(d["pos"].item()) == pos + 1 and torch.equal(d["kv_len"], kvl_in + 1)
            # the oracles see the GPU's own cache (its earlier appended rows included) and input ids
            key = (step, tuple(ids_in.tolist()))
            if step == 0 and key in first:
                (lb, rb), (lf, rf) = first[key]
            else:
                (lb, rb), (lf, rf) = _oracle_step(ob, ids_in, eng.kv, kvl_in, pos), _oracle_step(of, ids_in, eng.kv, kvl_in, pos)
                if step == 0:
                    first[key] = (lb, rb), (lf, rf)
            tag = f"B={B} {mode} step {step}"
            fl = nrel(lb, lf)
            e = nrel(logits, lb)
            print(f"[wide] {tag}: logits nrel {e:.3e} (floor {fl:.3e}, bar {_bar(fl):.3e})")
            assert e <= _bar(fl), f"{tag}: logits {e:.3e} > bar {_bar(fl):.3e}"
            for i in range(cfg.llm_layers):
                for j, kv_name in enumerate("kv"):
                    fr, er = nrel(rb[i, j], rf[i, j]), nrel(got_rows[i, j], rb[i, j])
                    print(f"[wide] {tag}: layer {i} appended {kv_name} nrel {er:.3e} (floor {fr:.3e})")
                    assert er <= _bar(fr), f"{tag}: layer {i} {kv_name} row {er:.3e} > bar {_bar(fr):.3e}"
            # greedy token: the oracle's, or a near-tie on both sides (fullsize.verdict's rule)
            lim = _bar(fl)
            got_ids = d["ids"].cpu()
            lg = logits.cpu()
            for b in range(B):
                gt, ot = int(got_ids[b]), int(lb[b].argmax())
                assert gt == int(lg[b].argmax())
                if gt != ot:
                    og = ((lb[b, ot] - lb[b, gt]) / lb[b].abs().max()).item()
                    gg = ((lg[b, gt] - lg[b, ot]) / lg[b].abs().max()).item()
                    print(f"[wide] {tag}: row {b} token {gt} vs oracle {ot}, gaps {og:.3e} / {gg:.3e} (limit {lim:.3e})")
                    assert og <= lim and gg <= lim, f"{tag}: row {b} token diverges outside the noise floor"
