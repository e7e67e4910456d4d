"""generate() with several prompts per image on the GPU: the grouped decode attention at Groma-7B head shapes against an fp64
attention and against the plain decode prologue (bit-exact appended row), eager / PDL / captured; and the miniature model's
grouped generate against the same rows run on repeated images."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from tests.parity import attention_ref, check_attention  # noqa: E402


def _rope_tables(n, D=128, theta=10000.0):
    inv = 1.0 / theta ** (torch.arange(0, D, 2, dtype=torch.float64) / D)
    fr = torch.outer(torch.arange(n, dtype=torch.float64), inv)
    return fr.cos().float().cuda().contiguous(), fr.sin().float().cuda().contiguous()


# ------------------------------------------------------------------------------------------------------- attention kernel
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n", [2, 7, 16, 64])
@pytest.mark.parametrize("P", [0, 1, 63, 64, 100, 965])   # 100: the launcher picks a 2-CTA cluster
@pytest.mark.parametrize("own", [1, 30, 158])
def test_grouped_attention(B, n, P, own):
    from groma_b200 import ops as G
    H, D, S = 32, 128, 3
    R = B * n
    rcap = own + 3
    pos_v = P + own - 1                       # own positions P .. pos_v, the last one appended by this step
    g = torch.Generator(device="cuda").manual_seed(B * 100000 + n * 1000 + P * 7 + own)
    pk = torch.randn(B, H, P, D, generator=g, device="cuda").bfloat16()
    pv = torch.randn(B, H, P, D, generator=g, device="cuda").bfloat16()
    rk = torch.randn(R, H, rcap, D, generator=g, device="cuda").bfloat16()
    rv = torch.randn(R, H, rcap, D, generator=g, device="cuda").bfloat16()
    ws = torch.randn(S, R, 3 * H * D, generator=g, device="cuda") * 0.5
    cos, sin = _rope_tables(pos_v + 1)
    pos = torch.tensor([pos_v], dtype=torch.int32, device="cuda")
    scale = 1.0 / math.sqrt(D)
    outs = []
    for pdl in (False, True):
        rk2, rv2 = rk.clone(), rv.clone()
        out = torch.empty(R, H * D, dtype=torch.bfloat16, device="cuda")
        G.decode_rope_attention_grouped(ws, pk, pv, rk2, rv2, pos, cos, sin, scale, out, n, pdl=pdl)
        outs.append((out, rk2, rv2))
    # inside a captured graph
    rk3, rv3 = rk.clone(), rv.clone()
    out3 = torch.empty(R, H * D, dtype=torch.bfloat16, device="cuda")
    G.decode_rope_attention_grouped(ws, pk, pv, rk3, rv3, pos, cos, sin, scale, out3, n)     # warm-up outside the capture
    out3.zero_()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            G.decode_rope_attention_grouped(ws, pk, pv, rk3, rv3, pos, cos, sin, scale, out3, n)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    outs.append((out3, rk3, rv3))
    torch.cuda.synchronize()
    out, rk2, rv2 = outs[0]
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(o, outs[0])), "two runs differ"
    # only index pos - P of the row cache changes
    s_new = pos_v - P
    keep = torch.ones(rcap, dtype=torch.bool, device="cuda")
    keep[s_new] = False
    assert torch.equal(rk2[:, :, keep], rk[:, :, keep]) and torch.equal(rv2[:, :, keep], rv[:, :, keep])
    # the plain reduce + RoPE + append on the gathered cache: q and the appended row, bit for bit
    ctx = pos_v + 1
    gk = torch.zeros(R, H, ctx + 1, D, dtype=torch.bfloat16, device="cuda")
    gv = torch.zeros_like(gk)
    rows = torch.arange(R, device="cuda")
    if P > 0:
        gk[:, :, :P] = pk[rows // n]
        gv[:, :, :P] = pv[rows // n]
    gk[:, :, P:pos_v] = rk[:, :, :s_new]
    gv[:, :, P:pos_v] = rv[:, :, :s_new]
    q = torch.empty(R, H * D, dtype=torch.bfloat16, device="cuda")
    G.decode_reduce_rope_kv(ws, q, gk, gv, cos, sin, pos, H, D, pdl=False)
    assert torch.equal(gk[:, :, pos_v], rk2[:, :, s_new]) and torch.equal(gv[:, :, pos_v], rv2[:, :, s_new])
    ref, pvm = attention_ref(q.reshape(R, 1, H, D), gk, gv, causal=False, scale=scale, sk=ctx)
    check_attention(out.reshape(R, 1, H * D), ref, pvm, what=f"grouped B={B} n={n} P={P} own={own}")


def test_grouped_attention_refuses():
    from groma_b200 import ops as G
    H, D = 4, 128
    ws = torch.zeros(1, 65, 3 * H * D, device="cuda")
    rk = torch.zeros(65, H, 4, D, dtype=torch.bfloat16, device="cuda")
    out = torch.empty(65, H * D, dtype=torch.bfloat16, device="cuda")
    cos, sin = _rope_tables(4)
    pos = torch.zeros(1, dtype=torch.int32, device="cuda")
    with pytest.raises(G._lib.GromaError, match="UNSUPPORTED"):
        G.decode_rope_attention_grouped(ws, None, None, rk, rk.clone(), pos, cos, sin, 1.0, out, 65)


# ------------------------------------------------------------------------------------------------------- generate on tiny_config
def _tiny_model(weights="bf16"):
    from groma.model.groma import GromaConfig, GromaModel
    from oracle.config import SyntheticTokenizer, tiny_config
    from oracle.weights import make_state_dict
    cfg = tiny_config(box_score_thres=0.0)
    sd = make_state_dict(cfg, seed=0)
    tok = SyntheticTokenizer(cfg.vocab)
    kw = dict(llm_weight_dtype=torch.float8_e4m3fn) if weights == "fp8" else {}
    model = GromaModel(GromaConfig.from_path_config(cfg), state_dict=sd, path_config=cfg, **kw)
    if weights == "nf4":
        model.quantize_nf4_(sd)
    model.init_special_token_id(tok)
    return model, tok


def _inputs(tok, n):
    """Two images; n questions per image that share the system text, image and regions, and differ in their last tokens (one
    row padded); the images' selections have 5 and 7 regions, so P is limited by the first image."""
    g = torch.Generator().manual_seed(n)
    images = torch.randn(2, 3, 448, 448, generator=g).cuda()
    base = torch.randint(10, 40, (20,), generator=g)
    base[3] = tok.map["<image>"]
    base[9] = tok.map["<region>"]
    ids = base.repeat(2 * n, 1)
    ids[:, 14:] = torch.randint(10, 40, (2 * n, 6), generator=g)
    ids[1, 17:] = tok.pad_token_id
    boxes = [torch.rand(5, 4, generator=g) * 0.6 + 0.2, torch.rand(7, 4, generator=g) * 0.6 + 0.2]
    return images, ids, boxes


def _run(model, ids, images, boxes, n, grouped, **kw):
    torch.manual_seed(1234)
    if grouped:
        out = model.generate(ids.clone().cuda(), images=images, _selected_override=boxes, _keep_logits=True,
                             return_dict_in_generate=True, output_hidden_states=True, **kw)
    else:
        out = model.generate(ids.clone().cuda(), images=images.repeat_interleave(n, 0),
                             _selected_override=[b for b in boxes for _ in range(n)], _keep_logits=True,
                             return_dict_in_generate=True, output_hidden_states=True, **kw)
    return out, [l.clone() for l in model._step_logits]


def _first_logits_match(got, ref):
    """The first-token logits: bit-identical when the suffix GEMMs pick the repeated run's tiles; else within 2^-7 of the
    row's logit range (the GEMM bound of bf16 activations at the miniature widths)."""
    if torch.equal(got, ref):
        return
    span = (ref.max(1, keepdim=True).values - ref.min(1, keepdim=True).values).clamp_min(1e-6)
    assert ((got - ref).abs() <= 2.0 ** -7 * span).all(), float(((got - ref).abs() / span).max())


def _agree_to_near_tie(seq_a, seq_b, logits_a, logits_b, L0, tol=2e-2, sampled=False):
    """Tokens equal step by step; at the first difference both runs' logits must make it a two-sided near-tie: each run's
    choice is within tol (relative to the row's logit range) of the other run's choice in both runs.  A sampled token
    turns on the cumulative distribution rather than on two logits, so there the two runs' logit rows must agree within tol."""
    new_a, new_b = seq_a[:, L0:], seq_b[:, L0:]
    steps = min(new_a.shape[1], new_b.shape[1], len(logits_a))
    for s in range(steps):
        diff = (new_a[:, s] != new_b[:, s]).nonzero().flatten().tolist()
        for r in diff:
            ta, tb = int(new_a[r, s]), int(new_b[r, s])
            if sampled:
                la, lb = logits_a[s][r], logits_b[s][r]
                span = float(lb.max() - lb.min()) or 1.0
                assert float((la - lb).abs().max()) <= tol * span, f"row {r} step {s}: sampled tokens differ on distinct logits"
                continue
            for lg in (logits_a[s][r], logits_b[s][r]):
                span = float(lg.max() - lg.min()) or 1.0
                assert abs(float(lg[ta] - lg[tb])) <= tol * span, f"row {r} step {s}: tokens {ta} / {tb} are not a near-tie"
        if diff:
            return s
    return steps


@pytest.fixture(scope="module")
def tiny():
    model, tok = _tiny_model()
    return dict(model=model, tok=tok)


@pytest.mark.parametrize("n", [2, 5])
@pytest.mark.parametrize("mode", ["greedy", "sample", "process"])
def test_grouped_generate_matches_repeated_images(tiny, n, mode):
    model, tok = tiny["model"], tiny["tok"]
    images, ids, boxes = _inputs(tok, n)
    kw = dict(max_new_tokens=10, eos_token_id=[])
    if mode == "sample":
        kw.update(do_sample=True, top_k=20, temperature=0.9)
    if mode == "process":
        kw.update(repetition_penalty=1.3, no_repeat_ngram_size=2)
    ref, ref_logits = _run(model, ids, images, boxes, n, grouped=False, **kw)
    eng = model.engine
    T = model._last["ids"].shape[1]
    ref_kv = eng.kv[:, :, ::n].clone()          # the first row of every image
    got, got_logits = _run(model, ids, images, boxes, n, grouped=True, **kw)
    grp = eng._group
    P = grp["P"]
    assert 0 < P < T
    # the prefix K/V: the same GEMM, RoPE and attention kernels on the same rows -> bit-identical
    assert torch.equal(grp["prefix"], ref_kv[:, :, :, :, :P])
    _first_logits_match(got_logits[0], ref_logits[0])
    assert got.sequences.shape[0] == 2 * n and got.past_key_values is None
    vis = got.hidden_states[0][-1]
    assert len(vis["pred_boxes"]) == 2 * n and vis["image_features"].shape[0] == 2
    for r in range(2 * n):
        assert torch.equal(vis["pred_boxes"][r].cpu(), boxes[r // n].float())
    if mode == "sample":
        # the Philox draw is keyed by (row, position): a grouped row draws what it draws ungrouped until the logits diverge
        s = _agree_to_near_tie(got.sequences.cpu(), ref.sequences.cpu(), got_logits, ref_logits, ids.shape[1], sampled=True)
    else:
        s = _agree_to_near_tie(got.sequences.cpu(), ref.sequences.cpu(), got_logits, ref_logits, ids.shape[1])
    assert s >= 1


def test_eager_equals_graph_and_plain_after_grouped(tiny):
    model, tok = tiny["model"], tiny["tok"]
    n = 4
    images, ids, boxes = _inputs(tok, n)
    kw = dict(max_new_tokens=8, eos_token_id=[])
    plain_ids = ids[::n].contiguous()
    model.use_cuda_graph = True
    plain0 = model.generate(plain_ids.clone().cuda(), images=images, _selected_override=boxes, **kw).cpu()
    plain_kernels = model._graph_kernels
    outs = []
    for graph in (False, True):
        model.use_cuda_graph = graph
        o, lg = _run(model, ids, images, boxes, n, grouped=True, **kw)
        outs.append((o.sequences.cpu(), lg))
    model.use_cuda_graph = True
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))
    # the grouped step keeps the plain step's launch count per layer (8 grouped rows vs 2 plain rows: the same kernels)
    assert model._graph_kernels == plain_kernels
    # a plain generate after a grouped one: bit-identical, same captured kernel count
    plain1 = model.generate(plain_ids.clone().cuda(), images=images, _selected_override=boxes, **kw).cpu()
    assert torch.equal(plain0, plain1) and model._graph_kernels == plain_kernels
    assert model.engine._group is None
    # a grouped call hands out no cache: a forward() continuation has nothing to continue from
    model.generate(ids.clone().cuda(), images=images, _selected_override=boxes, **kw)
    logits, pkv = model.forward(input_ids=plain_ids.clone().cuda(), images=images, use_cache=True, _selected_override=boxes)
    model.generate(ids.clone().cuda(), images=images, _selected_override=boxes, **kw)
    with pytest.raises(RuntimeError):
        model.forward(input_ids=torch.zeros(2, 1, dtype=torch.long).cuda(), past_key_values=pkv, use_cache=True)
    assert model.engine.kv_bytes() == (model.engine._group["prefix"].numel() + model.engine._group["row"].numel()) * 2
    # a forward() prefill frees the grouped caches
    model.forward(input_ids=plain_ids.clone().cuda(), images=images, use_cache=True, _selected_override=boxes)
    assert model.engine._group is None
    # a grouped call's override holds one selection per image, not one per row
    with pytest.raises(ValueError, match="one selection per image"):
        model.generate(ids.clone().cuda(), images=images, _selected_override=[b for b in boxes for _ in range(n)], **kw)


@pytest.mark.parametrize("weights", ["nf4", "fp8"])
def test_grouped_generate_quantized_weights(weights):
    model, tok = _tiny_model(weights)
    n = 3
    images, ids, boxes = _inputs(tok, n)
    kw = dict(max_new_tokens=8, eos_token_id=[])
    ref, ref_logits = _run(model, ids, images, boxes, n, grouped=False, **kw)
    got, got_logits = _run(model, ids, images, boxes, n, grouped=True, **kw)
    _first_logits_match(got_logits[0], ref_logits[0])
    assert _agree_to_near_tie(got.sequences.cpu(), ref.sequences.cpu(), got_logits, ref_logits, ids.shape[1]) >= 1
