"""Cost of the decode step of Groma-7B (random-init weights) when n prompts share one image: the grouped graph step at (B, n)
(B*n rows through the decode GEMMs, groma_decode_rope_attention_grouped over each image's shared prefix of P positions and each
row's own positions) against the plain graph step over the same B*n rows with a full prompt copy per row (the same prompts
run on repeated images).  Prompt ctx T = 1030 with P = 1000 shared positions (system text, 256 image tokens, the regions),
measured at generated index s = 64.  The steps are CUDA graphs timed alternately in one process with CUDA events.  Then the
attention alone (a graph of its 32 launches) in TB/s of algorithmic bytes: B*P*0.5 MiB of prefix K/V plus
B*n*(T - P + s + 1)*0.5 MiB of own K/V for the grouped kernel, B*n*(T + s + 1)*0.5 MiB for the plain one.
Then one image with 16 questions (a ~1000-token prompt of which the last 8 tokens differ, 100 regions, 10 new tokens), end to
end three ways: 16 batch-1 generate() calls, one generate() over 16 copies of the image, and one grouped generate(); with the
LLaMA prefill of the batched and grouped calls read off generate()'s stage marks (model.profile).  Last, the grouped prefill's
staging copies alone (32 layers of prefix broadcast + suffix copy into the row cache) at n = 16 and 64, and the grouped
prefill they sit in.
Prints the card and its power limit with the numbers, and one JSON line at the end.
    python tools/decode_groups.py [reps]"""
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from groma.model.groma import GromaConfig, GromaModel  # noqa: E402
from groma_b200 import ops as G  # noqa: E402
from groma_b200.config import PathConfig, SyntheticTokenizer  # noqa: E402
from groma_b200.synth import make_state_dict  # noqa: E402

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
T, P, S_GEN, MAX_NEW = 1030, 1000, 64, 128
if not torch.cuda.is_available():
    raise SystemExit("decode_groups.py measures on a CUDA device; none is visible")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
except Exception as e:  # the numbers are still printed, marked as taken on an unidentified card
    card = f"{torch.cuda.get_device_name()} (power limit unknown: {e})"
print(f"card: {card}", flush=True)

cfg = PathConfig(box_score_thres=0.0)
sd = make_state_dict(cfg, seed=0, perturb_norms=False, dtype=torch.bfloat16, device="cuda")
model = GromaModel(GromaConfig.from_path_config(cfg), state_dict=sd, path_config=cfg)
tok = SyntheticTokenizer(cfg.vocab)
model.init_special_token_id(tok)
eng = model.engine
del sd
eng.ensure_rope(T + MAX_NEW + 64)
HALF_MIB = cfg.llm_layers * 2 * cfg.llm_heads * cfg.head_dim * 2      # K/V bytes of one position over all layers (0.5 MiB)
POS = T + S_GEN


def med(ts):
    ts = sorted(ts)
    return ts[len(ts) // 2]


def graph_of(fn, reset):
    g = torch.cuda.CUDAGraph(); st = torch.cuda.Stream(); st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        reset(); fn(); reset()
        with torch.cuda.graph(g, stream=st, capture_error_mode="thread_local"):
            fn()
    torch.cuda.current_stream().wait_stream(st)
    return g


def timed(g, reset):
    reset()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1)


results = {}
for B, n in ((1, 16), (4, 4), (1, 64)):
    R = B * n
    eng.drop_kv(); eng.drop_group(); torch.cuda.empty_cache()
    d = eng._decode_buffers(R)

    def reset():
        d["ids"].fill_(1234); d["pos"].fill_(POS); d["kv_len"].fill_(POS + 1)
    # plain rows: a full prompt copy per row
    eng.alloc_kv(R, POS + 64)
    eng.kv.normal_(0, 0.5)
    g_rows = graph_of(lambda: eng.decode_step(R), reset)
    rows_kv = eng.kv
    # grouped: one prefix per image + each row's own positions
    st = eng.group_buffers(B, n, P, T, MAX_NEW)
    st["prefix"].normal_(0, 0.5); st["row"].normal_(0, 0.5)
    g_grp = graph_of(lambda: eng.decode_step(R, group=st), reset)
    ts = {"rows": [], "grouped": []}
    for it in range(reps + 3):                 # alternate the arms; the first 3 rounds warm up
        for k, g in (("rows", g_rows), ("grouped", g_grp)):
            t = timed(g, reset)
            if it >= 3:
                ts[k].append(t)
    res = {f"{k}_step_ms": round(med(v), 4) for k, v in ts.items()}
    # the attention alone: 32 launches, one per layer, in a graph
    sp = eng._decode_splits()
    ws = d["ws"][: sp["qkv"] * 3 * cfg.llm_hidden * R].view(sp["qkv"], R, 3 * cfg.llm_hidden)

    def attn_grp():
        for i in range(cfg.llm_layers):
            G.decode_rope_attention_grouped(ws, st["prefix"][i, 0], st["prefix"][i, 1], st["row"][i, 0], st["row"][i, 1], d["pos"],
                                            eng.rope_cos, eng.rope_sin, cfg.head_dim ** -0.5, d["a"], n)

    def attn_rows():
        for i in range(cfg.llm_layers):
            G.decode_rope_attention(ws, rows_kv[i, 0], rows_kv[i, 1], d["kv_len"], d["pos"], eng.rope_cos, eng.rope_sin,
                                    cfg.head_dim ** -0.5, d["a"])
    g_ag, g_ar = graph_of(attn_grp, reset), graph_of(attn_rows, reset)
    ta = {"grouped": [], "rows": []}
    for it in range(reps + 3):
        for k, g in (("grouped", g_ag), ("rows", g_ar)):
            t = timed(g, reset)
            if it >= 3:
                ta[k].append(t)
    t_ag, t_ar = med(ta["grouped"]), med(ta["rows"])
    b_grp = B * P * HALF_MIB + R * (POS - P + 1) * HALF_MIB
    b_rows = R * (POS + 1) * HALF_MIB
    res.update(grouped_attn_ms=round(t_ag, 4), grouped_attn_gb=round(b_grp / 1e9, 3), grouped_attn_tbs=round(b_grp / t_ag / 1e9, 3),
               rows_attn_ms=round(t_ar, 4), rows_attn_gb=round(b_rows / 1e9, 3), rows_attn_tbs=round(b_rows / t_ar / 1e9, 3))
    results[f"B={B},n={n}"] = res
    print(f"B={B} n={n}: step {res['rows_step_ms']} ms as repeated-image rows -> {res['grouped_step_ms']} ms grouped; attention "
          f"{t_ar:.3f} ms ({b_rows / 1e9:.2f} GB, {b_rows / t_ar / 1e9:.2f} TB/s) -> {t_ag:.3f} ms ({b_grp / 1e9:.2f} GB, "
          f"{b_grp / t_ag / 1e9:.2f} TB/s)", flush=True)
    del g_rows, g_grp, g_ag, g_ar, rows_kv
    eng.drop_kv(); eng.drop_group(); torch.cuda.empty_cache()

# ---------------- end to end: one image, 16 questions, 10 new tokens
N_Q, N_TEXT, NEW = 16, 500, 10
g = torch.Generator().manual_seed(7)
image = torch.randn(1, 3, cfg.image_size, cfg.image_size, generator=g).cuda()


def questions(nq):
    base = torch.randint(1000, cfg.vocab, (N_TEXT,), generator=g)
    base[4] = tok.map["<image>"]
    base[N_TEXT // 2] = tok.map["<region>"]
    ids = base.repeat(nq, 1)
    ids[:, -8:] = torch.randint(1000, cfg.vocab, (nq, 8), generator=g)
    return ids.cuda()


ids16 = questions(N_Q)


def call(ids, images):
    model.profile = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.generate(ids.clone(), images=images, max_new_tokens=NEW, eos_token_id=[])
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    marks = dict(model.profile)
    model.profile = None
    return wall, marks["assemble+embed"].elapsed_time(marks["llm_prefill"])


ways = {"16 batch-1 calls": lambda: (sum(call(ids16[i:i + 1], image)[0] for i in range(N_Q)), None),
        "repeated-image batch": lambda: call(ids16, image.repeat(N_Q, 1, 1, 1)),
        "grouped": lambda: call(ids16, image)}
e2e = {k: [] for k in ways}
pre = {k: [] for k in ways}
for k, fn in ways.items():                   # one block per way after a warm-up call: steady state keeps its decode graph
    fn()
    for _ in range(max(3, reps // 4)):
        wall, prefill = fn()
        e2e[k].append(wall)
        if prefill is not None:
            pre[k].append(prefill)
T16 = model._last["ids"].shape[1]
end_to_end = {k: dict(call_ms=round(med(v), 2), llm_prefill_ms=round(med(pre[k]), 2) if pre[k] else None) for k, v in e2e.items()}
for k, v in end_to_end.items():
    print(f"end to end, 1 image x {N_Q} questions, {NEW} new tokens, ctx {T16}: {k}: {v['call_ms']} ms"
          + (f" (LLaMA prefill {v['llm_prefill_ms']} ms)" if v["llm_prefill_ms"] is not None else ""), flush=True)

# ---------------- the grouped prefill's staging copies alone, and the grouped prefill at n = 64
staging = {}
for nq in (16, 64):
    ids = ids16 if nq == N_Q else questions(nq)
    pf = [call(ids, image)[1] for _ in range(3)][1:]
    st = eng._group
    Pq, Tq, R = st["P"], model._last["ids"].shape[1], nq
    stage = torch.empty((2, R, cfg.llm_heads, Tq, cfg.head_dim), dtype=torch.bfloat16, device="cuda")

    def copies():
        for i in range(cfg.llm_layers):
            stage.view(2, 1, R, cfg.llm_heads, Tq, cfg.head_dim)[:, :, :, :, :Pq].copy_(st["prefix"][i].unsqueeze(2))
            st["row"][i][:, :, :, :Tq - Pq].copy_(stage[:, :, :, Pq:])
    copies()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); copies(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    pos_bytes = 2 * cfg.llm_heads * cfg.head_dim * 2           # K and V of one position of one layer
    moved = cfg.llm_layers * pos_bytes * (Pq + R * Pq + 2 * R * (Tq - Pq))   # prefix read once, broadcast written, suffix copied
    staging[f"n={nq}"] = dict(ctx=Tq, prefix=Pq, grouped_llm_prefill_ms=round(med(pf), 2), staging_copies_ms=round(med(ts), 3),
                              staging_gb_moved=round(moved / 1e9, 2))
    print(f"grouped prefill, 1 image x {nq} questions, ctx {Tq}, P {Pq}: LLaMA prefill {med(pf):.2f} ms, of which staging copies "
          f"{med(ts):.3f} ms ({moved / 1e9:.2f} GB read + written)", flush=True)
    eng.drop_group(); torch.cuda.empty_cache()
    del stage
print(json.dumps(dict(card=card, ctx=T, prefix=P, gen_index=S_GEN, reps=reps, results=results, end_to_end=end_to_end,
                      staging=staging)))
