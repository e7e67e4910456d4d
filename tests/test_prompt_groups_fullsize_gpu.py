"""generate() with 16 prompts on one image at Groma-7B dimensions (H = 32, 100 regions, ctx ~1000, V = 32 114), against the same
16 rows run on 16 copies of the image, with the floor-relative bars of tests/fullsize.py: the floor is the distance between the
'bf16' and 'fp32' oracles' last-position logits of the first prompt.  This runs the grouped prefill at full size (the prefix pass
on the 2-CTA projections with the fused qkv + RoPE epilogue, the suffix pass at pos0 = P into the staging buffer, attention_tc
with q_pos0 = P over the staged cache) and the grouped decode attention inside the 32-layer CUDA-graph step."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_fullsize_prompt_groups_against_repeated_images():
    from groma.model.groma import GromaConfig, GromaModel
    from groma_b200.config import PathConfig, SyntheticTokenizer
    from groma_b200.synth import make_state_dict
    from oracle.groma_oracle import Oracle
    from tests.fullsize import BARS, make_inputs, nrel, widen_state_dict
    free, total = torch.cuda.mem_get_info()
    if total < 60 << 30:
        pytest.skip("needs a >= 60 GB GPU for the Groma-7B-shaped weights")
    n, n_new, n_text = 16, 8, 540
    cfg = PathConfig(box_score_thres=0.0)
    tok = SyntheticTokenizer(cfg.vocab)
    sd = make_state_dict(cfg, seed=0, perturb_norms=True, dtype=torch.bfloat16, device="cuda")
    model = GromaModel(GromaConfig.from_path_config(cfg), state_dict=sd, path_config=cfg)
    model.init_special_token_id(tok)
    sd_f32 = widen_state_dict(sd)
    del sd
    torch.cuda.empty_cache()
    images, ids1 = make_inputs(cfg, tok, n_text)
    g = torch.Generator().manual_seed(11)
    ids = ids1.repeat(n, 1)
    ids[:, -8:] = torch.randint(1000, cfg.vocab, (n, 8), generator=g)    # 16 questions after a shared 532-token text
    ids[0] = ids1[0]
    boxes = [torch.rand(cfg.max_region_num, 4, generator=g) * 0.6 + 0.2]
    L0 = ids.shape[1]
    kw = dict(max_new_tokens=n_new, eos_token_id=[], _keep_logits=True)
    ref = model.generate(ids.clone().cuda(), images=images.cuda().repeat_interleave(n, 0), _selected_override=boxes * n, **kw).cpu()
    ref_logits = [x.float().cpu() for x in model._step_logits]
    T = model._last["ids"].shape[1]
    got = model.generate(ids.clone().cuda(), images=images.cuda(), _selected_override=boxes, **kw).cpu()
    got_logits = [x.float().cpu() for x in model._step_logits]
    P = model.engine._group["P"]
    print(f"[fullsize groups] T={T} P={P}", flush=True)
    assert 900 <= T and T - P <= 16

    # the floor: bf16 vs fp32 oracle on the first prompt's prefill
    last = {}
    for prec in ("bf16", "fp32"):
        o = Oracle(cfg, sd_f32, prec, prerounded=True)
        o.init_special_token_id(tok)
        last[prec] = o.forward_prefill(ids[:1].clone(), images, selected_override=boxes)["logits"][:, -1].float()
        print(f"[fullsize groups] {prec} oracle prefill done", flush=True)
        del o
    floor = nrel(last["fp32"], last["bf16"])
    lim = BARS["floor_factor"] * floor + BARS["eps"]
    # the repeated-row run itself sits inside the bar of the bf16 oracle (what makes it the yardstick)
    d_ref = nrel(ref_logits[0][:1], last["bf16"])
    # first-token logits of every row, then each decode step's logits up to the first token difference
    d_first = max(nrel(got_logits[0][r], ref_logits[0][r]) for r in range(n))
    new_g, new_r = got[:, L0:], ref[:, L0:]
    steps = min(new_g.shape[1], new_r.shape[1])
    d_steps, first_diff = [], None
    for s in range(steps):
        d_steps.append(max(nrel(got_logits[s][r], ref_logits[s][r]) for r in range(n)))
        diff = (new_g[:, s] != new_r[:, s]).nonzero().flatten().tolist()
        if diff:
            first_diff = (s, diff)
            break
    print(f"[fullsize groups] floor {floor:.3e}, limit {lim:.3e}; repeated rows vs bf16 oracle {d_ref:.3e}; grouped vs repeated: "
          f"first token {d_first:.3e}, steps {[f'{x:.2e}' for x in d_steps]}, first token difference {first_diff}", flush=True)
    assert d_ref <= lim
    assert d_first <= lim and max(d_steps) <= lim
    if first_diff is not None:             # a two-sided near-tie inside the limit, in units of max |logit| of the step
        s, rows = first_diff
        for r in rows:
            tg, tr = int(new_g[r, s]), int(new_r[r, s])
            for lg, mine, other in ((got_logits[s][r], tg, tr), (ref_logits[s][r], tr, tg)):
                assert float(lg[mine] - lg[other]) / float(lg.abs().max()) <= lim, (s, r, tg, tr)
