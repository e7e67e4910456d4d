"""`groma.model.groma` surface: GromaConfig / GromaModel with the reference's forward / generate contract
(reference groma/model/groma.py:31-431), executed by the H100-native engine.

Kept from the reference (SURVEY.md section 8b): constructor + from_pretrained, init_special_token_id and the token-id
attributes, mutable config.{nms_thres, box_score_thres, max_region_num}, forward(...) -> CausalLMOutputWithPast with
hidden_states=(llm_hidden_states, vis_outputs), tuple-of-tuples past_key_values [B,32,ctx,128], in-place edit of the
caller's input_ids for <refer_box>/<ground_box> placeholders (T8), torch.randperm on the global CPU RNG (T6), the
all-ones decode mask (T7), generate(...).sequences / .hidden_states[0][-1].  There is no CPU path: construction fails
without a CUDA device."""
from __future__ import annotations

import copy
import glob
import json
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from transformers import AutoConfig, AutoModel, LlamaConfig, PretrainedConfig
from transformers.modeling_outputs import CausalLMOutputWithPast

from groma.constants import IGNORE_INDEX
from groma.model.ddetr import CustomDDETRConfig, CustomDDETRModel, perceiver_fields
from groma_b200 import ops as G
from groma_b200.config import PathConfig
from groma_b200.engine import GromaEngine


class GromaConfig(PretrainedConfig):
    model_type = "groma"

    def __init__(self, llm_cfg=None, perceiver_cfg=None, num_new_token=0, nms_thres=0.6, box_score_thres=0.15,
                 max_region_num=100, **kwargs):
        super().__init__(**kwargs)
        if perceiver_cfg is None:
            self.perceiver_cfg = CustomDDETRConfig()
        elif isinstance(perceiver_cfg, dict):
            self.perceiver_cfg = CustomDDETRConfig(**perceiver_cfg)
        elif isinstance(perceiver_cfg, CustomDDETRConfig):
            self.perceiver_cfg = perceiver_cfg
        else:
            raise NotImplementedError("currently only supports CustomDDETR as perceiver.")
        if llm_cfg is None:
            self.llm_cfg = LlamaConfig()
        elif isinstance(llm_cfg, dict):
            self.llm_cfg = LlamaConfig(**llm_cfg)
        elif isinstance(llm_cfg, LlamaConfig):
            self.llm_cfg = llm_cfg
        else:
            raise NotImplementedError("currently only supports LlamaModel as LLM.")
        self.nms_thres = nms_thres
        self.box_score_thres = box_score_thres
        self.max_region_num = max_region_num
        self.num_new_token = num_new_token
        self.vocab_size = self.llm_cfg.vocab_size + num_new_token

    def to_json_string(self, use_diff: bool = True) -> str:
        d = copy.deepcopy(self)
        if use_diff:
            d.perceiver_cfg = json.loads(d.perceiver_cfg.to_json_string(True))
            d.llm_cfg = d.llm_cfg.to_diff_dict()
            d = d.to_diff_dict()
        else:
            d.perceiver_cfg = json.loads(d.perceiver_cfg.to_json_string(False))
            d.llm_cfg = d.llm_cfg.to_dict()
            d = d.to_dict()
        return json.dumps(d, indent=2, sort_keys=True, default=str) + "\n"

    def to_path_config(self, image_size: int = 448, **overrides) -> PathConfig:
        l = self.llm_cfg
        f = perceiver_fields(self.perceiver_cfg)
        f.update(image_size=image_size, llm_hidden=l.hidden_size, llm_layers=l.num_hidden_layers, llm_heads=l.num_attention_heads,
                 llm_inter=l.intermediate_size, vocab=l.vocab_size, num_new_token=self.num_new_token, rms_eps=l.rms_norm_eps,
                 rope_theta=_rope_theta(l),
                 max_pos=l.max_position_embeddings, nms_thres=self.nms_thres, box_score_thres=self.box_score_thres,
                 max_region_num=self.max_region_num)
        if l.num_key_value_heads not in (None, l.num_attention_heads):
            raise NotImplementedError("Vicuna-7B is MHA; GQA is not on the path")
        f.update(overrides)
        return PathConfig(**f)

    @classmethod
    def from_path_config(cls, p: PathConfig) -> "GromaConfig":
        from transformers import Dinov2Config
        vis = Dinov2Config(hidden_size=p.vit_hidden, num_hidden_layers=p.vit_layers, num_attention_heads=p.vit_heads,
                           mlp_ratio=p.vit_mlp // p.vit_hidden, image_size=p.vit_pos_grid * p.patch, patch_size=p.patch,
                           layer_norm_eps=p.vit_ln_eps)
        det = _ddetr_cfg(p)
        llm = LlamaConfig(hidden_size=p.llm_hidden, num_hidden_layers=p.llm_layers, num_attention_heads=p.llm_heads,
                          num_key_value_heads=p.llm_heads, intermediate_size=p.llm_inter, vocab_size=p.vocab,
                          rms_norm_eps=p.rms_eps, max_position_embeddings=p.max_pos)
        return cls(llm_cfg=llm, perceiver_cfg=CustomDDETRConfig(vis_encoder_cfg=vis, ddetr_cfg=det), num_new_token=p.num_new_token,
                   nms_thres=p.nms_thres, box_score_thres=p.box_score_thres, max_region_num=p.max_region_num)


def _rope_theta(l) -> float:
    rt = getattr(l, "rope_theta", None)
    if rt is None:
        rt = (getattr(l, "rope_parameters", None) or {}).get("rope_theta", 10000.0)
    return float(rt)


def _ddetr_cfg(p: PathConfig):
    from transformers import DeformableDetrConfig
    kw = dict(d_model=p.d_model, encoder_layers=p.enc_layers, decoder_layers=p.dec_layers,
              encoder_attention_heads=p.ddetr_heads, decoder_attention_heads=p.ddetr_heads, encoder_n_points=p.n_points,
              decoder_n_points=p.n_points, encoder_ffn_dim=p.ddetr_ffn, decoder_ffn_dim=p.ddetr_ffn, num_queries=p.num_queries,
              two_stage_num_proposals=p.num_queries, num_feature_levels=1, two_stage=True, with_box_refine=True)
    try:
        return DeformableDetrConfig(use_timm_backbone=False, use_pretrained_backbone=False, **kw)
    except Exception:
        return DeformableDetrConfig(**kw)


@dataclass
class GenerateOutput:
    sequences: torch.Tensor
    hidden_states: Tuple
    past_key_values: Optional[Tuple] = None
    sequences_scores: Optional[torch.Tensor] = None     # beam search only: fp32 [B * num_return_sequences]


def _load_generation_config(path: Optional[str], config: "GromaConfig"):
    """`model.generation_config` as the reference's checkpoints carry it: train.py:108-112 stores the tokenizer's
    eos / pad / bos ids in `generation_config.json`, and every eval script passes it back to generate()
    (eval/run_groma.py:92).  Falls back to the ids in config.json (top level, then llm_cfg) when the file is absent."""
    from transformers import GenerationConfig
    if path is not None and os.path.isfile(os.path.join(path, "generation_config.json")):
        return GenerationConfig.from_pretrained(path)
    l = config.llm_cfg

    def pick(name):
        v = config.__dict__.get(name)
        return v if v is not None else getattr(l, name, None)
    return GenerationConfig(eos_token_id=pick("eos_token_id"), pad_token_id=pick("pad_token_id"), bos_token_id=pick("bos_token_id"))


def _eos_list(eos) -> List[int]:
    if eos is None:
        return []
    if isinstance(eos, torch.Tensor):
        return [int(v) for v in eos.reshape(-1).tolist()]
    if isinstance(eos, (list, tuple)):
        return [int(v) for v in eos]
    return [int(eos)]


_SAMPLING_DEFAULTS = dict(temperature=1.0, top_k=50, top_p=1.0)   # GenerationConfig() defaults of transformers 4.32


def resolve_sampling_params(generation_config=None, temperature=None, top_k=None, top_p=None) -> Tuple[float, int, float]:
    """(temperature, top_k, top_p) of a do_sample=True generate() call, as HF 4.32 `sample()` builds its warpers: an explicit
    argument wins, then the generation_config's value, then the 4.32 default (transformers 5.x leaves these None in
    GenerationConfig()).  top_k = 0 and top_p = 1.0 switch that warper off.  Raises ValueError where the 4.32 warpers do:
    temperature must be > 0, top_k a non-negative int, top_p in [0, 1]."""
    vals = {}
    for name, arg in (("temperature", temperature), ("top_k", top_k), ("top_p", top_p)):
        v = arg if arg is not None else getattr(generation_config, name, None)
        vals[name] = v if v is not None else _SAMPLING_DEFAULTS[name]
    t, k, p = vals["temperature"], vals["top_k"], vals["top_p"]
    if isinstance(t, bool) or not isinstance(t, (int, float)) or not t > 0:
        raise ValueError(f"`temperature` (={t}) has to be a strictly positive float")
    if isinstance(k, bool) or not isinstance(k, int) or k < 0:
        raise ValueError(f"`top_k` has to be a non-negative integer, but is {k}")
    if isinstance(p, bool) or not isinstance(p, (int, float)) or not 0.0 <= p <= 1.0:
        raise ValueError(f"`top_p` has to be a float >= 0 and <= 1, but is {p}")
    return float(t), int(k), float(p)


# GenerationConfig() defaults of transformers 4.32 (5.x leaves them None); each one switches its processor off
_PROCESSING_DEFAULTS = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, bad_words_ids=None, min_length=0, min_new_tokens=None,
                            suppress_tokens=None, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)


def resolve_processing_params(generation_config=None, eos_ids: Sequence[int] = (), vocab_size: int = 0, sampling: bool = False,
                              **knobs) -> Optional[dict]:
    """generate()'s logits processors and extra warpers as HF 4.32 `_get_logits_processor` / `_get_logits_warper` build them.
    Each knob (the keys of _PROCESSING_DEFAULTS) resolves like resolve_sampling_params: explicit argument, then the
    generation_config's value, then the 4.32 default.  A processor is on under 4.32's condition and raises ValueError where
    its 4.32 constructor does; typical / epsilon / eta only count with sampling.  Returns None when nothing is on, else a
    dict with the fields of ops.process_params (eos / ban / seqs lists) and of the extra warpers.  Deviations: a bad-words or
    suppress id outside the vocabulary raises ValueError here, before any work (4.32 raises at the first step; a suppress id
    in [-V, 0) indexes from the end, as 4.32's `scores[:, ids]` does), and an empty bad-words entry raises ValueError (4.32
    fails with IndexError at the first step)."""
    v = {}
    for name, default in _PROCESSING_DEFAULTS.items():
        a = knobs.get(name)
        a = a if a is not None else getattr(generation_config, name, None)
        v[name] = a if a is not None else default
    eos = [int(e) for e in eos_ids]
    out = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_length=0, min_new_tokens=0, eos=[], ban=[], seqs=[],
               bad_words=False, typical_p=1.0, epsilon_cutoff=0.0, eta_cutoff=0.0)
    on = False
    rp = v["repetition_penalty"]
    if rp != 1.0:
        if not isinstance(rp, float) or not rp > 0:
            raise ValueError(f"`penalty` has to be a strictly positive float, but is {rp}")
        out["repetition_penalty"], on = rp, True
    n = v["no_repeat_ngram_size"]
    if n > 0:
        if not isinstance(n, int) or n <= 0:
            raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {n}")
        out["no_repeat_ngram_size"], on = int(n), True
    bw = v["bad_words_ids"]
    if bw is not None:
        if not isinstance(bw, list) or len(bw) == 0:
            raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bw}.")
        if any(not isinstance(w, list) for w in bw):
            raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bw}.")
        if any(any(not isinstance(t, (int, np.integer)) or t < 0 for t in w) for w in bw):
            raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bw}.")
        if any(len(w) == 0 for w in bw):
            raise ValueError(f"`bad_words_ids` cannot hold an empty list: {bw}")
        bad = [t for w in bw for t in w if t >= vocab_size]
        if bad:
            raise ValueError(f"The model vocabulary size is {vocab_size}, but the following tokens were being biased: {bad}")
        for w in dict.fromkeys(tuple(int(t) for t in w) for w in bw if all(w != [e] for e in eos)):
            (out["ban"].append(w[0]) if len(w) == 1 else out["seqs"].append(list(w)))
        out["bad_words"] = on = True
    if eos:
        ml, mn = v["min_length"], v["min_new_tokens"]
        if ml > 0:
            if not isinstance(ml, int) or ml < 0:
                raise ValueError(f"`min_length` has to be a non-negative integer, but is {ml}")
            out["min_length"], out["eos"], on = int(ml), eos, True
        if mn is not None and mn > 0:
            if not isinstance(mn, int) or mn < 0:
                raise ValueError(f"`min_new_tokens` has to be a positive integer, but is {mn}")
            out["min_new_tokens"], out["eos"], on = int(mn), eos, True
    st = v["suppress_tokens"]
    if st is not None:
        for t in list(st):
            t = int(t)
            if not -vocab_size <= t < vocab_size:
                raise ValueError(f"suppress_tokens id {t} is outside the vocabulary of size {vocab_size}")
            out["ban"].append(t % vocab_size)
        on = True
    if sampling:
        tp = v["typical_p"]
        if tp < 1.0:
            if not float(tp) > 0:
                raise ValueError(f"`typical_p` has to be a float > 0 and < 1, but is {float(tp)}")
            out["typical_p"], on = float(tp), True
        for name in ("epsilon_cutoff", "eta_cutoff"):
            if 0.0 < v[name] < 1.0:
                out[name], on = float(v[name]), True
    return out if on else None


_BEAM_DEFAULTS = dict(length_penalty=1.0, early_stopping=False, num_return_sequences=1)   # GenerationConfig() of 4.32


def resolve_beam_params(generation_config=None, num_beams=None, length_penalty=None, early_stopping=None, num_return_sequences=None,
                        batch_size: int = 1, do_sample: bool = False, kv_cache_dtype=torch.bfloat16, eos_ids: Sequence[int] = (),
                        **kwargs) -> Optional[dict]:
    """Beam search of a generate() call, as HF 4.32 `beam_search` + `BeamSearchScorer` run it (oracle/beam_search.py).  None
    unless num_beams > 1 is passed explicitly: generation_config.num_beams alone keeps greedy search, as do_sample does.
    length_penalty, early_stopping and num_return_sequences resolve like the sampling knobs (argument, generation_config,
    4.32 default).  kwargs: num_beam_groups, diversity_penalty, constraints, force_words_ids (refused).  Raises ValueError for
    out-of-range values, more than ops.BEAM_MAX_BEAMS beams, batch_size * num_beams above ops.BEAM_MAX_ROWS, more than
    ops.BEAM_MAX_EOS EOS ids, and with an fp8 KV cache; NotImplementedError for beam sampling, group / diverse and constrained beam search."""
    nb = num_beams
    if nb is None:
        return None
    if isinstance(nb, bool) or not isinstance(nb, (int, np.integer)) or nb < 1:
        raise ValueError(f"`num_beams` has to be an integer >= 1, but is {nb}")
    nb = int(nb)
    if nb == 1:
        return None
    gc = generation_config
    if do_sample is True:
        raise NotImplementedError("num_beams > 1 with do_sample=True (beam_sample) is not implemented; supported: beam search "
                                  "(do_sample=False), or do_sample=True with num_beams=1")
    ng = kwargs.get("num_beam_groups") if kwargs.get("num_beam_groups") is not None else getattr(gc, "num_beam_groups", None)
    dp = kwargs.get("diversity_penalty") if kwargs.get("diversity_penalty") is not None else getattr(gc, "diversity_penalty", None)
    if (ng is not None and ng > 1) or (dp is not None and dp != 0.0):
        raise NotImplementedError("group / diverse beam search (num_beam_groups > 1, diversity_penalty) is not implemented; "
                                  "supported: beam search with num_beam_groups=1")
    fw = kwargs.get("force_words_ids") if kwargs.get("force_words_ids") is not None else getattr(gc, "force_words_ids", None)
    if kwargs.get("constraints") is not None or fw is not None:
        raise NotImplementedError("constrained beam search (constraints, force_words_ids) is not implemented; supported: beam "
                                  "search without constraints")
    if nb > G.BEAM_MAX_BEAMS:
        raise ValueError(f"num_beams={nb} exceeds the beam decode attention's limit of {G.BEAM_MAX_BEAMS} beams per image")
    if batch_size * nb > G.BEAM_MAX_ROWS:
        raise ValueError(f"batch size x num_beams = {batch_size} x {nb} exceeds the {G.BEAM_MAX_ROWS} rows of the decode GEMMs")
    if len(eos_ids) > G.BEAM_MAX_EOS:
        raise ValueError(f"beam search takes at most {G.BEAM_MAX_EOS} EOS ids, got {len(eos_ids)}")
    if kv_cache_dtype == torch.float8_e4m3fn:
        raise ValueError("beam search needs a bf16 KV cache: the fp8 cache's scales are aligned to 4-key groups, which a per-key "
                         "ancestry breaks; set model.kv_cache_dtype = torch.bfloat16")
    vals = {}
    for name, arg in (("length_penalty", length_penalty), ("early_stopping", early_stopping),
                      ("num_return_sequences", num_return_sequences)):
        v = arg if arg is not None else getattr(gc, name, None)
        vals[name] = v if v is not None else _BEAM_DEFAULTS[name]
    lp, es, nrs = vals["length_penalty"], vals["early_stopping"], vals["num_return_sequences"]
    if isinstance(lp, bool) or not isinstance(lp, (int, float)) or not np.isfinite(lp):
        raise ValueError(f"`length_penalty` has to be a finite float, but is {lp}")
    if not (es is True or es is False or es == "never"):
        raise ValueError(f"`early_stopping` has to be True, False or 'never', but is {es!r}")
    if isinstance(nrs, bool) or not isinstance(nrs, (int, np.integer)) or nrs < 1:
        raise ValueError(f"`num_return_sequences` has to be a positive integer, but is {nrs}")
    if nrs > nb:
        raise ValueError("`num_return_sequences` has to be smaller or equal to `num_beams`.")
    return dict(num_beams=nb, length_penalty=float(lp), early_stopping=es, num_return_sequences=int(nrs))


def beam_denominators(length_penalty: float, max_length: int) -> torch.Tensor:
    """float64 [max_length + 1]: n ** length_penalty as 4.32's BeamHypotheses computes it (a Python int to a float power)."""
    return torch.tensor([float(n) ** float(length_penalty) if n > 0 else 1.0 for n in range(max_length + 1)], dtype=torch.float64)


def resolve_prompt_groups(rows: int, n_images: int, refer_boxes=None, ground_boxes=None, kv_cache_dtype=torch.bfloat16,
                          num_beams=None) -> int:
    """n, the prompts per image of a generate(input_ids [rows, L], images [n_images, ...]) call: rows b*n .. b*n + n - 1 ask
    about image b, whose vision stage, region selection and shared prompt prefix run once (DESIGN.md section 4).  1 when
    rows == n_images (the plain call).  Raises ValueError when rows is not a multiple of n_images, and for n > 1 with refer /
    ground boxes (they change the region set per row), with an fp8 KV cache, with n > ops.GROUP_MAX_PROMPTS or with rows above
    ops.BEAM_MAX_ROWS; NotImplementedError for num_beams > 1 with n > 1."""
    if n_images < 1 or rows % n_images != 0:
        raise ValueError(f"input_ids has {rows} rows, which is not a multiple of the {n_images} images: the rows b*n .. b*n+n-1 "
                         "of a grouped generate() ask about image b")
    n = rows // n_images
    if n == 1:
        return 1
    if num_beams is not None and not isinstance(num_beams, bool) and isinstance(num_beams, (int, np.integer)) and num_beams > 1:
        raise NotImplementedError("num_beams > 1 with several prompts per image is not implemented; pass one row per image")
    if refer_boxes is not None or ground_boxes is not None:
        raise ValueError("refer_boxes / ground_boxes cannot be combined with several prompts per image: they change the region "
                         "set of each row, so the rows share nothing; pass one row per image")
    if kv_cache_dtype == torch.float8_e4m3fn:
        raise ValueError("several prompts per image need a bf16 KV cache; set model.kv_cache_dtype = torch.bfloat16")
    if n > G.GROUP_MAX_PROMPTS:
        raise ValueError(f"{n} prompts per image exceed the grouped decode attention's limit of {G.GROUP_MAX_PROMPTS}")
    if rows > G.BEAM_MAX_ROWS:
        raise ValueError(f"{rows} rows exceed the {G.BEAM_MAX_ROWS} rows of the decode GEMMs")
    return n


def rows_of_images(per_image: Sequence, n: int) -> list:
    """Row i of a grouped call takes image i // n's entry."""
    return [x for x in per_image for _ in range(n)]


def shared_prefix_len(ids: torch.Tensor, n: int) -> int:
    """P of a grouped generate(): over the assembled rows ids [B*n, T] (rows of an image consecutive), the minimum over images of
    the longest common prefix of that image's n rows, capped at T - 1 so that every row keeps at least one position of its
    own (the one whose logits give its first token)."""
    R, T = ids.shape
    g = ids.reshape(R // n, n, T)
    agree = (g == g[:, :1]).all(1).all(0)
    return min(int(agree.long().cumprod(0).sum()), T - 1)


def _c2c(b: torch.Tensor) -> torch.Tensor:
    return torch.cat([b[:, :2] - 0.5 * b[:, 2:], b[:, :2] + 0.5 * b[:, 2:]], -1)


def _box_iou(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    area_a = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = torch.max(a[:, None, :2], b[None, :, :2])
    rb = torch.min(a[:, None, 2:], b[None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (area_a[:, None] + area_b[None, :] - inter)


NF4_CONFIG = dict(load_in_4bit=True, bnb_4bit_quant_type="nf4", bnb_4bit_use_double_quant=False)
_NF4_HINT = ("supported: BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type='nf4', bnb_4bit_use_double_quant=False) "
             "(blocks of 64, any bnb_4bit_compute_dtype: the arithmetic is bf16 with fp32 accumulation)")


def resolve_quantization_config(load_in_8bit: bool = False, load_in_4bit: bool = False, quantization_config=None):
    """The quantization arguments of from_pretrained (transformers 4.32 names).  Returns the accepted config (recorded as
    config.quantization_config) or None for bf16; raises NotImplementedError, naming the supported config, for everything
    else: LLM.int8 (8-bit), FP4 -- also what a bare load_in_4bit=True means, HF's default quant type -- and double quant."""
    qc = quantization_config
    if qc is None:
        if load_in_8bit:
            raise NotImplementedError("load_in_8bit (LLM.int8 outlier decomposition) is not implemented; " + _NF4_HINT)
        if load_in_4bit:
            raise NotImplementedError("load_in_4bit=True without a quantization_config means bnb_4bit_quant_type='fp4' "
                                      "(the transformers default), which is not implemented; " + _NF4_HINT)
        return None
    get = (lambda k, d=None: qc.get(k, d)) if isinstance(qc, dict) else (lambda k, d=None: getattr(qc, k, d))
    if load_in_8bit or get("load_in_8bit", False):
        raise NotImplementedError("load_in_8bit (LLM.int8 outlier decomposition) is not implemented; " + _NF4_HINT)
    if not get("load_in_4bit", False):
        raise NotImplementedError("quantization_config without load_in_4bit=True is not implemented; " + _NF4_HINT)
    if get("bnb_4bit_quant_type", "fp4") != "nf4":
        raise NotImplementedError(f"bnb_4bit_quant_type={get('bnb_4bit_quant_type', 'fp4')!r} is not implemented; " + _NF4_HINT)
    if get("bnb_4bit_use_double_quant", False):
        raise NotImplementedError("bnb_4bit_use_double_quant=True (quantised absmax) is not implemented; " + _NF4_HINT)
    storage = get("bnb_4bit_quant_storage", None)
    if storage not in (None, torch.uint8, "uint8"):
        raise NotImplementedError(f"bnb_4bit_quant_storage={storage!r} is not implemented (codes are packed in uint8); " + _NF4_HINT)
    return qc


KV_CACHE_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


def resolve_kv_cache_dtype(kv_cache_dtype, head_dim: int = 128) -> torch.dtype:
    """The KV-cache storage of the LLaMA decode: torch.bfloat16 (the default, the reference's cache) or torch.float8_e4m3fn (e4m3
    codes + one fp32 scale per 128-element head vector, DESIGN.md section 4; it changes the decode numerics, like NF4 weights).
    Anything else raises ValueError, as does fp8 with a head dim other than 128 (the fp8 decode kernels' row)."""
    if not isinstance(kv_cache_dtype, torch.dtype) or kv_cache_dtype not in KV_CACHE_DTYPES:
        raise ValueError(f"kv_cache_dtype must be torch.bfloat16 or torch.float8_e4m3fn, got {kv_cache_dtype!r}")
    if kv_cache_dtype == torch.float8_e4m3fn and head_dim != 128:
        raise ValueError(f"an fp8 KV cache needs head_dim 128, the model has {head_dim}")
    return kv_cache_dtype


LLM_WEIGHT_DTYPES = (torch.bfloat16, torch.float8_e4m3fn)


def resolve_llm_weight_dtype(llm_weight_dtype, quantization_config=None) -> torch.dtype:
    """The storage of the LLaMA projections (32 x q/k/v/o/gate/up/down): torch.bfloat16 (the default, the reference's
    weights) or torch.float8_e4m3fn (e4m3 codes + one fp32 scale per weight row, with every GEMM input row quantised the same
    way at run time and multiplied on fp8 tensor cores, DESIGN.md section 4; it changes the numerics, like NF4).  Anything
    else raises ValueError, as does fp8 together with an NF4 quantization_config: a model has one weight format."""
    if not isinstance(llm_weight_dtype, torch.dtype) or llm_weight_dtype not in LLM_WEIGHT_DTYPES:
        raise ValueError(f"llm_weight_dtype must be torch.bfloat16 or torch.float8_e4m3fn, got {llm_weight_dtype!r}")
    if llm_weight_dtype == torch.float8_e4m3fn and quantization_config is not None:
        raise ValueError("llm_weight_dtype=torch.float8_e4m3fn cannot be combined with a 4-bit quantization_config: "
                         "a model has one weight format")
    return llm_weight_dtype


class GromaModel(torch.nn.Module):
    config_class = GromaConfig
    supports_gradient_checkpointing = False

    def __init__(self, config: GromaConfig, state_dict: Optional[Dict[str, torch.Tensor]] = None, image_size: int = 448,
                 path_config: Optional[PathConfig] = None, quantization_config=None, kv_cache_dtype: torch.dtype = torch.bfloat16,
                 llm_weight_dtype: torch.dtype = torch.bfloat16):
        """quantization_config: a BitsAndBytesConfig (or its dict) accepted by resolve_quantization_config -- quantise while
        packing, as from_pretrained(..., quantization_config=...) does.  kv_cache_dtype: see resolve_kv_cache_dtype and the
        kv_cache_dtype attribute.  llm_weight_dtype: see resolve_llm_weight_dtype; fixed for the model's lifetime."""
        super().__init__()
        if state_dict is None:
            raise ValueError("GromaModel needs weights: use GromaModel.from_pretrained(path) or pass state_dict=")
        qc = resolve_quantization_config(quantization_config=quantization_config)
        llm_weight_dtype = resolve_llm_weight_dtype(llm_weight_dtype, qc)
        self.config = config
        self._path_cfg = path_config if path_config is not None else config.to_path_config(image_size)
        kv_cache_dtype = resolve_kv_cache_dtype(kv_cache_dtype, self._path_cfg.head_dim)
        # a lazy checkpoint view (from_pretrained) holds file handles, not tensors: keep it so that quantize_nf4_() can re-read the
        # source weights.  An in-memory dict is never kept -- the caller may free it (bench.py does, for 14 GB of device weights)
        from groma_b200.checkpoint import ShardedStateDict
        self._source = state_dict if isinstance(state_dict, ShardedStateDict) else None
        self.engine = GromaEngine(self._path_cfg, state_dict, nf4=qc is not None, fp8=llm_weight_dtype == torch.float8_e4m3fn)
        self.engine.kv_dtype = kv_cache_dtype
        if qc is not None:
            self.config.quantization_config = qc
        self.perceiver = CustomDDETRModel(config.perceiver_cfg, engine=self.engine)
        self.generation_config = _load_generation_config(None, config)
        self.pad_token_id = None
        self.img_token_id = None
        self.reg_token_id = None
        self.refer_box_token_id = None
        self.refer_feat_token_id = None
        self.ground_box_token_id = None
        self.box_idx_token_ids = None
        self.use_cuda_graph = True
        self.kv_headroom = 64      # decode positions reserved by forward(use_cache=True) beyond the prompt (grows on demand)
        self._graph = None
        self.profile = None   # set to a list to collect (stage name, cuda event) marks during generate()

    @property
    def kv_cache_dtype(self) -> torch.dtype:
        """torch.bfloat16 (default) or torch.float8_e4m3fn.  Setting it drops the KV cache and any captured decode graph, so a
        forward(past_key_values=...) continuation has to start from a new prefill."""
        return self.engine.kv_dtype

    @kv_cache_dtype.setter
    def kv_cache_dtype(self, value):
        value = resolve_kv_cache_dtype(value, self._path_cfg.head_dim)
        self._graph = None
        self.engine.drop_kv()
        self.engine.kv_dtype = value

    @property
    def llm_weight_dtype(self) -> torch.dtype:
        """torch.bfloat16 (default) or torch.float8_e4m3fn: how the LLaMA projections are stored.  Read-only: another format
        needs the source weights, so build a new model."""
        return torch.float8_e4m3fn if self.engine.fp8 else torch.bfloat16

    def _mark(self, name: str):
        if self.profile is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.profile.append((name, ev))

    # ------------------------------------------------------------------ loading (SURVEY N4: HF checkpoint layout)
    @classmethod
    def from_pretrained(cls, path: str, *model_args, torch_dtype=None, config=None, **kwargs) -> "GromaModel":
        """`GromaModel.from_pretrained(dir)` (eval/run_groma.py:43-61) and `AutoModel.from_pretrained(dir)` (which resolves
        GromaConfig -> GromaModel through the registration at the bottom of this file and passes `config=`).  torch_dtype is
        accepted and ignored: the arithmetic type of the path is bf16 with fp32 accumulation (== the autocast region the
        reference's callers wrap generate() in)."""
        qc = resolve_quantization_config(kwargs.get("load_in_8bit", False), kwargs.get("load_in_4bit", False),
                                         kwargs.get("quantization_config"))
        llm_weight_dtype = resolve_llm_weight_dtype(kwargs.get("llm_weight_dtype", torch.bfloat16), qc)
        from groma_b200.checkpoint import ShardedStateDict, load_config_dict
        path = os.path.expanduser(str(path))
        cd = load_config_dict(path)
        cd.pop("model_type", None)
        if not isinstance(config, GromaConfig):
            config = GromaConfig(**cd)
        # lazy view over the (sharded) checkpoint: the engine packs tensor by tensor into its bf16 device arena
        view = ShardedStateDict(path)
        # region-encoder widths are code constants in the reference (roi_align.py:97-116,233-271), not config fields:
        # read them off the parameter shapes so any checkpoint of that architecture loads
        re_ = "region_encoder."
        geom = dict(region_mid=view.shape(re_ + "roi_align.flatten_linear.weight")[0],
                    pos_hidden=view.shape(re_ + "roi_align.pos_embedd.0.weight")[0],
                    fuse_rounds=sum(1 for k in view if k.startswith(re_ + "mlvl_fuse.fuse_convs.") and k.endswith(".conv.weight")))
        geom.update(cd.get("path_overrides") or {})     # e.g. {"gn_groups": 8} for miniature test checkpoints (reference: 64)
        model = cls(config, state_dict=view, path_config=config.to_path_config(**geom), quantization_config=qc,
                    kv_cache_dtype=kwargs.get("kv_cache_dtype", torch.bfloat16), llm_weight_dtype=llm_weight_dtype)
        model.generation_config = _load_generation_config(path, config)
        return model

    def quantize_nf4_(self, state_dict: Optional[Dict[str, torch.Tensor]] = None, quantization_config=None) -> "GromaModel":
        """Switch this model to 4-bit NF4 weights in place (what from_pretrained does with an nf4 BitsAndBytesConfig): the
        engine is re-packed from the source weights with every nn.Linear quantised (DESIGN.md section 4).  state_dict: the
        weights the model was built from; optional only for a model loaded by from_pretrained, which re-reads its checkpoint
        (the model keeps no reference to an in-memory dict).  Captured CUDA graphs are dropped.  quantization_config defaults
        to the supported nf4 config."""
        if self.engine.fp8:
            raise ValueError("this model has fp8 LLaMA weights (llm_weight_dtype): a model has one weight format")
        src = state_dict if state_dict is not None else self._source
        if src is None:
            raise ValueError("quantize_nf4_() needs the state dict this model was built from: model.quantize_nf4_(state_dict)")
        qc = resolve_quantization_config(quantization_config=quantization_config if quantization_config is not None else
                                         dict(NF4_CONFIG))
        self._graph = None
        kv_dtype = self.engine.kv_dtype
        self.engine = self.perceiver = None
        torch.cuda.empty_cache()
        self.engine = GromaEngine(self._path_cfg, src, nf4=True)
        self.engine.kv_dtype = kv_dtype
        self.perceiver = CustomDDETRModel(self.config.perceiver_cfg, engine=self.engine)
        self.config.quantization_config = qc
        return self

    def cuda(self, device=None):
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def init_special_token_id(self, tokenizer):
        from groma.constants import DEFAULT_TOKENS, REGION_IDX_TOKENS
        self.pad_token_id = tokenizer.pad_token_id
        self.img_token_id = tokenizer.convert_tokens_to_ids([DEFAULT_TOKENS["image"]])[0]
        self.reg_token_id = tokenizer.convert_tokens_to_ids([DEFAULT_TOKENS["region"]])[0]
        self.refer_box_token_id = tokenizer.convert_tokens_to_ids([DEFAULT_TOKENS["rbox"]])[0]
        self.refer_feat_token_id = tokenizer.convert_tokens_to_ids([DEFAULT_TOKENS["rfeat"]])[0]
        self.ground_box_token_id = tokenizer.convert_tokens_to_ids([DEFAULT_TOKENS["gbox"]])[0]
        self.box_idx_token_ids = tokenizer.convert_tokens_to_ids(REGION_IDX_TOKENS)

    def get_perceiver(self):
        return self.perceiver

    def get_llm(self):
        return None

    def prepare_inputs_for_generation(self, input_ids, past_key_values=None, attention_mask=None, inputs_embeds=None, **kwargs):
        if past_key_values:
            input_ids = input_ids[:, -1:]
        model_inputs = {"inputs_embeds": inputs_embeds} if (inputs_embeds is not None and past_key_values is None) else {"input_ids": input_ids}
        model_inputs.update({"past_key_values": past_key_values, "attention_mask": attention_mask, "use_cache": kwargs.get("use_cache"),
                             "images": kwargs.get("images"), "refer_boxes": kwargs.get("refer_boxes"), "ground_boxes": kwargs.get("ground_boxes")})
        return model_inputs

    # ------------------------------------------------------------------ host-side integer bookkeeping
    def _match(self, ids_h: torch.Tensor, labels_h, selected, refer_boxes, ground_boxes):
        """groma.py:283-309, on host copies; returns refer_box_inds."""
        refer_inds = []
        bidx = torch.tensor(self.box_idx_token_ids)
        for i in range(ids_h.shape[0]):
            if (ids_h[i] == self.refer_box_token_id).any():
                m = torch.max(_box_iou(_c2c(refer_boxes[i].float().cpu()), _c2c(selected[i])), dim=-1).indices
                refer_inds.append(m)
                ids_h[i].masked_scatter_(ids_h[i] == self.refer_box_token_id, bidx[m])
            else:
                refer_inds.append(torch.zeros(0, dtype=torch.long))
            if (ids_h[i] == self.ground_box_token_id).any():
                m = torch.max(_box_iou(_c2c(ground_boxes[i].float().cpu()), _c2c(selected[i])), dim=-1).indices
                mask = ids_h[i] == self.ground_box_token_id
                ids_h[i].masked_scatter_(mask, bidx[m])
                if labels_h is not None:
                    labels_h[i].masked_scatter_(mask, bidx[m])
        return refer_inds

    def _assemble(self, ids_h: torch.Tensor, labels_h, num_regions: List[int], n_img: int):
        """groma.py:317-357."""
        new_ids, new_labels = [], []
        for i in range(ids_h.shape[0]):
            ids = ids_h[i]
            ipos = (ids == self.img_token_id).nonzero(as_tuple=True)[0]
            rpos = (ids == self.reg_token_id).nonzero(as_tuple=True)[0]
            assert len(ipos) > 0 and len(rpos) > 0, "prompt needs one <image> and one <region> placeholder"
            ip, rp = int(ipos[0]), int(rpos[0])
            ppos = (ids == self.pad_token_id).nonzero(as_tuple=True)[0]
            pe = int(ppos[0]) if len(ppos) > 0 else len(ids)
            assert ip < rp
            regs = torch.tensor([v for j in range(num_regions[i]) for v in (self.box_idx_token_ids[j], self.reg_token_id)], dtype=torch.long)
            new_ids.append(torch.cat((ids[:ip], torch.full((n_img,), self.img_token_id, dtype=torch.long), ids[ip + 1:rp], regs, ids[rp + 1:pe])))
            if labels_h is not None:
                lb = labels_h[i]
                new_labels.append(torch.cat((lb[:ip], torch.full((n_img,), IGNORE_INDEX, dtype=torch.long), lb[ip + 1:rp],
                                             torch.full((2 * num_regions[i],), IGNORE_INDEX, dtype=torch.long), lb[rp + 1:pe])))
        ids_out = torch.nn.utils.rnn.pad_sequence(new_ids, batch_first=True, padding_value=self.pad_token_id)
        labels_out = torch.nn.utils.rnn.pad_sequence(new_labels, batch_first=True, padding_value=IGNORE_INDEX) if labels_h is not None else None
        return ids_out, labels_out

    # ------------------------------------------------------------------ vision + splice (groma.py:219-375)
    @torch.no_grad()
    def _prefill_inputs(self, input_ids, images, refer_boxes, ground_boxes, labels=None, selected_override=None, n: int = 1):
        """n > 1: rows b*n .. b*n + n - 1 of input_ids ask about image b (resolve_prompt_groups); the vision stage and the
        selection run per image, and each row is assembled with its image's image and region tokens."""
        eng, cfg = self.engine, self.config
        dev = eng.dev
        self._mark("start")
        # host copies of the ids / labels first (the GPU is idle here): reading them back later would wait for the whole vision stage
        ids_h0 = input_ids.detach().cpu()
        ids_h = ids_h0.clone()
        labels_h = labels.detach().cpu().clone() if labels is not None else None
        hs = eng.vit(images)
        self._mark("vit")
        img_tok = eng.image_tokens(hs[-1])
        n_extra = 0
        B = images.shape[0]
        if refer_boxes is not None or ground_boxes is not None:
            n_extra = max((len(refer_boxes[i]) if refer_boxes is not None else 0) + (len(ground_boxes[i]) if ground_boxes is not None else 0) for i in range(B))
        pc, px, sc, det_logits = eng.proposer(hs, n_extra)
        self._mark("proposer")
        # The fused maps of the region encoder do not depend on the selection: they are queued right behind the NMS read-back
        # copies, so the GPU works through them (~38 ms at B = 16) while the host waits for the keep lists, draws the
        # permutations, matches refer / ground boxes and builds the RoI list -- no idle gap at the one host sync of the vision stage.
        maps = {}

        def _queue_maps():
            maps["xs"] = eng.region_maps(hs)
        if selected_override is not None:
            selected = [b.float().cpu() for b in selected_override]
            _queue_maps()
        else:
            selected = eng.select_regions(pc, px, sc, refer_boxes, ground_boxes, cfg.nms_thres, cfg.box_score_thres, cfg.max_region_num,
                                          overlap=_queue_maps)
        sel_img = selected
        if n > 1:
            selected = rows_of_images(sel_img, n)
        refer_inds = self._match(ids_h, labels_h, selected, refer_boxes, ground_boxes)
        if not torch.equal(ids_h, ids_h0):
            input_ids.copy_(ids_h.to(input_ids.device))           # the reference edits the caller's tensor in place (T8)
            if labels is not None:
                labels.copy_(labels_h.to(labels.device))
        self._mark("select+maps")
        region = eng.region_tokens(maps["xs"], sel_img)
        self._mark("region_tokens")
        counts = [len(b) for b in selected]
        ids_new, labels_new = self._assemble(ids_h, labels_h, counts, img_tok.shape[1])
        Bn, T = ids_new.shape
        x = eng.embed(ids_new)
        flat = ids_new.reshape(-1)
        img_pos = (flat == self.img_token_id).nonzero(as_tuple=True)[0]
        reg_pos = (flat == self.reg_token_id).nonzero(as_tuple=True)[0]
        img_src, reg_src = img_tok.reshape(-1, x.shape[-1]), region
        if n > 1:
            # row i takes image i // n's tokens: gather the per-image rows into per-row order
            n_img = img_tok.shape[1]
            offs = np.cumsum([0] + [len(b) for b in sel_img])
            img_idx = torch.cat([torch.arange(n_img) + (i // n) * n_img for i in range(Bn)])
            reg_idx = torch.cat([torch.arange(offs[i // n], offs[i // n + 1]) for i in range(Bn)])
            img_src = G.gather_rows(img_idx.to(dev).contiguous(), img_src)
            reg_src = G.gather_rows(reg_idx.to(dev).contiguous(), region) if len(reg_idx) > 0 else region
        G.scatter_rows(img_pos.to(dev), img_src, x)
        if len(reg_pos) > 0:
            G.scatter_rows(reg_pos.to(dev), reg_src, x)
        ref_pos = (flat == self.refer_feat_token_id).nonzero(as_tuple=True)[0]
        if len(ref_pos) > 0:
            offs, o = [], 0
            for c, ind in zip(counts, refer_inds):
                offs.append(ind + o)
                o += c
            src = G.gather_rows(torch.cat(offs).to(dev).contiguous(), reg_src)
            G.scatter_rows(ref_pos.to(dev), src, x)
        attn_mask = ids_new.ne(self.pad_token_id)
        vis_outputs = {"pred_boxes": [b.to(dev) for b in selected], "image_features": img_tok, "region_features": region}
        aux = dict(pred_all=pc[:, :eng.cfg.num_queries], scores=sc[:, :eng.cfg.num_queries], det_logits=det_logits)
        return x, ids_new, labels_new, attn_mask, vis_outputs, aux

    def _kv_tuple(self, ctx: int, incremental: bool = False):
        """HF's tuple of per-layer (k, v) bf16 [B, H, ctx, D]: views of a bf16 cache.  With an fp8 cache they hold bf16_rn(x^):
        one dequantised copy, or with `incremental` (a forward() step loop) views of the engine's bf16 mirror, which each call
        extends by the positions added since the last one."""
        eng = self.engine
        if not eng.kv_fp8:
            kv = eng.kv
        elif incremental:
            kv = eng.kv_mirror_sync(ctx)
        else:
            kv = eng.kv_dequantized(ctx)
        return tuple((kv[i, 0][:, :, :ctx], kv[i, 1][:, :, :ctx]) for i in range(kv.shape[0]))

    # ------------------------------------------------------------------ forward (groma.py:202-427)
    @torch.no_grad()
    def forward(self, input_ids=None, inputs_embeds=None, labels=None, attention_mask=None, images=None, refer_boxes=None,
                ground_boxes=None, past_key_values=None, use_cache=False, output_attentions=False, output_hidden_states=False,
                return_dict=False, _selected_override=None, _reserve=0):
        eng = self.engine
        vis_outputs = None
        if past_key_values is None:
            if eng.drop_group():          # a prefill replaces the caches of an earlier grouped generate()
                self._graph = None
            x, ids_new, labels_new, mask, vis_outputs, aux = self._prefill_inputs(input_ids, images, refer_boxes, ground_boxes, labels,
                                                                                  _selected_override)
            B, T = ids_new.shape
            eng.ensure_rope(T + 1)
            # room for a step-wise decode loop over forward(past_key_values=...) (serve/model_worker.py:288-304, serve/cli.py
            # and HF generate all drive the model that way); the cache grows geometrically beyond it
            eng.alloc_kv(B, T + max(int(_reserve), self.kv_headroom))
            kv_len = mask.sum(1).to(torch.int32).to(eng.dev)
            logits = eng.llm_prefill(x, B, T, kv_len).reshape(B, T, -1)
            self._last = dict(ids=ids_new, mask=mask, aux=aux)
        else:
            B = past_key_values[0][0].shape[0]
            past = past_key_values[0][0].shape[-2]
            if eng.kv is None or past != eng.past or B != eng.kv.shape[2]:
                raise RuntimeError("past_key_values must be the cache returned by the previous forward() of this model")
            if past + 1 > eng.kv_cap:
                eng.grow_kv(max(past + 1, 2 * eng.kv_cap))      # new storage: the captured decode graph is keyed on it
            eng.ensure_rope(past + 1)
            d = eng._decode_buffers(B)
            d["ids"].copy_(input_ids.reshape(-1).to(eng.dev))
            d["pos"].fill_(past)
            d["kv_len"].fill_(past + 1)               # all-ones mask over past+1 (groma.py:376-379)
            # step-wise callers (serve/model_worker.py:288-304, serve/cli.py) get the same CUDA-graph step as generate() from
            # their second decode step on; the first one runs eagerly (it also warms every kernel up outside the capture)
            self._fwd_decode_steps = getattr(self, "_fwd_decode_steps", 0) + 1
            if self.use_cuda_graph and self._fwd_decode_steps >= 2:
                self._capture(B).replay()
                logits = d["logits"].clone().reshape(B, 1, -1)
            else:
                logits = eng.decode_step(B).clone().reshape(B, 1, -1)
            eng.check_decode_status()
            eng.past = past + 1
            labels_new = None
        loss = None
        if labels is not None and past_key_values is None:
            lab = labels_new.to(logits.device)
            loss = torch.nn.functional.cross_entropy(logits[:, :-1].reshape(-1, logits.shape[-1]).float(), lab[:, 1:].reshape(-1),
                                                     ignore_index=IGNORE_INDEX)
        if use_cache:
            pkv = self._kv_tuple(eng.past, incremental=True)
        else:
            pkv = None
            eng.kv_mirror, eng.kv_mirror_len = None, 0
        if not return_dict:
            out = (logits, pkv)
            return (loss,) + out if loss is not None else out
        return CausalLMOutputWithPast(loss=loss, logits=logits, past_key_values=pkv, hidden_states=(None, vis_outputs), attentions=None)

    __call__ = forward

    # ------------------------------------------------------------------ generate (HF greedy_search / sample contract)
    @torch.no_grad()
    def generate(self, input_ids, images=None, refer_boxes=None, ground_boxes=None, use_cache=True, do_sample=False,
                 max_new_tokens=None, return_dict_in_generate=False, output_hidden_states=False, generation_config=None,
                 eos_token_id=None, temperature=None, top_k=None, top_p=None, repetition_penalty=None, no_repeat_ngram_size=None,
                 bad_words_ids=None, min_length=None, min_new_tokens=None, suppress_tokens=None, typical_p=None, epsilon_cutoff=None,
                 eta_cutoff=None, num_beams=None, length_penalty=None, early_stopping=None, num_return_sequences=None,
                 _selected_override=None, **kwargs):
        """Greedy search, or with do_sample=True HF 4.32 `sample()`: temperature -> top-k -> top-p warpers
        (resolve_sampling_params) and a draw on the device (include/groma_b200.h: groma_sample_tokens).  The draw's seed comes
        from the CUDA default generator, so torch.manual_seed(s) makes a sampled generate() reproducible.  Unlike HF, sampling
        is on only when do_sample=True is passed: generation_config.do_sample alone (which the reference's training script sets
        in every checkpoint) keeps greedy search, the mode the eval scripts ask for.
        The logits processors repetition_penalty, no_repeat_ngram_size, bad_words_ids, min_length, min_new_tokens and
        suppress_tokens, and with do_sample=True the warpers typical_p, epsilon_cutoff and eta_cutoff, follow HF 4.32
        (resolve_processing_params; include/groma_b200.h: groma_logits_process, groma_sample_tokens_ex).  They see what HF
        passes as `input_ids`: the caller's prompt ids (after the in-place refer / ground edits) and the tokens generated so
        far, not the expanded image / region sequence.  With none of them on, the decode step is exactly the plain one.
        num_beams > 1 (passed explicitly; generation_config.num_beams alone keeps greedy search) runs HF 4.32 beam search with
        length_penalty, early_stopping and num_return_sequences (resolve_beam_params, oracle/beam_search.py): `sequences` is
        [B * num_return_sequences, L] with the rows of an image consecutive and GenerateOutput.sequences_scores is set.  The
        vision stage and the prefill run once per image, so hidden_states keeps one (None, vis_outputs) whose pred_boxes has B
        entries, and past_key_values is None (4.32's BeamSearchDecoderOnlyOutput).
        input_ids with n >= 2 rows per image (resolve_prompt_groups): rows b*n .. b*n + n - 1 ask about image b, and the result
        is that of the same rows on images.repeat_interleave(n, 0) with each image's selection repeated per row.  The vision
        stage and selection run once per image, the prefix the rows of an image share is prefilled once, and the decode
        attention reads it once per image (engine.group_buffers); pred_boxes has B*n entries and past_key_values is None."""
        sampling = do_sample is True
        gc = generation_config or self.generation_config
        if sampling:
            sample_args = resolve_sampling_params(gc, temperature, top_k, top_p)
        if max_new_tokens is None:
            max_new_tokens = getattr(gc, "max_new_tokens", None) or 20
        eos_ids = _eos_list(eos_token_id if eos_token_id is not None else getattr(gc, "eos_token_id", None))
        n_grp = 1 if images is None else resolve_prompt_groups(input_ids.shape[0], images.shape[0], refer_boxes, ground_boxes,
                                                                self.engine.kv_dtype, num_beams)
        if n_grp > 1 and _selected_override is not None and len(_selected_override) != images.shape[0]:
            raise ValueError(f"_selected_override of a grouped call holds one selection per image ({images.shape[0]}), "
                             f"got {len(_selected_override)}")
        beam = resolve_beam_params(gc, num_beams, length_penalty, early_stopping, num_return_sequences, input_ids.shape[0], do_sample,
                                   self.engine.kv_dtype, eos_ids, **kwargs)
        pad_id = getattr(gc, "pad_token_id", None)
        eng = self.engine
        dev = eng.dev
        proc = resolve_processing_params(
            gc, eos_ids, eng.cfg.vocab + eng.cfg.num_new_token, sampling, repetition_penalty=repetition_penalty,
            no_repeat_ngram_size=no_repeat_ngram_size, bad_words_ids=bad_words_ids, min_length=min_length,
            min_new_tokens=min_new_tokens, suppress_tokens=suppress_tokens, typical_p=typical_p, epsilon_cutoff=epsilon_cutoff,
            eta_cutoff=eta_cutoff)
        process = proc is not None
        if beam is not None:
            return self._generate_beam(input_ids, images, refer_boxes, ground_boxes, max_new_tokens, eos_ids, pad_id, proc, beam,
                                       return_dict_in_generate, output_hidden_states, _selected_override, kwargs.get("_keep_logits"))
        eng.kv_mirror, eng.kv_mirror_len = None, 0     # fp8: generate() hands out one dequantised copy at the end
        if eng.drop_beam():                            # a greedy call frees the beam cache of an earlier beam search
            self._graph = None                         # (and the beam graph that addressed it)
        if n_grp == 1 and eng.drop_group():            # and the caches of an earlier grouped call
            self._graph = None
        x, ids_new, _, mask, vis_outputs, aux = self._prefill_inputs(input_ids, images, refer_boxes, ground_boxes, None, _selected_override,
                                                                     n=n_grp)
        B, T = ids_new.shape
        eng.ensure_rope(T + max_new_tokens)        # HF's rotary cache extends on demand; ours is rebuilt before the kernels index it
        group = None
        if n_grp == 1:
            eng.alloc_kv(B, T + max_new_tokens)
        else:
            # prompt groups: shared prefix + per-row caches (engine.group_buffers); no per-row cache of the whole prompt exists
            eng.drop_kv()
            group = eng.group_buffers(B // n_grp, n_grp, shared_prefix_len(ids_new, n_grp), T, max_new_tokens)
        kv_len = mask.sum(1).to(torch.int32).to(dev)
        self._last = dict(ids=ids_new, mask=mask, aux=aux)
        self._mark("assemble+embed")
        if group is None:
            logits = eng.llm_prefill(x, B, T, kv_len, last_only=True)          # [B, V] at the last (padded) position
        else:
            logits = eng.llm_prefill_grouped(x, group, T, kv_len)
        self._mark("llm_prefill")
        d = eng._decode_buffers(B)
        if process:
            # the history HF's processors read: the caller's (edited) prompt ids, then one token per step
            L0 = input_ids.shape[1]
            lists = dict(eos=proc["eos"], ban=proc["ban"], seqs=proc["seqs"])
            d = eng.process_buffers(B, L0 + max_new_tokens, G.process_params_words(**lists))
            G.process_params(proc["repetition_penalty"], proc["no_repeat_ngram_size"], proc["min_length"], L0,
                             proc["min_new_tokens"], **lists, bad_words=proc["bad_words"], out=d["proc_params"])
            d["hist"][:, :L0].copy_(input_ids.to(device=dev, dtype=torch.int32))
            d["hist_len"].fill_(L0)
        if sampling:
            G.sample_params(*sample_args, out=d["sample_params"])
            if process:
                G.sample_params_ex(*sample_args, proc["typical_p"], proc["epsilon_cutoff"], proc["eta_cutoff"],
                                   out=d["sample_params_ex"])
            torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64, device=dev, out=d["seed"])
            d["pos"].fill_(T - 1)          # Philox step of the first token: the position of the prompt's last token
        eng.choose_tokens(logits, d, sampling, process)
        d["pos"].fill_(T)
        d["kv_len"].fill_(T + 1)
        out_tokens = torch.empty((max_new_tokens, B), dtype=torch.int64, device=dev)
        out_tokens[0].copy_(d["ids"])
        self._step_logits = [logits.clone()] if kwargs.get("_keep_logits") else None
        eos_t = torch.tensor(eos_ids, dtype=torch.int64, device=dev) if eos_ids else None
        graph = None
        steps_done = 1
        check_every = 16
        for s in range(1, max_new_tokens):
            if eos_t is not None and (s == 1 or s % check_every == 0):
                # one host sync every `check_every` steps: stop once every row has produced an EOS
                if bool(torch.isin(out_tokens[:steps_done], eos_t).any(0).all()):
                    break
            if self.use_cuda_graph and graph is None and s >= 2:
                graph = self._capture(B, sample=sampling, process=process, group=group)
            if graph is not None:
                graph.replay()
            else:
                eng.decode_step(B, sample=sampling, process=process, group=group)
            out_tokens[s].copy_(d["ids"])
            if self._step_logits is not None:
                self._step_logits.append(d["logits"].clone())
            steps_done = s + 1
        self._mark("decode")
        eng.check_decode_status()
        # a grouped call hands out no cache: forward(past_key_values=...) must start from a prefill
        eng.past = T + steps_done - 1 if group is None else -1
        new = out_tokens[:steps_done].t().contiguous()
        if eos_t is not None:
            # HF greedy_search semantics: a row that has emitted EOS is fed / reported as pad_token_id from then on, and
            # generation ends with the step at which the last unfinished row emits its EOS
            if pad_id is None:
                pad_id = self.pad_token_id if self.pad_token_id is not None else eos_ids[0]
            is_eos = torch.isin(new, eos_t)
            after = (is_eos.cumsum(1) - is_eos.long()) > 0
            new = torch.where(after, torch.full_like(new, pad_id), new)
            finished_at = torch.where(is_eos.any(1), is_eos.float().argmax(1) + 1, torch.full((B,), new.shape[1], device=dev))
            new = new[:, :int(finished_at.max())]
        sequences = torch.cat([input_ids.to(dev), new], 1)
        if not return_dict_in_generate:
            return sequences
        return GenerateOutput(sequences=sequences, hidden_states=((None, vis_outputs),) if output_hidden_states else (),
                              past_key_values=self._kv_tuple(eng.past) if use_cache and group is None else None)

    def _generate_beam(self, input_ids, images, refer_boxes, ground_boxes, max_new_tokens, eos_ids, pad_id, proc, beam,
                       return_dict_in_generate, output_hidden_states, _selected_override, keep_logits):
        """generate(num_beams > 1): one prefill per image, then B * nb decode rows over the shared prompt cache and a beam cache
        reordered through its ancestry table (engine.decode_step(beam=...)); finalize on the host from the hypothesis store."""
        eng = self.engine
        dev = eng.dev
        nb, process = beam["num_beams"], proc is not None
        if pad_id is None:
            pad_id = self.pad_token_id if self.pad_token_id is not None else (eos_ids[0] if eos_ids else 0)
        eng.kv_mirror, eng.kv_mirror_len = None, 0
        if eng.drop_group():
            self._graph = None
        x, ids_new, _, mask, vis_outputs, aux = self._prefill_inputs(input_ids, images, refer_boxes, ground_boxes, None, _selected_override)
        B, T = ids_new.shape
        R, L0 = B * nb, input_ids.shape[1]
        max_length = L0 + max_new_tokens
        eng.ensure_rope(T + max_new_tokens)
        eng.alloc_kv(B, T)                   # the prompt only: generated keys live in the beam cache
        kv_len = mask.sum(1).to(torch.int32).to(dev)
        self._last = dict(ids=ids_new, mask=mask, aux=aux)
        self._mark("assemble+embed")
        logits = eng.llm_prefill(x, B, T, kv_len, last_only=True)
        self._mark("llm_prefill")
        d = eng._decode_buffers(R)
        st = eng.beam_buffers(B, nb, max_new_tokens, max_length)
        params = G.beam_params(beam["early_stopping"], max_length, L0, pad_id, eos_ids, beam["length_penalty"], device=dev)
        eng.beam_reset(st, input_ids, T, params, beam_denominators(beam["length_penalty"], max_length).to(dev))
        if process:
            lists = dict(eos=proc["eos"], ban=proc["ban"], seqs=proc["seqs"])
            d = eng.process_buffers(R, max_length, G.process_params_words(**lists))
            G.process_params(proc["repetition_penalty"], proc["no_repeat_ngram_size"], proc["min_length"], L0,
                             proc["min_new_tokens"], **lists, bad_words=proc["bad_words"], out=d["proc_params"])
        d["logits"].copy_(logits.repeat_interleave(nb, 0))      # every beam of an image starts from its prefill logits
        eng.beam_tail(d["logits"], st, d, process)
        self._step_logits = [d["logits"].clone()] if keep_logits else None
        self._step_lp = [st["lp"].clone()] if keep_logits else None
        d["pos"].fill_(T)
        d["kv_len"].fill_(T + 1)
        graph = None
        for s in range(1, max_new_tokens):
            if s == 1 or s % 16 == 0:        # one host sync every 16 steps: stop once every image is done
                if int(st["flags"][0]) != 0:
                    break
            if self.use_cuda_graph and graph is None and s >= 2:
                graph = self._capture(R, process=process, beam=st)
            if graph is not None:
                graph.replay()
            else:
                eng.decode_step(R, process=process, beam=st)
            if keep_logits:
                self._step_logits.append(d["logits"].clone())
                self._step_lp.append(st["lp"].clone())
        self._mark("decode")
        eng.past = -1                        # no cache is handed out: forward(past_key_values=...) must start from a prefill
        h = {k: st[k].cpu() for k in ("hyp_tok", "hyp_len", "hyp_score", "hyp_order", "hyp_count", "worst", "done", "beam_scores",
                                      "hist", "hist_len", "flags")}
        if int(h["flags"][1]) != 0:
            raise ValueError(f"At most {nb} tokens in the candidates of a beam step can be equal to `eos_token_id: {eos_ids}`. "
                             "Make sure that `next_tokens` is correctly defined.")
        rows, scores = _beam_finalize(h, B, nb, L0, max_length, beam, pad_id, eos_ids)
        new = torch.tensor(rows, dtype=torch.int64).to(dev)
        sequences = torch.cat([input_ids.to(dev).repeat_interleave(beam["num_return_sequences"], 0), new], 1)
        if not return_dict_in_generate:
            return sequences
        return GenerateOutput(sequences=sequences, hidden_states=((None, vis_outputs),) if output_hidden_states else (),
                              past_key_values=None, sequences_scores=torch.tensor(scores, dtype=torch.float32).to(dev))

    def _capture(self, B: int, sample: bool = False, process: bool = False, beam: Optional[dict] = None, group: Optional[dict] = None):
        """Capture one decode step (all 32 layers + heads + [logits processors] + argmax or sampling + position advance) into a
        CUDA graph.  Sampling and processing read their parameters, seed and token history from device buffers, so one graph
        serves every setting whose buffers fit (the buffers' addresses are part of the key)."""
        eng = self.engine
        d = eng._decode_buffers(B)
        key = (B, eng.kv.data_ptr() if eng.kv is not None else 0, getattr(eng, "kv_cap", 0), eng.rope_cos.data_ptr(), eng.use_megakernel, eng.kv_dtype,
               eng.kv_scale.data_ptr() if eng.kv_scale is not None else 0, sample, process)
        if process:
            key += (d["hist"].data_ptr(), d["hist"].shape[1], d["proc_params"].data_ptr(), d["proc_params"].numel())
        if beam is not None:
            key += ("beam", beam["nb"], beam["kv"].data_ptr(), beam["src"].shape[1], beam["hist"].shape[1], beam["denom"].data_ptr())
        if group is not None:
            key += ("group", group["n"], group["P"], group["prefix"].data_ptr(), group["row"].data_ptr(), group["row"].shape[4])
        if self._graph is not None and self._graph[0] == key:
            return self._graph[1]
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        saved = {k: d[k].clone() for k in ("ids", "pos", "kv_len") + (("hist_len",) if process else ())}
        l0 = G.LAUNCHES
        with torch.cuda.stream(s):
            # thread_local: NCCL's watchdog thread may touch the CUDA API while this thread captures
            with torch.cuda.graph(g, stream=s, capture_error_mode="thread_local"):
                eng.decode_step(B, sample=sample, process=process, beam=beam, group=group)
        self._graph_kernels = G.LAUNCHES - l0
        torch.cuda.current_stream().wait_stream(s)
        for k, v in saved.items():      # capture does not execute; restore just in case of warm-up side effects
            d[k].copy_(v)
        self._graph = (key, g)
        return g


def _beam_finalize(h: dict, B: int, nb: int, L0: int, max_length: int, beam: dict, pad_id: int, eos_ids: Sequence[int]):
    """4.32 BeamSearchScorer.finalize on the host copy of the device state: every image not done adds its beams (full ids, fp32
    beam score) to its hypothesis list, then the best num_return_sequences per image are padded as 4.32 pads them.  Returns
    (generated-token rows, sequences_scores)."""
    cur = int(h["hist_len"][0])
    denom = beam_denominators(beam["length_penalty"], max_length).tolist()
    best, best_scores = [], []
    for b in range(B):
        n = int(h["hyp_count"][b])
        hyps = [(float(h["hyp_score"][b, k]), h["hyp_tok"][b, k, :int(h["hyp_len"][b, k])].tolist())
                for k in (int(v) for v in h["hyp_order"][b, :n])]
        worst = float(h["worst"][b])
        if not int(h["done"][b]):
            for j in range(nb):
                score = float(h["beam_scores"][b * nb + j]) / denom[cur]
                if len(hyps) < nb or score > worst:
                    hyps.append((score, h["hist"][b * nb + j, L0:cur].tolist()))
                    if len(hyps) > nb:
                        srt = sorted((s, i) for i, (s, _) in enumerate(hyps))
                        del hyps[srt[0][1]]
                        worst = srt[1][0]
                    else:
                        worst = min(score, worst)
        srt = sorted(hyps, key=lambda x: x[0])
        for _ in range(beam["num_return_sequences"]):
            s, toks = srt.pop()
            best.append(toks)
            best_scores.append(s)
    sent_max_len = min(max(len(t) for t in best) + L0 + 1, max_length)
    rows = []
    for toks in best:
        row = toks + [pad_id] * (sent_max_len - L0 - len(toks))
        if len(toks) + L0 < sent_max_len:
            row[len(toks)] = eos_ids[0]
        rows.append(row)
    return rows, best_scores


try:
    AutoConfig.register("groma", GromaConfig)
    AutoModel.register(GromaConfig, GromaModel)
except ValueError:
    pass
