"""GromaEngine -- host-side orchestration of the GPU (H100, sm_90a) forward path.

Holds the packed weight arena (bf16 matrices in the layouts the kernels want, fp32 vectors) and sequences the C-ABI
kernels of libgroma_b200.so for: DINOv2 encoder -> image tokens -> Deformable-DETR proposer -> region selection (NMS on
device, randperm on the host CPU RNG) -> region encoder -> LLaMA prefill / decode.  PyTorch provides device memory and
streams only.  Stage boundaries and rounding points are listed in DESIGN.md; the reference functions each stage
replaces are cited at the methods (paths relative to the FoundationVision/Groma tree).
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import ops as G
from .config import PathConfig


def _cat(*ts):
    return torch.cat(list(ts), 0)


class GromaEngine:
    def __init__(self, cfg: PathConfig, state_dict: Dict[str, torch.Tensor], device: str = "cuda", detector_only: bool = False,
                 nf4: bool = False, fp8: bool = False):
        """state_dict: any mapping key -> tensor with the reference's parameter names (a lazy `ShardedStateDict` reads each
        tensor from its shard exactly when it is packed).  detector_only: a `CustomDDETRModel` checkpoint (keys without the
        `perceiver.` prefix, no bridge / region encoder / LLaMA weights; reference ddetr.py:98-155) -- only vit() and
        proposer() are usable.  nf4: 4-bit NF4 weights (DESIGN.md section 4): the LLaMA projections and both heads are stored as
        NF4 codes + absmax only (`self.q4`), every other nn.Linear weight as its bf16 W~ = dequant(quant(W)).  fp8: e4m3 LLaMA
        projections (DESIGN.md section 4): q/k/v/o/gate/up/down as e4m3 codes + one fp32 scale per row (`self.q8`), multiplied
        with per-row quantised activations; the heads and every other weight stay bf16."""
        if not torch.cuda.is_available():
            raise RuntimeError("GromaEngine needs a CUDA device: the GPU path has no CPU fallback")
        self.cfg = cfg
        self.dev = torch.device(device)
        self.sms = torch.cuda.get_device_properties(self.dev).multi_processor_count
        self.detector_only = detector_only
        self.nf4 = nf4
        self.fp8 = fp8
        if nf4 and fp8:
            raise ValueError("NF4 and fp8 LLaMA weights are exclusive: a model has one weight format")
        self.q8: Dict[str, tuple] = {}   # fp8: name -> (codes float8_e4m3fn [N, K], fp32 scales [N]), row views of the fp8 arenas
        self.q4: Dict[str, tuple] = {}   # nf4: name -> (codes, absmax) in the decode tile layout (ops.nf4_tile), rows, K
        self._w_scratch = None
        self.w: Dict[str, torch.Tensor] = {}
        self._pack(state_dict)
        self._constants()
        self.kv = None
        self.kv_dtype = torch.bfloat16   # or torch.float8_e4m3fn: codes in self.kv + one fp32 scale per head vector (DESIGN.md section 4)
        self.kv_scale = None              # fp8: [layer, k/v, B, H, cap]
        self.kv_mirror = None             # fp8: bf16 copy of the first kv_mirror_len positions (kv_mirror_sync)
        self.kv_mirror_len = 0
        self.stages: Dict[str, torch.Tensor] = {}
        self.keep_stages = False
        self.fused_splitk = False
        self.decode_tiled = os.environ.get("GROMA_DECODE_TILED", "0") == "1"   # decode GEMMs stream a tile-major weight copy (+13 GB)
        self._wt: Dict[str, torch.Tensor] = {}
        self.use_2cta = True           # two-CTA cluster GEMM (B tile multicast) for the large prefill projections and 3x3 convs
        self.fused_head_tail = os.environ.get("GROMA_FUSED_HEAD_TAIL", "1") != "0"   # decode: head reduce + argmax + advance in one launch
        self.use_fused_rope = os.environ.get("GROMA_FUSED_ROPE", "1") != "0"   # RoPE + KV append in the qkv GEMM epilogue (prefill)
        self.fuse_gn_apply = os.environ.get("GROMA_FUSE_GN", "1") != "0"       # GroupNorm + ReLU of a fusion round applied by the next round's shuffle
        # wgmma flash attention (attention_wgmma.cu: two warpgroups of 64 query rows, P as register operand) for head dims 64 / 128
        # (DINOv2 and the LLaMA prefill); the mma.sync kernel stays for head dim 32 (Deformable-DETR self-attention) and the
        # miniature test shapes.  GROMA_TC_ATTENTION=0 switches back for A/B runs.
        self.use_tc_attention = os.environ.get("GROMA_TC_ATTENTION", "1") == "1"
        self.use_megakernel = os.environ.get("GROMA_DECODE_MEGA", "0") == "1"   # one persistent kernel per decode step (csrc/decode_megakernel.cu)
        self.fused_decode = True     # fused reduce epilogues + PDL in the decode step
        self.fused_rope_attn = os.environ.get("GROMA_FUSED_ROPE_ATTN", "1") == "1"   # qkv reduce + RoPE + KV append inside the attention launch
        self.use_pdl = True
        self.graph_proposer = os.environ.get("GROMA_GRAPH_PROPOSER", "1") == "1"
        self._prop_graphs: Dict[tuple, tuple] = {}
        self.topk_override = None  # tests: int64 [B, num_queries] token indices replacing the proposer's own top-k
        self.timing_hook = None   # bench.py: list collecting (start_event, end_event, algorithmic_bytes) per swap-AB GEMM

    # ------------------------------------------------------------------------------------------ weights
    def _mat(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(self.dev).to(torch.bfloat16).contiguous()

    def _lin(self, t: torch.Tensor) -> torch.Tensor:
        """An nn.Linear weight: bf16, or with nf4 its W~ (quantised and dequantised on the device, flat 64-element blocks of
        the tensor as stored in the checkpoint)."""
        m = self._mat(t)
        if self.nf4:
            codes, absmax = G.nf4_quantize(m)
            G.nf4_dequantize(codes, absmax, m.shape, out=m)
        return m

    def _vec(self, t: torch.Tensor) -> torch.Tensor:
        return t.to(self.dev).to(torch.float32).contiguous()

    def _pack(self, sd: Dict[str, torch.Tensor]):
        cfg, w = self.cfg, self.w
        H, D, T = cfg.vit_hidden, cfg.d_model, cfg.llm_hidden
        pfx = "" if self.detector_only else "perceiver."
        ve = pfx + "vis_encoder."
        pw = sd[ve + "embeddings.patch_embeddings.projection.weight"].reshape(H, -1).float()
        self.patch_ld = ((pw.shape[1] + 7) // 8) * 8
        pwp = torch.zeros(H, self.patch_ld)
        pwp[:, :pw.shape[1]] = pw
        w["vit.patch.w"], w["vit.patch.b"] = self._mat(pwp), self._vec(sd[ve + "embeddings.patch_embeddings.projection.bias"])
        w["vit.cls"] = self._vec(sd[ve + "embeddings.cls_token"].reshape(-1))
        w["vit.pos"] = self._vec(self._interp_pos(sd[ve + "embeddings.position_embeddings"].float()))
        for i in range(cfg.vit_layers):
            p, o = f"{ve}encoder.layer.{i}.", f"vit.{i}."
            w[o + "ln1.w"], w[o + "ln1.b"] = self._vec(sd[p + "norm1.weight"]), self._vec(sd[p + "norm1.bias"])
            w[o + "qkv.w"] = _cat(*[self._lin(sd[p + f"attention.attention.{n}.weight"]) for n in ("query", "key", "value")])
            w[o + "qkv.b"] = self._vec(_cat(*[sd[p + f"attention.attention.{n}.bias"] for n in ("query", "key", "value")]))
            w[o + "o.w"], w[o + "o.b"] = self._lin(sd[p + "attention.output.dense.weight"]), self._vec(sd[p + "attention.output.dense.bias"])
            w[o + "ls1"], w[o + "ls2"] = self._vec(sd[p + "layer_scale1.lambda1"]), self._vec(sd[p + "layer_scale2.lambda1"])
            w[o + "ln2.w"], w[o + "ln2.b"] = self._vec(sd[p + "norm2.weight"]), self._vec(sd[p + "norm2.bias"])
            w[o + "fc1.w"], w[o + "fc1.b"] = self._lin(sd[p + "mlp.fc1.weight"]), self._vec(sd[p + "mlp.fc1.bias"])
            w[o + "fc2.w"], w[o + "fc2.b"] = self._lin(sd[p + "mlp.fc2.weight"]), self._vec(sd[p + "mlp.fc2.bias"])
        if not self.detector_only:
            w["bridge0.w"], w["bridge0.b"] = self._lin(sd["img_txt_bridge.0.weight"]), self._vec(sd["img_txt_bridge.0.bias"])
            w["bridge2.w"], w["bridge2.b"] = self._lin(sd["img_txt_bridge.2.weight"]), self._vec(sd["img_txt_bridge.2.bias"])
        w["inproj.w"] = self._mat(sd[pfx + "input_proj.0.0.weight"].reshape(D, -1))
        w["inproj.b"] = self._vec(sd[pfx + "input_proj.0.0.bias"])
        w["inproj.ln.w"], w["inproj.ln.b"] = self._vec(sd[pfx + "input_proj.0.1.weight"]), self._vec(sd[pfx + "input_proj.0.1.bias"])
        dt = pfx + "ddetr_transformer."

        def lin(dst, src):
            w[dst + ".w"] = self._lin(sd[src + ".weight"])
            if src + ".bias" in sd:
                w[dst + ".b"] = self._vec(sd[src + ".bias"])

        def ln(dst, src):
            w[dst + ".w"], w[dst + ".b"] = self._vec(sd[src + ".weight"]), self._vec(sd[src + ".bias"])

        def msda(dst, src):
            w[dst + ".proj.w"] = _cat(self._lin(sd[src + ".sampling_offsets.weight"]), self._lin(sd[src + ".attention_weights.weight"]))
            w[dst + ".proj.b"] = self._vec(_cat(sd[src + ".sampling_offsets.bias"], sd[src + ".attention_weights.bias"]))
            lin(dst + ".value", src + ".value_proj")
            lin(dst + ".out", src + ".output_proj")

        for i in range(cfg.enc_layers):
            p, o = f"{dt}encoder.layers.{i}.", f"enc.{i}."
            msda(o + "sa", p + "self_attn"); ln(o + "ln1", p + "self_attn_layer_norm")
            lin(o + "fc1", p + "fc1"); lin(o + "fc2", p + "fc2"); ln(o + "ln2", p + "final_layer_norm")
        for i in range(cfg.dec_layers):
            p, o = f"{dt}decoder.layers.{i}.", f"dec.{i}."
            w[o + "qk.w"] = _cat(self._lin(sd[p + "self_attn.q_proj.weight"]), self._lin(sd[p + "self_attn.k_proj.weight"]))
            w[o + "qk.b"] = self._vec(_cat(sd[p + "self_attn.q_proj.bias"], sd[p + "self_attn.k_proj.bias"]))
            lin(o + "v", p + "self_attn.v_proj"); lin(o + "o", p + "self_attn.out_proj"); ln(o + "ln1", p + "self_attn_layer_norm")
            msda(o + "ca", p + "encoder_attn"); ln(o + "ln2", p + "encoder_attn_layer_norm")
            lin(o + "fc1", p + "fc1"); lin(o + "fc2", p + "fc2"); ln(o + "ln3", p + "final_layer_norm")
        w["level_embed"] = sd[dt + "level_embed"].float()
        w["query_tgt"] = self._mat(sd[dt + "query_position_embeddings.weight"])
        lin("enc_output", dt + "enc_output"); ln("enc_output_norm", dt + "enc_output_norm")
        lin("pos_trans", dt + "pos_trans"); ln("pos_trans_norm", dt + "pos_trans_norm")
        lin("cls_enc", dt + "class_embed_enc")
        L = cfg.dec_layers
        lin("cls_coco", f"{dt}class_embed_coco.{L - 1}"); lin("cls_sa1b", f"{dt}class_embed_sa1b.{L - 1}")
        for i in (L - 2, L - 1, L):
            if i < 0:
                continue
            for j in range(3):
                lin(f"bbox.{i}.{j}", f"{dt}bbox_embed.{i}.layers.{j}")
        if self.detector_only:
            return
        # region encoder
        re_ = "region_encoder."
        self.in_ld = H + 64
        for l in range(3):
            wi = torch.zeros(H, self.in_ld)
            wi[:, :H + 2] = sd[f"{re_}mlvl_fuse.input_conv.{l}.weight"].reshape(H, H + 2).float()
            w[f"inconv.{l}.w"], w[f"inconv.{l}.b"] = self._mat(wi), self._vec(sd[f"{re_}mlvl_fuse.input_conv.{l}.bias"])
        for k in range(cfg.fuse_rounds):
            cw = sd[f"{re_}mlvl_fuse.fuse_convs.{k}.conv.weight"]
            w[f"fuse.{k}.w"] = self._mat(cw.permute(0, 2, 3, 1).reshape(H, 9 * H))
            w[f"fuse.{k}.gn.w"], w[f"fuse.{k}.gn.b"] = self._vec(sd[f"{re_}mlvl_fuse.fuse_convs.{k}.gn.weight"]), self._vec(sd[f"{re_}mlvl_fuse.fuse_convs.{k}.gn.bias"])
        w["pconv.w"] = self._mat(torch.cat([sd[f"{re_}roi_align.pconvs.{l}.weight"].permute(0, 2, 3, 1).reshape(H, 9 * H) for l in range(3)], 1))
        w["pconv.b"] = self._vec(sum(sd[f"{re_}roi_align.pconvs.{l}.bias"].float() for l in range(3)))
        # bf16-rounded values kept in fp32 for the K=4 linear
        w["pos0.w"] = self._lin(sd[re_ + "roi_align.pos_embedd.0.weight"]).float().contiguous()
        w["pos0.b"] = self._vec(sd[re_ + "roi_align.pos_embedd.0.bias"])
        ln("pos2", re_ + "roi_align.pos_embedd.2"); lin("pos3", re_ + "roi_align.pos_embedd.3"); ln("pos5", re_ + "roi_align.pos_embedd.5")
        lin("updims", re_ + "roi_align.updims")
        fw = sd[re_ + "roi_align.flatten_linear.weight"]
        n_mid, ro = fw.shape[0], cfg.roi_out
        w["flatten.w"] = self._lin(fw).reshape(n_mid, H, ro * ro).permute(0, 2, 1).reshape(n_mid, ro * ro * H).contiguous()  # (c,h,w) -> (h,w,c)
        w["flatten.b"] = self._vec(sd[re_ + "roi_align.flatten_linear.bias"])
        # LLaMA.  The projections live in two arenas so that the persistent decode kernel addresses every weight tile through one
        # TMA descriptor each (include/groma_b200.h: groma_decode_step_args); the per-layer entries of `w` are row views into them
        w["embed"] = self._mat(sd["llm.model.embed_tokens.weight"])
        w["new_embed"] = self._mat(sd["new_input_embs.weight"])
        L, I, V = cfg.llm_layers, cfg.llm_inter, cfg.vocab + cfg.num_new_token
        if self.nf4:
            self._pack_llm_nf4(sd)
            return
        if self.fp8:
            self._pack_llm_fp8(sd)
            return
        RW = 4 * T + 2 * I
        arena = torch.empty((L * RW + V, T), dtype=torch.bfloat16, device=self.dev)
        down = torch.empty((L * T, I), dtype=torch.bfloat16, device=self.dev)
        lnw = torch.empty((2 * L + 1, T), dtype=torch.float32, device=self.dev)
        for i in range(L):
            p, o = f"llm.model.layers.{i}.", f"llm.{i}."
            r0 = i * RW
            for k, n in enumerate(("q", "k", "v")):
                arena[r0 + k * T: r0 + (k + 1) * T].copy_(sd[p + f"self_attn.{n}_proj.weight"])
            arena[r0 + 3 * T: r0 + 4 * T].copy_(sd[p + "self_attn.o_proj.weight"])
            g, u = sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]
            arena[r0 + 4 * T: r0 + RW].view(I, 2, T)[:, 0].copy_(g)          # rows (gate_j, up_j) interleaved
            arena[r0 + 4 * T: r0 + RW].view(I, 2, T)[:, 1].copy_(u)
            down[i * T: (i + 1) * T].copy_(sd[p + "mlp.down_proj.weight"])
            lnw[2 * i].copy_(sd[p + "input_layernorm.weight"])
            lnw[2 * i + 1].copy_(sd[p + "post_attention_layernorm.weight"])
            w[o + "qkv.w"], w[o + "o.w"], w[o + "gu.w"] = arena[r0: r0 + 3 * T], arena[r0 + 3 * T: r0 + 4 * T], arena[r0 + 4 * T: r0 + RW]
            w[o + "down.w"] = down[i * T: (i + 1) * T]
            w[o + "ln1"], w[o + "ln2"] = lnw[2 * i], lnw[2 * i + 1]
        lnw[2 * L].copy_(sd["llm.model.norm.weight"])
        arena[L * RW: L * RW + cfg.vocab].copy_(sd["llm.lm_head.weight"])
        arena[L * RW + cfg.vocab:].copy_(sd["extra_lm_head.weight"])
        w["llm.norm"] = lnw[2 * L]
        w["head.w"] = arena[L * RW:]
        self.llm_arena, self.llm_down, self.llm_ln = arena, down, lnw

    def _pack_llm_nf4(self, sd):
        """The LLaMA projections and lm_head || extra_lm_head as NF4 codes + absmax in the decode tile layout, one entry of
        `self.q4` per GEMM of the decode step.  Each checkpoint tensor is quantised on its own (blocks of 64 consecutive k
        of one row, since K % 64 == 0), so concatenating q/k/v, interleaving gate/up rows and stacking the heads only moves
        whole blocks.  No bf16 copy of these weights stays on the device."""
        cfg, w = self.cfg, self.w
        T, L, I = cfg.llm_hidden, cfg.llm_layers, cfg.llm_inter
        if T % 64 or I % 64:
            raise ValueError("4-bit NF4 weights need llm_hidden and llm_inter divisible by 64 (one block = 64 k of one row)")

        def quant(key):
            t = self._mat(sd[key])
            c, a = G.nf4_quantize(t)
            return c.view(t.shape[0], -1), a.view(t.shape[0], -1)

        def store(name, parts, interleave=False):
            if interleave:   # rows (gate_j, up_j)
                c = torch.stack([parts[0][0], parts[1][0]], 1).flatten(0, 1)
                a = torch.stack([parts[0][1], parts[1][1]], 1).flatten(0, 1)
            else:
                c, a = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
            n, k = c.shape[0], c.shape[1] * 2
            self.q4[name] = (*G.nf4_tile(c.reshape(-1), a.reshape(-1), n, k), n, k)

        lnw = torch.empty((2 * L + 1, T), dtype=torch.float32, device=self.dev)
        for i in range(L):
            p, o = f"llm.model.layers.{i}.", f"llm.{i}."
            store(o + "qkv.w", [quant(p + f"self_attn.{n}_proj.weight") for n in ("q", "k", "v")])
            store(o + "o.w", [quant(p + "self_attn.o_proj.weight")])
            store(o + "gu.w", [quant(p + "mlp.gate_proj.weight"), quant(p + "mlp.up_proj.weight")], interleave=True)
            store(o + "down.w", [quant(p + "mlp.down_proj.weight")])
            lnw[2 * i].copy_(sd[p + "input_layernorm.weight"])
            lnw[2 * i + 1].copy_(sd[p + "post_attention_layernorm.weight"])
            w[o + "ln1"], w[o + "ln2"] = lnw[2 * i], lnw[2 * i + 1]
        lnw[2 * L].copy_(sd["llm.model.norm.weight"])
        store("head.w", [quant("llm.lm_head.weight"), quant("extra_lm_head.weight")])
        w["llm.norm"] = lnw[2 * L]
        self.llm_arena = self.llm_down = None
        self.llm_ln = lnw

    def _pack_llm_fp8(self, sd):
        """The LLaMA projections as e4m3 codes in the row layout of the bf16 arenas ([q | k | v | o | gate/up interleaved] per
        layer, and down), plus one fp32 scale per row in a parallel scale arena.  Each checkpoint tensor is quantised per row
        from its bf16 values before q|k|v are concatenated and gate/up rows interleaved, so those steps only move whole rows.
        No bf16 copy of these weights stays on the device; lm_head || extra_lm_head stay bf16."""
        cfg, w = self.cfg, self.w
        T, L, I, V = cfg.llm_hidden, cfg.llm_layers, cfg.llm_inter, cfg.vocab + cfg.num_new_token
        if T % 16 or I % 16:
            raise ValueError("fp8 LLaMA weights need llm_hidden and llm_inter divisible by 16 (TMA rows of whole 16-byte units)")
        RW = 4 * T + 2 * I
        arena = torch.empty((L * RW, T), dtype=torch.float8_e4m3fn, device=self.dev)
        arena_s = torch.empty((L * RW,), dtype=torch.float32, device=self.dev)
        down = torch.empty((L * T, I), dtype=torch.float8_e4m3fn, device=self.dev)
        down_s = torch.empty((L * T,), dtype=torch.float32, device=self.dev)
        lnw = torch.empty((2 * L + 1, T), dtype=torch.float32, device=self.dev)

        def quant(key, codes, scales):
            G.fp8_quantize_rows(self._mat(sd[key]), codes, scales)

        for i in range(L):
            p, o = f"llm.model.layers.{i}.", f"llm.{i}."
            r0 = i * RW
            for k, n in enumerate(("q", "k", "v", "o")):
                quant(p + f"self_attn.{n}_proj.weight", arena[r0 + k * T: r0 + (k + 1) * T], arena_s[r0 + k * T: r0 + (k + 1) * T])
            gu, gu_s = arena[r0 + 4 * T: r0 + RW].view(I, 2, T), arena_s[r0 + 4 * T: r0 + RW].view(I, 2)
            for j, n in enumerate(("gate", "up")):   # rows (gate_j, up_j) interleaved
                c, sc = G.fp8_quantize_rows(self._mat(sd[p + f"mlp.{n}_proj.weight"]))
                gu[:, j].copy_(c)
                gu_s[:, j].copy_(sc)
            quant(p + "mlp.down_proj.weight", down[i * T: (i + 1) * T], down_s[i * T: (i + 1) * T])
            lnw[2 * i].copy_(sd[p + "input_layernorm.weight"])
            lnw[2 * i + 1].copy_(sd[p + "post_attention_layernorm.weight"])
            for name, a, b in (("qkv", 0, 3 * T), ("o", 3 * T, 4 * T), ("gu", 4 * T, RW)):
                self.q8[o + name + ".w"] = (arena[r0 + a: r0 + b], arena_s[r0 + a: r0 + b])
            self.q8[o + "down.w"] = (down[i * T: (i + 1) * T], down_s[i * T: (i + 1) * T])
            w[o + "ln1"], w[o + "ln2"] = lnw[2 * i], lnw[2 * i + 1]
        lnw[2 * L].copy_(sd["llm.model.norm.weight"])
        head = torch.empty((V, T), dtype=torch.bfloat16, device=self.dev)
        head[: cfg.vocab].copy_(sd["llm.lm_head.weight"])
        head[cfg.vocab:].copy_(sd["extra_lm_head.weight"])
        w["llm.norm"] = lnw[2 * L]
        w["head.w"] = head
        self.llm_arena = self.llm_down = None
        self.llm_ln = lnw
        self.fp8_arenas = (arena, arena_s, down, down_s)

    def fp8_weight_bytes(self) -> int:
        """Device bytes of the fp8 LLaMA projections: e4m3 codes + fp32 row scales (0 for other weight formats)."""
        if not self.fp8:
            return 0
        return sum(t.numel() * t.element_size() for t in self.fp8_arenas)

    def _fp8_scratch(self, rows: int, k: int):
        """(codes [rows, k], scales [rows]) views of one reusable buffer for the quantised input rows of a prefill GEMM (stream
        order keeps the previous GEMM's reads ahead of the overwrite)."""
        buf = getattr(self, "_q8_scratch", None)
        if buf is None or buf[0].numel() < rows * k or buf[1].numel() < rows:
            with torch.inference_mode(False):
                n = rows * max(self.cfg.llm_hidden, self.cfg.llm_inter)
                buf = self._q8_scratch = (torch.empty((n,), dtype=torch.float8_e4m3fn, device=self.dev),
                                          torch.empty((rows,), dtype=torch.float32, device=self.dev))
        return buf[0][: rows * k].view(rows, k), buf[1][:rows]

    def _proj(self, x: torch.Tensor, name: str, **kw) -> torch.Tensor:
        """A prefill LLaMA projection x @ W^T with gemm()'s epilogue keywords: bf16 / NF4 weights through gemm(); fp8 weights
        quantise the rows of x first and run the e4m3 GEMM."""
        if name not in self.q8:
            return G.gemm(x, self._wp(name), **kw)
        xq, xs = G.fp8_quantize_rows(x, *self._fp8_scratch(*x.shape))
        kw.pop("block_n", None)   # the fp8 kernel picks its own tile (at most 128 wide)
        return G.gemm_fp8(xq, xs, *self.q8[name], **kw)

    def nf4_bytes(self) -> int:
        """Device bytes of the NF4 weights (codes + absmax, including the padding of the last row tile)."""
        return sum(c.numel() + a.numel() * 4 for c, a, _, _ in self.q4.values())

    def _wp(self, name: str) -> torch.Tensor:
        """The bf16 weight a prefill GEMM reads.  An NF4 projection is dequantised into one reusable scratch buffer right before
        its GEMM (stream order keeps the previous GEMM's reads ahead of the overwrite)."""
        if name not in self.q4:
            return self.w[name]
        c, a, n, k = self.q4[name]
        if self._w_scratch is None:
            with torch.inference_mode(False):
                self._w_scratch = torch.empty((max(e[2] * e[3] for e in self.q4.values()),), dtype=torch.bfloat16, device=self.dev)
        return G.nf4_dequantize_tiles(c, a, n, k, out=self._w_scratch)

    def _interp_pos(self, pe: torch.Tensor) -> torch.Tensor:
        """transformers-4.32 Dinov2Embeddings.interpolate_pos_encoding: bicubic with scale_factor (g+0.1)/G (SURVEY T11).
        Input-independent -> computed once at load, on the host."""
        cfg = self.cfg
        Gp, g, dim = cfg.vit_pos_grid, cfg.grid, cfg.vit_hidden
        if g == Gp:
            return pe[0]
        patch = pe[:, 1:].reshape(1, Gp, Gp, dim).permute(0, 3, 1, 2)
        sf = (g + 0.1) / Gp
        patch = F.interpolate(patch, scale_factor=(sf, sf), mode="bicubic", align_corners=False)
        return torch.cat([pe[:, :1], patch.permute(0, 2, 3, 1).reshape(1, -1, dim)], 1)[0]

    def _constants(self):
        """Input-independent tensors of the proposer and region encoder (host-computed once)."""
        cfg = self.cfg
        g, D = cfg.grid, cfg.d_model
        S = g * g
        npf = D // 2
        ones = torch.ones(1, g, g)
        y_embed, x_embed = ones.cumsum(1, dtype=torch.float32), ones.cumsum(2, dtype=torch.float32)
        y_embed = (y_embed - 0.5) / (y_embed[:, -1:, :] + 1e-6) * (2 * math.pi)
        x_embed = (x_embed - 0.5) / (x_embed[:, :, -1:] + 1e-6) * (2 * math.pi)
        dim_t = 10000 ** (2 * torch.div(torch.arange(npf, dtype=torch.float32), 2, rounding_mode="floor") / npf)
        px, py = x_embed[:, :, :, None] / dim_t, y_embed[:, :, :, None] / dim_t
        px = torch.stack((px[..., 0::2].sin(), px[..., 1::2].cos()), dim=4).flatten(3)
        py = torch.stack((py[..., 0::2].sin(), py[..., 1::2].cos()), dim=4).flatten(3)
        sine = torch.cat((py, px), dim=3).reshape(S, D)
        self.enc_pos = (sine + self.w["level_embed"][0].cpu()).to(self.dev).to(torch.bfloat16).contiguous()
        lin = torch.linspace(0.5, g - 0.5, g, dtype=torch.float32) / g
        ry, rx = torch.meshgrid(lin, lin, indexing="ij")
        self.enc_ref1 = torch.stack((rx.reshape(-1), ry.reshape(-1)), -1).to(self.dev).contiguous()  # [S,2]
        ctr = (torch.arange(g, dtype=torch.float32) + 0.5) / g
        gy, gx = torch.meshgrid(ctr, ctr, indexing="ij")
        prop = torch.stack([gx.reshape(-1), gy.reshape(-1), torch.full((S,), 0.05), torch.full((S,), 0.05)], -1)
        valid = ((prop > 0.01) & (prop < 0.99)).all(-1)
        self.prop_logit = torch.log(prop / (1 - prop)).masked_fill(~valid[:, None], float("inf")).to(self.dev).contiguous()
        self.prop_valid_all = bool(valid.all())
        self.prop_valid = valid.to(torch.uint8).to(self.dev)
        self.coord = {}
        for s in (g * 4, g * 2, g):
            self.coord[s] = torch.linspace(-1, 1, s).to(self.dev)
        self.rope_len = 0
        self.ensure_rope(cfg.max_pos)

    def ensure_rope(self, n: int):
        """cos/sin tables [n, head_dim/2] for positions < n.  Built for max_position_embeddings at load; a longer sequence
        rebuilds them (HF's LlamaRotaryEmbedding extends its cache the same way, $HF/models/llama/modeling_llama.py:96-113 in
        4.32) instead of letting rope_kv / the decode kernels index past the end.  New storage invalidates captured graphs
        (the capture key in GromaModel._capture includes the table pointer)."""
        if n <= self.rope_len:
            return
        cfg = self.cfg
        hd = cfg.head_dim
        n = max(n, cfg.max_pos, 2 * self.rope_len)
        inv = 1.0 / (cfg.rope_theta ** (torch.arange(0, hd, 2).float() / hd))
        fr = torch.outer(torch.arange(n).float(), inv)
        with torch.inference_mode(False):
            self.rope_cos, self.rope_sin = fr.cos().to(self.dev).contiguous(), fr.sin().to(self.dev).contiguous()
        self.rope_len = n

    def _stage(self, name, t):
        if self.keep_stages:
            self.stages[name] = t

    # ------------------------------------------------------------------------------------------ a1/a2 DINOv2
    def vit(self, images: torch.Tensor) -> List[torch.Tensor]:
        """$HF/models/dinov2/modeling_dinov2.py:57-149 (embeddings) and :348-387 x24 (layers); returns the hidden states
        Groma reads: the last four layer outputs (groma.py:222-224,240-241,312)."""
        cfg, w = self.cfg, self.w
        B = images.shape[0]
        H, nh = cfg.vit_hidden, cfg.vit_heads
        hd = H // nh
        NP = cfg.grid ** 2
        S = NP + 1
        patches = G.vit_patchify(images.to(self.dev, torch.float32), self.patch_ld)
        emb = G.gemm(patches, w["vit.patch.w"], bias=w["vit.patch.b"])
        x = G.vit_embed(emb, w["vit.cls"], w["vit.pos"], B, NP).reshape(B * S, H)
        hs = []
        keep_from = cfg.vit_layers - 4
        for i in range(cfg.vit_layers):
            o = f"vit.{i}."
            y = G.layernorm(x, w[o + "ln1.w"], w[o + "ln1.b"], cfg.vit_ln_eps)
            qkv = G.gemm(y, w[o + "qkv.w"], bias=w[o + "qkv.b"]).reshape(B, S, 3, nh, hd)
            attn = G.attention_tc if (self.use_tc_attention and hd in (64, 128)) else G.attention
            a = attn(qkv[:, :, 0], qkv[:, :, 1].permute(0, 2, 1, 3), qkv[:, :, 2].permute(0, 2, 1, 3),
                     causal=False, scale=1.0 / math.sqrt(hd))
            xn = torch.empty_like(x) if i >= keep_from else x   # keep the hidden states that are read later intact
            G.gemm(a.reshape(B * S, H), w[o + "o.w"], bias=w[o + "o.b"], gamma=w[o + "ls1"], residual=x, out=xn)
            x = xn
            y = G.layernorm(x, w[o + "ln2.w"], w[o + "ln2.b"], cfg.vit_ln_eps)
            h = G.gemm(y, w[o + "fc1.w"], bias=w[o + "fc1.b"], act=G.ACT_GELU)
            G.gemm(h, w[o + "fc2.w"], bias=w[o + "fc2.b"], gamma=w[o + "ls2"], residual=x, out=x)
            if i >= keep_from:
                hs.append(x.reshape(B, S, H))
        return hs

    # ------------------------------------------------------------------------------------------ a3 image tokens
    def image_tokens(self, last: torch.Tensor) -> torch.Tensor:
        """groma.py:227-237 (2x2 token merge) + img_txt_bridge (groma.py:112-116,361)."""
        B = last.shape[0]
        f = G.space_to_depth(last, self.cfg.grid)
        h = G.gemm(f.reshape(-1, f.shape[-1]), self.w["bridge0.w"], bias=self.w["bridge0.b"], act=G.ACT_GELU)
        return G.gemm(h, self.w["bridge2.w"], bias=self.w["bridge2.b"]).reshape(B, -1, self.cfg.llm_hidden)

    # ------------------------------------------------------------------------------------------ a4..a9 proposer
    def _msda(self, pfx: str, query: torch.Tensor, value_src: torch.Tensor, ref: torch.Tensor, B: int, Q: int):
        cfg, w = self.cfg, self.w
        g = cfg.grid
        proj = G.gemm(query, w[pfx + ".proj.w"], bias=w[pfx + ".proj.b"], out_f32=True)
        value = G.gemm(value_src, w[pfx + ".value.w"], bias=w[pfx + ".value.b"])
        return G.msda(value.reshape(B, g * g, cfg.ddetr_heads, 32), proj, ref, [(g, g)], cfg.ddetr_heads, cfg.n_points).reshape(B * Q, -1)

    def proposer(self, hs: List[torch.Tensor], n_extra: int = 0):
        """groma.py:240-249, ddetr.py:147-151, ddetr_transformer.py:484-609,668-728 (inference subset, SURVEY T4).
        Returns fp32 (pred_cxcywh [B,N,4], pred_xyxy [B,N,4], scores [B,N]) with N = num_queries + n_extra slots.

        The ~200 launches after the token mean are tiny (d_model 256): eager they are launch-bound (2.9 ms at B = 16), so they are
        captured once per (B, n_extra) into a CUDA graph that reads the mean from a static buffer and writes static outputs --
        valid until the next proposer() call of the same shape.  Parity runs that record stages / teacher-force the top-k go eager."""
        cfg = self.cfg
        B = hs[0].shape[0]
        if not self.graph_proposer or self.keep_stages or self.topk_override is not None or torch.cuda.is_current_stream_capturing():
            x = G.mean_tokens(hs[-4:], 1).reshape(B * cfg.grid * cfg.grid, -1)
            return self._proposer_body(x, B, n_extra)
        key = (B, n_extra)
        ent = self._prop_graphs.get(key)
        if ent is None:
            with torch.inference_mode(False):
                xbuf = torch.empty((B * cfg.grid * cfg.grid, cfg.vit_hidden), dtype=torch.bfloat16, device=self.dev)
            G.mean_tokens(hs[-4:], 1, out=xbuf.view(B, cfg.grid * cfg.grid, -1))
            st = torch.cuda.Stream()
            st.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(st):
                self._proposer_body(xbuf, B, n_extra)                 # warm-up: one-time kernel attribute setup happens outside capture
                gr = torch.cuda.CUDAGraph()
                l0 = G.LAUNCHES
                with torch.inference_mode(False), torch.cuda.graph(gr, stream=st, capture_error_mode="thread_local"):
                    outs = self._proposer_body(xbuf, B, n_extra)
                n_kernels = G.LAUNCHES - l0
            torch.cuda.current_stream().wait_stream(st)
            ent = self._prop_graphs[key] = (gr, xbuf, outs, n_kernels)
        gr, xbuf, outs, n_kernels = ent
        G.mean_tokens(hs[-4:], 1, out=xbuf.view(B, cfg.grid * cfg.grid, -1))
        gr.replay()
        G.LAUNCHES += n_kernels          # the launch counter bench.py reports counts replayed graph nodes too
        return outs

    def _proposer_body(self, x: torch.Tensor, B: int, n_extra: int):
        cfg, w = self.cfg, self.w
        g, D, Qn = cfg.grid, cfg.d_model, cfg.num_queries
        S = g * g
        src = G.gemm(x, w["inproj.w"], bias=w["inproj.b"])
        x = G.layernorm(src, w["inproj.ln.w"], w["inproj.ln.b"], 1e-6)
        self._stage("ddetr_src", x.reshape(B, S, D))
        enc_ref = self.enc_ref1[None].expand(B, S, 2).contiguous()
        for i in range(cfg.enc_layers):
            o = f"enc.{i}."
            q = G.add_bcast(x, self.enc_pos, S)
            samp = self._msda(o + "sa", q, x, enc_ref, B, S)
            h = G.gemm(samp, w[o + "sa.out.w"], bias=w[o + "sa.out.b"], residual=x)
            x = G.layernorm(h, w[o + "ln1.w"], w[o + "ln1.b"], 1e-5)
            t = G.gemm(x, w[o + "fc1.w"], bias=w[o + "fc1.b"], act=G.ACT_RELU)
            h = G.gemm(t, w[o + "fc2.w"], bias=w[o + "fc2.b"], residual=x)
            x = G.layernorm(h, w[o + "ln2.w"], w[o + "ln2.b"], 1e-5)
        memory = x
        self._stage("memory", memory.reshape(B, S, D))
        oq = memory
        if not self.prop_valid_all:
            oq = G.mask_rows(memory.clone().reshape(B, S, D), self.prop_valid).reshape(B * S, D)
        eo = G.layernorm(G.gemm(oq, w["enc_output.w"], bias=w["enc_output.b"]), w["enc_output_norm.w"], w["enc_output_norm.b"], 1e-5)
        cls = G.gemm(eo, w["cls_enc.w"], bias=w["cls_enc.b"], out_f32=True).reshape(B, S)
        L = cfg.dec_layers
        t = G.gemm(eo, w[f"bbox.{L}.0.w"], bias=w[f"bbox.{L}.0.b"], act=G.ACT_RELU)
        t = G.gemm(t, w[f"bbox.{L}.1.w"], bias=w[f"bbox.{L}.1.b"], act=G.ACT_RELU)
        delta = G.gemm(t, w[f"bbox.{L}.2.w"], bias=w[f"bbox.{L}.2.b"], out_f32=True).reshape(B, S, 4)
        topk = G.topk_desc(cls, Qn)
        self._stage("topk_own", topk)
        if self.topk_override is not None:
            # parity tests only: continue with the oracle's query selection so that everything downstream of the (tie-sensitive)
            # two-stage top-k is comparable query by query; the engine's own selection is kept in stages['topk_own']
            topk = self.topk_override.to(self.dev, torch.int64).contiguous()
        ref, pos512 = G.ddetr_select(delta, self.prop_logit, topk, D // 2)
        self._stage("enc_cls", cls); self._stage("topk", topk); self._stage("ref_init", ref)
        pt = G.layernorm(G.gemm(pos512.reshape(B * Qn, 2 * D), w["pos_trans.w"], bias=w["pos_trans.b"]),
                         w["pos_trans_norm.w"], w["pos_trans_norm.b"], 1e-5)
        query_pos = pt[:, :D].contiguous()
        h = w["query_tgt"][None].expand(B, Qn, D).reshape(B * Qn, D).contiguous()
        nH = cfg.ddetr_heads
        hd = D // nH
        keep = {}
        for i in range(L):
            o = f"dec.{i}."
            qk_in = G.add(h, query_pos)
            qk = G.gemm(qk_in, w[o + "qk.w"], bias=w[o + "qk.b"]).reshape(B, Qn, 2, nH, hd)
            v = G.gemm(h, w[o + "v.w"], bias=w[o + "v.b"]).reshape(B, Qn, nH, hd)
            a = G.attention(qk[:, :, 0], qk[:, :, 1].permute(0, 2, 1, 3), v.permute(0, 2, 1, 3), causal=False, scale=hd ** -0.5)
            t = G.gemm(a.reshape(B * Qn, D), w[o + "o.w"], bias=w[o + "o.b"], residual=h)
            h = G.layernorm(t, w[o + "ln1.w"], w[o + "ln1.b"], 1e-5)
            qc = G.add(h, query_pos)
            samp = self._msda(o + "ca", qc, memory, ref, B, Qn)
            t = G.gemm(samp, w[o + "ca.out.w"], bias=w[o + "ca.out.b"], residual=h)
            h = G.layernorm(t, w[o + "ln2.w"], w[o + "ln2.b"], 1e-5)
            t = G.gemm(h, w[o + "fc1.w"], bias=w[o + "fc1.b"], act=G.ACT_RELU)
            t = G.gemm(t, w[o + "fc2.w"], bias=w[o + "fc2.b"], residual=h)
            h = G.layernorm(t, w[o + "ln3.w"], w[o + "ln3.b"], 1e-5)
            keep[i] = h
        self._stage("dec_last", keep[L - 1].reshape(B, Qn, D))

        def bbox(i, hh):
            t = G.gemm(hh, w[f"bbox.{i}.0.w"], bias=w[f"bbox.{i}.0.b"], act=G.ACT_RELU)
            t = G.gemm(t, w[f"bbox.{i}.1.w"], bias=w[f"bbox.{i}.1.b"], act=G.ACT_RELU)
            return G.gemm(t, w[f"bbox.{i}.2.w"], bias=w[f"bbox.{i}.2.b"], out_f32=True)

        d5 = bbox(L - 1, keep[L - 1])
        d4 = bbox(L - 2, keep[L - 2]) if L >= 2 else torch.zeros_like(d5)
        coco = G.gemm(keep[L - 1], w["cls_coco.w"], bias=w["cls_coco.b"], out_f32=True)
        sa1b = G.gemm(keep[L - 1], w["cls_sa1b.w"], bias=w["cls_sa1b.b"], out_f32=True)
        N = Qn + n_extra
        pc = torch.zeros((B, N, 4), dtype=torch.float32, device=self.dev)
        px = torch.zeros((B, N, 4), dtype=torch.float32, device=self.dev)
        sc = torch.zeros((B, N), dtype=torch.float32, device=self.dev)
        G.ddetr_finalize(d4, d5, ref, coco, sa1b, pc, px, sc)
        return pc, px, sc, {"coco": coco.reshape(B, Qn, 1), "sa1b": sa1b.reshape(B, Qn, 1)}

    # ------------------------------------------------------------------------------------------ a10 region selection
    def select_regions(self, pc, px, sc, refer_boxes: Optional[Sequence[torch.Tensor]], ground_boxes: Optional[Sequence[torch.Tensor]],
                       nms_thres: float, score_thres: float, max_num: int, overlap=None) -> List[torch.Tensor]:
        """groma.py:251-280.  NMS for the whole batch in one device kernel; the only host sync of the vision stage is the
        read-back of keep indices.  torch.randperm stays on the global CPU RNG, one draw per image in image order (T6).
        `overlap`: a callable that enqueues GPU work which does not depend on the selection (the fusion convs of the region
        encoder).  It is called after the read-back copies are queued and before the host waits for them, so the GPU keeps
        running while the host reads the keep lists, draws the permutations and builds the RoI list."""
        cfg = self.cfg
        B, N = sc.shape
        Qn = cfg.num_queries
        counts = torch.full((B,), Qn, dtype=torch.int32)
        if refer_boxes is not None or ground_boxes is not None:
            for i in range(B):
                extra = []
                if refer_boxes is not None and len(refer_boxes[i]) > 0:
                    extra.append((refer_boxes[i].to(self.dev, torch.float32), 1.0))
                if ground_boxes is not None and len(ground_boxes[i]) > 0:
                    extra.append((ground_boxes[i].to(self.dev, torch.float32), 0.2))
                o = Qn
                for bx, s in extra:
                    n = bx.shape[0]
                    pc[i, o:o + n] = bx
                    px[i, o:o + n] = torch.cat([bx[:, :2] - 0.5 * bx[:, 2:], bx[:, :2] + 0.5 * bx[:, 2:]], -1)
                    sc[i, o:o + n] = s
                    o += n
                counts[i] = o
        keep, num, amax = G.nms_batched(px, sc, nms_thres, score_thres, max_num, counts=counts.to(self.dev))
        if overlap is None:
            keep_h, num_h, amax_h, pc_h = keep.cpu(), num.cpu(), amax.cpu(), pc.cpu()   # single sync point
        else:
            # read-back into pinned buffers + an event: the host waits for these four copies only, not for what `overlap` queues
            srcs = (keep, num, amax, pc)
            key = tuple((tuple(t.shape), t.dtype) for t in srcs)
            if getattr(self, "_sel_pinned_key", None) != key:
                with torch.inference_mode(False):      # persistent buffers: ordinary tensors even under a caller's inference_mode()
                    self._sel_pinned = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in srcs]
                self._sel_pinned_key = key
            for dst, src in zip(self._sel_pinned, srcs):
                dst.copy_(src, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            # multi-rank: replayed_randperms all-gathers the keep counts on this stream right after the read-back; queue the
            # overlapped work behind those (tiny) collectives, not in front of them
            import torch.distributed as _dist
            overlap_late = _dist.is_available() and _dist.is_initialized() and _dist.get_world_size() > 1
            if not overlap_late:
                overlap()
            ev.synchronize()
            keep_h, num_h, amax_h, pc_h = (t.clone() for t in self._sel_pinned)
        self._stage("nms_keep", keep_h); self._stage("nms_num", num_h)
        from .dist import replayed_randperms
        perms = replayed_randperms([int(n) for n in num_h])   # == [torch.randperm(n)] in a single process
        if overlap is not None and overlap_late:
            overlap()
        selected = []
        for i in range(B):
            n = int(num_h[i])
            if n > 0:
                bx = pc_h[i][keep_h[i, :n]]
                bx = bx[perms[i]]
            else:
                mi = int(amax_h[i])
                bx = pc_h[i][mi:mi + 1]
            selected.append(bx)
        return selected

    # ------------------------------------------------------------------------------------------ a12/a13 region encoder
    def region_encoder(self, hs: List[torch.Tensor], boxes: Sequence[torch.Tensor]) -> torch.Tensor:
        """groma/model/roi_align.py:215-228 (upsample), :97-193 (MLVLFuseModule), :274-327 (MlvlRoIExtractor).
        boxes: per-image [R_i,4] cxcywh (host or device).  Returns region features [sum R, llm_hidden] bf16.
        = region_tokens(region_maps(hs), boxes); GromaModel calls the halves separately so that the maps (which do not depend on
        the selected boxes) are already being computed while the host reads the NMS result back."""
        return self.region_tokens(self.region_maps(hs), boxes)

    def region_maps(self, hs: List[torch.Tensor]) -> List[torch.Tensor]:
        """The box-independent part: upsample + coord channels + 1x1 input convs (roi_align.py:215-228,118-126) and the fusion
        rounds of MLVLFuseModule (:180-193).  Returns the three fused NHWC maps [B, s, s, C], s = 4g, 2g, g."""
        cfg, w = self.cfg, self.w
        g, C = cfg.grid, cfg.vit_hidden
        B = hs[0].shape[0]
        sizes = [g * 4, g * 2, g]
        xs = []
        for l in range(3):
            s = sizes[l]
            up = G.upsample_coords(hs[len(hs) - 3 + l], 1, g, s, s, self.in_ld, self.coord[s], self.coord[s])
            xs.append(G.gemm(up.reshape(-1, self.in_ld), w[f"inconv.{l}.w"], bias=w[f"inconv.{l}.b"]).reshape(B, s, s, C))
        # Between fusion rounds the maps stay RAW conv outputs + GroupNorm statistics: the next round's shuffle applies norm + ReLU
        # tap by tap (bit-identical to apply -> store -> shuffle, tests/test_ops_gpu.py), which drops one read + one write of every
        # map per round; only the last round's maps are materialised for RoIAlign.  GROMA_FUSE_GN=0: the three-kernel form.
        st = None                                       # per-level statistics of the maps in xs (None = xs is already activated)
        for k in range(cfg.fuse_rounds):
            new, new_st = [], []
            last = k == cfg.fuse_rounds - 1
            for l in range(3):
                s = sizes[l]
                t, d = min(l + 1, 2), max(l - 1, 0)
                if st is None:
                    xin = G.fuse_shuffle(xs[l], xs[t], xs[d])
                else:
                    xin = G.fuse_shuffle_gn(xs[l], xs[t], xs[d], st[l], st[t], st[d], w[f"fuse.{k - 1}.gn.w"], w[f"fuse.{k - 1}.gn.b"],
                                            cfg.gn_groups)
                y = G.conv3x3_flat(xin.reshape(-1, C), w[f"fuse.{k}.w"], B, s + 2, s + 2, block_n=512 if (self.use_2cta and C >= 512) else 0)
                if self.fuse_gn_apply and not last:
                    new_st.append(G.groupnorm_stats(y, cfg.gn_groups, 1e-5, B))
                    new.append(y.reshape(B, s, s, C))
                else:
                    new.append(G.groupnorm_relu(y, w[f"fuse.{k}.gn.w"], w[f"fuse.{k}.gn.b"], cfg.gn_groups, 1e-5, B, out=y).reshape(B, s, s, C))
            xs, st = new, (new_st if (self.fuse_gn_apply and not last) else None)
        if self.keep_stages:
            self.stages["fused_maps"] = xs
        return xs

    def region_tokens(self, xs: List[torch.Tensor], boxes: Sequence[torch.Tensor]) -> torch.Tensor:
        """MlvlRoIExtractor.forward (roi_align.py:274-327) on the fused maps of region_maps: RoIAlign x3 -> pconvs -> sum -> ReLU ->
        flatten_linear + box position MLP -> updims."""
        cfg, w = self.cfg, self.w
        C = cfg.vit_hidden
        allb = torch.cat([b.float() for b in boxes]).to(self.dev)
        K = allb.shape[0]
        if K == 0:
            return torch.zeros((0, cfg.llm_hidden), dtype=torch.bfloat16, device=self.dev)
        img_id = torch.cat([torch.full((len(b), 1), float(i)) for i, b in enumerate(boxes)]).to(self.dev)
        rois = torch.cat([img_id, allb * float(cfg.image_size)], 1).contiguous()    # cxcywh*448 fed as xyxy (T1)
        ro = cfg.roi_out
        rp = ro + 2
        rbuf = torch.empty((3, K, rp, rp, C), dtype=torch.bfloat16, device=self.dev)
        for l in range(3):
            G.roi_align(xs[l], rois, ro, (8, 4, 2)[l] / 14.0, cfg.roi_sampling, True, pad=True, out=rbuf[l])
        fused = G.conv3x3_flat(rbuf.reshape(-1, C), w["pconv.w"], K, rp, rp, bias=w["pconv.b"], act=G.ACT_RELU,
                               block_n=512 if (self.use_2cta and C >= 512 and K * rp * rp >= 2048) else 0)  # [K*ro*ro, C]
        self._stage("roi_fused", fused.reshape(K, ro, ro, C))
        flat_in = fused.reshape(K, ro * ro * C)
        kt = flat_in.shape[1]
        split = max(1, min(16, (self.sms * 2) // (((K + 127) // 128) * max(1, w["flatten.w"].shape[0] // 128))))
        split = min(split, max(1, kt // 1024))
        flat = G.gemm_splitk(flat_in, w["flatten.w"], split, bias=w["flatten.b"])
        self._stage("region_flat", flat)
        p = G.linear_smallk(allb, w["pos0.w"], w["pos0.b"], True)
        p = G.layernorm(p, w["pos2.w"], w["pos2.b"], 1e-5)
        p = G.gemm(p, w["pos3.w"], bias=w["pos3.b"], act=G.ACT_RELU)
        p = G.layernorm(p, w["pos5.w"], w["pos5.b"], 1e-5)
        z = G.add(flat, p)
        return G.gemm(z, w["updims.w"], bias=w["updims.b"])

    # ------------------------------------------------------------------------------------------ a15 embedding + splice
    def embed(self, ids: torch.Tensor) -> torch.Tensor:
        """groma.py:165-174: ids < vocab -> llm.embed_tokens, else new_input_embs[id - vocab]."""
        flat = ids.reshape(-1).to(self.dev, torch.int64).contiguous()
        return G.gather_rows(flat, self.w["embed"], self.w["new_embed"], self.cfg.vocab)

    # ------------------------------------------------------------------------------------------ a16/a17 LLaMA
    @property
    def kv_fp8(self) -> bool:
        return self.kv_dtype == torch.float8_e4m3fn

    def _kv_cap(self, cap: int) -> int:
        # fp8: the decode kernels copy scales in 16-byte units of 4 positions, which must not cross a (b, h) row
        return -(-cap // 4) * 4 if self.kv_fp8 else cap

    def _new_kv(self, shape):
        # persistent buffers are ordinary tensors even when the caller runs under torch.inference_mode()
        # (eval/run_groma.py:81): later calls outside it update them in place
        with torch.inference_mode(False):
            kv = torch.zeros(shape, dtype=self.kv_dtype, device=self.dev)
            sc = torch.zeros(shape[:-1], dtype=torch.float32, device=self.dev) if self.kv_fp8 else None
        return kv, sc

    def drop_kv(self):
        """Free the cache (and with it any fp8 mirror); the next prefill allocates a new one."""
        self.kv = self.kv_scale = self.kv_mirror = None
        self.kv_mirror_len = 0

    def alloc_kv(self, B: int, cap: int):
        cfg = self.cfg
        cap = self._kv_cap(cap)
        shape = (cfg.llm_layers, 2, B, cfg.llm_heads, cap, cfg.head_dim)
        if self.kv is None or tuple(self.kv.shape) != shape or self.kv.dtype != self.kv_dtype:
            self.drop_kv()
            self.kv, self.kv_scale = self._new_kv(shape)
        self.kv_mirror_len = 0           # the prefill rewrites every position
        self.kv_cap = cap

    def grow_kv(self, cap: int):
        """Re-home the cache with room for `cap` positions, keeping the first `past` of every (layer, k/v, row, head) -- fp8 codes
        and their scales alike."""
        old, old_sc, past = self.kv, self.kv_scale, self.past
        cap = self._kv_cap(cap)
        L, _, B, H, _, D = old.shape
        new, new_sc = self._new_kv((L, 2, B, H, cap, D))
        new[:, :, :, :, :past].copy_(old[:, :, :, :, :past])
        if new_sc is not None:
            new_sc[:, :, :, :, :past].copy_(old_sc[:, :, :, :, :past])
        self.kv, self.kv_scale, self.kv_cap = new, new_sc, cap

    def kv_bytes(self) -> int:
        """Device bytes of the KV caches: bf16 rows, or fp8 codes + fp32 scales, plus the prefix and row caches of a grouped
        generate() (group_buffers) while they are held."""
        n = 0 if self.kv is None else self.kv.numel() * self.kv.element_size()
        n += self.kv_scale.numel() * 4 if self.kv_scale is not None else 0
        g = getattr(self, "_group", None)
        if g is not None:
            n += (g["prefix"].numel() + g["row"].numel()) * 2
        return n

    def kv_layer(self, i: int):
        """(k, v, k scales, v scales) of layer i; the scales are None for a bf16 cache."""
        if self.kv_scale is None:
            return self.kv[i, 0], self.kv[i, 1], None, None
        return self.kv[i, 0], self.kv[i, 1], self.kv_scale[i, 0], self.kv_scale[i, 1]

    def kv_dequantized(self, ctx: int) -> torch.Tensor:
        """fp8: a new bf16 tensor [layer, k/v, B, H, ctx, D] holding bf16_rn(x^) of the first ctx positions (one launch)."""
        return G.kv_dequantize(self.kv, self.kv_scale, rows=ctx)

    def kv_mirror_sync(self, ctx: int) -> torch.Tensor:
        """fp8: bf16 view [layer, k/v, B, H, ctx, D] of an incrementally kept copy of the dequantised cache, for callers that take
        the cache after every step (forward(use_cache=True)): only positions the mirror does not hold yet are dequantised, so
        a step costs O(new rows).  It has the cache's capacity and is re-homed (one full copy) when the cache grows."""
        m = self.kv_mirror
        if m is None or m.shape[:4] != self.kv.shape[:4] or m.shape[4] < ctx:
            with torch.inference_mode(False):
                new = torch.empty(self.kv.shape, dtype=torch.bfloat16, device=self.dev)
            n = self.kv_mirror_len if m is not None and m.shape[:4] == self.kv.shape[:4] else 0
            if n:
                new[:, :, :, :, :n].copy_(m[:, :, :, :, :n])
            self.kv_mirror, self.kv_mirror_len = new, n
        n = self.kv_mirror_len
        if ctx > n:
            G.kv_dequantize(self.kv[:, :, :, :, n:], self.kv_scale[:, :, :, :, n:], out=self.kv_mirror[:, :, :, :, n:], rows=ctx - n)
            self.kv_mirror_len = ctx
        return self.kv_mirror[:, :, :, :, :ctx]

    def llm_prefill(self, x: torch.Tensor, B: int, T: int, kv_len: torch.Tensor, last_only: bool = False) -> torch.Tensor:
        """$HF/models/llama/modeling_llama.py LlamaModel forward (32 x LlamaDecoderLayer :292-340) + both heads
        (groma.py:399-402).  x [B*T, hidden] bf16 (consumed), kv_len int32 [B] = valid (non-pad) length per row."""
        cfg = self.cfg
        nh, hd = cfg.llm_heads, cfg.head_dim
        if self.kv_fp8:
            # the prefill attends over the bf16 K/V it computes (a per-layer staging buffer); groma_kv_quantize then writes them
            # into the fp8 cache
            stage = torch.empty((2, B, nh, T, hd), dtype=torch.bfloat16, device=self.dev)
            self._prefill_layers(x, B, T, kv_len, lambda i: (stage[0], stage[1]),
                                 written=lambda i: G.kv_quantize(stage, self.kv[i], self.kv_scale[i]))
        else:
            self._prefill_layers(x, B, T, kv_len, lambda i: (self.kv[i, 0], self.kv[i, 1]))
        self.past = T
        return self._prefill_head(x, B, T, last_only)

    def _prefill_head(self, x: torch.Tensor, B: int, T: int, last_only: bool) -> torch.Tensor:
        if last_only:
            x = x.reshape(B, T, -1)[:, -1].contiguous()
        h = G.rmsnorm(x, self.w["llm.norm"], self.cfg.rms_eps)
        return G.gemm(h, self._wp("head.w"), out_f32=True)

    def _prefill_layers(self, x: torch.Tensor, B: int, T: int, kv_len: torch.Tensor, kv_at, pos0: int = 0, written=None):
        """The decoder layers over x [B*T, hidden] (updated in place) at positions pos0 .. pos0 + T - 1.  kv_at(i) gives layer i's
        (k, v) [B, H, >= pos0 + T, D]: the rotated K/V are written at pos0 + t and the queries attend causally over positions
        [0, pos0 + T) of it, keys at or past kv_len[b] masked.  written(i), if given, runs after layer i's attention."""
        cfg, w = self.cfg, self.w
        nh, hd = cfg.llm_heads, cfg.head_dim
        q = torch.empty((B * T, nh * hd), dtype=torch.bfloat16, device=self.dev)
        # two-CTA cluster (256x256 tiles per CTA pair, B tile multicast) for the big projections; the 22016-wide
        # gate/up projection keeps the 128x256 tile
        bn2 = 512 if (self.use_2cta and B * T >= 2048 and cfg.llm_hidden >= 2048) else 0
        # RoPE + KV append in the qkv GEMM epilogue (one launch, no [B*T, 3*hidden] intermediate) whenever the 256-wide tile
        # applies: head_dim 128 and enough rows to fill the SMs; tiny test configs keep gemm + rope_kv (same values)
        # (fp8 weights: no fused form -- two accumulator sets do not fit the 256-wide tile's registers)
        fused_rope = self.use_fused_rope and hd == 128 and nh % 2 == 0 and (bn2 == 512 or B * T >= 1024) and not self.fp8
        for i in range(cfg.llm_layers):
            o = f"llm.{i}."
            y = G.rmsnorm(x, w[o + "ln1"], cfg.rms_eps)
            kc, vc = kv_at(i)
            if fused_rope:
                G.gemm_qkv_rope(y, self._wp(o + "qkv.w"), q, kc, vc, self.rope_cos, self.rope_sin, B, T, nh, hd, pos0,
                                block_n=bn2 or 256)
            else:
                qkv = self._proj(y, o + "qkv.w", block_n=bn2)
                G.rope_kv(qkv, q, kc, vc, self.rope_cos, self.rope_sin, B, T, nh, hd, pos0)
            attn = G.attention_tc if (self.use_tc_attention and hd in (64, 128)) else G.attention
            a = attn(q.reshape(B, T, nh, hd), kc, vc, causal=True, scale=1.0 / math.sqrt(hd), q_pos0=pos0, kv_len=kv_len,
                     sk=pos0 + T)
            if written is not None:
                written(i)
            self._proj(a.reshape(B * T, nh * hd), o + "o.w", residual=x, out=x, block_n=bn2)
            y = G.rmsnorm(x, w[o + "ln2"], cfg.rms_eps)
            gu = self._proj(y, o + "gu.w", act=G.ACT_SWIGLU)
            self._proj(gu, o + "down.w", residual=x, out=x, block_n=bn2)

    # ------------------------------------------------------------------------------------------ prompt groups
    def group_buffers(self, B: int, n: int, P: int, T: int, max_new: int):
        """Caches of a grouped generate() over B images x n prompts (decode_step(group=...), include/groma_b200.h:
        groma_decode_rope_attention_grouped): prefix [layer, k/v, B, H, P, D], the K/V of the P positions the rows of an image
        share, and row [layer, k/v, B*n, H, T - P + max_new, D], each row's own positions (position p at index p - P), both
        bf16.  They live apart from the plain cache `kv`; kept while the shapes are unchanged, so that a captured grouped step
        stays valid across calls; a plain or beam generate() frees them (drop_group)."""
        cfg = self.cfg
        L, H, D = cfg.llm_layers, cfg.llm_heads, cfg.head_dim
        rcap = T - P + max_new
        st = getattr(self, "_group", None)
        if st is not None and (st["B"], st["n"], st["P"], st["row"].shape[4]) == (B, n, P, rcap):
            return st
        self._group = st = None
        with torch.inference_mode(False):
            st = dict(B=B, n=n, P=P,
                      prefix=torch.zeros((L, 2, B, H, P, D), dtype=torch.bfloat16, device=self.dev),
                      row=torch.zeros((L, 2, B * n, H, rcap, D), dtype=torch.bfloat16, device=self.dev))
        self._group = st
        return st

    def drop_group(self) -> bool:
        """Free the caches of a grouped generate(); True if there were any."""
        had = getattr(self, "_group", None) is not None
        self._group = None
        return had

    def llm_prefill_grouped(self, x: torch.Tensor, st: dict, T: int, kv_len: torch.Tensor) -> torch.Tensor:
        """The prefill of B images x n prompts whose assembled rows (x [B*n*T, hidden], rows of an image consecutive) agree on
        their first P = st['P'] positions: the first row of each image runs positions [0, P) into st['prefix']; then every row
        runs [P, T), attending to its image's prefix and its own positions through a per-layer staging buffer [B*n, H, T, D],
        whose positions [P, T) go to st['row'].  kv_len int32 [B*n].  Returns fp32 logits [B*n, V] at the last position."""
        cfg = self.cfg
        B, n, P = st["B"], st["n"], st["P"]
        R, nh, hd = B * n, cfg.llm_heads, cfg.head_dim
        xr = x.view(B, n, T, -1)
        if P > 0:
            xp = xr[:, 0, :P].reshape(B * P, -1).contiguous()
            kvl = kv_len.view(B, n)[:, 0].contiguous()
            self._prefill_layers(xp, B, P, kvl, lambda i: (st["prefix"][i, 0], st["prefix"][i, 1]))
        xs = xr[:, :, P:].reshape(R * (T - P), -1).contiguous()
        stage = torch.empty((2, R, nh, T, hd), dtype=torch.bfloat16, device=self.dev)

        def kv_at(i):
            if P > 0:
                stage.view(2, B, n, nh, T, hd)[:, :, :, :, :P].copy_(st["prefix"][i].unsqueeze(2))
            return stage[0], stage[1]

        def written(i):
            st["row"][i][:, :, :, :T - P].copy_(stage[:, :, :, P:])
        self._prefill_layers(xs, R, T - P, kv_len, kv_at, pos0=P, written=written)
        self.past = T
        return self._prefill_head(xs, R, T - P, last_only=True)

    def _decode_buffers(self, B: int):
        cfg = self.cfg
        Hd, I, V = cfg.llm_hidden, cfg.llm_inter, cfg.vocab + cfg.num_new_token
        key = (B,)
        if getattr(self, "_dbuf_key", None) == key:
            return self._dbuf
        with torch.inference_mode(False):
            d = self._new_decode_buffers(B, Hd, I, V)
            if self.fp8:   # quantised input rows of the step's fp8 GEMMs
                d["xq"] = torch.empty((B * max(Hd, I),), dtype=torch.float8_e4m3fn, device=self.dev)
                d["xs"] = torch.empty((B,), dtype=torch.float32, device=self.dev)
        self._dbuf, self._dbuf_key = d, key
        return d

    def _new_decode_buffers(self, B, Hd, I, V):
        d = dict(
            ids=torch.zeros((B,), dtype=torch.int64, device=self.dev),
            x=torch.empty((B, Hd), dtype=torch.bfloat16, device=self.dev),
            y=torch.empty((B, Hd), dtype=torch.bfloat16, device=self.dev),
            qkv=torch.empty((B, 3 * Hd), dtype=torch.bfloat16, device=self.dev),
            q=torch.empty((B, Hd), dtype=torch.bfloat16, device=self.dev),
            a=torch.empty((B, 1, Hd), dtype=torch.bfloat16, device=self.dev),
            gu=torch.empty((B, I), dtype=torch.bfloat16, device=self.dev),
            ws=torch.empty((16 * max(3 * Hd, 2 * I, V) * B,), dtype=torch.float32, device=self.dev),
            logits=torch.empty((B, V), dtype=torch.float32, device=self.dev),
            pos=torch.zeros((1,), dtype=torch.int32, device=self.dev),
            cnt=torch.zeros((1024,), dtype=torch.int32, device=self.dev),   # split-K tile counters (self re-arming)
            kv_len=torch.zeros((B,), dtype=torch.int32, device=self.dev),
            # sampling step (decode_step(sample=True)): GromaSampleParams and the Philox seed; the Philox step is *pos
            sample_params=G.sample_params(1.0, 0, 1.0, device=self.dev),
            seed=torch.zeros((1,), dtype=torch.int64, device=self.dev),
        )
        return d

    # ------------------------------------------------------------------------------------------ persistent decode step
    def mega_supported(self, B: int) -> bool:
        cfg = self.cfg
        return (cfg.head_dim == 128 and B <= 16 and cfg.llm_hidden % 128 == 0 and cfg.llm_inter % 64 == 0 and
                (2 * cfg.llm_inter) % 128 == 0 and cfg.llm_hidden <= 8192)

    def _mega_state(self, B: int):
        """Scratch + argument block of groma_decode_step_fused for batch B (allocated once per B)."""
        st = getattr(self, "_mk", None)
        if st is not None and st["B"] == B:
            return st
        cfg = self.cfg
        L, H, Hd, I, V = cfg.llm_layers, cfg.llm_heads, cfg.llm_hidden, cfg.llm_inter, cfg.vocab + cfg.num_new_token
        n_flags, ws_tile, part, _ = G.decode_step_layout(L, B, H, Hd, I, V)
        sms = torch.cuda.get_device_properties(self.dev).multi_processor_count
        # every CTA needs at least one (row tile, k-block) unit of every projection (contributors of a tile are consecutive CTAs)
        units = min(3 * Hd // 128 * (Hd // 64), Hd // 128 * (Hd // 64), 2 * I // 128 * (Hd // 64), Hd // 128 * (I // 64), (V + 127) // 128 * (Hd // 64))
        grid = max(1, min(sms, units, int(os.environ.get("GROMA_MEGA_GRID", "100000"))))
        s_att = max(1, min(32, -(-int(os.environ.get("GROMA_MEGA_ITEMS_PER_CTA", "4")) * grid // (B * H))))
        f32 = lambda n: torch.empty((n,), dtype=torch.float32, device=self.dev)
        with torch.inference_mode(False):
            st = dict(B=B, grid=grid, s_att=s_att,
                      y2=torch.empty((B, Hd), dtype=torch.bfloat16, device=self.dev),
                      ws_qkv=f32(3 * Hd // 128 * ws_tile), ws_o=f32(Hd // 128 * ws_tile), ws_gu=f32(2 * I // 128 * ws_tile),
                      ws_down=f32(Hd // 128 * ws_tile), ws_head=f32((V + 127) // 128 * ws_tile),
                      att_part=f32(B * H * s_att * part), cand_val=f32((V + 127) // 128 * 16),
                      cand_idx=torch.empty(((V + 127) // 128 * 16,), dtype=torch.int32, device=self.dev),
                      flags=torch.zeros((n_flags,), dtype=torch.int32, device=self.dev),
                      status=torch.zeros((8 + 16 * sms,), dtype=torch.int32, device=self.dev), timeline=None)
        self._mk = st
        return st

    def decode_step_mega(self, B: int) -> torch.Tensor:
        """The same greedy step as decode_step() in ONE persistent kernel (csrc/decode_megakernel.cu): reads d['ids'], *pos,
        kv_len; appends K/V; writes d['logits'], the next ids, and advances pos / kv_len.  CUDA-graph capturable (the flag
        reset is a fill on the same stream)."""
        cfg, w = self.cfg, self.w
        d = self._decode_buffers(B)
        st = self._mega_state(B)
        a = G.DecodeStepArgs()
        a.L, a.B, a.H, a.Hd, a.I, a.V = cfg.llm_layers, B, cfg.llm_heads, cfg.llm_hidden, cfg.llm_inter, cfg.vocab + cfg.num_new_token
        a.vocab, a.S_att, a.cap = cfg.vocab, st["s_att"], self.kv_cap
        a.scale, a.eps = 1.0 / math.sqrt(cfg.head_dim), cfg.rms_eps
        ptr = lambda t: t.data_ptr()
        a.w_arena, a.w_down, a.embed, a.new_embed, a.ln_w = ptr(self.llm_arena), ptr(self.llm_down), ptr(w["embed"]), ptr(w["new_embed"]), ptr(self.llm_ln)
        a.kv, a.rope_cos, a.rope_sin = ptr(self.kv), ptr(self.rope_cos), ptr(self.rope_sin)
        a.ids, a.pos, a.kv_len = ptr(d["ids"]), ptr(d["pos"]), ptr(d["kv_len"])
        a.x, a.y_attn, a.y_mlp, a.a, a.gu, a.logits = ptr(d["x"]), ptr(d["y"]), ptr(st["y2"]), ptr(d["a"]), ptr(d["gu"]), ptr(d["logits"])
        for k in ("ws_qkv", "ws_o", "ws_gu", "ws_down", "ws_head", "att_part", "cand_val", "cand_idx", "flags", "status"):
            setattr(a, k, ptr(st[k]))
        a.grid = st["grid"]
        a.l2_prefetch_slots = int(os.environ.get("GROMA_MEGA_PREFETCH", "0"))
        a.timeline = st["timeline"].data_ptr() if st["timeline"] is not None else None
        if tuple(self.kv.shape[2:4]) != (B, cfg.llm_heads):
            raise RuntimeError("KV cache was allocated for a different batch")
        st["flags"].zero_()
        G.decode_step_fused(a)
        return d["logits"]

    def check_decode_status(self):
        """Raise if a dependency wait of the persistent decode kernel timed out (one device->host read; call outside graphs)."""
        st = getattr(self, "_mk", None)
        if st is None:
            return
        s = st["status"].cpu().tolist()
        if s[0] != 0:
            st["status"].zero_()
            from collections import Counter
            roles = ("stream-loader", "mma", "worker", "activation-loader")
            parked = Counter((roles[r], s[8 + (c * 4 + r) * 4], s[8 + (c * 4 + r) * 4 + 1] if os.environ.get("GROMA_MEGA_DEBUG") else 0)
                             for c in range(st["grid"]) for r in range(4) if s[8 + (c * 4 + r) * 4] != 0)
            detail = ""
            if os.environ.get("GROMA_MEGA_DEBUG"):
                detail = "\n" + "\n".join(f"cta {c} {roles[r]}: {s[8 + (c * 4 + r) * 4: 12 + (c * 4 + r) * 4]}" for c in range(st["grid"]) for r in range(4)
                                          if s[8 + (c * 4 + r) * 4] != 0)
            raise G._lib.GromaError(f"persistent decode kernel aborted: code {s[0]} (cta {s[1]}, role {roles[s[2]]}, thread {s[3]}, info {s[4:7]}); "
                                    f"parked waits (role, code, info): {sorted(parked.items(), key=lambda kv: -kv[1])[:12]}{detail}")

    def _decode_splits(self):
        """Split-K factors of the five decode GEMMs: (weight row-tiles of 128) x split should fill whole waves of the
        CTA slots (2 per SM)."""
        if getattr(self, "_splits", None) is None:
            cfg = self.cfg

            ncta = self.sms * max(1, int(os.environ.get("GROMA_GEMM_CTAS_PER_SM", "2")))   # the BN=16 kernel runs 2 CTAs per SM

            def pick(n_rows, k):
                tiles = (n_rows + 127) // 128
                kb = (k + 63) // 64
                best, best_eff = 1, 0.0
                for s in range(1, 17):
                    if s > kb:
                        break
                    per = (kb + s - 1) // s
                    s_eff = (kb + per - 1) // per          # splits that actually receive work
                    items = tiles * s_eff
                    waves = (items + ncta - 1) // ncta
                    eff = (tiles * kb) / (waves * ncta * per) - 0.004 * s   # small penalty: more fp32 partials to reduce
                    if eff > best_eff:
                        best, best_eff = s, eff
                return best
            Hd, I, V = cfg.llm_hidden, cfg.llm_inter, cfg.vocab + cfg.num_new_token
            self._splits = dict(qkv=pick(3 * Hd, Hd), o=pick(Hd, Hd), gu=pick(2 * I, Hd), down=pick(Hd, I), head=pick(V, Hd))
        return self._splits

    def _swap_gemm(self, x, wname, d, split, out, act=G.ACT_NONE, residual=None):
        """out[B, N] = epilogue(x[B,K] @ W[N,K]^T) through the swap-AB wgmma path (weights stream once)."""
        B = x.shape[0]
        if wname in self.q8:
            c, sc = self.q8[wname]
            N = c.shape[0]
            ws = d["ws"][: split * N * B].view(split, N, B)
            xq, xs = G.fp8_quantize_rows(x, d["xq"][: x.numel()].view(x.shape), d["xs"])
            if self.fused_splitk:
                return G.gemm_fp8_swap_ab_fused(xq, xs, c, sc, ws, d["cnt"], split, out, act=act, residual=residual)
            G.gemm_fp8_swap_ab(xq, xs, c, sc, ws, split_k=split)
            n_out = N // 2 if act == G.ACT_SWIGLU else N
            G.splitk_reduce(ws, out, act=act, residual=residual, bias_along_m=True, ld_m=1, ld_n=n_out)
            return out
        if self.nf4:
            if self.fused_splitk:
                raise G._lib.GromaError("the fused split-K decode GEMM has no NF4 form")
            c, a, N, _ = self.q4[wname]
            ws = d["ws"][: split * N * B].view(split, N, B)
            if self.timing_hook is not None:
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
            G.gemm_nf4_swap_ab(x, c, a, N, ws, split_k=split)
            if self.timing_hook is not None:
                ev1.record()
                self.timing_hook.append((ev0, ev1, c.numel() + a.numel() * 4 + x.numel() * 2 + ws.numel() * 4))
            n_out = N // 2 if act == G.ACT_SWIGLU else N
            G.splitk_reduce(ws, out, act=act, residual=residual, bias_along_m=True, ld_m=1, ld_n=n_out)
            return out
        W = self.w[wname]
        N = W.shape[0]
        ws = d["ws"][: split * N * B].view(split, N, B)
        if self.timing_hook is not None:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        if self.fused_splitk:
            # one launch: the CTA finishing a tile last reduces the partials (measured SLOWER at decode tile sizes: the
            # per-tile release fence + atomic sit on the epilogue's critical path; kept for larger-K uses, off by default)
            G.gemm_swap_ab_fused(x, W, ws, d["cnt"], split, out, act=act, residual=residual)
        else:
            G.gemm_swap_ab(x, W, ws, split_k=split)
        if self.timing_hook is not None:
            ev1.record()
            self.timing_hook.append((ev0, ev1, W.numel() * 2 + x.numel() * 2 + ws.numel() * 4))
        if not self.fused_splitk:
            n_out = N // 2 if act == G.ACT_SWIGLU else N
            G.splitk_reduce(ws, out, act=act, residual=residual, bias_along_m=True, ld_m=1, ld_n=n_out)
        return out

    def _tiled(self, wname: str) -> torch.Tensor:
        """Tile-major copy of a decode weight (every 128x64 TMA box = one contiguous 16 KB run of HBM); built on first use."""
        t = self._wt.get(wname)
        if t is None:
            t = self._wt[wname] = G.tile_weight(self.w[wname])
        return t

    def process_buffers(self, B: int, history_cap: int, params_words: int):
        """Device state of a processing step (decode_step(process=True)) in the decode buffers of batch B: d['hist'] int32
        [B, >= history_cap] with its length d['hist_len'], the GromaProcessParams block d['proc_params'] (>= params_words), the
        processed scores d['scores'] and GromaSampleParamsEx d['sample_params_ex'].  Grown, never shrunk, so a captured step
        keeps its buffers across calls whose sizes fit."""
        d = self._decode_buffers(B)
        V = d["logits"].shape[1]
        with torch.inference_mode(False):
            if "hist" not in d or d["hist"].shape[1] < history_cap:
                d["hist"] = torch.zeros((B, history_cap), dtype=torch.int32, device=self.dev)
            if "proc_params" not in d or d["proc_params"].numel() < params_words:
                d["proc_params"] = torch.zeros((max(params_words, 64),), dtype=torch.int32, device=self.dev)
            if "scores" not in d:
                d["scores"] = torch.empty((B, V), dtype=torch.float32, device=self.dev)
                d["hist_len"] = torch.zeros((1,), dtype=torch.int32, device=self.dev)
                d["sample_params_ex"] = G.sample_params_ex(1.0, 0, 1.0, device=self.dev)
        return d

    def beam_buffers(self, B: int, nb: int, max_new: int, hist_cap: int):
        """Device state of a beam search over B images x nb beams (decode_step(beam=...), include/groma_b200.h:
        groma_beam_select): the beam cache kv [layer, k/v, B*nb, H, max_new, D] bf16 with its ancestry table src, the token
        history (what the processors read), the scorer state and the hypothesis store.  Kept while (B, nb) and the sizes fit, so
        a captured beam step stays valid across beam generate() calls; a greedy or sampled generate() frees it (drop_beam)."""
        st = getattr(self, "_beam", None)
        if (st is not None and (st["B"], st["nb"]) == (B, nb) and st["src"].shape[1] >= max_new and st["hist"].shape[1] >= hist_cap):
            return st
        self._beam = st = None
        cfg = self.cfg
        R, V = B * nb, cfg.vocab + cfg.num_new_token
        dev = self.dev
        i32 = lambda *sh: torch.zeros(sh, dtype=torch.int32, device=dev)
        f32 = lambda *sh: torch.zeros(sh, dtype=torch.float32, device=dev)
        f64 = lambda *sh: torch.zeros(sh, dtype=torch.float64, device=dev)
        with torch.inference_mode(False):
            st = dict(B=B, nb=nb, kv=torch.zeros((cfg.llm_layers, 2, R, cfg.llm_heads, max_new, cfg.head_dim), dtype=torch.bfloat16, device=dev),
                      src=i32(R, max_new), src_tmp=i32(R, max_new), hist=i32(R, hist_cap), hist_tmp=i32(R, hist_cap), hist_len=i32(1),
                      plen=i32(1), lp=f32(R, V), cand_val=f32(R, 2 * nb), cand_tok=i32(R, 2 * nb), params=i32(16),
                      denom=f64(hist_cap + 1), beam_scores=f32(R), parents=i32(R), hyp_tok=i32(B, nb, max_new), hyp_len=i32(B, nb),
                      hyp_score=f64(B, nb), hyp_order=i32(B, nb), hyp_count=i32(B), worst=f64(B), done=i32(B), flags=i32(3))
        self._beam = st
        return st

    def drop_beam(self) -> bool:
        """Free the beam-search state (beam cache, ancestry table, history, hypothesis store); True if there was one."""
        had = getattr(self, "_beam", None) is not None
        self._beam = None
        return had

    def beam_reset(self, st, prompt_ids: torch.Tensor, T: int, params: torch.Tensor, denom: torch.Tensor):
        """Start a search: history = the caller's prompt ids in every row, beam scores 0 / -1e9, empty hypothesis lists,
        prompt length T of the prefill cache; params / denom as groma_beam_select reads them."""
        B, nb = st["B"], st["nb"]
        L0 = prompt_ids.shape[1]
        st["hist"][:, :L0].copy_(prompt_ids.to(device=self.dev, dtype=torch.int32).repeat_interleave(nb, 0))
        st["hist_len"].fill_(L0)
        st["plen"].fill_(T)
        st["beam_scores"].view(B, nb)[:, 0] = 0.0
        st["beam_scores"].view(B, nb)[:, 1:] = -1e9
        for k in ("hyp_count", "done", "flags", "src", "hyp_len"):
            st[k].zero_()
        st["worst"].fill_(1e9)
        st["params"].copy_(params)
        st["denom"][:denom.numel()].copy_(denom)

    def beam_tail(self, logits, st, d, process: bool):
        """The selection after a beam step's logits [B*nb, V]: log-softmax -> [processors] -> per-row top 2 nb -> per-image
        scorer step (next ids into d['ids'], history / src reordered, cur_len advanced)."""
        nb = st["nb"]
        lp = G.beam_logsoftmax(logits, out=st["lp"])
        sc = G.logits_process(lp, st["hist"], st["hist_len"], d["proc_params"], out=d["scores"]) if process else lp
        G.beam_topk(sc, st["beam_scores"], 2 * nb, st["cand_val"], st["cand_tok"])
        st["ids"] = d["ids"]
        G.beam_select(st, st["B"], nb, logits.shape[1])

    def choose_tokens(self, logits, d, sample: bool, process: bool):
        """Next ids (d['ids']) from fp32 logits [B, V]: with process, groma_logits_process (d['hist'], d['hist_len'],
        d['proc_params']) into d['scores'] first; then the argmax, or with sample the draw (d['sample_params'] /
        d['sample_params_ex'], d['seed'], Philox step = *pos of the input token); with process, the ids are appended to the
        history.  `logits` itself is left as it is."""
        if process:
            logits = G.logits_process(logits, d["hist"], d["hist_len"], d["proc_params"], out=d["scores"])
        if sample and process:
            G.sample_ex(logits, d["sample_params_ex"], d["seed"], d["pos"], out=d["ids"])
        elif sample:
            G.sample(logits, d["sample_params"], d["seed"], d["pos"], out=d["ids"])
        else:
            G.argmax(logits, out=d["ids"])
        if process:
            G.history_append(d["hist"], d["hist_len"], d["ids"])

    def decode_step(self, B: int, sample: bool = False, process: bool = False, beam: Optional[dict] = None,
                    group: Optional[dict] = None) -> torch.Tensor:
        """One greedy decode step for the whole batch (groma.py:376-402 + HF greedy argmax): reads d['ids'], appends K/V at
        *pos, attends to all kv_len[b] cached positions (all-ones mask, T7), writes next ids back to d['ids'].
        Every shape-dependent scalar lives on the device, so the step is CUDA-graph capturable.
        Per layer: 4 swap-AB wgmma GEMMs (weights prefetched under programmatic dependent launch), 4 fused reduce
        epilogues (RoPE+KV append / residual+RMSNorm / SwiGLU / residual+next RMSNorm) and the cluster decode attention.
        sample=True: the tail is head reduce -> groma_sample_tokens (d['sample_params'], d['seed']) -> advance instead of the
        fused reduce + argmax; the persistent kernel (GROMA_DECODE_MEGA=1) is greedy only, so a sampling step takes this path.
        process=True (generate()'s logits processors, state from process_buffers()): head reduce -> groma_logits_process ->
        argmax or groma_sample_tokens_ex -> history append -> advance; like sampling, it never takes the persistent kernel.
        beam (the state of beam_buffers()): B = images x beams rows; the attention is groma_decode_attention_beam over the prompt
        cache and the beam cache, and the tail is head reduce -> beam_tail -> advance.
        group (the caches of group_buffers()): B = images x n prompts rows; the attention is groma_decode_rope_attention_grouped
        over the image's shared prefix and the row's own positions; the rest of the step is the plain one."""
        if (self.use_megakernel and self.mega_supported(B) and not sample and not process and not self.nf4 and not self.kv_fp8
                and not self.fp8 and beam is None and group is None):
            return self.decode_step_mega(B)
        if not self.fused_decode:
            if beam is not None:
                raise G._lib.GromaError("the unfused decode step has no beam form")
            if group is not None:
                raise G._lib.GromaError("the unfused decode step has no prompt-group form")
            return self._decode_step_unfused(B, sample, process)
        cfg, w = self.cfg, self.w
        d = self._decode_buffers(B)
        nh, hd, Hd = cfg.llm_heads, cfg.head_dim, cfg.llm_hidden
        sp = self._decode_splits()
        pdl = self.use_pdl
        G.gather_rows(d["ids"], w["embed"], w["new_embed"], cfg.vocab, out=d["x"])
        x, y = d["x"], d["y"]
        G.rmsnorm(x, w["llm.0.ln1"], cfg.rms_eps, out=y)

        def gemm(inp, wname, split):
            if wname in self.q8:   # fp8: quantise the input rows, then the e4m3 swap-AB GEMM (both PDL-chained)
                c, sc = self.q8[wname]
                n = c.shape[0]
                ws = d["ws"][: split * n * B].view(split, B, n)
                xq, xs = G.fp8_quantize_rows(inp, d["xq"][: inp.numel()].view(inp.shape), d["xs"], pdl=pdl)
                if self.timing_hook is not None:
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                G.gemm_fp8_swap_ab(xq, xs, c, sc, ws, split_k=split, pdl=pdl, transposed=True)
                if self.timing_hook is not None:
                    ev1.record()
                    self.timing_hook.append((ev0, ev1, c.numel() + sc.numel() * 4 + xq.numel() + xs.numel() * 4 + ws.numel() * 4))
                return ws
            if self.nf4:
                c, a, n, _ = self.q4[wname]
                ws = d["ws"][: split * n * B].view(split, B, n)
                if self.timing_hook is not None:
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                G.gemm_nf4_swap_ab(inp, c, a, n, ws, split_k=split, pdl=pdl, transposed=True)
                if self.timing_hook is not None:
                    ev1.record()
                    self.timing_hook.append((ev0, ev1, c.numel() + a.numel() * 4 + inp.numel() * 2 + ws.numel() * 4))
                return ws
            W = w[wname]
            ws = d["ws"][: split * W.shape[0] * B].view(split, B, W.shape[0])
            if self.timing_hook is not None:
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
            if self.decode_tiled:
                G.gemm_swap_ab(inp, self._tiled(wname), ws, split_k=split, pdl=pdl, transposed=True, tiled=True, n_rows=W.shape[0])
            else:
                G.gemm_swap_ab(inp, W, ws, split_k=split, pdl=pdl, transposed=True)
            if self.timing_hook is not None:
                ev1.record()
                self.timing_hook.append((ev0, ev1, W.numel() * 2 + inp.numel() * 2 + ws.numel() * 4))
            return ws

        for i in range(cfg.llm_layers):
            o = f"llm.{i}."
            kc, vc, ks, vs = self.kv_layer(i) if group is None else (None,) * 4
            ws = gemm(y, o + "qkv.w", sp["qkv"])
            if group is not None:
                pre = group["prefix"][i] if group["P"] > 0 else (None, None)
                G.decode_rope_attention_grouped(ws, pre[0], pre[1], group["row"][i, 0], group["row"][i, 1], d["pos"], self.rope_cos,
                                                self.rope_sin, 1.0 / math.sqrt(hd), d["a"], group["n"], pdl=pdl)
            elif beam is not None:
                G.decode_attention_beam(ws, kc, vc, beam["kv"][i, 0], beam["kv"][i, 1], beam["src"], d["pos"], beam["plen"], self.rope_cos,
                                        self.rope_sin, 1.0 / math.sqrt(hd), d["a"], beam["nb"], pdl=pdl)
            elif hd == 128 and self.fused_rope_attn:
                G.decode_rope_attention(ws, kc, vc, d["kv_len"], d["pos"], self.rope_cos, self.rope_sin, 1.0 / math.sqrt(hd), d["a"], pdl=pdl,
                                        scales_k=ks, scales_v=vs)
            else:
                G.decode_reduce_rope_kv(ws, d["q"], kc, vc, self.rope_cos, self.rope_sin, d["pos"], nh, hd, pdl=pdl, scales_k=ks, scales_v=vs)
                if hd == 128:
                    G.decode_attention(d["q"], kc, vc, d["kv_len"], 1.0 / math.sqrt(hd), d["a"], pdl=pdl, scales_k=ks, scales_v=vs)
                else:
                    G.attention(d["q"].reshape(B, 1, nh, hd), kc, vc, causal=False, scale=1.0 / math.sqrt(hd), kv_len=d["kv_len"],
                                out=d["a"], sk=self.kv_cap)
            ws = gemm(d["a"].reshape(B, Hd), o + "o.w", sp["o"])
            G.decode_reduce_norm(ws, x, w[o + "ln2"], y, cfg.rms_eps, pdl=pdl)
            ws = gemm(y, o + "gu.w", sp["gu"])
            G.decode_reduce_swiglu(ws, d["gu"], pdl=pdl)
            ws = gemm(d["gu"], o + "down.w", sp["down"])
            nxt = w[f"llm.{i + 1}.ln1"] if i + 1 < cfg.llm_layers else w["llm.norm"]
            G.decode_reduce_norm(ws, x, nxt, y, cfg.rms_eps, pdl=pdl)
        ws = gemm(y, "head.w", sp["head"])
        if beam is not None:
            G.splitk_reduce(ws, d["logits"])
            self.beam_tail(d["logits"], beam, d, process)
            G.decode_advance(d["pos"], d["kv_len"])
        elif sample or process:
            G.splitk_reduce(ws, d["logits"])
            self.choose_tokens(d["logits"], d, sample, process)
            G.decode_advance(d["pos"], d["kv_len"])
        elif self.fused_head_tail:
            G.decode_head_argmax(ws, d["logits"], d["ids"], d["pos"], d["kv_len"], pdl=pdl)   # reduce + argmax + advance, one launch
        else:
            G.splitk_reduce(ws, d["logits"])
            G.argmax(d["logits"], out=d["ids"])
            G.decode_advance(d["pos"], d["kv_len"])
        return d["logits"]

    def _decode_step_unfused(self, B: int, sample: bool = False, process: bool = False) -> torch.Tensor:
        """Reference arrangement of the same step with stand-alone reduce / norm / RoPE kernels (kept for A/B tests)."""
        if self.kv_fp8:
            raise G._lib.GromaError("the unfused decode step has no fp8-cache form")
        cfg, w = self.cfg, self.w
        d = self._decode_buffers(B)
        nh, hd, Hd = cfg.llm_heads, cfg.head_dim, cfg.llm_hidden
        G.gather_rows(d["ids"], w["embed"], w["new_embed"], cfg.vocab, out=d["x"])
        x = d["x"]
        sp = self._decode_splits()
        for i in range(cfg.llm_layers):
            o = f"llm.{i}."
            G.rmsnorm(x, w[o + "ln1"], cfg.rms_eps, out=d["y"])
            self._swap_gemm(d["y"], o + "qkv.w", d, sp["qkv"], d["qkv"])
            kc, vc = self.kv[i, 0], self.kv[i, 1]
            G.rope_kv(d["qkv"], d["q"], kc, vc, self.rope_cos, self.rope_sin, B, 1, nh, hd, 0, pos_ptr=d["pos"])
            if hd == 128:
                G.decode_attention(d["q"], kc, vc, d["kv_len"], 1.0 / math.sqrt(hd), d["a"])
            else:
                G.attention(d["q"].reshape(B, 1, nh, hd), kc, vc, causal=False, scale=1.0 / math.sqrt(hd), kv_len=d["kv_len"],
                            out=d["a"], sk=self.kv_cap)
            self._swap_gemm(d["a"].reshape(B, Hd), o + "o.w", d, sp["o"], x, residual=x)
            G.rmsnorm(x, w[o + "ln2"], cfg.rms_eps, out=d["y"])
            self._swap_gemm(d["y"], o + "gu.w", d, sp["gu"], d["gu"], act=G.ACT_SWIGLU)
            self._swap_gemm(d["gu"], o + "down.w", d, sp["down"], x, residual=x)
        G.rmsnorm(x, w["llm.norm"], cfg.rms_eps, out=d["y"])
        self._swap_gemm(d["y"], "head.w", d, sp["head"], d["logits"])
        self.choose_tokens(d["logits"], d, sample, process)
        G.decode_advance(d["pos"], d["kv_len"])
        return d["logits"]
