/* groma_b200 -- C ABI of the H100-native Groma forward hot path (libgroma_b200.so, sm_90a).
 *
 * Conventions (every entry point):
 *   - returns int32_t status: 0 = GROMA_OK, otherwise a GROMA_ERR_* code; no exceptions cross the boundary
 *   - all pointers are DEVICE pointers unless a parameter says "host"; outputs and workspaces are caller-owned
 *   - `stream` is a cudaStream_t passed as void*; kernels are enqueued on it, nothing synchronises, nothing allocates
 *   - matrices are row-major bf16 (uint16 storage) unless stated; bias / norm / scale vectors are fp32
 *   - thread-compatible: no global mutable state beyond one-time kernel attribute setup
 *
 * Each declaration cites the reference interface it replaces (paths relative to the FoundationVision/Groma tree;
 * $HF = transformers 4.32 as pinned by the reference's pyproject.toml:19).
 */
#ifndef GROMA_B200_H
#define GROMA_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GROMA_OK 0
#define GROMA_ERR_ARG 1
#define GROMA_ERR_ALIGN 2
#define GROMA_ERR_CUDA 3
#define GROMA_ERR_DRIVER 4
#define GROMA_ERR_TMA_ENCODE 5
#define GROMA_ERR_UNSUPPORTED 6

/* epilogue activation / flags of groma_gemm_bf16 */
#define GROMA_ACT_NONE 0
#define GROMA_ACT_GELU 1   /* erf GELU (nn.GELU default) */
#define GROMA_ACT_RELU 2
#define GROMA_ACT_SWIGLU 3 /* columns (2j,2j+1) = (gate_j, up_j) -> out[:, j] = silu(gate)*up ; N_out = N/2 */
#define GROMA_GF_OUT_F32 1
#define GROMA_GF_BIAS_ALONG_M 2
#define GROMA_GF_PARTIAL 4
#define GROMA_GF_CONV_ROWS 8
#define GROMA_GF_CONV_COMPACT 16
#define GROMA_GF_A_TILED 32 /* A pre-tiled [m_tile][k_block][128][64] (lda must be 64): each TMA load is 16 KB contiguous */
#define GROMA_GF_PARTIAL_T 128 /* partials transposed: ws[split][n][m] */
#define GROMA_GF_PDL 64     /* programmatic dependent launch: A tiles are prefetched before waiting for the previous kernel */

/* D[M,N] = sum_{t<num_taps} A[m + a_row_off[t], 0:K] . B[n, t*K : (t+1)*K]   (+ bias, act, *gamma, + residual)
 * wgmma/TMA GEMM.  Replaces every torch.nn.Linear / nn.Conv2d(1x1, 3x3 pad 1) call on the path:
 *   groma/model/groma.py:112-119,389-401 ; groma/model/roi_align.py:128-143,251-264 ; groma/model/ddetr.py:147-151 ;
 *   $HF/models/{dinov2,llama,deformable_detr}/modeling_*.py Linear layers (cuBLAS / cuDNN in the reference).
 * A: [a_rows, lda] bf16, B: [b_rows, ldb] bf16 (lda, ldb multiples of 8; pointers 16-byte aligned).
 * num_taps > 1 = implicit-GEMM convolution over zero-bordered flat NHWC maps (a_row_off = tap row shifts, host array).
 * out[m*ld_m + n*ld_n] bf16 (or fp32 with GROMA_GF_OUT_F32); bias/gamma fp32 per column (per row with BIAS_ALONG_M);
 * residual bf16 with the strides of out.  GROMA_GF_PARTIAL: raw fp32 accumulators to ws[split][M][N] (split_k >= 1).
 * GROMA_GF_CONV_ROWS: rows are pixels of [img][conv_hp][conv_wp] maps, border rows are not written;
 * with GROMA_GF_CONV_COMPACT the row index is that of the un-padded [img][hp-2][wp-2] layout.
 * tile_counters (optional, with GROMA_GF_PARTIAL): zero-initialised int32[m_tiles*n_tiles]; the CTA that delivers the last
 * split of a tile sums ws over the splits in fixed order and applies the epilogue to `out` itself (no groma_splitk_reduce
 * launch); with GROMA_ACT_SWIGLU + GROMA_GF_BIAS_ALONG_M the (gate, up) pairs are adjacent ROWS (swap-AB decode layout).
 * block_n: 0 = auto, else 16/32/64/128/256. */
int32_t groma_gemm_bf16(const void* A, int64_t a_rows, int64_t lda, const void* B, int64_t b_rows, int64_t ldb,
                        int32_t M, int32_t N, int32_t K, int32_t num_taps, const int32_t* a_row_off /*host*/,
                        void* out, int64_t ld_m, int64_t ld_n, int32_t flags, int32_t act, const float* bias,
                        const float* gamma, const void* residual, float* ws, int32_t split_k,
                        int32_t* tile_counters, int32_t conv_hp, int32_t conv_wp, int32_t block_n, void* stream);

/* LLaMA attention input in ONE launch: x[B*T, K] @ w_qkv[3*H*D, K]^T (rows of w_qkv = [q heads | k heads | v heads]) with the
 * rotate-half RoPE of q and k and the KV-cache append done in the GEMM epilogue -- the [B*T, 3*H*D] intermediate of
 * groma_gemm_bf16 + groma_rope_kv never exists.  Replaces q_proj/k_proj/v_proj + apply_rotary_pos_emb + the cache torch.cat
 * of $HF/models/llama/modeling_llama.py:199-246 (called from groma/model/groma.py:389-397).  Values are bit-identical to the
 * two-launch form: the projection is rounded to bf16, rotated in fp32, rounded again.
 * q_out [B*T, H*D] bf16; cache_k / cache_v [B, H, ctx_cap, D] bf16; cos_t / sin_t fp32 [max_pos, D/2]; token t of every
 * sequence sits at position pos0 + t (pos0 + T <= ctx_cap).  D must be 128 and H even; block_n = 256 (one CTA per
 * 128x256 tile) or 512 (two-CTA cluster, 256x256). */
int32_t groma_gemm_qkv_rope(const void* x, int64_t ldx, const void* w_qkv, int64_t ldw, int32_t B, int32_t T, int32_t H,
                            int32_t D, int32_t K, void* q_out, void* cache_k, void* cache_v, const float* cos_t,
                            const float* sin_t, int32_t pos0, int64_t ctx_cap, int32_t block_n, void* stream);

/* out = epilogue(sum_s ws[s][M][N]) -- the deferred epilogue of a GROMA_GF_PARTIAL GEMM (same chain as above). */
int32_t groma_splitk_reduce(const float* ws, int32_t splits, int32_t M, int32_t N, int32_t act, int32_t flags,
                            const float* bias, const float* gamma, const void* residual, void* out, int64_t ld_m,
                            int64_t ld_n, void* stream);

/* softmax(QK^T*scale + mask)V, bf16, head_dim 32/64/128, online softmax, fp32 accumulate.
 * Replaces $HF/models/llama/modeling_llama.py:199-289 (eager attention, causal + key padding),
 * $HF/models/dinov2/modeling_dinov2.py:153-179 and $HF/models/deformable_detr/modeling_deformable_detr.py:453-516.
 * q[b*q_bs + i*q_rs + h*D + d], k[b*k_bs + h*k_hs + j*k_rs + d] (v alike), o[b*o_bs + i*o_rs + h*D + d].
 * causal: key j visible to query i iff j <= q_pos0 + i.  kv_len (optional, int32[B]): keys >= kv_len[b] masked. */
int32_t groma_attention(const void* q, int64_t q_bs, int64_t q_rs, const void* k, int64_t k_bs, int64_t k_hs,
                        int64_t k_rs, const void* v, int64_t v_bs, int64_t v_hs, int64_t v_rs, void* o, int64_t o_bs,
                        int64_t o_rs, const int32_t* kv_len, int32_t B, int32_t H, int32_t Sq, int32_t Sk, int32_t D,
                        int32_t causal, int32_t q_pos0, float scale, void* stream);

/* Precondition of both attention entry points: every K and V row a tile load can touch (rows up to the next multiple of 128 past
 * Sk / kv_len, inside the tensor) holds finite values.  Masked keys get probability exactly 0, and 0 * NaN would still poison O;
 * GromaEngine allocates the KV cache zero-filled.
 * The same attention on the Hopper tensor cores (wgmma, TMA-fed, S/O accumulators in registers), head_dim 64 / 128.
 * q/k/v are 2-D bf16 row-major views [rows, cols] (row stride ld); element (b, i|j, h, d) lives at
 *   q: row b*q_batch_rows + i,                 col h*q_head_cols + d
 *   k: row b*k_batch_rows + h*k_head_rows + j, col h*k_head_cols + d      (v alike)
 * -- covers the KV cache [B,H,cap,D] and fused qkv activations [B*S, 3*H*D] without copies.  o: [B*Sq, o_ld], col h*D + d. */
int32_t groma_attention_tc(const void* q, int64_t q_rows, int64_t q_cols, int64_t q_ld, int32_t q_batch_rows, int32_t q_head_cols,
                           const void* k, int64_t k_rows, int64_t k_cols, int64_t k_ld, int32_t k_batch_rows, int32_t k_head_rows,
                           int32_t k_head_cols, const void* v, int64_t v_rows, int64_t v_cols, int64_t v_ld, int32_t v_batch_rows,
                           int32_t v_head_rows, int32_t v_head_cols, void* o, int64_t o_ld, const int32_t* kv_len, int32_t B,
                           int32_t H, int32_t Sq, int32_t Sk, int32_t D, int32_t causal, int32_t q_pos0, float scale, void* stream);

/* Single-query (decode) attention over the KV cache: every cached position < kv_len[b] is visible (the all-ones mask of
 * groma/model/groma.py:376-379).  q, out [B, H*D]; cache_k/v [B, H, cap, D]; D = 128.  HBM-bound SIMT kernel. */
int32_t groma_decode_attention(const void* q, const void* cache_k, const void* cache_v, void* out, const int32_t* kv_len,
                               int32_t B, int32_t H, int32_t D, int64_t cap, float scale, int32_t pdl, void* stream);

/* groma_decode_reduce_rope_kv + groma_decode_attention in one launch (decode step, D = 128): q and the new token's K/V row
 * are reduced from the qkv GEMM's split-K partials ws[splits][B][3*H*D], rotated (rotate-half RoPE at position *pos_ptr,
 * $HF/models/llama/modeling_llama.py:138-168), the K/V row is appended to the cache at *pos_ptr (the tuple-cache torch.cat of
 * groma.py:376-379) and the attention over kv_len[b] positions follows; bit-identical to the two separate calls. */
int32_t groma_decode_rope_attention(const float* ws, int32_t splits, void* cache_k, void* cache_v, void* out,
                                    const int32_t* kv_len, const int32_t* pos_ptr, const float* cos_t, const float* sin_t,
                                    int32_t B, int32_t H, int32_t D, int64_t cap, float scale, int32_t pdl, void* stream);

/* The same two decode attentions over an FP8 (e4m3) KV cache (DESIGN.md section 4): codes_k/v uint8 [B, H, cap, D], scales_k/v
 * fp32 [B, H, cap] (16-byte aligned, cap % 4 == 0), key / value row x^ = fp32(code) * scale.  The _rope_ form quantises the
 * appended row (groma_kv_quantize's rule) and attends over its x^ like every other row.  Default (TMA ring) and
 * GROMA_DEC_ATTN_TMA=0 (LDG) kernels are bit-identical, as for bf16. */
int32_t groma_decode_attention_fp8(const void* q, const void* codes_k, const void* codes_v, const float* scales_k,
                                   const float* scales_v, void* out, const int32_t* kv_len, int32_t B, int32_t H, int32_t D,
                                   int64_t cap, float scale, int32_t pdl, void* stream);
int32_t groma_decode_rope_attention_fp8(const float* ws, int32_t splits, void* codes_k, void* codes_v, float* scales_k,
                                        float* scales_v, void* out, const int32_t* kv_len, const int32_t* pos_ptr, const float* cos_t,
                                        const float* sin_t, int32_t B, int32_t H, int32_t D, int64_t cap, float scale, int32_t pdl,
                                        void* stream);

/* y = w * bf16(h * rsqrt(mean(h^2)+eps)), h = bf16(x + residual) (h_out optional).  LlamaRMSNorm,
 * $HF/models/llama/modeling_llama.py:53-70 (+ the residual add of :292-340). */
int32_t groma_rmsnorm(const void* x, const void* residual, const float* w, void* y, void* h_out, int64_t rows,
                      int32_t dim, float eps, void* stream);

/* y = LayerNorm(x (+ residual)) * w + b over the last dim.  nn.LayerNorm call sites: modeling_dinov2.py:356-372,
 * modeling_deformable_detr.py:699-706,782-803 (post-LN), groma/model/ddetr.py:25-45 (channel LN == LN over NHWC C),
 * groma/model/roi_align.py:254-261, ddetr_transformer.py:311-314. */
int32_t groma_layernorm(const void* x, const void* residual, const float* w, const float* b, void* y, int64_t rows,
                        int32_t dim, float eps, int64_t x_row_stride, int64_t y_row_stride, void* stream);

/* y = relu(GroupNorm_G(x)) over NHWC [B, P, C]; mmcv ConvModule norm+act (mmcv/cnn/bricks/conv_module.py:196-206)
 * as used by groma/model/roi_align.py:133-143.  part: fp32 scratch [B*chunks*G*2]; stats: fp32 [B*G*2] (mean, rstd). */
int32_t groma_groupnorm_relu(const void* x, const float* gamma, const float* beta, void* y, float* part, float* stats,
                             int32_t B, int64_t P, int32_t C, int32_t G, float eps, int32_t chunks, void* stream);
/* The two halves of the call above: statistics only (stats [B,G,2] = mean, rstd) and apply + ReLU with given statistics.  The
 * fusion rounds of MLVLFuseModule (groma/model/roi_align.py:118-126,180-193) keep the RAW conv outputs and let the next round's
 * groma_fuse_shuffle_gn apply norm + act tap by tap; only the last round's maps are materialised with groma_groupnorm_apply_relu. */
int32_t groma_groupnorm_stats(const void* x, float* part, float* stats, int32_t B, int64_t P, int32_t C, int32_t G, float eps,
                              int32_t chunks, void* stream);
int32_t groma_groupnorm_apply_relu(const void* x, const float* stats, const float* gamma, const float* beta, void* y, int32_t B,
                                   int64_t P, int32_t C, int32_t G, void* stream);

/* Multi-scale deformable attention forward; twin of mmcv `ms_deform_attn_forward`
 * (mmcv/ops/csrc/pytorch/pybind.cpp:162,765; kernel common/cuda/ms_deform_attn_cuda_kernel.cuh:203-256) with the
 * softmax over (levels*points) and the sampling-location arithmetic of modeling_deformable_detr.py:586-610 fused in.
 * value [B,S,nH,32] bf16; proj [B*Q, nH*L*P*2 + nH*L*P] fp32 (offsets | logits); ref [B,Q,ref_dim] fp32;
 * out [B,Q,nH*32] bf16; level_hw host int32[2L] (h,w), level_start host int32[L]. */
int32_t groma_msda_forward(const void* value, const float* proj, const float* ref, void* out, int32_t B, int32_t Q,
                           int32_t S, int32_t n_heads, int32_t n_levels, int32_t n_points, int32_t ref_dim,
                           const int32_t* level_hw /*host*/, const int32_t* level_start /*host*/, void* stream);

/* RoIAlign forward (avg, aligned flag); twin of mmcv `roi_align_forward` (pybind.cpp:191,611; kernel
 * common/cuda/roi_align_cuda_kernel.cuh:17-108).  input NHWC bf16 [N,H,W,C]; rois fp32 [K,5] (batch, x1,y1,x2,y2);
 * output [K, ph+2p, pw+2p, C] bf16 with p = out_pad (0/1) zero border. */
int32_t groma_roi_align_forward(const void* input, const float* rois, void* output, int32_t K, int32_t C, int32_t H,
                                int32_t W, int32_t pooled_h, int32_t pooled_w, float spatial_scale,
                                int32_t sampling_ratio, int32_t aligned, int32_t out_pad, void* stream);

/* Batched greedy NMS; twin of mmcv `nms` (pybind.cpp:175,596; nms_cuda_kernel.cuh:18-74, nms_cuda.cu:5-54) plus the
 * score filter / max_num of mmcv/ops/nms.py:14-33, for all images of groma/model/groma.py:257-280 in one launch.
 * boxes [B,N,4] xyxy fp32, scores [B,N] fp32, counts int32[B] (optional valid prefix length per image).
 * keep int64 [B,max_out] (original indices, score order, -1 padded); num_keep int32[B];
 * argmax_idx int32[B] = first index of the max score (the reference's fallback when nothing is kept). */
int32_t groma_nms_batched(const float* boxes, const float* scores, const int32_t* counts, int32_t B, int32_t N,
                          float iou_threshold, float score_threshold, int32_t offset, int32_t max_num, int64_t* keep,
                          int32_t max_out, int32_t* num_keep, int32_t* argmax_idx, void* stream);

/* torch.topk(scores, k, dim=1)[1] (ddetr_transformer.py:556): indices of the k largest, descending. */
int32_t groma_topk_desc(const float* scores, int64_t ld, int32_t B, int32_t N, int32_t k, int64_t* out_idx, void* stream);

/* Two-stage proposal gather + sigmoid + sine embedding (ddetr_transformer.py:432-446,556-566). */
int32_t groma_ddetr_select(const float* delta, const float* proposals, const int64_t* topk, float* ref_out,
                           void* pos_out, int32_t B, int32_t S, int32_t k, int32_t num_pos_feats, void* stream);

/* Final box/score heads (ddetr_transformer.py:696-715 restricted to what inference reads, groma.py:246-249,268). */
int32_t groma_ddetr_finalize(const float* d4, const float* d5, const float* ref0, const float* coco, const float* sa1b,
                             float* pred_cxcywh, float* pred_xyxy, float* score, int32_t B, int32_t Q,
                             int64_t out_stride_boxes, int64_t out_stride_scores, void* stream);

/* zero rows of x [B,S,D] where valid[s]==0 (ddetr_transformer.py:424-426). */
int32_t groma_mask_rows(void* x, const uint8_t* valid, int32_t B, int32_t S, int32_t D, void* stream);

/* Region-encoder resampling (groma/model/roi_align.py:118-126,215-228 and :150-178). */
int32_t groma_upsample_coords(const void* tokens, int32_t skip, int32_t g, int32_t C, void* out, int32_t B, int32_t Ho,
                              int32_t Wo, int32_t ld, const float* xs, const float* ys, void* stream);
int32_t groma_fuse_shuffle(const void* tar, const void* top, const void* down, void* out, int32_t B, int32_t C,
                           int32_t Ht, int32_t Wt, int32_t Htop, int32_t Wtop, int32_t Hdn, int32_t Wdn, void* stream);
/* Same shuffle over the previous round's raw conv outputs: relu(GroupNorm_G) with per-level statistics and the round's shared
 * gamma / beta (mmcv ConvModule norm + act, conv_module.py:196-206) is applied to every tap and rounded to bf16 first, so the
 * result is bit-identical to groma_groupnorm_apply_relu on each map followed by groma_fuse_shuffle. */
int32_t groma_fuse_shuffle_gn(const void* tar, const void* top, const void* down, void* out, int32_t B, int32_t C,
                              int32_t Ht, int32_t Wt, int32_t Htop, int32_t Wtop, int32_t Hdn, int32_t Wdn,
                              const float* stats_tar, const float* stats_top, const float* stats_down, const float* gamma,
                              const float* beta, int32_t G, void* stream);

/* DINOv2 embeddings (modeling_dinov2.py:57-149): im2col of 14x14 patches and CLS/pos-embed assembly. */
int32_t groma_vit_patchify(const float* images, void* patches, int32_t B, int32_t S, int32_t ld, void* stream);
int32_t groma_vit_embed(const void* patch, const float* cls, const float* pos, void* out, int32_t B, int32_t NP,
                        int32_t C, void* stream);

/* groma.py:227-242: mean of the last hidden states (CLS dropped) and the 2x2 space-to-depth token merge. */
int32_t groma_mean_tokens(const void* a0, const void* a1, const void* a2, const void* a3, int32_t n, void* out,
                          int32_t B, int32_t T, int32_t C, int32_t skip, void* stream);
int32_t groma_space_to_depth(const void* in, void* out, int32_t B, int32_t g, int32_t C, void* stream);

/* groma.py:165-174,360-369: split-vocabulary embedding lookup and visual-token splice (row gather / scatter). */
int32_t groma_gather_rows(const int64_t* idx, const void* t0, const void* t1, int64_t split, void* out, int64_t n,
                          int32_t D, void* stream);
int32_t groma_scatter_rows(const int64_t* idx, const void* src, void* out, int64_t n, int32_t D, void* stream);

int32_t groma_add(const void* a, const void* b, void* c, int64_t n, void* stream);
int32_t groma_add_bcast(const void* a, const void* b, void* c, int64_t rows, int64_t period, int32_t D, void* stream);

/* rotate-half RoPE on fused QKV rows + KV-cache append (modeling_llama.py:138-168,225-289). */
int32_t groma_rope_kv(const void* qkv, void* q_out, void* cache_k, void* cache_v, const float* cos_t,
                      const float* sin_t, int32_t B, int32_t T, int32_t H, int32_t D, int32_t pos0,
                      const int32_t* pos_ptr /*device, optional: overrides pos0*/, int64_t ctx_cap, void* stream);

/* out = act(x[M,K] @ w[N,K]^T + b) for K <= 64 in fp32 (roi_align.py:255: Linear(4,256) on the fp32 boxes). */
int32_t groma_linear_smallk(const float* x, const float* w, const float* b, void* out, int64_t M, int32_t N, int32_t K,
                            int32_t relu, void* stream);

/* device-side decode bookkeeping (*pos += 1; kv_len[b] += 1) so a decode step is CUDA-graph capturable. */
int32_t groma_decode_advance(int32_t* pos, int32_t* kv_len, int32_t B, void* stream);

/* Fused decode epilogues over token-major split-K partials ws[split][token][feature] (GROMA_GF_PARTIAL_T); pdl != 0
 * launches them with programmatic stream serialisation (they wait for their producer in-kernel).
 *   reduce_norm   : x = bf16(sum + x) in place; y = LlamaRMSNorm(x)            (modeling_llama.py:292-340,53-70)
 *   reduce_swiglu : out[:, j] = silu(sum[2j]) * sum[2j+1]                        (modeling_llama.py:171-184)
 *   reduce_rope_kv: RoPE(q,k) at *pos_ptr, q -> q_out, k/v -> cache[b,h,*pos_ptr] (modeling_llama.py:138-168,225-289) */
int32_t groma_decode_reduce_norm(const float* ws, int32_t splits, int32_t B, int32_t N, void* x, const float* w, void* y,
                                 float eps, int32_t pdl, void* stream);
int32_t groma_decode_reduce_swiglu(const float* ws, int32_t splits, int32_t B, int32_t N, void* out, int32_t pdl, void* stream);
/* Tail of a decode step in one launch: logits[b, :] = sum_s ws[s][b][:] (fp32 [B, V], what lm_head returns,
 * groma/model/groma.py:399-402), ids[b] = first maximal index (HF greedy_search's torch.argmax), then *pos += 1 and
 * kv_len[b] += 1 for the next step.  Same values as groma_splitk_reduce + groma_argmax + groma_decode_advance. */
int32_t groma_decode_head_argmax(const float* ws, int32_t splits, int32_t B, int32_t V, float* logits, int64_t* ids,
                                 int32_t* pos, int32_t* kv_len, int32_t pdl, void* stream);
int32_t groma_decode_reduce_rope_kv(const float* ws, int32_t splits, int32_t B, int32_t H, int32_t D, void* q_out, void* cache_k,
                                    void* cache_v, const float* cos_t, const float* sin_t, const int32_t* pos_ptr, int64_t cap,
                                    int32_t pdl, void* stream);
/* reduce_rope_kv into an FP8 cache (D = 128): the rotated K row and the V row are quantised as groma_kv_quantize does. */
int32_t groma_decode_reduce_rope_kv_fp8(const float* ws, int32_t splits, int32_t B, int32_t H, int32_t D, void* q_out,
                                        void* codes_k, void* codes_v, float* scales_k, float* scales_v, const float* cos_t,
                                        const float* sin_t, const int32_t* pos_ptr, int64_t cap, int32_t pdl, void* stream);

/* ---- one persistent kernel per greedy decode step --------------------------------------------------------------------------
 * Replaces, for B <= 16 rows and head_dim 128, everything the reference executes per generated token: GromaModel.forward's
 * decode branch (groma/model/groma.py:376-402: embedding of the last id, 32 x LlamaDecoderLayer with KV append
 * -- $HF/models/llama/modeling_llama.py:292-340 -- final norm, lm_head || extra_lm_head) and the argmax of HF greedy search.
 * One launch of one CTA per SM; the weight / KV stream of each CTA is a single in-order ring filled by TMA that never waits for
 * activations (groma_b200/csrc/decode_megakernel.cu).  All pointers are device pointers owned by the caller:
 *   w_arena  [L*(3Hd + Hd + 2I) + V, Hd] bf16: per layer q|k|v rows, o rows, (gate_j, up_j)-interleaved rows; then lm_head || extra_lm_head
 *   w_down   [L*Hd, I] bf16;  ln_w [2L+1][Hd] fp32: input_layernorm_l, post_attention_layernorm_l (l = 0..L-1), final norm
 *   kv       [L][2][B][H][cap][128] bf16 cache; rope_cos/sin [>= pos+1][64] fp32
 *   ids [B] int64 (in: token to embed; out: next greedy token), pos [1], kv_len [B] (advanced by the kernel)
 *   x, y_attn, y_mlp, a [B][Hd] bf16, gu [B][I] bf16, logits [B][V] fp32 (written), ws_* fp32 scratch of
 *   tiles * layout[1] floats (tiles = rows/128 of the projection), att_part [B*H*S_att * layout[2]] floats,
 *   cand_val / cand_idx [ceil(V/128) * 16], flags int32[layout[0]] -- MUST be zero at entry (cudaMemsetAsync / fill before
 *   every step), status int32[8 + 16 * grid] -- zero at allocation; status[0] != 0 after the step = a dependency wait timed out
 *   (status[1..6]: CTA, role, thread, progress counters; from [8]: per (CTA, role) the wait it was parked in) and the outputs
 *   are invalid.
 * S_att: key segments per (row, head), merged in fixed order; choose it so that B*H*S_att is a few times the SM count.
 * grid: 0 = one CTA per SM (must not exceed the SM count: all CTAs have to be co-resident). */
typedef struct groma_decode_step_args {
    int32_t L, B, H, Hd, I, V, vocab, S_att;
    int64_t cap;
    float scale, eps;
    const void *w_arena, *w_down, *embed, *new_embed;
    const float* ln_w;
    void* kv;
    const float *rope_cos, *rope_sin;
    int64_t* ids;
    int32_t* pos;
    int32_t* kv_len;
    void *x, *y_attn, *y_mlp, *a, *gu;
    float* logits;
    float *ws_qkv, *ws_o, *ws_gu, *ws_down, *ws_head;
    float* att_part;
    float* cand_val;
    int32_t* cand_idx;
    int32_t* flags;
    int32_t* status;
    int32_t grid;
    int32_t l2_prefetch_slots; /* 16 KB slots the L2 prefetcher keeps ahead of the shared-memory ring (0 = no prefetch) */
    int64_t* timeline;   /* optional (may be null): int64[grid*4*32] %globaltimer stamps of the phase boundaries, for profiling */
} groma_decode_step_args;
int32_t groma_decode_step_fused(const groma_decode_step_args* args /*host*/, void* stream);
/* layout[0] = number of int32 dependency flags, [1] = fp32 scratch floats per 128-row weight tile, [2] = floats per attention
 * partial, [3] = max rows per step (host array of 4). */
int32_t groma_decode_step_layout(int32_t L, int32_t B, int32_t H, int32_t Hd, int32_t I, int32_t V, int64_t* layout /*host*/,
                                 void* stream);

/* greedy next-token argmax over fp32 logits (HF greedy_search). */
int32_t groma_argmax(const float* logits, int64_t* out, int32_t rows, int32_t V, int64_t ld, void* stream);

/* ---- sampled next token (generate(do_sample=True)) ---------------------------------------------------------------------------
 * The reference's sampling path is HF 4.32 `sample()` (its training script writes do_sample = True into every checkpoint's
 * generation_config.json, groma/train/train.py:108-112; the chat front ends sample at temperature 0.2-0.7,
 * groma/serve/cli.py:48-52, serve/model_worker.py:307-311): fp32 logits -> TemperatureLogitsWarper -> TopKLogitsWarper ->
 * TopPLogitsWarper -> softmax -> torch.multinomial ($HF/generation/utils.py `sample`, $HF/generation/logits_process.py).
 * Per row of logits [rows, V] (row stride ld), with s = l / temperature (fp32 division):
 *   top-k (top_k > 0): keep s_i >= the k-th largest s (every tie with it kept; k = min(k, V)), as TopKLogitsWarper;
 *   top-p (top_p < 1): p = softmax of s over the top-k survivors; keep token j iff the mass of survivors with s > s_j is
 *     < top_p -- what TopPLogitsWarper's ascending cumsum `cum <= 1 - top_p` removes, with the maximum always kept.  Every
 *     token equal to the boundary value is kept (HF's unstable sort makes that case arbitrary there).  The mass is integer fixed
 *     point, round(exp(s - max) * 2^40) per token, compared with ceil(top_p * sum); it agrees with exact arithmetic except when
 *     the boundary mass is within ~1e-6 of top_p.
 *   draw: torch.multinomial cannot be reproduced by a kernel, so the draw is this library's own.  Gumbel-max over the kept set:
 *     token = argmax_{i kept} (s_i - log(-log u_i)) in fp32, first index on a tie; that is exactly a draw from softmax(s) over
 *     the kept set, without sort, prefix sum or renormalisation.  u_i = ((x >> 8) + 0.5) * 2^-24 with x = word (i & 3) of
 *     Philox4x32-10(counter = (i >> 2, row, *step, 0), key = (low, high) 32 bits of *seed).  The perturbation lies in
 *     [-2.86, 17.33], so a token whose probability relative to the best kept token is below about e^-20 is never drawn.
 * params (device): temperature > 0, top_k >= 0 (0 = off), 0 <= top_p <= 1 (1 = off); seed int64 and step int32 are device scalars
 * too, so a captured CUDA graph stays valid when a later call changes any of them.  Logits must be finite.  ids int64 [rows].
 * Deterministic: the same logits, params, seed and step give the same token on every run (integer or fixed-order reductions).
 * One CTA per row stages the row in shared memory: GROMA_ERR_UNSUPPORTED when 4 * V bytes (+ 11 KB) exceed the device's
 * per-block limit (V up to about 55 000 on H100). */
typedef struct GromaSampleParams {
    float temperature;
    int32_t top_k;
    float top_p;
    int32_t reserved;
} GromaSampleParams;
int32_t groma_sample_tokens(const float* logits, int64_t ld, int32_t rows, int32_t V, const GromaSampleParams* params,
                            const int64_t* seed, const int32_t* step, int64_t* ids, void* stream);

/* groma_sample_tokens plus HF 4.32's remaining warpers, applied after top-p in _get_logits_warper's order with
 * min_tokens_to_keep = 1.  Each works on the distribution left by the ones before it (softmax of s over the tokens still kept):
 *   typical (0 < typical_p < 1; >= 1 = off), TypicalLogitsWarper: with H = -sum p log p, order the kept tokens by
 *     |-log p_i - H| ascending and keep every token whose distance is <= that of the first token at which the ascending mass
 *     reaches typical_p (ties kept).  The mass is the same integer fixed point as top-p, compared with ceil(typical_p * sum).
 *   epsilon (0 < epsilon_cutoff < 1, else off), EpsilonLogitsWarper: drop p_i < epsilon_cutoff unless s_i is the kept maximum.
 *   eta (0 < eta_cutoff < 1, else off), EtaLogitsWarper: drop p_i < min(eta, sqrt(eta) * exp(-H)) unless s_i is the kept
 *     maximum.
 * p and H come from double sums in a fixed order, so draws stay deterministic; a decision within about 1e-6 (relative) of its
 * boundary may differ from HF's fp32 arithmetic.  Then the draw is groma_sample_tokens' Gumbel-max over the kept set.
 * Logits may contain -inf (the output of groma_logits_process): such a token has zero mass and is never drawn.  A row with no
 * finite logit gives token 0, the token greedy search's argmax gives there (HF `sample` raises in torch.multinomial instead).
 * groma_sample_tokens with the extended warpers off draws exactly what groma_sample_tokens draws. */
typedef struct GromaSampleParamsEx {
    float temperature;
    int32_t top_k;
    float top_p;
    float typical_p;
    float epsilon_cutoff;
    float eta_cutoff;
    int32_t reserved[2];
} GromaSampleParamsEx;
int32_t groma_sample_tokens_ex(const float* logits, int64_t ld, int32_t rows, int32_t V, const GromaSampleParamsEx* params,
                               const int64_t* seed, const int32_t* step, int64_t* ids, void* stream);

/* ---- generate()'s logits processors ------------------------------------------------------------------------------------------
 * HF 4.32 `_get_logits_processor`, in its order, on fp32 logits [rows, V] (row stride ld), written to scores (row stride
 * ld_scores; logits are not modified).  history int32 [rows, history_cap] holds what HF passes as `input_ids`: the caller's
 * prompt ids followed by the tokens generated so far; cur_len = *history_len (a device scalar, common to all rows).
 *   repetition penalty (!= 1), RepetitionPenaltyLogitsProcessor: every distinct token of the row's history, once:
 *     s < 0 ? s * penalty : s / penalty (IEEE fp32).
 *   no-repeat n-gram (n > 0), NoRepeatNGramLogitsProcessor: -inf for every token t such that (last n - 1 history tokens, t)
 *     is an n-gram of the history.  n = 1 bans every token of the history.
 *   bad words, NoBadWordsLogitsProcessor: an entry of length len <= cur_len bans its last token when the history ends with
 *     its first len - 1 tokens (single-token entries are in the static ban list).  HF applies them as scores + bias, so
 *     while bad_words is set every score gets + 0.0f (a -0.0 logit becomes +0.0).
 *   min length, MinLengthLogitsProcessor / MinNewTokensLengthLogitsProcessor: every EOS id gets -inf while
 *     cur_len < min_length or cur_len - prompt_length < min_new_tokens.
 *   suppress tokens, SuppressTokensLogitsProcessor: the static ban list gets -inf.
 * Every step other than the penalty only sets -inf, so their order does not matter after it.  Token ids outside [0, V) in the
 * history or the lists are ignored.  params: a GromaProcessParams header followed by the packed int32 lists; each *_off is
 * a word offset from the start of the block, params_words its total length (a list outside the block is ignored).  Bad-word
 * entries of two or more tokens are stored back to back; seq_off points at n_seq + 1 word offsets into the block (CSR):
 * entry e is block[offs[e] .. offs[e + 1]).  Everything lives on the device, so a captured CUDA graph stays valid when a
 * later call changes any value (but not the block's address or length).  GROMA_ERR_UNSUPPORTED when V > 196 608. */
typedef struct GromaProcessParams {
    float repetition_penalty;   /* 1 = off */
    int32_t no_repeat_ngram_size; /* 0 = off */
    int32_t min_length;         /* 0 = off */
    int32_t prompt_length;
    int32_t min_new_tokens;     /* 0 = off */
    int32_t n_eos, eos_off;     /* the EOS ids the length processors ban (n_eos = 0: both off, as in HF without an EOS) */
    int32_t n_ban, ban_off;     /* static bans: suppress_tokens and single-token bad words */
    int32_t n_seq, seq_off;     /* bad words of two or more tokens */
    int32_t bad_words;          /* 1 when bad_words_ids is set: HF adds its -inf bias to every score, which turns -0.0 into +0.0 */
    int32_t reserved[4];
} GromaProcessParams;
int32_t groma_logits_process(const float* logits, int64_t ld, float* scores, int64_t ld_scores, int32_t rows, int32_t V,
                             const int32_t* history, int64_t history_cap, const int32_t* history_len, const int32_t* params,
                             int32_t params_words, void* stream);
/* history[r, *history_len] = ids[r] for every row, then *history_len += 1; a full history (len == cap) is left as it is. */
int32_t groma_history_append(int32_t* history, int64_t history_cap, int32_t* history_len, const int64_t* ids, int32_t rows,
                             void* stream);

/* ---- beam search (generate(num_beams > 1); DESIGN.md sections 3 and 4, restated in oracle/beam_search.py) -----------------
 * Replaces HF 4.32 `beam_search` + `BeamSearchScorer` ($HF/generation/utils.py, $HF/generation/beam_search.py) and LLaMA's
 * `_reorder_cache` (index_select of every cached K/V on the batch dimension; the reference's GromaModel has no such hook, so
 * its beam search cannot run).  Rows r = b * nb + j: beam j of image b, B * nb <= GROMA_BEAM_MAX_ROWS, nb <= GROMA_BEAM_MAX_BEAMS.
 *
 * groma_decode_attention_beam: the decode attention of every beam, bf16 caches, D = 128.  prompt_k/v [B, H, prompt_cap, 128]:
 * the prefill's cache, read once per image and group of up to 4 beams (positions 0 .. *prompt_len - 1).  beam_k/v [B * nb, H, gen_cap,
 * 128]: the generated keys; src int32 [B * nb, gen_cap]: generated position g of beam r lives in slot src[r][g] (the ancestry
 * table groma_beam_select maintains, so a reorder never moves the cache).  Fused prologue as groma_decode_rope_attention: ws
 * [splits, B * nb, 3 * H * 128] are the qkv split-K partials; q and the new K/V row are reduced, rounded to bf16 and rotated at
 * position *pos_ptr = T + s (T = *prompt_len) and the row is stored at beam-cache index s of slot r.  Beam r attends to the
 * prompt and its generated positions 0 .. s; the caller keeps 0 <= s < gen_cap.  out bf16 [B * nb, H * 128].  pdl: programmatic
 * stream serialisation. */
#define GROMA_BEAM_MAX_BEAMS 8
#define GROMA_BEAM_MAX_K (2 * GROMA_BEAM_MAX_BEAMS)
#define GROMA_BEAM_MAX_ROWS 256
int32_t groma_decode_attention_beam(const float* ws, int32_t splits, const void* prompt_k, const void* prompt_v, int64_t prompt_cap,
                                    void* beam_k, void* beam_v, int32_t gen_cap, const int32_t* src, const int32_t* pos_ptr,
                                    const int32_t* prompt_len, const float* cos_t, const float* sin_t, void* out, int32_t B,
                                    int32_t nb, int32_t H, int32_t D, float scale, int32_t pdl, void* stream);
/* ---- prompt groups (generate() with n prompts per image; DESIGN.md sections 3 and 4) ------------------------------------------
 * groma_decode_rope_attention_grouped: the decode attention of B images x n prompts, rows r = b * n + j, bf16 caches, D = 128,
 * n <= GROMA_GROUP_MAX_PROMPTS, B * n <= GROMA_BEAM_MAX_ROWS.  prefix_k/v [B, H, prefix_len, 128]: the K/V of the P = prefix_len
 * positions every row of an image shares, read once per (image, head) and multiplied on the tensor cores (P may be 0).
 * row_k/v [B * n, H, row_cap, 128]: each row's own positions, position p at index p - P.  Fused prologue as
 * groma_decode_rope_attention: ws [splits, B * n, 3 * H * 128] are the qkv split-K partials; q and the new K/V row are reduced,
 * rounded to bf16 and rotated at position *pos_ptr, and the row is stored at row-cache index *pos_ptr - P.  Row r attends to its
 * image's prefix and its own positions P .. *pos_ptr; the caller keeps P <= *pos_ptr < P + row_cap.  out bf16 [B * n, H * 128].
 * pdl: programmatic stream serialisation. */
#define GROMA_GROUP_MAX_PROMPTS 64
int32_t groma_decode_rope_attention_grouped(const float* ws, int32_t splits, const void* prefix_k, const void* prefix_v,
                                            int32_t prefix_len, void* row_k, void* row_v, int64_t row_cap, const int32_t* pos_ptr,
                                            const float* cos_t, const float* sin_t, void* out, int32_t B, int32_t n, int32_t H,
                                            int32_t D, float scale, int32_t pdl, void* stream);
/* lp = log_softmax(logits) per row (4.32: `nn.functional.log_softmax(next_token_logits, dim=-1)`): the sum of exp(x - max) and
 * x - (max + log sum) are formed in double in a fixed order, then rounded to fp32. */
int32_t groma_beam_logsoftmax(const float* logits, int64_t ld, int32_t rows, int32_t V, float* lp, int64_t ld_out, void* stream);
/* Per row r: the K best of cand = scores[r] + beam_scores[r] (fp32 add), in decreasing order, a tie going to the lower token
 * (4.32's torch.topk leaves the order of ties unspecified; this is the defined rule).  cand_val fp32 / cand_tok int32 [rows, K],
 * K <= GROMA_BEAM_MAX_K <= V.  One CTA per row stages the row in shared memory (the limit of groma_sample_tokens). */
int32_t groma_beam_topk(const float* scores, int64_t ld, int32_t rows, int32_t V, const float* beam_scores, int32_t K,
                        float* cand_val, int32_t* cand_tok, void* stream);
/* One scorer step per image (4.32 BeamSearchScorer.process, BeamHypotheses.add / is_done), then the beam update of
 * beam_search: merges the nb rows' K = 2 nb candidates by (value desc, flat index j * V + t asc); an EOS of rank < nb adds a
 * hypothesis (score = value / denom[cur_len], double; list semantics of BeamHypotheses kept in hyp_order), an EOS of rank >= nb
 * is skipped, other tokens fill the nb next beams; fewer than nb filled sets flags[1] = 1 (4.32 raises ValueError).
 * done[b] |= is_done(rank-0 value, cur_len).  A done image takes pad tokens, score 0 and parent beam 0 of the image.  Then
 * ids / parents / beam_scores are written, the history rows and src rows are reordered by parent (staged through hist_tmp /
 * src_tmp), hist[r][cur_len] = token, src[r][cur_len - L0] = r, and the last CTA sets *cur_len += 1 and flags[0] = all done.
 * params int32 (device): {early_stopping (0 False, 1 True, 2 "never"), max_length, L0, pad_token_id, n_eos,
 * never_uses_max_length (early_stopping "never" and length_penalty > 0), up to 10 eos ids}; denom fp64 [max_length + 1]: n **
 * length_penalty as Python computes it.  Every knob is device data, so one captured graph serves every setting.
 * Hypothesis store per image: hyp_count, worst (fp64, starts at 1e9), hyp_order [nb] (list order -> slot), and per slot
 * hyp_score (fp64), hyp_len (generated tokens) and hyp_tok [gen_cap]. */
typedef struct GromaBeamArgs {
    int32_t B, nb, V, K;          /* images, beams per image, vocabulary, candidates per row (2 nb) */
    int32_t hist_cap, gen_cap;    /* row capacity of hist / hist_tmp, of src / src_tmp / hyp_tok */
    const float* cand_val;        /* [B * nb, K] */
    const int32_t* cand_tok;      /* [B * nb, K] */
    const int32_t* params;
    const double* denom;
    int32_t* cur_len;             /* the history length (device scalar, shared with groma_logits_process) */
    float* beam_scores;           /* [B * nb] */
    int64_t* ids;                 /* [B * nb] next tokens */
    int32_t* parents;             /* [B * nb] parent row */
    int32_t* hist; int32_t* hist_tmp;
    int32_t* src; int32_t* src_tmp;
    int32_t* hyp_tok; int32_t* hyp_len; double* hyp_score; int32_t* hyp_order; int32_t* hyp_count; double* worst;
    int32_t* done;                /* [B] */
    int32_t* flags;               /* [3]: all done, status, CTA ticket (kept 0 between launches) */
} GromaBeamArgs;
int32_t groma_beam_select(const GromaBeamArgs* args /*host*/, void* stream);

/* ---- 4-bit NF4 weights (bitsandbytes nf4, block 64, no double quant; DESIGN.md section 4) ---------------------------------
 * Replace bitsandbytes' quantize_4bit / dequantize_4bit / gemv_4bit, which HF 4.32 calls for every nn.Linear of a model loaded
 * with BitsAndBytesConfig(load_in_4bit=True, bnb_4bit_quant_type='nf4') (groma/eval/run_groma.py:43-61).
 * w: the bf16 weight flattened row-major, numel elements, in blocks of 64 (the last may be shorter).
 * absmax_b = max|w| (fp32); s = w * (1.0f / absmax_b); code = dQuantizeNF4(s) (strict > against the fp32 midpoints of the
 * codebook; an all-zero block gives code 0); codes: uint8 [(numel + 1) / 2], even element in the high nibble.
 * Dequantised value W~ = bf16_rn(fp32(bf16_rn(NF4[code])) * absmax_b); out bf16 [numel] (4-byte aligned). */
int32_t groma_nf4_quantize(const void* w, int64_t numel, void* codes, float* absmax, void* stream);
int32_t groma_nf4_dequantize(const void* codes, const float* absmax, int64_t numel, void* out, void* stream);
/* The same W~ [n_rows, K] (row-major bf16, K % 64 == 0) from the decode tile layout below: the per-projection dequantisation in
 * front of the bf16 prefill GEMMs of a 4-bit model (bitsandbytes' own multi-token strategy). */
int32_t groma_nf4_dequantize_tiles(const void* codes, const float* absmax, int32_t n_rows, int32_t K, void* out, void* stream);

/* ws = W~[n_rows, K] @ x[n_tok, K]^T as raw fp32 split-K partials, W~ dequantised on chip from NF4 codes + absmax in the decode
 * tile layout of csrc/gemm_nf4.cuh (groma_b200.ops.nf4_tile).  The NF4 counterpart of groma_gemm_bf16's swap-AB decode call
 * (weights as the 128-row operand, GROMA_GF_PARTIAL, BN = 16): same split-K ranges and k order, so with the same split_k the
 * partials equal those of groma_gemm_bf16 on a bf16 tensor holding W~.  flags: GROMA_GF_PARTIAL_T (ws[split][n][m], else
 * ws[split][m][n]) | GROMA_GF_PDL (weights prefetched before waiting for the previous kernel).  K % 64 == 0; any n_tok (tiles of
 * 16 tokens: more than 16 re-read each weight tile once per token tile, mostly from L2). */
int32_t groma_gemm_nf4_swap_ab(const void* x, int64_t ldx, int32_t n_tok, const void* codes, const float* absmax,
                               int32_t n_rows, int32_t K, float* ws, int32_t split_k, int32_t flags, void* stream);

/* ---- FP8 (e4m3) KV cache (opt-in, DESIGN.md section 4) ----------------------------------------------------------------------
 * One fp32 scale per 128-element head vector x (bf16 values): s = fp32(amax / 448) (IEEE division), code_i =
 * e4m3_rn_satfinite(fp32(x_i) / s); amax = 0 gives s = 0 and every code +0, so no NaN is ever stored.  Dequantised value
 * x^_i = fp32(code_i) * s.  Rows are addressed as n_groups groups of `rows` consecutive 128-element rows; group g starts at
 * row g * src_gs of the source and g * dst_gs of the destination (a [.., cap, 128] cache, or a [.., T, 128] staging buffer).
 *   kv_quantize  : bf16 src (8-byte aligned) -> uint8 codes + fp32 scales
 *   kv_dequantize: codes + scales -> bf16 out = bf16_rn(x^) */
int32_t groma_kv_quantize(const void* src, int64_t src_gs, int32_t n_groups, int32_t rows, void* codes, float* scales, int64_t dst_gs,
                          void* stream);
int32_t groma_kv_dequantize(const void* codes, const float* scales, int64_t src_gs, int32_t n_groups, int32_t rows, void* out,
                            int64_t dst_gs, void* stream);

/* ---- FP8 (e4m3) LLaMA weights (opt-in, DESIGN.md section 4) ------------------------------------------------------------------
 * Row quantiser: the rule of groma_kv_quantize applied to whole rows of a bf16 [M, K] matrix (row stride lds): one fp32 scale
 * per row into scales[M], the e4m3 codes into codes [M, K] (row stride ldc).  Used at load for every q/k/v/o/gate/up/down
 * weight (replacing the bf16 copy into the projection arenas) and before every fp8 GEMM for its input rows.  K, lds, ldc % 8 == 0.
 * pdl: launched with programmatic stream serialisation (it releases its dependents at entry and waits for its producer). */
int32_t groma_fp8_quantize_rows(const void* src, int64_t lds, int32_t M, int32_t K, void* codes, int64_t ldc, float* scales,
                                int32_t pdl, void* stream);
/* groma_gemm_bf16 with e4m3 codes as A [a_rows, K] and B [b_rows, K] (K-major, lda / ldb / K % 16 == 0) and their fp32 row scales
 * scale_a [M], scale_b [N]: the fp32 accumulator (promoted into a second register set after every 64-deep k chunk) is multiplied
 * by fp32(scale_a[m] * scale_b[n]) before the unchanged epilogue, or before a split-K partial is stored.  Replaces
 * groma_gemm_bf16 for the LLaMA projections of an fp8-weight model: the prefill calls (A = activations, B = weights; the qkv
 * projection takes this + groma_rope_kv instead of groma_gemm_qkv_rope) and the swap-AB decode calls (A = weights, B = <= 16
 * activation rows, GROMA_GF_PARTIAL[_T], GROMA_GF_PDL, tile_counters).  No bias / LayerScale / taps / tiled A; block_n: 0
 * (auto, at most 128), 16, 32, 64 or 128. */
int32_t groma_gemm_fp8(const void* A, int64_t a_rows, int64_t lda, const float* scale_a, const void* B, int64_t b_rows, int64_t ldb,
                       const float* scale_b, int32_t M, int32_t N, int32_t K, void* out, int64_t ld_m, int64_t ld_n, int32_t flags,
                       int32_t act, const void* residual, float* ws, int32_t split_k, int32_t* tile_counters, int32_t block_n,
                       void* stream);

int32_t groma_cast_f32_bf16(const float* a, void* b, int64_t n, void* stream);
int32_t groma_cast_bf16_f32(const void* a, float* b, int64_t n, void* stream);

/* ---- image preprocessing in front of the ViT (SURVEY.md §8f N3) ----------------------------------------------------------
 * Replaces, per image, the reference's CPU pass  PIL `Image.resize((448, 448))` (BICUBIC, uint8; groma/eval/run_groma.py:78,
 * groma/data/datasets/groma.py:94) + `BitImageProcessor.preprocess` with do_resize=False, do_center_crop=False (rescale 1/255,
 * ImageNet mean/std, CHW float32; run_groma.py:79, run_ddetr.py:39-45).
 * img: uint8 RGB, HWC, row_stride bytes between rows (device).  The resize reproduces Pillow's two-pass fixed-point resampler
 * bit for bit.  lut: float32 [3][256] = normalised value of every byte per channel (host computes it once with the processor's
 * mean/std).  tmp: uint8 [H][out_size][3] scratch.  coef: int32 scratch of GROMA_PREPROCESS_COEF_INTS(out_size).
 * out_f32: float32 [3][out_size][out_size] pixel_values (may be null), out_u8: resized uint8 [out_size][out_size][3] (may be null).
 * Sides up to 15 x out_size. */
#define GROMA_PREPROCESS_COEF_INTS(out_size) (2 * (out_size) * (2 + 64))
int32_t groma_preprocess_image(const uint8_t* img, int32_t H, int32_t W, int64_t row_stride, const float* lut,
                               int32_t out_size, uint8_t* tmp, int32_t* coef, float* out_f32, uint8_t* out_u8, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GROMA_B200_H */
