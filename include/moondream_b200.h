/*
 * moondream_b200 — C-ABI of the H100-native (sm_90a) moondream hot path (libmoondream_b200.so).
 *
 * Conventions (all entry points):
 *   - plain pointers and sizes; device pointers unless marked HOST; bf16 = raw uint16 storage;
 *   - `stream` is a cudaStream_t passed as void*; entry points never synchronise and never
 *     allocate device memory: the caller passes outputs and workspaces (see the *_workspace_bytes
 *     queries); all launches are CUDA-graph capturable;
 *   - return 0 on success, non-zero on error; md_last_error() returns the message (thread-local);
 *   - leading dimensions (`ld*`) and strides are in elements.
 *
 * The reference (vikhyat/moondream, /root/reference) has no FFI: its swap seam is the four bound
 * methods MoondreamModel._vis_enc/_vis_proj/_prefill/_decode_one_tok (moondream/torch/moondream.py
 * :168-192) that compile() rebinds (:194-204).  The model-level entry points below are those four
 * methods generalised with a leading batch dimension; each cites the reference lines whose
 * arithmetic it replaces.  INTEGRATION.md shows the ctypes stubs that bind them.
 */
#ifndef MOONDREAM_B200_H
#define MOONDREAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MD_ABI_VERSION 3

/* epilogue selectors for the linear entry points */
#define MD_EPI_BIAS 0          /* y = bf16(x W^T + b)                        layers.py:34-35   */
#define MD_EPI_BIAS_GELU 1     /* y = bf16(gelu_tanh(bf16(x W^T + b)))       layers.py:130,137 */
#define MD_EPI_BIAS_RESIDUAL 2 /* y = bf16(bf16(x W^T + b) + r)              vision.py:70-71, text.py:158 */

#define MD_PAGE_TOKENS 64      /* tokens per KV page */

const char* md_last_error(void);
int md_abi_version(void);
/* number of kernels this library has launched since the last reset (bench.py's gpu_launches) */
long long md_launch_count(void);
void md_reset_launch_count(void);
/* Optional CUDA-event timing around every md_linear_bf16-class launch made outside graph capture
 * (bench.py's roofline leg): enable, run, then read the summed device time, algorithmic FLOPs
 * (2*M*N*K) and launch count.  md_profile_linear_read synchronises on the recorded events. */
void md_profile_linear(int enable);
int md_profile_linear_read(double* total_ms, double* total_flops, long long* launches);
/* Kept for ABI compatibility: sm_90 has no CTA-pair MMA, so every row-form tile is one CTA whatever the argument. */
void md_debug_force_cta_group(int cta_group);

/* ------------------------------------------------------------------------------------------------
 * Operator level
 * ---------------------------------------------------------------------------------------------- */

/*
 * y[M,N] = epilogue(x[M,K] @ w[N,K]^T + bias[N])            (wgmma + TMA GEMM, bf16 in/out)
 * Replaces F.linear at layers.py:35 and its nn.Linear call sites vision.py:67 (patch_emb),
 * layers.py:159-165 (ViT qkv/proj), layers.py:130,139 (fc1/fc2), vision.py:89 (proj_mlp),
 * text.py:30,53 (decoder qkv/proj) for prefill-sized M.
 *   residual: [*, N] rows of stride ldr; when res_mod > 0 the residual row is (row % res_mod)
 *             (pos_emb broadcast over crops, vision.py:68).
 *   remap:    when remap_gin > 0 output row r is written at (r / gin) * gout + r % gin + goff
 *             (places the 729 projected image rows after the BOS row, moondream.py:254).
 * Requirements: N % 8 == 0, K % 8 == 0, 16-byte aligned pointers and row pitches.
 */
int md_linear_bf16(const void* x, long long ldx, const void* w, long long ldw, int M, int N, int K,
                   int epilogue, const void* bias, const void* residual, long long ldr, int res_mod,
                   void* out, long long ldo, int remap_gin, int remap_gout, int remap_goff,
                   void* stream);

/*
 * Same contraction for a small batch (decode step, LM head, region head): the weight matrix is the
 * M side of the MMA so every SM streams weights at HBM rate; K is split across CTAs and the fp32
 * partial sums are reduced in a fixed order (deterministic).  Replaces the M=1 F.linear calls the
 * reference issues per generated token (text.py:30,53,166; layers.py:130,139; region.py:43-93).
 */
int md_linear_small_batch_splits(int n_out, int K);
long long md_linear_small_batch_workspace_bytes(int n_out, int batch, int K);
int md_linear_small_batch_bf16(const void* x, long long ldx, const void* w, long long ldw, int batch,
                               int n_out, int K, int epilogue, const void* bias, const void* residual,
                               long long ldr, void* out, long long ldo, void* workspace, void* stream);

/* dequantize_tensor (layers.py:38-44) for a stream-layout matrix: out bf16 [N][K] (row pitch ldo) =
 * bf16( bf16(q - zero) * scale ); bits in {4, 8}, K % 128 == 0. */
int md_dequantize_weights(int bits, const void* wq, const float* scale, const float* zero, int N, int K, void* out,
                          long long ldo, void* stream);
/* md_linear_small_batch_bf16 with packed weights (see md_model_set_quantized_block for the layout): the result
 * equals md_linear_small_batch_bf16 on the dequantised matrix bit for bit (same split plan and summation order). */
int md_linear_small_batch_quant(int bits, const void* x, long long ldx, const void* wq, const float* scale,
                                const float* zero, int batch, int n_out, int K, int epilogue, const void* bias,
                                const void* residual, long long ldr, void* out, long long ldo, void* workspace,
                                void* stream);

/*
 * Image preprocessing on the device: the resize of overlap_crop_image (image_crops.py:124-150, PIL branch) as the two
 * passes of Pillow's 8-bit resampler (libImaging/Resample.c).  One call = one pass over a uint8 HWC image with 3
 * channels: axis 1 resizes the width (in_w -> out_size), axis 0 the height.  bounds int32 [out_size][2] = (first
 * source index, taps), coeffs int32 [out_size][ksize] = Pillow's 22-bit fixed-point Lanczos-3 weights
 * (moondream_b200/resample.py computes them with Pillow's expressions); out = clamp((2^21 + sum src * coeff) >> 22).
 * Bit-exact against PIL.Image.resize(..., LANCZOS).  md_extract_windows_u8 cuts the rows x cols overlapping
 * crop x crop windows (stride = crop - 2 * margin pixels, image_crops.py:152-165) out of the resized canvas.
 */
int md_resample_u8(const uint8_t* src, int in_h, int in_w, int axis, const int* bounds, const int* coeffs, int ksize,
                   int out_size, uint8_t* dst, void* stream);
int md_extract_windows_u8(const uint8_t* canvas, int h, int w, int rows, int cols, int stride, int crop, uint8_t* crops,
                          void* stream);

/* y = LayerNorm(x) * w + b, eps 1e-5, fp32 statistics (layers.py:118-119). dim % 8 == 0, <= 4096. */
/* prepare_crops' normalisation + create_patches (vision.py:36-40, 44-61): crops uint8 NHWC [n_crops, crop, crop, 3] ->
 * patches bf16 [n_crops * (crop / patch)^2, k_pad], feature order (channel, row, column) as the reference's
 * reshape/permute produces, columns [3 * patch^2, k_pad) zero; pixel_lut = bf16[256], the reference's op chain per byte. */
int md_patchify_u8(const uint8_t* crops, int n_crops, int crop, int patch, int k_pad, const void* pixel_lut, void* out,
                   void* stream);
/* reconstruct_from_crops(patch_size = 1) + adaptive_avg_pool2d + concat (image_crops.py:170-231, vision.py:83-88) for a
 * batch: feats bf16 [sum crops * grid^2, dim] (crop 0 of each image = global) -> out bf16 [n_images * grid^2, 2 * dim]
 * = [global | pooled stitched local]; crop_offsets [n_images + 1], tilings [n_images][2] (device int32). */
int md_stitch_pool_concat_bf16(const void* feats, const int* crop_offsets, const int* tilings, int n_images, int grid,
                               int margin, int dim, void* out, void* stream);
int md_layernorm_bf16(const void* x, long long ldx, const void* w, const void* b, void* y,
                      long long ldy, int rows, int dim, void* stream);

/*
 * ViT self-attention over the fused qkv activations (layers.py:155-166): qkv [n_crops*seq, 3*H*72]
 * -> out [n_crops*seq, H*72]; softmax(QK^T / sqrt(72)) V, no mask.
 */
int md_vit_attention_bf16(const void* qkv, int n_crops, int seq, int n_heads, void* out, void* stream);

/* Paged KV cache handle: pool bf16 [layers][n_pages][2][kv_heads][64 tokens][64 dims];
 * block_tables int32 [n_seqs][max_blocks] (page of positions 64*i..64*i+63 of each sequence). */
typedef struct md_kv {
  void* pool;
  int n_pages;
  const int* block_tables;
  int max_blocks;
  int n_layers;            /* layers in the pool (bounds the TMA view of the pool) */
  int n_kv_heads;          /* heads in the pool; 0 = as many as query heads.  Fewer = grouped-query attention
                            * (text.py:49 enable_gqa): query head h reads KV head h / (n_heads / n_kv_heads) */
} md_kv;

/* Partial RoPE (first 32 of 64 dims, split-half in / interleaved out, rope.py:20-48) on q and k of
 * fused qkv [tokens, 3*H*64]; q -> q_out [tokens, H*64]; k, v -> KV pages (moondream.py:74-78).
 * q_offsets == NULL means one token per sequence at position start_pos[seq] (decode). */
/* (multi-head layout only: kv->n_kv_heads must be 0 or n_heads; grouped-query models go through the model-level
 * entry points, whose QKV epilogues handle the narrower k / v column blocks) */
int md_rope_kv_write_bf16(const void* qkv, int n_tokens, int n_heads, const int* q_offsets,
                          const int* start_pos, int n_seqs, const float* rope_table, void* q_out,
                          const md_kv* kv, int layer, void* stream);

/* Prefix-LM attention for prefill (text.py:46-50 under the mask of moondream.py:138-146):
 * wgmma/TMA flash attention; q / out are [total_tokens, H*64].  The pool must hold finite values
 * in unused slots (zero-initialise it): masked keys still flow through the P V product as 0 * v. */
int md_prefill_attention_bf16(const void* q, int n_heads, int total_tokens, const int* q_offsets,
                              const int* start_pos, int n_seqs, int max_q, int prefix_len,
                              const md_kv* kv, int layer, void* out, void* stream);
/* Testing / A-B timing only: 1 = the legacy mma.sync kernels, 4 = the wgmma kernels launched with one CTA per work item
 * instead of persistent CTAs; any other value = the wgmma kernels with persistent CTAs (the default).
 * Decode attention (md_decode_attention_bf16 and the decode step): 2 = the kernel that loads K/V into registers instead
 * of the one streaming them through a bulk-copy ring (the same bits).  Prefill and ViT attention treat 2 as the
 * default. */
void md_debug_attention_impl(int impl);
/* Testing / A-B timing only: programmatic dependent launch between consecutive kernels (default on). */
void md_debug_set_pdl(int enable);
/* Ablation timing only (results are garbage when non-zero): skip kernels of md_text_decode_step;
 * bit0 [qkv;fc1] GEMM, bit1 its epilogue, bit2 attention, bit3 [proj|fc2] GEMM, bit4 residual+LN epilogue. */
void md_debug_skip_decode_kernels(int mask);
/* Timing experiments only: bit5 stops the row-form GEMM from releasing its dependent grid early (programmatic dependent
 * launch); bit7 runs the patch embedding as patchify kernel + row-form GEMM instead of the im2col-fused kernel; bit8
 * makes the row-form GEMM use 128-wide column tiles for every N >= 96 instead of the planned 192 / 256 (same results,
 * for A/B timing and tests).  Other bits are ignored. */
void md_debug_gemm(int flags);
/* Experiments only: cap the persistent row-form GEMM's grid at `sms` SMs (0 = all, the default), leaving the others
 * to kernels of a concurrent stream (encode / decode overlap experiments). */
void md_debug_gemm_sm_cap(int sms);
/* Profiling only: while `records` is non-NULL every CTA of the decode-step kernels (weight-stream GEMMs, decode
 * attention, residual+LayerNorm epilogue) appends one record of 6 uint64 to records[capacity][6]:
 * {tag << 32 | block, t_entry, t_after_dependency_wait, t_mid0, t_mid1, t_exit} in %globaltimer ns; tag bits 31..28:
 * 1 GEMM (bits 27..24 epilogue mode, 23..0 rows), 2 decode attention, 3 residual+LN epilogue.  `count` is a
 * device uint32 the caller zeroes.  Pass NULL to remove.  (tools/decode_timeline.py) */
int md_debug_timeline(void* records, void* count, unsigned int capacity);

/* One-query attention for decode (text.py:46-50 with the [1,1,2048] mask of moondream.py:472-474). */
int md_decode_attention_bf16(const void* q, int n_heads, const int* pos, int n_seqs, const md_kv* kv,
                             int layer, void* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Model level (the four seam methods, batched)
 * ---------------------------------------------------------------------------------------------- */
typedef struct md_dims {
  /* vision (VisionConfig, config.py:19-31); vis_ff and patch_k are the PADDED sizes the prepared
   * weights use (multiples of 8: 588 -> 592, 2690 -> 2696) */
  int vis_dim, vis_ff, vis_layers, vis_heads, crop, patch, patch_k, grid, margin, proj_inner;
  /* text (TextConfig, config.py:5-15) */
  int txt_dim, txt_ff, txt_layers, txt_heads, vocab, max_context, prefix_len;
  /* region (RegionConfig, config.py:34-41) */
  int reg_inner, coord_feat, coord_out, size_feat, size_out;
  /* 1: the decoder weights use the fused decode layout.  Per text block the canonical pointers are
   * views into two buffers:  W1 = [qkv.weight ; fc1.weight]  ([3D + FF, D], bias likewise), and
   * W2 = [proj.weight | fc2.weight]  ([D, D + FF], row pitch D + FF).  md_model_create checks the
   * pointer relationships.  md_text_decode_step requires it (one weight stream per pair). */
  int txt_fused;
  /* KV heads of the decoder (TextConfig.n_kv_heads, config.py:13); 0 = txt_heads.  qkv.weight then has
   * txt_dim + 2 * txt_kv_heads * 64 rows (text.py:36-38) and the KV pool txt_kv_heads heads. */
  int txt_kv_heads;
} md_dims;

typedef struct md_model md_model;

/* Number of weight tensors md_model_create expects: the canonical state_dict order of the
 * reference (SURVEY.md §2.4; moondream_b200/synth.py:state_dict_spec). */
int md_model_num_weights(const md_dims* dims);

/*
 * weights: HOST array of device pointers in canonical order (bf16, contiguous, prepared/padded);
 * pixel_lut: device bf16[256] = the reference's pixel normalisation chain (vision.py:36-40);
 * rope_table: device f32 [max_context][16][2] = precompute_freqs_cis (rope.py:6-17, text.py:215-219).
 * The model object only stores pointers (host memory); it owns no device memory.
 */
int md_model_create(const md_dims* dims, const void* const* weights, int n_weights,
                    const void* pixel_lut, const float* rope_table, md_model** out);
void md_model_destroy(md_model* model);

/*
 * Weight-only quantised decoder blocks — the reference's int4 group-128 QuantizedLinear (layers.py:38-110, selected by
 * TextConfig.group_size, text.py:178) and int8.  Per block the packed tensors of the two fused decode streams, in the
 * STREAM layout (moondream_b200/quant.py converts the reference checkpoint layout; values untouched):
 *   bits = 4: wq[n][K / 2] bytes, low nibble = input feature 2j, high nibble = 2j + 1;  bits = 8: wq[n][K] signed bytes;
 *   scale / zero: fp32 [n][K / 128];   W[n][k] = bf16( bf16(q - zero) * scale )   (dequantize_tensor, layers.py:38-44)
 *   W1 = [qkv ; fc1]: n = txt_dim + 2 * txt_kv_heads * 64 + txt_ff rows, K = txt_dim;
 *   W2 = [proj | fc2]: n = txt_dim rows, K = txt_dim + txt_ff (groups never straddle the boundary).
 * Call it for EVERY block.  The bf16 weight pointers of all decoder blocks given to md_model_create must then alias
 * ONE scratch pair (W1 / W2): md_text_prefill(_lora) rebuilds block i's bf16 weights there before its GEMMs, and
 * md_text_decode_step streams the packed bytes (a quarter / half of the bf16 traffic), producing bit for bit what the
 * bf16 path produces on W.  The model stores the pointers only.
 */
int md_model_set_quantized_block(md_model* model, int layer, int bits, const void* w1q, const float* w1_scale,
                                 const float* w1_zero, const void* w2q, const float* w2_scale, const float* w2_zero);

/* _vis_enc (vision.py:64-74 + prepare_crops' normalisation :36-40 + create_patches :44-61):
 * crops uint8 NHWC [n_crops, crop, crop, 3] -> feats bf16 [n_crops * grid^2, vis_dim]. */
long long md_vision_encode_workspace_bytes(const md_model* model, int n_crops);
int md_vision_encode(md_model* model, const uint8_t* crops, int n_crops, void* feats, void* workspace,
                     void* stream);

/* reconstruct_from_crops + _vis_proj (image_crops.py:170-231, vision.py:77-89) for n_images at once:
 * crop_offsets int32 [n_images+1] (first crop of an image is its global crop), tilings int32
 * [n_images][2].  Writes the projected rows of image i to embeds rows i*prefix_len+1 .. +grid^2
 * (row i*prefix_len is left for the BOS embedding, moondream.py:250-254); embeds is
 * [n_images*rows_per_image, txt_dim] bf16 with rows_per_image >= prefix_len (prefix_len when 0 is passed): a larger
 * value leaves room after each image for prompt embeddings so image and prompt prefill in one pass. */
long long md_vision_project_workspace_bytes(const md_model* model, int n_images);
int md_vision_project(md_model* model, const void* feats, const int* crop_offsets, const int* tilings,
                      int n_images, void* embeds, int rows_per_image, void* workspace, void* stream);

/* `_vis_proj(g, r)` with the reference's own signature (moondream.py:171-172, vision.py:77-89) for one image:
 * global_feats bf16 [grid^2, vis_dim], stitched bf16 [height, width, vis_dim] (reconstruct_from_crops' output)
 * -> out bf16 [grid^2, txt_dim].  Workspace: md_vision_project_workspace_bytes(model, 1). */
int md_vision_project_stitched(md_model* model, const void* global_feats, const void* stitched, int height, int width,
                               void* out, void* workspace, void* stream);

/* text_encoder (text.py:12-13): out[i] = wte[ids[i * id_stride]]. */
int md_embed_tokens(md_model* model, const int* ids, long long id_stride, int n, void* out,
                    long long ldo, void* stream);

/* _prefill (text.py:128-160) over a ragged batch: x [total_tokens, txt_dim] embeddings in, hidden
 * states out (in place); sequence s owns rows q_offsets[s]..q_offsets[s+1] at positions
 * start_pos[s]...; K/V are written to the pages.
 * prefix_len: positions < prefix_len attend bidirectionally among themselves (the image prefix of
 * moondream.py:143-145); -1 = the model's (730); 0 = pure causal, which is the mask the reference builds for
 * a text-only query (moondream.py:565-574). */
long long md_text_prefill_workspace_bytes(const md_model* model, int total_tokens);
int md_text_prefill(md_model* model, void* x, int total_tokens, const int* q_offsets,
                    const int* start_pos, int n_seqs, int max_q, int prefix_len, const md_kv* kv,
                    void* workspace, void* stream);

/* _prefill under a LoRA variant (settings["variant"], lora.py:55-79): text.py:31-32,54-56 and layers.py:131-143 add
 * `B (A x)` to every Linear of a decoder block.  lora: HOST array of 8 * txt_layers device pointers, per block
 * (A_qkv [r, D], B_qkv [3D, r], A_proj [r, D], B_proj [D, r], A_fc1 [r, D], B_fc1 [FF, r], A_fc2 [r, FF], B_fc2 [D, r]),
 * bf16, row-major; rank r a multiple of 8.  Same arguments and cache behaviour as md_text_prefill otherwise; one row
 * per sequence (q_offsets = 0, 1, 2, ...) makes it the decode step under a variant. */
long long md_text_prefill_lora_workspace_bytes(const md_model* model, int total_tokens, int rank);
int md_text_prefill_lora(md_model* model, void* x, int total_tokens, const int* q_offsets, const int* start_pos,
                         int n_seqs, int max_q, int prefix_len, const md_kv* kv, const void* const* lora, int rank,
                         void* workspace, void* stream);

/* _decode_one_tok's decoder half (text.py:128-160 with T=1) for `batch` sequences:
 * x [batch, txt_dim] embeddings in, hidden out (in place); pos int32 [batch] (device).
 * normed_out (optional) receives post_ln(hidden) [batch, txt_dim] (text.py:165) computed by the last
 * block's fused epilogue; pass it to md_lm_head_argmax with prenormed = 1.
 * Per block: one [qkv;fc1] weight stream, RoPE/KV-write/GELU epilogue, paged attention, one
 * [proj|fc2] weight stream, residual + next-LayerNorm epilogue (5 launches). */
long long md_text_decode_workspace_bytes(const md_model* model, int batch);
int md_text_decode_step(md_model* model, void* x, const int* pos, int batch, const md_kv* kv,
                        void* normed_out, void* workspace, void* stream);

/* lm_head + greedy argmax (text.py:163-167, moondream.py:313-314,517-524): hidden rows
 * [batch] x txt_dim (stride ld_hidden).  Token ids go to out_ids[b * out_stride + *out_index]
 * (out_index: device int or NULL = 0); mask_id / mask_id2 >= 0 are excluded (answer_id in
 * _generate_answer, moondream.py:517; eos_id and size_id in _generate_reasoning, :395-396).
 * prenormed != 0: `hidden` already holds post_ln(hidden) (from md_text_decode_step's normed_out).
 * Optional: out_margin (same addressing, top1 - top2 of the bf16 logits), out_logits bf16 [batch, vocab]. */
long long md_lm_head_workspace_bytes(const md_model* model, int batch);
int md_lm_head_argmax(md_model* model, const void* hidden, long long ld_hidden, int prenormed, int batch,
                      int mask_id, int mask_id2, int* out_ids, long long out_stride, const int* out_index,
                      float* out_margin, void* out_logits, void* workspace, void* stream);

/* Temperature / top-p sampling on the device (moondream.py:270-278 `_apply_top_p`, :312-318, :524-530), one CTA per
 * sequence, no sort: probs = softmax(logits / temperature) rounded like the reference's bf16 tensors; the kept set
 * is the prefix of (probability descending, index ascending) order whose preceding mass, in the reference's bf16
 * arithmetic, does not exceed top_p (found through a histogram of probability values); the kept probabilities are
 * renormalised and one token is drawn by inverse CDF in index order from a uniform u: uniforms[b] when given
 * (tests), else Philox4x32-10 keyed by *seed with counter (b, *step + out_offset), so CUDA-graph replays draw fresh
 * numbers as the device-side step advances.  logits bf16 [batch, vocab] (md_lm_head_argmax's out_logits, masks
 * already applied); scratch bf16 [batch, vocab]; when keep_probs != 0 scratch returns the reference's `next_probs`.
 * The token goes to out_ids[b * out_stride + *step + out_offset] (step NULL = 0). */
int md_sample_top_p(const void* logits, int batch, int vocab, float temperature, float top_p,
                    const unsigned long long* seed, const int* step, const float* uniforms, void* scratch,
                    int keep_probs, int* out_ids, long long out_stride, int out_offset, void* stream);

/* text_encoder with substitution (moondream.py:381-391): out[i] = ids[i*id_stride] == sel_id ? alt[i] : wte[id]. */
int md_embed_tokens_select(md_model* model, const int* ids, long long id_stride, int n, int sel_id,
                           const void* alt, long long ld_alt, void* out, long long ldo, void* stream);

/* dst[i * stride + *index + offset] = src[i] (per-step record of decoded coordinates; index NULL = 0). */
int md_store_column_f32(const float* src, int n, float* dst, long long stride, const int* index, int offset,
                        void* stream);

/* Decode-loop bookkeeping on the device (the generator loop of moondream.py:481-530 without the
 * per-token .item() sync): cur_tok[b] = (forced ? forced : preds)[b*stride + step+1]; pos[b] += 1;
 * finished[b] |= (cur_tok[b] == eos_id); step += 1. */
int md_decode_advance(int* cur_tok, int* pos, int* step, const int* preds, const int* forced,
                      long long stride, int batch, int eos_id, int* finished, void* stream);

/* out[i, :] = src[row_index[i], :] (picks each sequence's last prompt row, text.py:164). */
int md_gather_rows_bf16(const void* src, long long ld_src, const int* row_index, int n, int dim,
                        void* out, long long ldo, void* stream);

/* Region head (region.py).  which: 0 = coordinate (decode: 1024 bins -> out_bins [batch]),
 * 1 = size (decode: view(2,-1) -> out_bins [batch][2] = (w_bin, h_bin)). */
long long md_region_workspace_bytes(const md_model* model, int batch);
int md_region_decode(md_model* model, int which, const void* hidden, long long ld_hidden, int batch,
                     int* out_bins, void* workspace, void* stream);
/* values fp32 [batch][1 or 2] (coordinate in [0,1] / (w, h)); out bf16 [batch, txt_dim]
 * (region.py:32-43, 60-71 incl. fourier_features :12-29). */
int md_region_encode(md_model* model, int which, const float* values, int batch, void* out,
                     long long ldo, void* workspace, void* stream);
/* bins -> values (moondream.py:673,683,701-702): coord = bin / n_bins (n_bins = coord_out_dim, the size of the
 * logits' last dimension); size = 2^(bin/1023*10 - 10) (the reference hard-codes 1023). */
int md_region_bins_to_values(int which, const int* bins, int n, int n_bins, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Native checkpoint reader (replaces the file-reading half of load_weights_into_model, weights.py:156-171)
 * ---------------------------------------------------------------------------------------------- */
/* safetensors file -> mmap + parsed header.  md_safetensors_info: name / dtype strings live as long as the handle;
 * shape8 receives up to 8 extents.  md_safetensors_read copies one tensor's bytes (dst_bytes must equal its size)
 * from the mapping into device memory (cudaMemcpyAsync on `stream`; the mapping must stay open until the stream has
 * drained) or, with dst_is_device == 0, into host memory. */
typedef struct md_file md_file;
int md_safetensors_open(const char* path, md_file** out);
int md_safetensors_count(const md_file* file);
int md_safetensors_info(const md_file* file, int index, const char** name, const char** dtype, int* ndim,
                        long long* shape8, long long* nbytes);
int md_safetensors_find(const md_file* file, const char* name);
int md_safetensors_read(const md_file* file, int index, void* dst, long long dst_bytes, int dst_is_device, void* stream);
void md_safetensors_close(md_file* file);

#ifdef __cplusplus
}
#endif
#endif /* MOONDREAM_B200_H */
