// Internal (C++) interface between the kernel translation units and the C-ABI layer (api.cu).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace md {

// epilogue modes shared by the GEMM kernels (values are part of the C-ABI, see include/moondream_b200.h)
enum : int {
  EPI_BIAS = 0,            // out = bf16(acc + bias)
  EPI_BIAS_GELU = 1,       // out = bf16(gelu_tanh(bf16(acc + bias)))
  EPI_BIAS_RESIDUAL = 2,   // out = bf16(bf16(acc + bias) + residual)
  EPI_PARTIAL = 3,         // small-batch kernel: fp32 partial sums to workspace (timeline tag only)
  EPI_QKV_ROPE = 5,        // row form, decoder QKV projection: bias + partial RoPE, q -> q_out, k/v -> KV pages
};

// error plumbing: every entry point returns 0 on success; the message is kept per thread.
int set_error(const char* msg);
const char* last_error();
void count_launch();
long long launch_count();
void reset_launch_count();
int num_sms();

// cudaFuncSetAttribute is per device: one flag per (call site, device), so a second model on another GPU of the
// same process configures its kernels too.
struct DeviceOnce {
  bool done[64] = {};
  bool first() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 64) return true;
    if (done[d]) return false;
    done[d] = true;
    return true;
  }
};

// Launch with programmatic stream serialization (PDL) when enabled: the kernel must call pdl_wait()
// before touching memory its predecessor produced.
extern int g_pdl;
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = g_pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// debug timeline (ptx.cuh): each kernel translation unit holds its own __constant__ copy
struct Timeline;
int timeline_install_all(unsigned long long* buf, unsigned int* count, unsigned int cap);
void timeline_install_attention(const Timeline& t);
void timeline_install_elementwise(const Timeline& t);
void timeline_install_attention_tc(const Timeline& t);

// ---- gemm.cu ----
int make_tmap_bf16_2d(CUtensorMap* tm, const void* base, long long rows, long long cols,
                      long long ld, int box_rows);
int make_tmap_bf16_3d(CUtensorMap* tm, const void* base, long long d0, long long d1, long long d2,
                      long long s1_bytes, long long s2_bytes, int b0, int b1, int b2, int swizzle_bytes);
int make_tmap_u8_2d(CUtensorMap* tm, const void* base, long long rows, long long row_bytes, long long pitch_bytes,
                    int box_rows, int box_bytes);
int gemm_rowform(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M,
                 int N, int K, int mode, const __nv_bfloat16* bias, const __nv_bfloat16* res,
                 long long ldr, int res_mod, __nv_bfloat16* out, long long ldo, int remap_gin,
                 int remap_gout, int remap_goff, cudaStream_t stream);
void gemm_force_cta_group(int cg);
void gemm_debug_flags(int flags);
void gemm_debug_sm_cap(int sms);
void gemm_profile_enable(int on);
int gemm_profile_read(double* total_ms, double* total_flops, long long* launches);
struct StreamPlan { int tile_rows, kb, splits; };
StreamPlan plan_smallbatch(int n_out, int K, int kb_divisor);
int gemm_smallbatch_splits(int n_out, int K);
int gemm_smallbatch(const __nv_bfloat16* W, long long ldw, const __nv_bfloat16* X, long long ldx,
                 int n_out, int batch, int K, int splits, float* ws, cudaStream_t stream);
// Prefill QKV projection with RoPE and the KV-cache write fused into the GEMM epilogue (text.py:30-43,
// rope.py:20-48, moondream.py:74-78): output column block -> (q|k|v, head, half-head); row -> (sequence, position).
struct RopeEpilogue {
  int D, n_heads, n_kv_heads, n_seqs;   // n_kv_heads < n_heads: grouped-query attention (text.py:49 enable_gqa)
  const int* q_offsets;           // [n_seqs + 1] token rows of each sequence
  const int* start_pos;           // [n_seqs]
  const float* freqs;             // rope table [ctx][16][2]
  __nv_bfloat16* q_out;           // [tokens, D]
  __nv_bfloat16* kv_pool;
  int n_pages;
  const int* block_tables;
  int max_blocks, layer;
};
int gemm_rowform_qkv_rope(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M,
                          int K, const __nv_bfloat16* bias, const RopeEpilogue& epi, cudaStream_t stream);
// K-concatenated stream W = [A | B] (seg_K = width of A): no split straddles the boundary
struct StreamPlan2 { int tile_rows, splits_a, kb_a, splits_b, kb_b; };
StreamPlan2 plan_smallbatch_2seg(int n_out, int K, int seg_K);
int gemm_smallbatch_2seg(const __nv_bfloat16* W, long long ldw, const __nv_bfloat16* X, long long ldx,
                      int n_out, int batch, int K, int seg_K, float* ws, cudaStream_t stream);
// One weight stream (decode-time Linear): ws[split][b][n] fp32 partial sums of X[batch,K] * W[n_out,K]^T.
struct StreamArgs {
  int bits;                          // 16: bf16 W (ldw elements per row); 4 / 8: packed rows of K * bits / 8 bytes
  const void* W;
  long long ldw;
  const float* scale;                // packed only: [n_out][K / 128] fp32 scale and zero point per group of 128
  const float* zero;
  const __nv_bfloat16* X;
  long long ldx;
  int n_out, batch, K;
  int tile_n;                        // 64 or 128 weight rows per CTA
  int kb_per_split, seg_kb, kb_per_split2;   // seg_kb > 0: [0, seg_kb) and [seg_kb, K / 64) split separately
  float* ws;
};
int weight_stream(const StreamArgs& a, cudaStream_t stream);   // returns the number of splits, -1 on error
int splitk_epilogue(const float* ws, int splits, int B, int N, int mode, const __nv_bfloat16* bias,
                    const __nv_bfloat16* res, long long ldr, __nv_bfloat16* out, long long ldo,
                    cudaStream_t stream);

// ---- gemm_quant.cu: weight-only int4 (group 128) / int8 decode weight stream (layers.py:38-110) ----
int dequant_weights(int bits, const uint8_t* q, const float* scale, const float* zero, int N, int K,
                    __nv_bfloat16* out, long long ldo, cudaStream_t stream);
int gemm_smallbatch_quant(int bits, const uint8_t* Wq, const float* scale, const float* zero, const __nv_bfloat16* X,
                          long long ldx, int n_out, int batch, int K, int seg_K, float* ws, cudaStream_t stream);

// ---- patch_embed.cu: im2col-fused patch embedding (vision.py:25-68) ----
int patch_embed_fused(const uint8_t* crops, int n_crops, int crop, int patch, const __nv_bfloat16* lut,
                      const __nv_bfloat16* W, int k_pad, const __nv_bfloat16* bias, const __nv_bfloat16* pos_emb, int N,
                      __nv_bfloat16* out, cudaStream_t stream);
extern int g_patch_embed_unfused;

// ---- elementwise.cu ----
int layernorm(const __nv_bfloat16* x, long long ldx, const __nv_bfloat16* w, const __nv_bfloat16* b,
              __nv_bfloat16* y, long long ldy, int rows, int dim, float eps, cudaStream_t stream);
int patchify(const uint8_t* crops, int n_crops, int crop, int patch, int k_pad,
             const __nv_bfloat16* lut, __nv_bfloat16* out, cudaStream_t stream);
int stitch_pool_concat(const __nv_bfloat16* feats, const int* crop_offsets, const int* tilings,
                       int n_images, int grid, int margin, int dim, __nv_bfloat16* out,
                       cudaStream_t stream);
int gelu_rows(const __nv_bfloat16* x, __nv_bfloat16* y, long long n, cudaStream_t stream);
int add3_rows(const __nv_bfloat16* x, const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* y, long long n,
              cudaStream_t stream);
int pool_concat(const __nv_bfloat16* global_feats, const __nv_bfloat16* stitched, int H, int W, int grid, int dim,
                __nv_bfloat16* out, cudaStream_t stream);
int embed_tokens(const int* ids, long long id_stride, int n, const __nv_bfloat16* wte, int dim,
                 int vocab, __nv_bfloat16* out, long long ldo, cudaStream_t stream);
int rope_kv_write(const __nv_bfloat16* qkv, int n_tokens, int n_heads, const int* q_offsets,
                  const int* start_pos, int n_seqs, const float* freqs, __nv_bfloat16* q_out,
                  __nv_bfloat16* kv_pool, int n_pages, const int* block_tables, int max_blocks,
                  int layer, cudaStream_t stream);
int argmax_logits(const float* ws, int splits, int B, int V, const __nv_bfloat16* bias, int bias_period,
                  int mask_id, int mask_id2, int* out_ids, long long out_stride, const int* out_index,
                  float* out_margin, __nv_bfloat16* out_logits, float* scratch, cudaStream_t stream);
long long argmax_scratch_floats(int B);
int decode_advance(int* cur_tok, int* pos, int* step, const int* preds, const int* forced,
                   long long stride, int batch, int eos_id, int* finished, cudaStream_t stream);
int gather_rows(const __nv_bfloat16* src, long long ld_src, const int* idx, int n, int dim,
                __nv_bfloat16* out, long long ldo, cudaStream_t stream);
int bins_to_values(int which, const int* bins, int n, int n_bins, float* out, cudaStream_t stream);
int decode_residual_ln_epilogue(const float* ws, int splits, int proj_splits, int B, int D,
                                const __nv_bfloat16* bias_proj, const __nv_bfloat16* bias_fc2,
                                __nv_bfloat16* x, const __nv_bfloat16* ln_w, const __nv_bfloat16* ln_b,
                                __nv_bfloat16* ln_out, cudaStream_t stream);
int fourier_features(const float* x, int B, int n_in, const __nv_bfloat16* w, int half,
                     __nv_bfloat16* out, long long ldo, cudaStream_t stream);

// ---- attention_tc.cu ----
int prefill_attention_tc(const __nv_bfloat16* q, int n_heads, int n_kv_heads, int total_tokens, const int* q_offsets,
                         const int* start_pos, int n_seqs, int max_q, int prefix_len,
                         const __nv_bfloat16* kv_pool, int n_pages, int n_layers, const int* block_tables,
                         int max_blocks, int layer, __nv_bfloat16* out, cudaStream_t stream);
int vit_attention_tc(const __nv_bfloat16* qkv, int n_crops, int seq, int n_heads, __nv_bfloat16* out,
                     cudaStream_t stream);
// 1: the mma.sync kernels of attention.cu; otherwise the wgmma kernels.  Decode attention: 2 = the kernel that loads
// K/V into registers instead of the bulk-copy ring (same bits).
extern int g_attention_impl;

// ---- attention.cu ----
int vit_attention(const __nv_bfloat16* qkv, int n_crops, int seq, int n_heads, __nv_bfloat16* out,
                  cudaStream_t stream);
int prefill_attention(const __nv_bfloat16* q, int n_heads, const int* q_offsets, const int* start_pos,
                      int n_seqs, int max_q, int prefix_len, const __nv_bfloat16* kv_pool, int n_pages,
                      const int* block_tables, int max_blocks, int layer, __nv_bfloat16* out,
                      cudaStream_t stream);
int decode_attention(const __nv_bfloat16* q, int n_heads, int n_kv_heads, const int* pos, int n_seqs,
                     const __nv_bfloat16* kv_pool, int n_pages, const int* block_tables,
                     int max_blocks, int layer, __nv_bfloat16* out, long long ld_out, cudaStream_t stream);
int decode_attention_fused(const float* ws, int splits, int D, int FF, const __nv_bfloat16* bias, const float* freqs,
                           __nv_bfloat16* hid, long long ld_hid, int n_heads, const int* pos, int n_seqs,
                           __nv_bfloat16* kv_pool, int n_pages, const int* block_tables, int max_blocks, int layer,
                           __nv_bfloat16* out, long long ld_out, cudaStream_t stream);
int decode_qkv_finish(const float* ws, int splits, int B, int D, int n_kv_heads, int FF, const __nv_bfloat16* bias,
                      const float* freqs, const int* pos, __nv_bfloat16* q_out, __nv_bfloat16* kv_pool, int n_pages,
                      const int* block_tables, int max_blocks, int layer, __nv_bfloat16* hid, long long ld_hid,
                      cudaStream_t stream);

// ---- preprocess.cu ----
int resample_u8(const uint8_t* src, int in_h, int in_w, int axis, const int* bounds, const int* coeffs, int ksize,
                int out_size, uint8_t* dst, cudaStream_t stream);
int extract_windows_u8(const uint8_t* canvas, int h, int w, int rows, int cols, int stride, int crop, uint8_t* crops,
                       cudaStream_t stream);

// ---- sampling.cu ----
int sample_top_p(const __nv_bfloat16* logits, int B, int V, float temperature, float top_p,
                 const unsigned long long* seed, const int* step, const float* uniforms, __nv_bfloat16* scratch,
                 int keep_probs, int* out_ids, long long out_stride, int out_offset, cudaStream_t stream);
int embed_select(const int* ids, long long id_stride, int n, const __nv_bfloat16* wte, int dim, int vocab, int sel_id,
                 const __nv_bfloat16* alt, long long ld_alt, __nv_bfloat16* out, long long ldo, cudaStream_t stream);
int store_column_f32(const float* src, int n, float* dst, long long stride, const int* index, int offset,
                     cudaStream_t stream);

}  // namespace md
