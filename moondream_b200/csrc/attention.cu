// Attention kernels.
//
//  * flash_attention_kernel<HD, DP, PAGED>: tiled online-softmax attention, 64 queries x 64 keys per
//    step, bf16 mma.sync m16n8k16 with fp32 accumulation, cp.async double-buffered K/V tiles.
//      - PAGED=false: ViT self-attention (reference layers.py:155-166: softmax(QK^T/sqrt(72))V, no
//        mask, 729 tokens, head_dim 72 padded to 80 in shared memory only), reading Q/K/V straight
//        out of the fused qkv GEMM output [B*729, 3*D] and writing token-major [B*729, D].
//      - PAGED=true: decoder prefill (reference text.py:46-50 under the mask of moondream.py:138-146):
//        prefix-LM mask computed from indices (positions < prefix attend bidirectionally inside the
//        prefix, causal afterwards); K/V come from the paged KV pool and only the pos+T keys that
//        exist are visited (the reference scans all 2048 cache slots under a bool mask).
//  * decode_attention_ring_kernel: one query per (sequence, head), that head's K/V pages streamed by bulk copy
//    through a shared-memory ring; HBM-bound (reference text.py:46-50 with the [1,1,2048] mask of
//    moondream.py:472-474,514).  decode_attention_kernel, the same computation with loads into registers, stays for
//    A/B timing and as the tests' independent comparison.
//
// KV pool layout (bf16): [layer][page][2 (k,v)][head][64 tokens][64 dims]; block_tables[seq][i] is
// the page holding positions 64*i .. 64*i+63 of that sequence.
#include <math.h>

#include "kernels.cuh"
#include "ptx.cuh"

namespace md {

constexpr int kPageTokens = 64;

struct FlashParams {
  // dense (ViT) addressing
  const __nv_bfloat16* q;
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  long long q_stride, kv_stride;   // row strides in elements
  int seq_len;                     // dense: rows per batch item
  // paged (text) addressing
  const int* q_offsets;            // [n_seqs + 1] row offsets into q/out
  const int* start_pos;            // [n_seqs]
  const __nv_bfloat16* kv_pool;
  const int* block_tables;
  int max_blocks, layer, n_pages, prefix_len;
  // common
  __nv_bfloat16* out;
  long long out_stride;
  int n_heads;
  float scale_log2;                // softmax scale * log2(e)
};

template <int HD, int DP, bool PAGED>
__global__ void __launch_bounds__(128)
flash_attention_kernel(const FlashParams p) {
  constexpr int BM = 64, BN = 64;
  constexpr int LDS = DP + 8;                 // padded row pitch (elements): conflict-free ldmatrix
  constexpr int CH = HD / 8;                  // 16-byte chunks per global row
  constexpr int KSTEPS = DP / 16;             // k16 steps of QK^T
  constexpr int DT = (HD + 7) / 8;            // n8 tiles of the output (head dim)
  extern __shared__ __align__(16) uint8_t fa_smem[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(fa_smem);
  __nv_bfloat16* sK = sQ + BM * LDS;          // [2][BN][LDS]
  __nv_bfloat16* sV = sK + 2 * BN * LDS;      // [2][BN][LDS]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int head = blockIdx.y;
  const int item = blockIdx.z;
  const int q0 = blockIdx.x * BM;

  int n_q, kv_len, q_pos0;
  long long q_row0;
  const int* btab = nullptr;
  if (PAGED) {
    const int off = p.q_offsets[item];
    n_q = p.q_offsets[item + 1] - off;
    q_pos0 = p.start_pos[item];
    kv_len = q_pos0 + n_q;
    q_row0 = off;
    btab = p.block_tables + static_cast<long long>(item) * p.max_blocks;
  } else {
    n_q = p.seq_len;
    q_pos0 = 0;
    kv_len = p.seq_len;
    q_row0 = static_cast<long long>(item) * p.seq_len;
  }
  if (q0 >= n_q) return;

  // zero the padding columns [HD, DP) of Q and K tiles once (cp.async never touches them)
  if constexpr (DP > HD) {
    for (int i = tid; i < (BM + 2 * BN) * (DP - HD); i += 128) {
      const int r = i / (DP - HD), c = HD + i % (DP - HD);
      sQ[r * LDS + c] = __float2bfloat16(0.f);   // sQ and sK are contiguous: rows 0..BM+2BN-1
    }
  }

  // ---- async tile loaders ----
  auto load_q = [&]() {
    for (int i = tid; i < BM * CH; i += 128) {
      const int r = i / CH, c = i % CH;
      const bool ok = q0 + r < n_q;
      const __nv_bfloat16* src =
          p.q + (q_row0 + (ok ? q0 + r : 0)) * p.q_stride + head * HD + c * 8;
      cp_async_16(sQ + r * LDS + c * 8, src, ok);
    }
  };
  auto load_kv = [&](int tile, int buf) {
    const int k0 = tile * BN;
    const __nv_bfloat16 *kbase, *vbase;
    long long stride;
    if (PAGED) {
      const int page = btab[tile];
      const long long pbase =
          ((static_cast<long long>(p.layer) * p.n_pages + page) * 2) * p.n_heads * (kPageTokens * 64);
      kbase = p.kv_pool + pbase + static_cast<long long>(head) * (kPageTokens * 64);
      vbase = kbase + static_cast<long long>(p.n_heads) * (kPageTokens * 64);
      stride = 64;
    } else {
      kbase = p.k + (q_row0 + k0) * p.kv_stride + head * HD;
      vbase = p.v + (q_row0 + k0) * p.kv_stride + head * HD;
      stride = p.kv_stride;
    }
    __nv_bfloat16* dk = sK + buf * BN * LDS;
    __nv_bfloat16* dv = sV + buf * BN * LDS;
    for (int i = tid; i < BN * CH; i += 128) {
      const int r = i / CH, c = i % CH;
      const bool ok = k0 + r < kv_len;
      const long long ro = ok ? r * stride : 0;
      cp_async_16(dk + r * LDS + c * 8, kbase + ro + c * 8, ok);
      cp_async_16(dv + r * LDS + c * 8, vbase + ro + c * 8, ok);
    }
  };

  // how many key tiles this query tile can see
  int n_tiles;
  {
    const int q_hi = q_pos0 + min(q0 + BM, n_q) - 1;     // last query position of the tile
    int reach = q_hi + 1;
    if (PAGED) {
      if (q_pos0 + q0 < p.prefix_len) reach = max(reach, p.prefix_len);
      reach = min(reach, kv_len);
    } else {
      reach = kv_len;
    }
    n_tiles = (reach + BN - 1) / BN;
  }

  load_q();
  load_kv(0, 0);
  cp_async_commit();

  float o_acc[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
  float row_max[2] = {-INFINITY, -INFINITY};
  float row_sum[2] = {0.f, 0.f};
  uint32_t qf[KSTEPS][4];

  const int r_lo = warp * 16 + (lane >> 2);            // this thread's two query rows in the tile
  const int qpos_lo = q_pos0 + q0 + r_lo, qpos_hi = qpos_lo + 8;

  for (int tile = 0; tile < n_tiles; ++tile) {
    const int buf = tile & 1;
    if (tile + 1 < n_tiles) load_kv(tile + 1, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();

    if (tile == 0) {
#pragma unroll
      for (int ks = 0; ks < KSTEPS; ++ks)
        ldmatrix_x4(qf[ks], smem_u32(sQ + (warp * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8));
    }

    // ---- S = Q K^T ----
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    const __nv_bfloat16* bK = sK + buf * BN * LDS;
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {             // pairs of n8 tiles
        uint32_t kb[4];
        ldmatrix_x4(kb, smem_u32(bK + (np * 16 + (lane & 7) + (lane >> 4) * 8) * LDS + ks * 16 +
                                 ((lane >> 3) & 1) * 8));
        const uint32_t b0[2] = {kb[0], kb[1]};
        const uint32_t b1[2] = {kb[2], kb[3]};
        mma_bf16_16816(s[2 * np], qf[ks], b0);
        mma_bf16_16816(s[2 * np + 1], qf[ks], b1);
      }
    }

    // ---- mask + online softmax ----
    const int kcol0 = tile * BN + (lane & 3) * 2;
    const bool need_mask = PAGED ? true : (tile * BN + BN > kv_len);
    if (need_mask) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int kpos = kcol0 + nt * 8 + (e & 1);
          const int qpos = (e < 2) ? qpos_lo : qpos_hi;
          bool ok = kpos < kv_len;
          if (PAGED) ok = ok && (kpos <= qpos || (kpos < p.prefix_len && qpos < p.prefix_len));
          if (!ok) s[nt][e] = -INFINITY;
        }
      }
    }
    float mx[2] = {row_max[0], row_max[1]};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float corr[2], base[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // a fully masked row so far keeps max = -inf: use 0 as the exponent base to avoid inf - inf
      base[h] = (mx[h] == -INFINITY) ? 0.f : mx[h] * p.scale_log2;
      corr[h] = (row_max[h] == -INFINITY) ? 0.f : exp2f(row_max[h] * p.scale_log2 - base[h]);
      row_max[h] = mx[h];
      row_sum[h] *= corr[h];
    }
#pragma unroll
    for (int i = 0; i < DT; ++i) {
      o_acc[i][0] *= corr[0]; o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1]; o_acc[i][3] *= corr[1];
    }
    uint32_t pf[4][4];                              // P as A fragments for 4 k16 steps
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = exp2f(s[nt][0] * p.scale_log2 - base[0]);
      const float p1 = exp2f(s[nt][1] * p.scale_log2 - base[0]);
      const float p2 = exp2f(s[nt][2] * p.scale_log2 - base[1]);
      const float p3 = exp2f(s[nt][3] * p.scale_log2 - base[1]);
      row_sum[0] += p0 + p1;
      row_sum[1] += p2 + p3;
      pf[nt >> 1][(nt & 1) * 2 + 0] = pack_bf16x2(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_bf16x2(p2, p3);
    }

    // ---- O += P V ----
    const __nv_bfloat16* bV = sV + buf * BN * LDS;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {                // 16 keys per step
#pragma unroll
      for (int dp = 0; dp < DT / 2; ++dp) {         // pairs of n8 tiles over the head dim
        uint32_t vb[4];
        ldmatrix_x4_trans(vb, smem_u32(bV + (ks * 16 + (lane & 15)) * LDS + dp * 16 + (lane >> 4) * 8));
        const uint32_t b0[2] = {vb[0], vb[1]};
        const uint32_t b1[2] = {vb[2], vb[3]};
        mma_bf16_16816(o_acc[2 * dp], pf[ks], b0);
        mma_bf16_16816(o_acc[2 * dp + 1], pf[ks], b1);
      }
      if (DT & 1) {                                  // odd tile count (head_dim 72 -> 9 tiles)
        uint32_t vb[2];
        ldmatrix_x2_trans(vb, smem_u32(bV + (ks * 16 + (lane & 15)) * LDS + (DT - 1) * 8));
        mma_bf16_16816(o_acc[DT - 1], pf[ks], vb);
      }
    }
    __syncthreads();                                 // everyone done with `buf` before it is refilled
  }
  cp_async_wait<0>();

  // ---- normalise and store ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    row_sum[h] += __shfl_xor_sync(0xffffffffu, row_sum[h], 1);
    row_sum[h] += __shfl_xor_sync(0xffffffffu, row_sum[h], 2);
  }
  const float inv0 = row_sum[0] > 0.f ? 1.f / row_sum[0] : 0.f;
  const float inv1 = row_sum[1] > 0.f ? 1.f / row_sum[1] : 0.f;
  const int col = (lane & 3) * 2;
  if (q0 + r_lo < n_q) {
    __nv_bfloat16* o = p.out + (q_row0 + q0 + r_lo) * p.out_stride + head * HD + col;
#pragma unroll
    for (int i = 0; i < DT; ++i)
      *reinterpret_cast<uint32_t*>(o + i * 8) = pack_bf16x2(o_acc[i][0] * inv0, o_acc[i][1] * inv0);
  }
  if (q0 + r_lo + 8 < n_q) {
    __nv_bfloat16* o = p.out + (q_row0 + q0 + r_lo + 8) * p.out_stride + head * HD + col;
#pragma unroll
    for (int i = 0; i < DT; ++i)
      *reinterpret_cast<uint32_t*>(o + i * 8) = pack_bf16x2(o_acc[i][2] * inv1, o_acc[i][3] * inv1);
  }
}

template <int HD, int DP, bool PAGED>
static int launch_flash(const FlashParams& p, dim3 grid, cudaStream_t stream) {
  constexpr int smem = (64 + 4 * 64) * (DP + 8) * 2;
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(flash_attention_kernel<HD, DP, PAGED>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  }
  flash_attention_kernel<HD, DP, PAGED><<<grid, 128, smem, stream>>>(p);
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

int vit_attention(const __nv_bfloat16* qkv, int n_crops, int seq, int n_heads, __nv_bfloat16* out,
                  cudaStream_t stream) {
  if (n_crops <= 0) return set_error("vit_attention: empty batch");
  const int D = n_heads * 72;
  FlashParams p{};
  p.q = qkv; p.k = qkv + D; p.v = qkv + 2 * D;
  p.q_stride = 3LL * D; p.kv_stride = 3LL * D;
  p.seq_len = seq;
  p.out = out; p.out_stride = D;
  p.n_heads = n_heads;
  p.scale_log2 = (1.0f / sqrtf(72.0f)) * 1.4426950408889634f;
  dim3 grid((seq + 63) / 64, n_heads, n_crops);
  return launch_flash<72, 80, false>(p, grid, stream);
}

int prefill_attention(const __nv_bfloat16* q, int n_heads, const int* q_offsets, const int* start_pos,
                      int n_seqs, int max_q, int prefix_len, const __nv_bfloat16* kv_pool, int n_pages,
                      const int* block_tables, int max_blocks, int layer, __nv_bfloat16* out,
                      cudaStream_t stream) {
  if (n_seqs <= 0 || max_q <= 0) return set_error("prefill_attention: empty batch");
  FlashParams p{};
  p.q = q; p.q_stride = static_cast<long long>(n_heads) * 64;
  p.q_offsets = q_offsets; p.start_pos = start_pos;
  p.kv_pool = kv_pool; p.block_tables = block_tables; p.max_blocks = max_blocks;
  p.layer = layer; p.n_pages = n_pages; p.prefix_len = prefix_len;
  p.out = out; p.out_stride = static_cast<long long>(n_heads) * 64;
  p.n_heads = n_heads;
  p.scale_log2 = 0.125f * 1.4426950408889634f;
  dim3 grid((max_q + 63) / 64, n_heads, n_seqs);
  return launch_flash<64, 64, true>(p, grid, stream);
}

// ------------------------------------------------------------------------------------------------
// decode attention: one (sequence, head) per CTA, 4 warps split the keys, 8 lanes per key row.
// FUSED = true additionally finishes the [qkv ; fc1] weight stream of the block for this (sequence, head)
// before attending: sums the fp32 split-K partials of its 3 x 64 q/k/v features (+ bias, bf16 round, partial
// RoPE, K/V row -> KV page; reference text.py:30-43, moondream.py:74-78) and of a 1/H slice of the fc1
// features (+ bias, round, GELU -> hid; layers.py:130,137).  That replaces a separate epilogue kernel.
// ------------------------------------------------------------------------------------------------
struct DecodeFuse {
  const float* ws;                 // [splits][B][3D + FF]
  int splits, B, D, FF;
  const __nv_bfloat16* bias;       // [3D + FF]
  const float* freqs;              // rope table
  __nv_bfloat16* hid;              // gelu(fc1) output rows, pitch ld_hid
  long long ld_hid;
};

// 7 CTAs per SM (<= 72 registers): batch 32 x 32 heads = 1024 CTAs, of which 132 SMs hold 924 at once; the rest run
// as a short second wave
template <bool FUSED>
__global__ void __launch_bounds__(128, 7)
decode_attention_kernel(const __nv_bfloat16* __restrict__ q, int n_heads, int n_kv_heads, const int* __restrict__ pos,
                        __nv_bfloat16* __restrict__ kv_pool, int n_pages,
                        const int* __restrict__ block_tables, int max_blocks, int layer,
                        __nv_bfloat16* __restrict__ out, long long ld_out, float scale_log2, const DecodeFuse fz) {
  // all CTAs of this grid are resident at once, so the trigger fires immediately: the next kernel (the
  // [proj|fc2] weight stream) may start prefetching weights while this one is streaming K/V
  const bool tl = tl_on() && threadIdx.x == 0;
  __shared__ unsigned long long tl_s[4];               // debug timeline stamps (thread 0 only; smem keeps them out of registers)
  if (tl) tl_s[0] = tl_now();
  pdl_launch_dependents();
  pdl_wait();
  if (tl) tl_s[1] = tl_now();
  const int head = blockIdx.x, seq = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane & 7;            // which 16-byte chunk (8 dims) of the 64-dim row
  const int rowi = lane >> 3;          // 4 key rows per warp step
  const int cur = pos[seq];
  const int kv_len = cur + 1;          // the current token's K/V row is part of the context
  const int* btab = block_tables + static_cast<long long>(seq) * max_blocks;
  // grouped-query attention (text.py:49 enable_gqa): query head h reads KV head h / (H / KVH).  The G query heads
  // of a group are neighbouring CTAs, so the group's K/V rows come from HBM once and from L2 for the others.
  // (The fused prologue writes the new K/V row of its own head and therefore needs KVH == H; engine.cu routes
  // grouped models through decode_qkv_finish + the plain kernel.)
  const int kv_head = FUSED ? head : head / (n_heads / n_kv_heads);
  const long long head_off = static_cast<long long>(kv_head) * (kPageTokens * 64);
  const long long v_off = static_cast<long long>(n_kv_heads) * (kPageTokens * 64);

  __shared__ float sq[64];
  float qv[8];
  // The prologue is a chain of dependent L2 round trips during which HBM would sit idle (~5 us measured,
  // tools/decode_timeline.py), so (a) every independent load is issued before the first use of any of them
  // and (b) the first 128 keys' K and V rows (one 128-byte line per thread and plane) are requested into L2
  // up front: the main loop then starts on L2 hits with the stream already running.
  auto prefetch_head = [&]() {
    if (tid < kv_len) {
      const int page = btab[tid >> 6];
      const __nv_bfloat16* kp = kv_pool +
          ((static_cast<long long>(layer) * n_pages + page) * 2) * n_kv_heads * (kPageTokens * 64) + head_off + (tid & 63) * 64;
      prefetch_l2(kp);
      prefetch_l2(kp + v_off);
    }
  };
  if (FUSED) {
    const int NF = 3 * fz.D + fz.FF;
    const long long sstride = static_cast<long long>(fz.B) * NF;
    const float* ws0 = fz.ws + static_cast<long long>(seq) * NF;            // split 0 of this sequence
    const int per = fz.FF / n_heads;
    // features this thread finishes: (fa, fb) of q / k / v (warps 0..2) and (fh, fh + 1) of the fc1 slice
    const bool rot = warp < 2 && lane < 16;                  // dims 0..31 of q and k rotate as pairs (j, j + 16)
    const int f0 = warp * fz.D + head * 64;
    const int fa = rot ? f0 + lane : f0 + 2 * lane;
    const int fb = rot ? f0 + 16 + lane : f0 + 2 * lane + 1;
    const int fh = 3 * fz.D + head * per + tid * 2;
    const bool has_h = tid * 2 < per;
    float ra = 0.f, rb = 0.f, ba = 0.f, bb = 0.f;
    float2 rh = make_float2(0.f, 0.f);
    uint32_t bh = 0;
    if (warp < 3) {
      ra = ws0[fa]; rb = ws0[fb];
      ba = __bfloat162float(fz.bias[fa]); bb = __bfloat162float(fz.bias[fb]);
    }
    if (has_h) {
      rh = *reinterpret_cast<const float2*>(ws0 + fh);
      bh = *reinterpret_cast<const uint32_t*>(fz.bias + fh);
    }
    prefetch_head();                                         // first use of the position / block table
    float cs = 0.f, sn = 0.f;
    int new_page = 0;
    if (rot) { cs = fz.freqs[(cur * 16 + lane) * 2]; sn = fz.freqs[(cur * 16 + lane) * 2 + 1]; }
    if (warp == 1 || warp == 2) new_page = btab[cur >> 6];
    // same summation order as before: split 0, 1, 2, ... then the bias, rounded to bf16 like the Linear output
    auto finish = [&](float a, int f, float b) {
#pragma unroll 1
      for (int s2 = 1; s2 < fz.splits; ++s2) a += ws0[s2 * sstride + f];
      return bf16_round(a + b);
    };
    if (has_h) {
      const float g0 = gelu_tanh(finish(rh.x, fh, bf16_lo(bh))), g1 = gelu_tanh(finish(rh.y, fh + 1, bf16_hi(bh)));
      *reinterpret_cast<uint32_t*>(fz.hid + seq * fz.ld_hid + head * per + tid * 2) = pack_bf16x2(g0, g1);
    }
    for (int i2 = tid * 2 + 256; i2 < per; i2 += 256) {      // slices wider than 256 features
      const int f = 3 * fz.D + head * per + i2;
      const float g0 = gelu_tanh(finish(ws0[f], f, __bfloat162float(fz.bias[f])));
      const float g1 = gelu_tanh(finish(ws0[f + 1], f + 1, __bfloat162float(fz.bias[f + 1])));
      *reinterpret_cast<uint32_t*>(fz.hid + seq * fz.ld_hid + head * per + i2) = pack_bf16x2(g0, g1);
    }
    if (warp < 3) {                                          // warp 0: q, 1: k, 2: v of this head
      const float va = finish(ra, fa, ba), vb = finish(rb, fb, bb);
      float o0 = va, o1 = vb;
      if (rot) {
        o0 = __fsub_rn(__fmul_rn(va, cs), __fmul_rn(vb, sn));
        o1 = __fadd_rn(__fmul_rn(va, sn), __fmul_rn(vb, cs));
      }
      if (warp == 0) {
        sq[2 * lane] = bf16_round(o0);
        sq[2 * lane + 1] = bf16_round(o1);
      } else {
        __nv_bfloat16* dst = kv_pool + ((static_cast<long long>(layer) * n_pages + new_page) * 2 + (warp - 1)) * v_off +
                             head_off + (cur & 63) * 64 + 2 * lane;
        *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(o0, o1);
      }
    }
    __syncthreads();                                       // q in smem, new K/V row visible to the block
#pragma unroll
    for (int j = 0; j < 8; ++j) qv[j] = sq[sub * 8 + j];
  } else {
    prefetch_head();
    const uint4 qq = *reinterpret_cast<const uint4*>(q + (static_cast<long long>(seq) * n_heads + head) * 64 + sub * 8);
    const uint32_t w[4] = {qq.x, qq.y, qq.z, qq.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { qv[2 * j] = bf16_lo(w[j]); qv[2 * j + 1] = bf16_hi(w[j]); }
  }
  if (tl) tl_s[2] = tl_now();
  float m = -INFINITY, l = 0.f;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;

  // each warp takes 16 consecutive keys (4 steps of 4 rows) per iteration, warps interleave
  for (int k0 = warp * 16; k0 < kv_len; k0 += 64) {
    const int page = btab[k0 >> 6];
    const __nv_bfloat16* kp = kv_pool +
        ((static_cast<long long>(layer) * n_pages + page) * 2) * n_kv_heads * (kPageTokens * 64) + head_off;
    uint4 kq[4], vq[4];
#pragma unroll
    for (int st = 0; st < 4; ++st) {
      const int kpos = k0 + st * 4 + rowi;
      const bool ok = kpos < kv_len;
      const long long ro = static_cast<long long>(kpos & 63) * 64 + sub * 8;
      kq[st] = ok ? *reinterpret_cast<const uint4*>(kp + ro) : make_uint4(0, 0, 0, 0);
      vq[st] = ok ? *reinterpret_cast<const uint4*>(kp + v_off + ro) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int st = 0; st < 4; ++st) {
      const int kpos = k0 + st * 4 + rowi;
      const uint32_t w[4] = {kq[st].x, kq[st].y, kq[st].z, kq[st].w};
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) d += qv[2 * j] * bf16_lo(w[j]) + qv[2 * j + 1] * bf16_hi(w[j]);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      if (kpos < kv_len) {               // uniform within the 8-lane group
        const float sc = d * scale_log2;
        const float mn = fmaxf(m, sc);
        const float c = exp2f(m - mn);   // m = -inf on the first key: exp2(-inf) = 0
        const float pw = exp2f(sc - mn);
        l = l * c + pw;
        const uint32_t u[4] = {vq[st].x, vq[st].y, vq[st].z, vq[st].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[2 * j] = acc[2 * j] * c + pw * bf16_lo(u[j]);
          acc[2 * j + 1] = acc[2 * j + 1] * c + pw * bf16_hi(u[j]);
        }
        m = mn;
      }
    }
  }

  if (tl) tl_s[3] = tl_now();
  // merge the 16 partial states (4 row groups x 4 warps) that share each dim chunk
  __shared__ float sm_m[16][8], sm_l[16][8], sm_acc[16][8][8];
  const int slot = warp * 4 + rowi;
  sm_m[slot][sub] = m;
  sm_l[slot][sub] = l;
#pragma unroll
  for (int j = 0; j < 8; ++j) sm_acc[slot][sub][j] = acc[j];
  __syncthreads();
  if (tid < 64) {
    const int c = tid >> 3, j = tid & 7;   // output dim = c * 8 + j
    float M = -INFINITY;
#pragma unroll
    for (int s2 = 0; s2 < 16; ++s2) M = fmaxf(M, sm_m[s2][c]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int s2 = 0; s2 < 16; ++s2) {
      const float w = (sm_m[s2][c] == -INFINITY) ? 0.f : exp2f(sm_m[s2][c] - M);
      L += sm_l[s2][c] * w;
      A += sm_acc[s2][c][j] * w;
    }
    out[static_cast<long long>(seq) * ld_out + head * 64 + c * 8 + j] = __float2bfloat16_rn(A / L);
  }
  if (tl) tl_emit((2u << 28) | (FUSED ? 1u : 0u), tl_s[0], tl_s[1], tl_s[2], tl_s[3], tl_now());
}

// ------------------------------------------------------------------------------------------------
// decode attention with a bulk-copy ring: the same work split, lane mapping and arithmetic as decode_attention_kernel
// (one CTA per (sequence, head); in every page warp w takes rows 16w .. 16w + 15, 4 rows per step, 8 lanes per
// 128-byte row), so the two give the same bits.  What differs is how the K/V rows arrive: one thread streams them by
// 1-D bulk copy into a 3-stage mbarrier ring instead of every lane loading into registers, so the bytes in flight no
// longer depend on the compiler keeping the loads ahead of the math.  A stage is half a page in the order the warps
// consume it: for each warp its rows 16w + 8h .. 16w + 8h + 7 of K and of V (h = 0, 1), 8 copies of 1 KB (the pool
// keeps a (layer, page, plane, head) block contiguous).  Rows past the context arrive with the page and are left out
// by a branch on the position, never multiplied by p = 0.
//
// 24 KB of ring and <= 64 registers give 8 CTAs per SM: the bench's 32 x 32 (sequence, head) pairs fit the 132 SMs in
// one wave (the register-loading kernel fits 7 per SM, 924 at once, and streams its last 100 CTAs as a thin second
// wave).  The following [proj | fc2] weight-stream CTA sizes its own ring to ~226 KB of shared memory and so starts on
// SMs the attention has left, as before.
//
// FUSED: the new K / V row is written to the pool and also kept in shared memory, where the consumer takes it from
// for key `pos` (selected by position).  The copies of that page are issued before the prologue computes the row and
// may or may not see the generic-proxy global write, so their copy of the row is never used: that avoids a proxy fence
// + block barrier in front of the first copies.
// ------------------------------------------------------------------------------------------------
constexpr int kDecStages = 3;
constexpr int kDecStageElems = 2 * 4 * 8 * 64;                         // [K, V][warp][8 rows][64 dims]
constexpr int kDecSmem = kDecStages * kDecStageElems * 2;              // 24 KB
constexpr int kDecCtasPerSm = 8;

template <bool FUSED>
__global__ void __launch_bounds__(128, kDecCtasPerSm)
decode_attention_ring_kernel(const __nv_bfloat16* __restrict__ q, int n_heads, int n_kv_heads, const int* __restrict__ pos,
                             __nv_bfloat16* __restrict__ kv_pool, int n_pages,
                             const int* __restrict__ block_tables, int max_blocks, int layer,
                             __nv_bfloat16* __restrict__ out, long long ld_out, float scale_log2, const DecodeFuse fz) {
  const bool tl = tl_on() && threadIdx.x == 0;
  __shared__ unsigned long long tl_s[4];
  if (tl) tl_s[0] = tl_now();
  pdl_launch_dependents();
  pdl_wait();
  if (tl) tl_s[1] = tl_now();
  extern __shared__ __align__(128) uint8_t dec_smem[];
  __nv_bfloat16* ring = reinterpret_cast<__nv_bfloat16*>(dec_smem);
  __shared__ uint64_t full_bar[kDecStages];
  __shared__ __align__(16) __nv_bfloat16 s_new[2][64];                  // FUSED: the new K and V rows
  __shared__ float sq[64];

  const int head = blockIdx.x, seq = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane & 7, rowi = lane >> 3;
  const int cur = pos[seq];
  const int kv_len = cur + 1;
  const int n_stages = 2 * ((kv_len + kPageTokens - 1) / kPageTokens);  // two per page
  const int* btab = block_tables + static_cast<long long>(seq) * max_blocks;
  const int kv_head = FUSED ? head : head / (n_heads / n_kv_heads);
  const long long head_off = static_cast<long long>(kv_head) * (kPageTokens * 64);
  const long long v_off = static_cast<long long>(n_kv_heads) * (kPageTokens * 64);
  const long long layer_off = static_cast<long long>(layer) * n_pages;

  auto issue = [&](int k) {                              // half k & 1 of page k >> 1 into slot k % kDecStages
    const int page = btab[k >> 1];
    const __nv_bfloat16* src = kv_pool + (layer_off + page) * 2 * v_off + head_off + (k & 1) * 8 * 64;
    __nv_bfloat16* dst = ring + (k % kDecStages) * kDecStageElems;
    uint64_t* bar = &full_bar[k % kDecStages];
    mbar_arrive_expect_tx(bar, kDecStageElems * 2);
#pragma unroll
    for (int pl = 0; pl < 2; ++pl)
#pragma unroll
      for (int w = 0; w < 4; ++w)
        bulk_load_1d(dst + (pl * 4 + w) * 8 * 64, src + pl * v_off + w * 16 * 64, 8 * 64 * 2, bar);
  };
  if (tid == 0) {
    for (int s = 0; s < kDecStages; ++s) mbar_init(&full_bar[s], 1);
    fence_barrier_init();
    for (int k = 0; k < kDecStages && k < n_stages; ++k) issue(k);
  }

  float qv[8];
  if (FUSED) {
    // the prologue of decode_attention_kernel: same features per thread, same summation order
    const int NF = 3 * fz.D + fz.FF;
    const long long sstride = static_cast<long long>(fz.B) * NF;
    const float* ws0 = fz.ws + static_cast<long long>(seq) * NF;
    const int per = fz.FF / n_heads;
    const bool rot = warp < 2 && lane < 16;
    const int f0 = warp * fz.D + head * 64;
    const int fa = rot ? f0 + lane : f0 + 2 * lane;
    const int fb = rot ? f0 + 16 + lane : f0 + 2 * lane + 1;
    const int fh = 3 * fz.D + head * per + tid * 2;
    const bool has_h = tid * 2 < per;
    float ra = 0.f, rb = 0.f, ba = 0.f, bb = 0.f;
    float2 rh = make_float2(0.f, 0.f);
    uint32_t bh = 0;
    if (warp < 3) {
      ra = ws0[fa]; rb = ws0[fb];
      ba = __bfloat162float(fz.bias[fa]); bb = __bfloat162float(fz.bias[fb]);
    }
    if (has_h) {
      rh = *reinterpret_cast<const float2*>(ws0 + fh);
      bh = *reinterpret_cast<const uint32_t*>(fz.bias + fh);
    }
    float cs = 0.f, sn = 0.f;
    int new_page = 0;
    if (rot) { cs = fz.freqs[(cur * 16 + lane) * 2]; sn = fz.freqs[(cur * 16 + lane) * 2 + 1]; }
    if (warp == 1 || warp == 2) new_page = btab[cur >> 6];
    auto finish = [&](float a, int f, float b) {
#pragma unroll 1
      for (int s2 = 1; s2 < fz.splits; ++s2) a += ws0[s2 * sstride + f];
      return bf16_round(a + b);
    };
    if (has_h) {
      const float g0 = gelu_tanh(finish(rh.x, fh, bf16_lo(bh))), g1 = gelu_tanh(finish(rh.y, fh + 1, bf16_hi(bh)));
      *reinterpret_cast<uint32_t*>(fz.hid + seq * fz.ld_hid + head * per + tid * 2) = pack_bf16x2(g0, g1);
    }
    for (int i2 = tid * 2 + 256; i2 < per; i2 += 256) {
      const int f = 3 * fz.D + head * per + i2;
      const float g0 = gelu_tanh(finish(ws0[f], f, __bfloat162float(fz.bias[f])));
      const float g1 = gelu_tanh(finish(ws0[f + 1], f + 1, __bfloat162float(fz.bias[f + 1])));
      *reinterpret_cast<uint32_t*>(fz.hid + seq * fz.ld_hid + head * per + i2) = pack_bf16x2(g0, g1);
    }
    if (warp < 3) {                                      // warp 0: q, 1: k, 2: v of this head
      const float va = finish(ra, fa, ba), vb = finish(rb, fb, bb);
      float o0 = va, o1 = vb;
      if (rot) {
        o0 = __fsub_rn(__fmul_rn(va, cs), __fmul_rn(vb, sn));
        o1 = __fadd_rn(__fmul_rn(va, sn), __fmul_rn(vb, cs));
      }
      if (warp == 0) {
        sq[2 * lane] = bf16_round(o0);
        sq[2 * lane + 1] = bf16_round(o1);
      } else {
        const uint32_t row = pack_bf16x2(o0, o1);
        __nv_bfloat16* dst = kv_pool + ((layer_off + new_page) * 2 + (warp - 1)) * v_off + head_off + (cur & 63) * 64 + 2 * lane;
        *reinterpret_cast<uint32_t*>(dst) = row;
        *reinterpret_cast<uint32_t*>(&s_new[warp - 1][2 * lane]) = row;
      }
    }
    __syncthreads();                                     // q, the new row and the ring's barriers visible to the block
#pragma unroll
    for (int j = 0; j < 8; ++j) qv[j] = sq[sub * 8 + j];
  } else {
    const uint4 qq = *reinterpret_cast<const uint4*>(q + (static_cast<long long>(seq) * n_heads + head) * 64 + sub * 8);
    const uint32_t w[4] = {qq.x, qq.y, qq.z, qq.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) { qv[2 * j] = bf16_lo(w[j]); qv[2 * j + 1] = bf16_hi(w[j]); }
    __syncthreads();                                     // the ring's barriers initialised
  }
  if (tl) tl_s[2] = tl_now();
  float m = -INFINITY, l = 0.f;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;

  for (int k = 0; k < n_stages; ++k) {
    mbar_wait(&full_bar[k % kDecStages], (k / kDecStages) & 1);
    const uint4* sk = reinterpret_cast<const uint4*>(ring + (k % kDecStages) * kDecStageElems + warp * 8 * 64);
    const uint4* sv = sk + 4 * 8 * 8;                   // the V plane: 4 warps x 8 rows x 8 chunks further
    const int k0 = (k >> 1) * kPageTokens + warp * 16 + (k & 1) * 8;
    uint4 kq[2], vq[2];
#pragma unroll
    for (int st = 0; st < 2; ++st) {
      const int r = st * 4 + rowi;
      const bool fresh = FUSED && k0 + r == cur;
      kq[st] = fresh ? reinterpret_cast<const uint4*>(s_new[0])[sub] : sk[r * 8 + sub];
      vq[st] = fresh ? reinterpret_cast<const uint4*>(s_new[1])[sub] : sv[r * 8 + sub];
    }
#pragma unroll
    for (int st = 0; st < 2; ++st) {
      const int kpos = k0 + st * 4 + rowi;
      const uint32_t w[4] = {kq[st].x, kq[st].y, kq[st].z, kq[st].w};
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) d += qv[2 * j] * bf16_lo(w[j]) + qv[2 * j + 1] * bf16_hi(w[j]);
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      if (kpos < kv_len) {               // uniform within the 8-lane group
        const float sc = d * scale_log2;
        const float mn = fmaxf(m, sc);
        const float c = exp2f(m - mn);
        const float pw = exp2f(sc - mn);
        l = l * c + pw;
        const uint32_t u[4] = {vq[st].x, vq[st].y, vq[st].z, vq[st].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[2 * j] = acc[2 * j] * c + pw * bf16_lo(u[j]);
          acc[2 * j + 1] = acc[2 * j + 1] * c + pw * bf16_hi(u[j]);
        }
        m = mn;
      }
    }
    __syncthreads();                                     // the stage is consumed: refill it
    if (tid == 0 && k + kDecStages < n_stages) issue(k + kDecStages);
  }

  if (tl) tl_s[3] = tl_now();
  // merge the 16 partial states as decode_attention_kernel does; the ring is idle now and holds them
  float* sm_m = reinterpret_cast<float*>(dec_smem);      // [16][8]
  float* sm_l = sm_m + 128;                              // [16][8]
  float* sm_acc = sm_l + 128;                            // [16][8][8]
  const int slot = warp * 4 + rowi;
  sm_m[slot * 8 + sub] = m;
  sm_l[slot * 8 + sub] = l;
#pragma unroll
  for (int j = 0; j < 8; ++j) sm_acc[(slot * 8 + sub) * 8 + j] = acc[j];
  __syncthreads();
  if (tid < 64) {
    const int c = tid >> 3, j = tid & 7;
    float M = -INFINITY;
#pragma unroll
    for (int s2 = 0; s2 < 16; ++s2) M = fmaxf(M, sm_m[s2 * 8 + c]);
    float L = 0.f, A = 0.f;
#pragma unroll
    for (int s2 = 0; s2 < 16; ++s2) {
      const float w = (sm_m[s2 * 8 + c] == -INFINITY) ? 0.f : exp2f(sm_m[s2 * 8 + c] - M);
      L += sm_l[s2 * 8 + c] * w;
      A += sm_acc[(s2 * 8 + c) * 8 + j] * w;
    }
    out[static_cast<long long>(seq) * ld_out + head * 64 + c * 8 + j] = __float2bfloat16_rn(A / L);
  }
  if (tl) tl_emit((2u << 28) | (FUSED ? 1u : 0u), tl_s[0], tl_s[1], tl_s[2], tl_s[3], tl_now());
}

void timeline_install_attention(const Timeline& t) { timeline_install(t); }

template <bool FUSED>
static int launch_decode_attention(const __nv_bfloat16* q, int n_heads, int n_kv_heads, const int* pos, int n_seqs,
                                   __nv_bfloat16* kv_pool, int n_pages, const int* block_tables, int max_blocks,
                                   int layer, __nv_bfloat16* out, long long ld_out, const DecodeFuse& fz,
                                   cudaStream_t stream) {
  const float scale_log2 = 0.125f * 1.4426950408889634f;
  const dim3 grid(n_heads, n_seqs);
  count_launch();
  const cudaError_t e =
      g_attention_impl == 2
          ? launch_k(decode_attention_kernel<FUSED>, grid, dim3(128), 0, stream, q, n_heads, n_kv_heads, pos, kv_pool,
                     n_pages, block_tables, max_blocks, layer, out, ld_out, scale_log2, fz)
          : launch_k(decode_attention_ring_kernel<FUSED>, grid, dim3(128), kDecSmem, stream, q, n_heads, n_kv_heads,
                     pos, kv_pool, n_pages, block_tables, max_blocks, layer, out, ld_out, scale_log2, fz);
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

int decode_attention(const __nv_bfloat16* q, int n_heads, int n_kv_heads, const int* pos, int n_seqs,
                     const __nv_bfloat16* kv_pool, int n_pages, const int* block_tables,
                     int max_blocks, int layer, __nv_bfloat16* out, long long ld_out, cudaStream_t stream) {
  if (n_seqs <= 0) return set_error("decode_attention: empty batch");
  if (n_kv_heads <= 0) n_kv_heads = n_heads;
  if (n_heads % n_kv_heads) return set_error("decode_attention: n_heads must be a multiple of n_kv_heads");
  return launch_decode_attention<false>(q, n_heads, n_kv_heads, pos, n_seqs, const_cast<__nv_bfloat16*>(kv_pool),
                                        n_pages, block_tables, max_blocks, layer, out, ld_out, DecodeFuse{}, stream);
}

// fused form: q/k/v/fc1 are finished from the split-K partials `ws` inside the kernel (see DecodeFuse)
int decode_attention_fused(const float* ws, int splits, int D, int FF, const __nv_bfloat16* bias, const float* freqs,
                           __nv_bfloat16* hid, long long ld_hid, int n_heads, const int* pos, int n_seqs,
                           __nv_bfloat16* kv_pool, int n_pages, const int* block_tables, int max_blocks, int layer,
                           __nv_bfloat16* out, long long ld_out, cudaStream_t stream) {
  if (n_seqs <= 0) return set_error("decode_attention: empty batch");
  if (FF % n_heads || (FF / n_heads) % 2) return set_error("decode_attention_fused: FF must split evenly over the heads");
  DecodeFuse fz{ws, splits, n_seqs, D, FF, bias, freqs, hid, ld_hid};
  return launch_decode_attention<true>(static_cast<const __nv_bfloat16*>(nullptr), n_heads, n_heads, pos, n_seqs,
                                       kv_pool, n_pages, block_tables, max_blocks, layer, out, ld_out, fz, stream);
}

// ------------------------------------------------------------------------------------------------
// Grouped-query models (n_kv_heads < n_heads): finish the [qkv ; fc1] weight stream in a separate small kernel —
// split-K sum in fixed order + bias + bf16 rounding (the Linear outputs, text.py:30 / layers.py:130), partial RoPE on
// q and k (rope.py:20-48), the new K/V row into its page (moondream.py:74-78), GELU on the fc1 slice — then run the
// plain decode attention.  Columns of the stream: q [0, D) | k [D, D + KVW) | v [.., D + 2 KVW) | fc1 [.., + FF).
// One CTA per sequence; a thread owns one rotation pair (j, j + 16) or two neighbouring pass-through features.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
decode_qkv_finish_kernel(const float* __restrict__ ws, int splits, int B, int D, int n_kv_heads, int FF,
                         const __nv_bfloat16* __restrict__ bias, const float* __restrict__ freqs,
                         const int* __restrict__ pos, __nv_bfloat16* __restrict__ q_out,
                         __nv_bfloat16* __restrict__ kv_pool, int n_pages, const int* __restrict__ block_tables,
                         int max_blocks, int layer, __nv_bfloat16* __restrict__ hid, long long ld_hid) {
  pdl_launch_dependents();
  pdl_wait();
  const int seq = blockIdx.x;
  const int kvw = n_kv_heads * 64;
  const int NF = D + 2 * kvw + FF;
  const long long sstride = static_cast<long long>(B) * NF;
  const float* ws0 = ws + static_cast<long long>(seq) * NF;
  const int cur = pos[seq];
  const int page = block_tables[static_cast<long long>(seq) * max_blocks + (cur >> 6)];
  __nv_bfloat16* krow = kv_pool + ((static_cast<long long>(layer) * n_pages + page) * 2) * n_kv_heads * (kPageTokens * 64) +
                        (cur & 63) * 64;
  const long long v_off = static_cast<long long>(n_kv_heads) * (kPageTokens * 64);
  auto lin = [&](int f) {
    float a = ws0[f];
    for (int s2 = 1; s2 < splits; ++s2) a += ws0[s2 * sstride + f];
    return bf16_round(a + __bfloat162float(bias[f]));
  };
  // q and k heads: 32 work items per head = 16 rotation pairs + 16 pass-through pairs
  const int qk_heads = D / 64 + n_kv_heads;
  for (int w = threadIdx.x; w < qk_heads * 32; w += blockDim.x) {
    const int h = w >> 5, i = w & 31;
    const bool is_q = h < D / 64;
    const int base = is_q ? h * 64 : D + (h - D / 64) * 64;
    __nv_bfloat16* dst = is_q ? q_out + static_cast<long long>(seq) * D + h * 64
                              : krow + static_cast<long long>(h - D / 64) * (kPageTokens * 64);
    if (i < 16) {
      const float re = lin(base + i), im = lin(base + 16 + i);
      const float cs = freqs[(cur * 16 + i) * 2], sn = freqs[(cur * 16 + i) * 2 + 1];
      const float o0 = __fsub_rn(__fmul_rn(re, cs), __fmul_rn(im, sn));
      const float o1 = __fadd_rn(__fmul_rn(re, sn), __fmul_rn(im, cs));
      *reinterpret_cast<uint32_t*>(dst + 2 * i) = pack_bf16x2(o0, o1);          // interleaved (re', im')
    } else {
      const int d = 32 + 2 * (i - 16);
      *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16x2(lin(base + d), lin(base + d + 1));
    }
  }
  for (int w = threadIdx.x; w < kvw / 2; w += blockDim.x) {                       // v rows
    const int h = (2 * w) >> 6, d = (2 * w) & 63;
    const int f = D + kvw + 2 * w;
    *reinterpret_cast<uint32_t*>(krow + v_off + static_cast<long long>(h) * (kPageTokens * 64) + d) =
        pack_bf16x2(lin(f), lin(f + 1));
  }
  for (int w = threadIdx.x; w < FF / 2; w += blockDim.x) {                        // gelu(fc1)
    const int f = D + 2 * kvw + 2 * w;
    *reinterpret_cast<uint32_t*>(hid + seq * ld_hid + 2 * w) = pack_bf16x2(gelu_tanh(lin(f)), gelu_tanh(lin(f + 1)));
  }
}

int decode_qkv_finish(const float* ws, int splits, int B, int D, int n_kv_heads, int FF, const __nv_bfloat16* bias,
                      const float* freqs, const int* pos, __nv_bfloat16* q_out, __nv_bfloat16* kv_pool, int n_pages,
                      const int* block_tables, int max_blocks, int layer, __nv_bfloat16* hid, long long ld_hid,
                      cudaStream_t stream) {
  if (B <= 0) return set_error("decode_qkv_finish: empty batch");
  if (D % 64 || FF % 2 || n_kv_heads <= 0) return set_error("decode_qkv_finish: unsupported shape");
  count_launch();
  cudaError_t e = launch_k(decode_qkv_finish_kernel, dim3(B), dim3(256), 0, stream, ws, splits, B, D, n_kv_heads, FF, bias,
                           freqs, pos, q_out, kv_pool, n_pages, block_tables, max_blocks, layer, hid, ld_hid);
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

}  // namespace md
