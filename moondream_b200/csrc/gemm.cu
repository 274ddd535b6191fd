// Persistent, warp-specialised bf16 GEMMs for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T  (fp32 accum).
//
// Replaces every F.linear on the hot path of the reference (moondream/torch/layers.py:34-35,
// vision.py:67, text.py:30,53,166, layers.py:130,139, region.py:43,57,71,93).
//
//   warpgroup 0     : TMA producer  (one thread: cp.async.bulk.tensor, 128B-swizzled K-major tiles, mbarrier ring)
//   warpgroups 1, 2 : consumers     (wgmma m64 x BN x 16 from shared memory, accumulators in registers, then the
//                                    fused epilogue straight from the registers)
//
// Row form: BN = 256 / 192 for the wide layers (per k16 step a warpgroup reads 64 x 16 of A and BN x 16 of B from
// shared memory, so a wider tile needs fewer shared-memory bytes per MMA), with the producer warpgroup's registers
// handed to the consumers (setmaxnreg) for the 128 / 96 accumulators per thread.  The consumers keep one k-block of
// MMAs in flight while they wait for the next stage; each accumulator still sums K in the order its MMAs are issued.
//
// Tails in M, N and K are handled by TMA out-of-bounds zero fill plus masked stores, so the awkward reference
// shapes (K=588->592, N=4304, M=B*729) need no padded copies of activations.
//
// Two kernels:
//   * gemm_bf16_kernel (row form, prefill / ViT sized M): bf16 out[M,N] with a fused epilogue.
//   * smallbatch_gemm_kernel (decode sized batches, <= 128 rows per launch): one CTA per (weight-row tile, K split)
//     streams its slice of the weight matrix once, weights as the 64-row wgmma A operand and the activations as the
//     N = 16..128 B operand; fp32 partial sums ws[split][b][n] are finished by the consumer (splitk_epilogue_kernel,
//     the decode attention prologue, the residual + LayerNorm epilogue, argmax).  The same kernel streams int4 / int8
//     weights (gemm_quant.cu): the packed tile is staged by TMA and dequantised into the A slot by the consumers.
#include <vector>

#include "kernels.cuh"
#include "ptx.cuh"

namespace md {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int kGemmThreads = 384;       // producer warpgroup + two consumer warpgroups of 64 accumulator rows

static int g_gemm_debug = 0;            // md_debug_gemm: timing experiments only
static int g_gemm_sm_cap = 0;           // md_debug_gemm_sm_cap: 0 = every SM (default)

struct GemmParams {
  int M, N, K;
  int m_blocks, n_blocks, k_blocks;    // k_blocks = ceil(K / BK)
  int mode;                            // EPI_BIAS / EPI_BIAS_GELU / EPI_BIAS_RESIDUAL / EPI_QKV_ROPE
  __nv_bfloat16* out;
  long long ldo;
  const __nv_bfloat16* bias;           // [N] or nullptr
  const __nv_bfloat16* res;            // residual [*, N]
  long long ldr;
  int res_mod;                         // residual row = row % res_mod when > 0 (pos_emb broadcast)
  int remap_gin, remap_gout, remap_goff;  // out row = (r / gin) * gout + r % gin + goff when gin > 0
  RopeEpilogue rope;                   // EPI_QKV_ROPE
  int early_trigger;                   // release the dependent grid at once (its prologue overlaps this kernel's tail wave)
};

// wgmma m64nN accumulator layout: warp w of the warpgroup holds rows 16w .. 16w+15; lane l holds rows 16w + l/4 and
// 16w + l/4 + 8 (h = 0, 1) and, in every 8-column block j, columns 8j + 2 (l % 4) and the one after it:
// acc[4j + 2h + e] = D[16w + l/4 + 8h][8j + 2 (l % 4) + e].

// Fused epilogue of the prefill QKV projection: row `row` (h selects it in the fragment), output columns
// col0 .. col0+31 = one half of one head of q, k or v.  dims 0..31 of q and k rotate (pairs (j, j+16) are both in
// this thread), everything else passes through; q goes to q_out, k / v to the KV page of (seq, pos).
struct RopeRow { int pos; long long kv_row; };   // kv_row: element offset of (page, token) for head 0, k plane
__device__ __forceinline__ RopeRow rope_locate(const RopeEpilogue& e, int row) {
  int lo = 0, hi = e.n_seqs;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (e.q_offsets[mid] <= row) lo = mid; else hi = mid;
  }
  RopeRow r;
  r.pos = e.start_pos[lo] + (row - e.q_offsets[lo]);
  const int page = e.block_tables[static_cast<long long>(lo) * e.max_blocks + (r.pos >> 6)];
  r.kv_row = ((static_cast<long long>(e.layer) * e.n_pages + page) * 2) * e.n_kv_heads * (64 * 64) + (r.pos & 63) * 64;
  return r;
}
// x[jj][e] = bf16(acc + bias) of columns col0 + 8 jj + 2 qd + e of this thread's row
__device__ __forceinline__ void rope_store_frag(const GemmParams& p, const float (&x)[4][2], int row, int col0, int qd,
                                                const RopeRow& rr) {
  const RopeEpilogue& e = p.rope;
  // columns: q [0, D) | k [D, D + KVW) | v [D + KVW, D + 2 KVW), KVW = n_kv_heads * 64 (text.py:36-38)
  const int kvw = e.n_kv_heads * 64;
  const int part = col0 < e.D ? 0 : (col0 < e.D + kvw ? 1 : 2);
  const int within = col0 - (part == 0 ? 0 : e.D + (part - 1) * kvw);
  const int head = within >> 6, half = (within >> 5) & 1;
  __nv_bfloat16* dst;
  if (part == 0) dst = e.q_out + static_cast<long long>(row) * e.D + head * 64 + half * 32;
  else dst = e.kv_pool + rr.kv_row + (static_cast<long long>(part - 1) * e.n_kv_heads + head) * (64 * 64) + half * 32;
  if (part < 2 && half == 0) {
    const float* tab = e.freqs + static_cast<long long>(rr.pos) * 32;    // 16 x (cos, sin)
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      uint32_t w[2];
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int j = 8 * jj + 2 * qd + s;            // pairs with j + 16; output (re', im') lands at 2j, 2j+1
        const float c = tab[2 * j], sn = tab[2 * j + 1];
        const float re = __fsub_rn(__fmul_rn(x[jj][s], c), __fmul_rn(x[jj + 2][s], sn));
        const float im = __fadd_rn(__fmul_rn(x[jj][s], sn), __fmul_rn(x[jj + 2][s], c));
        w[s] = pack_bf16x2(re, im);
      }
      *reinterpret_cast<uint2*>(dst + 16 * jj + 4 * qd) = make_uint2(w[0], w[1]);
    }
  } else {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
      *reinterpret_cast<uint32_t*>(dst + 8 * jj + 2 * qd) = pack_bf16x2(x[jj][0], x[jj][1]);
  }
}

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarOffset = STAGES * kStageBytes;
  static constexpr int kTotal = kBarOffset + 2 * STAGES * 8 + 1024;  // +1024 align slack
};

template <int BN, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using S = GemmSmem<BN, STAGES>;
  static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 192 || BN == 256, "BN");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;

  __shared__ unsigned long long tl_s[5];    // debug timeline stamps (see ptx.cuh), untouched unless installed
  const bool tl = tl_on();
  if (tl && threadIdx.x == 0) tl_s[0] = tl_now();
  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmA);
    prefetch_tensormap(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);            // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  // every dependent kernel waits (griddepcontrol.wait) before it touches global memory, so releasing it here only moves
  // its launch latency and prologue under this kernel's last, partially filled wave of tiles
  if (p.early_trigger) pdl_launch_dependents();

  const int total_tiles = p.m_blocks * p.n_blocks;
  const int wg = threadIdx.x >> 7;

  // 384 threads launch with 168 registers each; 40 x 128 + 232 x 256 <= 65536 moves the producer's share to the
  // consumers' accumulators
  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      pdl_wait();
      if (tl) tl_s[1] = tl_now();
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_blk = tile % p.n_blocks;
        const int m_blk = tile / p.n_blocks;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          uint8_t* sa = smem + stage * S::kStageBytes;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
          tma_load_2d(sa + S::kABytes, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ------------------------------ consumers: MMA + epilogue ------------------------------
    setmaxnreg_inc<232>();
    const int c = wg - 1;                      // accumulator rows 64c .. 64c+63 of the tile
    const int t = threadIdx.x & 127;
    const int lane = t & 31, w = t >> 5, qd = lane & 3;
    pdl_wait();                                // global reads (residual) and writes must follow the predecessor
    int stage = 0;
    uint32_t phase = 0;
    bool first = true;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_blk = tile % p.n_blocks;
      const int m_blk = tile / p.n_blocks;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;                           // stage whose MMAs are still in flight
      for (int kb = 0; kb < p.k_blocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (tl && first && t == 0 && c == 0) tl_s[2] = tl_now();      // first operands landed
        first = false;
        const uint32_t sa = smem_u32(smem + stage * S::kStageBytes);
        const uint64_t da = make_desc_k_sw128(sa + c * (64 * 128));
        const uint64_t db = make_desc_k_sw128(sa + S::kABytes);
        wgmma_fence();
        fence_regs(acc);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)      // 16 elements (32 B) along K inside the 128-byte swizzle row: +2
          wgmma_ss<BN>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                       (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                       // k-block kb - 1 is done: its operands may be overwritten
        fence_regs(acc);
        if (t == 0 && prev >= 0) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (t == 0) mbar_arrive(&empty_bar[prev]);
      if (tl && t == 0 && c == 0) tl_s[3] = tl_now();                   // (last) accumulator complete

#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = m_blk * BM + c * 64 + w * 16 + (lane >> 2) + 8 * h;
        if (row >= p.M) continue;
        if (p.mode == EPI_QKV_ROPE) {
          const RopeRow rr = rope_locate(p.rope, row);
#pragma unroll
          for (int cc = 0; cc < BN / 32; ++cc) {
            const int col0 = n_blk * BN + cc * 32;
            if (col0 >= p.N) continue;
            float x[4][2];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const uint32_t bw = *reinterpret_cast<const uint32_t*>(p.bias + col0 + 8 * jj + 2 * qd);
              x[jj][0] = bf16_round(acc[(4 * cc + jj) * 4 + 2 * h] + bf16_lo(bw));
              x[jj][1] = bf16_round(acc[(4 * cc + jj) * 4 + 2 * h + 1] + bf16_hi(bw));
            }
            rope_store_frag(p, x, row, col0, qd, rr);
          }
          continue;
        }
        long long out_row = row;
        if (p.remap_gin > 0)
          out_row = static_cast<long long>(row / p.remap_gin) * p.remap_gout + row % p.remap_gin + p.remap_goff;
        const int res_row = (p.res_mod > 0) ? (row % p.res_mod) : row;
        __nv_bfloat16* orow = p.out + out_row * p.ldo;
        const __nv_bfloat16* rrow = p.mode == EPI_BIAS_RESIDUAL ? p.res + static_cast<long long>(res_row) * p.ldr : nullptr;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n_blk * BN + 8 * j + 2 * qd;
          if (col >= p.N) continue;            // N is a multiple of 8 (checked on the host): col + 1 < N too
          const uint32_t bw = p.bias ? *reinterpret_cast<const uint32_t*>(p.bias + col) : 0u;
          // the reference rounds the Linear output to bf16 before anything else touches it
          float v0 = bf16_round(acc[4 * j + 2 * h] + bf16_lo(bw));
          float v1 = bf16_round(acc[4 * j + 2 * h + 1] + bf16_hi(bw));
          if (p.mode == EPI_BIAS_GELU) {
            v0 = gelu_tanh(v0);
            v1 = gelu_tanh(v1);
          } else if (p.mode == EPI_BIAS_RESIDUAL) {
            const uint32_t rw = *reinterpret_cast<const uint32_t*>(rrow + col);
            v0 += bf16_lo(rw);
            v1 += bf16_hi(rw);
          }
          *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(v0, v1);
        }
      }
    }
  }

  __syncthreads();
  if (tl && threadIdx.x == 0 && blockIdx.x < total_tiles)
    tl_emit((1u << 28) | (static_cast<uint32_t>(p.mode) << 24) | (static_cast<uint32_t>(p.M) & 0xFFFFFFu),
            tl_s[0], tl_s[1], tl_s[2], tl_s[3], tl_now());
}


// ------------------------------------------------------------------------------------------------
// Small-batch weight stream (decode-time Linear layers, batch <= 128 rows of activations).
//
// ws[split][b][n] = sum_{k in split} X[b][k] * W[n][k]  (fp32 partials, finished by the consumer kernel).
//
// The weight tile is the wgmma A operand (64 rows per consumer warpgroup, tile_n = 64 or 128 rows per CTA) and the
// activations the B operand (N = the batch rounded up to 16 / 32 / 64 / 128; TMA zero-fills the rows past the batch),
// so the weights enter the tensor core once per k-block whatever the batch.
//
// One CTA per (weight-row tile, K split), all resident at once where the plan allows.  Under programmatic dependent
// launch the weight tiles of the first ring of stages are requested before the dependency wait (no earlier kernel
// writes weights); only the activation loads, and everything downstream of them, wait for the predecessor.
//
// BITS = 16: bf16 weights, loaded by TMA straight into the swizzled A slot.  BITS = 4 / 8: packed weights
// (gemm_quant.cu) are staged by TMA, and each consumer warpgroup rebuilds its 64 rows of the bf16 tile in the A slot
// exactly as the reference dequantises (layers.py:38-44) before its MMAs: the partial sums equal the bf16 stream's
// on the dequantised matrix bit for bit.
// ------------------------------------------------------------------------------------------------
constexpr int kSbMaxStages = 8;

struct SmallBatchParams {
  int batch, batch_total, n_out, k_blocks;   // this launch covers `batch` (<= 128) rows of a batch_total-row problem
  int tile_n, k_splits;
  int kb_per_split, seg_splits, seg_kb, kb_per_split2;   // split -> k-block range (two segments when seg_kb < k_blocks)
  int stages, w_bytes, x_bytes, q_bytes, stage_bytes;    // stage = [W tile | X tile | packed staging], 1 KB multiple
  int groups, max_groups;                  // packed: scale / zero row pitch (K / 128); groups one split can touch
  int trigger_early;
  float* ws;
  const float* scale;
  const float* zero;
};

template <int NB, int BITS>
__global__ void __launch_bounds__(kGemmThreads, 1)
smallbatch_gemm_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                       const SmallBatchParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  // [stage: W (bf16, swizzled) | X | packed staging] x stages | scale table | zero table | barriers
  float* s_scale = reinterpret_cast<float*>(smem + p.stages * p.stage_bytes);
  float* s_zero = s_scale + p.tile_n * p.max_groups;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(
      (reinterpret_cast<uintptr_t>(s_zero + p.tile_n * p.max_groups) + 7) & ~static_cast<uintptr_t>(7));
  uint64_t* qfull = full_bar + kSbMaxStages;
  uint64_t* empty_bar = qfull + kSbMaxStages;
  __shared__ unsigned long long tl_s[5];    // debug timeline stamps (see ptx.cuh), untouched unless installed
  const bool tl = tl_on();
  if (tl && threadIdx.x == 0) tl_s[0] = tl_now();

  const int wg = threadIdx.x >> 7;
  const int n_wg = p.tile_n / 64;
  if (p.trigger_early) pdl_launch_dependents();
  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmX);
    prefetch_tensormap(&tmW);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&qfull[i], 1);
      mbar_init(&empty_bar[i], n_wg);
    }
    fence_barrier_init();
  }

  const int split = blockIdx.x % p.k_splits;
  const int tile = blockIdx.x / p.k_splits;
  int kb0, kb1;
  if (split < p.seg_splits) {
    kb0 = split * p.kb_per_split;
    kb1 = min(p.seg_kb, kb0 + p.kb_per_split);
  } else {
    kb0 = p.seg_kb + (split - p.seg_splits) * p.kb_per_split2;
    kb1 = min(p.k_blocks, kb0 + p.kb_per_split2);
  }
  const int nk = kb1 - kb0;
  const int n0 = tile * p.tile_n;
  const int g0 = kb0 >> 1;                       // first quantisation group of this split (128 = two k-blocks)
  if (BITS != 16 && wg >= 1) {
    // scale / zero-point table of this (tile, split): constants, so no dependency wait
    for (int i = threadIdx.x - 128; i < p.tile_n * p.max_groups; i += n_wg * 128) {
      const int row = i / p.max_groups, g = i - row * p.max_groups;
      const int n = min(n0 + row, p.n_out - 1), gg = min(g0 + g, p.groups - 1);
      s_scale[i] = p.scale[static_cast<long long>(n) * p.groups + gg];
      s_zero[i] = p.zero[static_cast<long long>(n) * p.groups + gg];
    }
  }
  __syncthreads();

  if (wg == 0) {
    if (threadIdx.x == 0) {
      // bf16: W and X of a stage complete full_bar together; packed: the staging tile completes qfull
      const uint32_t w_tx = BITS == 16 ? static_cast<uint32_t>(p.w_bytes + p.x_bytes) : static_cast<uint32_t>(p.q_bytes);
      uint64_t* wbar = BITS == 16 ? full_bar : qfull;
      const int w_off = BITS == 16 ? 0 : p.w_bytes + p.x_bytes;
      const int w_c0 = BITS == 16 ? BK : BK * BITS / 8;       // tensor-map units per k-block (elements / bytes)
      const int pre = min(p.stages, nk);
      for (int i = 0; i < pre; ++i) {
        mbar_arrive_expect_tx(&wbar[i], w_tx);
        tma_load_2d(smem + i * p.stage_bytes + w_off, &tmW, &wbar[i], (kb0 + i) * w_c0, n0);
      }
      pdl_wait();
      if (tl) tl_s[1] = tl_now();
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < nk; ++j) {
        uint8_t* sx = smem + stage * p.stage_bytes;
        if (j >= pre) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&wbar[stage], w_tx);
          tma_load_2d(sx + w_off, &tmW, &wbar[stage], (kb0 + j) * w_c0, n0);
        }
        if (BITS != 16) mbar_arrive_expect_tx(&full_bar[stage], static_cast<uint32_t>(p.x_bytes));
        tma_load_2d(sx + p.w_bytes, &tmX, &full_bar[stage], (kb0 + j) * BK, 0);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    const int c = wg - 1;                        // weight rows 64c .. 64c+63 of the tile
    const int t = threadIdx.x & 127;
    const int lane = t & 31, w = t >> 5, qd = lane & 3;
    float acc[NB / 2];
#pragma unroll
    for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (int j = 0; j < nk; ++j) {
      uint8_t* sw = smem + stage * p.stage_bytes;
      if (BITS != 16) {
        const int gl = ((kb0 + j) >> 1) - g0;
        const uint8_t* sq = sw + p.w_bytes + p.x_bytes;
        const int cch = t & 7;                   // 8 weights = one 16-byte chunk of the 128-byte row
        mbar_wait(&qfull[stage], phase);
        for (int row = c * 64 + (t >> 3); row < c * 64 + 64; row += 16) {
          const float sc = s_scale[row * p.max_groups + gl], z = s_zero[row * p.max_groups + gl];
          float v[8];
          unpack8<BITS>(sq + row * (BK * BITS / 8) + cch * BITS, v);
          uint4 o;
          o.x = pack_bf16x2(dequant1(v[0], z, sc), dequant1(v[1], z, sc));
          o.y = pack_bf16x2(dequant1(v[2], z, sc), dequant1(v[3], z, sc));
          o.z = pack_bf16x2(dequant1(v[4], z, sc), dequant1(v[5], z, sc));
          o.w = pack_bf16x2(dequant1(v[6], z, sc), dequant1(v[7], z, sc));
          *reinterpret_cast<uint4*>(sw + row * 128 + ((cch ^ (row & 7)) << 4)) = o;
        }
        fence_proxy_async_smem();                // generic-proxy stores -> visible to the tensor core's reads
        named_barrier(1 + c, 128);
      }
      mbar_wait(&full_bar[stage], phase);
      if (tl && j == 0 && t == 0 && c == 0) tl_s[2] = tl_now();        // first operands landed
      const uint32_t sa = smem_u32(sw);
      const uint64_t dw = make_desc_k_sw128(sa + c * (64 * 128));
      const uint64_t dx = make_desc_k_sw128(sa + static_cast<uint32_t>(p.w_bytes));
      wgmma_fence();
      fence_regs(acc);
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        wgmma_ss<NB>(acc, dw + static_cast<uint64_t>(2 * k), dx + static_cast<uint64_t>(2 * k), (j > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(acc);
      if (t == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    pdl_wait();                                  // ws is still being read by the predecessor's consumers
    if (tl && t == 0 && c == 0) tl_s[3] = tl_now();                     // accumulator complete
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int nr = c * 64 + w * 16 + (lane >> 2) + 8 * h;             // weight row inside the tile
      const int n = n0 + nr;
      if (nr >= p.tile_n || n >= p.n_out) continue;
      float* dst = p.ws + static_cast<long long>(split) * p.batch_total * p.n_out + n;
#pragma unroll
      for (int jb = 0; jb < NB / 8; ++jb)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int b = 8 * jb + 2 * qd + e;
          if (b < p.batch) dst[static_cast<long long>(b) * p.n_out] = acc[4 * jb + 2 * h + e];
        }
    }
  }

  __syncthreads();
  if (tl && threadIdx.x == 0)
    tl_emit((1u << 28) | (static_cast<uint32_t>(EPI_PARTIAL) << 24) | (static_cast<uint32_t>(p.n_out) & 0xFFFFFFu),
            tl_s[0], tl_s[1], tl_s[2], tl_s[3], tl_now());
}

// Finishes a small-batch GEMM: out[b][n] = epi( sum_s ws[s][b][n] + bias[n] ) in a fixed
// summation order (deterministic, unlike atomics).
__global__ void splitk_epilogue_kernel(const float* __restrict__ ws, int splits, int B, int N,
                                       int mode, const __nv_bfloat16* __restrict__ bias,
                                       const __nv_bfloat16* __restrict__ res, long long ldr,
                                       __nv_bfloat16* __restrict__ out, long long ldo) {
  pdl_launch_dependents();
  pdl_wait();
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 2;
  const int b = blockIdx.y;
  if (n >= N) return;
  float a0 = 0.f, a1 = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float2 v = *reinterpret_cast<const float2*>(ws + (static_cast<long long>(s) * B + b) * N + n);
    a0 += v.x;
    a1 += v.y;
  }
  if (bias) {
    const uint32_t bw = *reinterpret_cast<const uint32_t*>(bias + n);
    a0 += bf16_lo(bw);
    a1 += bf16_hi(bw);
  }
  a0 = bf16_round(a0);
  a1 = bf16_round(a1);
  if (mode == EPI_BIAS_GELU) {
    a0 = gelu_tanh(a0);
    a1 = gelu_tanh(a1);
  } else if (mode == EPI_BIAS_RESIDUAL) {
    const uint32_t rw = *reinterpret_cast<const uint32_t*>(res + static_cast<long long>(b) * ldr + n);
    a0 += bf16_lo(rw);
    a1 += bf16_hi(rw);
  }
  *reinterpret_cast<uint32_t*>(out + static_cast<long long>(b) * ldo + n) = pack_bf16x2(a0, a1);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) return nullptr;
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// bf16 row-major [rows, cols] with row stride ld (elements); box = [box_rows, 64] 128B-swizzled.
int make_tmap_bf16_2d(CUtensorMap* tm, const void* base, long long rows, long long cols,
                      long long ld, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (ld * 2) % 16)
    return set_error("TMA operand must be 16-byte aligned with a 16-byte multiple row pitch");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                  box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled failed");
  return 0;
}

// raw bytes, row-major [rows][row_bytes] with row pitch pitch_bytes; box = [box_rows, box_bytes], no swizzle
// (staging tiles of packed int4 / int8 weights, gemm_quant.cu)
int make_tmap_u8_2d(CUtensorMap* tm, const void* base, long long rows, long long row_bytes, long long pitch_bytes,
                    int box_rows, int box_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) || pitch_bytes % 16 || box_bytes % 16 || box_rows < 1 || box_rows > 256)
    return set_error("TMA byte operand must be 16-byte aligned with 16-byte multiple pitch and box");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(row_bytes), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(pitch_bytes)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_bytes), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled (bytes) failed");
  return 0;
}

// ---- optional per-launch timing of the row-form GEMM (bench.py's roofline leg) ----
struct GemmProfile {
  bool on = false;
  std::vector<cudaEvent_t> pool;
  size_t used = 0;
  double flops = 0.0;
  long long launches = 0;
};
static GemmProfile g_prof;

void gemm_profile_enable(int on) {
  g_prof.on = on != 0;
  if (on) { g_prof.used = 0; g_prof.flops = 0.0; g_prof.launches = 0; }
}
// Sums the recorded start/stop pairs (synchronises on the last event). Returns 0 on success.
int gemm_profile_read(double* total_ms, double* total_flops, long long* launches) {
  double ms = 0.0;
  for (size_t i = 0; i + 1 < g_prof.used; i += 2) {
    if (cudaEventSynchronize(g_prof.pool[i + 1]) != cudaSuccess) return set_error("profile: event sync failed");
    float t = 0.f;
    if (cudaEventElapsedTime(&t, g_prof.pool[i], g_prof.pool[i + 1]) != cudaSuccess)
      return set_error("profile: elapsed time failed");
    ms += t;
  }
  *total_ms = ms; *total_flops = g_prof.flops; *launches = g_prof.launches;
  return 0;
}
static cudaEvent_t profile_event() {
  if (g_prof.used == g_prof.pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    g_prof.pool.push_back(e);
  }
  return g_prof.pool[g_prof.used++];
}

// bf16 3-D tensor [d2][d1][d0] (d0 contiguous) with byte strides s1, s2; box {b0, b1, b2}.
int make_tmap_bf16_3d(CUtensorMap* tm, const void* base, long long d0, long long d1, long long d2,
                      long long s1_bytes, long long s2_bytes, int b0, int b1, int b2, int swizzle_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (s1_bytes % 16) || (s2_bytes % 16))
    return set_error("TMA operand must be 16-byte aligned with 16-byte multiple strides");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1), static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(s1_bytes), static_cast<cuuint64_t>(s2_bytes)};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(b0), static_cast<cuuint32_t>(b1), static_cast<cuuint32_t>(b2)};
  cuuint32_t estr[3] = {1, 1, 1};
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                              : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                              : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled (3-D) failed");
  return 0;
}

static int g_num_sms = 0;
int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

template <int BN, int STAGES>
static int launch_gemm(const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p,
                       cudaStream_t stream) {
  using S = GemmSmem<BN, STAGES>;
  static_assert(S::kTotal <= 227 * 1024, "shared memory budget");
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<BN, STAGES>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  }
  const int total = p.m_blocks * p.n_blocks;
  int max_ctas = num_sms();
  if (g_gemm_sm_cap > 0 && g_gemm_sm_cap < max_ctas) max_ctas = g_gemm_sm_cap;   // experiments: leave SMs to a concurrent stream
  const int ctas = total < max_ctas ? total : max_ctas;
  const cudaError_t e = launch_k(gemm_bf16_kernel<BN, STAGES>, dim3(ctas), dim3(kGemmThreads),
                                 static_cast<size_t>(S::kTotal), stream, tA, tB, p);
  count_launch();
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

int g_patch_embed_unfused = 0;   // md_debug_gemm bit 7: patchify kernel + row-form GEMM instead of the fused kernel (A/B, tests)
void gemm_debug_flags(int flags) { g_gemm_debug = flags; g_patch_embed_unfused = (flags & 128) ? 1 : 0; }
void gemm_debug_sm_cap(int sms) { g_gemm_sm_cap = sms < 0 ? 0 : sms; }
// sm_90 has no CTA-pair MMA: every row-form tile is one CTA, so the selection has nothing to choose between
void gemm_force_cta_group(int) {}
// Installs (buf != nullptr) or removes the debug timeline buffer in every kernel translation unit.
int timeline_install_all(unsigned long long* buf, unsigned int* count, unsigned int cap) {
  Timeline t{buf, count, buf ? cap : 0u};
  if (timeline_install(t) != cudaSuccess) return set_error("timeline: cudaMemcpyToSymbol failed");
  timeline_install_attention(t);
  timeline_install_elementwise(t);
  timeline_install_attention_tc(t);
  return 0;
}

static int dispatch_gemm(int bn, const CUtensorMap& tA, const CUtensorMap& tB, const GemmParams& p,
                         cudaStream_t stream) {
  switch (bn) {      // stage = 16 KB of A + BN x 128 B of B; one stage is held by the MMAs in flight
    case 256: return launch_gemm<256, 4>(tA, tB, p, stream);
    case 192: return launch_gemm<192, 5>(tA, tB, p, stream);
    case 128: return launch_gemm<128, 6>(tA, tB, p, stream);
    case 64: return launch_gemm<64, 8>(tA, tB, p, stream);
    case 32: return launch_gemm<32, 10>(tA, tB, p, stream);
  }
  return set_error("unsupported BN");
}

// Row-form tile width: the widest of 256 / 192 / 128 whose padding of the last column tile costs at most 5 % of N
// (256 for N = 2048, 3456, 4304, 6144, 8192; 192 for N = 1152), 64 / 32 for narrow N.  md_debug_gemm bit 8 keeps
// every wide N at 128 (A/B timing and tests).
static int pick_bn_rows(int N) {
  if (N < 96) return N >= 48 ? 64 : 32;
  if (!(g_gemm_debug & 256))
    for (int bn : {256, 192})
      if (static_cast<long long>((N + bn - 1) / bn * bn - N) * 20 <= N) return bn;
  return 128;
}

static int run_rowform(const CUtensorMap& tA, const CUtensorMap& tB, int bn, GemmParams& p, cudaStream_t stream) {
  p.m_blocks = (p.M + BM - 1) / BM;
  p.n_blocks = (p.N + bn - 1) / bn;
  p.k_blocks = (p.K + BK - 1) / BK;
  p.early_trigger = (g_pdl && !(g_gemm_debug & 32)) ? 1 : 0;      // md_debug_gemm bit 5: off (A/B)
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  const bool prof = g_prof.on && cudaStreamIsCapturing(stream, &cap) == cudaSuccess &&
                    cap == cudaStreamCaptureStatusNone;
  if (prof) cudaEventRecord(profile_event(), stream);
  const int rc = dispatch_gemm(bn, tA, tB, p, stream);
  if (prof) {
    cudaEventRecord(profile_event(), stream);
    g_prof.flops += 2.0 * p.M * static_cast<double>(p.N) * p.K;
    g_prof.launches += 1;
  }
  return rc;
}

int gemm_rowform(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M,
                 int N, int K, int mode, const __nv_bfloat16* bias, const __nv_bfloat16* res,
                 long long ldr, int res_mod, __nv_bfloat16* out, long long ldo, int remap_gin,
                 int remap_gout, int remap_goff, cudaStream_t stream) {
  if (M <= 0 || N <= 0 || K <= 0) return set_error("gemm: empty problem");
  if (N % 8 || K % 8) return set_error("gemm: N and K must be multiples of 8");
  if (mode == EPI_BIAS_RESIDUAL && !res) return set_error("gemm: residual mode without residual");
  if ((ldo % 8) || (res && (ldr % 8))) return set_error("gemm: ldo/ldr must be multiples of 8");
  const int bn = pick_bn_rows(N);
  CUtensorMap tA, tB;
  if (make_tmap_bf16_2d(&tA, A, M, K, lda, BM)) return 1;
  if (make_tmap_bf16_2d(&tB, W, N, K, ldw, bn)) return 1;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.mode = mode;
  p.out = out; p.ldo = ldo; p.bias = bias; p.res = res; p.ldr = ldr; p.res_mod = res_mod;
  p.remap_gin = remap_gin; p.remap_gout = remap_gout; p.remap_goff = remap_goff;
  return run_rowform(tA, tB, bn, p, stream);
}

int gemm_rowform_qkv_rope(const __nv_bfloat16* A, long long lda, const __nv_bfloat16* W, long long ldw, int M,
                          int K, const __nv_bfloat16* bias, const RopeEpilogue& epi, cudaStream_t stream) {
  const int N = epi.D + 2 * epi.n_kv_heads * 64;
  if (M <= 0 || K <= 0) return set_error("gemm_qkv_rope: empty problem");
  if (K % 8 || epi.D % 64 || epi.D != epi.n_heads * 64 || epi.n_kv_heads <= 0 || epi.n_heads % epi.n_kv_heads || !bias)
    return set_error("gemm_qkv_rope: unsupported shape");
  const int bn = pick_bn_rows(N);                    // 2 to 4 heads per column tile: N and BN are multiples of 64
  CUtensorMap tA, tB;
  if (make_tmap_bf16_2d(&tA, A, M, K, lda, BM)) return 1;
  if (make_tmap_bf16_2d(&tB, W, N, K, ldw, bn)) return 1;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.mode = EPI_QKV_ROPE;
  p.bias = bias;
  p.rope = epi;
  return run_rowform(tA, tB, bn, p, stream);
}


// Plan of a small-batch weight stream: tile height (64 or 128 rows of W per CTA, one consumer warpgroup per 64) and
// k-blocks per split such that (tiles x splits) fills whole waves of the SMs.  cost = waves x tile_rows x kb is the
// critical path in units of 128-byte weight rows, plus this SM's share of the fp32 partial-sum traffic (written and
// re-read once per split, nominal batch 32); ties prefer fewer splits.  kb_divisor > 0 restricts kb to divisors of it.
StreamPlan plan_smallbatch(int n_out, int K, int kb_divisor) {
  const int k_blocks = (K + BK - 1) / BK;
  const int sms = num_sms();
  StreamPlan best{BM, k_blocks, 1};
  long long best_cost = -1;
  for (int kb = k_blocks; kb >= 1; --kb) {
    if (kb_divisor > 0 ? (kb > kb_divisor || kb_divisor % kb) : false) continue;
    const int splits = (k_blocks + kb - 1) / kb;
    if (splits > 32) break;
    if (kb_divisor == 0 && kb < 4 && k_blocks >= 4) break;           // keep >= 256 of K per split
    for (int rows = BM; rows >= 64; rows -= 64) {
      const int tiles = (n_out + rows - 1) / rows;
      const long long waves = (1LL * tiles * splits + sms - 1) / sms;
      const long long cost = waves * rows * kb + (1LL * splits * n_out * 32 * 8) / (128LL * sms);
      if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = StreamPlan{rows, kb, splits}; }
    }
  }
  return best;
}

// Plan for a K-concatenated weight stream [A | B] whose halves must not share a split (seg_K = width of A, a
// multiple of 64): the k-blocks of the longest CTA, as many short splits as keep every CTA resident at once.
StreamPlan2 plan_smallbatch_2seg(int n_out, int K, int seg_K) {
  const int k_blocks = (K + BK - 1) / BK;
  const int ka = seg_K / BK, kbt = k_blocks - ka;
  const int sms = num_sms();
  StreamPlan2 best{BM, 1, ka, 1, kbt};
  long long best_cost = -1;
  for (int rows = BM; rows >= 64; rows -= 64) {
    const int tiles = (n_out + rows - 1) / rows;
    for (int sa = 1; sa <= ka && sa <= 8; ++sa) {
      const int kba = (ka + sa - 1) / sa;
      if (kba * (sa - 1) >= ka) continue;                       // a split would be empty
      for (int sb = 1; sb <= kbt && sb <= 24; ++sb) {
        const int kbb = (kbt + sb - 1) / sb;
        if (kbb * (sb - 1) >= kbt) continue;
        const long long waves = (1LL * tiles * (sa + sb) + sms - 1) / sms;
        const long long cost = waves * rows * (kba > kbb ? kba : kbb) +
                               (1LL * (sa + sb) * n_out * 32 * 8) / (128LL * sms);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = StreamPlan2{rows, sa, kba, sb, kbb}; }
      }
    }
  }
  return best;
}

template <int NB, int BITS>
static cudaError_t launch_stream(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, const CUtensorMap& tX,
                                 const CUtensorMap& tW, const SmallBatchParams& p) {
  static DeviceOnce configured;
  if (configured.first()) {
    const cudaError_t e = cudaFuncSetAttribute(smallbatch_gemm_kernel<NB, BITS>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
    if (e != cudaSuccess) return e;
  }
  return launch_k(smallbatch_gemm_kernel<NB, BITS>, grid, block, smem, stream, tX, tW, p);
}
template <int BITS>
static cudaError_t launch_stream_nb(int nb, dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                    const CUtensorMap& tX, const CUtensorMap& tW, const SmallBatchParams& p) {
  switch (nb) {
    case 16: return launch_stream<16, BITS>(grid, block, smem, stream, tX, tW, p);
    case 32: return launch_stream<32, BITS>(grid, block, smem, stream, tX, tW, p);
    case 64: return launch_stream<64, BITS>(grid, block, smem, stream, tX, tW, p);
    default: return launch_stream<128, BITS>(grid, block, smem, stream, tX, tW, p);
  }
}

// ws[splits][batch][n_out] (fp32) = W[n_out,K] * X[batch,K]^T partial sums; split s owns k-blocks
// [s * kb_per_split, (s+1) * kb_per_split).  With seg_kb > 0 the k-blocks split in two segments: [0, seg_kb) in
// pieces of kb_per_split, the rest in pieces of kb_per_split2.  Batches above 128 rows run as consecutive 128-row
// launches.  Returns the number of splits (> 0), -1 on error.
int weight_stream(const StreamArgs& a, cudaStream_t stream) {
  if (a.n_out <= 0 || a.batch <= 0 || a.K <= 0) { set_error("small-batch GEMM: empty problem"); return -1; }
  if (a.K % 8) { set_error("small-batch GEMM: K must be a multiple of 8"); return -1; }
  if (a.bits != 16 && a.bits != 8 && a.bits != 4) { set_error("small-batch GEMM: bits must be 16, 8 or 4"); return -1; }
  if (a.tile_n != 64 && a.tile_n != 128) { set_error("small-batch GEMM: tile height must be 64 or 128"); return -1; }
  SmallBatchParams p{};
  p.batch_total = a.batch; p.n_out = a.n_out;
  p.k_blocks = (a.K + BK - 1) / BK;
  p.tile_n = a.tile_n;
  const int n_tiles = (a.n_out + p.tile_n - 1) / p.tile_n;
  int kb_per_split = a.kb_per_split < 1 ? 1 : (a.kb_per_split > p.k_blocks ? p.k_blocks : a.kb_per_split);
  p.kb_per_split = kb_per_split;
  int kb_max = kb_per_split;
  if (a.seg_kb > 0 && a.seg_kb < p.k_blocks) {
    const int kb2 = a.kb_per_split2 < 1 ? 1 : a.kb_per_split2;
    p.seg_kb = a.seg_kb;
    p.seg_splits = (a.seg_kb + kb_per_split - 1) / kb_per_split;
    p.kb_per_split2 = kb2;
    p.k_splits = p.seg_splits + (p.k_blocks - a.seg_kb + kb2 - 1) / kb2;
    if (kb2 > kb_max) kb_max = kb2;
  } else {
    p.k_splits = (p.k_blocks + kb_per_split - 1) / kb_per_split;   // every split owns >= 1 k-block
    p.seg_splits = p.k_splits; p.seg_kb = p.k_blocks; p.kb_per_split2 = kb_per_split;
  }
  p.trigger_early = g_pdl >= 2 ? 1 : 0;
  p.scale = a.scale; p.zero = a.zero;
  if (a.bits != 16) {
    p.groups = a.K / 128;
    p.max_groups = kb_max / 2 + 2;                     // a split starting on an odd k-block touches one more group
  }
  CUtensorMap tW;
  if (a.bits == 16) {
    if (make_tmap_bf16_2d(&tW, a.W, a.n_out, a.K, a.ldw, p.tile_n)) return -1;
  } else {
    const long long row_bytes = static_cast<long long>(a.K) * a.bits / 8;
    if (make_tmap_u8_2d(&tW, a.W, a.n_out, row_bytes, row_bytes, p.tile_n, BK * a.bits / 8)) return -1;
  }
  constexpr int kSmemMax = 227 * 1024 - 1024;          // leave room for the kernel's few static __shared__ words
  for (int b0 = 0; b0 < a.batch; b0 += BM) {
    p.batch = a.batch - b0 < BM ? a.batch - b0 : BM;
    const int nb = p.batch <= 16 ? 16 : p.batch <= 32 ? 32 : p.batch <= 64 ? 64 : 128;
    p.w_bytes = p.tile_n * BK * 2;                     // a multiple of 8 KB: every tile stays swizzle-aligned
    p.x_bytes = nb * BK * 2;
    p.q_bytes = a.bits == 16 ? 0 : p.tile_n * BK * a.bits / 8;
    p.stage_bytes = (p.w_bytes + p.x_bytes + p.q_bytes + 1023) / 1024 * 1024;
    const int fixed = 1024 + 2 * p.tile_n * p.max_groups * 4 + 8 + 3 * kSbMaxStages * 8;
    p.stages = (kSmemMax - fixed) / p.stage_bytes;
    if (p.stages > kSbMaxStages) p.stages = kSbMaxStages;
    if (p.stages < 2) { set_error("small-batch GEMM: tile does not fit shared memory"); return -1; }
    p.ws = a.ws + static_cast<long long>(b0) * a.n_out;
    CUtensorMap tX;                                    // rows past the batch are zero-filled up to nb
    if (make_tmap_bf16_2d(&tX, a.X + static_cast<long long>(b0) * a.ldx, p.batch, a.K, a.ldx, nb)) return -1;
    const size_t smem = static_cast<size_t>(p.stages) * p.stage_bytes + fixed;
    const dim3 grid(n_tiles * p.k_splits), block(128 * (1 + p.tile_n / 64));
    count_launch();
    const cudaError_t e = a.bits == 16 ? launch_stream_nb<16>(nb, grid, block, smem, stream, tX, tW, p)
                        : a.bits == 8  ? launch_stream_nb<8>(nb, grid, block, smem, stream, tX, tW, p)
                                       : launch_stream_nb<4>(nb, grid, block, smem, stream, tX, tW, p);
    if (e != cudaSuccess) { set_error(cudaGetErrorString(e)); return -1; }
  }
  return p.k_splits;
}

// upper bound over the plans a launch may pick (callers size their partial-sum workspace with it)
int gemm_smallbatch_splits(int n_out, int K) { return plan_smallbatch(n_out, K, 0).splits; }

int gemm_smallbatch(const __nv_bfloat16* W, long long ldw, const __nv_bfloat16* X, long long ldx,
                 int n_out, int batch, int K, int splits, float* ws, cudaStream_t stream) {
  (void)splits;                                  // the plan decides (callers size ws with gemm_smallbatch_splits)
  const StreamPlan pl = plan_smallbatch(n_out, K, 0);
  StreamArgs a{};
  a.bits = 16; a.W = W; a.ldw = ldw; a.X = X; a.ldx = ldx; a.n_out = n_out; a.batch = batch; a.K = K;
  a.tile_n = pl.tile_rows; a.kb_per_split = pl.kb; a.ws = ws;
  return weight_stream(a, stream);
}

// same as gemm_smallbatch for W = [A | B] along K with the split boundaries of plan_smallbatch_2seg: splits
// [0, splits_a) hold A's partial sums, the rest B's.  Returns the number of splits, -1 on error.
int gemm_smallbatch_2seg(const __nv_bfloat16* W, long long ldw, const __nv_bfloat16* X, long long ldx,
                      int n_out, int batch, int K, int seg_K, float* ws, cudaStream_t stream) {
  if (seg_K <= 0 || seg_K >= K || seg_K % BK) { set_error("gemm_smallbatch_2seg: segment boundary must be a multiple of 64 inside K"); return -1; }
  const StreamPlan2 pl = plan_smallbatch_2seg(n_out, K, seg_K);
  StreamArgs a{};
  a.bits = 16; a.W = W; a.ldw = ldw; a.X = X; a.ldx = ldx; a.n_out = n_out; a.batch = batch; a.K = K;
  a.tile_n = pl.tile_rows; a.kb_per_split = pl.kb_a; a.seg_kb = seg_K / BK; a.kb_per_split2 = pl.kb_b; a.ws = ws;
  return weight_stream(a, stream);
}

int splitk_epilogue(const float* ws, int splits, int B, int N, int mode, const __nv_bfloat16* bias,
                    const __nv_bfloat16* res, long long ldr, __nv_bfloat16* out, long long ldo,
                    cudaStream_t stream) {
  if (N % 2) return set_error("splitk_epilogue: N must be even");
  dim3 grid((N / 2 + 127) / 128, B);
  cudaError_t e = launch_k(splitk_epilogue_kernel, grid, dim3(128), 0, stream, ws, splits, B, N, mode, bias, res, ldr, out, ldo);
  count_launch();
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

}  // namespace md
