// Patch embedding as ONE im2col-fused wgmma GEMM (reference vision.py:25-41 prepare_crops' normalisation, :44-61
// create_patches, :67-68 `patch_emb(x) + pos_emb`):
//
//     x[r][n] = bf16( bf16( sum_k lut[pixel(r, k)] * W[n][k] + bias[n] ) + pos_emb[r % tokens][n] )
//
// r = (crop, patch row, patch column), k = (channel, py, px).  The [tokens, 588] patch matrix never exists in HBM: the
// A operand of the MMAs is gathered from the uint8 NHWC crops (256-entry LUT = the reference's bf16 rounding chain per
// byte, so the pixel path stays bit-exact) straight into 128B-swizzled shared-memory tiles by the CTA's own warps.
//
//   warpgroup 0     : TMA producer for the weight tiles W[n chunk of 128][k-block of 64]  (3-stage ring, K tail zero-filled)
//   warpgroups 1, 2 : gather the 128 x 640 A tile of a row tile (10 k-blocks; columns 588..639 zero), then for each n
//                     chunk run wgmma m64 x 128 x 16 on their 64 rows and drain the registers: + bias, round, + pos_emb,
//                     round, stores
// Persistent over row tiles (one CTA per SM).  The accumulation order over K is the row-form GEMM's (the same K = 16
// steps in the same order; the row form's wider n192 / n256 instruction gives the same bits per element), so the result
// equals patchify + gemm_rowform bit for bit (tests/test_model_parity_gpu.py).
#include "kernels.cuh"
#include "ptx.cuh"

namespace md {

namespace pe {
constexpr int BM = 128, BN = 128, BK = 64;
constexpr int kStages = 3;
constexpr int kThreads = 384;
constexpr int kWorkers = 256;                    // warpgroups 1, 2
constexpr int kMaxKBlocks = 10;                  // K <= 640 (patch 14 x 14 x 3 = 588)
constexpr int kATile = BM * BK * 2;              // 16 KB per k-block
constexpr int kWTile = BN * BK * 2;              // 16 KB
}  // namespace pe

struct PatchEmbedParams {
  const uint8_t* crops;                          // [n_crops, crop, crop, 3]
  int n_crops, crop, patch, grid, tokens;        // tokens = grid * grid
  int T, N, K, k_blocks, n_chunks, row_tiles;    // T = n_crops * tokens, N = enc_dim, K = 3 * patch^2
  const __nv_bfloat16* lut;                      // [256]
  const __nv_bfloat16* bias;                     // [N]
  const __nv_bfloat16* pos_emb;                  // [tokens, N]
  __nv_bfloat16* out;                            // [T, N]
};

__global__ void __launch_bounds__(pe::kThreads, 1)
patch_embed_kernel(const __grid_constant__ CUtensorMap tmW, const PatchEmbedParams p) {
  using namespace pe;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;                                            // [k_blocks][128 x 64] bf16, 128B-swizzled
  uint8_t* sW = sA + kMaxKBlocks * kATile;                       // [kStages][128 x 64]
  int* s_koff = reinterpret_cast<int*>(sW + kStages * kWTile);   // [k_blocks * 64] byte offset of feature k in a patch, -1 = pad
  __nv_bfloat16* s_lut = reinterpret_cast<__nv_bfloat16*>(s_koff + kMaxKBlocks * BK);
  uint64_t* wfull = reinterpret_cast<uint64_t*>(s_lut + 256);
  uint64_t* wempty = wfull + kStages;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmW);
    for (int i = 0; i < kStages; ++i) { mbar_init(&wfull[i], 1); mbar_init(&wempty[i], 2); }
    fence_barrier_init();
  }
  // feature k = (c, py, px) -> byte offset inside the patch's pixel window; constants of the launch
  for (int k = threadIdx.x; k < p.k_blocks * BK; k += kThreads) {
    int off = -1;
    if (k < p.K) {
      const int pp = p.patch * p.patch;
      const int c = k / pp, rem = k - c * pp, py = rem / p.patch, px = rem - py * p.patch;
      off = (py * p.crop + px) * 3 + c;
    }
    s_koff[k] = off;
  }
  for (int i = threadIdx.x; i < 256; i += kThreads) s_lut[i] = p.lut[i];
  __syncthreads();
  pdl_launch_dependents();

  const int n_my_tiles = (p.row_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x);
  const int wg = threadIdx.x >> 7;

  if (wg == 0) {
    // ------------------------------ weight tiles (constants: no dependency wait) ------------------------------
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = 0; t < n_my_tiles; ++t)
        for (int nc = 0; nc < p.n_chunks; ++nc)
          for (int kb = 0; kb < p.k_blocks; ++kb) {
            mbar_wait(&wempty[stage], phase ^ 1);
            mbar_arrive_expect_tx(&wfull[stage], kWTile);
            tma_load_2d(sW + stage * kWTile, &tmW, &wfull[stage], kb * BK, nc * BN);
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
    }
  } else {
    const int wt = threadIdx.x - 128;
    const int c = wg - 1;                           // accumulator rows 64c .. 64c+63 of the row tile
    const int t128 = threadIdx.x & 127;
    const int lane = t128 & 31, w = t128 >> 5, qd = lane & 3;
    pdl_wait();                                     // crops may come from a preceding kernel (device preprocessing)
    int stage = 0;
    uint32_t phase = 0;
    for (int t = 0; t < n_my_tiles; ++t) {
      const int tile = static_cast<int>(blockIdx.x) + t * static_cast<int>(gridDim.x);
      const int r0 = tile * BM;
      // ---- gather: (row, 16-byte chunk of 8 features) items; a warp writes four full 128-byte lines per store ----
      if (t > 0) named_barrier(1, kWorkers);        // both warpgroups' MMAs of the previous row tile have read A
      const int chunks = p.k_blocks * 8;
      for (int i = wt; i < BM * chunks; i += kWorkers) {
        const int row = i / chunks, cc = i - row * chunks;
        const int r = r0 + row;
        uint4 o = make_uint4(0, 0, 0, 0);
        if (r < p.T) {
          const int n = r / p.tokens, tok = r - n * p.tokens, gy = tok / p.grid, gx = tok - gy * p.grid;
          const uint8_t* base = p.crops + ((static_cast<long long>(n) * p.crop + gy * p.patch) * p.crop + gx * p.patch) * 3;
          uint32_t wd[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int o0 = s_koff[cc * 8 + 2 * j], o1 = s_koff[cc * 8 + 2 * j + 1];
            const uint32_t lo = o0 >= 0 ? static_cast<uint32_t>(__bfloat16_as_ushort(s_lut[base[o0]])) : 0u;
            const uint32_t hi = o1 >= 0 ? static_cast<uint32_t>(__bfloat16_as_ushort(s_lut[base[o1]])) : 0u;
            wd[j] = lo | (hi << 16);
          }
          o = make_uint4(wd[0], wd[1], wd[2], wd[3]);
        }
        *reinterpret_cast<uint4*>(sA + (cc >> 3) * kATile + row * 128 + (((cc & 7) ^ (row & 7)) << 4)) = o;
      }
      fence_proxy_async_smem();                     // generic-proxy stores -> visible to the tensor core's reads
      named_barrier(1, kWorkers);
      // ---- this row tile's n chunks ----
      for (int nc = 0; nc < p.n_chunks; ++nc) {
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait(&wfull[stage], phase);
          const uint64_t da = make_desc_k_sw128(smem_u32(sA + kb * kATile + c * (64 * 128)));
          const uint64_t db = make_desc_k_sw128(smem_u32(sW + stage * kWTile));
          wgmma_fence();
          fence_regs(acc);
#pragma unroll
          for (int k = 0; k < BK / 16; ++k)
            wgmma_ss<BN>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                         (kb > 0 || k > 0) ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          fence_regs(acc);
          if (t128 == 0) mbar_arrive(&wempty[stage]);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + c * 64 + w * 16 + (lane >> 2) + 8 * h;
          if (row >= p.T) continue;
          const __nv_bfloat16* prow = p.pos_emb + static_cast<long long>(row % p.tokens) * p.N;
          __nv_bfloat16* orow = p.out + static_cast<long long>(row) * p.N;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = nc * BN + 8 * j + 2 * qd;
            if (col >= p.N) continue;                                 // N is a multiple of 8
            const uint32_t bw = *reinterpret_cast<const uint32_t*>(p.bias + col);
            const uint32_t pw = *reinterpret_cast<const uint32_t*>(prow + col);
            // the Linear output is a bf16 tensor before pos_emb is added (vision.py:67-68)
            const float v0 = bf16_round(acc[4 * j + 2 * h] + bf16_lo(bw)) + bf16_lo(pw);
            const float v1 = bf16_round(acc[4 * j + 2 * h + 1] + bf16_hi(bw)) + bf16_hi(pw);
            *reinterpret_cast<uint32_t*>(orow + col) = pack_bf16x2(v0, v1);
          }
        }
      }
    }
  }
}

// x [n_crops * grid^2, N] = patch_emb(patches(crops)) + pos_emb   (W: [N, k_pad] with zero columns >= 3 * patch^2)
int patch_embed_fused(const uint8_t* crops, int n_crops, int crop, int patch, const __nv_bfloat16* lut,
                      const __nv_bfloat16* W, int k_pad, const __nv_bfloat16* bias, const __nv_bfloat16* pos_emb, int N,
                      __nv_bfloat16* out, cudaStream_t stream) {
  using namespace pe;
  if (n_crops <= 0) return set_error("patch_embed: empty batch");
  const int K = 3 * patch * patch;
  if (crop % patch || k_pad < K || k_pad % 8 || N % 8) return set_error("patch_embed: bad geometry");
  const int k_blocks = (k_pad + BK - 1) / BK;
  if (k_blocks > kMaxKBlocks) return set_error("patch_embed: patch too large for the shared-memory A tile");
  PatchEmbedParams p{};
  p.crops = crops; p.n_crops = n_crops; p.crop = crop; p.patch = patch; p.grid = crop / patch;
  p.tokens = p.grid * p.grid;
  p.T = n_crops * p.tokens; p.N = N; p.K = K; p.k_blocks = k_blocks;
  p.n_chunks = (N + BN - 1) / BN;
  p.row_tiles = (p.T + BM - 1) / BM;
  p.lut = lut; p.bias = bias; p.pos_emb = pos_emb; p.out = out;
  CUtensorMap tW;
  if (make_tmap_bf16_2d(&tW, W, N, k_pad, k_pad, BN)) return 1;
  constexpr int kSmem = kMaxKBlocks * kATile + kStages * kWTile + kMaxKBlocks * BK * 4 + 512 + 2 * kStages * 8 + 1024;
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
  static DeviceOnce configured;
  if (configured.first()) {
    cudaError_t e = cudaFuncSetAttribute(patch_embed_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
    if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  }
  const int ctas = p.row_tiles < num_sms() ? p.row_tiles : num_sms();
  count_launch();
  cudaError_t e = launch_k(patch_embed_kernel, dim3(ctas), dim3(kThreads), static_cast<size_t>(kSmem), stream, tW, p);
  if (e != cudaSuccess) return set_error(cudaGetErrorString(e));
  return 0;
}

}  // namespace md
