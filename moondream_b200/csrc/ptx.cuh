// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait, descriptors; the MMAs are in wgmma.cuh),
// cp.async, ldmatrix, mma.sync.  No CUTLASS dependency; descriptor bit layouts follow the PTX ISA wgmma
// "matrix descriptor" table.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace md {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

// ----------------------------------------------------------------------------------------------
// programmatic dependent launch: a kernel may start (prologue) while its predecessor drains;
// pdl_wait() blocks until the predecessor grid has completed and its writes are visible.
// Both are no-ops for a kernel launched without the attribute.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must become a trap (reported launch failure), never a hung GPU.
// try_wait may itself suspend for a system-dependent time, so the bound is on elapsed clocks.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done = 0;
  long long t0 = 0;
  for (uint32_t spins = 0; !done; ++spins) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    if (!done && (spins & 0xFF) == 0xFF) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > 4000000000LL) __trap();      // ~2 s at 2 GHz
    }
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
// hint: bring the 128-byte line holding `p` into L2 (no register result, no fault on the data path)
__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
// 2-D tiled load: c0 = innermost (contiguous) coordinate, c1 = row coordinate.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// 1-D bulk copy of `bytes` (a multiple of 16, both addresses 16-byte aligned) global -> this CTA's shared memory
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(gsrc)), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// 3-D tiled load (c0 innermost)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tm, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA): the four warps of a warpgroup issue together; accumulators live in registers.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Per-thread register budget of the executing warpgroup (all 128 threads execute it): `dec` hands registers back to
// the CTA's pool, `inc` takes them from it.  R is a multiple of 8 in [24, 256].
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
// barrier over `threads` threads (a multiple of 32) under hardware barrier `id` (0 is __syncthreads)
__device__ __forceinline__ void named_barrier(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// Shared-memory matrix descriptors (PTX ISA "matrix descriptor" for wgmma): start address >> 4 at [0,14), leading
// byte offset >> 4 at [16,30), stride byte offset >> 4 at [32,46), layout at [62,64) (1 = 128B, 3 = 32B swizzle).
// Tiles are written by TMA with the matching CU_TENSOR_MAP_SWIZZLE_* and start on a swizzle-atom boundary.
//
// K-major bf16 tile stored as rows of 64 elements (128 B) with the 128-byte swizzle: 8-row groups are 1024 B apart
// (SBO); LBO is unused for swizzled K-major layouts.  Advancing 16 elements along K inside the row is +32 B, i.e. +2
// on the descriptor.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}
// 32-byte-swizzled tiles (rows of 32 B = 16 bf16, 8-row groups 256 B apart) for the 16-wide tail of a 72-wide head:
// K-major (Q, K: rows = tokens) and MN-major (V: rows = keys, 16 dims along N).
__device__ __forceinline__ uint64_t make_desc_sw32(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(256 >> 4) << 16;
  d |= static_cast<uint64_t>(256 >> 4) << 32;
  d |= static_cast<uint64_t>(3) << 62;
  return d;
}
// MN-major 128B-swizzled tile (rows = K index, the 64 elements of a row run along N): V in O += P V, straight from the
// [keys, 64] image TMA writes.  SBO = 1024 B between 8-row K groups; N = 64 is a single swizzle row, so LBO (the
// distance between 64-wide N blocks) is never used.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1024 >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// Ampere-style async copy / ldmatrix / mma.sync (used by the attention kernels)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;  // src-size 0 => zero-fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(sz)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t (&r)[2], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];"
               : "=r"(r[0]), "=r"(r[1])
               : "r"(saddr));
}
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t (&r)[2], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];"
               : "=r"(r[0]), "=r"(r[1])
               : "r"(saddr));
}
// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4],
                                               const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, "
      "{%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ----------------------------------------------------------------------------------------------
// numerics helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }
// ---- weight-only quantisation (gemm_quant.cu layout) ----
// 8 packed weights -> 8 fp32 values (exact)
template <int BITS>
__device__ __forceinline__ void unpack8(const uint8_t* src, float (&v)[8]) {
  if (BITS == 4) {
    const uint32_t w = *reinterpret_cast<const uint32_t*>(src);
#pragma unroll
    for (int j = 0; j < 8; ++j)       // 2^23 + nibble is exact in fp32; so is the difference
      v[j] = __uint_as_float(0x4B000000u | ((w >> (4 * j)) & 15u)) - 8388608.f;
  } else {
    const uint2 w = *reinterpret_cast<const uint2*>(src);
    const uint32_t ws2[2] = {w.x ^ 0x80808080u, w.y ^ 0x80808080u};     // signed byte + 128
#pragma unroll
    for (int j = 0; j < 8; ++j)
      v[j] = __uint_as_float(0x4B000000u | ((ws2[j >> 2] >> (8 * (j & 3))) & 255u)) - 8388736.f;   // 2^23 + 128
  }
}

// the reference's dequantisation of one value (layers.py:42-43: `W_r.sub_(zero).mul_(scale)` on a bf16 tensor with
// fp32 parameters: each step is evaluated in fp32 and rounded to bf16)
__device__ __forceinline__ float dequant1(float v, float zero, float scale) {
  return __fmul_rn(bf16_round(__fsub_rn(v, zero)), scale);      // the caller rounds the product to bf16 when packing
}

// tanh-approximated GELU exactly as F.gelu(approximate="tanh") states it
// (reference: moondream/torch/layers.py:24-25), evaluated in fp32.
__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5 x (1 + tanh(u)) == x * sigmoid(2u) == x / (1 + 2^(-2u log2 e)),  u = sqrt(2/pi) (x + 0.044715 x^3)
  const float kA = -2.0f * 0.7978845608028654f * 1.4426950408889634f;   // -2 sqrt(2/pi) log2(e)
  const float kKappa = 0.044715f;
  const float t = kA * (x + kKappa * x * x * x);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));                   // ~2 ulp
  return __fdividef(x, 1.0f + e);
}

// ---- debug timeline (md_debug_timeline) ----
// Per-CTA %globaltimer stamps, written only while a buffer is installed (tools/decode_timeline.py): the
// ground truth for where a decode step's time goes once PDL overlaps adjacent kernels and CUDA events
// or ncu (which serialises launches) can no longer tell.  One __constant__ copy per translation unit.
struct Timeline { unsigned long long* buf; unsigned int* count; unsigned int cap; };
constexpr int kTimelineWords = 6;   // {tag << 32 | block, entry, after dependency wait, mid0, mid1, exit}
static __constant__ Timeline c_timeline;
__device__ __forceinline__ bool tl_on() { return c_timeline.buf != nullptr; }
__device__ __forceinline__ unsigned long long tl_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void tl_emit(uint32_t tag, unsigned long long t0, unsigned long long t1,
                                        unsigned long long t2, unsigned long long t3, unsigned long long t4) {
  const unsigned int i = atomicAdd(c_timeline.count, 1u);
  if (i >= c_timeline.cap) return;
  unsigned long long* r = c_timeline.buf + static_cast<size_t>(i) * kTimelineWords;
  const uint32_t blk = blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z);
  r[0] = (static_cast<unsigned long long>(tag) << 32) | blk;
  r[1] = t0; r[2] = t1; r[3] = t2; r[4] = t3; r[5] = t4;
}
static inline cudaError_t timeline_install(const Timeline& t) {
  return cudaMemcpyToSymbol(c_timeline, &t, sizeof(t));
}

}  // namespace md
