// Device helpers shared by the wgmma kernels (sm_90a): shared-memory operand tiles, descriptors, wgmma fences, the
// 3xTF32 operand split.
//
// Operand tiles are K-major with the 128-byte swizzle: one tile row holds 32 consecutive k (128 bytes), 16-byte chunk
// j of row m sits at chunk j ^ (m & 7), rows follow each other every 128 bytes (8-row groups of 1024 bytes).  Tiles
// start at 1024-byte boundaries, so a wgmma descriptor addresses the k-step ks (8 tf32 = 32 bytes) of a tile by adding
// 32 * ks bytes to the start address.  The wide tiles of conv_wg_kernel hold 16 k per row instead, with the 64-byte
// swizzle: chunk j of row m at chunk j ^ ((m >> 1) & 3), rows every 64 bytes (8-row groups of 512 bytes).
#pragma once
#include <stdint.h>
#include "../../include/cape_b200.h"
#include "wgmma_tf32.cuh"

namespace cape {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory matrix descriptor: K-major, tile rows of ROW_BYTES = 128 (SWIZZLE_128B, layout type 1) or 64
// (SWIZZLE_64B, layout type 2), stride between 8-row groups 8 * ROW_BYTES
template <int ROW_BYTES = 128>
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  static_assert(ROW_BYTES == 128 || ROW_BYTES == 64, "128- or 64-byte swizzle");
  return (uint64_t)((smem_addr >> 4) & 0x3fffu) | (1ull << 16) | ((uint64_t)(8 * ROW_BYTES >> 4) << 32) |
         ((ROW_BYTES == 128 ? 1ull : 2ull) << 62);
}

// byte offset of element (m, k) (k = 0..31) of a tile
__device__ __forceinline__ uint32_t sw_off(int m, int k) {
  return (uint32_t)(m * 128 + ((((k >> 2) ^ (m & 7)) << 4) | ((k & 3) << 2)));
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// waits until at most N of this warpgroup's committed wgmma groups are still pending
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// shared-memory mbarriers for producer/consumer rings: thread arrivals, and the transaction bytes of TMA loads
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// makes the initialised mbarriers visible to the asynchronous proxy (TMA completions), before the __syncthreads
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// arrives and adds `bytes` to the transaction count the phase waits for (issued before the loads that complete them)
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA: the box at coordinates (x0 innermost, x1) of a 2-d tensor map into shared memory (`dst` 1024-byte aligned for
// the 128-byte swizzle), completing its bytes on `bar`; elements outside the tensor are filled with zeros
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, int x0, int x1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(x0), "r"(x1), "r"(smem_u32(bar)) : "memory");
}
// waits until the phase of parity `parity` has completed (a fresh barrier counts its phase "before 0" as parity 1)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!done);
}
// named barrier over a subset of the CTA's warps (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// per-warpgroup register budget (all four warps of the warpgroup execute it)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// keeps the compiler from moving accumulator reads or writes across the asynchronous MMAs
template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// 3xTF32 operand split: hi = x with the low 13 mantissa bits cleared (exactly representable in tf32), lo = x - hi
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

// four consecutive k of one tile row (16-byte aligned chunk) into the hi and lo tiles
__device__ __forceinline__ void split_store4(float4 v, char* hi_tile, char* lo_tile, uint32_t off) {
  float4 h, l;
  h.x = tf32_hi(v.x); l.x = v.x - h.x;
  h.y = tf32_hi(v.y); l.y = v.y - h.y;
  h.z = tf32_hi(v.z); l.z = v.z - h.z;
  h.w = tf32_hi(v.w); l.w = v.w - h.w;
  *reinterpret_cast<float4*>(hi_tile + off) = h;
  *reinterpret_cast<float4*>(lo_tile + off) = l;
}
__device__ __forceinline__ void split_store1(float v, char* hi_tile, char* lo_tile, uint32_t off) {
  const float h = tf32_hi(v);
  *reinterpret_cast<float*>(hi_tile + off) = h;
  *reinterpret_cast<float*>(lo_tile + off) = v - h;
}

// acc += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo over the KS k-steps of 8 of one tile row (KS = 4: a 32-deep chunk with
// the 128-byte swizzle; KS = 2: the 16-deep half of one with the 64-byte swizzle), A = 64 rows of this warpgroup
template <int N, int KS = 4>
__device__ __forceinline__ void mma3_chunk(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                           uint32_t b_lo, int scale_first) {
  constexpr int RB = 32 * KS;
#pragma unroll
  for (int ks = 0; ks < KS; ++ks) {
    const uint32_t adv = 32u * ks;
    wg::mma_tf32<N>(d, make_desc<RB>(a_hi + adv), make_desc<RB>(b_hi + adv), ks == 0 ? scale_first : 1);
    wg::mma_tf32<N>(d, make_desc<RB>(a_lo + adv), make_desc<RB>(b_hi + adv), 1);
    wg::mma_tf32<N>(d, make_desc<RB>(a_hi + adv), make_desc<RB>(b_lo + adv), 1);
  }
}

// accumulator fragment of m64nNk8 (f32): element i of thread `t` of the warpgroup is at
//   row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),   col = 8 * (i / 4) + 2 * (t % 4) + (i % 2)
__device__ __forceinline__ int frag_row(int t, int i) { return 16 * (t >> 5) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int frag_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

}  // namespace tc
}  // namespace cape
