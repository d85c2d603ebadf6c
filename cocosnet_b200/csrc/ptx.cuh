// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (fence / commit / wait, accumulator staging) and the shared-memory
// matrix descriptors wgmma consumes.  No CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "wgmma_ops.cuh"

namespace cocos {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a launch failure by the
// C-ABI) instead of hanging the GPU.
#ifndef COCOS_MBAR_SPIN_LIMIT
#define COCOS_MBAR_SPIN_LIMIT (1u << 24)
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > COCOS_MBAR_SPIN_LIMIT) {
      printf("cocos: mbarrier timeout block(%d,%d) thread %d bar 0x%x parity %u\n", blockIdx.x, blockIdx.y,
             threadIdx.x, bar, parity);
      __trap();
    }
  }
}
// The same bound without the report, for every wait of a kernel that issues wgmma, its producer warp included: ptxas
// serialises all wgmma of a kernel that contains a function call (the printf above is one), waiting for each wgmma to
// complete before the next is issued.
__device__ __forceinline__ void mbar_wait_quiet(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > COCOS_MBAR_SPIN_LIMIT) __trap();
  }
}

// ----------------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// -------------------------------------------------------------------- wgmma
// Warpgroup MMA (sm_90a): D (registers, fp32) (+)= A * B over a 64-row slab per warpgroup; see wgmma_ops.cuh.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// named barrier over `n` threads (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// Accumulator fragment of m64nN (thread t of the warpgroup: rows 16*(t/32) + (t%32)/4 and +8, column pairs
// 8j + 2*(t%4), registers d[4j, 4j + 4)) -> row-major fp32 tile rows [row0, row0 + 64), pitch `ld` floats (even).
// One 8-column block: fragment block j (d4 = d + 4j) -> tile columns [8 jd, 8 jd + 8).
__device__ __forceinline__ void acc_block_to_smem(const float* d4, float* tile, int ld, int row0, int jd) {
  const int t = threadIdx.x & 127;
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 8 * jd + 2 * (t & 3);
  *reinterpret_cast<float2*>(tile + r * ld + c) = make_float2(d4[0], d4[1]);
  *reinterpret_cast<float2*>(tile + (r + 8) * ld + c) = make_float2(d4[2], d4[3]);
}
template <int N>
__device__ __forceinline__ void acc_to_smem(const float* d, float* tile, int ld, int row0) {
#pragma unroll
  for (int j = 0; j < N / 8; ++j) acc_block_to_smem(d + 4 * j, tile, ld, row0, j);
}
// N consecutive fp32 of a staged accumulator row (16-byte aligned) as raw bits
template <int N>
__device__ __forceinline__ void acc_ld(const float* src, uint32_t* r) {
#pragma unroll
  for (int i = 0; i < N / 4; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
  }
}
__device__ __forceinline__ void acc_ld32(const float* src, uint32_t* r) { acc_ld<32>(src, r); }

// --------------------------------------------------------------- descriptors
// K-major operand tile staged by TMA with SWIZZLE_128B: rows of 64 16-bit elements (128 B), 8-row groups 1024 B apart.
// wgmma matrix descriptor: start[0,14) lbo[16,30) sbo[32,46) layout[62,64)=1 (128B swizzle), addresses in 16 B units.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;            // leading byte offset (unused for swizzled K-major)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // stride byte offset: 8 rows * 128 B
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}
// MN-major operand, SWIZZLE_128B: 64-element (128 B) rows along MN, 8 K-rows 1024 B apart (SBO), the next 64-element
// block along MN `lbo_bytes` further.
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo_bytes >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// descriptor for the next 16-element K step inside a 128B swizzle atom (+32 bytes)
__device__ __forceinline__ uint64_t desc_advance_k16(uint64_t d, int steps) { return d + static_cast<uint64_t>(2 * steps); }

// ------------------------------------------------------- 128-row tile main loop
// The GEMM-like kernels run two consumer warpgroups (warps 0-7; warpgroup g owns accumulator rows [64g, 64g + 64))
// and one TMA producer warp (warp 8).  Stage `st` of the ring is released with one arrive per consumer warp, so the
// `empty` barriers are initialised with CONSUMER_WARPS.
constexpr int CONSUMER_WARPS = 8;
constexpr int TILE_THREADS = 32 * CONSUMER_WARPS + 32;

// The consumers' position in the ring (stage, phase); a persistent kernel carries it from tile to tile.
struct RingPos {
  uint32_t st = 0, ph = 0;
  __device__ __forceinline__ void advance(int stages) {
    if (++st == static_cast<uint32_t>(stages)) { st = 0; ph ^= 1; }
  }
};

// one arrive per consumer warp on `empty`: the stage's buffers go back to the producer
__device__ __forceinline__ void release_stage(uint64_t* empty) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(smem_u32(empty));
}

// d (+)= sum over `iters` stages of 4 K16 steps; desc(st, k, da, db) gives this warpgroup's descriptors.  One commit
// group (the 4 wgmmas of a stage) stays in flight while the next stage is waited for and issued: stage s - 1 is
// released once wait<1> after stage s's commit shows it complete.  The stages are summed in the same order either way.
template <int BN, bool BF16, typename Desc>
__device__ __forceinline__ void consume_stages_t(float* d, int iters, int stages, uint64_t* full, uint64_t* empty,
                                                 int tnsp, Desc desc, RingPos& rp) {
  uint32_t prev = 0;
  for (int it = 0; it < iters; ++it) {
    mbar_wait_quiet(smem_u32(&full[rp.st]), rp.ph);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint64_t da, db;
      desc(rp.st, k, da, db);
      wgmma_ss<BN, BF16>(d, da, db, (it | k) != 0 ? 1 : 0, tnsp);
    }
    wgmma_commit();
    wgmma_wait<1>();
    if (it > 0) release_stage(&empty[prev]);
    prev = rp.st;
    rp.advance(stages);
  }
  wgmma_wait<0>();
  if (iters > 0) release_stage(&empty[prev]);
}
template <int BN, typename Desc>
__device__ __forceinline__ void consume_stages(float* d, int iters, int stages, uint64_t* full, uint64_t* empty,
                                               bool bf16, int tnsp, Desc desc, RingPos& rp) {
  if (bf16) consume_stages_t<BN, true>(d, iters, stages, full, empty, tnsp, desc, rp);
  else consume_stages_t<BN, false>(d, iters, stages, full, empty, tnsp, desc, rp);
}
template <int BN, typename Desc>
__device__ __forceinline__ void consume_stages(float* d, int iters, int stages, uint64_t* full, uint64_t* empty,
                                               bool bf16, int tnsp, Desc desc) {
  RingPos rp;
  consume_stages<BN>(d, iters, stages, full, empty, bf16, tnsp, desc, rp);
}

// After the main loop: both warpgroups write their accumulators into the (drained) operand ring as a row-major fp32
// tile of 128 rows, pitch BN + 4, for an epilogue that reads one row per thread.
template <int BN>
__device__ __forceinline__ float* stage_acc(const float* d, uint8_t* ring) {
  float* tile = reinterpret_cast<float*>(ring);
  bar_sync(1, 32 * CONSUMER_WARPS);  // every consumer warp is past its last wgmma on the ring
  acc_to_smem<BN>(d, tile, BN + 4, 64 * (threadIdx.x >> 7));
  bar_sync(1, 32 * CONSUMER_WARPS);
  return tile;
}

// one lane of a converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

}  // namespace cocos
