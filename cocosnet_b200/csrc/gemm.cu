// Plain batched wgmma GEMM for sm_90a:
//   C[b] (M x N fp32, row-major) = alpha * A[b] (M x K fp16) * B[b]^T (N x K fp16)  [+ C]
// Both operands K-contiguous ("K-major"), staged by TMA into 128B-swizzled
// shared memory; 128 x BN output tile per CTA, 64-wide K chunks through a
// multi-stage mbarrier ring; accumulators in the registers of two warpgroups.
//   warp 8: TMA producer, warps 0-7: wgmma (64 rows each) + epilogue.
// Used by the correspondence backward (dQ = dS K, dK = dS^T Q) and by the
// SAGAN-attention / 1x1-conv paths.
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

#include <stdlib.h>

namespace cocos {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int ATOM_BYTES = 128 * BK * 2;
constexpr int MAX_STAGES = 6;
constexpr int NUM_THREADS = TILE_THREADS;

struct GemmParams {
  int M, N, K, ldc;
  long long stride_c;
  float alpha;
  int accumulate;
  int bf16;
  float* c;
};

struct GemmBars {
  uint64_t full[MAX_STAGES];
  uint64_t empty[MAX_STAGES];
};

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_f16_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                const GemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));
  constexpr int STAGES = (BN == 128) ? 6 : 4;
  constexpr int STAGE_BYTES = ATOM_BYTES + (BN / 128) * ATOM_BYTES;
  GemmBars* bars = reinterpret_cast<GemmBars*>(smem_gen + STAGES * STAGE_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN, bz = blockIdx.z;
  const int kc_count = (p.K + BK - 1) / BK;

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(smem_u32(&bars->full[i]), 1);
      mbar_init(smem_u32(&bars->empty[i]), CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      uint32_t st = 0, ph = 0;
      for (int kc = 0; kc < kc_count; ++kc) {
        mbar_wait_quiet(smem_u32(&bars->empty[st]), ph ^ 1);
        const uint32_t full = smem_u32(&bars->full[st]);
        mbar_expect_tx(full, STAGE_BYTES);
        tma_load_3d(smem0 + st * STAGE_BYTES, &tm_a, full, kc * BK, m0, bz);
        tma_load_3d(smem0 + st * STAGE_BYTES + ATOM_BYTES, &tm_b, full, kc * BK, n0, bz);
        if (++st == STAGES) { st = 0; ph ^= 1; }
      }
    }
    __syncwarp();
  } else {
    float d[BN / 2];
    const uint32_t a_off = (tid >> 7) * 64 * 128;  // this warpgroup's 64 rows of the A atom
    consume_stages<BN>(d, kc_count, STAGES, bars->full, bars->empty, p.bf16 != 0, 0,
                       [&](uint32_t st, int k, uint64_t& da, uint64_t& db) {
                         const uint32_t a_addr = smem0 + st * STAGE_BYTES;
                         da = desc_advance_k16(make_desc_k_sw128(a_addr + a_off), k);
                         db = desc_advance_k16(make_desc_k_sw128(a_addr + ATOM_BYTES), k);
                       });
    const float* tile = stage_acc<BN>(d, smem_gen);
    if (warp < 4) {
      const int row = m0 + tid;
      const float* arow = tile + tid * (BN + 4);
      float* crow = p.c + static_cast<size_t>(bz) * p.stride_c + static_cast<size_t>(row) * p.ldc + n0;
      const bool vec_ok = ((p.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.c) & 15) == 0) &&
                          ((p.stride_c & 3) == 0);
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        uint32_t r[32];
        acc_ld32(arow + c * 32, r);
        if (row < p.M) {
          const int nbase = n0 + c * 32;
          if (vec_ok && nbase + 32 <= p.N) {
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              float4 v;
              v.x = __uint_as_float(r[i]) * p.alpha;
              v.y = __uint_as_float(r[i + 1]) * p.alpha;
              v.z = __uint_as_float(r[i + 2]) * p.alpha;
              v.w = __uint_as_float(r[i + 3]) * p.alpha;
              float4* dst = reinterpret_cast<float4*>(crow + c * 32 + i);
              if (p.accumulate) {
                const float4 o = *dst;
                v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
              }
              *dst = v;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              if (nbase + i < p.N) {
                float v = __uint_as_float(r[i]) * p.alpha;
                if (p.accumulate) v += crow[c * 32 + i];
                crow[c * 32 + i] = v;
              }
            }
          }
        }
      }
    }
  }
}

}  // namespace

int gemm_f16_launch(const void* a, const void* b, float* c, int batch, int M, int N, int K, int lda, int ldb,
                    int ldc, long long stride_a, long long stride_b, long long stride_c, float alpha,
                    int accumulate, int bf16, cudaStream_t stream) {
  if (batch <= 0 || M <= 0 || N <= 0 || K <= 0) {
    set_error("gemm_f16: empty problem (batch=%d M=%d N=%d K=%d)", batch, M, N, K);
    return -1;
  }
  if ((lda % 8) || (ldb % 8) || (stride_a % 8) || (stride_b % 8)) {
    set_error("gemm_f16: lda/ldb/strides must be multiples of 8 fp16 elements");
    return -1;
  }
  CUtensorMap tm_a, tm_b;
  int rc;
  const uint64_t sa = batch > 1 ? (uint64_t)stride_a * 2 : (uint64_t)M * lda * 2;
  const uint64_t sb = batch > 1 ? (uint64_t)stride_b * 2 : (uint64_t)N * ldb * 2;
  if ((rc = make_tmap_f16_3d(&tm_a, a, K, M, batch, (uint64_t)lda * 2, sa, BK, BM, 1))) return rc;
  static const int bn = [] {
    const char* e = getenv("COCOS_GEMM_BN");
    return (e && atoi(e) == 128) ? 128 : 256;
  }();
  const int BN = (bn == 256 && N > 128) ? 256 : 128;
  if ((rc = make_tmap_f16_3d(&tm_b, b, K, N, batch, (uint64_t)ldb * 2, sb, BK, BN, 1))) return rc;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.stride_c = stride_c; p.alpha = alpha; p.accumulate = accumulate; p.bf16 = bf16;
  p.c = c;
  const int smem_bytes = 1024 + 196608 + 256;  // 6 x 32 KiB or 4 x 48 KiB
  dim3 grid((M + BM - 1) / BM, (N + BN - 1) / BN, batch);
  if (BN == 256) {
    COCOS_CUDA_CHECK(
        cudaFuncSetAttribute(gemm_f16_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    gemm_f16_kernel<256><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_a, tm_b, p);
  } else {
    COCOS_CUDA_CHECK(
        cudaFuncSetAttribute(gemm_f16_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    gemm_f16_kernel<128><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_a, tm_b, p);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
