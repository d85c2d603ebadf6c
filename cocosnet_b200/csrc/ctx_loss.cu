// Row kernels of the contextual loss (reference models/networks/ContextualLoss.py:93-137) on the correlation matrix
// S = Xhat^T Yhat [B, N, N] (fp32, produced by the wgmma GEMM cocos_gemm_f16; N <= 1024 positions of a VGG map):
//   d = 1 - S,  m_i = min_j d_ij,  w_ij = exp((1 - d_ij / (m_i + 1e-3)) / h),  A_ij = w_ij / sum_j w_ij,
//   CX_i = max_j A_ij = 1 / sum_j q_ij,  q_ij = exp(-a_i (d_ij - m_i)),  a_i = 1 / (h (m_i + 1e-3))
// (w is decreasing in d, so the row maximum sits at the row minimum of d).  The reference materialises d, d_norm, w,
// A and the max as five [B, N, N] fp32 tensors per layer plus their autograd copies; here a warp owns a row, keeps it
// in registers, and writes per-row scalars only.  Backward (autograd's formula, min routed to its arg-min j*):
//   dCX_i/dd_ij  = CX_i^2 a_i q_ij                                         (j != j*)
//   dCX_i/dd_ij* = -CX_i^2 a_i sum_{j != j*} q_ij (1 + (d_ij - m_i) / (m_i + 1e-3))
// and dS = -dd.  Launch: one warp per row, 8 rows per block.
#include <cuda_bf16.h>

#include "corr_kernels.h"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int MAXPER = 32;  // N <= 1024: up to 32 values of the row per lane

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct RowStats {
  float m, a, sumq, sumqd;  // min d, 1/(h(m+eps)), sum_j q, sum_{j != j*} q (d - m)
  int arg;
};

__device__ __forceinline__ RowStats row_stats(const float* __restrict__ srow, int N, float h, float eps, float* d,
                                              int lane) {
  float best = 3.4e38f;
  int arg = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < MAXPER; ++k) {
    const int j = lane + 32 * k;
    d[k] = j < N ? 1.0f - srow[j] : 3.4e38f;
    if (d[k] < best) { best = d[k]; arg = j; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // min with the smallest index on ties (torch.min's first occurrence)
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob < best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  RowStats r;
  r.m = best;
  r.arg = arg;
  r.a = 1.0f / (h * (best + eps));
  float sq = 0.f, sqd = 0.f;
#pragma unroll
  for (int k = 0; k < MAXPER; ++k) {
    const int j = lane + 32 * k;
    if (j < N) {
      const float q = __expf(-r.a * (d[k] - best));
      sq += q;
      if (j != arg) sqd = fmaf(q, d[k] - best, sqd);
    }
  }
  r.sumq = wsum(sq);
  r.sumqd = wsum(sqd);
  return r;
}

// cx[b, i] = 1 / sum_j q_ij
__global__ void __launch_bounds__(256)
ctx_rows_fwd_kernel(const float* __restrict__ S, float* __restrict__ cx, int rows, int N, float h, float eps) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  float d[MAXPER];
  const RowStats r = row_stats(S + row * N, N, h, eps, d, lane);
  if (lane == 0) cx[row] = 1.0f / r.sumq;
}

// dS[b, i, j] (bf16, row pitch ldd) = -g[b, i] * dCX_i / dd_ij
__global__ void __launch_bounds__(256)
ctx_rows_bwd_kernel(const float* __restrict__ S, const float* __restrict__ g, __nv_bfloat16* __restrict__ dS, int rows,
                    int N, int ldd, float h, float eps) {
  const int lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  float d[MAXPER];
  const RowStats r = row_stats(S + row * N, N, h, eps, d, lane);
  const float cx = 1.0f / r.sumq;
  const float c = g[row] * cx * cx * r.a;
  // sum_{j != j*} q (1 + (d - m)/(m + eps)) = (sumq - 1) + sumqd / (m + eps)     (q_{j*} = 1)
  const float at_min = c * ((r.sumq - 1.0f) + r.sumqd / (r.m + eps));
  __nv_bfloat16* out = dS + row * ldd;
#pragma unroll
  for (int k = 0; k < MAXPER; ++k) {
    const int j = lane + 32 * k;
    if (j < N) {
      const float dd = (j == r.arg) ? -at_min : c * __expf(-r.a * (d[k] - r.m));
      out[j] = __float2bfloat16_rn(-dd);
    }
  }
}

}  // namespace

int ctx_rows_fwd_launch(const float* S, float* cx, int B, int N, float h, float eps, cudaStream_t stream) {
  if (B <= 0 || N <= 0 || N > 32 * MAXPER || h <= 0.f) {
    set_error("ctx_rows_fwd: bad arguments (B=%d N=%d)", B, N);
    return -1;
  }
  const int rows = B * N;
  ctx_rows_fwd_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(S, cx, rows, N, h, eps);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int ctx_rows_bwd_launch(const float* S, const float* g, void* dS, int B, int N, int ldd, float h, float eps,
                        cudaStream_t stream) {
  if (B <= 0 || N <= 0 || N > 32 * MAXPER || ldd < N || h <= 0.f) {
    set_error("ctx_rows_bwd: bad arguments (B=%d N=%d ldd=%d)", B, N, ldd);
    return -1;
  }
  const int rows = B * N;
  ctx_rows_bwd_kernel<<<(rows + 7) / 8, 256, 0, stream>>>(S, g, static_cast<__nv_bfloat16*>(dS), rows, N, ldd, h, eps);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
