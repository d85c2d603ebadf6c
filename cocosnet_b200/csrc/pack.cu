// HBM-bound layout/precision prologue kernels for K1.
//   pack_rows_f16 : fp32 [B, C, N] (channel-major, the reference's
//                   theta/phi layout, correspondence.py:274-289) ->
//                   fp16 [B, N, Kt] (position-major, K contiguous) that TMA
//                   stages as the K-major MMA operand; optional 2-term fp16
//                   split laid out along K so ONE GEMM accumulates
//                   hi*hi + lo*hi + hi*lo.
//   pack_v_f16    : fp32 [B, Cv, Nk] -> fp16 [B, Cvp, Nkp], zero padded.
#include "corr_kernels.h"
#include "tmap.h"

#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace cocos {

namespace {

constexpr int TC = 64;  // channels per tile
constexpr int TN = 32;  // positions per tile

// split_mode 0: [h]; 1: [h, l, h] (query side); 2: [h, h, l] (key side)
__global__ void __launch_bounds__(256)
pack_rows_kernel(const float* __restrict__ src, __half* __restrict__ dst, int C, int N, int Kp, int split_mode,
                 const float* __restrict__ rowscale, int bf16) {
  __shared__ float tile[TC][TN + 1];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * TC;
  const int n0 = blockIdx.x * TN;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const float* s = src + static_cast<size_t>(b) * C * N;
#pragma unroll
  for (int i = 0; i < TC; i += 8) {
    const int c = c0 + ty + i, n = n0 + tx;
    tile[ty + i][tx] = (c < C && n < N) ? s[static_cast<size_t>(c) * N + n] : 0.f;
  }
  __syncthreads();
  const int nseg = split_mode ? 3 : 1;
  const int Kt = Kp * nseg;
  __half* d = dst + static_cast<size_t>(b) * N * Kt;
  // each thread writes 2 adjacent channels (half2) for 4 positions
  const int cx = (threadIdx.x & 31) * 2;  // 0..62
  const int nrow = threadIdx.x >> 5;      // 0..7
#pragma unroll
  for (int i = 0; i < TN; i += 8) {
    const int n = n0 + nrow + i;
    const int c = c0 + cx;
    if (n < N && c < Kp) {
      const float rs = rowscale ? rowscale[static_cast<size_t>(b) * N + n] : 1.0f;
      const float x0 = tile[cx][nrow + i] * rs, x1 = tile[cx + 1][nrow + i] * rs;
      const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
      const __half2 hi = __halves2half2(h0, h1);
      __half* row = d + static_cast<size_t>(n) * Kt + c;
      if (bf16) {  // same 2-byte slots, bfloat16 rounding (gradient operands: fp32 range)
        const __nv_bfloat162 bb = __floats2bfloat162_rn(x0, x1);
        *reinterpret_cast<uint32_t*>(row) = *reinterpret_cast<const uint32_t*>(&bb);
      } else if (!split_mode) {
        *reinterpret_cast<__half2*>(row) = hi;
      } else {
        const __half2 lo = __halves2half2(__float2half_rn(x0 - __half2float(h0)),
                                          __float2half_rn(x1 - __half2float(h1)));
        *reinterpret_cast<__half2*>(row) = hi;
        *reinterpret_cast<__half2*>(row + Kp) = (split_mode == 1) ? lo : hi;
        *reinterpret_cast<__half2*>(row + 2 * Kp) = (split_mode == 1) ? hi : lo;
      }
    }
  }
}

__global__ void __launch_bounds__(256)
pack_v_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, int Cv, int Nk, int Cvp, int Nkp, int bf16) {
  const int b = blockIdx.z, c = blockIdx.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nkp) return;
  float v = 0.f;
  if (c < Cv && n < Nk) v = src[(static_cast<size_t>(b) * Cv + c) * Nk + n];
  uint16_t bits;
  if (bf16) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    bits = *reinterpret_cast<const uint16_t*>(&h);
  } else {
    const __half h = __float2half_rn(v);
    bits = *reinterpret_cast<const uint16_t*>(&h);
  }
  dst[(static_cast<size_t>(b) * Cvp + c) * Nkp + n] = bits;
}

// r[b,n] = min(1 / max_c |src[b,c,n]|, 2^126)  (1 where the column is all zero)
__global__ void __launch_bounds__(256)
rowscale_kernel(const float* __restrict__ src, float* __restrict__ r, int C, int N) {
  const int b = blockIdx.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float* s = src + static_cast<size_t>(b) * C * N + n;
  float m = 0.f;
  for (int c = 0; c < C; ++c) m = fmaxf(m, fabsf(s[static_cast<size_t>(c) * N]));
  // 1/m overflows fp32 for a subnormal m <= 2^-128: cap r at 2^126 so that r * x stays <= 1 and the divide-back
  // (scale / r in stage A) stays finite; every normal m keeps r = 1/m exactly
  r[static_cast<size_t>(b) * N + n] = (m > 0.f && isfinite(m)) ? fminf(1.0f / m, 0x1p126f) : 1.0f;
}

}  // namespace

int pack_rows_f16_launch(const float* src, void* dst, int B, int C, int N, int Kp, int split_mode,
                         float* rowscale_out, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || N <= 0 || Kp < C || (Kp % 2) != 0 || split_mode < 0 || (split_mode > 2 && split_mode != 4)) {
    set_error("pack_rows_f16: bad arguments (B=%d C=%d N=%d Kp=%d split=%d)", B, C, N, Kp, split_mode);
    return -1;
  }
  if (rowscale_out != nullptr) {
    rowscale_kernel<<<dim3((N + 255) / 256, B), 256, 0, stream>>>(src, rowscale_out, C, N);
    COCOS_CUDA_CHECK(cudaGetLastError());
  }
  dim3 grid((N + TN - 1) / TN, (Kp + TC - 1) / TC, B);
  pack_rows_kernel<<<grid, 256, 0, stream>>>(src, static_cast<__half*>(dst), C, N, Kp, split_mode & 3, rowscale_out,
                                             (split_mode & 4) != 0);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int pack_v_f16_launch(const float* src, void* dst, int B, int Cv, int Nk, int Cvp, int Nkp, int bf16,
                      cudaStream_t stream) {
  if (B <= 0 || Cv <= 0 || Nk <= 0 || Cvp < Cv || Nkp < Nk) {
    set_error("pack_v_f16: bad arguments (B=%d Cv=%d Nk=%d Cvp=%d Nkp=%d)", B, Cv, Nk, Cvp, Nkp);
    return -1;
  }
  dim3 grid((Nkp + 255) / 256, Cvp, B);
  pack_v_kernel<<<grid, 256, 0, stream>>>(src, static_cast<uint16_t*>(dst), Cv, Nk, Cvp, Nkp, bf16);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
