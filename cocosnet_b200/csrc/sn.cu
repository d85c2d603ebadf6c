// Spectral normalisation of ALL convolutions of a network in three launches (HBM bound: two passes over the weights).
//
// torch.nn.utils.spectral_norm (reference normalization.py:30-31 wraps every generator / adaptor / discriminator conv)
// runs, per layer and per forward, one power iteration on persistent vectors u [rows], v [cols] of the weight matrix
// W [rows, cols] = weight_orig.view(Cout, -1):
//     v <- normalize(W^T u),  u <- normalize(W v),  sigma = u^T W v,  weight = weight_orig / sigma
// -- about ten small launches per layer, ~100 layer invocations per training iteration.  Here a device-resident table
// lists the layers of one network forward and each phase is ONE launch over all of them:
//   phase A: t = W^T u (column sums, coalesced), |t|^2 partial per block            -> v holds t
//   phase B: s = W t / max(|t|, eps) (one warp per row), |s|^2 partial per block    -> u holds s
//   phase C: v = t / max(|t|, eps), u = s / max(|s|, eps), inv_sigma = 1 / (u^T W v) = max(|s|, eps) / |s|^2
// (u^T W v = u^T s = |s|^2 / max(|s|, eps)).  The division weight_orig / sigma never happens: the convolution kernels
// take inv_sigma as an epilogue scale.  Evaluation mode (no power iteration): phase B' computes W v with the stored v
// and phase C' only the dot product with the stored u.  The per-block partials go to a workspace and are added per layer
// in block order (no floating-point atomics): the same weights give the same sigma on every call.
#include "corr_kernels.h"
#include "tmap.h"

namespace cocos {

namespace {

struct SnEntry {          // one layer; lives in device memory (int64 x 8)
  float* W; float* u; float* v;
  long long rows, cols, block_a, block_b, snap;  // snap: offset of this layer's [u | v] copy in the snapshot buffer
};

__device__ __forceinline__ float warp_sum_sn(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int find_entry(const SnEntry* __restrict__ tab, int n, long long block, bool phase_b) {
  int i = 0;
  while (i + 1 < n && (phase_b ? tab[i + 1].block_b : tab[i + 1].block_a) <= block) ++i;
  return i;
}

// phase A: block = 128 columns (32 threads x 4) x 8 row lanes
__global__ void __launch_bounds__(256)
sn_cols_kernel(const SnEntry* __restrict__ tab, int n, float* __restrict__ part_a) {
  __shared__ float red[8][32][4];
  const int e = find_entry(tab, n, blockIdx.x, false);
  const SnEntry L = tab[e];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const long long c = (blockIdx.x - L.block_a) * 128 + tx * 4;
  float a[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < L.cols) {
    const bool vec = (L.cols & 3) == 0;
    for (long long r = ty; r < L.rows; r += 8) {
      const float ur = L.u[r];
      const float* w = L.W + r * L.cols + c;
      if (vec) {
        const float4 t = *reinterpret_cast<const float4*>(w);
        a[0] = fmaf(t.x, ur, a[0]); a[1] = fmaf(t.y, ur, a[1]); a[2] = fmaf(t.z, ur, a[2]); a[3] = fmaf(t.w, ur, a[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (c + j < L.cols) a[j] = fmaf(w[j], ur, a[j]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[ty][tx][j] = a[j];
  __syncthreads();
  if (ty == 0) {
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += red[k][tx][j];
      if (c + j < L.cols) {
        L.v[c + j] = t;
        sq = fmaf(t, t, sq);
      }
    }
    sq = warp_sum_sn(sq);
    if (tx == 0) part_a[blockIdx.x] = sq;
  }
}

// |t|^2 of layer L: its phase-A partials in block order
__device__ __forceinline__ float sum_t2(const SnEntry& L, const float* __restrict__ part_a) {
  float t2 = 0.f;
  for (long long k = 0; k < (L.cols + 127) / 128; ++k) t2 += part_a[L.block_a + k];
  return t2;
}

// phase B: one warp per row; scale_v: multiply v by 1 / max(|t|, eps) on the fly (training) or use it as stored
__global__ void __launch_bounds__(256)
sn_rows_kernel(const SnEntry* __restrict__ tab, int n, const float* __restrict__ part_a, float* __restrict__ part_b,
               float eps, int scale_v) {
  __shared__ float red[8];
  const int e = find_entry(tab, n, blockIdx.x, true);
  const SnEntry L = tab[e];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long r = (blockIdx.x - L.block_b) * 8 + warp;
  float acc = 0.f;
  if (r < L.rows) {
    const float* w = L.W + r * L.cols;
    if ((L.cols & 3) == 0) {
      for (long long c = lane * 4; c < L.cols; c += 128) {
        const float4 t = *reinterpret_cast<const float4*>(w + c);
        const float4 vv = *reinterpret_cast<const float4*>(L.v + c);
        acc += (t.x * vv.x + t.y * vv.y) + (t.z * vv.z + t.w * vv.w);
      }
    } else {
      for (long long c = lane; c < L.cols; c += 32) acc = fmaf(w[c], L.v[c], acc);
    }
  }
  acc = warp_sum_sn(acc);
  float contrib = 0.f;
  if (r < L.rows && lane == 0) {
    if (scale_v) {
      const float s = acc / fmaxf(sqrtf(sum_t2(L, part_a)), eps);
      L.u[r] = s;  // unnormalised W v
      contrib = s * s;
    } else {
      contrib = acc * L.u[r];  // u^T (W v) with the stored u, v
    }
  }
  if (lane == 0) red[warp] = contrib;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k];
    part_b[blockIdx.x] = t;
  }
}

// phase C: normalise u, v in place and emit 1 / sigma; one block per layer
// `snapshot` (may be NULL) receives a copy [u | v] of the vectors sigma was computed with: the backward of THIS forward
// needs them (d sigma / dW = u v^T) after later forwards of the same layer have advanced the persistent ones.
__global__ void __launch_bounds__(256)
sn_finish_kernel(const SnEntry* __restrict__ tab, const float* __restrict__ part_a, const float* __restrict__ part_b,
                 float* __restrict__ scratch, float eps, int training, float* __restrict__ inv_sigma,
                 float* __restrict__ snapshot) {
  const int e = blockIdx.x;
  const SnEntry L = tab[e];
  float sb = 0.f;  // |s|^2 (training) or u^T W v (evaluation): the layer's phase-B partials in block order
  for (long long k = 0; k < (L.rows + 7) / 8; ++k) sb += part_b[L.block_b + k];
  const float t2 = training ? sum_t2(L, part_a) : 0.f;
  if (threadIdx.x == 0) {
    scratch[2 * e] = t2;
    scratch[2 * e + 1] = sb;
  }
  float tn = 1.f, sn = 1.f;
  if (training) {
    tn = fmaxf(sqrtf(t2), eps);
    const float sn2 = sb;
    sn = fmaxf(sqrtf(sn2), eps);
    if (threadIdx.x == 0) inv_sigma[e] = sn / sn2;
  } else if (threadIdx.x == 0) {
    inv_sigma[e] = 1.0f / sb;
  }
  float* su = snapshot ? snapshot + L.snap : nullptr;
  for (long long r = threadIdx.x; r < L.rows; r += 256) {
    const float t = L.u[r] / sn;
    if (training) L.u[r] = t;
    if (su) su[r] = t;
  }
  for (long long c = threadIdx.x; c < L.cols; c += 256) {
    const float t = L.v[c] / tn;
    if (training) L.v[c] = t;
    if (su) su[L.rows + c] = t;
  }
}

}  // namespace

int sn_power_iter_launch(const void* table, int n, int blocks_a, int blocks_b, float* scratch, float* inv_sigma,
                         float* snapshot, float eps, int training, cudaStream_t stream) {
  if (!table || !scratch || !inv_sigma || n <= 0 || blocks_a <= 0 || blocks_b <= 0) {
    set_error("sn_power_iter: bad arguments (n=%d blocks_a=%d blocks_b=%d)", n, blocks_a, blocks_b);
    return -1;
  }
  const SnEntry* tab = static_cast<const SnEntry*>(table);
  float* part_a = scratch + 2 * n;  // per-block partials of phase A, then of phase B
  float* part_b = part_a + blocks_a;
  if (training) sn_cols_kernel<<<blocks_a, 256, 0, stream>>>(tab, n, part_a);
  sn_rows_kernel<<<blocks_b, 256, 0, stream>>>(tab, n, part_a, part_b, eps, training);
  sn_finish_kernel<<<n, 256, 0, stream>>>(tab, part_a, part_b, scratch, eps, training, inv_sigma, snapshot);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
