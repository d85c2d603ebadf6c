// HBM-bound layout and gradient kernels of the SAGAN non-local block (architecture.py:97-127) on the 16-bit NHWC
// tape, sm_90a.  The block is  y = x + gamma * o(attend(theta(x), maxpool2(phi(x)), maxpool2(g(x))));  its three
// 1x1 input convolutions run as ONE tap convolution with filters [theta | phi | g] and its matmul / softmax / matmul
// on K1 (cocos_corr_warp_fwd, scale 1) and K1's backward (cocos_corr_warp_bwd_ds + three bf16 cocos_gemm_f16).
// What lies between them is here:
//
//   nhwc_to_op      : raw NHWC activation (fp32 / fp16) -> fp16 conv operand [hi | lo]
//   attn_pack_nhwc  : raw [theta | phi | g] conv output -> the K1 operands Q, maxpool2(phi) as K rows, maxpool2(g) as
//                     channel-major V, and the position-major / bf16 channel-major copies the backward contracts with
//   attn_do_rows    : bf16 NHWC gradient of the attention output -> row-scaled fp16 dO rows + bf16 channel-major dO
//   attn_grad_unpack: dQ, dK, dV (channel-major fp32 GEMM outputs) -> bf16 NHWC gradient of the [theta | phi | g]
//                     conv output, dK / dV routed to the first maximum of each 2x2 window (F.max_pool2d's backward)
//
// Every output element is written by exactly one thread, nothing reduces across threads: no atomics, no workspace,
// the same bits on every run.  Transposes go through a 32 x 33 shared-memory tile, so both the NHWC side and the
// channel-major side are read / written along their contiguous dimension.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/cocos_b200.h"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int TILE = 32;

__device__ __forceinline__ float ld1(const void* base, int kind, size_t idx) {
  if (kind == 3) return static_cast<const float*>(base)[idx];
  const uint16_t u = static_cast<const uint16_t*>(base)[idx];
  if (kind == 1) return __half2float(__ushort_as_half(u));
  return __bfloat162float(__ushort_as_bfloat16(u));
}

__device__ __forceinline__ uint16_t f16bits(float v) { return __half_as_ushort(__float2half_rn(v)); }
__device__ __forceinline__ uint16_t bf16bits(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }

long long blocks_of(long long n, int per) { return (n + per - 1) / per; }

// ----------------------------------------------------------------------------------------------- raw -> operand
// y[pix, c] = fp16(x[pix, c]) and, with lo_off, y[pix, lo_off + c] = fp16(x - fp16(x)), c < Cs (4 channels per thread)
__global__ void __launch_bounds__(256)
to_op_kernel(const void* __restrict__ x, int kind, int Cs, uint16_t* __restrict__ y, int y_Cs, int lo_off,
             long long npix) {
  const int n4 = Cs >> 2;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= npix * n4) return;
  const int c = static_cast<int>(idx % n4) * 4;
  const long long pix = idx / n4;
  const size_t src = static_cast<size_t>(pix) * Cs + c;
  float v[4];
  if (kind == 3) {
    const float4 f = *reinterpret_cast<const float4*>(static_cast<const float*>(x) + src);
    v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = ld1(x, kind, src + i);
  }
  uint16_t hi[4], lo[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const __half h = __float2half_rn(v[i]);
    hi[i] = __half_as_ushort(h);
    lo[i] = f16bits(v[i] - __half2float(h));
  }
  uint16_t* row = y + static_cast<size_t>(pix) * y_Cs;
  *reinterpret_cast<uint2*>(row + c) = make_uint2(hi[0] | (static_cast<uint32_t>(hi[1]) << 16),
                                                  hi[2] | (static_cast<uint32_t>(hi[3]) << 16));
  if (lo_off)
    *reinterpret_cast<uint2*>(row + lo_off + c) = make_uint2(lo[0] | (static_cast<uint32_t>(lo[1]) << 16),
                                                             lo[2] | (static_cast<uint32_t>(lo[3]) << 16));
}

// ----------------------------------------------------------------------------------------------- forward pack
struct AttnPack {
  const void* z;
  int z_kind, z_Cs;
  int H, W, Kd, Cv, Kp, split;
  uint16_t* q;     // [B, Nq, Kt]  fp16, Kt = Kp * (split ? 3 : 1): [hi] or [hi, lo, hi]
  uint16_t* k;     // [B, Nk, Kt]  fp16: [hi] or [hi, hi, lo]
  uint16_t* vt;    // [B, Cvp, Nkp] fp16 channel-major
  int Cvp, Nkp;
  uint16_t* v16;   // [B, Nk, Cvk] fp16 position-major, zero beyond Cv (optional)
  int Cvk;
  uint16_t* q_cm;  // [B, Kd, Nqp] bf16 (optional)
  int Nqp;
  uint16_t* k_cm;  // [B, Kd, Nkp] bf16 (optional)
};

__device__ __forceinline__ void store_rows(uint16_t* row, int Kp, int c, float v, int split, bool query) {
  const __half h = __float2half_rn(v);
  const uint16_t hb = __half_as_ushort(h);
  row[c] = hb;
  if (split) {
    const uint16_t lb = f16bits(v - __half2float(h));
    row[Kp + c] = query ? lb : hb;
    row[2 * Kp + c] = query ? hb : lb;
  }
}

// theta: 32 query positions x 32 channels per block (channels [0, Kp), zero beyond Kd)
__global__ void __launch_bounds__(256) attn_q_kernel(const AttnPack p) {
  __shared__ float tile[TILE][TILE + 1];  // [position][channel]
  const int b = blockIdx.z, c0 = blockIdx.y * TILE, n0 = blockIdx.x * TILE;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int Nq = p.H * p.W;
  for (int i = ty; i < TILE; i += 8) {
    const int n = n0 + i, c = c0 + tx;
    tile[i][tx] = (n < Nq && c < p.Kd) ? ld1(p.z, p.z_kind, (static_cast<size_t>(b) * Nq + n) * p.z_Cs + c) : 0.f;
  }
  __syncthreads();
  const int Kt = p.split ? 3 * p.Kp : p.Kp;
  for (int i = ty; i < TILE; i += 8) {
    const int n = n0 + i;
    if (n < Nq) store_rows(p.q + (static_cast<size_t>(b) * Nq + n) * Kt, p.Kp, c0 + tx, tile[i][tx], p.split, true);
  }
  if (p.q_cm != nullptr) {
    for (int i = ty; i < TILE; i += 8) {
      const int c = c0 + i, n = n0 + tx;
      if (c < p.Kd && n < Nq) p.q_cm[(static_cast<size_t>(b) * p.Kd + c) * p.Nqp + n] = bf16bits(tile[tx][i]);
    }
  }
}

// maxpool2(phi) and maxpool2(g): 32 pooled positions x 32 channels per block; channel tiles [0, Kp) are phi, the
// tiles from Kp on are g (channels [0, Cvk))
__global__ void __launch_bounds__(256) attn_kv_kernel(const AttnPack p) {
  __shared__ float tile[TILE][TILE + 1];  // [pooled position][channel]
  const int b = blockIdx.z, n0 = blockIdx.x * TILE;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const bool is_k = static_cast<int>(blockIdx.y) * TILE < p.Kp;
  const int cbase = is_k ? blockIdx.y * TILE : blockIdx.y * TILE - p.Kp;
  const int lim = is_k ? p.Kd : p.Cv;
  const int src0 = is_k ? p.Kd : 2 * p.Kd;
  const int Wo = p.W >> 1, Nk = (p.H >> 1) * Wo, Nq = p.H * p.W;
  for (int i = ty; i < TILE; i += 8) {
    const int n = n0 + i, cl = cbase + tx;
    float m = 0.f;
    if (n < Nk && cl < lim) {
      const int ho = n / Wo, wo = n - ho * Wo;
      const size_t px = (static_cast<size_t>(b) * Nq + static_cast<size_t>(2 * ho) * p.W + 2 * wo) * p.z_Cs + src0 + cl;
      const size_t row = static_cast<size_t>(p.W) * p.z_Cs;
      m = ld1(p.z, p.z_kind, px);
      const float a1 = ld1(p.z, p.z_kind, px + p.z_Cs), a2 = ld1(p.z, p.z_kind, px + row),
                  a3 = ld1(p.z, p.z_kind, px + row + p.z_Cs);
      if (a1 > m) m = a1;
      if (a2 > m) m = a2;
      if (a3 > m) m = a3;
    }
    tile[i][tx] = m;
  }
  __syncthreads();
  if (is_k) {
    const int Kt = p.split ? 3 * p.Kp : p.Kp;
    for (int i = ty; i < TILE; i += 8) {
      const int n = n0 + i;
      if (n < Nk) store_rows(p.k + (static_cast<size_t>(b) * Nk + n) * Kt, p.Kp, cbase + tx, tile[i][tx], p.split, false);
    }
    if (p.k_cm != nullptr) {
      for (int i = ty; i < TILE; i += 8) {
        const int c = cbase + i, n = n0 + tx;
        if (c < p.Kd && n < Nk) p.k_cm[(static_cast<size_t>(b) * p.Kd + c) * p.Nkp + n] = bf16bits(tile[tx][i]);
      }
    }
    return;
  }
  if (p.v16 != nullptr) {  // [B][Nk][Cvk]
    uint16_t* dst = p.v16 + static_cast<size_t>(b) * Nk * p.Cvk + cbase + tx;
    for (int i = ty; i < TILE; i += 8) {
      const int n = n0 + i;
      if (n < Nk) dst[static_cast<size_t>(n) * p.Cvk] = f16bits(tile[i][tx]);
    }
  }
  for (int i = ty; i < TILE; i += 8) {  // V channel-major, zero in the padding columns [Nk, Nkp) and rows [Cv, Cvp)
    const int c = cbase + i, n = n0 + tx;
    if (c < p.Cvp && n < p.Nkp) p.vt[(static_cast<size_t>(b) * p.Cvp + c) * p.Nkp + n] = f16bits(n < Nk ? tile[tx][i] : 0.f);
  }
}

// ----------------------------------------------------------------------------------------------- dO rows
// dy bf16 [B, N, dy_Cs] (Cv channels) -> do16 fp16 [B, N, Cvk] = r * dy (zero beyond Cv), r = min(1 / max_c |dy|,
// 2^126) (1 for an all-zero row), and do_cm bf16 [B, Cv, Nqp] = dy channel-major.  32 positions per block, one warp per
// row for the maxima.
__global__ void __launch_bounds__(256)
attn_do_rows_kernel(const uint16_t* __restrict__ dy, int dy_Cs, int N, int Cv, uint16_t* __restrict__ do16, int Cvk,
                    float* __restrict__ rscale, uint16_t* __restrict__ do_cm, int Nqp) {
  __shared__ float tile[TILE][TILE + 1];
  __shared__ float rs[TILE];
  const int b = blockIdx.y, n0 = blockIdx.x * TILE;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const uint16_t* base = dy + static_cast<size_t>(b) * N * dy_Cs;
  for (int i = ty; i < TILE; i += 8) {
    const int n = n0 + i;
    float m = 0.f;
    if (n < N)
      for (int c = tx; c < Cv; c += 32)
        m = fmaxf(m, fabsf(__bfloat162float(__ushort_as_bfloat16(base[static_cast<size_t>(n) * dy_Cs + c]))));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (tx == 0) {
      // capped at 2^126: 1/m overflows fp32 for a subnormal maximum m <= 2^-128 (rowscale_kernel in pack.cu)
      const float r = (m > 0.f && isfinite(m)) ? fminf(1.0f / m, 0x1p126f) : 1.0f;
      rs[i] = r;
      if (n < N) rscale[static_cast<size_t>(b) * N + n] = r;
    }
  }
  for (int c0 = 0; c0 < Cvk; c0 += TILE) {
    __syncthreads();
    for (int i = ty; i < TILE; i += 8) {
      const int n = n0 + i, c = c0 + tx;
      tile[i][tx] = (n < N && c < Cv) ? __bfloat162float(__ushort_as_bfloat16(base[static_cast<size_t>(n) * dy_Cs + c]))
                                      : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < TILE; i += 8) {
      const int n = n0 + i;
      if (n < N) do16[(static_cast<size_t>(b) * N + n) * Cvk + c0 + tx] = f16bits(tile[i][tx] * rs[i]);
    }
    for (int i = ty; i < TILE; i += 8) {
      const int c = c0 + i, n = n0 + tx;
      if (c < Cv && n < N) do_cm[(static_cast<size_t>(b) * Cv + c) * Nqp + n] = bf16bits(tile[tx][i]);
    }
  }
}

// ----------------------------------------------------------------------------------------------- gradient unpack
struct AttnUnpack {
  const float* dq;  // [B, Kd, Nq]
  const float* dk;  // [B, Kd, Nk]
  const float* dv;  // [B, Cv, Nk]
  const void* z;
  int z_kind, z_Cs;
  int H, W, Kd, Cv;
  uint16_t* dz;     // [B, H, W, dz_Cs] bf16
  int dz_Cs;
};

// 32 pooled positions (= their 128 window pixels) x 32 channels of dz per block
__global__ void __launch_bounds__(256) attn_grad_unpack_kernel(const AttnUnpack p) {
  __shared__ float g[TILE][4][TILE + 1];  // [channel][window slot][pooled position]
  const int b = blockIdx.z, c0 = blockIdx.y * TILE, n0 = blockIdx.x * TILE;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int Wo = p.W >> 1, Nk = (p.H >> 1) * Wo, Nq = p.H * p.W;
  {
    const int n = n0 + tx;
    if (n < Nk) {
      const int ho = n / Wo, wo = n - ho * Wo;
      const int pix0 = 2 * ho * p.W + 2 * wo;
      for (int i = ty; i < TILE; i += 8) {
        const int c = c0 + i;
        if (c < p.Kd) {
          const float* src = p.dq + (static_cast<size_t>(b) * p.Kd + c) * Nq + pix0;
          g[i][0][tx] = src[0];
          g[i][1][tx] = src[1];
          g[i][2][tx] = src[p.W];
          g[i][3][tx] = src[p.W + 1];
        } else if (c < 2 * p.Kd) {
          g[i][0][tx] = p.dk[(static_cast<size_t>(b) * p.Kd + c - p.Kd) * Nk + n];
        } else if (c < 2 * p.Kd + p.Cv) {
          g[i][0][tx] = p.dv[(static_cast<size_t>(b) * p.Cv + c - 2 * p.Kd) * Nk + n];
        }
      }
    }
  }
  __syncthreads();
  const int c = c0 + tx;
  if (c >= p.dz_Cs) return;
  for (int i = ty; i < TILE; i += 8) {
    const int n = n0 + i;
    if (n >= Nk) break;
    const int ho = n / Wo, wo = n - ho * Wo;
    const size_t pix[4] = {static_cast<size_t>(b) * Nq + static_cast<size_t>(2 * ho) * p.W + 2 * wo,
                           static_cast<size_t>(b) * Nq + static_cast<size_t>(2 * ho) * p.W + 2 * wo + 1,
                           static_cast<size_t>(b) * Nq + static_cast<size_t>(2 * ho + 1) * p.W + 2 * wo,
                           static_cast<size_t>(b) * Nq + static_cast<size_t>(2 * ho + 1) * p.W + 2 * wo + 1};
    float o[4] = {0.f, 0.f, 0.f, 0.f};
    if (c < p.Kd) {
#pragma unroll
      for (int s = 0; s < 4; ++s) o[s] = g[tx][s][i];
    } else if (c < 2 * p.Kd + p.Cv) {
      // the window's first maximum in scan order, as the pooling forward saw it (F.max_pool2d's index)
      float best = ld1(p.z, p.z_kind, pix[0] * p.z_Cs + c);
      int arg = 0;
#pragma unroll
      for (int s = 1; s < 4; ++s) {
        const float t = ld1(p.z, p.z_kind, pix[s] * p.z_Cs + c);
        if (t > best) { best = t; arg = s; }
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) o[s] = (s == arg) ? g[tx][0][i] : 0.f;
    }
#pragma unroll
    for (int s = 0; s < 4; ++s) p.dz[pix[s] * p.dz_Cs + c] = bf16bits(o[s]);
  }
}

bool kind_ok(int k) { return k == 1 || k == 3; }

}  // namespace

}  // namespace cocos

using namespace cocos;

extern "C" {

int cocos_nhwc_to_op(const void* x, int x_kind, int Cs, void* y, int y_Cs, int lo_off, long long npix, void* stream) {
  if (!x || !y) {
    set_error("cocos_nhwc_to_op: null pointer argument");
    return -1;
  }
  if (npix <= 0 || Cs <= 0 || (Cs % 8) || !kind_ok(x_kind) || (y_Cs % 8) || lo_off < 0 || (lo_off % 8) ||
      (lo_off ? (lo_off < Cs || lo_off + Cs > y_Cs) : y_Cs < Cs)) {
    set_error("cocos_nhwc_to_op: bad arguments (kind=%d Cs=%d y_Cs=%d lo_off=%d npix=%lld)", x_kind, Cs, y_Cs, lo_off,
              npix);
    return -1;
  }
  to_op_kernel<<<static_cast<unsigned>(blocks_of(npix * (Cs / 4), 256)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, x_kind, Cs, static_cast<uint16_t*>(y), y_Cs, lo_off, npix);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int cocos_attn_pack_nhwc(const void* z, int z_kind, int z_Cs, int B, int H, int W, int Kd, int Cv, int split, void* q,
                         void* k, void* vt, int Cvp, int Nkp, void* v16, int Cvk, void* q_cm, int Nqp, void* k_cm,
                         void* stream) {
  if (!z || !q || !k || !vt) {
    set_error("cocos_attn_pack_nhwc: null pointer argument");
    return -1;
  }
  const int Kp = (Kd + 63) / 64 * 64;
  const long long Nq = static_cast<long long>(H) * W, Nk = Nq / 4;
  if (B <= 0 || H <= 0 || W <= 0 || (H % 2) || (W % 2) || Kd <= 0 || Cv <= 0 || !kind_ok(z_kind) ||
      z_Cs < 2 * Kd + Cv || Cvp < Cv || (Cvp % 16) || Nkp < Nk || (Nkp % 8) || Nqp < Nq || (Nqp % 8) ||
      (v16 && (Cvk < Cvp || (Cvk % 64))) || (split != 0 && split != 1) || (!q_cm) != (!k_cm)) {
    set_error("cocos_attn_pack_nhwc: bad arguments (B=%d H=%d W=%d Kd=%d Cv=%d z_Cs=%d Cvp=%d Nkp=%d Cvk=%d Nqp=%d)", B,
              H, W, Kd, Cv, z_Cs, Cvp, Nkp, Cvk, Nqp);
    return -1;
  }
  AttnPack p;
  p.z = z; p.z_kind = z_kind; p.z_Cs = z_Cs;
  p.H = H; p.W = W; p.Kd = Kd; p.Cv = Cv; p.Kp = Kp; p.split = split;
  p.q = static_cast<uint16_t*>(q); p.k = static_cast<uint16_t*>(k); p.vt = static_cast<uint16_t*>(vt);
  p.Cvp = Cvp; p.Nkp = Nkp;
  p.v16 = static_cast<uint16_t*>(v16); p.Cvk = v16 ? Cvk : 0;
  p.q_cm = static_cast<uint16_t*>(q_cm); p.Nqp = Nqp; p.k_cm = static_cast<uint16_t*>(k_cm);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dim3 blk(TILE, 8);
  attn_q_kernel<<<dim3(static_cast<unsigned>(blocks_of(Nq, TILE)), Kp / TILE, B), blk, 0, s>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  // V channel tiles up to Cvk when the position-major copy is written (Cvk >= Cvp covers both copies), else up to Cvp
  const long long kv_tiles = Kp / TILE + blocks_of(v16 ? Cvk : Cvp, TILE);
  attn_kv_kernel<<<dim3(static_cast<unsigned>(blocks_of(Nkp, TILE)), static_cast<unsigned>(kv_tiles), B), blk, 0, s>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int cocos_attn_do_rows(const void* dy, int dy_Cs, int B, int N, int Cv, void* do16, int Cvk, float* rscale, void* do_cm,
                       int Nqp, void* stream) {
  if (!dy || !do16 || !rscale || !do_cm) {
    set_error("cocos_attn_do_rows: null pointer argument");
    return -1;
  }
  if (B <= 0 || N <= 0 || Cv <= 0 || dy_Cs < Cv || Cvk < Cv || (Cvk % 64) || Nqp < N || (Nqp % 8)) {
    set_error("cocos_attn_do_rows: bad arguments (B=%d N=%d Cv=%d dy_Cs=%d Cvk=%d Nqp=%d)", B, N, Cv, dy_Cs, Cvk, Nqp);
    return -1;
  }
  attn_do_rows_kernel<<<dim3(static_cast<unsigned>(blocks_of(N, TILE)), B), dim3(TILE, 8), 0,
                        static_cast<cudaStream_t>(stream)>>>(static_cast<const uint16_t*>(dy), dy_Cs, N, Cv,
                                                             static_cast<uint16_t*>(do16), Cvk, rscale,
                                                             static_cast<uint16_t*>(do_cm), Nqp);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int cocos_attn_grad_unpack(const float* dq, const float* dk, const float* dv, const void* z, int z_kind, int z_Cs, int B,
                           int H, int W, int Kd, int Cv, void* dz, int dz_Cs, void* stream) {
  if (!dq || !dk || !dv || !z || !dz) {
    set_error("cocos_attn_grad_unpack: null pointer argument");
    return -1;
  }
  if (B <= 0 || H <= 0 || W <= 0 || (H % 2) || (W % 2) || Kd <= 0 || Cv <= 0 || !kind_ok(z_kind) ||
      z_Cs < 2 * Kd + Cv || dz_Cs < 2 * Kd + Cv || (dz_Cs % 8)) {
    set_error("cocos_attn_grad_unpack: bad arguments (B=%d H=%d W=%d Kd=%d Cv=%d z_Cs=%d dz_Cs=%d)", B, H, W, Kd, Cv,
              z_Cs, dz_Cs);
    return -1;
  }
  AttnUnpack p;
  p.dq = dq; p.dk = dk; p.dv = dv;
  p.z = z; p.z_kind = z_kind; p.z_Cs = z_Cs;
  p.H = H; p.W = W; p.Kd = Kd; p.Cv = Cv;
  p.dz = static_cast<uint16_t*>(dz); p.dz_Cs = dz_Cs;
  const long long Nk = static_cast<long long>(H / 2) * (W / 2);
  attn_grad_unpack_kernel<<<dim3(static_cast<unsigned>(blocks_of(Nk, TILE)), static_cast<unsigned>(blocks_of(dz_Cs, TILE)),
                                 B), dim3(TILE, 8), 0, static_cast<cudaStream_t>(stream)>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // extern "C"
