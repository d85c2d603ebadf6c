// HBM-bound elementwise / normalisation kernels of the 16-bit NHWC pipeline (everything between two tap
// convolutions), sm_90a.  Tensor "kinds": 1 = fp16, 2 = bf16, 3 = fp32; activations NHWC [B, H, W, Cs] with channel
// stride Cs >= C; gradients bf16.  `op` tensors (the A operand of the next convolution) are fp16, optionally carry
// a reflection halo of p pixels ([B, H+2p, W+2p, Cs], p < H, W: F.pad(mode="reflect"); p = dilation of the SPADE block
// that reads it, 1, 2 or 4) and optionally a second fp16 term lo = x - fp16(x) at channel offset lo_off (2-term split
// operands of the correspondence path).  Halo gradients are folded back by the exact adjoint of the padding.
//
//   spade_mod_nhwc   : PONO + SPADE modulation + LeakyReLU + ReflectionPad2d (normalization.py:63-68,149;
//                      architecture.py:73-74,94-95) raw -> op, forward / backward
//   in_stats_nhwc    : per-(image, channel) sum / sum of squares (InstanceNorm2d statistics)
//   inst_act_nhwc    : InstanceNorm2d(affine=False) [+ residual] + LeakyReLU / PReLU [+ reflection halo]
//                      (generator.py:104-113, discriminator.py:92-115, correspondence.py:13-36), forward / backward
//   nhwc_pack        : fp32 NCHW -> op (nearest down-sampling by an integer factor, halo, split)
//   nhwc_unpack      : NHWC (halo folded back) -> fp32 NCHW, overwrite or accumulate, strided scatter
//   colsum_nhwc      : bias gradient  db[c] = sum over pixels
//   pack_w           : fp32 [Cout, Cin, KS, KS] -> the K-major 16-bit weight matrix of a tap-group list
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/cocos_b200.h"
#include "corr_kernels.h"
#include "tmap.h"

namespace cocos {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// source index of padded coordinate i + pad, i in [-pad, n + pad), pad < n (one reflection per side)
__device__ __forceinline__ int reflect1(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// 4 consecutive channels starting at element index `idx` (multiple of 4)
__device__ __forceinline__ float4 ld4(const void* base, int kind, size_t idx) {
  if (kind == 3) return *reinterpret_cast<const float4*>(static_cast<const float*>(base) + idx);
  const uint2 u = *reinterpret_cast<const uint2*>(static_cast<const uint16_t*>(base) + idx);
  if (kind == 1) {
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
  }
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ void st4(void* base, int kind, size_t idx, float4 v) {
  if (kind == 3) {
    *reinterpret_cast<float4*>(static_cast<float*>(base) + idx) = v;
    return;
  }
  uint2 u;
  if (kind == 1) {
    const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
    u.x = *reinterpret_cast<const uint32_t*>(&a);
    u.y = *reinterpret_cast<const uint32_t*>(&b);
  } else {
    const __nv_bfloat162 a = __floats2bfloat162_rn(v.x, v.y), b = __floats2bfloat162_rn(v.z, v.w);
    u.x = *reinterpret_cast<const uint32_t*>(&a);
    u.y = *reinterpret_cast<const uint32_t*>(&b);
  }
  *reinterpret_cast<uint2*>(static_cast<uint16_t*>(base) + idx) = u;
}

__device__ __forceinline__ float lo16(float v) { return v - __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float4 lo4(float4 v) { return make_float4(lo16(v.x), lo16(v.y), lo16(v.z), lo16(v.w)); }
__device__ __forceinline__ float lrelu(float v, float s) { return v > 0.f ? v : v * s; }

// ----------------------------------------------------------------------------------------------- SPADE modulation
struct SpadeFwd {
  const void* x; int x_kind, x_Cs;
  const void* gb; int gb_kind, gb_Cs;   // gamma at channel [0,C), beta at [C,2C)
  void* y; int y_Cs, y_lo_off;          // fp16 op, [B, H+2p, W+2p, y_Cs]
  float* mean; float* rstd;             // [B,H,W]
  int B, C, H, W, pad;
  float slope, eps;
};

// one warp per (padded) output pixel
__global__ void __launch_bounds__(256) spade_mod_nhwc_fwd_kernel(const SpadeFwd p) {
  const int Hp = p.H + 2 * p.pad, Wp = p.W + 2 * p.pad;
  const int lane = threadIdx.x & 31;
  const long long op = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (op >= static_cast<long long>(p.B) * Hp * Wp) return;
  const int b = static_cast<int>(op / (Hp * Wp));
  const int r = static_cast<int>(op - static_cast<long long>(b) * Hp * Wp);
  const int ho = r / Wp, wo = r - ho * Wp;
  const int hs = reflect1(ho - p.pad, p.H), ws = reflect1(wo - p.pad, p.W);
  const size_t spix = (static_cast<size_t>(b) * p.H + hs) * p.W + ws;
  const size_t xo = spix * p.x_Cs, go = spix * p.gb_Cs, yo = static_cast<size_t>(op) * p.y_Cs;
  const int n4 = p.C >> 2;
  float sum = 0.f;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = ld4(p.x, p.x_kind, xo + 4 * i);
    sum += (v.x + v.y) + (v.z + v.w);
  }
  const float mean = warp_sum(sum) / p.C;
  float ss = 0.f;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = ld4(p.x, p.x_kind, xo + 4 * i);
    const float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    ss += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(ss) / (p.C - 1) + p.eps);
  if (lane == 0 && ho - p.pad == hs && wo - p.pad == ws) {
    p.mean[spix] = mean;
    p.rstd[spix] = rstd;
  }
  for (int i = lane; i < n4; i += 32) {
    const float4 v = ld4(p.x, p.x_kind, xo + 4 * i);
    const float4 g = ld4(p.gb, p.gb_kind, go + 4 * i), be = ld4(p.gb, p.gb_kind, go + p.C + 4 * i);
    float4 z;
    z.x = lrelu(fmaf((v.x - mean) * rstd, 1.0f + g.x, be.x), p.slope);
    z.y = lrelu(fmaf((v.y - mean) * rstd, 1.0f + g.y, be.y), p.slope);
    z.z = lrelu(fmaf((v.z - mean) * rstd, 1.0f + g.z, be.z), p.slope);
    z.w = lrelu(fmaf((v.w - mean) * rstd, 1.0f + g.w, be.w), p.slope);
    st4(p.y, 1, yo + 4 * i, z);
    if (p.y_lo_off) st4(p.y, 1, yo + p.y_lo_off + 4 * i, lo4(z));
  }
}

// per-pixel PONO statistics for the SPADE epilogue of the tap convolution: one warp per pixel, two passes (L1-resident)
__global__ void __launch_bounds__(256)
pono_stats_nhwc_kernel(const void* __restrict__ x, int kind, int Cs, int C, long long npix, float eps,
                       float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int lane = threadIdx.x & 31;
  const long long pix = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (pix >= npix) return;
  const size_t xo = static_cast<size_t>(pix) * Cs;
  const int n4 = C >> 2;
  float sum = 0.f;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = ld4(x, kind, xo + 4 * i);
    sum += (v.x + v.y) + (v.z + v.w);
  }
  const float mean = warp_sum(sum) / C;
  float ss = 0.f;
  for (int i = lane; i < n4; i += 32) {
    const float4 v = ld4(x, kind, xo + 4 * i);
    const float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    ss += (a * a + bb * bb) + (c * c + d * d);
  }
  const float rstd = rsqrtf(warp_sum(ss) / (C - 1) + eps);
  if (lane == 0) {
    mean_out[pix] = mean;
    rstd_out[pix] = rstd;
  }
}

struct SpadeBwd {
  const void* dy; int dy_Cs;            // bf16 [B, H+2p, W+2p, dy_Cs]
  const void* x; int x_kind, x_Cs;
  const void* gb; int gb_kind, gb_Cs;
  int gb_W;                             // 0: gb / dgb = [gamma | beta]; W: per 2W channels [gamma of W | beta of W]
  const float* mean; const float* rstd;
  void* dx; int dx_Cs, dx_acc;          // bf16 [B,H,W,dx_Cs]; dx_acc: add to what is there
  void* dgb; int dgb_Cs;                // bf16 [B,H,W,dgb_Cs]: d gamma [0,C), d beta [C,2C)
  int B, C, H, W, pad;
  float slope;
};

// gradient of the padded output folded back onto source pixel (h, w): up to 3 x 3 halo images (pad < H, W: at most
// one mirror image per side and dimension)
struct Fold {
  int hc[3], wc[3], nh, nw;
};
__device__ __forceinline__ Fold make_fold(int h, int w, int H, int W, int pad) {
  Fold f;
  f.nh = f.nw = 0;
  f.hc[f.nh++] = h + pad;
  f.wc[f.nw++] = w + pad;
  if (pad) {
    if (h >= 1 && h <= pad) f.hc[f.nh++] = pad - h;
    if (h <= H - 2 && h >= H - 1 - pad) f.hc[f.nh++] = 2 * (H - 1) - h + pad;
    if (w >= 1 && w <= pad) f.wc[f.nw++] = pad - w;
    if (w <= W - 2 && w >= W - 1 - pad) f.wc[f.nw++] = 2 * (W - 1) - w + pad;
  }
  return f;
}
__device__ __forceinline__ float4 folded4(const void* dy, int kind, const Fold& f, size_t img_off, int Wp, int Cs,
                                          int c) {
  float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int a = 0; a < f.nh; ++a)
    for (int e = 0; e < f.nw; ++e) {
      const float4 t = ld4(dy, kind, (img_off + static_cast<size_t>(f.hc[a]) * Wp + f.wc[e]) * Cs + c);
      d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
    }
  return d;
}

// one warp per source pixel; two passes over the channels (sums, then the outputs)
__global__ void __launch_bounds__(256) spade_mod_nhwc_bwd_kernel(const SpadeBwd p) {
  const int Hp = p.H + 2 * p.pad, Wp = p.W + 2 * p.pad;
  const int lane = threadIdx.x & 31;
  const long long pixl = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (pixl >= static_cast<long long>(p.B) * p.H * p.W) return;
  const size_t spix = static_cast<size_t>(pixl);
  const int b = static_cast<int>(pixl / (p.H * p.W));
  const int r = static_cast<int>(pixl - static_cast<long long>(b) * p.H * p.W);
  const int h = r / p.W, w = r - h * p.W;
  const Fold f = make_fold(h, w, p.H, p.W, p.pad);
  const size_t img = static_cast<size_t>(b) * Hp * Wp;
  const size_t xo = spix * p.x_Cs, go = spix * p.gb_Cs;
  const int n4 = p.C >> 2;
  const float mean = p.mean[spix], rstd = p.rstd[spix];
  float s1 = 0.f, s2 = 0.f;
  // channel c -> position of gamma_c (beta_c is `boff` further) in gb / dgb
  const int boff = p.gb_W ? p.gb_W : p.C;
  for (int i = lane; i < n4; i += 32) {
    const int gi = p.gb_W ? ((4 * i) / p.gb_W) * 2 * p.gb_W + (4 * i) % p.gb_W : 4 * i;
    float4 d = folded4(p.dy, 2, f, img, Wp, p.dy_Cs, 4 * i);
    const float4 v = ld4(p.x, p.x_kind, xo + 4 * i);
    const float4 g = ld4(p.gb, p.gb_kind, go + gi), be = ld4(p.gb, p.gb_kind, go + gi + boff);
    const float xh0 = (v.x - mean) * rstd, xh1 = (v.y - mean) * rstd, xh2 = (v.z - mean) * rstd,
                xh3 = (v.w - mean) * rstd;
    d.x = fmaf(xh0, 1.0f + g.x, be.x) > 0.f ? d.x : d.x * p.slope;
    d.y = fmaf(xh1, 1.0f + g.y, be.y) > 0.f ? d.y : d.y * p.slope;
    d.z = fmaf(xh2, 1.0f + g.z, be.z) > 0.f ? d.z : d.z * p.slope;
    d.w = fmaf(xh3, 1.0f + g.w, be.w) > 0.f ? d.w : d.w * p.slope;
    st4(p.dgb, 2, spix * p.dgb_Cs + gi, make_float4(d.x * xh0, d.y * xh1, d.z * xh2, d.w * xh3));
    st4(p.dgb, 2, spix * p.dgb_Cs + gi + boff, d);
    const float e0 = d.x * (1.0f + g.x), e1 = d.y * (1.0f + g.y), e2 = d.z * (1.0f + g.z), e3 = d.w * (1.0f + g.w);
    s1 += (e0 + e1) + (e2 + e3);
    s2 += (e0 * xh0 + e1 * xh1) + (e2 * xh2 + e3 * xh3);
  }
  const float m1 = warp_sum(s1) / p.C, m2 = warp_sum(s2) / (p.C - 1);
  for (int i = lane; i < n4; i += 32) {
    // d beta was just written by this lane: dz = d beta, no need to fold again
    const int gi = p.gb_W ? ((4 * i) / p.gb_W) * 2 * p.gb_W + (4 * i) % p.gb_W : 4 * i;
    const float4 d = ld4(p.dgb, 2, spix * p.dgb_Cs + gi + boff);
    const float4 v = ld4(p.x, p.x_kind, xo + 4 * i);
    const float4 g = ld4(p.gb, p.gb_kind, go + gi);
    float4 t;
    t.x = rstd * (d.x * (1.0f + g.x) - m1 - (v.x - mean) * rstd * m2);
    t.y = rstd * (d.y * (1.0f + g.y) - m1 - (v.y - mean) * rstd * m2);
    t.z = rstd * (d.z * (1.0f + g.z) - m1 - (v.z - mean) * rstd * m2);
    t.w = rstd * (d.w * (1.0f + g.w) - m1 - (v.w - mean) * rstd * m2);
    const size_t o = spix * p.dx_Cs + 4 * i;
    if (p.dx_acc) {
      const float4 old = ld4(p.dx, 2, o);
      t.x += old.x; t.y += old.y; t.z += old.z; t.w += old.w;
    }
    st4(p.dx, 2, o, t);
  }
}

// ----------------------------------------------------------------------------------------------- instance norm
// Common shape of the four kernels: blockDim = (TX <= 32 channel quads, 8 pixel lanes); a thread owns 4 channels
// (c = (blockIdx.y * TX + tx) * 4) of one image, loads its per-channel coefficients ONCE and walks a pixel range with
// stride 8, so the inner loop is loads / FMAs / stores only.  TX is chosen so that the channel groups are evenly
// filled (C = 408: 4 groups of 26 quads instead of 3 full + 1 with 6).  grid (pixel chunks, channel groups, B).
struct Coef4 {
  float mean[4], rstd[4];
};
// stats [B or 1][C][2] = {sum, sumsq} over `1 / inv` values: per image (InstanceNorm2d) or, with bstride 0, over the
// whole batch (BatchNorm2d in training mode; running statistics in eval mode are passed in the same form)
__device__ __forceinline__ Coef4 load_coef4(const float* __restrict__ stats, int b, int C, int c, float inv, float eps,
                                            int bstride = 1) {
  Coef4 k;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 st = *reinterpret_cast<const float2*>(stats + (static_cast<size_t>(b) * bstride * C + c + j) * 2);
    k.mean[j] = st.x * inv;
    k.rstd[j] = rsqrtf(fmaxf(st.y * inv - k.mean[j] * k.mean[j], 0.f) + eps);
  }
  return k;
}

// part[chunk][b][c] = {sum, sumsq} over the chunk's pixels (blockIdx.x = chunk); ordered_sum() adds the chunks.
__global__ void __launch_bounds__(256)
in_stats_nhwc_kernel(const void* __restrict__ x, int kind, int Cs, int C, int HW, int pix_per_block,
                     float* __restrict__ stats) {
  __shared__ float red[8][32][8];
  const int b = blockIdx.z;
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  const int p0 = blockIdx.x * pix_per_block;
  int p1 = p0 + pix_per_block;
  if (p1 > HW) p1 = HW;
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < C) {
#pragma unroll 4
    for (int pix = p0 + threadIdx.y; pix < p1; pix += 8) {
      const float4 v = ld4(x, kind, (static_cast<size_t>(b) * HW + pix) * Cs + c);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
      q[0] = fmaf(v.x, v.x, q[0]); q[1] = fmaf(v.y, v.y, q[1]); q[2] = fmaf(v.z, v.z, q[2]); q[3] = fmaf(v.w, v.w, q[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    red[threadIdx.y][threadIdx.x][j] = s[j];
    red[threadIdx.y][threadIdx.x][4 + j] = q[j];
  }
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = 0.f, bq = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        a += red[k][threadIdx.x][j];
        bq += red[k][threadIdx.x][4 + j];
      }
      if (c + j < C) {
        float* dst = stats + (static_cast<size_t>(blockIdx.x) * gridDim.z * C + static_cast<size_t>(b) * C + c + j) * 2;
        dst[0] = a;
        dst[1] = bq;
      }
    }
  }
}

struct InstFwd {
  const void* x; int x_kind, x_Cs;
  const float* stats;                    // [B, C, 2] sum / sumsq
  const void* res; int res_kind, res_Cs; // optional residual added after the normalisation
  const float* slope_ptr; float slope;   // PReLU parameter (device scalar) or a constant slope (1 = none)
  void* y; int y_kind, y_Cs, y_lo_off, y_pad;   // op (fp16 [+lo], halo) or any kind without halo
  void* y2; int y2_Cs;                   // optional second output: fp32 NHWC, no halo (residual source of the next block)
  int B, C, H, W;
  float eps;
  // SPADE with instance / batch statistics (normalization.py:96-104,132-149): z = norm(x) * (1 + gamma) + beta
  const void* gb; int gb_kind, gb_Cs;    // optional [gamma | beta] at channels [0,C) and [C,2C)
  int batch_stats;                       // 1: stats are [1][C][2] over B*H*W values (BatchNorm2d)
};

// walks the (padded) OUTPUT pixels: halo pixels re-read their mirror source
__global__ void __launch_bounds__(256) inst_act_nhwc_fwd_kernel(const InstFwd p, int pix_per_block) {
  const int Hp = p.H + 2 * p.y_pad, Wp = p.W + 2 * p.y_pad;
  const int b = blockIdx.z;
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  if (c >= p.C) return;
  const int p0 = blockIdx.x * pix_per_block;
  int p1 = p0 + pix_per_block;
  if (p1 > Hp * Wp) p1 = Hp * Wp;
  const float slope = p.slope_ptr ? *p.slope_ptr : p.slope;
  const float cnt = p.batch_stats ? static_cast<float>(p.B) * p.H * p.W : static_cast<float>(p.H * p.W);
  const Coef4 k = load_coef4(p.stats, b, p.C, c, 1.0f / cnt, p.eps, p.batch_stats ? 0 : 1);
#pragma unroll 2
  for (int op = p0 + threadIdx.y; op < p1; op += 8) {
    const int ho = op / Wp, wo = op - ho * Wp;
    const int hs = reflect1(ho - p.y_pad, p.H), ws = reflect1(wo - p.y_pad, p.W);
    const size_t spix = (static_cast<size_t>(b) * p.H + hs) * p.W + ws;
    const float4 v = ld4(p.x, p.x_kind, spix * p.x_Cs + c);
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.res) t = ld4(p.res, p.res_kind, spix * p.res_Cs + c);
    float4 g1 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (p.gb) {
      const float4 g = ld4(p.gb, p.gb_kind, spix * p.gb_Cs + c), be = ld4(p.gb, p.gb_kind, spix * p.gb_Cs + p.C + c);
      g1 = make_float4(1.f + g.x, 1.f + g.y, 1.f + g.z, 1.f + g.w);
      t.x += be.x; t.y += be.y; t.z += be.z; t.w += be.w;
    }
    float4 o;
    o.x = lrelu(fmaf((v.x - k.mean[0]) * k.rstd[0], g1.x, t.x), slope);
    o.y = lrelu(fmaf((v.y - k.mean[1]) * k.rstd[1], g1.y, t.y), slope);
    o.z = lrelu(fmaf((v.z - k.mean[2]) * k.rstd[2], g1.z, t.z), slope);
    o.w = lrelu(fmaf((v.w - k.mean[3]) * k.rstd[3], g1.w, t.w), slope);
    const size_t yo = (static_cast<size_t>(b) * Hp * Wp + op) * p.y_Cs + c;
    st4(p.y, p.y_kind, yo, o);
    if (p.y_lo_off) st4(p.y, 1, yo + p.y_lo_off, lo4(o));
    if (p.y2 && ho - p.y_pad == hs && wo - p.y_pad == ws) st4(p.y2, 3, spix * p.y2_Cs + c, o);
  }
}

struct InstBwd {
  const void* dy; int dy_Cs, dy_pad;     // bf16 [B, H+2p, W+2p, dy_Cs]
  const void* dy2; int dy2_Cs;           // optional second upstream gradient (of y2), bf16 [B,H,W,dy2_Cs]
  const void* x; int x_kind, x_Cs;
  const float* stats;
  const void* res; int res_kind, res_Cs;
  const float* slope_ptr; float slope;
  float* bstats;                         // [B, C, 2]: sum dz, sum dz*z (pass 1 output, pass 2 input)
  float* dslope;                         // optional PReLU gradient accumulator (pass 1)
  void* dx; int dx_Cs, dx_acc;           // bf16
  void* dres; int dres_Cs, dres_acc;     // optional bf16
  int B, C, H, W;
  float eps;
  const void* gb; int gb_kind, gb_Cs;    // optional SPADE modulation [gamma | beta]
  void* dgb; int dgb_Cs;                 // bf16 [B,H,W,dgb_Cs]: d gamma [0,C), d beta [C,2C) (pass 2 output)
  int batch_stats;                       // statistics over the whole batch: stats / bstats are [1][C][2]
  int const_stats;                       // eval-mode BatchNorm: the statistics do not depend on x (no mean terms)
};

// dz for 4 channels of one source pixel (shared by both passes).  MODE < 0: every option read from the descriptor at run
// time; MODE = xf32 | res << 1 | pad << 2 | dy2 << 3 (no modulation, residual of x's kind): the options are compile-time
// constants, so the loop bodies are straight-line code whose loads the compiler can hoist and batch.
template <int MODE>
__device__ __forceinline__ void inst_bwd_dz(const InstBwd& p, const Coef4& k, int b, int pix, int c, float slope,
                                            float* z, float* dz, float* u_neg_dy, float* dact) {
  constexpr bool GEN = MODE < 0;
  const int xk = GEN ? p.x_kind : ((MODE & 1) ? 3 : 1);
  const bool has_res = GEN ? (p.res != nullptr) : ((MODE & 2) != 0);
  const bool has_pad = GEN ? (p.dy_pad != 0) : ((MODE & 4) != 0);
  const bool has_dy2 = GEN ? (p.dy2 != nullptr) : ((MODE & 8) != 0);
  const size_t spix = static_cast<size_t>(b) * p.H * p.W + pix;
  float4 d;
  if (has_pad) {
    const int Wp = p.W + 2 * p.dy_pad, Hp = p.H + 2 * p.dy_pad;
    const int h = pix / p.W, w = pix - h * p.W;
    const Fold f = make_fold(h, w, p.H, p.W, p.dy_pad);
    d = folded4(p.dy, 2, f, static_cast<size_t>(b) * Hp * Wp, Wp, p.dy_Cs, c);
  } else {
    d = ld4(p.dy, 2, spix * p.dy_Cs + c);
  }
  if (has_dy2) {
    const float4 t = ld4(p.dy2, 2, spix * p.dy2_Cs + c);
    d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
  }
  const float4 v = ld4(p.x, xk, spix * p.x_Cs + c);
  float rs[4] = {0.f, 0.f, 0.f, 0.f};
  if (has_res) {
    const float4 t = ld4(p.res, GEN ? p.res_kind : xk, spix * p.res_Cs + c);
    rs[0] = t.x; rs[1] = t.y; rs[2] = t.z; rs[3] = t.w;
  }
  float g1[4] = {1.f, 1.f, 1.f, 1.f};
  if (GEN && p.gb) {
    const float4 g = ld4(p.gb, p.gb_kind, spix * p.gb_Cs + c), be = ld4(p.gb, p.gb_kind, spix * p.gb_Cs + p.C + c);
    g1[0] += g.x; g1[1] += g.y; g1[2] += g.z; g1[3] += g.w;
    rs[0] += be.x; rs[1] += be.y; rs[2] += be.z; rs[3] += be.w;
  }
  const float in[4] = {v.x, v.y, v.z, v.w}, dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    z[j] = (in[j] - k.mean[j]) * k.rstd[j];
    const float u = fmaf(z[j], g1[j], rs[j]);
    dact[j] = u > 0.f ? dd[j] : dd[j] * slope;   // gradient behind the activation: d beta, d residual
    dz[j] = dact[j] * g1[j];                      // gradient of the normalised value
    u_neg_dy[j] = u > 0.f ? 0.f : dd[j] * u;
  }
}

// pass 1: per-block partials of {sum dz, sum dz*z} (bstats) and of sum dy*u*[u<=0] (dslope)
template <int MODE>
__global__ void __launch_bounds__(256) inst_act_nhwc_bwd_stats_kernel(const InstBwd p, int pix_per_block) {
  __shared__ float red[8][32][8];
  __shared__ float red_s[8][32];
  const int b = blockIdx.z;
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  const int HW = p.H * p.W;
  const int p0 = blockIdx.x * pix_per_block;
  int p1 = p0 + pix_per_block;
  if (p1 > HW) p1 = HW;
  const float slope = p.slope_ptr ? *p.slope_ptr : p.slope;
  float s[4] = {0.f, 0.f, 0.f, 0.f}, q[4] = {0.f, 0.f, 0.f, 0.f}, ds = 0.f;
  if (c < p.C) {
    const float cnt = p.batch_stats ? static_cast<float>(p.B) * HW : static_cast<float>(HW);
    const Coef4 k = load_coef4(p.stats, b, p.C, c, 1.0f / cnt, p.eps, p.batch_stats ? 0 : 1);
#pragma unroll 4
    for (int pix = p0 + threadIdx.y; pix < p1; pix += 8) {
      float z[4], dz[4], un[4], da[4];
      inst_bwd_dz<MODE>(p, k, b, pix, c, slope, z, dz, un, da);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[j] += dz[j];
        q[j] = fmaf(dz[j], z[j], q[j]);
        ds += un[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    red[threadIdx.y][threadIdx.x][j] = s[j];
    red[threadIdx.y][threadIdx.x][4 + j] = q[j];
  }
  red_s[threadIdx.y][threadIdx.x] = ds;
  __syncthreads();
  if (threadIdx.y == 0) {
    if (c < p.C) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = 0.f, bq = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          a += red[k][threadIdx.x][j];
          bq += red[k][threadIdx.x][4 + j];
        }
        if (c + j < p.C) {
          // partial of (chunk, b): part[(chunk * B + b) * 2C + 2c] -- ordered_sum() adds the chunks (and, for batch
          // statistics, the images) in a fixed order
          float* dst = p.bstats + (static_cast<size_t>(blockIdx.x) * p.B + b) * 2 * p.C + 2 * (c + j);
          dst[0] = a;
          dst[1] = bq;
        }
      }
    }
    if (p.dslope && threadIdx.x == 0) {  // (a block row can be narrower than a warp: no shuffles here)
      float t = 0.f;
      for (int k = 0; k < 8; ++k)
        for (int xx = 0; xx < static_cast<int>(blockDim.x); ++xx) t += red_s[k][xx];
      p.dslope[blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)] = t;  // one partial per block
    }
  }
}

// pass 2: dx = rstd * (dz - mean(dz) - z * mean(dz*z)); dres = dz
template <int MODE>
__global__ void __launch_bounds__(256) inst_act_nhwc_bwd_apply_kernel(const InstBwd p, int pix_per_block) {
  const int b = blockIdx.z;
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  if (c >= p.C) return;
  const int HW = p.H * p.W;
  const int p0 = blockIdx.x * pix_per_block;
  int p1 = p0 + pix_per_block;
  if (p1 > HW) p1 = HW;
  const float slope = p.slope_ptr ? *p.slope_ptr : p.slope;
  const float inv = 1.0f / (p.batch_stats ? static_cast<float>(p.B) * HW : static_cast<float>(HW));
  const Coef4 k = load_coef4(p.stats, b, p.C, c, inv, p.eps, p.batch_stats ? 0 : 1);
  float m1[4], m2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 bs = *reinterpret_cast<const float2*>(p.bstats + (static_cast<size_t>(p.batch_stats ? 0 : b) * p.C + c + j) * 2);
    m1[j] = p.const_stats ? 0.f : bs.x * inv;
    m2[j] = p.const_stats ? 0.f : bs.y * inv;
  }
#pragma unroll 4
  for (int pix = p0 + threadIdx.y; pix < p1; pix += 8) {
    float z[4], dz[4], un[4], o[4], da[4];
    inst_bwd_dz<MODE>(p, k, b, pix, c, slope, z, dz, un, da);
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = k.rstd[j] * (dz[j] - m1[j] - z[j] * m2[j]);
    const size_t spix = static_cast<size_t>(b) * HW + pix;
    if (p.dgb) {
      st4(p.dgb, 2, spix * p.dgb_Cs + c, make_float4(da[0] * z[0], da[1] * z[1], da[2] * z[2], da[3] * z[3]));
      st4(p.dgb, 2, spix * p.dgb_Cs + p.C + c, make_float4(da[0], da[1], da[2], da[3]));
    }
    float4 t = make_float4(o[0], o[1], o[2], o[3]);
    if (p.dx_acc) {
      const float4 old = ld4(p.dx, 2, spix * p.dx_Cs + c);
      t.x += old.x; t.y += old.y; t.z += old.z; t.w += old.w;
    }
    st4(p.dx, 2, spix * p.dx_Cs + c, t);
    if (p.dres) {
      float4 t2 = make_float4(da[0], da[1], da[2], da[3]);
      if (p.dres_acc) {
        const float4 old = ld4(p.dres, 2, spix * p.dres_Cs + c);
        t2.x += old.x; t2.y += old.y; t2.z += old.z; t2.w += old.w;
      }
      st4(p.dres, 2, spix * p.dres_Cs + c, t2);
    }
  }
}

// ----------------------------------------------------------------------------------------------- activation backward
// dz = fold_halo(dy) * act'(y) for an activation fused into a convolution epilogue (ReLU / LeakyReLU): y is the op
// tensor the epilogue wrote (halo `pad`), dy its gradient (bf16, same geometry), dz bf16 without halo.
__global__ void __launch_bounds__(256)
act_bwd_nhwc_kernel(const void* __restrict__ dy, int dy_Cs, const void* __restrict__ y, int y_kind, int y_Cs, int pad,
                    void* __restrict__ dz, int dz_Cs, int B, int C, int H, int W, int act, float slope) {
  const int n4 = C >> 2;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(B) * H * W * n4) return;
  const int c = static_cast<int>(idx % n4) * 4;
  const long long pixl = idx / n4;
  const int b = static_cast<int>(pixl / (H * W));
  const int r = static_cast<int>(pixl - static_cast<long long>(b) * H * W);
  const int h = r / W, w = r - h * W;
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const Fold f = make_fold(h, w, H, W, pad);
  float4 d = folded4(dy, 2, f, static_cast<size_t>(b) * Hp * Wp, Wp, dy_Cs, c);
  const float4 v = ld4(y, y_kind, ((static_cast<size_t>(b) * Hp + h + pad) * Wp + w + pad) * y_Cs + c);
  const float neg = act == 1 ? 0.f : slope;
  d.x = v.x > 0.f ? d.x : d.x * neg;
  d.y = v.y > 0.f ? d.y : d.y * neg;
  d.z = v.z > 0.f ? d.z : d.z * neg;
  d.w = v.w > 0.f ? d.w : d.w * neg;
  st4(dz, 2, static_cast<size_t>(pixl) * dz_Cs + c, d);
}

// ----------------------------------------------------------------------------------------------- feature losses
// out[0] += scale * sum_b w[b] * sum_{pixels, c < C} |x - y|  (mode 0: criterionFeat / weighted_l1_loss,
// pix2pix_model.py:240,253; util/util.py:36-40) or (x - y)^2 (mode 1: the perceptual MSE, pix2pix_model.py:256) over two
// fp16 NHWC feature tensors -- the discriminator / VGG19 features never leave the 16-bit NHWC pipeline for their loss.
// One block = 8 pixel lanes x 32 threads x 8 channels; block reduction, one partial per block (added in block order by ordered_sum).
__global__ void __launch_bounds__(256)
pair_loss_nhwc_fwd_kernel(const uint16_t* __restrict__ x, int x_Cs, const uint16_t* __restrict__ y, int y_Cs,
                          const float* __restrict__ w, int B, long long HW, int C8, float scale, int mode,
                          float* __restrict__ out) {
  __shared__ float red[8];
  const long long total = static_cast<long long>(B) * HW * C8;
  float acc = 0.f;
  for (long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * 256) {
    const int c = static_cast<int>(idx % C8) * 8;
    const long long pix = idx / C8;
    const float wb = w ? w[pix / HW] : 1.0f;
    const uint4 a = *reinterpret_cast<const uint4*>(x + pix * x_Cs + c);
    const uint4 b = *reinterpret_cast<const uint4*>(y + pix * y_Cs + c);
    const __half2* ha = reinterpret_cast<const __half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]);
      const float d0 = fa.x - fb.x, d1 = fa.y - fb.y;
      s += mode ? (d0 * d0 + d1 * d1) : (fabsf(d0) + fabsf(d1));
    }
    acc = fmaf(wb, s, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k];
    out[blockIdx.x] = t * scale;  // one partial per block
  }
}

// dx (bf16) (+)= g[0] * scale * w[b] * sign(x - y)  (mode 0)  or  2 (x - y)  (mode 1)
__global__ void __launch_bounds__(256)
pair_loss_nhwc_bwd_kernel(const uint16_t* __restrict__ x, int x_Cs, const uint16_t* __restrict__ y, int y_Cs,
                          const float* __restrict__ w, int B, long long HW, int C8, float scale, int mode,
                          const float* __restrict__ g, uint16_t* __restrict__ dx, int dx_Cs, int acc) {
  const long long total = static_cast<long long>(B) * HW * C8;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % C8) * 8;
  const long long pix = idx / C8;
  const float k = __ldg(g) * scale * (w ? w[pix / HW] : 1.0f);
  const uint4 a = *reinterpret_cast<const uint4*>(x + pix * x_Cs + c);
  const uint4 b = *reinterpret_cast<const uint4*>(y + pix * y_Cs + c);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&b);
  uint4 o = make_uint4(0u, 0u, 0u, 0u);
  if (acc) o = *reinterpret_cast<const uint4*>(dx + pix * dx_Cs + c);
  __nv_bfloat162* ob = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 fa = __half22float2(ha[i]), fb = __half22float2(hb[i]);
    const float d0 = fa.x - fb.x, d1 = fa.y - fb.y;
    float g0, g1;
    if (mode) {
      g0 = 2.f * k * d0; g1 = 2.f * k * d1;
    } else {
      g0 = d0 > 0.f ? k : (d0 < 0.f ? -k : 0.f);
      g1 = d1 > 0.f ? k : (d1 < 0.f ? -k : 0.f);
    }
    float2 old = make_float2(0.f, 0.f);
    if (acc) old = __bfloat1622float2(ob[i]);
    ob[i] = __floats2bfloat162_rn(old.x + g0, old.y + g1);
  }
  *reinterpret_cast<uint4*>(dx + pix * dx_Cs + c) = o;
}

// ----------------------------------------------------------------------------------------------- fp16 -> bf16 operand
// The backward-weights GEMM multiplies dY (bf16: gradients need the fp32 exponent range) with the activation X the
// forward saved (fp16 [hi | lo]); wgmma cannot mix fp16 x bf16 operands, and converting X inside the GEMM kernel
// repeats the conversion for every output-channel tile.  So X is converted here, once per tensor, in an HBM-bound
// pass: dst[pix][c] = bf16(hi + lo), 8 channels (16 bytes) per thread, halo pixels included.
__global__ void __launch_bounds__(256)
cast_op_bf16_kernel(const uint16_t* __restrict__ src, int src_Cs, int lo_off, uint16_t* __restrict__ dst, int dst_Cs,
                    long long npix) {
  const int n8 = dst_Cs >> 3;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= npix * n8) return;
  const int c = static_cast<int>(idx % n8) * 8;
  const long long pix = idx / n8;
  const uint4 hi = *reinterpret_cast<const uint4*>(src + pix * src_Cs + c);
  uint4 lo = make_uint4(0u, 0u, 0u, 0u);
  if (lo_off) lo = *reinterpret_cast<const uint4*>(src + pix * src_Cs + lo_off + c);
  const __half2* h = reinterpret_cast<const __half2*>(&hi);
  const __half2* l = reinterpret_cast<const __half2*>(&lo);
  uint4 o;
  __nv_bfloat162* ob = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 a = __half22float2(h[i]), b = __half22float2(l[i]);
    ob[i] = __floats2bfloat162_rn(a.x + b.x, a.y + b.y);
  }
  *reinterpret_cast<uint4*>(dst + pix * dst_Cs + c) = o;
}

// ----------------------------------------------------------------------------------------------- 2x2 max pooling
// nn.MaxPool2d(kernel_size=2, stride=2) of the VGG19 feature net (correspondence.py:84-100) over fp16 NHWC
// [B, 2*Ho, 2*Wo, Cs] -> [B, Ho, Wo, Cs]; 8 channels (one 16-byte vector) per thread.
__global__ void __launch_bounds__(256)
maxpool2_nhwc_fwd_kernel(const uint16_t* __restrict__ x, uint16_t* __restrict__ y, int B, int Cs, int Ho, int Wo) {
  const int n8 = Cs >> 3;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(B) * Ho * Wo * n8) return;
  const int c = static_cast<int>(idx % n8) * 8;
  const long long pix = idx / n8;
  const int b = static_cast<int>(pix / (Ho * Wo));
  const int r = static_cast<int>(pix - static_cast<long long>(b) * Ho * Wo);
  const int ho = r / Wo, wo = r - ho * Wo;
  const size_t W2 = 2 * static_cast<size_t>(Wo);
  const size_t base = ((static_cast<size_t>(b) * 2 * Ho + 2 * ho) * W2 + 2 * wo) * Cs + c;
  const uint4 v00 = *reinterpret_cast<const uint4*>(x + base);
  const uint4 v01 = *reinterpret_cast<const uint4*>(x + base + Cs);
  const uint4 v10 = *reinterpret_cast<const uint4*>(x + base + W2 * Cs);
  const uint4 v11 = *reinterpret_cast<const uint4*>(x + base + W2 * Cs + Cs);
  uint4 o;
  const __half2* a = reinterpret_cast<const __half2*>(&v00);
  const __half2* bb = reinterpret_cast<const __half2*>(&v01);
  const __half2* cc = reinterpret_cast<const __half2*>(&v10);
  const __half2* d = reinterpret_cast<const __half2*>(&v11);
  __half2* oo = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) oo[i] = __hmax2(__hmax2(a[i], bb[i]), __hmax2(cc[i], d[i]));
  *reinterpret_cast<uint4*>(y + static_cast<size_t>(pix) * Cs + c) = o;
}

// dx[b, 2ho+i, 2wo+j, c] = dy[b, ho, wo, c] at the FIRST maximum of the window in scan order (what ATen's
// max_pool2d_with_indices keeps), 0 elsewhere.  x fp16, dy / dx bf16.
__global__ void __launch_bounds__(256)
maxpool2_nhwc_bwd_kernel(const uint16_t* __restrict__ dy, const uint16_t* __restrict__ x, uint16_t* __restrict__ dx,
                         int B, int Cs, int Ho, int Wo) {
  const int n8 = Cs >> 3;
  const long long idx = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x;
  if (idx >= static_cast<long long>(B) * Ho * Wo * n8) return;
  const int c = static_cast<int>(idx % n8) * 8;
  const long long pix = idx / n8;
  const int b = static_cast<int>(pix / (Ho * Wo));
  const int r = static_cast<int>(pix - static_cast<long long>(b) * Ho * Wo);
  const int ho = r / Wo, wo = r - ho * Wo;
  const size_t W2 = 2 * static_cast<size_t>(Wo);
  const size_t base = ((static_cast<size_t>(b) * 2 * Ho + 2 * ho) * W2 + 2 * wo) * Cs + c;
  const size_t off[4] = {0, static_cast<size_t>(Cs), W2 * Cs, W2 * Cs + Cs};
  uint4 v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = *reinterpret_cast<const uint4*>(x + base + off[k]);
  const uint4 g = *reinterpret_cast<const uint4*>(dy + static_cast<size_t>(pix) * Cs + c);
  const uint16_t* gs = reinterpret_cast<const uint16_t*>(&g);
  uint4 o[4];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float best = __half2float(__ushort_as_half(reinterpret_cast<const uint16_t*>(&v[0])[e]));
    int arg = 0;
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const float t = __half2float(__ushort_as_half(reinterpret_cast<const uint16_t*>(&v[k])[e]));
      if (t > best) { best = t; arg = k; }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) reinterpret_cast<uint16_t*>(&o[k])[e] = (k == arg) ? gs[e] : static_cast<uint16_t>(0);
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) *reinterpret_cast<uint4*>(dx + base + off[k]) = o[k];
}

// ----------------------------------------------------------------------------------------------- pack / unpack
// fp32 NCHW [B, C, Hs, Ws] -> NHWC kind `kind` [B, H+2p, W+2p, Cs]: dst pixel (h, w) = src pixel (h*f, w*f)
// (nearest down-sampling by the integer factor f, F.interpolate(mode='nearest')), reflection halo, channels
// [C, Cs) zero, optional lo term.  blockDim (32, 8): smem-tiled transpose, 32 pixels x 32 channels per block.
__global__ void __launch_bounds__(256)
nhwc_pack_kernel(const float* __restrict__ src, void* __restrict__ dst, int kind, int C, int Cs, int cspan, int lo_off,
                 int Hs, int Ws, int H, int W, int f, int pad) {
  __shared__ float tile[32][33];
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32;
  const int op0 = blockIdx.x * 32;
  // load: thread x = pixel, thread y (+8k) = channel
  {
    const int op = op0 + threadIdx.x;
    const bool live = op < Hp * Wp;
    const int opc = live ? op : 0;
    const int ho = opc / Wp, wo = opc - ho * Wp;
    const int hs = reflect1(ho - pad, H) * f, ws = reflect1(wo - pad, W) * f;
#pragma unroll
    for (int k = 0; k < 32; k += 8) {
      const int c = c0 + threadIdx.y + k;
      tile[threadIdx.y + k][threadIdx.x] =
          (live && c < C) ? src[((static_cast<size_t>(b) * C + c) * Hs + hs) * Ws + ws] : 0.f;
    }
  }
  __syncthreads();
  // store: thread x = channel, thread y (+8k) = pixel
  const int c = c0 + threadIdx.x;
#pragma unroll
  for (int k = 0; k < 32; k += 8) {
    const int op = op0 + threadIdx.y + k;
    if (op < Hp * Wp && c < cspan) {
      const float v = tile[threadIdx.x][threadIdx.y + k];
      const size_t o = (static_cast<size_t>(b) * Hp * Wp + op) * Cs + c;
      if (kind == 3) static_cast<float*>(dst)[o] = v;
      else if (kind == 2) static_cast<uint16_t*>(dst)[o] = __bfloat16_as_ushort(__float2bfloat16_rn(v));
      else {
        static_cast<uint16_t*>(dst)[o] = __half_as_ushort(__float2half_rn(v));
        if (lo_off) static_cast<uint16_t*>(dst)[o + lo_off] = __half_as_ushort(__float2half_rn(lo16(v)));
      }
    }
  }
}

// NHWC kind `kind` [B, H+2p, W+2p, Cs] (channels [c_lo, c_lo + C)) -> fp32 NCHW [B, Cd, Hd, Wd] channels
// [cd_lo, cd_lo + C) at pixels (h*f, w*f); the reflection halo is folded back; acc: add instead of overwrite.
__global__ void __launch_bounds__(256)
nhwc_unpack_kernel(const void* __restrict__ src, int kind, int Cs, int c_lo, int C, int H, int W, int pad,
                   float* __restrict__ dst, int Cd, int cd_lo, int Hd, int Wd, int f, int acc) {
  __shared__ float tile[32][33];
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32;
  const int p0 = blockIdx.x * 32;
  {
    const int c = c0 + threadIdx.x;
#pragma unroll
    for (int k = 0; k < 32; k += 8) {
      const int pix = p0 + threadIdx.y + k;
      float v = 0.f;
      if (pix < H * W && c < C) {
        const int h = pix / W, w = pix - h * W;
        const Fold fo = make_fold(h, w, H, W, pad);
        for (int a = 0; a < fo.nh; ++a)
          for (int e = 0; e < fo.nw; ++e) {
            const size_t o = ((static_cast<size_t>(b) * Hp + fo.hc[a]) * Wp + fo.wc[e]) * Cs + c_lo + c;
            if (kind == 3) v += static_cast<const float*>(src)[o];
            else if (kind == 2) v += __bfloat162float(__ushort_as_bfloat16(static_cast<const uint16_t*>(src)[o]));
            else v += __half2float(__ushort_as_half(static_cast<const uint16_t*>(src)[o]));
          }
      }
      tile[threadIdx.y + k][threadIdx.x] = v;
    }
  }
  __syncthreads();
  const int pix = p0 + threadIdx.x;
  if (pix < H * W) {
    const int h = pix / W, w = pix - h * W;
#pragma unroll
    for (int k = 0; k < 32; k += 8) {
      const int c = c0 + threadIdx.y + k;
      if (c < C) {
        float* d = dst + ((static_cast<size_t>(b) * Cd + cd_lo + c) * Hd + static_cast<size_t>(h) * f) * Wd +
                   static_cast<size_t>(w) * f;
        const float v = tile[threadIdx.x][threadIdx.y + k];
        *d = acc ? *d + v : v;
      }
    }
  }
}

// Fast path of nhwc_unpack for 16-bit sources without halo (the common case: features handed to torch): a block moves
// 32 pixels x 64 channels; 16-byte loads along the channels, 128-byte stores along the pixels.
__global__ void __launch_bounds__(256)
nhwc_unpack16_kernel(const uint16_t* __restrict__ src, int bf16, int Cs, int c_lo, int C, int HW, float* __restrict__ dst,
                     int Cd, int cd_lo, int acc) {
  __shared__ float tile[64][33];
  const int b = blockIdx.z, c0 = blockIdx.y * 64, p0 = blockIdx.x * 32;
  {
    const int cv = (threadIdx.x & 7) * 8, pix = p0 + (threadIdx.x >> 3);
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (pix < HW && c0 + cv < C) {
      const uint4 u = *reinterpret_cast<const uint4*>(src + (static_cast<size_t>(b) * HW + pix) * Cs + c_lo + c0 + cv);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float2 f;
        if (bf16) f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
        else f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
        v[2 * i] = f.x; v[2 * i + 1] = f.y;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) tile[cv + i][threadIdx.x >> 3] = v[i];
  }
  __syncthreads();
  const int pix = p0 + (threadIdx.x & 31);
  if (pix >= HW) return;
#pragma unroll
  for (int k = 0; k < 64; k += 8) {
    const int c = c0 + k + (threadIdx.x >> 5);
    if (c < C) {
      float* d = dst + (static_cast<size_t>(b) * Cd + cd_lo + c) * HW + pix;
      const float v = tile[k + (threadIdx.x >> 5)][threadIdx.x & 31];
      *d = acc ? *d + v : v;
    }
  }
}

// part[chunk][c] = sum over the chunk's rows of a 16-bit / fp32 [rows, Cs] matrix; grid (row chunks, C/128)
__global__ void __launch_bounds__(256)
colsum_nhwc_kernel(const void* __restrict__ x, int kind, int Cs, int C, long long rows, int rows_per_block,
                   float* __restrict__ out) {
  __shared__ float red[8][32][4];
  const int c = blockIdx.y * 128 + threadIdx.x * 4;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block;
  long long r1 = r0 + rows_per_block;
  if (r1 > rows) r1 = rows;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    for (long long r = r0 + threadIdx.y; r < r1; r += 8) {
      const float4 v = ld4(x, kind, static_cast<size_t>(r) * Cs + c);
      s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x][j] = s[j];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) a += red[k][threadIdx.x][j];
      if (c + j < C) out[static_cast<size_t>(blockIdx.x) * C + c + j] = a;
    }
  }
}

// Weight matrix of a tap-group list: dst[row][g*Kc + c] for row < rows (rows_alloc >= rows: the rest zero),
// g < ngroups, c < Kc.  transposed == 0 (forward): row = output channel, c = input channel, value = W[row][c][r][s];
// transposed == 1 (backward-data): row = input channel, c = output channel, value = W[c][row][r][s].
// term 0: the 16-bit rounding of the value; term 1: lo = fp16(value - fp16(value)).
struct PackW {
  const float* w; int Cout, Cin, KS;
  void* dst; int rows, rows_alloc, Kc, ngroups, transposed, bf16;
  int8_t r[COCOS_TAPCONV_MAX_GROUPS], s[COCOS_TAPCONV_MAX_GROUPS], term[COCOS_TAPCONV_MAX_GROUPS];
};
// One block = a 32 (output channels) x 32 (input channels) tile of the filter, staged through shared memory: the fp32
// source [Cout, Cin, KS, KS] is read in runs of 32*KS*KS contiguous floats (one per output channel); then each warp
// owns destination rows and writes, per tap group, 32 consecutive 16-bit elements (lane = the contiguous index of the
// destination: input channel for the plain layout, output channel for the transposed one).  dst is fully written
// (zeros beyond the filter's extents: no memset).  grid (ceil(Kc or rows_alloc / 32) input, ... output tiles).
__global__ void __launch_bounds__(256) pack_w_kernel(const PackW p) {
  extern __shared__ float tile[];  // [32][32 * KS*KS + 1]
  const int kk = p.KS * p.KS;
  const int pitch = 32 * kk + 1;
  const int ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  const int lane = threadIdx.x, warp = threadIdx.y;
  const int run = (p.Cin - ci0 < 32 ? p.Cin - ci0 : 32) * kk;  // contiguous floats per output channel (<= 0: none)
  for (int co = warp; co < 32; co += 8) {
    const bool ok = co0 + co < p.Cout;
    const float* src = p.w + (static_cast<size_t>(co0 + co) * p.Cin + ci0) * kk;
    for (int e = lane; e < 32 * kk; e += 32) tile[co * pitch + e] = (ok && e < run) ? src[e] : 0.f;
  }
  __syncthreads();
  uint16_t* dst = static_cast<uint16_t*>(p.dst);
  const size_t Kt = static_cast<size_t>(p.ngroups) * p.Kc;
  // plain: row = co0 + r, column = ci0 + lane, element tile[r][lane];  transposed: row = ci0 + r, column = co0 + lane,
  // element tile[lane][r]
  const int row0 = p.transposed ? ci0 : co0, col = (p.transposed ? co0 : ci0) + lane;
  if (col >= p.Kc) return;
  for (int r = warp; r < 32; r += 8) {
    if (row0 + r >= p.rows_alloc) break;
    const float* t = p.transposed ? tile + lane * pitch + r * kk : tile + r * pitch + lane * kk;
    uint16_t* d = dst + static_cast<size_t>(row0 + r) * Kt + col;
    for (int g = 0; g < p.ngroups; ++g) {
      const float v = t[p.r[g] * p.KS + p.s[g]];
      d[static_cast<size_t>(g) * p.Kc] = p.bf16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v))
                                                : __half_as_ushort(__float2half_rn(p.term[g] ? lo16(v) : v));
    }
  }
}

// ----------------------------------------------------------------------------------------------- squeeze-excitation
// SELayer (architecture.py:182-197) on the raw output dx of a SPADE block's conv_1, fused with the block's residual sum:
// y = res + s[b, c] * dx with s = sigmoid(W2 relu(W1 mean_hw(dx))), W1 [Cr, C], W2 [C, Cr] (bias-free nn.Linear).

// s[b] = sigmoid(W2 relu(W1 m[b])) with m = the per-(image, channel) sums of cocos_in_stats_nhwc / HW: one block per
// image; m and the hidden activations are kept for the backward.  Every sum runs in a fixed order.
__global__ void __launch_bounds__(256)
se_excite_kernel(const float* __restrict__ stats, const float* __restrict__ w1, const float* __restrict__ w2, int C,
                 int Cr, float inv_hw, float* __restrict__ m, float* __restrict__ hid, float* __restrict__ s) {
  extern __shared__ float sh[];  // m [C] | hidden [Cr]
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float v = stats[(static_cast<size_t>(b) * C + c) * 2] * inv_hw;
    sh[c] = v;
    m[static_cast<size_t>(b) * C + c] = v;
  }
  __syncthreads();
  for (int j = warp; j < Cr; j += blockDim.x >> 5) {
    float t = 0.f;
    for (int c = lane; c < C; c += 32) t = fmaf(w1[static_cast<size_t>(j) * C + c], sh[c], t);
    t = fmaxf(warp_sum(t), 0.f);
    if (lane == 0) {
      sh[C + j] = t;
      hid[static_cast<size_t>(b) * Cr + j] = t;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float z = 0.f;
    for (int j = 0; j < Cr; ++j) z = fmaf(w2[static_cast<size_t>(c) * Cr + j], sh[C + j], z);
    s[static_cast<size_t>(b) * C + c] = 1.f / (1.f + expf(-z));
  }
}

// y[b, p, c] = res[b, p, c] + s[b, c] * dx[b, p, c]; one thread per 4 channels of a pixel
__global__ void __launch_bounds__(256)
se_apply_nhwc_kernel(const void* __restrict__ dx, int dx_kind, int dx_Cs, const void* __restrict__ res, int res_kind,
                     int res_Cs, const float* __restrict__ s, void* __restrict__ y, int y_kind, int y_Cs, int C, int HW,
                     long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c4 = C >> 2;
  const long long px = i / c4;
  const int c = static_cast<int>(i - px * c4) * 4;
  const float4 v = ld4(dx, dx_kind, px * dx_Cs + c), r = ld4(res, res_kind, px * res_Cs + c);
  const float4 g = *reinterpret_cast<const float4*>(s + (px / HW) * C + c);
  st4(y, y_kind, px * y_Cs + c, make_float4(fmaf(g.x, v.x, r.x), fmaf(g.y, v.y, r.y), fmaf(g.z, v.z, r.z),
                                            fmaf(g.w, v.w, r.w)));
}

// part[chunk][b][c] = sum over the chunk's pixels of dx * dy (dy bf16): the gradient of the gate; ordered_sum() adds
// the chunks.  Grid / block as in_stats_nhwc_kernel.
__global__ void __launch_bounds__(256)
se_dot_nhwc_kernel(const void* __restrict__ dx, int dx_kind, int dx_Cs, const void* __restrict__ dy, int dy_Cs, int C,
                   int HW, int pix_per_block, float* __restrict__ part) {
  __shared__ float red[8][32][4];
  const int b = blockIdx.z;
  const int c = (blockIdx.y * blockDim.x + threadIdx.x) * 4;
  const int p0 = blockIdx.x * pix_per_block;
  const int p1 = p0 + pix_per_block < HW ? p0 + pix_per_block : HW;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < C) {
#pragma unroll 4
    for (int pix = p0 + threadIdx.y; pix < p1; pix += 8) {
      const size_t px = static_cast<size_t>(b) * HW + pix;
      const float4 v = ld4(dx, dx_kind, px * dx_Cs + c), d = ld4(dy, 2, px * dy_Cs + c);
      s[0] = fmaf(v.x, d.x, s[0]); s[1] = fmaf(v.y, d.y, s[1]); s[2] = fmaf(v.z, d.z, s[2]); s[3] = fmaf(v.w, d.w, s[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x][j] = s[j];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float a = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) a += red[k][threadIdx.x][j];
      if (c + j < C) part[(static_cast<size_t>(blockIdx.x) * gridDim.z + b) * C + c + j] = a;
    }
  }
}

// backward of the gate of image b from ds = sum_hw dx * dy: e2 = ds s (1 - s) (before the sigmoid), e1 = relu'(hid)
// (W2^T e2) (before the ReLU), dm = W1^T e1 / HW (what every pixel of dx receives through the mean)
__global__ void __launch_bounds__(256)
se_excite_bwd_kernel(const float* __restrict__ ds, const float* __restrict__ s, const float* __restrict__ hid,
                     const float* __restrict__ w1, const float* __restrict__ w2, int C, int Cr, float inv_hw,
                     float* __restrict__ e2, float* __restrict__ e1, float* __restrict__ dm) {
  extern __shared__ float sh[];  // e2 [C] | e1 [Cr]
  const int b = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const size_t i = static_cast<size_t>(b) * C + c;
    const float sv = s[i], v = ds[i] * sv * (1.f - sv);
    sh[c] = v;
    e2[i] = v;
  }
  __syncthreads();
  for (int j = warp; j < Cr; j += blockDim.x >> 5) {
    float t = 0.f;
    for (int c = lane; c < C; c += 32) t = fmaf(w2[static_cast<size_t>(c) * Cr + j], sh[c], t);
    t = warp_sum(t);
    if (lane == 0) {
      const float v = hid[static_cast<size_t>(b) * Cr + j] > 0.f ? t : 0.f;
      sh[C + j] = v;
      e1[static_cast<size_t>(b) * Cr + j] = v;
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
    for (int j = 0; j < Cr; ++j) t = fmaf(w1[static_cast<size_t>(j) * C + c], sh[C + j], t);
    dm[static_cast<size_t>(b) * C + c] = t * inv_hw;
  }
}

// dW1[j, c] = sum_b e1[b, j] m[b, c] and dW2[c, j] = sum_b e2[b, c] hid[b, j], images in ascending order
__global__ void __launch_bounds__(256)
se_wgrad_kernel(const float* __restrict__ e1, const float* __restrict__ e2, const float* __restrict__ m,
                const float* __restrict__ hid, int B, int C, int Cr, float* __restrict__ dw1, float* __restrict__ dw2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = C * Cr;
  if (i >= 2 * n) return;
  float t = 0.f;
  if (i < n) {
    const int j = i / C, c = i - j * C;
    for (int b = 0; b < B; ++b) t = fmaf(e1[b * Cr + j], m[static_cast<size_t>(b) * C + c], t);
    dw1[i] = t;
  } else {
    const int k = i - n, c = k / Cr, j = k - c * Cr;
    for (int b = 0; b < B; ++b) t = fmaf(e2[static_cast<size_t>(b) * C + c], hid[b * Cr + j], t);
    dw2[k] = t;
  }
}

// d dx[b, p, c] = s[b, c] dy[b, p, c] + dm[b, c] (bf16)
__global__ void __launch_bounds__(256)
se_dx_nhwc_kernel(const void* __restrict__ dy, int dy_Cs, const float* __restrict__ s, const float* __restrict__ dm,
                  void* __restrict__ ddx, int ddx_Cs, int C, int HW, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c4 = C >> 2;
  const long long px = i / c4;
  const int c = static_cast<int>(i - px * c4) * 4;
  const size_t bc = (px / HW) * C + c;
  const float4 d = ld4(dy, 2, px * dy_Cs + c);
  const float4 g = *reinterpret_cast<const float4*>(s + bc), k = *reinterpret_cast<const float4*>(dm + bc);
  st4(ddx, 2, px * ddx_Cs + c, make_float4(fmaf(g.x, d.x, k.x), fmaf(g.y, d.y, k.y), fmaf(g.z, d.z, k.z),
                                           fmaf(g.w, d.w, k.w)));
}

inline int blocks_for(long long n, int per) { return static_cast<int>((n + per - 1) / per); }

}  // namespace

// ------------------------------------------------------------------------------------------------- launchers
int spade_mod_nhwc_fwd_launch(const void* x, int x_kind, int x_Cs, const void* gb, int gb_kind, int gb_Cs, void* y,
                              int y_Cs, int y_lo_off, float* mean, float* rstd, int B, int C, int H, int W, int pad,
                              float slope, float eps, cudaStream_t stream) {
  if (B <= 0 || C < 4 || (C % 4) || H <= pad || W <= pad || pad < 0 || (x_Cs % 4) || (gb_Cs % 4) ||
      (y_Cs % 4) || (y_lo_off % 4) || (x_kind != 1 && x_kind != 3) || (gb_kind != 1 && gb_kind != 3)) {
    set_error("spade_mod_nhwc_fwd: bad arguments (B=%d C=%d H=%d W=%d pad=%d)", B, C, H, W, pad);
    return -1;
  }
  SpadeFwd p{x, x_kind, x_Cs, gb, gb_kind, gb_Cs, y, y_Cs, y_lo_off, mean, rstd, B, C, H, W, pad, slope, eps};
  const long long pix = static_cast<long long>(B) * (H + 2 * pad) * (W + 2 * pad);
  spade_mod_nhwc_fwd_kernel<<<blocks_for(pix, 8), 256, 0, stream>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int pono_stats_nhwc_launch(const void* x, int kind, int Cs, int C, long long npix, float eps, float* mean, float* rstd,
                           cudaStream_t stream) {
  if (npix <= 0 || C < 4 || (C % 4) || (Cs % 4) || Cs < C || (kind != 1 && kind != 3)) {
    set_error("pono_stats_nhwc: bad arguments (C=%d Cs=%d kind=%d npix=%lld)", C, Cs, kind, npix);
    return -1;
  }
  pono_stats_nhwc_kernel<<<blocks_for(npix, 8), 256, 0, stream>>>(x, kind, Cs, C, npix, eps, mean, rstd);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int spade_mod_nhwc_bwd_launch(const void* dy, int dy_Cs, const void* x, int x_kind, int x_Cs, const void* gb,
                              int gb_kind, int gb_Cs, int gb_W, const float* mean, const float* rstd, void* dx,
                              int dx_Cs, int dx_acc, void* dgb, int dgb_Cs, int B, int C, int H, int W, int pad,
                              float slope, cudaStream_t stream) {
  if (B <= 0 || C < 4 || (C % 4) || H <= pad || W <= pad || pad < 0 || (dy_Cs % 4) || (x_Cs % 4) ||
      (gb_Cs % 4) || (dx_Cs % 4) || (dgb_Cs % 4) || (x_kind != 1 && x_kind != 3) || (gb_kind != 1 && gb_kind != 3) ||
      gb_W < 0 || (gb_W && ((gb_W % 4) || (C % gb_W)))) {
    set_error("spade_mod_nhwc_bwd: bad arguments (B=%d C=%d H=%d W=%d pad=%d)", B, C, H, W, pad);
    return -1;
  }
  SpadeBwd p{dy, dy_Cs, x, x_kind, x_Cs, gb, gb_kind, gb_Cs, gb_W, mean, rstd, dx, dx_Cs, dx_acc, dgb, dgb_Cs,
             B, C, H, W, pad, slope};
  spade_mod_nhwc_bwd_kernel<<<blocks_for(static_cast<long long>(B) * H * W, 8), 256, 0, stream>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// grid / block of the instance-norm kernels: TX channel quads per block row (evenly filled groups), ~8 waves of
// blocks, at least 64 pixels per block
static void stats_grid(int HW, int C, int B, dim3* grid, dim3* block, int* ppb) {
  const int c4 = (C + 3) / 4;
  const int cg = (c4 + 31) / 32;
  const int tx = (c4 + cg - 1) / cg;
  int chunks = (8 * num_sms() + cg * B - 1) / (cg * B);
  const int max_chunks = (HW + 63) / 64;
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1) chunks = 1;
  *ppb = (HW + chunks - 1) / chunks;
  *grid = dim3((HW + *ppb - 1) / *ppb, cg, B);
  *block = dim3(tx, 8);
}

int in_stats_nhwc_launch(const void* x, int kind, int Cs, int B, int C, int HW, float* stats, float* ws,
                         long long* ws_floats, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || (C % 4) || (Cs % 4) || HW <= 0 || kind < 1 || kind > 3) {
    set_error("in_stats_nhwc: bad arguments (B=%d C=%d HW=%d)", B, C, HW);
    return -1;
  }
  dim3 grid, block;
  int ppb;
  stats_grid(HW, C, B, &grid, &block, &ppb);
  const long long n = 2ll * B * C;
  const int wc = workspace_check(ws, ws_floats, grid.x * n, "in_stats_nhwc");
  if (wc) return wc < 0 ? -1 : 0;
  float* part = ws;
  in_stats_nhwc_kernel<<<grid, block, 0, stream>>>(x, kind, Cs, C, HW, ppb, part);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return ordered_sum(part, grid.x, n, stats, 0, stream);
}

int inst_act_nhwc_fwd_launch(const void* x, int x_kind, int x_Cs, const float* stats, const void* res, int res_kind,
                             int res_Cs, const float* slope_ptr, float slope, void* y, int y_kind, int y_Cs,
                             int y_lo_off, int y_pad, void* y2, int y2_Cs, int B, int C, int H, int W, float eps,
                             const void* gb, int gb_kind, int gb_Cs, int batch_stats, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || (C % 4) || (x_Cs % 4) || (y_Cs % 4) || (y_lo_off % 4) || H <= y_pad || W <= y_pad ||
      y_pad < 0 || x_kind < 1 || x_kind > 3 || y_kind < 1 || y_kind > 3 || (y_lo_off && y_kind != 1) ||
      (res && (res_kind < 1 || res_kind > 3 || (res_Cs % 4))) || (y2 && (y2_Cs % 4)) ||
      (gb && ((gb_kind != 1 && gb_kind != 3) || (gb_Cs % 4) || gb_Cs < 2 * C))) {
    set_error("inst_act_nhwc_fwd: bad arguments (B=%d C=%d H=%d W=%d pad=%d)", B, C, H, W, y_pad);
    return -1;
  }
  InstFwd p{x, x_kind, x_Cs, stats, res, res_kind, res_Cs, slope_ptr, slope, y, y_kind, y_Cs, y_lo_off, y_pad,
            y2, y2_Cs, B, C, H, W, eps, gb, gb_kind, gb_Cs, batch_stats};
  dim3 grid, block;
  int ppb;
  stats_grid((H + 2 * y_pad) * (W + 2 * y_pad), C, B, &grid, &block, &ppb);
  inst_act_nhwc_fwd_kernel<<<grid, block, 0, stream>>>(p, ppb);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int inst_act_nhwc_bwd_launch(const void* dy, int dy_Cs, int dy_pad, const void* dy2, int dy2_Cs, const void* x,
                             int x_kind, int x_Cs, const float* stats, const void* res, int res_kind, int res_Cs,
                             const float* slope_ptr, float slope, float* bstats, float* dslope, void* dx, int dx_Cs,
                             int dx_acc, void* dres, int dres_Cs, int dres_acc, int B, int C, int H, int W, float eps,
                             const void* gb, int gb_kind, int gb_Cs, void* dgb, int dgb_Cs, int batch_stats,
                             int const_stats, int phase, float* ws, long long* ws_floats, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || (C % 4) || (dy_Cs % 4) || (x_Cs % 4) || (dx_Cs % 4) || H <= dy_pad || W <= dy_pad ||
      dy_pad < 0 || x_kind < 1 || x_kind > 3 || (res && (res_kind < 1 || res_kind > 3 || (res_Cs % 4))) ||
      (dy2 && (dy2_Cs % 4)) || (dres && (dres_Cs % 4)) || !bstats || phase < 0 || phase > 2 ||
      (gb && ((gb_kind != 1 && gb_kind != 3) || (gb_Cs % 4) || gb_Cs < 2 * C || !dgb || (dgb_Cs % 4) || dgb_Cs < 2 * C))) {
    set_error("inst_act_nhwc_bwd: bad arguments (B=%d C=%d H=%d W=%d pad=%d)", B, C, H, W, dy_pad);
    return -1;
  }
  InstBwd p{dy, dy_Cs, dy_pad, dy2, dy2_Cs, x, x_kind, x_Cs, stats, res, res_kind, res_Cs, slope_ptr, slope, bstats,
            dslope, dx, dx_Cs, dx_acc, dres, dres_Cs, dres_acc, B, C, H, W, eps, gb, gb_kind, gb_Cs, dgb, dgb_Cs,
            batch_stats, const_stats};
  dim3 grid, block;
  int ppb;
  stats_grid(H * W, C, B, &grid, &block, &ppb);
  // phase 1: statistics only, phase 2: apply only (a synchronised BatchNorm all-reduces bstats in between), 0: both
  // specialised variants: no modulation, 16-bit or fp32 x, residual (if any) of x's kind
  int mode = -1;
  if (!gb && (x_kind == 1 || x_kind == 3) && (!res || res_kind == x_kind))
    mode = (x_kind == 3 ? 1 : 0) | (res ? 2 : 0) | (dy_pad ? 4 : 0) | (dy2 ? 8 : 0);
  // the statistics kernel writes per-block partials into the workspace: [chunk][b][2C] for bstats, then one per block
  // for dslope; ordered_sum() reduces them in a fixed order before the apply kernel reads bstats
  const long long nb = 2ll * B * C, nblocks = static_cast<long long>(grid.x) * grid.y * grid.z;
  const int wc = workspace_check(ws, ws_floats, phase != 2 ? grid.x * nb + nblocks : 0, "inst_act_nhwc_bwd");
  if (wc) return wc < 0 ? -1 : 0;
  if (phase != 2) {
    float* part = ws;
    InstBwd ps = p;
    ps.bstats = part;
    ps.dslope = dslope ? part + grid.x * nb : nullptr;
#define COCOS_INST_BWD(M) \
  case M: inst_act_nhwc_bwd_stats_kernel<M><<<grid, block, 0, stream>>>(ps, ppb); break;
    switch (mode) {
      COCOS_INST_BWD(0) COCOS_INST_BWD(1) COCOS_INST_BWD(2) COCOS_INST_BWD(3) COCOS_INST_BWD(4) COCOS_INST_BWD(5)
      COCOS_INST_BWD(6) COCOS_INST_BWD(7) COCOS_INST_BWD(8) COCOS_INST_BWD(9) COCOS_INST_BWD(10) COCOS_INST_BWD(11)
      COCOS_INST_BWD(12) COCOS_INST_BWD(13) COCOS_INST_BWD(14) COCOS_INST_BWD(15)
      default: inst_act_nhwc_bwd_stats_kernel<-1><<<grid, block, 0, stream>>>(ps, ppb);
    }
#undef COCOS_INST_BWD
    COCOS_CUDA_CHECK(cudaGetLastError());
    int rc;
    // batch statistics: [chunk * B + b][2C] summed over chunks and images; per image: [chunk][2BC] over chunks
    if ((rc = batch_stats ? ordered_sum(part, grid.x * B, 2ll * C, bstats, 0, stream)
                          : ordered_sum(part, grid.x, nb, bstats, 0, stream)))
      return rc;
    if (dslope && (rc = ordered_sum(part + grid.x * nb, static_cast<int>(nblocks), 1, dslope, 1, stream))) return rc;
  }
  if (phase != 1) {
#define COCOS_INST_BWD(M) \
  case M: inst_act_nhwc_bwd_apply_kernel<M><<<grid, block, 0, stream>>>(p, ppb); break;
    switch (mode) {
      COCOS_INST_BWD(0) COCOS_INST_BWD(1) COCOS_INST_BWD(2) COCOS_INST_BWD(3) COCOS_INST_BWD(4) COCOS_INST_BWD(5)
      COCOS_INST_BWD(6) COCOS_INST_BWD(7) COCOS_INST_BWD(8) COCOS_INST_BWD(9) COCOS_INST_BWD(10) COCOS_INST_BWD(11)
      COCOS_INST_BWD(12) COCOS_INST_BWD(13) COCOS_INST_BWD(14) COCOS_INST_BWD(15)
      default: inst_act_nhwc_bwd_apply_kernel<-1><<<grid, block, 0, stream>>>(p, ppb);
    }
#undef COCOS_INST_BWD
    COCOS_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

int act_bwd_nhwc_launch(const void* dy, int dy_Cs, const void* y, int y_kind, int y_Cs, int pad, void* dz, int dz_Cs,
                        int B, int C, int H, int W, int act, float slope, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || (C % 4) || (dy_Cs % 4) || (y_Cs % 4) || (dz_Cs % 4) || H <= pad || W <= pad || pad < 0 ||
      y_kind < 1 || y_kind > 3 || (act != 1 && act != 2)) {
    set_error("act_bwd_nhwc: bad arguments (B=%d C=%d H=%d W=%d pad=%d act=%d)", B, C, H, W, pad, act);
    return -1;
  }
  const long long n = static_cast<long long>(B) * H * W * (C / 4);
  act_bwd_nhwc_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(dy, dy_Cs, y, y_kind, y_Cs, pad, dz, dz_Cs, B, C, H, W,
                                                              act, slope);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int nhwc_pack_launch(const float* src, void* dst, int kind, int B, int C, int Cs, int lo_off, int c_lo, int c_span,
                     int Hs, int Ws, int H, int W, int f, int pad, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || Cs < C || H <= pad || W <= pad || f < 1 || (H - 1) * f >= Hs || (W - 1) * f >= Ws || pad < 0 ||
      kind < 1 || kind > 3 || (lo_off && (kind != 1 || lo_off < C || 2 * lo_off != Cs)) || c_lo < 0 ||
      c_span < 0 || (c_span && (c_span < C || c_lo + c_span > (lo_off ? lo_off : Cs)))) {
    set_error("nhwc_pack: bad arguments (B=%d C=%d Cs=%d c_lo=%d c_span=%d Hs=%d Ws=%d H=%d W=%d f=%d pad=%d)", B, C, Cs,
              c_lo, c_span, Hs, Ws, H, W, f, pad);
    return -1;
  }
  const int npix = (H + 2 * pad) * (W + 2 * pad);
  // the channel window [c_lo, c_lo + cspan) of dst is written (zeros beyond C); default: everything up to the lo terms
  const int cspan = c_span ? c_span : (lo_off ? lo_off : Cs) - c_lo;
  dst = static_cast<char*>(dst) + static_cast<size_t>(c_lo) * (kind == 3 ? 4 : 2);
  dim3 grid((npix + 31) / 32, (cspan + 31) / 32, B);
  nhwc_pack_kernel<<<grid, dim3(32, 8), 0, stream>>>(src, dst, kind, C, Cs, cspan, lo_off, Hs, Ws, H, W, f, pad);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int nhwc_unpack_launch(const void* src, int kind, int Cs, int c_lo, int C, int B, int H, int W, int pad, float* dst,
                       int Cd, int cd_lo, int Hd, int Wd, int f, int acc, cudaStream_t stream) {
  if (B <= 0 || C <= 0 || c_lo < 0 || c_lo + C > Cs || cd_lo < 0 || cd_lo + C > Cd || H <= pad || W <= pad || f < 1 ||
      (H - 1) * f >= Hd || (W - 1) * f >= Wd || pad < 0 || kind < 1 || kind > 3) {
    set_error("nhwc_unpack: bad arguments (B=%d C=%d Cs=%d H=%d W=%d f=%d pad=%d)", B, C, Cs, H, W, f, pad);
    return -1;
  }
  if (kind != 3 && pad == 0 && f == 1 && Hd == H && Wd == W && (Cs % 8) == 0 && (c_lo % 8) == 0 &&
      (C % 8 == 0 || c_lo + ((C + 7) / 8) * 8 <= Cs)) {
    // (channels up to the next multiple of 8 may be read: they exist whenever the padded extent fits in Cs)
    dim3 grid16((H * W + 31) / 32, (C + 63) / 64, B);
    nhwc_unpack16_kernel<<<grid16, 256, 0, stream>>>(static_cast<const uint16_t*>(src), kind == 2, Cs, c_lo, C, H * W,
                                                     dst, Cd, cd_lo, acc);
    COCOS_CUDA_CHECK(cudaGetLastError());
    return 0;
  }
  dim3 grid((H * W + 31) / 32, (C + 31) / 32, B);
  nhwc_unpack_kernel<<<grid, dim3(32, 8), 0, stream>>>(src, kind, Cs, c_lo, C, H, W, pad, dst, Cd, cd_lo, Hd, Wd, f,
                                                        acc);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int pair_loss_nhwc_fwd_launch(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                              float scale, int mode, float* out, float* ws, long long* ws_floats,
                              cudaStream_t stream) {
  if (B <= 0 || HW <= 0 || C <= 0 || (C % 8) || (x_Cs % 8) || (y_Cs % 8) || x_Cs < C || y_Cs < C || mode < 0 || mode > 1) {
    set_error("pair_loss_nhwc_fwd: bad arguments (B=%d HW=%lld C=%d x_Cs=%d y_Cs=%d)", B, HW, C, x_Cs, y_Cs);
    return -1;
  }
  const long long total = static_cast<long long>(B) * HW * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > num_sms() * 8ll) blocks = num_sms() * 8ll;
  const int wc = workspace_check(ws, ws_floats, blocks, "pair_loss_nhwc_fwd");
  if (wc) return wc < 0 ? -1 : 0;
  float* part = ws;
  pair_loss_nhwc_fwd_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(
      static_cast<const uint16_t*>(x), x_Cs, static_cast<const uint16_t*>(y), y_Cs, w, B, HW, C / 8, scale, mode, part);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return ordered_sum(part, static_cast<int>(blocks), 1, out, 1, stream);  // out += the loss
}

int pair_loss_nhwc_bwd_launch(const void* x, int x_Cs, const void* y, int y_Cs, const float* w, int B, long long HW, int C,
                              float scale, int mode, const float* g, void* dx, int dx_Cs, int acc, cudaStream_t stream) {
  if (B <= 0 || HW <= 0 || C <= 0 || (C % 8) || (x_Cs % 8) || (y_Cs % 8) || (dx_Cs % 8) || x_Cs < C || y_Cs < C ||
      dx_Cs < C || mode < 0 || mode > 1) {
    set_error("pair_loss_nhwc_bwd: bad arguments (B=%d HW=%lld C=%d)", B, HW, C);
    return -1;
  }
  const long long total = static_cast<long long>(B) * HW * (C / 8);
  pair_loss_nhwc_bwd_kernel<<<blocks_for(total, 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(x), x_Cs, static_cast<const uint16_t*>(y), y_Cs, w, B, HW, C / 8, scale, mode, g,
      static_cast<uint16_t*>(dx), dx_Cs, acc);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int cast_op_bf16_launch(const void* src, int src_Cs, int lo_off, void* dst, int dst_Cs, long long npix,
                        cudaStream_t stream) {
  if (npix <= 0 || dst_Cs <= 0 || (dst_Cs % 8) || (src_Cs % 8) || (lo_off % 8) || lo_off < 0 ||
      (lo_off ? lo_off : src_Cs) < dst_Cs || (lo_off && lo_off + dst_Cs > src_Cs)) {
    set_error("cast_op_bf16: bad arguments (src_Cs=%d lo_off=%d dst_Cs=%d npix=%lld)", src_Cs, lo_off, dst_Cs, npix);
    return -1;
  }
  cast_op_bf16_kernel<<<blocks_for(npix * (dst_Cs / 8), 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(src), src_Cs, lo_off, static_cast<uint16_t*>(dst), dst_Cs, npix);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int maxpool2_nhwc_fwd_launch(const void* x, void* y, int B, int Cs, int Ho, int Wo, cudaStream_t stream) {
  if (B <= 0 || Cs <= 0 || (Cs % 8) || Ho <= 0 || Wo <= 0) {
    set_error("maxpool2_nhwc_fwd: bad arguments (B=%d Cs=%d Ho=%d Wo=%d)", B, Cs, Ho, Wo);
    return -1;
  }
  const long long n = static_cast<long long>(B) * Ho * Wo * (Cs / 8);
  maxpool2_nhwc_fwd_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(static_cast<const uint16_t*>(x),
                                                                   static_cast<uint16_t*>(y), B, Cs, Ho, Wo);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int maxpool2_nhwc_bwd_launch(const void* dy, const void* x, void* dx, int B, int Cs, int Ho, int Wo,
                             cudaStream_t stream) {
  if (B <= 0 || Cs <= 0 || (Cs % 8) || Ho <= 0 || Wo <= 0) {
    set_error("maxpool2_nhwc_bwd: bad arguments (B=%d Cs=%d Ho=%d Wo=%d)", B, Cs, Ho, Wo);
    return -1;
  }
  const long long n = static_cast<long long>(B) * Ho * Wo * (Cs / 8);
  maxpool2_nhwc_bwd_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(
      static_cast<const uint16_t*>(dy), static_cast<const uint16_t*>(x), static_cast<uint16_t*>(dx), B, Cs, Ho, Wo);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int colsum_nhwc_launch(const void* x, int kind, int Cs, int C, long long rows, float* out, float* ws,
                       long long* ws_floats, cudaStream_t stream) {
  if (C <= 0 || (C % 4) || (Cs % 4) || rows <= 0 || kind < 1 || kind > 3) {
    set_error("colsum_nhwc: bad arguments (C=%d Cs=%d rows=%lld)", C, Cs, rows);
    return -1;
  }
  const int cg = (C + 127) / 128;
  long long chunks = (4ll * num_sms() + cg - 1) / cg;
  const long long max_chunks = (rows + 63) / 64;
  if (chunks > max_chunks) chunks = max_chunks;
  const int rpb = static_cast<int>((rows + chunks - 1) / chunks);
  dim3 grid(static_cast<unsigned>((rows + rpb - 1) / rpb), cg);
  const int wc = workspace_check(ws, ws_floats, static_cast<long long>(grid.x) * C, "colsum_nhwc");
  if (wc) return wc < 0 ? -1 : 0;
  float* part = ws;
  colsum_nhwc_kernel<<<grid, dim3(32, 8), 0, stream>>>(x, kind, Cs, C, rows, rpb, part);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return ordered_sum(part, grid.x, C, out, 0, stream);
}

int pack_w_launch(const float* w, int Cout, int Cin, int KS, void* dst, int rows, int rows_alloc, int Kc, int ngroups,
                  const signed char* r, const signed char* s, const signed char* term, int transposed, int bf16,
                  cudaStream_t stream) {
  if (!w || !dst || !r || !s || !term || Cout <= 0 || Cin <= 0 || KS <= 0 || rows <= 0 || rows_alloc < rows || Kc <= 0 ||
      (Kc % 64) || ngroups <= 0 || ngroups > COCOS_TAPCONV_MAX_GROUPS) {
    set_error("pack_w: bad arguments (Cout=%d Cin=%d KS=%d rows=%d Kc=%d groups=%d)", Cout, Cin, KS, rows, Kc, ngroups);
    return -1;
  }
  PackW p;
  p.w = w; p.Cout = Cout; p.Cin = Cin; p.KS = KS; p.dst = dst; p.rows = rows; p.rows_alloc = rows_alloc; p.Kc = Kc;
  p.ngroups = ngroups; p.transposed = transposed; p.bf16 = bf16;
  for (int g = 0; g < ngroups; ++g) {
    if (r[g] < 0 || r[g] >= KS || s[g] < 0 || s[g] >= KS) {
      set_error("pack_w: tap (%d,%d) of group %d outside the %dx%d filter", r[g], s[g], g, KS, KS);
      return -1;
    }
    p.r[g] = r[g]; p.s[g] = s[g]; p.term[g] = term[g];
  }
  // the grid covers the padded extents of dst: rows_alloc x Kc (zeros beyond the filter)
  const int n_in = transposed ? rows_alloc : Kc, n_out = transposed ? Kc : rows_alloc;
  const size_t smem = sizeof(float) * 32 * (32 * KS * KS + 1);
  if (smem > 48 * 1024) {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(pack_w_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          static_cast<int>(smem)));
  }
  pack_w_kernel<<<dim3((n_in + 31) / 32, (n_out + 31) / 32), dim3(32, 8), smem, stream>>>(p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static bool se_bad_shape(int B, int C, int Cr, int HW) {
  return B <= 0 || C < 4 || C > 4096 || (C % 4) || Cr <= 0 || Cr > C || HW <= 0;
}

int se_nhwc_fwd_launch(const void* dx, int dx_kind, int dx_Cs, const void* res, int res_kind, int res_Cs,
                       const float* w1, const float* w2, void* y, int y_kind, int y_Cs, float* m, float* hid, float* s,
                       int B, int C, int Cr, int HW, float* ws, long long* ws_floats, cudaStream_t stream) {
  if (se_bad_shape(B, C, Cr, HW) || (dx_Cs % 4) || (res_Cs % 4) || (y_Cs % 4) || dx_Cs < C || res_Cs < C || y_Cs < C ||
      (dx_kind != 1 && dx_kind != 3) || (res_kind != 1 && res_kind != 3) || (y_kind != 1 && y_kind != 3)) {
    set_error("se_nhwc_fwd: bad arguments (B=%d C=%d Cr=%d HW=%d)", B, C, Cr, HW);
    return -1;
  }
  // workspace: the [B, C, 2] statistics of cocos_in_stats_nhwc, then its own partials
  const long long nstats = 2ll * B * C;
  long long need = 0;
  int rc = in_stats_nhwc_launch(dx, dx_kind, dx_Cs, B, C, HW, nullptr, nullptr, &need, stream);
  if (rc) return rc;
  const int wc = workspace_check(ws, ws_floats, nstats + need, "se_nhwc_fwd");
  if (wc) return wc < 0 ? -1 : 0;
  if ((rc = in_stats_nhwc_launch(dx, dx_kind, dx_Cs, B, C, HW, ws, ws + nstats, &need, stream))) return rc;
  se_excite_kernel<<<B, 256, (C + Cr) * sizeof(float), stream>>>(ws, w1, w2, C, Cr, 1.f / HW, m, hid, s);
  COCOS_CUDA_CHECK(cudaGetLastError());
  const long long n = static_cast<long long>(B) * HW * (C / 4);
  se_apply_nhwc_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(dx, dx_kind, dx_Cs, res, res_kind, res_Cs, s, y, y_kind,
                                                               y_Cs, C, HW, n);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int se_nhwc_bwd_launch(const void* dy, int dy_Cs, const void* dx, int dx_kind, int dx_Cs, const float* w1,
                       const float* w2, const float* m, const float* hid, const float* s, void* ddx, int ddx_Cs,
                       float* dw1, float* dw2, int B, int C, int Cr, int HW, float* ws, long long* ws_floats,
                       cudaStream_t stream) {
  if (se_bad_shape(B, C, Cr, HW) || (dy_Cs % 4) || (dx_Cs % 4) || (ddx_Cs % 4) || dy_Cs < C || dx_Cs < C ||
      ddx_Cs < C || (dx_kind != 1 && dx_kind != 3)) {
    set_error("se_nhwc_bwd: bad arguments (B=%d C=%d Cr=%d HW=%d)", B, C, Cr, HW);
    return -1;
  }
  dim3 grid, block;
  int ppb;
  stats_grid(HW, C, B, &grid, &block, &ppb);
  // workspace: ds [B, C] | e2 [B, C] | dm [B, C] | e1 [B, Cr] | per-chunk partials of ds [chunks][B][C]
  const long long bc = static_cast<long long>(B) * C, fixed = 3 * bc + static_cast<long long>(B) * Cr;
  const int wc = workspace_check(ws, ws_floats, fixed + grid.x * bc, "se_nhwc_bwd");
  if (wc) return wc < 0 ? -1 : 0;
  float *ds = ws, *e2 = ws + bc, *dm = ws + 2 * bc, *e1 = ws + 3 * bc, *part = ws + fixed;
  se_dot_nhwc_kernel<<<grid, block, 0, stream>>>(dx, dx_kind, dx_Cs, dy, dy_Cs, C, HW, ppb, part);
  COCOS_CUDA_CHECK(cudaGetLastError());
  int rc = ordered_sum(part, grid.x, bc, ds, 0, stream);
  if (rc) return rc;
  se_excite_bwd_kernel<<<B, 256, (C + Cr) * sizeof(float), stream>>>(ds, s, hid, w1, w2, C, Cr, 1.f / HW, e2, e1, dm);
  COCOS_CUDA_CHECK(cudaGetLastError());
  se_wgrad_kernel<<<blocks_for(2ll * C * Cr, 256), 256, 0, stream>>>(e1, e2, m, hid, B, C, Cr, dw1, dw2);
  COCOS_CUDA_CHECK(cudaGetLastError());
  const long long n = static_cast<long long>(B) * HW * (C / 4);
  se_dx_nhwc_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(dy, dy_Cs, s, dm, ddx, ddx_Cs, C, HW, n);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
