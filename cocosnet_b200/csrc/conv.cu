// K2: TMA-fed wgmma implicit-GEMM convolution, forward (3x3 / 1x1, stride 1), sm_90a.
//
//   Y[b, n, h, w] = bias[n] + sum_{r,s,c} X[b, h + r - off, w + s - off, c] * Wt[n, (r*KS + s)*Cp + c]
//
// The 3x3 convolutions of the SPADE blocks / domain adaptor / residual blocks (reference architecture.py:31-33,
// 73-74; normalization.py:112-120; correspondence.py:17-22) as one GEMM: M = 128 output pixels (a TH x TW patch of
// one image), N = 128 or 256 output channels, K = KS*KS*Cp looped tap by tap.
//   * X is NHWC fp16 [B, Hin, Win, Cp] (Cp % 64 == 0).  `pre_padded`: Hin = H + KS - 1 (reflection padding was done
//     by the producer, off = 0); otherwise Hin = H and the halo is TMA out-of-bounds zero fill (off = KS/2).
//   * the A tile of tap (r, s), channel chunk kc is ONE 4-D TMA box {64 ch, TW, TH, 1} at (kc*64, w0+s-off, h0+r-off, b):
//     its TH*TW rows of 128 B land in (h, w) order with the 128B swizzle -- exactly the K-major operand layout of
//     wgmma, no im2col buffer anywhere.
//   * B tile = weights [Cout, KS*KS*Cp] fp16 K-major, box {64, BN}.
//   * accumulators in registers (fp32, two warpgroups of 64 rows), staged through shared memory; the epilogue adds
//     the bias and writes NCHW fp32, coalesced along w.
// warp 8: TMA producer, warps 0-7: wgmma (N = BN), warps 0-3: epilogue.
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int ATOM_BYTES = 128 * BK * 2;
constexpr int NUM_THREADS = TILE_THREADS;

struct ConvParams {
  int B, H, W, Cout, Cp, KS, off;
  int TH, TW, tiles_h, tiles_w;
  int bf16;           // operands are bf16 (backward-data path) instead of fp16
  const float* bias;  // [Cout] or null
  float* y;           // [B, Cout, H, W]
};

struct ConvBars {
  uint64_t full[6];
  uint64_t empty[6];
};

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_fwd_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                const ConvParams p) {
  constexpr int STAGES = (BN == 128) ? 6 : 4;
  constexpr int STAGE_BYTES = ATOM_BYTES + (BN / 128) * ATOM_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));
  ConvBars* bars = reinterpret_cast<ConvBars*>(smem_gen + STAGES * STAGE_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  int tile = blockIdx.x;
  const int tw_i = tile % p.tiles_w; tile /= p.tiles_w;
  const int th_i = tile % p.tiles_h;
  const int b = tile / p.tiles_h;
  const int h0 = th_i * p.TH, w0 = tw_i * p.TW;
  const int n0 = blockIdx.y * BN;
  const int kc_per_tap = p.Cp / BK;
  const int iters = p.KS * p.KS * kc_per_tap;
  const uint32_t a_bytes = static_cast<uint32_t>(p.TH * p.TW) * 128u;

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(smem_u32(&bars->full[i]), 1);
      mbar_init(smem_u32(&bars->empty[i]), CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_w);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (elect_one()) {
      uint32_t st = 0, ph = 0;
      for (int it = 0; it < iters; ++it) {
        const int tap = it / kc_per_tap, kc = it - tap * kc_per_tap;
        const int r = tap / p.KS, s = tap - r * p.KS;
        mbar_wait_quiet(smem_u32(&bars->empty[st]), ph ^ 1);
        const uint32_t full = smem_u32(&bars->full[st]);
        mbar_expect_tx(full, a_bytes + (BN / 128) * ATOM_BYTES);
        tma_load_4d(smem0 + st * STAGE_BYTES, &tm_x, full, kc * BK, w0 + s - p.off, h0 + r - p.off, b);
        tma_load_3d(smem0 + st * STAGE_BYTES + ATOM_BYTES, &tm_w, full, tap * p.Cp + kc * BK, n0, 0);
        if (++st == STAGES) { st = 0; ph ^= 1; }
      }
    }
  } else {
    float d[BN / 2];
    const uint32_t a_off = (tid >> 7) * 64 * 128;
    consume_stages<BN>(d, iters, STAGES, bars->full, bars->empty, p.bf16 != 0, 0,
                       [&](uint32_t st, int k, uint64_t& da, uint64_t& db) {
                         const uint32_t a_addr = smem0 + st * STAGE_BYTES;
                         da = desc_advance_k16(make_desc_k_sw128(a_addr + a_off), k);
                         db = desc_advance_k16(make_desc_k_sw128(a_addr + ATOM_BYTES), k);
                       });
    const float* tile = stage_acc<BN>(d, smem_gen);
    if (warp < 4) {
      const int m = tid;  // accumulator row == pixel (th, tw) of the patch
      const int th = m / p.TW, tw = m - th * p.TW;
      const int h = h0 + th, w = w0 + tw;
      const bool ok = (m < p.TH * p.TW) && h < p.H && w < p.W;
      const size_t hw = static_cast<size_t>(p.H) * p.W;
      float* ybase = p.y + (static_cast<size_t>(b) * p.Cout) * hw + static_cast<size_t>(h) * p.W + w;
#pragma unroll 1
      for (int c = 0; c < BN / 32; ++c) {
        uint32_t r[32];
        acc_ld32(tile + m * (BN + 4) + c * 32, r);
        if (ok) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int n = n0 + c * 32 + i;
            if (n < p.Cout) ybase[static_cast<size_t>(n) * hw] = __uint_as_float(r[i]) + (p.bias ? p.bias[n] : 0.f);
          }
        }
      }
    }
  }
}

}  // namespace

int conv_fwd_launch(const void* x, const void* wt, const float* bias, float* y, int B, int H, int W, int Hin, int Win,
                    int Cp, int Cout, int KS, int off, int bf16, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || W <= 0 || Hin <= 0 || Win <= 0 || Cp <= 0 || (Cp % BK) || Cout <= 0 || (KS != 1 && KS != 3) ||
      off < 0 || off >= 2 * KS) {
    set_error("conv_fwd: bad shape (B=%d H=%d W=%d Hin=%d Win=%d Cp=%d Cout=%d KS=%d off=%d)", B, H, W, Hin, Win, Cp,
              Cout, KS, off);
    return -1;
  }
  ConvParams p;
  p.B = B; p.H = H; p.W = W; p.Cout = Cout; p.Cp = Cp; p.KS = KS;
  p.off = off; p.bf16 = bf16;
  // patch shape: TH x TW <= 128 pixels minimising the number of (partly empty) tiles; ties -> wider patch (the
  // epilogue stores are coalesced along w).  258x258 (backward-data of a reflection-padded 256x256 layer) gets
  // 4x32 patches (89% full) instead of 1x128 (67%).
  {
    long long best = -1;
    for (int tw = (W < 128 ? W : 128); tw >= 1; --tw) {
      int th = 128 / tw;
      if (th > H) th = H;
      const long long tiles = (long long)((W + tw - 1) / tw) * ((H + th - 1) / th);
      if (best < 0 || tiles < best) { best = tiles; p.TW = tw; p.TH = th; }
    }
  }
  p.tiles_w = (W + p.TW - 1) / p.TW;
  p.tiles_h = (H + p.TH - 1) / p.TH;
  p.bias = bias; p.y = y;
  CUtensorMap tm_x, tm_w;
  const uint64_t dims[4] = {(uint64_t)Cp, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
  const uint64_t pitches[3] = {(uint64_t)Cp * 2, (uint64_t)Win * Cp * 2, (uint64_t)Hin * Win * Cp * 2};
  const uint32_t box[4] = {BK, (uint32_t)p.TW, (uint32_t)p.TH, 1};
  int rc;
  if ((rc = make_tmap_f16_4d(&tm_x, x, dims, pitches, box))) return rc;
  const int BN = Cout > 128 ? 256 : 128;
  const uint64_t Kt = (uint64_t)KS * KS * Cp;
  if ((rc = make_tmap_f16_3d(&tm_w, wt, Kt, Cout, 1, Kt * 2, (uint64_t)Cout * Kt * 2, BK, BN, 1))) return rc;
  const int smem_bytes = 1024 + 196608 + 256;
  dim3 grid(p.tiles_w * p.tiles_h * B, (Cout + BN - 1) / BN);
  if (BN == 256) {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(conv_fwd_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    conv_fwd_kernel<256><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_x, tm_w, p);
  } else {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(conv_fwd_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    conv_fwd_kernel<128><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_x, tm_w, p);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
