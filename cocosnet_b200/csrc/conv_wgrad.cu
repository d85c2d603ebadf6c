// K2w: TMA-fed wgmma implicit-GEMM convolution, backward-weights (3x3 / 1x1, stride 1), sm_90a.
//
//   dW[n, c, r, s] = sum_{b,h,w} dY[b, n, h, w] * X[b, c, h + r - off, w + s - off]
//
// One GEMM per filter tap: M = 128 output channels n, N = 128/256 input channels c, K = the B*H*W output pixels.
// Both operands are K-major with K = pixels, which is exactly what NCHW gives for free:
//   * A tile = dY, 16-bit NCHW [B, Cout, H, Wp]: one 4-D TMA box {bw, bh, 128, 1} = 64 pixels (bh rows of bw) of 128
//     channels; each channel's 64 pixels land as one 128-byte swizzled row -- the wgmma K-major layout.
//   * B tile = X, 16-bit [KS][B, Cin, Hin, Wp]: KS column-shifted NCHW copies (copy s holds columns s-off .. s-off+W-1;
//     a TMA box has to start on a 16-byte boundary of the innermost dimension, so the tap's column shift is baked into
//     the copy and only the row shift is a coordinate): box {bw, bh, BN, 1} at (w0, h0 + r - off, c0, s*B + b).
//     Rows outside the image and ragged edges are TMA out-of-bounds zero fill (a pixel that does not exist has
//     dY == 0 from the same fill, so it contributes nothing).
//   * Wp: row pitch rounded up to 8 elements (TMA needs 16-byte strides); cocos_cast_pitch makes all these copies.
//   * the pixel range is split over gridDim.z (split-K) so that every layer fills the SMs; split k stores its
//     partial tile into slice k of a workspace and ordered_sum() adds the slices in split order into ws[tap][c][n]
//     (fp32, n contiguous), which the host permutes to [n][c][r][s].
// dY is bf16 (gradient range) and X must have the same 16-bit format (wgmma takes one operand type).
// warp 8: TMA producer, warps 0-7: wgmma, warps 0-3: epilogue.
#include <cstdlib>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int ATOM_BYTES = 128 * BK * 2;
constexpr int NUM_THREADS = TILE_THREADS;

struct WgradParams {
  int B, H, W, Cout, Cin, KS, off;
  int bw, bh, chunks_w, chunks_h;  // a K chunk = bh rows x bw columns = 64 pixels
  int total_chunks, chunks_per_split, splits;
  int a_bf16, b_bf16;
  int dbg;  // COCOS_WG_DBG bring-up knock-outs: 1 no x load, 2 no dy load, 4 no MMA, 8 no stores
  float* ws;  // [KS*KS, Cin, Cout], or with splits > 1 the workspace [splits][KS*KS, Cin, Cout]
  long long ws_size;
};

struct WgradBars {
  uint64_t full[6];
  uint64_t empty[6];
};

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tm_dy, const __grid_constant__ CUtensorMap tm_x,
                  const WgradParams p) {
  constexpr int STAGES = (BN == 128) ? 6 : 4;
  constexpr int STAGE_BYTES = ATOM_BYTES + (BN / 128) * ATOM_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));
  WgradBars* bars = reinterpret_cast<WgradBars*>(smem_gen + STAGES * STAGE_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * BM;  // output channels (rows of dY)
  const int c0 = blockIdx.y * BN;  // input channels
  const int tap = blockIdx.z / p.splits, split = blockIdx.z - tap * p.splits;
  const int r = tap / p.KS, s = tap - r * p.KS;
  const int chunk_lo = split * p.chunks_per_split;
  int chunk_hi = chunk_lo + p.chunks_per_split;
  if (chunk_hi > p.total_chunks) chunk_hi = p.total_chunks;
  const int iters = chunk_hi - chunk_lo;  // >= 1 by construction of `splits`

  if (tid == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(smem_u32(&bars->full[i]), 1);
      mbar_init(smem_u32(&bars->empty[i]), CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tm_dy);
    tma_prefetch_desc(&tm_x);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (elect_one()) {
      uint32_t st = 0, ph = 0;
      int chunk = chunk_lo;
      int cw = chunk % p.chunks_w;
      int tmp = chunk / p.chunks_w;
      int ch = tmp % p.chunks_h;
      int b = tmp / p.chunks_h;
      for (int it = 0; it < iters; ++it) {
        mbar_wait_quiet(smem_u32(&bars->empty[st]), ph ^ 1);
        const uint32_t full = smem_u32(&bars->full[st]);
        mbar_expect_tx(full, ((p.dbg & 2) ? 0 : ATOM_BYTES) + ((p.dbg & 1) ? 0 : (BN / 128) * ATOM_BYTES));
        const int w0 = cw * p.bw, h0 = ch * p.bh;
        if (!(p.dbg & 2)) tma_load_4d(smem0 + st * STAGE_BYTES, &tm_dy, full, w0, h0, n0, b);
        if (!(p.dbg & 1)) tma_load_4d(smem0 + st * STAGE_BYTES + ATOM_BYTES, &tm_x, full, w0, h0 + r - p.off, c0, s * p.B + b);
        if (++st == STAGES) { st = 0; ph ^= 1; }
        if (++cw == p.chunks_w) {
          cw = 0;
          if (++ch == p.chunks_h) { ch = 0; ++b; }
        }
      }
    }
  } else {
    float d[BN / 2];
    const uint32_t a_off = (tid >> 7) * 64 * 128;
    consume_stages<BN>(d, (p.dbg & 4) ? 0 : iters, STAGES, bars->full, bars->empty, p.a_bf16 != 0, 0,
                       [&](uint32_t st, int k, uint64_t& da, uint64_t& db) {
                         const uint32_t a_addr = smem0 + st * STAGE_BYTES;
                         da = desc_advance_k16(make_desc_k_sw128(a_addr + a_off), k);
                         db = desc_advance_k16(make_desc_k_sw128(a_addr + ATOM_BYTES), k);
                       });
    if (p.dbg & 4) {  // no MMA: the stages still have to be released for the producer
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
      uint32_t st = 0, ph = 0;
      for (int it = 0; it < iters; ++it) {
        mbar_wait_quiet(smem_u32(&bars->full[st]), ph);
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars->empty[st]));
        if (++st == STAGES) { st = 0; ph ^= 1; }
      }
    }
    const float* tile = stage_acc<BN>(d, smem_gen);
    if (warp < 4) {
      const int n = n0 + tid;  // accumulator row == output channel
      float* wbase = p.ws + split * p.ws_size + (static_cast<size_t>(tap) * p.Cin) * p.Cout + n;
#pragma unroll 1
      for (int cc = 0; cc < BN / 32; ++cc) {
        uint32_t v[32];
        acc_ld32(tile + tid * (BN + 4) + cc * 32, v);
        if (n < p.Cout && !(p.dbg & 8)) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int c = c0 + cc * 32 + i;
            if (c < p.Cin) {
              wbase[static_cast<size_t>(c) * p.Cout] = __uint_as_float(v[i]);
            }
          }
        }
      }
    }
  }
}

// fp32 [rows, Win] -> 16-bit [nshift, rows, Wp]: copy s holds dst[s][row][w] = src[row][w + s - off] for w < Wout (zero
// where that column does not exist).  Pad columns w >= Wout are left untouched: the tensor maps never read them.
// nshift = 1, off = 0, Wout = Win is a plain cast with a padded pitch.
__global__ void __launch_bounds__(256)
cast_pitch_kernel(const float* __restrict__ src, uint16_t* __restrict__ dst, long long rows, int Win, int Wout, int Wp,
                  int nshift, int off, int bf16) {
  const int wq = (Wout + 3) >> 2;
  const long long total = rows * wq;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * 256) {
    const long long row = i / wq;
    const int w = static_cast<int>(i - row * wq) * 4;
    const float* sp = src + row * Win;
    for (int s = 0; s < nshift; ++s) {
      uint16_t o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = w + j + s - off;
        const float x = (w + j < Wout && col >= 0 && col < Win) ? __ldg(sp + col) : 0.f;
        o[j] = bf16 ? __bfloat16_as_ushort(__float2bfloat16_rn(x)) : __half_as_ushort(__float2half_rn(x));
      }
      // Wp % 8 == 0 and w % 4 == 0: the 8-byte store is aligned and stays inside the padded row
      *reinterpret_cast<uint2*>(dst + (static_cast<long long>(s) * rows + row) * Wp + w) =
          make_uint2(o[0] | (uint32_t(o[1]) << 16), o[2] | (uint32_t(o[3]) << 16));
    }
  }
}

}  // namespace

int cast_pitch_launch(const float* src, void* dst, long long rows, int Win, int Wout, int Wp, int nshift, int off,
                      int bf16, cudaStream_t stream) {
  if (rows <= 0 || Win <= 0 || Wout <= 0 || Wp < Wout || (Wp % 8) != 0 || nshift < 1 || nshift > 3 || off < 0) {
    set_error("cast_pitch: bad shape (rows=%lld Win=%d Wout=%d Wp=%d nshift=%d off=%d)", rows, Win, Wout, Wp, nshift, off);
    return -1;
  }
  const long long total = rows * ((Wout + 3) / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > num_sms() * 16ll) blocks = num_sms() * 16ll;
  cast_pitch_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(src, static_cast<uint16_t*>(dst), rows, Win, Wout, Wp,
                                                                  nshift, off, bf16);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

int conv_wgrad_launch(const void* dy, const void* x, float* ws, int B, int H, int W, int Hin, int Win, int Cout, int Cin,
                      int KS, int off, int a_bf16, int b_bf16, float* ws_part, long long* ws_floats,
                      cudaStream_t stream) {
  if (B <= 0 || H <= 0 || W <= 0 || Hin <= 0 || Win <= 0 || Cout <= 0 || Cin <= 0 || (KS != 1 && KS != 3) || off < 0 ||
      off >= KS) {
    set_error("conv_wgrad: bad shape (B=%d H=%d W=%d Hin=%d Win=%d Cout=%d Cin=%d KS=%d off=%d)", B, H, W, Hin, Win,
              Cout, Cin, KS, off);
    return -1;
  }
  WgradParams p;
  p.B = B; p.H = H; p.W = W; p.Cout = Cout; p.Cin = Cin; p.KS = KS; p.off = off;
  int bw = 8;
  while (bw < W && bw < 64) bw *= 2;
  if (bw < 64) {
    // a {bw < 64, bh, C, 1} box does not land as dense 128-byte swizzled rows, so
    // narrow layers are not taken here; the host routes them to the library wgrad.
    set_error("conv_wgrad: W=%d < 64 is not supported", W);
    return -1;
  }
  p.bw = bw; p.bh = 64 / bw;
  p.chunks_w = (W + bw - 1) / bw;
  p.chunks_h = (H + p.bh - 1) / p.bh;
  p.total_chunks = B * p.chunks_h * p.chunks_w;
  if (a_bf16 != b_bf16) {
    set_error("conv_wgrad: dY and X must share one 16-bit format (a_bf16=%d b_bf16=%d)", a_bf16, b_bf16);
    return -1;
  }
  p.a_bf16 = a_bf16; p.b_bf16 = b_bf16;
  {
    const char* e = getenv("COCOS_WG_DBG");
    p.dbg = e ? atoi(e) : 0;
  }
  p.ws = ws;
  const int BN = Cin > 128 ? 256 : 128;
  const int mt = (Cout + BM - 1) / BM, nt = (Cin + BN - 1) / BN, taps = KS * KS;
  // split-K: aim at ~2 waves of CTAs, keep >= 8 chunks (512 pixels) per CTA so the prologue/epilogue amortise
  int splits = (2 * num_sms() + mt * nt * taps - 1) / (mt * nt * taps);
  const int max_splits = (p.total_chunks + 7) / 8;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  p.chunks_per_split = (p.total_chunks + splits - 1) / splits;
  p.splits = (p.total_chunks + p.chunks_per_split - 1) / p.chunks_per_split;  // no empty CTA
  p.ws_size = (long long)taps * Cin * Cout;
  const int wc = workspace_check(ws_part, ws_floats, p.splits > 1 ? p.splits * p.ws_size : 0, "conv_wgrad");
  if (wc) return wc < 0 ? -1 : 0;
  if (p.splits > 1) p.ws = ws_part;

  const int Wp = (W + 7) / 8 * 8;
  (void)Win;
  CUtensorMap tm_dy, tm_x;
  int rc;
  {
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)H, (uint64_t)Cout, (uint64_t)B};
    const uint64_t pitches[3] = {(uint64_t)Wp * 2, (uint64_t)H * Wp * 2, (uint64_t)Cout * H * Wp * 2};
    const uint32_t box[4] = {(uint32_t)p.bw, (uint32_t)p.bh, BM, 1};
    if ((rc = make_tmap_f16_4d(&tm_dy, dy, dims, pitches, box))) return rc;
  }
  {
    // x arrives as KS column-shifted copies [KS][B][Cin][Hin][Wp] (copy s starts at column s - off), because a TMA
    // box must start on a 16-byte boundary of the innermost dimension: the tap's column shift cannot be a coordinate.
    const uint64_t dims[4] = {(uint64_t)W, (uint64_t)Hin, (uint64_t)Cin, (uint64_t)B * KS};
    const uint64_t pitches[3] = {(uint64_t)Wp * 2, (uint64_t)Hin * Wp * 2, (uint64_t)Cin * Hin * Wp * 2};
    const uint32_t box[4] = {(uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)(BN > 256 ? 256 : BN), 1};
    if ((rc = make_tmap_f16_4d(&tm_x, x, dims, pitches, box))) return rc;
  }
  const int smem_bytes = 1024 + 196608 + 256;
  dim3 grid(mt, nt, taps * p.splits);
  if (BN == 256) {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(conv_wgrad_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    conv_wgrad_kernel<256><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_dy, tm_x, p);
  } else {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(conv_wgrad_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    conv_wgrad_kernel<128><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_dy, tm_x, p);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  if (p.splits > 1) return ordered_sum(p.ws, p.splits, p.ws_size, ws, 0, stream);
  return 0;
}

}  // namespace cocos
