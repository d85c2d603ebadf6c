// K2w-n: backward-weights of the tap convolution (tapconv.cu) over 16-bit NHWC tensors, sm_90a.
//
//   dW[g, n, c] = sum_{b,h,w} dY[b, h, w, n] * X[b, s*h + dh[g], s*w + dw[g], coff + c]
//
// (the wgrad half of autograd's convolution_backward for every nn.Conv2d the tap convolution serves; same reference
// call sites).  One GEMM per tap group g: M = 128 output channels n, N = 128/256 input channels c, K = pixels.
// With NHWC activations the channels are the contiguous dimension of BOTH operands, i.e. both are "MN-major" for
// wgmma: a K step is a run of pixels, each pixel a 128-byte row of 64 channels - exactly what the same 5-D TMA
// boxes the forward kernel uses deliver ({64 ch, TW, 1, TH, 1} with TW*TH = 64 pixels, 128B swizzle), so there are no
// transposed / shifted operand copies at all (the NCHW version needed KS shifted 16-bit copies of X per layer).
//   * A = dY (bf16), 2 atoms of 64 channels; B = X, BN/64 atoms, the tap's offset / stride-2 parity in the coordinates;
//     smem descriptors: MN-major, SWIZZLE_128B, LBO = bytes between 64-channel atoms (64 pixels * 128 B),
//     SBO = 1024 B between 8-pixel groups; a K=16 step advances the start address by 16 pixels = 2048 B.
//   * X is what the forward saved: fp16.  wgmma cannot mix fp16 x bf16 operands and gradients need the bf16 range,
//     so the consumer warps convert the landed X atoms fp16 -> bf16 IN PLACE in shared memory (elementwise, so the
//     swizzle does not matter) and fence to the async proxy before their wgmma reads the stage.  The main loop keeps
//     one stage's wgmmas in flight, so stage s + 1 is converted while stage s is multiplied.
//   * the pixel range is split over the grid (split-K): split k stores its partial tile into slice k of a workspace
//     and ordered_sum() adds the slices in split order into ws[g][n][c] (same bits on every run; a thread owns 32
//     consecutive c of one n: 128-byte runs).
// warp 8: TMA producer, warps 0-7: converter + wgmma (64 output channels each), warps 0-3: epilogue.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/cocos_b200.h"
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int BM = 128;
constexpr int KP = 64;                    // pixels per pipeline stage
constexpr int ATOM = KP * 128;            // one 64-channel atom: 64 pixel rows of 128 B
constexpr int NUM_THREADS = TILE_THREADS;
constexpr int MAXG = COCOS_TAPCONV_MAX_GROUPS;

struct WgParams {
  int B, H, W, Cout, Cin, Cin_s;
  int TH, TW, tiles_h, tiles_w, total_chunks, chunks_per_split, splits;
  int a_stride, Ca, x_f16;
  int ngroups;
  int8_t dh[MAXG], dw[MAXG];
  int16_t coff[MAXG];
  float* ws;  // [ngroups, Cout, Cin_s], or with splits > 1 the workspace [splits][ngroups, Cout, Cin_s]
  long long ws_size;
};

struct WgBars {
  uint64_t full[4];
  uint64_t empty[4];
};

__device__ __forceinline__ void tma_load_5d_w(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                              int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

__device__ __forceinline__ uint32_t h2_to_bf2(uint32_t h) {
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
  const __nv_bfloat162 b = __floats2bfloat162_rn(f.x, f.y);
  return *reinterpret_cast<const uint32_t*>(&b);
}

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapwgrad_kernel(const __grid_constant__ CUtensorMap tm_dy, const __grid_constant__ CUtensorMap tm_x,
                const __grid_constant__ WgParams p) {
  constexpr int STAGES = 4;
  constexpr int NB = BN / 64;  // atoms of the B operand
  constexpr int STAGE_BYTES = (2 + NB) * ATOM;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));
  WgBars* bars = reinterpret_cast<WgBars*>(smem_gen + STAGES * STAGE_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n0 = blockIdx.x * BM;  // output channels
  const int c0 = blockIdx.y * BN;  // input channels
  const int g = blockIdx.z / p.splits, split = blockIdx.z - g * p.splits;
  const int chunk_lo = split * p.chunks_per_split;
  int chunk_hi = chunk_lo + p.chunks_per_split;
  if (chunk_hi > p.total_chunks) chunk_hi = p.total_chunks;
  const int iters = chunk_hi - chunk_lo;  // >= 1 by construction

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
      int dh = p.dh[g], dw = p.dw[g], hpar = 0, cbase = p.coff[g] + c0;
      if (p.a_stride == 2) {
        hpar = dh & 1;
        dh >>= 1;
        cbase += (dw & 1) * p.Ca;
        dw >>= 1;
      }
      uint32_t st = 0, ph = 0;
      int chunk = chunk_lo;
      int tw_i = chunk % p.tiles_w;
      int tmp = chunk / p.tiles_w;
      int th_i = tmp % p.tiles_h;
      int b = tmp / p.tiles_h;
      for (int it = 0; it < iters; ++it) {
        mbar_wait_quiet(smem_u32(&bars->empty[st]), ph ^ 1);
        const uint32_t full = smem_u32(&bars->full[st]);
        mbar_expect_tx(full, STAGE_BYTES);
        const int w0 = tw_i * p.TW, h0 = th_i * p.TH;
        const uint32_t base = smem0 + st * STAGE_BYTES;
#pragma unroll
        for (int a = 0; a < 2; ++a) tma_load_5d_w(base + a * ATOM, &tm_dy, full, n0 + a * 64, w0, 0, h0, b);
#pragma unroll
        for (int a = 0; a < NB; ++a)
          tma_load_5d_w(base + (2 + a) * ATOM, &tm_x, full, cbase + a * 64, w0 + dw, hpar, h0 + dh, b);
        if (++st == STAGES) { st = 0; ph ^= 1; }
        if (++tw_i == p.tiles_w) {
          tw_i = 0;
          if (++th_i == p.tiles_h) { th_i = 0; ++b; }
        }
      }
    }
  } else {
    constexpr int CT = 32 * CONSUMER_WARPS;
    const int wg = tid >> 7;  // output channels [n0 + 64 wg, n0 + 64 wg + 64) = dY atom wg
    float d[BN / 2];
    RingPos rp;
    uint32_t prev = 0;
    for (int it = 0; it < iters; ++it) {
      const uint32_t st = rp.st;
      mbar_wait_quiet(smem_u32(&bars->full[st]), rp.ph);
      if (p.x_f16) {
        // ------------------------------------------------------------ converter: X atoms fp16 -> bf16 in place,
        // while the previous stage's wgmmas are still in flight
        uint4* xb = reinterpret_cast<uint4*>(smem_gen + st * STAGE_BYTES + 2 * ATOM);
#pragma unroll
        for (int i = 0; i < NB * ATOM / 16 / CT; ++i) {
          uint4 v = xb[i * CT + tid];
          v.x = h2_to_bf2(v.x); v.y = h2_to_bf2(v.y); v.z = h2_to_bf2(v.z); v.w = h2_to_bf2(v.w);
          xb[i * CT + tid] = v;
        }
        fence_proxy_async_smem();
        bar_sync(1, CT);
      }
      const uint32_t a_addr = smem0 + st * STAGE_BYTES;
      const uint64_t da = make_desc_mn_sw128(a_addr + wg * ATOM, ATOM), db = make_desc_mn_sw128(a_addr + 2 * ATOM, ATOM);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < KP / 16; ++k)  // 16 pixels = 2048 B further along K
        wgmma_ss<BN, true>(d, da + static_cast<uint64_t>(k * 128), db + static_cast<uint64_t>(k * 128),
                           (it | k) != 0 ? 1 : 0, 1);
      wgmma_commit();
      wgmma_wait<1>();  // one stage in flight; the one before it is complete and goes back to the producer
      if (it > 0) release_stage(&bars->empty[prev]);
      prev = st;
      rp.advance(STAGES);
    }
    wgmma_wait<0>();
    release_stage(&bars->empty[prev]);
    const float* tile = stage_acc<BN>(d, smem_gen);
    // ------------------------------------------------------------------ epilogue
    if (warp < 4) {
      const int n = n0 + tid;  // accumulator row == output channel
      float* wrow = p.ws + split * p.ws_size + (static_cast<size_t>(g) * p.Cout + n) * p.Cin_s;
#pragma unroll 1
      for (int cc = 0; cc < BN / 32; ++cc) {
        const int cb = c0 + cc * 32;
        if (cb >= p.Cin) break;
        uint32_t v[32];
        acc_ld32(tile + tid * (BN + 4) + cc * 32, v);
        if (n < p.Cout) {
          if (cb + 32 <= p.Cin_s) {
            float* dst = wrow + cb;
#pragma unroll
            for (int q = 0; q < 8; ++q) {
              const float a = __uint_as_float(v[4 * q]), b = __uint_as_float(v[4 * q + 1]),
                          c = __uint_as_float(v[4 * q + 2]), d = __uint_as_float(v[4 * q + 3]);
              *reinterpret_cast<float4*>(dst + 4 * q) = make_float4(a, b, c, d);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i)
              if (cb + i < p.Cin_s) wrow[cb + i] = __uint_as_float(v[i]);
          }
        }
      }
    }
  }
}

}  // namespace

int tapwgrad_launch(const cocos_tapwgrad_desc* d, long long* need_out, cudaStream_t stream) {
  if (!d || !d->dy || !d->x || !d->ws) {
    set_error("tapwgrad: null pointer argument");
    return -1;
  }
  const int s = d->a_stride;
  if (d->B <= 0 || d->H <= 0 || d->W <= 0 || d->Hin <= 0 || d->Win <= 0 || d->Ca <= 0 || (d->Ca % 8) || d->Cout <= 0 ||
      d->Cin <= 0 || d->dy_Cs <= 0 || (d->dy_Cs % 8) || (s != 1 && s != 2) || (s == 2 && ((d->Hin | d->Win) & 1)) ||
      d->ngroups <= 0 || d->ngroups > MAXG || d->Cin_s < d->Cin || (d->Cin_s % 4)) {
    set_error("tapwgrad: bad descriptor (B=%d H=%d W=%d Hin=%d Win=%d Ca=%d Cout=%d Cin=%d stride=%d groups=%d)", d->B,
              d->H, d->W, d->Hin, d->Win, d->Ca, d->Cout, d->Cin, s, d->ngroups);
    return -1;
  }
  WgParams p;
  p.B = d->B; p.H = d->H; p.W = d->W; p.Cout = d->Cout; p.Cin = d->Cin; p.Cin_s = d->Cin_s;
  int tw = 8;
  while (tw < d->W && tw < 64) tw *= 2;
  p.TW = tw; p.TH = KP / tw;  // always exactly 64 pixel rows per box (out-of-image pixels are zero fill)
  p.tiles_w = (d->W + p.TW - 1) / p.TW;
  p.tiles_h = (d->H + p.TH - 1) / p.TH;
  p.total_chunks = d->B * p.tiles_h * p.tiles_w;
  p.a_stride = s; p.Ca = d->Ca; p.x_f16 = d->x_f16;
  p.ngroups = d->ngroups;
  for (int g = 0; g < d->ngroups; ++g) {
    p.dh[g] = d->dh[g]; p.dw[g] = d->dw[g]; p.coff[g] = d->coff[g];
    if (d->coff[g] < 0 || (d->coff[g] % 8)) {
      set_error("tapwgrad: channel offset of group %d (%d) must be a non-negative multiple of 8", g, d->coff[g]);
      return -1;
    }
  }
  p.ws = d->ws;
  const int BN = d->Cin > 128 ? 256 : 128;
  const int mt = (d->Cout + BM - 1) / BM, nt = (d->Cin + BN - 1) / BN;
  // split-K: ~2 waves of CTAs, at least 8 chunks (512 pixels) per CTA so prologue / epilogue amortise
  int splits = (2 * num_sms() + mt * nt * d->ngroups - 1) / (mt * nt * d->ngroups);
  const int max_splits = (p.total_chunks + 7) / 8;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  p.chunks_per_split = (p.total_chunks + splits - 1) / splits;
  p.splits = (p.total_chunks + p.chunks_per_split - 1) / p.chunks_per_split;
  p.ws_size = (long long)d->ngroups * d->Cout * d->Cin_s;
  const long long need = p.splits > 1 ? p.splits * p.ws_size : 0;
  if (need_out) {  // size query: nothing is launched
    *need_out = need;
    return 0;
  }
  if (need > 0 && (!d->part || d->part_floats < need)) {
    set_error("tapwgrad: split-K workspace of %lld floats, %lld needed", d->part ? d->part_floats : 0ll, need);
    return -1;
  }
  if (p.splits > 1) {
    // slices are zeroed like ws would be: a tile does not store the channels of a row past its last 32-channel run
    p.ws = d->part;
    COCOS_CUDA_CHECK(cudaMemsetAsync(p.ws, 0, sizeof(float) * p.splits * p.ws_size, stream));
  }

  CUtensorMap tm_dy, tm_x;
  int rc;
  {
    const uint64_t C = (uint64_t)d->dy_Cs, W = (uint64_t)d->W, H = (uint64_t)d->H;
    const uint64_t dims[5] = {C, W, 1, H, (uint64_t)d->B};
    const uint64_t pitches[4] = {C * 2, W * C * 2, W * C * 2, H * W * C * 2};
    const uint32_t box[5] = {64, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if ((rc = make_tmap_16_5d(&tm_dy, d->dy, dims, pitches, box))) return rc;
  }
  {
    const uint64_t Ca = (uint64_t)d->Ca, Win = (uint64_t)d->Win, Hin = (uint64_t)d->Hin;
    const uint64_t dims[5] = {Ca * s, Win / s, (uint64_t)s, Hin / s, (uint64_t)d->B};
    const uint64_t pitches[4] = {Ca * s * 2, Win * Ca * 2, Win * Ca * s * 2, Hin * Win * Ca * 2};
    const uint32_t box[5] = {64, (uint32_t)p.TW, 1, (uint32_t)p.TH, 1};
    if ((rc = make_tmap_16_5d(&tm_x, d->x, dims, pitches, box))) return rc;
  }
  dim3 grid(mt, nt, d->ngroups * p.splits);
  if (BN == 256) {
    const int smem_bytes = 1024 + 4 * (2 + 4) * ATOM + 256;
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(tapwgrad_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    tapwgrad_kernel<256><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_dy, tm_x, p);
  } else {
    const int smem_bytes = 1024 + 4 * (2 + 2) * ATOM + 256;
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(tapwgrad_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    tapwgrad_kernel<128><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_dy, tm_x, p);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  if (p.splits > 1) return ordered_sum(p.ws, p.splits, p.ws_size, d->ws, 0, stream);
  return 0;
}

}  // namespace cocos
