// K2n: TMA-fed wgmma implicit-GEMM "tap convolution" over 16-bit NHWC activations, sm_90a.
//
//   Y[b, h, w, n] = epilogue( sum_{g < ngroups} sum_{c < 64*kchunks}
//                             X[b, s*h + dh[g], s*w + dw[g], coff[g] + c] * Wt[n, (g*kchunks)*64 + c] )
//
// One kernel for every convolution of the SPADE generator / domain adaptor / residual blocks / PatchGAN / VGG19
// (reference architecture.py:31-33,73-74; normalization.py:112-120; correspondence.py:17-22,79-146;
// discriminator.py:92-115; generator.py:104-113), forward AND backward-data:
//   * forward KSxKS stride s: one group per filter tap, dh = r - pad (+ the producer's materialised halo);
//   * backward-data of a stride-1 conv: x = dY, flipped taps, Wt = W^T;
//   * backward-data of a stride-2 conv: one launch per input-pixel parity class (a stride-1 tap conv over dY with the
//     taps of matching parity), scattered to the class's pixels through (y_sh, y_sw, y_oh, y_ow);
//   * 2-term fp16 split operands ([hi | lo] along channels): three groups per tap (hi*Whi, lo*Whi, hi*Wlo) - the
//     host lays the weight rows out in the same order; `coff` selects the hi or lo half of x.
// Operands:
//   * A tile = ONE 5-D TMA box {64 ch, TW, 1, TH, TB} of the activation tensor seen as
//     [B, Hin/s, s (row parity), Win/s, s (col parity) * Ca]: its TB*TH*TW rows of 128 B land pixel after pixel with
//     the 128B swizzle, i.e. directly in the K-major operand layout of wgmma (no im2col, no strided gather:
//     a stride-2 tap is a plain tile of the parity-split view).  Out-of-image taps and channels >= Ca are TMA
//     zero fill (zero padding for free; reflection halos are materialised by the producing epilogue).
//   * B tile = weights [Cout, ngroups*kchunks*64] K-major, box {64, BN}.
//   * accumulators: registers of two warpgroups (64 rows x BN fp32 each), staged 32 columns at a time through a
//     shared-memory slab of their own for the epilogue.
// Epilogue (8 warps, two threads per output pixel): + bias, + residual, activation, then store as fp16 / bf16 / fp32
// NHWC (optionally with a 1-pixel halo filled by reflection, optionally as a 2-term [hi | lo] split) or fp32 NCHW.
// warp 8: TMA producer, warps 0-7: wgmma (M=64 each, N=BN) and epilogue.  Persistent: min(tiles, SMs) CTAs, each walking
// a fixed stride of tiles, with the next tile's operands loading during the epilogue.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/cocos_b200.h"
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

namespace cocos {

namespace {

constexpr int BM = 128, BK = 64;
constexpr int ATOM_BYTES = 128 * BK * 2;
// Two consumer warpgroups and a whole third warpgroup around the producer warp: setmaxnreg moves registers between
// warpgroups, so the consumers (BN = 256 keeps 128 accumulators per thread live through the epilogue) get 232 while
// the producer warpgroup drops to 40; 168 each is all a CTA of this size can start with.
constexpr int NUM_THREADS = 32 * CONSUMER_WARPS + 128;
constexpr int MAXG = COCOS_TAPCONV_MAX_GROUPS;

struct TapParams {
  int B, H, W, Cout;
  int TB, TH, TW, tiles_b, tiles_h, tiles_w, tiles_n, num_tiles;
  int a_stride, Ca, bf16;
  int ngroups, kchunks;
  int8_t dh[MAXG], dw[MAXG];
  int16_t coff[MAXG];
  // epilogue
  const float* scale;
  const float* bias;
  const void* res;
  int res_kind, res_Cs;
  int act;
  float slope;
  void* y;
  int y_kind, y_H, y_W, y_Cs, y_coff, y_lo_off, y_pad, y_reflect;
  int y_sh, y_sw, y_oh, y_ow;
  // SPADE modulation epilogue (mod_W > 0): an N tile holds [gamma of mod_W channels | beta of the same channels]
  int mod_W;
  const void* mod_x; int mod_x_kind, mod_x_Cs;
  const float* mod_mean; const float* mod_rstd;
  void* gb; int gb_kind, gb_Cs;
};

struct TapBars {
  uint64_t full[6];
  uint64_t empty[6];
};

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

__device__ __forceinline__ int floordiv2(int v) { return v >> 1; }  // arithmetic shift: floor for negatives

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  if (act == 1) return fmaxf(v, 0.f);
  if (act == 2) return v > 0.f ? v : v * slope;
  if (act == 3) return tanhf(v);
  return v;
}

__device__ __forceinline__ uint32_t pack2(float a, float b, bool bf16) {
  if (bf16) {
    const __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&t);
  }
  const __half2 t = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&t);
}

__device__ __forceinline__ float lo_of(float v) { return v - __half2float(__float2half_rn(v)); }

// N consecutive channels of one pixel -> 16-bit NHWC at `dst` (16-byte aligned when `vec`), n_ok valid channels
template <int N>
__device__ __forceinline__ void store16(uint16_t* dst, const float* v, int n_ok, bool vec, bool bf16) {
  if (vec && n_ok == N) {
    uint4* d4 = reinterpret_cast<uint4*>(dst);
#pragma unroll
    for (int q = 0; q < N / 8; ++q)
      d4[q] = make_uint4(pack2(v[8 * q], v[8 * q + 1], bf16), pack2(v[8 * q + 2], v[8 * q + 3], bf16),
                         pack2(v[8 * q + 4], v[8 * q + 5], bf16), pack2(v[8 * q + 6], v[8 * q + 7], bf16));
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i)
      if (i < n_ok)
        dst[i] = bf16 ? __bfloat16_as_ushort(__float2bfloat16_rn(v[i])) : __half_as_ushort(__float2half_rn(v[i]));
  }
}

template <int N>
__device__ __forceinline__ void store32(float* dst, const float* v, int n_ok, bool vec) {
  if (vec && n_ok == N) {
    float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll
    for (int q = 0; q < N / 4; ++q) d4[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  } else {
#pragma unroll
    for (int i = 0; i < N; ++i)
      if (i < n_ok) dst[i] = v[i];
  }
}

struct TileCoord {
  int n_i, tw_i, th_i, tb_i;
};
// tile index -> coordinates, the N tile innermost (both N tiles of an M tile run back to back and share A in L2)
__device__ __forceinline__ TileCoord tile_coord(int t, const TapParams& p) {
  TileCoord c;
  c.n_i = t % p.tiles_n; t /= p.tiles_n;
  c.tw_i = t % p.tiles_w; t /= p.tiles_w;
  c.th_i = t % p.tiles_h;
  c.tb_i = t / p.tiles_h;
  return c;
}

// The epilogue stages the accumulators through a slab of SLAB_COLS columns that does not alias the operand ring, so
// the producer keeps loading the next tile's stages while it runs.  Pitch 36 (= 4 mod 32 banks): the row reads of
// the epilogue threads are conflict-free.
constexpr int SLAB_COLS = 32, SLAB_LD = SLAB_COLS + 4;
constexpr int SLAB_BYTES = BM * SLAB_LD * 4;
constexpr int RING_BYTES = 196608;  // 6 stages of 32 KB (BN = 128) or 4 of 48 KB (BN = 256)
constexpr int SMEM_BYTES = 1024 + RING_BYTES + SLAB_BYTES + static_cast<int>(sizeof(TapBars));

// Persistent: CTA i runs tiles i, i + gridDim.x, ...  The producer streams the stages of its tiles without a break
// (the ring's phases carry over from tile to tile); each consumer warpgroup keeps its accumulators in registers
// through the epilogue, which writes them into the slab 32 columns per pass.  All 8 consumer warps run the epilogue,
// two threads per output pixel, 16 columns each (SPADE: 8 gamma and the 8 matching beta columns each).
template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tapconv_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
               const __grid_constant__ TapParams p) {
  constexpr int STAGES = (BN == 128) ? 6 : 4;
  constexpr int STAGE_BYTES = ATOM_BYTES + (BN / 128) * ATOM_BYTES;
  static_assert(STAGES * STAGE_BYTES == RING_BYTES, "ring size");
  constexpr int NC = SLAB_COLS / 2;  // columns per epilogue thread and pass
  constexpr int NR = 8;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));
  float* slab = reinterpret_cast<float*>(smem_gen + RING_BYTES);
  TapBars* bars = reinterpret_cast<TapBars*>(smem_gen + RING_BYTES + SLAB_BYTES);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int iters = p.ngroups * p.kchunks;
  const uint32_t a_bytes = static_cast<uint32_t>(p.TB * p.TH * p.TW) * 128u;

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

  if (warp >= CONSUMER_WARPS) {
    setmaxnreg_dec<40>();
    // ------------------------------------------------------------------ TMA producer (warps 9-11 idle)
    if (warp == CONSUMER_WARPS && elect_one()) {
      uint32_t st = 0, ph = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(tile, p);
        const int h0 = tc.th_i * p.TH, w0 = tc.tw_i * p.TW, b0 = tc.tb_i * p.TB, n0 = tc.n_i * BN;
        for (int g = 0; g < p.ngroups; ++g) {
          int dh = p.dh[g], dw = p.dw[g], hpar = 0, cbase = p.coff[g];
          if (p.a_stride == 2) {
            hpar = dh & 1;
            dh = floordiv2(dh);
            cbase += (dw & 1) * p.Ca;
            dw = floordiv2(dw);
          }
          for (int kc = 0; kc < p.kchunks; ++kc) {
            mbar_wait_quiet(smem_u32(&bars->empty[st]), ph ^ 1);
            const uint32_t full = smem_u32(&bars->full[st]);
            mbar_expect_tx(full, a_bytes + (BN / 128) * ATOM_BYTES);
            tma_load_5d(smem0 + st * STAGE_BYTES, &tm_x, full, cbase + kc * BK, w0 + dw, hpar, h0 + dh, b0);
            tma_load_3d(smem0 + st * STAGE_BYTES + ATOM_BYTES, &tm_w, full, (g * p.kchunks + kc) * BK, n0, 0);
            if (++st == STAGES) { st = 0; ph ^= 1; }
          }
        }
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  float d[BN / 2];
  RingPos rp;
  const int row0 = 64 * (tid >> 7);  // this warpgroup's accumulator rows
  const uint32_t a_off = (tid >> 7) * 64 * 128;
  // epilogue role: output pixel m of the tile, columns [NC * half, NC * half + NC) of each pass
  const int m = tid >> 1, half = tid & 1;
  const int rows_per_img = p.TH * p.TW;
  const int tb = m / rows_per_img, rem = m - tb * rows_per_img;
  const int th = rem / p.TW, tw = rem - th * p.TW;
  const int yHp = p.y_H + 2 * p.y_pad, yWp = p.y_W + 2 * p.y_pad;
  const bool out16 = p.y_kind == 1 || p.y_kind == 2;
  const bool obf = p.y_kind == 2;
  const float scale = p.scale ? __ldg(p.scale) : 1.0f;
  const float* acc = slab + m * SLAB_LD;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    // ------------------------------------------------------------------ wgmma main loop
    consume_stages<BN>(d, iters, STAGES, bars->full, bars->empty, p.bf16 != 0, 0,
                       [&](uint32_t st, int k, uint64_t& da, uint64_t& db) {
                         const uint32_t a_addr = smem0 + st * STAGE_BYTES;
                         da = desc_advance_k16(make_desc_k_sw128(a_addr + a_off), k);
                         db = desc_advance_k16(make_desc_k_sw128(a_addr + ATOM_BYTES), k);
                       }, rp);
    // ------------------------------------------------------------------ epilogue
    const TileCoord tc = tile_coord(tile, p);
    const int b = tc.tb_i * p.TB + tb, h = tc.th_i * p.TH + th, w = tc.tw_i * p.TW + tw;
    const int n0 = tc.n_i * BN;
    const bool ok = (tb < p.TB) && b < p.B && h < p.H && w < p.W;
    const int yh = h * p.y_sh + p.y_oh, yw = w * p.y_sw + p.y_ow;
    // store targets: the pixel itself, plus its mirror images in the reflection halo of width q < y_H, y_W (at most
    // one per side: padded row q - yh for 1 <= yh <= q, 2 (y_H - 1) - yh + q for y_H - 1 - q <= yh <= y_H - 2)
    int rt[3], ct[3], nr = 0, nc = 0;
    const int q = p.y_pad;
    rt[nr++] = yh + q;
    ct[nc++] = yw + q;
    if (p.y_reflect && q) {
      if (yh >= 1 && yh <= q) rt[nr++] = q - yh;
      if (yh <= p.y_H - 2 && yh >= p.y_H - 1 - q) rt[nr++] = 2 * (p.y_H - 1) - yh + q;
      if (yw >= 1 && yw <= q) ct[nc++] = q - yw;
      if (yw <= p.y_W - 2 && yw >= p.y_W - 1 - q) ct[nc++] = 2 * (p.y_W - 1) - yw + q;
    }
    const size_t spix = (static_cast<size_t>(b) * p.y_H + yh) * p.y_W + yw;
    float mean = 0.f, rstd = 0.f;
    if (p.mod_W && ok) { mean = __ldg(p.mod_mean + spix); rstd = __ldg(p.mod_rstd + spix); }
#pragma unroll 1
    for (int c = 0; c < BN / SLAB_COLS; ++c) {
      if (!p.mod_W && n0 + c * SLAB_COLS >= p.Cout) break;  // uniform
      bar_sync(1, 32 * CONSUMER_WARPS);  // every reader of the previous pass is done with the slab
      // pass c of the slab: accumulator columns [32c, 32c + 32), or for SPADE (mod_W = BN / 2) gamma [16c, 16c + 16)
      // then the matching beta columns [BN / 2 + 16c, BN / 2 + 16c + 16).  Register indices must be constants, so the
      // pass is selected from an unrolled loop.
#pragma unroll
      for (int cc = 0; cc < BN / SLAB_COLS; ++cc) {
        if (cc != c) continue;
        if (p.mod_W) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            acc_block_to_smem(d + 4 * (2 * cc + q), slab, SLAB_LD, row0, q);
            acc_block_to_smem(d + 4 * (BN / 16 + 2 * cc + q), slab, SLAB_LD, row0, 2 + q);
          }
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) acc_block_to_smem(d + 4 * (4 * cc + q), slab, SLAB_LD, row0, q);
        }
      }
      bar_sync(1, 32 * CONSUMER_WARPS);
      if (!ok) continue;
      if (p.mod_W) {
        // ---- SPADE: y = reflect_pad(lrelu(PONO(x) * (1 + gamma) + beta)) straight from the gamma / beta accumulators
        // (normalization.py:132-149 + architecture.py:73-74); the raw [gamma | beta] pair is stored too when the
        // backward will need it.  Tile n_i covers channels [n_i * mod_W, (n_i + 1) * mod_W) of x / y.
        constexpr int NS = NC / 2;
        uint32_t rg[NS], rb[NS];
        acc_ld<NS>(acc + NS * half, rg);
        acc_ld<NS>(acc + NC + NS * half, rb);
        const int ch = tc.n_i * p.mod_W + c * NC + NS * half;  // channel of x / y
        const int ng = n0 + c * NC + NS * half, nbt = ng + p.mod_W;  // columns (= rows of the interleaved weight / bias)
        float v[NS], g[NS], be[NS];
#pragma unroll
        for (int i = 0; i < NS; ++i) {
          g[i] = __uint_as_float(rg[i]) * scale;
          be[i] = __uint_as_float(rb[i]) * scale;
        }
        if (p.bias) {
#pragma unroll
          for (int i = 0; i < NS; ++i) {
            g[i] += __ldg(p.bias + ng + i);
            be[i] += __ldg(p.bias + nbt + i);
          }
        }
        if (p.gb) {
          const size_t go = spix * p.gb_Cs;
          if (p.gb_kind == 3) {
            store32<NS>(static_cast<float*>(p.gb) + go + ng, g, NS, true);
            store32<NS>(static_cast<float*>(p.gb) + go + nbt, be, NS, true);
          } else {
            store16<NS>(static_cast<uint16_t*>(p.gb) + go + ng, g, NS, true, false);
            store16<NS>(static_cast<uint16_t*>(p.gb) + go + nbt, be, NS, true, false);
          }
        }
        if (p.mod_x_kind == 3) {
          const float4* xp = reinterpret_cast<const float4*>(static_cast<const float*>(p.mod_x) + spix * p.mod_x_Cs + ch);
#pragma unroll
          for (int q = 0; q < NS / 4; ++q) {
            const float4 t = xp[q];
            v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
          }
        } else {
          const uint4* xp = reinterpret_cast<const uint4*>(static_cast<const __half*>(p.mod_x) + spix * p.mod_x_Cs + ch);
#pragma unroll
          for (int q = 0; q < NS / 8; ++q) {
            const uint4 t = xp[q];
            const __half2* h2 = reinterpret_cast<const __half2*>(&t);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const float2 f = __half22float2(h2[e]);
              v[8 * q + 2 * e] = f.x; v[8 * q + 2 * e + 1] = f.y;
            }
          }
        }
#pragma unroll
        for (int i = 0; i < NS; ++i) {
          const float z = fmaf((v[i] - mean) * rstd, 1.0f + g[i], be[i]);
          v[i] = z > 0.f ? z : z * p.slope;
        }
        float lo[NS];
        if (p.y_lo_off) {
#pragma unroll
          for (int i = 0; i < NS; ++i) lo[i] = lo_of(v[i]);
        }
        for (int a = 0; a < nr; ++a)
          for (int e = 0; e < nc; ++e) {
            const size_t po = ((static_cast<size_t>(b) * yHp + rt[a]) * yWp + ct[e]) * p.y_Cs + ch;
            store16<NS>(static_cast<uint16_t*>(p.y) + po, v, NS, true, false);
            if (p.y_lo_off) store16<NS>(static_cast<uint16_t*>(p.y) + po + p.y_lo_off, lo, NS, true, false);
          }
        continue;
      }
      // this thread's NC columns, NR at a time (the accumulators stay live in registers through the epilogue)
#pragma unroll 1
      for (int s = 0; s < NC / NR; ++s) {
        const int nb = n0 + c * SLAB_COLS + NC * half + NR * s;
        const int n_ok = min(NR, p.Cout - nb);
        if (n_ok <= 0) break;
        uint32_t r[NR];
        acc_ld<NR>(acc + NC * half + NR * s, r);
        float v[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) v[i] = __uint_as_float(r[i]) * scale;
        if (p.bias) {
#pragma unroll
          for (int i = 0; i < NR; ++i)
            if (i < n_ok) v[i] += __ldg(p.bias + nb + i);
        }
        if (p.res) {
          const size_t ro = ((static_cast<size_t>(b) * p.y_H + yh) * p.y_W + yw) * p.res_Cs + nb;
          if (p.res_kind == 3) {
            const float* rp_ = static_cast<const float*>(p.res) + ro;
#pragma unroll
            for (int i = 0; i < NR; ++i)
              if (i < n_ok) v[i] += rp_[i];
          } else {
            const __half* rp_ = static_cast<const __half*>(p.res) + ro;
#pragma unroll
            for (int i = 0; i < NR; ++i)
              if (i < n_ok) v[i] += __half2float(rp_[i]);
          }
        }
        if (p.act) {
#pragma unroll
          for (int i = 0; i < NR; ++i) v[i] = apply_act(v[i], p.act, p.slope);
        }
        if (p.y_kind == 0) {  // fp32 NCHW
          const size_t hw = static_cast<size_t>(p.y_H) * p.y_W;
          float* yb = static_cast<float*>(p.y) + (static_cast<size_t>(b) * p.y_Cs + p.y_coff + nb) * hw +
                      static_cast<size_t>(yh) * p.y_W + yw;
#pragma unroll
          for (int i = 0; i < NR; ++i)
            if (i < n_ok) yb[static_cast<size_t>(i) * hw] = v[i];
        } else {
          const int ch = p.y_coff + nb;
          const bool vec = ((ch | p.y_Cs | p.y_lo_off) & 7) == 0;
          float lo[NR];
          if (p.y_lo_off) {
#pragma unroll
            for (int i = 0; i < NR; ++i) lo[i] = lo_of(v[i]);
          }
          for (int a = 0; a < nr; ++a)
            for (int e = 0; e < nc; ++e) {
              const size_t po = ((static_cast<size_t>(b) * yHp + rt[a]) * yWp + ct[e]) * p.y_Cs + ch;
              if (out16) {
                store16<NR>(static_cast<uint16_t*>(p.y) + po, v, n_ok, vec, obf);
                if (p.y_lo_off) store16<NR>(static_cast<uint16_t*>(p.y) + po + p.y_lo_off, lo, n_ok, vec, false);
              } else {
                store32<NR>(static_cast<float*>(p.y) + po, v, n_ok, vec && ((ch | p.y_Cs) & 3) == 0);
              }
            }
        }
      }
    }
  }
}

}  // namespace

// Tile shape of the M dimension: TB images x TH rows x TW columns <= 128 pixels, minimising the number of tiles.
void tapconv_tile_shape(int B, int H, int W, int* TB, int* TH, int* TW) {
  if (H * W <= 64) {  // tiny maps (8x8): several images per tile
    *TW = W; *TH = H;
    int tb = 128 / (H * W);
    if (tb > B) tb = B;
    *TB = tb;
    return;
  }
  *TB = 1;
  long long best = -1;
  for (int tw = (W < 128 ? W : 128); tw >= 1; --tw) {
    int th = 128 / tw;
    if (th > H) th = H;
    const long long tiles = (long long)((W + tw - 1) / tw) * ((H + th - 1) / th);
    if (best < 0 || tiles < best) { best = tiles; *TW = tw; *TH = th; }
  }
}

int tapconv_launch(const cocos_tapconv_desc* d, cudaStream_t stream) {
  if (!d || !d->x || !d->w || !d->y) {
    set_error("tapconv: null pointer argument");
    return -1;
  }
  const int s = d->a_stride;
  if (d->B <= 0 || d->H <= 0 || d->W <= 0 || d->Hin <= 0 || d->Win <= 0 || d->Ca <= 0 || (d->Ca % 8) || d->Cout <= 0 ||
      (s != 1 && s != 2) || (s == 2 && ((d->Hin | d->Win) & 1)) || d->ngroups <= 0 || d->ngroups > MAXG ||
      d->kchunks <= 0 || d->y_kind < 0 || d->y_kind > 3 || d->y_pad < 0 || d->y_Cs <= 0 ||
      (d->y_reflect && (d->y_pad >= d->y_H || d->y_pad >= d->y_W)) ||
      d->y_sh <= 0 || d->y_sw <= 0 || d->act < 0 || d->act > 3 || (d->res && d->res_kind != 1 && d->res_kind != 3) ||
      (d->res && (d->y_sh != 1 || d->y_sw != 1 || d->y_oh || d->y_ow)) || (d->y_lo_off && d->y_kind != 1) ||
      (d->y_kind == 0 && (d->y_pad || d->y_lo_off))) {
    set_error("tapconv: bad descriptor (B=%d H=%d W=%d Hin=%d Win=%d Ca=%d Cout=%d stride=%d groups=%d kchunks=%d "
              "y_kind=%d y_pad=%d)", d->B, d->H, d->W, d->Hin, d->Win, d->Ca, d->Cout, s, d->ngroups, d->kchunks,
              d->y_kind, d->y_pad);
    return -1;
  }
  TapParams p;
  p.B = d->B; p.H = d->H; p.W = d->W; p.Cout = d->Cout;
  tapconv_tile_shape(d->B, d->H, d->W, &p.TB, &p.TH, &p.TW);
  p.tiles_b = (d->B + p.TB - 1) / p.TB;
  p.tiles_h = (d->H + p.TH - 1) / p.TH;
  p.tiles_w = (d->W + p.TW - 1) / p.TW;
  const int BN = d->mod_W ? 2 * d->mod_W : (d->Cout > 128 ? 256 : 128);
  p.tiles_n = (d->Cout + BN - 1) / BN;
  p.num_tiles = p.tiles_b * p.tiles_h * p.tiles_w * p.tiles_n;
  p.a_stride = s; p.Ca = d->Ca; p.bf16 = d->bf16;
  p.ngroups = d->ngroups; p.kchunks = d->kchunks;
  for (int g = 0; g < d->ngroups; ++g) {
    p.dh[g] = d->dh[g]; p.dw[g] = d->dw[g]; p.coff[g] = d->coff[g];
    if (d->coff[g] < 0 || (d->coff[g] % 8)) {
      set_error("tapconv: channel offset of group %d (%d) must be a non-negative multiple of 8", g, d->coff[g]);
      return -1;
    }
  }
  p.scale = d->scale; p.bias = d->bias; p.res = d->res; p.res_kind = d->res_kind; p.res_Cs = d->res_Cs;
  p.act = d->act; p.slope = d->slope;
  p.y = d->y; p.y_kind = d->y_kind; p.y_H = d->y_H; p.y_W = d->y_W; p.y_Cs = d->y_Cs; p.y_coff = d->y_coff;
  p.y_lo_off = d->y_lo_off; p.y_pad = d->y_pad; p.y_reflect = d->y_reflect;
  p.y_sh = d->y_sh; p.y_sw = d->y_sw; p.y_oh = d->y_oh; p.y_ow = d->y_ow;
  p.mod_W = d->mod_W; p.mod_x = d->mod_x; p.mod_x_kind = d->mod_x_kind; p.mod_x_Cs = d->mod_x_Cs;
  p.mod_mean = d->mod_mean; p.mod_rstd = d->mod_rstd; p.gb = d->gb; p.gb_kind = d->gb_kind; p.gb_Cs = d->gb_Cs;
  if (d->mod_W) {
    const int C = d->Cout / 2;
    if ((d->mod_W != 64 && d->mod_W != 128) || (d->Cout % (2 * d->mod_W)) || (d->mod_W == 64 && C != 64) || !d->mod_x ||
        !d->mod_mean || !d->mod_rstd || (d->mod_x_kind != 1 && d->mod_x_kind != 3) || (d->mod_x_Cs % 8) || d->y_kind != 1 ||
        (d->y_Cs % 8) || (d->y_lo_off % 8) || d->y_coff || d->res || d->act != 2 || d->y_sh != 1 || d->y_sw != 1 ||
        d->y_oh || d->y_ow || d->H != d->y_H || d->W != d->y_W ||
        (d->gb && ((d->gb_kind != 1 && d->gb_kind != 3) || (d->gb_Cs % 8) || d->gb_Cs < d->Cout))) {
      set_error("tapconv: bad SPADE-epilogue descriptor (Cout=%d mod_W=%d x_kind=%d y_kind=%d act=%d)", d->Cout, d->mod_W,
                d->mod_x_kind, d->y_kind, d->act);
      return -1;
    }
  }
  if ((d->H - 1) * d->y_sh + d->y_oh >= d->y_H || (d->W - 1) * d->y_sw + d->y_ow >= d->y_W) {
    set_error("tapconv: output pixels fall outside y (%dx%d into %dx%d)", d->H, d->W, d->y_H, d->y_W);
    return -1;
  }
  CUtensorMap tm_x, tm_w;
  int rc;
  {
    // [B, Hin/s, s, Win/s, s*Ca]: innermost = (column parity, channel)
    const uint64_t Ca = (uint64_t)d->Ca, Win = (uint64_t)d->Win, Hin = (uint64_t)d->Hin;
    const uint64_t dims[5] = {Ca * s, Win / s, (uint64_t)s, Hin / s, (uint64_t)d->B};
    const uint64_t pitches[4] = {Ca * s * 2, Win * Ca * 2, Win * Ca * s * 2, Hin * Win * Ca * 2};
    const uint32_t box[5] = {BK, (uint32_t)p.TW, 1, (uint32_t)p.TH, (uint32_t)p.TB};
    if ((rc = make_tmap_16_5d(&tm_x, d->x, dims, pitches, box))) return rc;
  }
  const uint64_t Kt = (uint64_t)d->ngroups * d->kchunks * BK;
  const uint64_t wrows = (uint64_t)(d->w_rows >= d->Cout ? d->w_rows : d->Cout);
  if ((rc = make_tmap_f16_3d(&tm_w, d->w, Kt, wrows, 1, Kt * 2, wrows * Kt * 2, BK, BN, 1))) return rc;
  const int smem_bytes = SMEM_BYTES;
  const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
  if (BN == 256) {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(tapconv_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    tapconv_kernel<256><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_x, tm_w, p);
  } else {
    COCOS_CUDA_CHECK(cudaFuncSetAttribute(tapconv_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    tapconv_kernel<128><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_x, tm_w, p);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
