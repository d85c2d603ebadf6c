// K1 backward, stage A: recompute the correlation tile by tile and emit the
// softmax-Jacobian product
//     dS[i,j] = P[i,j] * (dP[i,j] - D[i]) * scale,   P = exp(scale*S - lse),
//     dP = dO V^T,  D[i] = sum_c dO[c,i] O[c,i]
// as bf16 (dO enters row-scaled in fp16, the scale is divided back out) in BOTH
// orientations -- dS [B,Nq,Nkp] and dS^T [B,Nk,Nqp] -- plus optionally P^T.
// Two plain wgmma GEMMs (gemm.cu) then give dQ^T = K^T-major x dS and
// dK^T = Q^T-major x dS^T; a third gives dV from P^T.  This is what autograd
// does through reference correspondence.py:291-318, without keeping the three
// fp32 N x N tensors alive.
//
// CTA = 128 query rows, streams 128-key tiles.  warp 8: TMA, warps 0-7: two
// warpgroups of 64 query rows; S and dP by wgmma into registers, the softmax
// Jacobian on the accumulator fragments, dS staged through one smem tile.
//
// Two shared-memory plans.  Resident (Cvk <= 192): the CTA's dO tile stays in smem, each key tile's V tile is loaded
// whole.  Streamed (Cvk > 192, where dO + V no longer fit beside a 2-stage ring): the 64-channel atoms of dO and V go
// through the same ring as the Q / K atoms, [dO atom | V atom] after the tile's [Q atom | K atom] stages, and
// dP = dO V^T is a longer wgmma K loop accumulated in registers.  dS, dS^T and P^T are written once per tile either way.
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

#include <cuda_bf16.h>

namespace cocos {

namespace {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int ATOM_BYTES = 128 * BK * 2;
constexpr int NUM_THREADS = 32 * CONSUMER_WARPS + 32;
constexpr int CT = 32 * CONSUMER_WARPS;  // consumer threads
constexpr int MAX_STAGES = 5;
constexpr int MAX_RESIDENT_STAGES = 4;
constexpr int TPITCH = 136;                     // staging tile pitch (fp16 elements)
constexpr int TILE_BYTES = 128 * TPITCH * 2;    // 34816

struct BwdParams {
  int B, Nq, Nk, Kd, Cv, Cvk;
  int kc_count, vc_count, n_tiles, ns;
  int Nkp, Nqp;
  float scale, scale_log2;
  const __half* do16;  // [B, Nq, Cvk] row-scaled dO (the dP operand)
  const float* rscale; // [B, Nq] the row scale r_i applied to dO
  const float* out;    // [B, Cv, Nq]
  const float* lse;    // [B, Nq]
  uint16_t* ds;        // bf16 [B, Nq, Nkp]
  uint16_t* dst;       // bf16 [B, Nk, Nqp]
  uint16_t* pt;        // bf16 [B, Nk, Nqp] or null
};

struct BwdBars {
  uint64_t do_full;
  uint64_t k_full[MAX_STAGES];
  uint64_t k_empty[MAX_STAGES];
  uint64_t v_full;
  uint64_t v_empty;
};

__device__ __forceinline__ void wg_sync() { bar_sync(1, CT); }

// copy a staged 128x128 fp16 tile (pitch TPITCH) to global rows of pitch `gpitch`
__device__ __forceinline__ uint32_t pack_bf2(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ void copy_tile_out(const uint8_t* tile, uint16_t* gbase, int gpitch, int valid_rows,
                                              int valid_cols, int tid) {
  const int chunk = tid & 15;
  if (chunk * 8 >= valid_cols) return;
#pragma unroll 4
  for (int it = 0; it < 128 / (CT / 16); ++it) {
    const int r = (tid >> 4) + it * (CT / 16);
    if (r < valid_rows) {
      const uint4 v = *reinterpret_cast<const uint4*>(tile + (r * TPITCH + chunk * 8) * 2);
      *reinterpret_cast<uint4*>(gbase + static_cast<size_t>(r) * gpitch + chunk * 8) = v;
    }
  }
}

// STREAM: the streamed plan (dO / V atoms through the ring) instead of the resident one
template <bool STREAM>
__global__ void __launch_bounds__(NUM_THREADS, 1)
corr_bwd_ds_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                   const __grid_constant__ CUtensorMap tm_do, const __grid_constant__ CUtensorMap tm_v,
                   const BwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * BM, bidx = blockIdx.y;
  const int T = p.n_tiles;

  const uint32_t stage_bytes = 2 * ATOM_BYTES;                 // [Q chunk | K chunk] (streamed: or [dO | V])
  const uint32_t op_bytes = STREAM ? 0 : p.vc_count * ATOM_BYTES;  // resident dO tile / V tile
  const uint32_t k_ring = smem0;
  const uint32_t do_smem = k_ring + p.ns * stage_bytes;
  const uint32_t v_smem = do_smem + op_bytes;
  const uint32_t stg_off = (v_smem + op_bytes) - smem0;        // staging tiles A, B
  uint8_t* tile = smem_gen + stg_off;  // one staging tile, reused for dS, dS^T (and P^T)
  BwdBars* bars = reinterpret_cast<BwdBars*>(tile + TILE_BYTES);

  if (tid == 0) {
    mbar_init(smem_u32(&bars->do_full), 1);
    for (int i = 0; i < p.ns; ++i) {
      mbar_init(smem_u32(&bars->k_full[i]), 1);
      mbar_init(smem_u32(&bars->k_empty[i]), CONSUMER_WARPS);
    }
    mbar_init(smem_u32(&bars->v_full), 1);
    mbar_init(smem_u32(&bars->v_empty), CONSUMER_WARPS);
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_do);
    tma_prefetch_desc(&tm_v);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    if (lane == 0) {
      if constexpr (!STREAM) {
        mbar_expect_tx(smem_u32(&bars->do_full), op_bytes);
        for (int vc = 0; vc < p.vc_count; ++vc)
          tma_load_3d(do_smem + vc * ATOM_BYTES, &tm_do, smem_u32(&bars->do_full), vc * BK, q0, bidx);
      }
      uint32_t ks = 0, kph = 0;
      for (int j = 0; j < T; ++j) {
        for (int kc = 0; kc < p.kc_count; ++kc) {
          mbar_wait(smem_u32(&bars->k_empty[ks]), kph ^ 1);
          const uint32_t full = smem_u32(&bars->k_full[ks]);
          mbar_expect_tx(full, stage_bytes);
          tma_load_3d(k_ring + ks * stage_bytes, &tm_q, full, kc * BK, q0, bidx);
          tma_load_3d(k_ring + ks * stage_bytes + ATOM_BYTES, &tm_k, full, kc * BK, j * BN, bidx);
          if (++ks == static_cast<uint32_t>(p.ns)) { ks = 0; kph ^= 1; }
        }
        if constexpr (STREAM) {
          for (int vc = 0; vc < p.vc_count; ++vc) {
            mbar_wait(smem_u32(&bars->k_empty[ks]), kph ^ 1);
            const uint32_t full = smem_u32(&bars->k_full[ks]);
            mbar_expect_tx(full, stage_bytes);
            tma_load_3d(k_ring + ks * stage_bytes, &tm_do, full, vc * BK, q0, bidx);
            tma_load_3d(k_ring + ks * stage_bytes + ATOM_BYTES, &tm_v, full, vc * BK, j * BN, bidx);
            if (++ks == static_cast<uint32_t>(p.ns)) { ks = 0; kph ^= 1; }
          }
        } else {
          mbar_wait(smem_u32(&bars->v_empty), (j & 1) ^ 1);
          mbar_expect_tx(smem_u32(&bars->v_full), op_bytes);
          for (int vc = 0; vc < p.vc_count; ++vc)
            tma_load_3d(v_smem + vc * ATOM_BYTES, &tm_v, smem_u32(&bars->v_full), vc * BK, j * BN, bidx);
        }
      }
    }
    __syncwarp();
    return;
  }

  const int wg = tid >> 7, t = tid & 127;
  const int r0 = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);  // fragment rows r0, r0 + 8
  const int cq = 2 * (t & 3);
  const uint32_t a_off = wg * 64 * 128;
  const float c2 = p.scale_log2;
  // D'[i] = sum_c dO'[i,c] * O[c,i] with the SAME fp16-rounded, row-scaled dO' the dP MMA consumes, so
  // that sum_j P[i,j] (dP'[i,j] - D'[i]) cancels to rounding noise instead of to an fp16-vs-fp32 bias.
  float lse2[2], dsum[2], gs[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + r0 + 8 * r;
    lse2[r] = INFINITY; dsum[r] = 0.f; gs[r] = 0.f;
    if (q < p.Nq) {
      lse2[r] = p.lse[static_cast<size_t>(bidx) * p.Nq + q] * 1.4426950408889634f;
      const __half* drow = p.do16 + (static_cast<size_t>(bidx) * p.Nq + q) * p.Cvk;
      for (int c = 0; c < p.Cv; ++c)
        dsum[r] = fmaf(__half2float(drow[c]), p.out[(static_cast<size_t>(bidx) * p.Cv + c) * p.Nq + q], dsum[r]);
      gs[r] = p.scale / p.rscale[static_cast<size_t>(bidx) * p.Nq + q];  // undo the row scale: true dS in bf16
    }
  }
  const int valid_rows = min(BM, p.Nq - q0);
  if constexpr (!STREAM) mbar_wait(smem_u32(&bars->do_full), 0);

  uint32_t ks = 0, kph = 0;
  for (int j = 0; j < T; ++j) {
    const int valid_cols = min(BN, p.Nk - j * BN);
    float s[BN / 2], dp[BN / 2];
    for (int kc = 0; kc < p.kc_count; ++kc) {
      mbar_wait_quiet(smem_u32(&bars->k_full[ks]), kph);
      const uint32_t a_addr = k_ring + ks * stage_bytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<BN, false>(s, desc_advance_k16(make_desc_k_sw128(a_addr + a_off), k),
                            desc_advance_k16(make_desc_k_sw128(a_addr + ATOM_BYTES), k), (kc | k) != 0 ? 1 : 0, 0);
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars->k_empty[ks]));
      if (++ks == static_cast<uint32_t>(p.ns)) { ks = 0; kph ^= 1; }
    }
    if constexpr (STREAM) {
      for (int vc = 0; vc < p.vc_count; ++vc) {
        mbar_wait_quiet(smem_u32(&bars->k_full[ks]), kph);
        const uint32_t st = k_ring + ks * stage_bytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss<BN, false>(dp, desc_advance_k16(make_desc_k_sw128(st + a_off), k),
                              desc_advance_k16(make_desc_k_sw128(st + ATOM_BYTES), k), (vc | k) != 0 ? 1 : 0, 0);
        wgmma_commit();
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars->k_empty[ks]));
        if (++ks == static_cast<uint32_t>(p.ns)) { ks = 0; kph ^= 1; }
      }
    } else {
      mbar_wait_quiet(smem_u32(&bars->v_full), j & 1);
      wgmma_fence();
      for (int vc = 0; vc < p.vc_count; ++vc) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_ss<BN, false>(dp, desc_advance_k16(make_desc_k_sw128(do_smem + vc * ATOM_BYTES + a_off), k),
                              desc_advance_k16(make_desc_k_sw128(v_smem + vc * ATOM_BYTES), k), (vc | k) != 0 ? 1 : 0,
                              0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars->v_empty));
    }

    // fragment element i: row r0 + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + cq + (i & 1)
    uint32_t dsp[BN / 4];  // bf16 pairs (i, i + 1) for even i
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int r = (i >> 1) & 1, col = 8 * (i >> 2) + cq + (i & 1);
      const float pv = ex2(fmaf(s[i], c2, -lse2[r]));
      s[i] = (col < valid_cols) ? pv : 0.f;
    }
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int r = (i >> 1) & 1;
      dsp[i >> 1] = pack_bf2(s[i] * (dp[i] - dsum[r]) * gs[r], s[i + 1] * (dp[i + 1] - dsum[r]) * gs[r]);
    }

    // stage dS row-major, then transposed, (then P^T) through one smem tile
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + cq;
      *reinterpret_cast<uint32_t*>(tile + (row * TPITCH + col) * 2) = dsp[i >> 1];
    }
    wg_sync();
    copy_tile_out(tile, p.ds + (static_cast<size_t>(bidx) * p.Nq + q0) * p.Nkp + j * BN, p.Nkp, valid_rows,
                  valid_cols, tid);
    wg_sync();
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + cq;
      *reinterpret_cast<uint16_t*>(tile + (col * TPITCH + row) * 2) = static_cast<uint16_t>(dsp[i >> 1] & 0xFFFF);
      *reinterpret_cast<uint16_t*>(tile + ((col + 1) * TPITCH + row) * 2) = static_cast<uint16_t>(dsp[i >> 1] >> 16);
    }
    wg_sync();
    copy_tile_out(tile, p.dst + (static_cast<size_t>(bidx) * p.Nk + j * BN) * p.Nqp + q0, p.Nqp, valid_cols,
                  valid_rows, tid);
    wg_sync();
    if (p.pt != nullptr) {
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + cq;
        const uint32_t h = pack_bf2(s[i], s[i + 1]);
        *reinterpret_cast<uint16_t*>(tile + (col * TPITCH + row) * 2) = static_cast<uint16_t>(h & 0xFFFF);
        *reinterpret_cast<uint16_t*>(tile + ((col + 1) * TPITCH + row) * 2) = static_cast<uint16_t>(h >> 16);
      }
      wg_sync();
      copy_tile_out(tile, p.pt + (static_cast<size_t>(bidx) * p.Nk + j * BN) * p.Nqp + q0, p.Nqp, valid_cols,
                    valid_rows, tid);
      wg_sync();
    }
  }
}

}  // namespace

int corr_bwd_ds_launch(const void* q, const void* k, const void* do16, const void* v16, const float* rscale,
                       const float* out, const float* lse, void* ds, void* dst, void* pt, int B, int Nq, int Nk,
                       int Kd, int Cv, int Cvk, int Nkp, int Nqp, float scale, cudaStream_t stream) {
  if (B <= 0 || Nq <= 0 || Nk <= 0 || Kd <= 0 || (Kd % BK) || Cvk <= 0 || (Cvk % BK) || Cv <= 0 || Cv > Cvk) {
    set_error("corr_bwd_ds: bad shape (B=%d Nq=%d Nk=%d Kd=%d Cv=%d Cvk=%d)", B, Nq, Nk, Kd, Cv, Cvk);
    return -1;
  }
  if (Nkp < Nk || Nqp < Nq || (Nkp % 8) || (Nqp % 8)) {
    set_error("corr_bwd_ds: pitches must be >= extent and multiples of 8 (Nkp=%d Nqp=%d)", Nkp, Nqp);
    return -1;
  }
  BwdParams p;
  p.B = B; p.Nq = Nq; p.Nk = Nk; p.Kd = Kd; p.Cv = Cv; p.Cvk = Cvk;
  p.kc_count = Kd / BK; p.vc_count = Cvk / BK; p.n_tiles = (Nk + BN - 1) / BN;
  p.Nkp = Nkp; p.Nqp = Nqp;
  p.scale = scale; p.scale_log2 = scale * 1.4426950408889634f;
  p.do16 = static_cast<const __half*>(do16); p.rscale = rscale; p.out = out; p.lse = lse;
  p.ds = static_cast<uint16_t*>(ds); p.dst = static_cast<uint16_t*>(dst); p.pt = static_cast<uint16_t*>(pt);
  // resident plan up to Cvk = 192 (dO and V tiles beside a ring of >= 2 stages); streamed beyond, where the ring
  // also carries the dO / V atoms and its depth no longer depends on Cvk
  const bool stream_vo = Cvk > 192;
  const int budget = 227 * 1024 - 1024 - 512;
  const int fixed = (stream_vo ? 0 : 2 * p.vc_count * ATOM_BYTES) + TILE_BYTES;
  p.ns = (budget - fixed) / (2 * ATOM_BYTES);
  if (p.ns > (stream_vo ? MAX_STAGES : MAX_RESIDENT_STAGES)) p.ns = stream_vo ? MAX_STAGES : MAX_RESIDENT_STAGES;
  if (p.ns < 2) {
    set_error("corr_bwd_ds: shared memory plan failed (Cvk=%d)", Cvk);
    return -1;
  }
  const int smem_bytes = 1024 + p.ns * 2 * ATOM_BYTES + fixed + 512;
  CUtensorMap tm_q, tm_k, tm_do, tm_v;
  int rc;
  if ((rc = make_tmap_f16_3d(&tm_q, q, Kd, Nq, B, (uint64_t)Kd * 2, (uint64_t)Nq * Kd * 2, BK, BM, 1))) return rc;
  if ((rc = make_tmap_f16_3d(&tm_k, k, Kd, Nk, B, (uint64_t)Kd * 2, (uint64_t)Nk * Kd * 2, BK, BN, 1))) return rc;
  if ((rc = make_tmap_f16_3d(&tm_do, do16, Cvk, Nq, B, (uint64_t)Cvk * 2, (uint64_t)Nq * Cvk * 2, BK, BM, 1)))
    return rc;
  if ((rc = make_tmap_f16_3d(&tm_v, v16, Cvk, Nk, B, (uint64_t)Cvk * 2, (uint64_t)Nk * Cvk * 2, BK, BN, 1)))
    return rc;
  auto kernel = stream_vo ? corr_bwd_ds_kernel<true> : corr_bwd_ds_kernel<false>;
  COCOS_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  dim3 grid((Nq + BM - 1) / BM, B);
  kernel<<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_q, tm_k, tm_do, tm_v, p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // namespace cocos
