// K1: fused correlation -> softmax -> warp for sm_90a.
//
//   O[b,c,i] = sum_j softmax_j(scale * <Q[b,i,:], K[b,j,:]>) * V[b,j,c]
//
// Replaces reference correspondence.py:291 (matmul theta^T phi), :304
// (/temperature), :307 (row softmax) and :318/:334 (matmul with the exemplar /
// its mask) without ever writing the HWxHW matrix to HBM.
//
// One CTA owns 128 query rows and streams 64-key tiles:
//   warp 8   : TMA producer (Q once or chunk-streamed, K chunks, V tiles)
//   warps 0-7: two warpgroups of 64 query rows each.  S = Q K^T by wgmma into registers, online softmax on the
//              accumulator fragments (row max / sum over the 4 threads sharing a row), then
//              * PVN > 0: O += P V by wgmma with P as the fp16 register operand (O in registers, N = PVN >= Cvp);
//              * CV > 0 (Cv <= 4 value channels, fp32 V): P V on the CUDA cores inside the exp loop, P and V stay
//                fp32 (no fp16 rounding of the probabilities).
// More than 256 padded value channels (a TMA box and a wgmma N stop at 256): V is split into chunks of 256 rows along
// grid z, each CTA recomputes S and the online softmax for its chunk, and a second launch takes a partial last chunk
// with the PVN that fits it.  lse (and the raw logits) come from chunk 0 only.
#include "corr_kernels.h"
#include "ptx.cuh"
#include "tmap.h"

#include <stdlib.h>

namespace cocos {

namespace {

constexpr int BM = 128;  // queries per CTA
constexpr int BN = 64;   // keys per tile
constexpr int BK = 64;   // 16-bit elements per 128B swizzle atom row
constexpr int Q_ATOM = BM * BK * 2;  // 16 KiB: 128 rows x 64 fp16
constexpr int K_ATOM = BN * BK * 2;  // 8 KiB: 64 rows x 64 fp16
constexpr int NUM_THREADS = 32 * CONSUMER_WARPS + 32;
constexpr int MAX_KSTAGES = 8;
constexpr int MAX_VSTAGES = 2;
constexpr int VCHUNK = 256;  // value rows per chunk: the TMA box limit and the widest wgmma N

struct FwdParams {
  int B, Nq, Nk, Kd, Cv, Cvp;
  int kc_count;    // Kd / 64
  int n_tiles;     // ceil(Nk / 64)
  int q_resident;  // Q tile kept in smem for the whole CTA
  int ns_k, ns_v;
  int v_stage;     // bytes per V stage
  int v_rows;      // value rows per chunk (the V box), <= PVN
  int c0;          // first value row of chunk blockIdx.z == 0; chunk z starts at c0 + z * VCHUNK
  float scale, scale_log2;
  float* out;   // [B, Cv, Nq]
  float* lse;   // [B, Nq] (natural log) or null
  float* corr;  // [B, Nq, Nk] scaled logits or null (return_corr / debug)
};

struct Barriers {
  uint64_t q_full;
  uint64_t k_full[MAX_KSTAGES];
  uint64_t k_empty[MAX_KSTAGES];
  uint64_t v_full[MAX_VSTAGES];
  uint64_t v_empty[MAX_VSTAGES];
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// PVN: wgmma N of the P V product (tensor path) or 0; CV: value channels of the CUDA-core path or 0
template <int PVN, int CV>
__global__ void __launch_bounds__(NUM_THREADS, 1)
corr_fwd_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                const __grid_constant__ CUtensorMap tm_v, const FwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment for the 128B swizzle atoms
  const uint32_t smem0 = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem0 - smem_u32(smem_raw));

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int q0 = blockIdx.x * BM;
  const int bidx = blockIdx.y;
  const int cbase = p.c0 + blockIdx.z * VCHUNK;

  const uint32_t stage_bytes = p.q_resident ? K_ATOM : Q_ATOM + K_ATOM;
  const uint32_t q_smem = smem0;
  const uint32_t k_ring = q_smem + (p.q_resident ? p.kc_count * Q_ATOM : 0);
  const uint32_t v_ring = k_ring + p.ns_k * stage_bytes;
  const uint32_t bar_off = v_ring + p.ns_v * p.v_stage - smem0;
  Barriers* bars = reinterpret_cast<Barriers*>(smem_gen + ((bar_off + 7) & ~7u));

  if (tid == 0) {
    mbar_init(smem_u32(&bars->q_full), 1);
    for (int i = 0; i < p.ns_k; ++i) {
      mbar_init(smem_u32(&bars->k_full[i]), 1);
      mbar_init(smem_u32(&bars->k_empty[i]), CONSUMER_WARPS);
    }
    for (int i = 0; i < p.ns_v; ++i) {
      mbar_init(smem_u32(&bars->v_full[i]), 1);
      mbar_init(smem_u32(&bars->v_empty[i]), CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  if (warp == CONSUMER_WARPS && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
  }
  __syncthreads();
  const int T = p.n_tiles;

  if (warp == CONSUMER_WARPS) {
    // ------------------------------------------------------------ TMA producer
    if (lane == 0) {
      if (p.q_resident) {
        mbar_expect_tx(smem_u32(&bars->q_full), p.kc_count * Q_ATOM);
        for (int kc = 0; kc < p.kc_count; ++kc)
          tma_load_3d(q_smem + kc * Q_ATOM, &tm_q, smem_u32(&bars->q_full), kc * BK, q0, bidx);
      }
      const uint32_t v_bytes = PVN ? static_cast<uint32_t>(p.v_rows) * BN * 2 : static_cast<uint32_t>(CV) * BN * 4;
      uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
      for (int j = 0; j < T; ++j) {
        for (int kc = 0; kc < p.kc_count; ++kc) {
          mbar_wait(smem_u32(&bars->k_empty[ks]), kph ^ 1);
          const uint32_t full = smem_u32(&bars->k_full[ks]);
          mbar_expect_tx(full, stage_bytes);
          uint32_t dst = k_ring + ks * stage_bytes;
          if (!p.q_resident) {
            tma_load_3d(dst, &tm_q, full, kc * BK, q0, bidx);
            dst += Q_ATOM;
          }
          tma_load_3d(dst, &tm_k, full, kc * BK, j * BN, bidx);
          if (++ks == static_cast<uint32_t>(p.ns_k)) { ks = 0; kph ^= 1; }
        }
        mbar_wait(smem_u32(&bars->v_empty[vs]), vph ^ 1);
        const uint32_t vfull = smem_u32(&bars->v_full[vs]);
        mbar_expect_tx(vfull, v_bytes);
        tma_load_3d(v_ring + vs * p.v_stage, &tm_v, vfull, j * BN, cbase, bidx);
        if (++vs == static_cast<uint32_t>(p.ns_v)) { vs = 0; vph ^= 1; }
      }
    }
    __syncwarp();
    return;
  }

  // ------------------------------------------------- softmax warpgroups (warps 0..7)
  const int wg = tid >> 7, t = tid & 127;
  const int r0 = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2);  // fragment rows r0 and r0 + 8
  const int cq = 2 * (t & 3);                                 // fragment column offset
  const float c2 = p.scale_log2;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  constexpr int ON = PVN ? PVN / 2 : 1;
  float o[ON];
  float oc[2][CV > 0 ? CV : 1];
#pragma unroll
  for (int i = 0; i < ON; ++i) o[i] = 0.f;
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int c = 0; c < (CV > 0 ? CV : 1); ++c) oc[r][c] = 0.f;

  if (p.q_resident) mbar_wait(smem_u32(&bars->q_full), 0);
  uint32_t ks = 0, kph = 0, vs = 0, vph = 0;
  for (int j = 0; j < T; ++j) {
    float s[BN / 2];
    for (int kc = 0; kc < p.kc_count; ++kc) {
      mbar_wait_quiet(smem_u32(&bars->k_full[ks]), kph);
      const uint32_t st = k_ring + ks * stage_bytes;
      const uint32_t a_addr = (p.q_resident ? (q_smem + kc * Q_ATOM) : st) + wg * 64 * 128;
      const uint32_t b_addr = p.q_resident ? st : (st + Q_ATOM);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<BN, false>(s, desc_advance_k16(make_desc_k_sw128(a_addr), k),
                            desc_advance_k16(make_desc_k_sw128(b_addr), k), (kc | k) != 0 ? 1 : 0, 0);
      wgmma_commit();
      wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars->k_empty[ks]));
      if (++ks == static_cast<uint32_t>(p.ns_k)) { ks = 0; kph ^= 1; }
    }

    const int kbase = j * BN + cq;
    if (p.corr != nullptr && cbase == 0) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) {
        const int q = q0 + r0 + ((i >> 1) & 1) * 8, key = kbase + 8 * (i >> 2) + (i & 1);
        if (q < p.Nq && key < p.Nk) p.corr[(static_cast<size_t>(bidx) * p.Nq + q) * p.Nk + key] = s[i] * p.scale;
      }
    }
    if (j == T - 1 && (p.Nk % BN) != 0) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i)
        if (kbase + 8 * (i >> 2) + (i & 1) >= p.Nk) s[i] = -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float tmax = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) tmax = fmaxf(tmax, fmaxf(s[4 * jj + 2 * r], s[4 * jj + 2 * r + 1]));
      const float m_new = fmaxf(m[r], quad_max(tmax));  // finite: every tile has a valid key
      alpha[r] = ex2((m[r] - m_new) * c2);                // exact online softmax; 0 on the first tile
      m[r] = m_new;
      l[r] *= alpha[r];
    }
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int r = (i >> 1) & 1;
      s[i] = ex2(fmaf(s[i], c2, -m[r] * c2));
      l[r] += s[i];
    }
    mbar_wait_quiet(smem_u32(&bars->v_full[vs]), vph);
    if constexpr (PVN > 0) {
#pragma unroll
      for (int i = 0; i < ON; ++i) o[i] *= alpha[(i >> 1) & 1];
      const uint32_t vb = v_ring + vs * p.v_stage;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BN / 16; ++kk) {
        uint32_t a[4];
        a[0] = pack_h2(s[8 * kk + 0], s[8 * kk + 1]);
        a[1] = pack_h2(s[8 * kk + 2], s[8 * kk + 3]);
        a[2] = pack_h2(s[8 * kk + 4], s[8 * kk + 5]);
        a[3] = pack_h2(s[8 * kk + 6], s[8 * kk + 7]);
        wgmma_rs<PVN>(o, a, desc_advance_k16(make_desc_k_sw128(vb), kk), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
    } else {
      const float* vt = reinterpret_cast<const float*>(smem_gen + (v_ring - smem0) + vs * p.v_stage);
#pragma unroll
      for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < CV; ++c) oc[r][c] *= alpha[r];
#pragma unroll
      for (int jj = 0; jj < BN / 8; ++jj) {
#pragma unroll
        for (int c = 0; c < CV; ++c) {
          const float2 v = *reinterpret_cast<const float2*>(vt + c * BN + 8 * jj + cq);
#pragma unroll
          for (int r = 0; r < 2; ++r) oc[r][c] = fmaf(s[4 * jj + 2 * r], v.x, fmaf(s[4 * jj + 2 * r + 1], v.y, oc[r][c]));
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&bars->v_empty[vs]));
    if (++vs == static_cast<uint32_t>(p.ns_v)) { vs = 0; vph ^= 1; }
  }

  // epilogue: O / l -> out[b, c, q]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const float lt = quad_sum(l[r]);
    const float inv_l = 1.0f / lt;
    const int q = q0 + r0 + 8 * r;
    if constexpr (PVN > 0) {
      if (q < p.Nq) {
#pragma unroll
        for (int i = 0; i < ON; ++i) {
          if (((i >> 1) & 1) != r) continue;
          const int c = cbase + 8 * (i >> 2) + cq + (i & 1);
          if (c < p.Cv) p.out[(static_cast<size_t>(bidx) * p.Cv + c) * p.Nq + q] = o[i] * inv_l;
        }
      }
    } else {
#pragma unroll
      for (int c = 0; c < CV; ++c) {
        const float v = quad_sum(oc[r][c]);
        if (q < p.Nq && (t & 3) == c) p.out[(static_cast<size_t>(bidx) * p.Cv + c) * p.Nq + q] = v * inv_l;
      }
    }
    if (p.lse != nullptr && cbase == 0 && q < p.Nq && (t & 3) == 0)
      p.lse[static_cast<size_t>(bidx) * p.Nq + q] = (m[r] * c2 + log2f(lt)) * 0.6931471805599453f;
  }
}

template <int PVN, int CV>
int launch_fwd(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const CUtensorMap& tm_v, const FwdParams& p,
               int smem_bytes, cudaStream_t stream, int n_chunks = 1) {
  COCOS_CUDA_CHECK(
      cudaFuncSetAttribute(corr_fwd_kernel<PVN, CV>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
  dim3 grid((p.Nq + BM - 1) / BM, p.B, n_chunks);
  corr_fwd_kernel<PVN, CV><<<grid, NUM_THREADS, smem_bytes, stream>>>(tm_q, tm_k, tm_v, p);
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// shared memory plan (<= 227 KiB): [Q] [K ring] [V ring] [barriers]; sets q_resident / ns_k / ns_v from p.v_stage
int plan_smem(FwdParams& p) {
  const int budget = 227 * 1024 - 1024 /*alignment slack*/ - 512 /*barriers*/;
  p.q_resident = (p.Kd <= 256) ? 1 : 0;
  const int q_bytes = p.q_resident ? p.kc_count * Q_ATOM : 0;
  const int stage = p.q_resident ? K_ATOM : Q_ATOM + K_ATOM;
  p.ns_v = 2;
  p.ns_k = (budget - q_bytes - p.ns_v * p.v_stage) / stage;
  if (p.ns_k > MAX_KSTAGES) p.ns_k = MAX_KSTAGES;
  if (p.ns_k < 2) {
    set_error("corr_warp_fwd: shared memory plan failed (Kd=%d Cvp=%d)", p.Kd, p.Cvp);
    return -1;
  }
  return 1024 + q_bytes + p.ns_k * stage + p.ns_v * p.v_stage + 512;
}

// tensor-core P V over n_chunks chunks of `rows` value rows, the first at row c0
int launch_tensor_pv(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const void* vt, FwdParams p, int Nkp, int rows,
                     int c0, int n_chunks, cudaStream_t stream) {
  const int pvn = rows <= 64 ? 64 : rows <= 128 ? 128 : 256;
  // a V stage holds PVN rows of 64 keys (the wgmma reads PVN >= rows rows)
  p.v_stage = pvn * BN * 2;
  p.v_rows = rows;
  p.c0 = c0;
  const int smem_bytes = plan_smem(p);
  if (smem_bytes < 0) return -1;
  CUtensorMap tm_v;
  int rc;
  if ((rc = make_tmap_f16_3d(&tm_v, vt, p.Nk, p.Cvp, p.B, (uint64_t)Nkp * 2, (uint64_t)p.Cvp * Nkp * 2, BK, rows, 1)))
    return rc;
  if (pvn == 64) return launch_fwd<64, 0>(tm_q, tm_k, tm_v, p, smem_bytes, stream, n_chunks);
  if (pvn == 128) return launch_fwd<128, 0>(tm_q, tm_k, tm_v, p, smem_bytes, stream, n_chunks);
  return launch_fwd<256, 0>(tm_q, tm_k, tm_v, p, smem_bytes, stream, n_chunks);
}

}  // namespace

int corr_warp_fwd_launch(const void* q, const void* k, const void* vt, const float* v32, float* out, float* lse,
                         float* corr, int B, int Nq, int Nk, int Kd, int Cv, int Cvp, int Nkp, float scale,
                         cudaStream_t stream) {
  if (B <= 0 || Nq <= 0 || Nk <= 0) {
    set_error("corr_warp_fwd: empty problem (B=%d Nq=%d Nk=%d)", B, Nq, Nk);
    return -1;
  }
  if (Kd <= 0 || (Kd % BK) != 0) {
    set_error("corr_warp_fwd: Kd=%d must be a positive multiple of 64 (pad in the pack kernel)", Kd);
    return -1;
  }
  // Cv <= 4 with fp32 values: P V on the CUDA cores (no fp16 rounding of P); otherwise the tensor-core P V
  const bool cuda_pv = v32 != nullptr && corr == nullptr && Cv >= 1 && Cv <= 4 && (Nk % 4) == 0 &&
                       (reinterpret_cast<uintptr_t>(v32) & 15) == 0;
  if (!cuda_pv) {
    if (vt == nullptr) {
      set_error("corr_warp_fwd: packed fp16 values (vt) are required for this shape (Cv=%d)", Cv);
      return -1;
    }
    if (Cv <= 0 || Cvp < Cv || (Cvp % 16) != 0) {
      set_error("corr_warp_fwd: need 0 < Cv <= Cvp, Cvp %% 16 == 0 (Cv=%d Cvp=%d)", Cv, Cvp);
      return -1;
    }
    if (Cvp / VCHUNK > 65535) {
      set_error("corr_warp_fwd: Cvp=%d needs more than 65535 value chunks of %d", Cvp, VCHUNK);
      return -1;
    }
    if (Nkp < Nk || (Nkp % 8) != 0) {
      set_error("corr_warp_fwd: V row pitch Nkp=%d must be >= Nk=%d and a multiple of 8", Nkp, Nk);
      return -1;
    }
  }
  FwdParams p;
  p.B = B; p.Nq = Nq; p.Nk = Nk; p.Kd = Kd; p.Cv = Cv; p.Cvp = Cvp;
  p.kc_count = Kd / BK;
  p.n_tiles = (Nk + BN - 1) / BN;
  p.scale = scale;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.out = out; p.lse = lse; p.corr = corr;
  p.v_rows = Cvp;
  p.c0 = 0;

  CUtensorMap tm_q, tm_k;
  int rc;
  if ((rc = make_tmap_f16_3d(&tm_q, q, Kd, Nq, B, (uint64_t)Kd * 2, (uint64_t)Nq * Kd * 2, BK, BM, 1))) return rc;
  if ((rc = make_tmap_f16_3d(&tm_k, k, Kd, Nk, B, (uint64_t)Kd * 2, (uint64_t)Nk * Kd * 2, BK, BN, 1))) return rc;
  if (cuda_pv) {
    p.v_stage = 1024;  // Cv fp32 rows of 64 keys
    const int smem_bytes = plan_smem(p);
    if (smem_bytes < 0) return -1;
    CUtensorMap tm_v;
    if ((rc = make_tmap_f32_3d_plain(&tm_v, v32, Nk, Cv, B, (uint64_t)Nk * 4, (uint64_t)Cv * Nk * 4, BN, Cv, 1)))
      return rc;
    switch (Cv) {
      case 1: return launch_fwd<0, 1>(tm_q, tm_k, tm_v, p, smem_bytes, stream);
      case 2: return launch_fwd<0, 2>(tm_q, tm_k, tm_v, p, smem_bytes, stream);
      case 3: return launch_fwd<0, 3>(tm_q, tm_k, tm_v, p, smem_bytes, stream);
      default: return launch_fwd<0, 4>(tm_q, tm_k, tm_v, p, smem_bytes, stream);
    }
  }
  // up to 256 rows: one chunk, grid z = 1.  Beyond: every full chunk of 256 rows in one launch (grid z = chunk), then
  // the partial last chunk, if any, in a second launch with the PVN that fits it.  Each chunk recomputes S = Q K^T.
  const int n_full = Cvp > VCHUNK ? Cvp / VCHUNK : 0;
  const int tail = Cvp - n_full * VCHUNK;
  if (n_full > 0 && (rc = launch_tensor_pv(tm_q, tm_k, vt, p, Nkp, VCHUNK, 0, n_full, stream))) return rc;
  if (tail > 0 && (rc = launch_tensor_pv(tm_q, tm_k, vt, p, Nkp, tail, n_full * VCHUNK, 1, stream))) return rc;
  return 0;
}

}  // namespace cocos
