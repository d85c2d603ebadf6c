#include "tmap.h"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace cocos {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

int workspace_check(float* ws, long long* ws_floats, long long need, const char* what) {
  if (!ws_floats) {
    set_error("%s: null workspace size pointer", what);
    return -1;
  }
  if (!ws) {
    *ws_floats = need;
    return 1;
  }
  if (*ws_floats < need) {
    set_error("%s: workspace of %lld floats, %lld needed", what, *ws_floats, need);
    return -1;
  }
  return 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        n <= 0)
      n = 132;
  }
  return n;
}

namespace {
// few partials per output (split-K slices): one thread per output adds them in order
__global__ void __launch_bounds__(256)
ordered_sum_kernel(const float* __restrict__ part, int nparts, long long n, float* __restrict__ out, int accumulate) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * 256) {
    float t = 0.f;
    for (int p = 0; p < nparts; ++p) t += part[p * n + i];
    out[i] = accumulate ? out[i] + t : t;
  }
}
// many partials per output (per-block statistics, losses): one block per output, thread k adds partials k, k + 256, ...
// and a fixed tree combines the 256 sums
__global__ void __launch_bounds__(256)
ordered_sum_wide_kernel(const float* __restrict__ part, int nparts, long long n, float* __restrict__ out,
                        int accumulate) {
  __shared__ float red[256];
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    float t = 0.f;
    for (int p = threadIdx.x; p < nparts; p += 256) t += part[p * n + i];
    red[threadIdx.x] = t;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[i] = accumulate ? out[i] + red[0] : red[0];
    __syncthreads();
  }
}
}  // namespace

int ordered_sum(const float* part, int nparts, long long n, float* out, int accumulate, cudaStream_t stream) {
  if (nparts > 32) {
    const long long blocks = n < num_sms() * 8ll ? n : num_sms() * 8ll;
    ordered_sum_wide_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(part, nparts, n, out, accumulate);
  } else {
    long long blocks = (n + 255) / 256;
    if (blocks > num_sms() * 8ll) blocks = num_sms() * 8ll;
    ordered_sum_kernel<<<static_cast<int>(blocks), 256, 0, stream>>>(part, nparts, n, out, accumulate);
  }
  COCOS_CUDA_CHECK(cudaGetLastError());
  return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int make_tmap_f16_3d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t pitch1,
                     uint64_t pitch2, uint32_t b0, uint32_t b1, uint32_t b2) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -3;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitch1 & 15) || (pitch2 & 15)) {
    set_error("tensor map: base/pitches must be 16-byte aligned (base=%p pitch1=%llu pitch2=%llu)", base,
              (unsigned long long)pitch1, (unsigned long long)pitch2);
    return -1;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {pitch1, pitch2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  static const int promo = [] {
    const char* e = getenv("COCOS_TMA_L2PROMO");
    return e ? atoi(e) : 256;
  }();
  const CUtensorMapL2promotion l2p = promo == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE
                                     : promo == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                                     : promo == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                                                    : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2p, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: CUresult %d (dims %llu,%llu,%llu box %u,%u,%u)", (int)r,
              (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, b0, b1, b2);
    return -3;
  }
  return 0;
}

int make_tmap_f16_4d(CUtensorMap* map, const void* base, const uint64_t dims[4], const uint64_t pitches[3],
                     const uint32_t box[4]) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -3;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitches[0] & 15) || (pitches[1] & 15) || (pitches[2] & 15)) {
    set_error("tensor map (4d): base/pitches must be 16-byte aligned");
    return -1;
  }
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t st[3] = {pitches[0], pitches[1], pitches[2]};
  cuuint32_t bx[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t es[4] = {1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), d, st, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(4d) failed: CUresult %d (dims %llu,%llu,%llu,%llu box %u,%u,%u,%u)", (int)r,
              (unsigned long long)d[0], (unsigned long long)d[1], (unsigned long long)d[2], (unsigned long long)d[3],
              bx[0], bx[1], bx[2], bx[3]);
    return -3;
  }
  return 0;
}

int make_tmap_16_5d(CUtensorMap* map, const void* base, const uint64_t dims[5], const uint64_t pitches[4],
                    const uint32_t box[5]) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -3;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitches[0] & 15) || (pitches[1] & 15) || (pitches[2] & 15) ||
      (pitches[3] & 15)) {
    set_error("tensor map (5d): base/pitches must be 16-byte aligned");
    return -1;
  }
  cuuint64_t d[5] = {dims[0], dims[1], dims[2], dims[3], dims[4]};
  cuuint64_t st[4] = {pitches[0], pitches[1], pitches[2], pitches[3]};
  cuuint32_t bx[5] = {box[0], box[1], box[2], box[3], box[4]};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(base), d, st, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(5d) failed: CUresult %d (dims %llu,%llu,%llu,%llu,%llu box %u,%u,%u,%u,%u)", (int)r,
              (unsigned long long)d[0], (unsigned long long)d[1], (unsigned long long)d[2], (unsigned long long)d[3],
              (unsigned long long)d[4], bx[0], bx[1], bx[2], bx[3], bx[4]);
    return -3;
  }
  return 0;
}

int make_tmap_f32_3d_plain(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t pitch1,
                           uint64_t pitch2, uint32_t b0, uint32_t b1, uint32_t b2) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return -3;
  if ((reinterpret_cast<uintptr_t>(base) & 15) || (pitch1 & 15) || (pitch2 & 15)) {
    set_error("tensor map (fp32): base/pitches must be 16-byte aligned");
    return -1;
  }
  cuuint64_t dims[3] = {d0, d1, d2};
  cuuint64_t strides[2] = {pitch1, pitch2};
  cuuint32_t box[3] = {b0, b1, b2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(fp32) failed: CUresult %d", (int)r);
    return -3;
  }
  return 0;
}

}  // namespace cocos
