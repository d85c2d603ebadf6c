// Host-side helpers: CUtensorMap construction through the driver entry point
// (no -lcuda link dependency), error recording for the C-ABI.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cocos {

void set_error(const char* fmt, ...);
const char* get_error();

// fp16 tensor [d2][d1][d0] (d0 contiguous), row pitches in BYTES, box
// (b0,b1,b2) elements, 128B swizzle, OOB -> zero fill.
// Returns 0 on success.
int make_tmap_f16_3d(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t pitch1,
                     uint64_t pitch2, uint32_t b0, uint32_t b1, uint32_t b2);

// fp16 tensor [d3][d2][d1][d0] (d0 contiguous), pitches in BYTES, box (b0,b1,b2,b3), 128B swizzle, OOB -> zero.
int make_tmap_f16_4d(CUtensorMap* map, const void* base, const uint64_t dims[4], const uint64_t pitches[3],
                     const uint32_t box[4]);

// 16-bit tensor of rank 5 (d0 contiguous), pitches in BYTES, 128B swizzle, OOB -> zero.
int make_tmap_16_5d(CUtensorMap* map, const void* base, const uint64_t dims[5], const uint64_t pitches[4],
                    const uint32_t box[5]);

// fp32 tensor [d2][d1][d0], no swizzle (plain row-major box in shared memory), OOB -> zero fill.
int make_tmap_f32_3d_plain(CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t pitch1,
                           uint64_t pitch2, uint32_t b0, uint32_t b1, uint32_t b2);

// Multi-block reductions write one partial sum per block into a caller-provided fp32 workspace and ordered_sum() adds
// the partials in a fixed order (no floating-point atomics: the same inputs give the same bits on every run).
// Workspace protocol of such an entry point (ws, ws_floats): ws == NULL is a size query -- *ws_floats receives the
// floats it needs and nothing is launched (returns 1 here, the entry point returns 0); otherwise *ws_floats is the
// capacity of ws, checked against the need (returns -1 after set_error() when too small, 0 to proceed).
int workspace_check(float* ws, long long* ws_floats, long long need, const char* what);
// out[i] (+)= sum_{p < nparts} part[p * n + i], p ascending
int ordered_sum(const float* part, int nparts, long long n, float* out, int accumulate, cudaStream_t stream);
// multiprocessor count of the current device (queried once)
int num_sms();

#define COCOS_CUDA_CHECK(expr)                                                            \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      cocos::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return -2;                                                                          \
    }                                                                                     \
  } while (0)

}  // namespace cocos
