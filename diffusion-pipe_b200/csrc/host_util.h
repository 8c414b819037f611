// Host-side helpers shared by the C-ABI entry points: error reporting and TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/dpipe.h"

namespace dpipe {

void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

#define DPIPE_CUDA_CHECK(expr)                                                                   \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      return ::dpipe::fail(DPIPE_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                           __FILE__, __LINE__);                                                  \
  } while (0)

// 2-D bf16 tensor map with 128B swizzle.  dim0 is the contiguous dimension.
// Returns 0 or a negative DPIPE_E* code.
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1,
                      uint64_t stride1_elems, uint32_t box0, uint32_t box1);
// 3-D variant (dim0 contiguous), strides in elements
int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                      uint64_t stride1_elems, uint64_t stride2_elems, uint32_t box0, uint32_t box1,
                      uint32_t box2);

// 4-D variant for token-major [batch, seq, heads, 128] activations viewed as {d, seq, head, batch}
int make_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint64_t strides_elems[3],
                      const uint32_t box[4]);

int num_sms();  // SM count of the current device (cached per device)

// true when `p` is not a multiple of `bytes`, the width of the vector loads / stores a kernel makes through it
inline bool misaligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) & (uintptr_t)(bytes - 1)) != 0; }

}  // namespace dpipe
