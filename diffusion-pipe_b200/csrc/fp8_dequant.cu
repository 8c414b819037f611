// fp8 -> bf16 expansion of a frozen weight matrix into a GEMM operand buffer.
//
// The reference stores the frozen base of a LoRA run as torch.float8_e4m3fn / float8_e5m2 without scales
// (`transformer_dtype = 'float8'`: models/flux.py:172,203-205, models/qwen_image.py:249-262, utils/common.py:18-20) and
// lets autocast widen the weight to bf16 inside every nn.Linear.  Every fp8 value is exactly representable in bf16, so the
// widening is a table lookup; the GEMMs then run on the same wgmma kernel as the bf16 path.
//
// HBM-bound: 1 B read + 2 B written per element.  One thread expands 16 codes (one 16-byte load, two 16-byte stores)
// through a 256-entry bf16 table in shared memory; the grid is a multiple of the SM count and strides over the matrix.
#include "host_util.h"

namespace dpipe {

// ---- the code tables (host + device: dpipe_fp8_code_table exposes exactly what the kernel uses) ----
__host__ __device__ inline int msb3(unsigned m) { return m >= 4 ? 2 : (m >= 2 ? 1 : 0); }

// e4m3fn: 1 sign, 4 exponent (bias 7), 3 mantissa; no infinities, S.1111.111 is NaN; subnormals m * 2^-9
__host__ __device__ inline uint16_t e4m3_to_bf16_bits(unsigned b) {
  const unsigned s = (b >> 7) & 1u, e = (b >> 3) & 15u, m = b & 7u;
  if (e == 15u && m == 7u) return (uint16_t)((s << 15) | 0x7FC0u);
  if (e == 0u) {
    if (m == 0u) return (uint16_t)(s << 15);
    const int p = msb3(m);                                  // m * 2^-9 = 2^(p-9) * (1 + (m - 2^p) / 2^p)
    return (uint16_t)((s << 15) | ((unsigned)(p - 9 + 127) << 7) | ((m - (1u << p)) << (7 - p)));
  }
  return (uint16_t)((s << 15) | ((e + 120u) << 7) | (m << 4));   // 2^(e-7) * (1 + m/8):  e - 7 + 127, m << (7 - 3)
}

// e5m2: 1 sign, 5 exponent (bias 15), 2 mantissa; IEEE-like (e = 31: inf / NaN); subnormals m * 2^-16
__host__ __device__ inline uint16_t e5m2_to_bf16_bits(unsigned b) {
  const unsigned s = (b >> 7) & 1u, e = (b >> 2) & 31u, m = b & 3u;
  if (e == 31u) return (uint16_t)((s << 15) | (m ? 0x7FC0u : 0x7F80u));
  if (e == 0u) {
    if (m == 0u) return (uint16_t)(s << 15);
    const int p = msb3(m);                                  // m * 2^-16 = 2^(p-16) * (1 + (m - 2^p) / 2^p)
    return (uint16_t)((s << 15) | ((unsigned)(p - 16 + 127) << 7) | ((m - (1u << p)) << (7 - p)));
  }
  return (uint16_t)((s << 15) | ((e + 112u) << 7) | (m << 5));   // e - 15 + 127, m << (7 - 2)
}

template <int FMT>
__global__ void __launch_bounds__(256) fp8_to_bf16_kernel(const uint8_t* __restrict__ src, uint16_t* __restrict__ dst,
                                                           int64_t rows, int64_t chunks_per_row, int64_t ld_src,
                                                           int64_t ld_dst) {
  __shared__ uint16_t lut[256];
  lut[threadIdx.x] = FMT == DPIPE_FP8_E4M3 ? e4m3_to_bf16_bits(threadIdx.x) : e5m2_to_bf16_bits(threadIdx.x);
  __syncthreads();
  const int64_t total = rows * chunks_per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / chunks_per_row, c = i - r * chunks_per_row;
    const uint4 in = *reinterpret_cast<const uint4*>(src + r * ld_src + c * 16);
    const uint32_t w[4] = {in.x, in.y, in.z, in.w};
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      o[2 * k] = (uint32_t)lut[w[k] & 0xFFu] | ((uint32_t)lut[(w[k] >> 8) & 0xFFu] << 16);
      o[2 * k + 1] = (uint32_t)lut[(w[k] >> 16) & 0xFFu] | ((uint32_t)lut[w[k] >> 24] << 16);
    }
    uint4* out = reinterpret_cast<uint4*>(dst + r * ld_dst + c * 16);
    out[0] = make_uint4(o[0], o[1], o[2], o[3]);
    out[1] = make_uint4(o[4], o[5], o[6], o[7]);
  }
}

}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_fp8_code_table(int format, uint16_t* bf16_bits_256) {
  if (!bf16_bits_256) return fail(DPIPE_EINVAL, "dpipe_fp8_code_table: null output");
  if (format != DPIPE_FP8_E4M3 && format != DPIPE_FP8_E5M2)
    return fail(DPIPE_EINVAL, "dpipe_fp8_code_table: unknown format %d", format);
  for (unsigned b = 0; b < 256; ++b)
    bf16_bits_256[b] = format == DPIPE_FP8_E4M3 ? e4m3_to_bf16_bits(b) : e5m2_to_bf16_bits(b);
  return 0;
}

extern "C" int dpipe_fp8_to_bf16(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows, int64_t cols,
                                 int format, void* stream) {
  if (format != DPIPE_FP8_E4M3 && format != DPIPE_FP8_E5M2)
    return fail(DPIPE_EINVAL, "dpipe_fp8_to_bf16: unknown format %d", format);
  if (rows < 0 || cols < 0) return fail(DPIPE_EINVAL, "dpipe_fp8_to_bf16: negative shape");
  if (rows == 0 || cols == 0) return 0;
  if (!src || !dst) return fail(DPIPE_EINVAL, "dpipe_fp8_to_bf16: null pointer");
  if (cols % 16 != 0 || ld_src % 16 != 0 || ld_dst % 8 != 0 || ld_src < cols || ld_dst < cols)
    return fail(DPIPE_EINVAL, "dpipe_fp8_to_bf16: cols (%lld) and ld_src (%lld) must be multiples of 16, ld_dst (%lld) of 8, "
                "and both strides >= cols", (long long)cols, (long long)ld_src, (long long)ld_dst);
  if ((reinterpret_cast<uintptr_t>(src) & 15) != 0 || (reinterpret_cast<uintptr_t>(dst) & 15) != 0)
    return fail(DPIPE_EINVAL, "dpipe_fp8_to_bf16: src and dst must be 16-byte aligned");
  const int64_t chunks_per_row = cols / 16;
  const int64_t total = rows * chunks_per_row;
  const int64_t want = (total + 255) / 256;
  const int64_t cap = (int64_t)num_sms() * 8;
  const int grid = (int)(want < cap ? want : cap);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (format == DPIPE_FP8_E4M3)
    fp8_to_bf16_kernel<DPIPE_FP8_E4M3><<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), static_cast<uint16_t*>(dst),
                                                            rows, chunks_per_row, ld_src, ld_dst);
  else
    fp8_to_bf16_kernel<DPIPE_FP8_E5M2><<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(src), static_cast<uint16_t*>(dst),
                                                            rows, chunks_per_row, ld_src, ld_dst);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
