#include "host_util.h"

#include <stdarg.h>
#include <string.h>

namespace dpipe {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1,
                      uint64_t stride1_elems, uint32_t box0, uint32_t box1) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (stride1_elems * 2) % 16 != 0)
    return fail(DPIPE_EINVAL, "TMA operand must be 16B aligned with a 16B-multiple row stride (base=%p ld=%llu)",
                base, (unsigned long long)stride1_elems);
  cuuint64_t dims[2] = {dim0, dim1};
  cuuint64_t strides[1] = {stride1_elems * 2};
  cuuint32_t box[2] = {box0, box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled(2d) failed: %d (dims %llu x %llu ld %llu box %u x %u)", (int)r,
                (unsigned long long)dim0, (unsigned long long)dim1, (unsigned long long)stride1_elems, box0, box1);
  return 0;
}

int make_tmap_3d_bf16(CUtensorMap* out, const void* base, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                      uint64_t stride1_elems, uint64_t stride2_elems, uint32_t box0, uint32_t box1,
                      uint32_t box2) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0 || (stride1_elems * 2) % 16 != 0 ||
      (stride2_elems * 2) % 16 != 0)
    return fail(DPIPE_EINVAL, "TMA operand must be 16B aligned with 16B-multiple strides");
  cuuint64_t dims[3] = {dim0, dim1, dim2};
  cuuint64_t strides[2] = {stride1_elems * 2, stride2_elems * 2};
  cuuint32_t box[3] = {box0, box1, box2};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled(3d) failed: %d", (int)r);
  return 0;
}

int make_tmap_4d_bf16(CUtensorMap* out, const void* base, const uint64_t dims[4], const uint64_t strides_elems[3],
                      const uint32_t box[4]) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return fail(DPIPE_EINVAL, "TMA operand must be 16B aligned");
  cuuint64_t d[4], st[3];
  cuuint32_t bx[4], es[4] = {1, 1, 1, 1};
  for (int i = 0; i < 4; ++i) { d[i] = dims[i]; bx[i] = box[i]; }
  for (int i = 0; i < 3; ++i) {
    st[i] = strides_elems[i] * 2;
    if (st[i] % 16 != 0) return fail(DPIPE_EINVAL, "TMA strides must be multiples of 16 bytes");
  }
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), d, st, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(DPIPE_ECUDA, "cuTensorMapEncodeTiled(4d) failed: %d", (int)r);
  return 0;
}

int num_sms() {
  static int cached[64];
  static bool have[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!have[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
    have[dev] = true;
  }
  return cached[dev];
}

}  // namespace dpipe

extern "C" const char* dpipe_last_error(void) { return dpipe::g_err; }
extern "C" int dpipe_abi_version(void) { return 1; }
extern "C" int dpipe_check_device(int dev) {
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return dpipe::fail(DPIPE_ECUDA, "cudaGetDeviceProperties(%d): %s", dev, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return dpipe::fail(DPIPE_ENOTSUP, "device %d is sm_%d%d; this library is sm_90a only", dev, prop.major, prop.minor);
  return 0;
}
