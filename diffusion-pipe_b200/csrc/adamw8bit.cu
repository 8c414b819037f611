// bitsandbytes' AdamW8bit step (`type = 'adamw8bit'`) as one multi-tensor kernel over up to 64 tensors per launch:
//
//   a8_step_kernel   one warp per block of 256 elements of one tensor, 8 consecutive elements per lane.
//                    8-bit states: dequantize m, v with the stored absmax, Adam update, new absmax by a warp max
//                    (exact and order-free: no atomics, replicas stay bit-identical), p update, quantize m / absmax
//                    and v / absmax to the nearest map entry.        10 B / bf16 parameter (p, g r/w 2+2+2, codes 2+2)
//                    fp32 states (tensors below min_8bit_size): the same update on fp32 m, v.
//
// The maps sit in shared memory, each with its 255 midpoints in breadth-first (Eytzinger) order, so the nearest-entry
// search is 8 probes whose first six levels touch at most 32 consecutive words (no bank conflicts).  Every float
// operation is an IEEE round-to-nearest intrinsic in the order of oracle/adamw8bit_ref.py (bit-identical to
// adamw8bit_emulated); bf16 weights round to bf16 after the update and after the weight decay.  16-byte vectors for
// p and g when a lane's 8 elements are 16-byte aligned, element-wise access otherwise.
//                                                      replaces bitsandbytes.optim.AdamW8bit.step (train.py:650-700).
#include <cuda_bf16.h>

#include "host_util.h"
#include "optim_common.cuh"

namespace dpipe {
namespace {

constexpr int A8_MAX = 64;
constexpr int A8_THREADS = 256;
constexpr int A8_WARPS = A8_THREADS / 32;
constexpr int A8_BLOCK = 256;             // elements per absmax block (one warp)
constexpr int A8_PER_LANE = A8_BLOCK / 32;

struct A8List {
  dpipe_adamw8bit_tensor t[A8_MAX];
  long long blk0[A8_MAX + 1];             // prefix sums of the 256-element blocks per tensor
  int n;
};

// number of midpoints below x: the nearest map entry (tree[1..255] in breadth-first order; NaN goes left: 0)
__device__ __forceinline__ int nearest_code(const float* __restrict__ tree, float x) {
  int i = 1;
#pragma unroll
  for (int k = 0; k < 8; ++k) i = 2 * i + (tree[i] < x ? 1 : 0);
  return i - 256;
}

template <bool BF16>
__device__ __forceinline__ void load8(const void* base, long long e, int valid, bool vec, float (&x)[A8_PER_LANE]) {
  if (BF16) {
    const __nv_bfloat16* a = reinterpret_cast<const __nv_bfloat16*>(base) + e;
    if (vec) {
      const uint4 q = *reinterpret_cast<const uint4*>(a);
      const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        x[2 * k] = __uint_as_float(w[k] << 16);
        x[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u);
      }
    } else {
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j) x[j] = j < valid ? __bfloat162float(a[j]) : 0.f;
    }
  } else {
    const float* a = reinterpret_cast<const float*>(base) + e;
    if (vec) {
      const float4 q0 = reinterpret_cast<const float4*>(a)[0], q1 = reinterpret_cast<const float4*>(a)[1];
      x[0] = q0.x; x[1] = q0.y; x[2] = q0.z; x[3] = q0.w;
      x[4] = q1.x; x[5] = q1.y; x[6] = q1.z; x[7] = q1.w;
    } else {
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j) x[j] = j < valid ? a[j] : 0.f;
    }
  }
}

template <bool BF16>
__device__ __forceinline__ void store8(void* base, long long e, int valid, bool vec, const float (&x)[A8_PER_LANE]) {
  if (BF16) {
    __nv_bfloat16* a = reinterpret_cast<__nv_bfloat16*>(base) + e;
    if (vec) {
      uint32_t w[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const __nv_bfloat162 r = __floats2bfloat162_rn(x[2 * k], x[2 * k + 1]);
        w[k] = *reinterpret_cast<const uint32_t*>(&r);
      }
      *reinterpret_cast<uint4*>(a) = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j)
        if (j < valid) a[j] = __float2bfloat16_rn(x[j]);
    }
  } else {
    float* a = reinterpret_cast<float*>(base) + e;
    if (vec) {
      reinterpret_cast<float4*>(a)[0] = make_float4(x[0], x[1], x[2], x[3]);
      reinterpret_cast<float4*>(a)[1] = make_float4(x[4], x[5], x[6], x[7]);
    } else {
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j)
        if (j < valid) a[j] = x[j];
    }
  }
}

__device__ __forceinline__ bool aligned16(const void* base, long long e, int esz) {
  return ((reinterpret_cast<uintptr_t>(base) + (uintptr_t)(e * esz)) & 15) == 0;
}

// one lane's 8 elements of block `blk` of tensor t; e: its first element, valid: how many of the 8 exist
template <bool BF16, bool Q8>
__device__ __forceinline__ void a8_lane(const dpipe_adamw8bit_tensor& t, long long blk, long long e, int valid,
                                        const float* __restrict__ q1, const float* __restrict__ q2,
                                        const float* __restrict__ tree1, const float* __restrict__ tree2) {
  constexpr int ESZ = BF16 ? 2 : 4;
  const bool vec = valid == A8_PER_LANE && aligned16(t.p, e, ESZ) && aligned16(t.g, e, ESZ);
  float p[A8_PER_LANE], g[A8_PER_LANE], m[A8_PER_LANE], v[A8_PER_LANE];
  load8<BF16>(t.g, e, valid, vec, g);
  const float b1 = t.beta1, b2 = t.beta2;
  const float omb1 = __fsub_rn(1.0f, b1), omb2 = __fsub_rn(1.0f, b2);
  unsigned char c1[A8_PER_LANE], c2[A8_PER_LANE];
  if (Q8) {
    const unsigned char* s1 = reinterpret_cast<const unsigned char*>(t.state1) + e;
    const unsigned char* s2 = reinterpret_cast<const unsigned char*>(t.state2) + e;
    if (valid == A8_PER_LANE && ((reinterpret_cast<uintptr_t>(s1) | reinterpret_cast<uintptr_t>(s2)) & 7) == 0) {
      const uint2 w1 = *reinterpret_cast<const uint2*>(s1), w2 = *reinterpret_cast<const uint2*>(s2);
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j) {
        c1[j] = (unsigned char)(((j < 4 ? w1.x : w1.y) >> (8 * (j & 3))) & 0xff);
        c2[j] = (unsigned char)(((j < 4 ? w2.x : w2.y) >> (8 * (j & 3))) & 0xff);
      }
    } else {
#pragma unroll
      for (int j = 0; j < A8_PER_LANE; ++j) {
        c1[j] = j < valid ? s1[j] : 0;
        c2[j] = j < valid ? s2[j] : 0;
      }
    }
    const float a1 = t.absmax1[blk], a2 = t.absmax2[blk];
#pragma unroll
    for (int j = 0; j < A8_PER_LANE; ++j) {
      if (isfinite(g[j])) {
        v[j] = __fadd_rn(__fmul_rn(__fmul_rn(q2[c2[j]], a2), b2), __fmul_rn(__fmul_rn(omb2, g[j]), g[j]));
        m[j] = __fadd_rn(__fmul_rn(__fmul_rn(q1[c1[j]], a1), b1), __fmul_rn(omb1, g[j]));
      } else {
        m[j] = 0.f;
        v[j] = 0.f;
      }
    }
  } else {
    const bool svec = valid == A8_PER_LANE && aligned16(t.state1, e, 4) && aligned16(t.state2, e, 4);
    load8<false>(t.state1, e, valid, svec, m);
    load8<false>(t.state2, e, valid, svec, v);
#pragma unroll
    for (int j = 0; j < A8_PER_LANE; ++j) {
      m[j] = __fadd_rn(__fmul_rn(m[j], b1), __fmul_rn(omb1, g[j]));
      v[j] = __fadd_rn(__fmul_rn(v[j], b2), __fmul_rn(__fmul_rn(omb2, g[j]), g[j]));
    }
    store8<false>(t.state1, e, valid, svec, m);
    store8<false>(t.state2, e, valid, svec, v);
  }
  load8<BF16>(t.p, e, valid, vec, p);
#pragma unroll
  for (int j = 0; j < A8_PER_LANE; ++j) {
    if (Q8 && !isfinite(g[j])) continue;                                 // bnb skips the element: p stays
    const float den = __fadd_rn(__fsqrt_rn(v[j]), t.eps_c2);
    const float pn = R<BF16>(__fadd_rn(p[j], __fmul_rn(t.step_size, __fdiv_rn(m[j], den))));
    p[j] = R<BF16>(__fmul_rn(pn, t.decay));
  }
  store8<BF16>(t.p, e, valid, vec, p);
  if (!Q8) return;
  // new absmax of the block: |m|, v >= 0 (fmaxf drops NaN), so the fp32 bits order as unsigned integers
  float mx1 = 0.f, mx2 = 0.f;
#pragma unroll
  for (int j = 0; j < A8_PER_LANE; ++j)
    if (j < valid) {
      mx1 = fmaxf(mx1, fabsf(m[j]));
      mx2 = fmaxf(mx2, fabsf(v[j]));
    }
  const float am1 = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(mx1)));
  const float am2 = __uint_as_float(__reduce_max_sync(0xffffffffu, __float_as_uint(mx2)));
  if ((threadIdx.x & 31) == 0) {
    t.absmax1[blk] = am1;
    t.absmax2[blk] = am2;
  }
#pragma unroll
  for (int j = 0; j < A8_PER_LANE; ++j) {
    int k1 = nearest_code(tree1, am1 > 0.f ? __fdiv_rn(m[j], am1) : 0.f);
    if (signbit(q1[k1]) != signbit(m[j])) k1 += m[j] > 0.f ? 1 : -1;    // keep the sign of the first moment
    c1[j] = (unsigned char)k1;
    c2[j] = (unsigned char)nearest_code(tree2, am2 > 0.f ? __fdiv_rn(v[j], am2) : 0.f);
  }
  unsigned char* s1 = reinterpret_cast<unsigned char*>(t.state1) + e;
  unsigned char* s2 = reinterpret_cast<unsigned char*>(t.state2) + e;
  if (valid == A8_PER_LANE && ((reinterpret_cast<uintptr_t>(s1) | reinterpret_cast<uintptr_t>(s2)) & 7) == 0) {
    uint2 w1 = make_uint2(0, 0), w2 = make_uint2(0, 0);
#pragma unroll
    for (int j = 0; j < A8_PER_LANE; ++j) {
      (j < 4 ? w1.x : w1.y) |= (uint32_t)c1[j] << (8 * (j & 3));
      (j < 4 ? w2.x : w2.y) |= (uint32_t)c2[j] << (8 * (j & 3));
    }
    *reinterpret_cast<uint2*>(s1) = w1;
    *reinterpret_cast<uint2*>(s2) = w2;
  } else {
#pragma unroll
    for (int j = 0; j < A8_PER_LANE; ++j)
      if (j < valid) {
        s1[j] = c1[j];
        s2[j] = c2[j];
      }
  }
}

// the midpoint of in-order position k, for breadth-first node i of the perfect 255-node tree
__device__ __forceinline__ float tree_node(const float* __restrict__ q, int i) {
  const int level = 31 - __clz(i);
  const int k = ((2 * (i - (1 << level)) + 1) << (7 - level)) - 1;
  return __fmul_rn(__fadd_rn(q[k], q[k + 1]), 0.5f);
}

__global__ void __launch_bounds__(A8_THREADS) a8_step_kernel(const __grid_constant__ A8List tl,
                                                            const float* __restrict__ qmap1,
                                                            const float* __restrict__ qmap2) {
  __shared__ float q1[256], q2[256], tree1[256], tree2[256];
  if (qmap1) {
    const int i = threadIdx.x;
    q1[i] = qmap1[i];
    q2[i] = qmap2[i];
    __syncthreads();
    if (i > 0) {
      tree1[i] = tree_node(q1, i);
      tree2[i] = tree_node(q2, i);
    }
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long total = tl.blk0[tl.n];
  int ti = 0;
  for (long long w = (long long)blockIdx.x * A8_WARPS + warp; w < total; w += (long long)gridDim.x * A8_WARPS) {
    while (w >= tl.blk0[ti + 1]) ++ti;                                   // w only grows: one pass over the tensors
    const dpipe_adamw8bit_tensor& t = tl.t[ti];
    const long long blk = w - tl.blk0[ti];
    const long long e = blk * A8_BLOCK + lane * A8_PER_LANE;
    const long long left = t.numel - e;
    const int valid = left >= A8_PER_LANE ? A8_PER_LANE : (left > 0 ? (int)left : 0);
    const bool q8 = t.absmax1 != nullptr;
    if (t.dtype == 0) {
      if (q8) a8_lane<true, true>(t, blk, e, valid, q1, q2, tree1, tree2);
      else if (valid) a8_lane<true, false>(t, blk, e, valid, q1, q2, tree1, tree2);
    } else {
      if (q8) a8_lane<false, true>(t, blk, e, valid, q1, q2, tree1, tree2);
      else if (valid) a8_lane<false, false>(t, blk, e, valid, q1, q2, tree1, tree2);
    }
  }
}

long long blocks_of(const dpipe_adamw8bit_tensor& t) { return (t.numel + A8_BLOCK - 1) / A8_BLOCK; }

// the next chunk of up to 64 non-empty tensors from *pos; returns its block count
long long fill(A8List& tl, const dpipe_adamw8bit_tensor* t, int n, int* pos) {
  tl.n = 0;
  tl.blk0[0] = 0;
  for (; *pos < n && tl.n < A8_MAX; ++*pos) {
    if (t[*pos].numel == 0) continue;
    tl.t[tl.n] = t[*pos];
    tl.blk0[tl.n + 1] = tl.blk0[tl.n] + blocks_of(t[*pos]);
    ++tl.n;
  }
  return tl.blk0[tl.n];
}

}  // namespace
}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_adamw8bit_step(const dpipe_adamw8bit_tensor* t, int n, const float* qmap1, const float* qmap2,
                                    void* stream) {
  if (n < 0 || (n > 0 && !t)) return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: null tensor array or n < 0");
  // every tensor is checked before the first launch: a bad argument leaves all tensors untouched
  for (int i = 0; i < n; ++i) {
    const dpipe_adamw8bit_tensor& a = t[i];
    if (a.numel < 0) return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: tensor %d has numel < 0", i);
    if (a.dtype != 0 && a.dtype != 1)
      return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: tensor %d has dtype %d (0 = bf16, 1 = fp32)", i, a.dtype);
    if (a.numel == 0) continue;
    if (!a.p || !a.g || !a.state1 || !a.state2) return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: tensor %d has a null pointer", i);
    if (!a.absmax1 != !a.absmax2)
      return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: tensor %d: absmax1 and absmax2 must both be given (8-bit) or both null", i);
    if (a.absmax1 && (!qmap1 || !qmap2))
      return fail(DPIPE_EINVAL, "dpipe_adamw8bit_step: tensor %d has 8-bit states but the maps are null", i);
  }
  const int grid_cap = 4 * num_sms();
  for (int pos = 0; pos < n;) {
    A8List tl;
    const long long blocks = fill(tl, t, n, &pos);
    if (tl.n == 0) continue;
    long long ctas = (blocks + A8_WARPS - 1) / A8_WARPS;
    if (ctas > grid_cap) ctas = grid_cap;
    a8_step_kernel<<<(unsigned)ctas, A8_THREADS, 0, (cudaStream_t)stream>>>(tl, qmap1, qmap2);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}
