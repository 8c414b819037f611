// HBM-bound kernels either side of the block stack in one optimizer step:
//
//   grad_sumsq_multi   sum of squares of up to 64 gradient tensors per launch (bf16 or fp32), fp32 per-thread accumulation,
//                      one partial per CTA; grad_sumsq_finish folds the partials in double precision (fixed order:
//                      deterministic) into the squared global L2 norm.                      replaces the per-parameter
//                      `g.float().norm(2)` loop of clip_grad_norm_ (utils/patches.py:204-224), which materialises an fp32
//                      copy of every gradient.
//   grad_scale_multi   g *= coef for the same tensor lists, coef read from device memory; every CTA returns at once when
//                      coef >= 1 (the common case: no clipping, no pass over 24 GB of gradients).
//                                                                                           replaces utils/patches.py:238-243.
//   noise_pack         x_t = (1-t) x_1 + t x_0 and target = x_0 - x_1 in fp32 with IEEE round-to-nearest multiplies and adds
//                      (no FMA contraction: bit-identical to the three separate ATen ops of the host path), written either in
//                      the input layout or packed 2x2 -> [bs, (h/2)(w/2), 4c] (diffusers `_pack_latents`).
//                                                                                           replaces models/flux.py:368-378,
//                                                                                           qwen_image.py:447-455, wan.py:400-404.
//   adamw_step_multi   one pass of optimi's AdamW over up to 64 (p, g, m, v, c) tensor sets per launch, with Kahan-summed
//                      bf16 weights when c is given.  Every operation is an IEEE round-to-nearest intrinsic in the order of
//                      the torch ops it replaces, rounded to the state dtype where a bf16 torch op rounds (no FMA
//                      contraction): bit-identical to oracle/optim_ref.py adamw_step_emulated.
//                                                                                           replaces optimi.AdamW.step
//                                                                                           (train.py:676-678).
#include <cuda_bf16.h>

#include "host_util.h"
#include "optim_common.cuh"

namespace dpipe {

constexpr int ST_MAX_TENSORS = 64;
constexpr int ST_THREADS = 256;

struct TensorList {
  const void* ptr[ST_MAX_TENSORS];
  long long numel[ST_MAX_TENSORS];
  int dtype[ST_MAX_TENSORS];   // 0 = bf16, 1 = fp32
  int n;
};

__device__ __forceinline__ float bf16_bits_to_float(uint32_t bits16) { return __uint_as_float(bits16 << 16); }

__device__ __forceinline__ float block_sum(float v, float* smem) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  float s = 0.f;
  if (warp == 0) {
    s = lane < (blockDim.x >> 5) ? smem[lane] : 0.f;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  }
  __syncthreads();
  return s;   // valid in warp 0
}

__global__ void __launch_bounds__(ST_THREADS) grad_sumsq_multi_kernel(const TensorList tl, float* __restrict__ partials) {
  __shared__ float red[ST_THREADS / 32];
  float acc = 0.f;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (int i = 0; i < tl.n; ++i) {
    const long long n = tl.numel[i];
    if (tl.dtype[i] == 0) {
      const uint16_t* p = reinterpret_cast<const uint16_t*>(tl.ptr[i]);
      const int head = (int)(((16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15) >> 1);   // elements before 16-byte alignment
      const long long h = head < n ? head : n;
      if (tid < h) { const float v = bf16_bits_to_float(p[tid]); acc = fmaf(v, v, acc); }
      const uint4* p4 = reinterpret_cast<const uint4*>(p + h);
      const long long nv = (n - h) >> 3;
      for (long long j = tid; j < nv; j += nthreads) {
        const uint4 q = __ldg(p4 + j);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float lo = __uint_as_float(w[k] << 16), hi = __uint_as_float(w[k] & 0xffff0000u);
          acc = fmaf(lo, lo, acc);
          acc = fmaf(hi, hi, acc);
        }
      }
      const long long tail0 = h + (nv << 3);
      if (tail0 + tid < n) { const float v = bf16_bits_to_float(p[tail0 + tid]); acc = fmaf(v, v, acc); }
    } else {
      const float* p = reinterpret_cast<const float*>(tl.ptr[i]);
      for (long long j = tid; j < n; j += nthreads) { const float v = p[j]; acc = fmaf(v, v, acc); }
    }
  }
  const float s = block_sum(acc, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void grad_sumsq_finish_kernel(const float* __restrict__ partials, int n, float* __restrict__ out) {
  __shared__ double red[ST_THREADS / 32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += (double)partials[i];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    *out = (float)s;
  }
}

__global__ void __launch_bounds__(ST_THREADS) grad_scale_multi_kernel(const TensorList tl, const float* __restrict__ coef_p) {
  const float coef = *coef_p;
  if (!(coef < 1.0f)) return;   // also leaves the gradients alone when the norm is NaN/inf-free and small
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (int i = 0; i < tl.n; ++i) {
    const long long n = tl.numel[i];
    if (tl.dtype[i] == 0) {
      __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(tl.ptr[i]));
      const int head = (int)(((16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15) >> 1);
      const long long h = head < n ? head : n;
      if (tid < h) p[tid] = __float2bfloat16_rn(__bfloat162float(p[tid]) * coef);
      uint4* p4 = reinterpret_cast<uint4*>(p + h);
      const long long nv = (n - h) >> 3;
      for (long long j = tid; j < nv; j += nthreads) {
        uint4 q = p4[j];
        uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float lo = __uint_as_float(w[k] << 16) * coef, hi = __uint_as_float(w[k] & 0xffff0000u) * coef;
          const __nv_bfloat162 r = __floats2bfloat162_rn(lo, hi);
          w[k] = *reinterpret_cast<const uint32_t*>(&r);
        }
        p4[j] = make_uint4(w[0], w[1], w[2], w[3]);
      }
      const long long tail0 = h + (nv << 3);
      if (tail0 + tid < n) p[tail0 + tid] = __float2bfloat16_rn(__bfloat162float(p[tail0 + tid]) * coef);
    } else {
      float* p = reinterpret_cast<float*>(const_cast<void*>(tl.ptr[i]));
      for (long long j = tid; j < n; j += nthreads) p[j] *= coef;
    }
  }
}

// one thread per output element of the packed layout (or the plain layout when pack == 0)
__global__ void noise_pack_kernel(const float* __restrict__ x1, const float* __restrict__ x0, const float* __restrict__ t,
                                  float* __restrict__ xt, float* __restrict__ target, int bs, int c, long long frames_hw,
                                  int h, int w, int pack) {
  const long long per = (long long)c * frames_hw;   // elements per sample
  const long long total = (long long)bs * per;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < total; o += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(o / per);
    long long src;
    if (pack) {
      // out[b, (i*(w/2) + j), (ch*4 + di*2 + dj)] = in[b, ch, 2i+di, 2j+dj]      (frames_hw == h*w)
      const long long r = o - (long long)b * per;
      const int feat = c * 4;
      const long long tok = r / feat;
      const int f = (int)(r - tok * feat);
      const int ch = f >> 2, di = (f >> 1) & 1, dj = f & 1;
      const int i = (int)(tok / (w >> 1)), j = (int)(tok - (long long)i * (w >> 1));
      src = (long long)b * per + ((long long)ch * h + (2 * i + di)) * w + (2 * j + dj);
    } else {
      src = o;
    }
    const float tb = t[b];
    const float a = x1[src], n0 = x0[src];
    const float om = __fsub_rn(1.0f, tb);
    xt[o] = __fadd_rn(__fmul_rn(om, a), __fmul_rn(tb, n0));
    target[o] = __fsub_rn(n0, a);
  }
}

struct AdamwList {
  void* p[ST_MAX_TENSORS];
  const void* g[ST_MAX_TENSORS];
  void* m[ST_MAX_TENSORS];
  void* v[ST_MAX_TENSORS];
  void* c[ST_MAX_TENSORS];     // null: no Kahan compensation for this tensor
  long long numel[ST_MAX_TENSORS];
  int dtype[ST_MAX_TENSORS];   // 0 = bf16, 1 = fp32 (all five tensors of a set share it)
  int n;
};

struct AdamwScalars {
  float lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps, decay;
};

// one element; p, m, v, c are exact values of the state dtype on entry and on exit
template <bool BF16, bool KAHAN>
__device__ __forceinline__ void adamw_elem(float& p, const float g, float& m, float& v, float& c, const AdamwScalars& s) {
  p = R<BF16>(__fmul_rn(p, s.decay));                                            // p.mul_(1 - lr*wd)
  const float w = s.beta1_comp;                                                  // m.lerp_(g, w), torch's two-sided form
  const float d = __fsub_rn(g, m);
  m = R<BF16>(fabsf(w) < 0.5f ? __fadd_rn(m, __fmul_rn(w, d)) : __fsub_rn(g, __fmul_rn(d, __fsub_rn(1.0f, w))));
  v = R<BF16>(__fmul_rn(v, s.beta2_hat));                                        // v.mul_(beta2_hat)
  v = R<BF16>(__fadd_rn(v, __fmul_rn(__fmul_rn(s.one_minus_beta2_hat, g), g)));          // .addcmul_(g, g, 1-beta2_hat)
  const float den = R<BF16>(__fadd_rn(R<BF16>(__fsqrt_rn(v)), s.eps));                    // v.sqrt().add_(eps)
  const float upd = __fdiv_rn(__fmul_rn(-s.lr, m), den);                         // addcdiv's value * m / den
  if (KAHAN) {
    c = R<BF16>(__fadd_rn(c, upd));
    const float old = p;
    p = R<BF16>(__fadd_rn(p, c));
    c = R<BF16>(__fadd_rn(c, R<BF16>(__fsub_rn(old, p))));
  } else {
    p = R<BF16>(__fadd_rn(p, upd));
  }
}

template <bool BF16, bool KAHAN>
__device__ __forceinline__ void adamw_scalar(const AdamwList& tl, int i, long long j, const AdamwScalars& s) {
  float p = ld1<BF16>(tl.p[i], j), m = ld1<BF16>(tl.m[i], j), v = ld1<BF16>(tl.v[i], j);
  float c = KAHAN ? ld1<BF16>(tl.c[i], j) : 0.f;
  adamw_elem<BF16, KAHAN>(p, ld1<BF16>(tl.g[i], j), m, v, c, s);
  st1<BF16>(tl.p[i], j, p);
  st1<BF16>(tl.m[i], j, m);
  st1<BF16>(tl.v[i], j, v);
  if (KAHAN) st1<BF16>(tl.c[i], j, c);
}

// one 32-bit word of each of the five 16-byte vectors: two bf16 elements or one fp32 element, updated in place (the
// vectors stay packed in registers: unpacking all five at once does not fit 64 registers)
template <bool BF16, bool KAHAN>
__device__ __forceinline__ void adamw_word(uint32_t& pw, const uint32_t gw, uint32_t& mw, uint32_t& vw, uint32_t& cw,
                                           const AdamwScalars& s) {
  if (BF16) {
    constexpr uint32_t HI = 0xffff0000u;
    // the results are bf16 values: their fp32 bits end in 16 zeros
    {   // low halves
      float p = __uint_as_float(pw << 16), m = __uint_as_float(mw << 16), v = __uint_as_float(vw << 16), c = __uint_as_float(cw << 16);
      adamw_elem<true, KAHAN>(p, __uint_as_float(gw << 16), m, v, c, s);
      pw = (pw & HI) | (__float_as_uint(p) >> 16);
      mw = (mw & HI) | (__float_as_uint(m) >> 16);
      vw = (vw & HI) | (__float_as_uint(v) >> 16);
      if (KAHAN) cw = (cw & HI) | (__float_as_uint(c) >> 16);
    }
    {   // high halves
      float p = __uint_as_float(pw & HI), m = __uint_as_float(mw & HI), v = __uint_as_float(vw & HI), c = __uint_as_float(cw & HI);
      adamw_elem<true, KAHAN>(p, __uint_as_float(gw & HI), m, v, c, s);
      pw = (pw & ~HI) | __float_as_uint(p);
      mw = (mw & ~HI) | __float_as_uint(m);
      vw = (vw & ~HI) | __float_as_uint(v);
      if (KAHAN) cw = (cw & ~HI) | __float_as_uint(c);
    }
  } else {
    float p = __uint_as_float(pw), m = __uint_as_float(mw), v = __uint_as_float(vw), c = 0.f;
    adamw_elem<false, false>(p, __uint_as_float(gw), m, v, c, s);
    pw = __float_as_uint(p); mw = __float_as_uint(m); vw = __float_as_uint(v);
  }
}

template <bool BF16, bool KAHAN>
__device__ __forceinline__ void adamw_tensor(const AdamwList& tl, int i, long long tid, long long nthreads, const AdamwScalars& s) {
  constexpr int VEC = BF16 ? 8 : 4;            // elements per 16-byte vector
  constexpr int ESZ = BF16 ? 2 : 4;
  const long long n = tl.numel[i];
  const uintptr_t mis = reinterpret_cast<uintptr_t>(tl.p[i]) & 15;
  const bool same = (reinterpret_cast<uintptr_t>(tl.g[i]) & 15) == mis && (reinterpret_cast<uintptr_t>(tl.m[i]) & 15) == mis &&
                    (reinterpret_cast<uintptr_t>(tl.v[i]) & 15) == mis &&
                    (!KAHAN || (reinterpret_cast<uintptr_t>(tl.c[i]) & 15) == mis);
  if (!same) {                                 // views at different offsets mod 16 B: element-wise loads
    for (long long j = tid; j < n; j += nthreads) adamw_scalar<BF16, KAHAN>(tl, i, j, s);
    return;
  }
  const int head = (int)(((16 - mis) & 15) / ESZ);   // elements before 16-byte alignment
  const long long h = head < n ? head : n;
  if (tid < h) adamw_scalar<BF16, KAHAN>(tl, i, tid, s);
  const long long nv = (n - h) / VEC;
  uint4* p4 = reinterpret_cast<uint4*>(static_cast<char*>(tl.p[i]) + h * ESZ);
  const uint4* g4 = reinterpret_cast<const uint4*>(static_cast<const char*>(tl.g[i]) + h * ESZ);
  uint4* m4 = reinterpret_cast<uint4*>(static_cast<char*>(tl.m[i]) + h * ESZ);
  uint4* v4 = reinterpret_cast<uint4*>(static_cast<char*>(tl.v[i]) + h * ESZ);
  uint4* c4 = KAHAN ? reinterpret_cast<uint4*>(static_cast<char*>(tl.c[i]) + h * ESZ) : nullptr;
  for (long long j = tid; j < nv; j += nthreads) {
    uint4 P = p4[j], M = m4[j], V = v4[j], C = KAHAN ? c4[j] : make_uint4(0, 0, 0, 0);
    const uint4 G = __ldg(g4 + j);
    adamw_word<BF16, KAHAN>(P.x, G.x, M.x, V.x, C.x, s);
    adamw_word<BF16, KAHAN>(P.y, G.y, M.y, V.y, C.y, s);
    adamw_word<BF16, KAHAN>(P.z, G.z, M.z, V.z, C.z, s);
    adamw_word<BF16, KAHAN>(P.w, G.w, M.w, V.w, C.w, s);
    p4[j] = P;
    m4[j] = M;
    v4[j] = V;
    if (KAHAN) c4[j] = C;
  }
  const long long tail0 = h + nv * VEC;
  if (tail0 + tid < n) adamw_scalar<BF16, KAHAN>(tl, i, tail0 + tid, s);
}

__global__ void __launch_bounds__(ST_THREADS, 4) adamw_step_multi_kernel(const AdamwList tl, const AdamwScalars s) {
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * blockDim.x;
  for (int i = 0; i < tl.n; ++i) {
    if (tl.dtype[i] == 1) adamw_tensor<false, false>(tl, i, tid, nthreads, s);
    else if (tl.c[i]) adamw_tensor<true, true>(tl, i, tid, nthreads, s);
    else adamw_tensor<true, false>(tl, i, tid, nthreads, s);
  }
}

static int fill_list(TensorList& tl, const void* const* ptrs, const int64_t* numels, const int* dtypes, int begin, int n) {
  tl.n = 0;
  for (int i = begin; i < n && tl.n < ST_MAX_TENSORS; ++i) {
    if (!ptrs[i] || numels[i] < 0 || (dtypes[i] != 0 && dtypes[i] != 1)) return -1;
    if (numels[i] == 0) continue;
    tl.ptr[tl.n] = ptrs[i]; tl.numel[tl.n] = numels[i]; tl.dtype[tl.n] = dtypes[i];
    ++tl.n;
  }
  return 0;
}

}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_grad_sumsq_blocks(void) { return 4 * num_sms(); }

extern "C" int dpipe_grad_sumsq(const void* const* ptrs, const int64_t* numels, const int* dtypes, int n, float* partials,
                                int64_t partials_len, float* out, void* stream) {
  if (n < 0 || (n > 0 && (!ptrs || !numels || !dtypes)) || !partials || !out) return fail(DPIPE_EINVAL, "dpipe_grad_sumsq: null argument");
  const int blocks = dpipe_grad_sumsq_blocks();
  const int launches = (n + ST_MAX_TENSORS - 1) / ST_MAX_TENSORS;
  if (partials_len < (int64_t)blocks * (launches > 0 ? launches : 1)) return fail(DPIPE_EINVAL, "dpipe_grad_sumsq: partials too small");
  cudaStream_t s = (cudaStream_t)stream;
  int used = 0;
  for (int l = 0; l < launches; ++l) {
    TensorList tl;
    if (fill_list(tl, ptrs, numels, dtypes, l * ST_MAX_TENSORS, n < (l + 1) * ST_MAX_TENSORS ? n : (l + 1) * ST_MAX_TENSORS))
      return fail(DPIPE_EINVAL, "dpipe_grad_sumsq: bad tensor %d..", l * ST_MAX_TENSORS);
    if (tl.n == 0) continue;
    grad_sumsq_multi_kernel<<<blocks, ST_THREADS, 0, s>>>(tl, partials + (int64_t)used * blocks);
    DPIPE_CUDA_CHECK(cudaGetLastError());
    ++used;
  }
  grad_sumsq_finish_kernel<<<1, ST_THREADS, 0, s>>>(partials, used * blocks, out);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_grad_scale(const void* const* ptrs, const int64_t* numels, const int* dtypes, int n, const float* coef,
                                void* stream) {
  if (n < 0 || (n > 0 && (!ptrs || !numels || !dtypes)) || !coef) return fail(DPIPE_EINVAL, "dpipe_grad_scale: null argument");
  const int blocks = dpipe_grad_sumsq_blocks();
  for (int l = 0; l * ST_MAX_TENSORS < n; ++l) {
    TensorList tl;
    if (fill_list(tl, ptrs, numels, dtypes, l * ST_MAX_TENSORS, n < (l + 1) * ST_MAX_TENSORS ? n : (l + 1) * ST_MAX_TENSORS))
      return fail(DPIPE_EINVAL, "dpipe_grad_scale: bad tensor %d..", l * ST_MAX_TENSORS);
    if (tl.n == 0) continue;
    grad_scale_multi_kernel<<<blocks, ST_THREADS, 0, (cudaStream_t)stream>>>(tl, coef);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int dpipe_adamw_step(void* const* params, const void* const* grads, void* const* exp_avgs, void* const* exp_avg_sqs,
                                void* const* kahan_comps, const int64_t* numels, const int* dtypes, int n, float lr,
                                float beta1_comp, float beta2_hat, float one_minus_beta2_hat, float eps, float decay,
                                void* stream) {
  if (n < 0) return fail(DPIPE_EINVAL, "dpipe_adamw_step: n < 0");
  if (n > 0 && (!params || !grads || !exp_avgs || !exp_avg_sqs || !numels || !dtypes))
    return fail(DPIPE_EINVAL, "dpipe_adamw_step: null argument");
  // every tensor is checked before the first launch: a bad argument leaves all tensors untouched
  for (int i = 0; i < n; ++i) {
    if (numels[i] < 0) return fail(DPIPE_EINVAL, "dpipe_adamw_step: tensor %d has numel < 0", i);
    if (dtypes[i] != 0 && dtypes[i] != 1) return fail(DPIPE_EINVAL, "dpipe_adamw_step: tensor %d has dtype %d (0 = bf16, 1 = fp32)", i, dtypes[i]);
    if (numels[i] == 0) continue;
    if (!params[i] || !grads[i] || !exp_avgs[i] || !exp_avg_sqs[i]) return fail(DPIPE_EINVAL, "dpipe_adamw_step: tensor %d has a null pointer", i);
    if (kahan_comps && kahan_comps[i] && dtypes[i] != 0)
      return fail(DPIPE_EINVAL, "dpipe_adamw_step: tensor %d: Kahan compensation is for bf16 tensors only", i);
  }
  const AdamwScalars s{lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps, decay};
  int i = 0;
  while (i < n) {
    AdamwList tl;
    tl.n = 0;
    for (; i < n && tl.n < ST_MAX_TENSORS; ++i) {
      if (numels[i] == 0) continue;
      tl.p[tl.n] = params[i]; tl.g[tl.n] = grads[i]; tl.m[tl.n] = exp_avgs[i]; tl.v[tl.n] = exp_avg_sqs[i];
      tl.c[tl.n] = kahan_comps ? kahan_comps[i] : nullptr;
      tl.numel[tl.n] = numels[i]; tl.dtype[tl.n] = dtypes[i];
      ++tl.n;
    }
    if (tl.n == 0) continue;
    adamw_step_multi_kernel<<<dpipe_grad_sumsq_blocks(), ST_THREADS, 0, (cudaStream_t)stream>>>(tl, s);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int dpipe_noise_pack(const float* x1, const float* x0, const float* t, float* xt, float* target, int bs, int c,
                                int64_t frames, int h, int w, int pack, void* stream) {
  if (!x1 || !x0 || !t || !xt || !target || bs <= 0 || c <= 0 || frames <= 0 || h <= 0 || w <= 0)
    return fail(DPIPE_EINVAL, "dpipe_noise_pack: bad arguments");
  if (pack && (frames != 1 || (h & 1) || (w & 1))) return fail(DPIPE_EINVAL, "dpipe_noise_pack: 2x2 packing needs one frame and even h, w");
  const long long total = (long long)bs * c * frames * h * w;
  long long blocks = (total + 255) / 256;
  const long long cap = 8LL * num_sms();
  if (blocks > cap) blocks = cap;
  noise_pack_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x1, x0, t, xt, target, bs, c, (long long)frames * h * w, h, w, pack);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
