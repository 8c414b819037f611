// AdaLayerNorm modulation linears:  mod[b, :] = W · silu(temb[b, :]) + bias   with batch b = micro-batch size (1..8).
//
// These are rank-`batch` problems (M = batch): 113 MB of weights are streamed once per call, so they are HBM-bound and do
// not belong on the tensor-core GEMM (a 128-row MMA tile would be >99% padding).  Forward: one warp per output row.
// Backward: ONE pass over W and dW with one thread per 8 columns — it forms dW (+)= dmod^T · silu(temb), d bias and the
// per-CTA partials of d silu = dmod · W; a finish kernel folds the partials through silu' into d temb.
//
// Replaces nn.Linear(SiLU(temb)) inside diffusers AdaLayerNormZero / AdaLayerNormZeroSingle / AdaLayerNormContinuous
// (reference call sites models/flux.py:502,525,547) and its autograd backward.
#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int MOD_MAX_B = 8;
constexpr int MOD_ROWS = 64;   // weight rows per CTA in the backward pass

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_grad_f(float x) {
  const float s = 1.0f / (1.0f + __expf(-x));
  return s * (1.0f + x * (1.0f - s));
}
__device__ __forceinline__ void unpack8f(const uint4& q, float* f) {
  f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
  f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
}

// grid = N / 8 CTAs of 256 threads; warp w of CTA c owns output row n = 8c + w.  smem: [B][K] fp32 silu(temb)
__global__ void mod_fwd_kernel(const __nv_bfloat16* __restrict__ temb, const __nv_bfloat16* __restrict__ W,
                               const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ out, int B, int N, int K) {
  extern __shared__ float s_smem[];
  for (int i = threadIdx.x; i < B * K; i += blockDim.x)
    s_smem[i] = bf16_round(silu_f(__bfloat162float(temb[i])));   // SiLU output is a bf16 tensor in the reference
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * 8 + warp;
  if (n >= N) return;
  float acc[MOD_MAX_B];
#pragma unroll
  for (int b = 0; b < MOD_MAX_B; ++b) acc[b] = 0.f;
  const uint4* wrow = reinterpret_cast<const uint4*>(W + (int64_t)n * K);
  for (int c = lane; c < K / 8; c += 32) {
    float w[8];
    unpack8f(wrow[c], w);
#pragma unroll
    for (int b = 0; b < MOD_MAX_B; ++b) {
      if (b < B) {
        const float* s = s_smem + b * K + c * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[b] = fmaf(w[j], s[j], acc[b]);
      }
    }
  }
#pragma unroll
  for (int b = 0; b < MOD_MAX_B; ++b) {
    if (b < B) {
      float v = acc[b];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if (lane == 0) out[(int64_t)b * N + n] = __float2bfloat16_rn(v + (bias ? __bfloat162float(bias[n]) : 0.f));
    }
  }
}

// grid = N / MOD_ROWS CTAs of K/8 threads; thread t owns columns [8t, 8t+8)
template <int BMAX>
__global__ void mod_bwd_kernel(const float* __restrict__ dmod, int64_t ldd, const __nv_bfloat16* __restrict__ temb,
                               const __nv_bfloat16* __restrict__ W, __nv_bfloat16* __restrict__ dW, int accumulate,
                               float* __restrict__ dbias, float* __restrict__ partials, int B, int N, int K) {
  __shared__ float dm[BMAX][MOD_ROWS];
  const int n0 = blockIdx.x * MOD_ROWS;
  for (int i = threadIdx.x; i < B * MOD_ROWS; i += blockDim.x) {
    const int b = i / MOD_ROWS, r = i % MOD_ROWS;
    dm[b][r] = (n0 + r < N) ? bf16_round(dmod[(int64_t)b * ldd + n0 + r]) : 0.f;   // the reference's grad is a bf16 tensor
  }
  const int col = threadIdx.x * 8;
  float s[BMAX][8], acc[BMAX][8];
#pragma unroll
  for (int b = 0; b < BMAX; ++b) {
    if (b < B) {
      float t[8];
      unpack8f(*reinterpret_cast<const uint4*>(temb + (int64_t)b * K + col), t);
#pragma unroll
      for (int j = 0; j < 8; ++j) { s[b][j] = bf16_round(silu_f(t[j])); acc[b][j] = 0.f; }
    }
  }
  __syncthreads();
  if (dbias) {
    for (int r = threadIdx.x; r < MOD_ROWS && n0 + r < N; r += blockDim.x) {   // blockDim may be smaller than MOD_ROWS
      float v = 0.f;
      for (int b = 0; b < B; ++b) v += dm[b][r];
      dbias[n0 + r] = v;
    }
  }
  const int rows = min(MOD_ROWS, N - n0);
#pragma unroll 4
  for (int r = 0; r < rows; ++r) {
    const int64_t off = (int64_t)(n0 + r) * K + col;
    float w[8], g[8];
    unpack8f(*reinterpret_cast<const uint4*>(W + off), w);
    if (dW && accumulate) {
      unpack8f(*reinterpret_cast<const uint4*>(dW + off), g);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = 0.f;
    }
#pragma unroll
    for (int b = 0; b < BMAX; ++b) {
      if (b < B) {
        const float d = dm[b][r];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[b][j] = fmaf(d, w[j], acc[b][j]);
          g[j] = fmaf(d, s[b][j], g[j]);
        }
      }
    }
    if (dW) {
      uint4 o;
      o.x = pack_bf16(g[0], g[1]); o.y = pack_bf16(g[2], g[3]); o.z = pack_bf16(g[4], g[5]); o.w = pack_bf16(g[6], g[7]);
      *reinterpret_cast<uint4*>(dW + off) = o;
    }
  }
#pragma unroll
  for (int b = 0; b < BMAX; ++b) {
    if (b < B) {
      float* pp = partials + ((int64_t)blockIdx.x * B + b) * K + col;
#pragma unroll
      for (int j = 0; j < 8; ++j) pp[j] = acc[b][j];
    }
  }
}

// d temb[b,k] += silu'(temb[b,k]) * bf16(sum_c partials[c][b][k]);   block = 32 columns x 8 chunk groups
__global__ void mod_bwd_finish_kernel(const float* __restrict__ partials, int nchunk, const __nv_bfloat16* __restrict__ temb,
                                      float* __restrict__ dtemb, int B, int K) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + tx, b = blockIdx.y;
  float acc = 0.f;
  if (k < K)
    for (int c = ty; c < nchunk; c += 8) acc += partials[((int64_t)c * B + b) * K + k];
  red[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && k < K) {
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) v += red[i][tx];
    dtemb[(int64_t)b * K + k] += bf16_round(v) * silu_grad_f(__bfloat162float(temb[(int64_t)b * K + k]));
  }
}

}  // namespace dpipe

using namespace dpipe;
typedef __nv_bfloat16 bf16;

extern "C" int dpipe_mod_fwd(const void* temb, const void* W, const void* bias, void* out, int B, int N, int K, void* stream) {
  if (!temb || !W || !out || B < 1 || B > MOD_MAX_B || K % 8 || N < 1) return fail(DPIPE_EINVAL, "dpipe_mod_fwd: bad arguments (B=%d N=%d K=%d)", B, N, K);
  const size_t smem = (size_t)B * K * sizeof(float);
  if (smem > 200 * 1024) return fail(DPIPE_EINVAL, "dpipe_mod_fwd: B*K too large for shared memory");
  static bool configured = false;
  if (!configured) {
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(mod_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    configured = true;
  }
  mod_fwd_kernel<<<(N + 7) / 8, 256, smem, (cudaStream_t)stream>>>((const bf16*)temb, (const bf16*)W, (const bf16*)bias, (bf16*)out, B, N, K);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_mod_bwd_chunks(int N) { return (N + MOD_ROWS - 1) / MOD_ROWS; }

extern "C" int dpipe_mod_bwd(const float* dmod, int64_t ldd, const void* temb, const void* W, void* dW, int accumulate,
                             float* dbias, float* partials, float* dtemb, int B, int N, int K, void* stream) {
  if (!dmod || !temb || !W || !partials || !dtemb || B < 1 || B > MOD_MAX_B || K % 256 || K / 8 > 1024)
    return fail(DPIPE_EINVAL, "dpipe_mod_bwd: bad arguments (B=%d N=%d K=%d)", B, N, K);
  if (B > 4 && K > 3328)   // mod_bwd_kernel<8>: 155 registers x K/8 threads must fit the register file
    return fail(DPIPE_EINVAL, "dpipe_mod_bwd: batch %d with K=%d is not supported (batch <= 4 for K > 3328)", B, K);
  const int nchunk = dpipe_mod_bwd_chunks(N);
  cudaStream_t s = (cudaStream_t)stream;
  if (B <= 2)
    mod_bwd_kernel<2><<<nchunk, K / 8, 0, s>>>(dmod, ldd, (const bf16*)temb, (const bf16*)W, (bf16*)dW, accumulate, dbias, partials, B, N, K);
  else if (B <= 4)
    mod_bwd_kernel<4><<<nchunk, K / 8, 0, s>>>(dmod, ldd, (const bf16*)temb, (const bf16*)W, (bf16*)dW, accumulate, dbias, partials, B, N, K);
  else
    mod_bwd_kernel<8><<<nchunk, K / 8, 0, s>>>(dmod, ldd, (const bf16*)temb, (const bf16*)W, (bf16*)dW, accumulate, dbias, partials, B, N, K);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  mod_bwd_finish_kernel<<<dim3((K + 31) / 32, B), 256, 0, s>>>(partials, nchunk, (const bf16*)temb, dtemb, B, K);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
