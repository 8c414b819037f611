// Wan attention pre-processing: RMSNorm over the FULL model width (not per head), RoPE, and the scatter from the
// token-major projection output [rows, C] into the head-major [B, H, L, 128] layout the attention kernels read.
//
// Reference (models/wan/model.py): WanRMSNorm :71-87 (`_norm(x.float()).type_as(x) * weight`, eps 1e-6, width = dim),
// WanSelfAttention.forward :137-156 (q = norm_q(q(x)), k = norm_k(k(x)), v = v(x); rope_apply on q and k :41-68 —
// complex multiply of interleaved pairs in fp32, result cast to bf16 by flash_attention :54-78), WanCrossAttention
// :171-183 (same without RoPE; k, v from the text context).  Flux / Qwen normalise per head, which fits in the GEMM
// epilogue (gemm_sm90.cu EPI_QKV_ROPE); a 5120-wide row statistic spans 20 N-tiles and cannot, hence these
// HBM-bound kernels: one CTA per token row, C/8 threads, 16-byte accesses on both layouts.
//
// Algorithmic bytes per token and projection: forward reads 2C (+ 4*128 table bytes per head-row, L2-resident),
// writes 2C (head-major) + 2C (x_hat, saved for backward); backward reads 2C (dy) + 2C (x_hat), writes 2C.
#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int WN_ROWS = 16;   // token rows per CTA in the backward pass (amortises the d weight partial)

__device__ __forceinline__ void wn_unpack8(const uint4& q, float* f) {
  f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
  f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
}
__device__ __forceinline__ uint4 wn_pack8(const float* f) {
  uint4 q;
  q.x = pack_bf16(f[0], f[1]); q.y = pack_bf16(f[2], f[3]); q.z = pack_bf16(f[4], f[5]); q.w = pack_bf16(f[6], f[7]);
  return q;
}

// CTA-wide sum of one value, broadcast to every thread.  `red` is smem [32].
__device__ __forceinline__ float wn_block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < nwarp; ++w) s += red[w];
  return s;
}

struct WanNormProj {
  const __nv_bfloat16* src;     // [rows, ld] token-major projection output (bias already added)
  int64_t ld;
  const __nv_bfloat16* weight;  // [C] RMSNorm scale, or nullptr: no normalisation (v)
  __nv_bfloat16* dst;           // [B, H, L, 128]
  __nv_bfloat16* xhat;          // [rows, C] normalised rows before the scale (saved for backward), or nullptr
  float* rstd;                  // [rows], or nullptr
  int rope;                     // apply the rotation (q, k of self-attention)
};

struct WanNormFwdParams {
  WanNormProj proj[3];
  const float* cos;             // [L, 128] fp32, every frequency repeated twice
  const float* sin;
  int B, L, H;
  float eps;
};

// grid (B * L, nproj), block C / 8
__global__ void wan_norm_rope_fwd_kernel(const WanNormFwdParams p) {
  __shared__ float red[32];
  const WanNormProj& pr = p.proj[blockIdx.y];
  const int row = blockIdx.x;
  const int b = row / p.L, l = row - b * p.L;
  const int col = threadIdx.x * 8;
  const int C = p.H * 128;
  float x[8];
  wn_unpack8(*reinterpret_cast<const uint4*>(pr.src + (int64_t)row * pr.ld + col), x);
  float y[8];
  if (pr.weight) {
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += x[j] * x[j];
    ss = wn_block_sum(ss, red);
    const float rstd = rsqrtf(ss / C + p.eps);
    float w[8], xh[8];
    wn_unpack8(*reinterpret_cast<const uint4*>(pr.weight + col), w);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      xh[j] = bf16_round(x[j] * rstd);          // `.type_as(x)`
      y[j] = bf16_round(xh[j] * w[j]);          // bf16 * bf16 -> bf16
    }
    if (pr.xhat) *reinterpret_cast<uint4*>(pr.xhat + (int64_t)row * C + col) = wn_pack8(xh);
    if (pr.rstd && threadIdx.x == 0) pr.rstd[row] = rstd;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = x[j];
  }
  const int head = col >> 7, d0 = col & 127;
  if (pr.rope) {
    const float4 c0 = *reinterpret_cast<const float4*>(p.cos + (int64_t)l * 128 + d0);
    const float4 c1 = *reinterpret_cast<const float4*>(p.cos + (int64_t)l * 128 + d0 + 4);
    const float4 s0 = *reinterpret_cast<const float4*>(p.sin + (int64_t)l * 128 + d0);
    const float4 s1 = *reinterpret_cast<const float4*>(p.sin + (int64_t)l * 128 + d0 + 4);
    const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
    const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; j += 2) {             // (a + ib)(c + is): pairs (2i, 2i+1)
      o[j] = y[j] * cs[j] - y[j + 1] * sn[j];
      o[j + 1] = y[j + 1] * cs[j + 1] + y[j] * sn[j + 1];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = o[j];
  }
  __nv_bfloat16* out = pr.dst + (((int64_t)b * p.H + head) * p.L + l) * 128 + d0;
  *reinterpret_cast<uint4*>(out) = wn_pack8(y);
}

struct WanNormBwdProj {
  const __nv_bfloat16* dy;      // [B, H, L, 128] gradient of the head-major output
  const __nv_bfloat16* xhat;    // [rows, C] saved by the forward (nullptr with weight == nullptr)
  const float* rstd;            // [rows]
  const __nv_bfloat16* weight;  // [C] or nullptr (v: pure layout change)
  __nv_bfloat16* dx;            // [rows, ld] gradient of the projection output
  int64_t ld;
  float* dw_partials;           // [nchunk, C] fp32 partial sums of d weight (nullptr with weight == nullptr)
  int rope;
};

struct WanNormBwdParams {
  WanNormBwdProj proj[3];
  const float* cos;
  const float* sin;
  int B, L, H;
};

// grid (ceil(B * L / WN_ROWS), nproj), block C / 8
__global__ void wan_norm_rope_bwd_kernel(const WanNormBwdParams p) {
  __shared__ float red[32];
  const WanNormBwdProj& pr = p.proj[blockIdx.y];
  const int col = threadIdx.x * 8;
  const int C = p.H * 128;
  const int head = col >> 7, d0 = col & 127;
  const int rows = p.B * p.L;
  float w[8], dw[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { w[j] = 0.f; dw[j] = 0.f; }
  if (pr.weight) wn_unpack8(*reinterpret_cast<const uint4*>(pr.weight + col), w);
  const int r0 = blockIdx.x * WN_ROWS;
  const int r1 = min(r0 + WN_ROWS, rows);
  for (int row = r0; row < r1; ++row) {
    const int b = row / p.L, l = row - b * p.L;
    float g[8];
    wn_unpack8(*reinterpret_cast<const uint4*>(pr.dy + (((int64_t)b * p.H + head) * p.L + l) * 128 + d0), g);
    if (pr.rope) {   // transpose of the rotation
      const float4 c0 = *reinterpret_cast<const float4*>(p.cos + (int64_t)l * 128 + d0);
      const float4 c1 = *reinterpret_cast<const float4*>(p.cos + (int64_t)l * 128 + d0 + 4);
      const float4 s0 = *reinterpret_cast<const float4*>(p.sin + (int64_t)l * 128 + d0);
      const float4 s1 = *reinterpret_cast<const float4*>(p.sin + (int64_t)l * 128 + d0 + 4);
      const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      float t[8];
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        t[j] = g[j] * cs[j] + g[j + 1] * sn[j + 1];
        t[j + 1] = g[j + 1] * cs[j + 1] - g[j] * sn[j];
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) g[j] = t[j];
    }
    float o[8];
    if (pr.weight) {
      float xh[8], dxh[8];
      wn_unpack8(*reinterpret_cast<const uint4*>(pr.xhat + (int64_t)row * C + col), xh);
      float dot = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dw[j] += g[j] * xh[j];
        dxh[j] = g[j] * w[j];
        dot += dxh[j] * xh[j];
      }
      dot = wn_block_sum(dot, red) / C;
      const float rs = pr.rstd[row];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rs * (dxh[j] - xh[j] * dot);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = g[j];
    }
    *reinterpret_cast<uint4*>(pr.dx + (int64_t)row * pr.ld + col) = wn_pack8(o);
  }
  if (pr.weight && pr.dw_partials) {
    float* pp = pr.dw_partials + (int64_t)blockIdx.x * C + col;
#pragma unroll
    for (int j = 0; j < 8; ++j) pp[j] = dw[j];
  }
}

}  // namespace dpipe

using namespace dpipe;

static int wn_check(const char* fn, int B, int L, int H, int nproj) {
  if (B < 1 || L < 1 || H < 1 || H > 56 || (H * 128) % 256 || nproj < 1 || nproj > 3)   // 16 H threads x 72 registers per CTA
    return fail(DPIPE_EINVAL, "%s: bad geometry B=%d L=%d H=%d nproj=%d (width H*128 must be a multiple of 256, <= 7168)", fn, B, L, H, nproj);
  return 0;
}

extern "C" int dpipe_wan_norm_rows(void) { return WN_ROWS; }

extern "C" int dpipe_wan_norm_rope_fwd(const dpipe_wan_norm_fwd_args* a, void* stream) {
  if (!a) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_fwd: null args");
  int rc = wn_check("dpipe_wan_norm_rope_fwd", a->batch, a->seq, a->heads, a->nproj);
  if (rc) return rc;
  WanNormFwdParams p;
  for (int i = 0; i < 3; ++i) p.proj[i] = WanNormProj{nullptr, 0, nullptr, nullptr, nullptr, nullptr, 0};
  for (int i = 0; i < a->nproj; ++i) {
    const dpipe_wan_norm_proj& s = a->proj[i];
    if (!s.src || !s.dst || s.ld % 8 || s.ld < a->heads * 128) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_fwd: projection %d: bad pointers / ld", i);
    if (s.rope && (!a->cos || !a->sin)) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_fwd: rope requested without tables");
    p.proj[i] = WanNormProj{(const __nv_bfloat16*)s.src, s.ld, (const __nv_bfloat16*)s.weight, (__nv_bfloat16*)s.dst,
                            (__nv_bfloat16*)s.xhat, s.rstd, s.rope};
  }
  p.cos = a->cos; p.sin = a->sin; p.B = a->batch; p.L = a->seq; p.H = a->heads; p.eps = a->eps;
  dim3 grid(a->batch * a->seq, a->nproj);
  wan_norm_rope_fwd_kernel<<<grid, a->heads * 16, 0, (cudaStream_t)stream>>>(p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_wan_norm_rope_bwd(const dpipe_wan_norm_bwd_args* a, void* stream) {
  if (!a) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_bwd: null args");
  int rc = wn_check("dpipe_wan_norm_rope_bwd", a->batch, a->seq, a->heads, a->nproj);
  if (rc) return rc;
  WanNormBwdParams p;
  for (int i = 0; i < 3; ++i) p.proj[i] = WanNormBwdProj{nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, 0};
  for (int i = 0; i < a->nproj; ++i) {
    const dpipe_wan_norm_bwd_proj& s = a->proj[i];
    if (!s.dy || !s.dx || s.ld % 8 || s.ld < a->heads * 128) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_bwd: projection %d: bad pointers / ld", i);
    if (s.weight && (!s.xhat || !s.rstd || !s.dw_partials)) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_bwd: projection %d: missing saved statistics", i);
    if (s.rope && (!a->cos || !a->sin)) return fail(DPIPE_EINVAL, "dpipe_wan_norm_rope_bwd: rope requested without tables");
    p.proj[i] = WanNormBwdProj{(const __nv_bfloat16*)s.dy, (const __nv_bfloat16*)s.xhat, s.rstd, (const __nv_bfloat16*)s.weight,
                               (__nv_bfloat16*)s.dx, s.ld, s.dw_partials, s.rope};
  }
  p.cos = a->cos; p.sin = a->sin; p.B = a->batch; p.L = a->seq; p.H = a->heads;
  const int rows = a->batch * a->seq;
  dim3 grid((rows + WN_ROWS - 1) / WN_ROWS, a->nproj);
  wan_norm_rope_bwd_kernel<<<grid, a->heads * 16, 0, (cudaStream_t)stream>>>(p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
