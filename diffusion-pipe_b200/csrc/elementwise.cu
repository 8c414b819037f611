// HBM-bound kernels around the GEMMs of a DiT block: LayerNorm+modulation (fwd/bwd), gated-residual backward,
// q/k RMSNorm + RoPE backward, column sums (bias grads), and the masked MSE loss.
//
// Layout conventions: activations are token-major bf16 [batch*rows_per_batch, ld]; modulation vectors are
// bf16 [batch, mod_stride] slices; reductions over rows are done without atomics in two stages:
// every CTA owns DPIPE_ROW_CHUNK rows of one sample and writes fp32 partial column sums
// partials[batch][nchunk][2][D]; dpipe_colreduce_finish folds them.
//
// Thread mapping: one thread owns 8 consecutive columns (one 16-byte vector); a CTA of D/8 threads covers a row.
//
// Replaces the unfused ATen elementwise / LayerNorm kernels the reference runs inside the diffusers Flux blocks
// (AdaLayerNormZero, gate*out+residual, RMSNorm(q,k), apply_rotary_emb; reference call sites models/flux.py:502,525)
// and F.mse_loss in models/base.py:418-436.
#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int ROW_CHUNK = 16;  // rows handled by one CTA in the backward reductions
constexpr int RG = 4;          // rows processed together (amortises block reductions)

__device__ __forceinline__ void unpack8(const uint4& q, float* f) {
  f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
  f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 q;
  q.x = pack_bf16(f[0], f[1]); q.y = pack_bf16(f[2], f[3]); q.z = pack_bf16(f[4], f[5]); q.w = pack_bf16(f[6], f[7]);
  return q;
}

// sums NV values per thread across the CTA; result broadcast to all threads.  `red` is smem [32][NV].
template <int NV>
__device__ __forceinline__ void block_sum(float* v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], off);
  }
  __syncthreads();  // protect `red` from the previous use
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < NV; ++i) red[warp * NV + i] = v[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float s = 0.f;
    for (int w = 0; w < nwarp; ++w) s += red[w * NV + i];
    v[i] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (no affine) + modulation:  out = LN(x) * bf16(1 + scale[b]) + shift[b]
// grid (ceil(rows_per_batch / RG), batch), block D/8 threads
// ---------------------------------------------------------------------------------------------
__global__ void ln_modulate_fwd_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                       const __nv_bfloat16* __restrict__ scale, const __nv_bfloat16* __restrict__ shift,
                                       int64_t mod_stride, __nv_bfloat16* __restrict__ out, int64_t ldo,
                                       float* __restrict__ mean_out, float* __restrict__ rstd_out, int rows_per_batch,
                                       int D, float eps, int flags) {
  __shared__ float red[32 * RG];
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * RG;
  const int col = threadIdx.x * 8;
  float xv[RG][8];
  float s[RG];
#pragma unroll
  for (int i = 0; i < RG; ++i) {
    const int r = r0 + i;
    if (r < rows_per_batch) {
      unpack8(*reinterpret_cast<const uint4*>(x + ((int64_t)b * rows_per_batch + r) * ldx + col), xv[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) xv[i][j] = 0.f;
    }
    s[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s[i] += xv[i][j];
  }
  block_sum<RG>(s, red);
  float mean[RG], var[RG];
#pragma unroll
  for (int i = 0; i < RG; ++i) {
    mean[i] = s[i] / D;
    var[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = xv[i][j] - mean[i]; var[i] += d * d; }
  }
  block_sum<RG>(var, red);
  float sc[8], sh[8];
  unpack8(*reinterpret_cast<const uint4*>(scale + (int64_t)b * mod_stride + col), sc);
  unpack8(*reinterpret_cast<const uint4*>(shift + (int64_t)b * mod_stride + col), sh);
  if (!(flags & DPIPE_LN_MULT_DIRECT)) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sc[j] = bf16_round(1.0f + sc[j]);  // (1 + scale) is formed in bf16 by the reference
  }
  const bool steps = flags & DPIPE_LN_ROUND_STEPS;
#pragma unroll
  for (int i = 0; i < RG; ++i) {
    const int r = r0 + i;
    if (r >= rows_per_batch) continue;
    const float rstd = rsqrtf(var[i] / D + eps);
    float o[8];
    if (steps) {   // every elementwise op of the reference yields a bf16 tensor (Wan: norm(x) * (1 + e1) + e0)
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = bf16_round(bf16_round((xv[i][j] - mean[i]) * rstd) * sc[j]) + sh[j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (xv[i][j] - mean[i]) * rstd * sc[j] + sh[j];
    }
    const int64_t row = (int64_t)b * rows_per_batch + r;
    *reinterpret_cast<uint4*>(out + row * ldo + col) = pack8(o);
    if (threadIdx.x == 0 && mean_out) { mean_out[row] = mean[i]; rstd_out[row] = rstd; }
  }
}

// backward: g = dxn * bf16(1+scale);  dx = rstd * (g - mean(g) - xhat * mean(g*xhat)) (+ dres)
// partial column sums: slot 0 = sum_rows dxn * xhat (dscale), slot 1 = sum_rows dxn (dshift)
// grid (nchunk, batch), block D/8 threads.  RGT rows are processed together; MAXT bounds the block size so that the
// register file holds it: <4, 512> (128 registers, D <= 4096: Flux / Qwen 3072) and <2, 1024> (64 registers, D <= 8192:
// Wan 5120 = 640 threads, which 128 registers per thread do not fit).
template <int RGT, int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) ln_modulate_bwd_kernel(const __nv_bfloat16* __restrict__ dxn, int64_t lddxn,
                                       const __nv_bfloat16* __restrict__ x, int64_t ldx,
                                       const __nv_bfloat16* __restrict__ scale, int64_t mod_stride,
                                       const float* __restrict__ mean_in, const float* __restrict__ rstd_in,
                                       const __nv_bfloat16* __restrict__ dres, int64_t lddres,
                                       __nv_bfloat16* __restrict__ dx, int64_t lddx, float* __restrict__ partials,
                                       int rows_per_batch, int D, int flags) {
  __shared__ float red[32 * 2 * RGT];
  const int b = blockIdx.y;
  const int col = threadIdx.x * 8;
  float sc[8];
  unpack8(*reinterpret_cast<const uint4*>(scale + (int64_t)b * mod_stride + col), sc);
  if (!(flags & DPIPE_LN_MULT_DIRECT)) {
#pragma unroll
    for (int j = 0; j < 8; ++j) sc[j] = bf16_round(1.0f + sc[j]);
  }
  float acc_scale[8], acc_shift[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { acc_scale[j] = 0.f; acc_shift[j] = 0.f; }
  const int rbeg = blockIdx.x * ROW_CHUNK;
  for (int r0 = rbeg; r0 < rbeg + ROW_CHUNK; r0 += RGT) {
    float g[RGT][8], xh[RGT][8], rs[RGT];
    float sums[2 * RGT];
    uint4 rraw[RGT];
#pragma unroll
    for (int i = 0; i < RGT; ++i) {
      const int r = r0 + i;
      sums[2 * i] = 0.f; sums[2 * i + 1] = 0.f;
      if (r < rows_per_batch) {
        const int64_t row = (int64_t)b * rows_per_batch + r;
        float xv[8], dv[8];
        // all three inputs of the row are requested before the block reduction (r2: the residual gradient used to be loaded
        // after it, a third serialised DRAM latency per row group in a kernel that runs at 1-2 CTAs per SM)
        const uint4 xraw = *reinterpret_cast<const uint4*>(x + row * ldx + col);
        const uint4 draw = *reinterpret_cast<const uint4*>(dxn + row * lddxn + col);
        if (dres) rraw[i] = *reinterpret_cast<const uint4*>(dres + row * lddres + col);
        unpack8(xraw, xv);
        unpack8(draw, dv);
        const float m = mean_in[row];
        rs[i] = rstd_in[row];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          xh[i][j] = (xv[j] - m) * rs[i];
          g[i][j] = dv[j] * sc[j];
          acc_scale[j] += dv[j] * xh[i][j];
          acc_shift[j] += dv[j];
          sums[2 * i] += g[i][j];
          sums[2 * i + 1] += g[i][j] * xh[i][j];
        }
      } else {
        rs[i] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { g[i][j] = 0.f; xh[i][j] = 0.f; }
      }
    }
    block_sum<2 * RGT>(sums, red);
#pragma unroll
    for (int i = 0; i < RGT; ++i) {
      const int r = r0 + i;
      if (r >= rows_per_batch) continue;
      const int64_t row = (int64_t)b * rows_per_batch + r;
      const float m1 = sums[2 * i] / D, m2 = sums[2 * i + 1] / D;
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = rs[i] * (g[i][j] - m1 - xh[i][j] * m2);
      if (dres) {
        float rv[8];
        unpack8(rraw[i], rv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] += rv[j];
      }
      *reinterpret_cast<uint4*>(dx + row * lddx + col) = pack8(o);
    }
  }
  float* pp = partials + (((int64_t)b * gridDim.x + blockIdx.x) * 2) * D + col;
#pragma unroll
  for (int j = 0; j < 8; ++j) { pp[j] = acc_scale[j]; pp[D + j] = acc_shift[j]; }
}

// gated residual backward:  x_new = res + gate[b]*y   =>   dy = gate*dx ; dgate[b] = sum_rows dx*y ; dbias = sum dy
// partial slot 0 = dx*y (per sample), slot 1 = dy.  grid (nchunk, batch), block D/8 threads
__global__ void gate_bwd_kernel(const __nv_bfloat16* __restrict__ dxo, int64_t lddx, const __nv_bfloat16* __restrict__ y,
                                int64_t ldy, const __nv_bfloat16* __restrict__ gate, int64_t gate_stride,
                                __nv_bfloat16* __restrict__ dy, int64_t lddy, float* __restrict__ partials,
                                int rows_per_batch, int D) {
  const int b = blockIdx.y;
  const int col = threadIdx.x * 8;
  float gv[8];
  unpack8(*reinterpret_cast<const uint4*>(gate + (int64_t)b * gate_stride + col), gv);
  float a0[8], a1[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { a0[j] = 0.f; a1[j] = 0.f; }
  const int rbeg = blockIdx.x * ROW_CHUNK;
  const int rend = min(rbeg + ROW_CHUNK, rows_per_batch);
#pragma unroll 4
  for (int r = rbeg; r < rend; ++r) {
    const int64_t row = (int64_t)b * rows_per_batch + r;
    float dv[8], yv[8], o[8];
    unpack8(*reinterpret_cast<const uint4*>(dxo + row * lddx + col), dv);
    unpack8(*reinterpret_cast<const uint4*>(y + row * ldy + col), yv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j] = bf16_round(gv[j] * dv[j]);
      a0[j] += dv[j] * yv[j];
      a1[j] += o[j];
    }
    *reinterpret_cast<uint4*>(dy + row * lddy + col) = pack8(o);
  }
  float* pp = partials + (((int64_t)b * gridDim.x + blockIdx.x) * 2) * D + col;
#pragma unroll
  for (int j = 0; j < 8; ++j) { pp[j] = a0[j]; pp[D + j] = a1[j]; }
}

// plain column sums of a bf16 matrix (bias gradients): slot 0 = sum_rows x.  grid (nchunk, 1), block N/8 threads
__global__ void colsum_kernel(const __nv_bfloat16* __restrict__ x, int64_t ldx, float* __restrict__ partials, int rows,
                              int N, int rows_per_cta) {
  const int col = (blockIdx.y * blockDim.x + threadIdx.x) * 8;
  if (col >= N) return;
  float a[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) a[j] = 0.f;
  const int rbeg = blockIdx.x * rows_per_cta;
  const int rend = min(rbeg + rows_per_cta, rows);
#pragma unroll 4
  for (int r = rbeg; r < rend; ++r) {
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(x + (int64_t)r * ldx + col), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += v[j];
  }
  float* pp = partials + (int64_t)blockIdx.x * N + col;
#pragma unroll
  for (int j = 0; j < 8; ++j) pp[j] = a[j];
}

// folds partials[batch][nchunk][nslot][D]; slot s goes to per_sample[s][b*ld[s] + d] (if non-null) and/or
// summed[s][d] (sum over samples, if non-null)
struct FinishArgs {
  float* per_sample[2];
  int64_t ld[2];
  float* summed[2];
};
__global__ void colreduce_finish_kernel(const float* __restrict__ partials, int batch, int nchunk, int nslot, int D,
                                        FinishArgs fa) {
  // block = 32 columns x 8 chunk groups; grid = (D/32, nslot)
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int d = blockIdx.x * 32 + tx;
  const int s = blockIdx.y;
  float total = 0.f;
  for (int b = 0; b < batch; ++b) {
    float acc = 0.f;
    if (d < D) {
      const float* p = partials + (((int64_t)b * nchunk) * nslot + s) * D + d;
      for (int c = ty; c < nchunk; c += 8) acc += p[(int64_t)c * nslot * D];
    }
    red[ty][tx] = acc;
    __syncthreads();
    if (ty == 0) {
      float v = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) v += red[k][tx];
      if (d < D && fa.per_sample[s]) fa.per_sample[s][(int64_t)b * fa.ld[s] + d] = v;
      total += v;
    }
    __syncthreads();
  }
  if (ty == 0 && d < D && fa.summed[s]) fa.summed[s][d] = total;
}

// ---------------------------------------------------------------------------------------------
// backward of (bias ->) per-head RMSNorm -> RoPE for q and k, plus the head-major -> token-major gather of dq/dk/dv.
// One warp walks the tokens of one (sample, head, which in {q,k,v}) slice; each lane owns 4 of the 128 channels.
// grid (ceil(rows_per_batch / TOK_PER_WARP / warps), heads*3, batch)
// ---------------------------------------------------------------------------------------------
constexpr int QK_TOK_PER_WARP = 32;    // (r2: 128 left 17 warps per SM in flight: 0.35 of the HBM peak under ncu)
struct QkBwdParams {
  const __nv_bfloat16 *dq, *dk, *dv;      // [B,H,seq_total,128]
  const __nv_bfloat16 *qhat, *khat;       // [B,H,seq_total,128]
  const float *q_rstd, *k_rstd;           // [B,H,seq_total]
  const __nv_bfloat16 *wq, *wk;           // [128]
  const float *cos, *sin;                 // [seq_total,128]
  __nv_bfloat16* dqkv; int64_t ld;        // [B*rows_per_batch, >= 3*H*128] token-major
  float* dbias;                           // fp32 [3*H*128], atomically accumulated (must be zeroed by the caller)
  float* dw;                              // fp32 [2][128] norm-weight grads, atomically accumulated
  int heads, seq_total, seq_offset, rows_per_batch;
};
__global__ void qknorm_rope_bwd_kernel(const QkBwdParams p) {
  const int lane = threadIdx.x & 31;
  const int wglobal = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int head = blockIdx.y % p.heads, which = blockIdx.y / p.heads;
  const int b = blockIdx.z;
  __shared__ float cta_sum[4][2][128];   // per-warp partial column sums, folded before touching global atomics
  const int t0 = min(wglobal * QK_TOK_PER_WARP, p.rows_per_batch);
  const int t1 = min(t0 + QK_TOK_PER_WARP, p.rows_per_batch);   // (possibly empty: the warp still joins the reduction)
  const int c0 = lane * 4;
  const __nv_bfloat16* src = which == 0 ? p.dq : (which == 1 ? p.dk : p.dv);
  const int64_t hb = ((int64_t)b * p.heads + head) * p.seq_total;
  float bsum[4] = {0.f, 0.f, 0.f, 0.f}, wsum[4] = {0.f, 0.f, 0.f, 0.f};
  float wv[4] = {0.f, 0.f, 0.f, 0.f};
  if (which < 2) {
    const uint2 w2 = *reinterpret_cast<const uint2*>((which == 0 ? p.wq : p.wk) + c0);
    wv[0] = bf16_lo(w2.x); wv[1] = bf16_hi(w2.x); wv[2] = bf16_lo(w2.y); wv[3] = bf16_hi(w2.y);
  }
  constexpr int TB = 4;   // tokens in flight per warp: all loads of a group are issued before any dependent math
  const __nv_bfloat16* hat = which == 0 ? p.qhat : p.khat;
  const float* rstd_p = which == 0 ? p.q_rstd : p.k_rstd;
  for (int tb = t0; tb < t1; tb += TB) {
    uint2 g2[TB], h2[TB];
    float4 cs[TB], sn[TB];
    float rs[TB];
#pragma unroll
    for (int u = 0; u < TB; ++u) {
      const int t = min(tb + u, t1 - 1);
      const int pos = p.seq_offset + t;
      g2[u] = *reinterpret_cast<const uint2*>(src + (hb + pos) * 128 + c0);
      if (which < 2) {
        cs[u] = *reinterpret_cast<const float4*>(p.cos + (int64_t)pos * 128 + c0);
        sn[u] = *reinterpret_cast<const float4*>(p.sin + (int64_t)pos * 128 + c0);
        h2[u] = *reinterpret_cast<const uint2*>(hat + (hb + pos) * 128 + c0);
        rs[u] = rstd_p[hb + pos];
      }
    }
    float o[TB][4], xh[TB][4], dxh[TB][4], dot[TB];
#pragma unroll
    for (int u = 0; u < TB; ++u) {
      const float g[4] = {bf16_lo(g2[u].x), bf16_hi(g2[u].x), bf16_lo(g2[u].y), bf16_hi(g2[u].y)};
      const bool live = tb + u < t1;
      if (which == 2) {
#pragma unroll
        for (int j = 0; j < 4; ++j) o[u][j] = g[j];
      } else {
        // transpose of the rotation  out[2i] = y[2i]c[2i] - y[2i+1]s[2i] ;  out[2i+1] = y[2i+1]c[2i+1] + y[2i]s[2i+1]
        float dy[4];
        dy[0] = g[0] * cs[u].x + g[1] * sn[u].y;
        dy[1] = g[1] * cs[u].y - g[0] * sn[u].x;
        dy[2] = g[2] * cs[u].z + g[3] * sn[u].w;
        dy[3] = g[3] * cs[u].w - g[2] * sn[u].z;
        xh[u][0] = bf16_lo(h2[u].x); xh[u][1] = bf16_hi(h2[u].x); xh[u][2] = bf16_lo(h2[u].y); xh[u][3] = bf16_hi(h2[u].y);
        dot[u] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (live) wsum[j] += dy[j] * xh[u][j];
          dxh[u][j] = dy[j] * wv[j];
          dot[u] += dxh[u][j] * xh[u][j];
        }
      }
    }
    if (which < 2) {
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
        for (int u = 0; u < TB; ++u) dot[u] += __shfl_xor_sync(0xffffffffu, dot[u], off);
      }
#pragma unroll
      for (int u = 0; u < TB; ++u) {
        const float d = dot[u] * (1.0f / 128.0f);
#pragma unroll
        for (int j = 0; j < 4; ++j) o[u][j] = rs[u] * (dxh[u][j] - xh[u][j] * d);
      }
    }
#pragma unroll
    for (int u = 0; u < TB; ++u) {
      if (tb + u >= t1) continue;
      const int t = tb + u;
      uint2 ov;
      ov.x = pack_bf16(o[u][0], o[u][1]);
      ov.y = pack_bf16(o[u][2], o[u][3]);
      bsum[0] += bf16_lo(ov.x); bsum[1] += bf16_hi(ov.x); bsum[2] += bf16_lo(ov.y); bsum[3] += bf16_hi(ov.y);
      *reinterpret_cast<uint2*>(p.dqkv + ((int64_t)b * p.rows_per_batch + t) * p.ld + (which * p.heads + head) * 128 + c0) = ov;
    }
  }
  const int wid = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 4; ++j) { cta_sum[wid][0][c0 + j] = bsum[j]; cta_sum[wid][1][c0 + j] = wsum[j]; }
  __syncthreads();
  // 256 threads-worth of sums (2 x 128): every thread of the CTA folds one or two entries over the 4 warps
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    const int kind = i >> 7, c = i & 127;
    float v = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) v += cta_sum[w][kind][c];
    if (kind == 0) atomicAdd(p.dbias + (which * p.heads + head) * 128 + c, v);
    else if (which < 2) atomicAdd(p.dw + which * 128 + c, v);
  }
}

// ---------------------------------------------------------------------------------------------
// masked MSE: loss = mean((out - target)^2 * mask) ; dout = 2 (out - target) mask / numel   (models/base.py:418-436)
// ---------------------------------------------------------------------------------------------
__global__ void mse_loss_kernel(const __nv_bfloat16* __restrict__ out, const float* __restrict__ target,
                                const float* __restrict__ mask, int64_t numel, float* __restrict__ block_sums,
                                __nv_bfloat16* __restrict__ dout) {
  __shared__ float red[32];
  float acc = 0.f;
  const float inv_n = 1.0f / (float)numel;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = __bfloat162float(out[i]) - target[i];
    const float m = mask ? mask[i] : 1.0f;
    acc += d * d * m;
    if (dout) dout[i] = __float2bfloat16_rn(2.0f * d * m * inv_n);
  }
  float v[1] = {acc};
  block_sum<1>(v, red);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = v[0];
}
__global__ void mse_finish_kernel(const float* __restrict__ block_sums, int n, int64_t numel, float* __restrict__ loss) {
  __shared__ float red[32];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += block_sums[i];
  float v[1] = {acc};
  block_sum<1>(v, red);
  if (threadIdx.x == 0) *loss = v[0] / (float)numel;
}

static int check_cols(const char* what, int D) {
  // D/8 threads per CTA must be whole warps (full-mask shuffles) and fit one CTA
  if (D % 256 != 0 || D / 8 > 1024 || D <= 0) return fail(DPIPE_EINVAL, "%s: D=%d must be a multiple of 256 and <= 8192", what, D);
  return 0;
}

}  // namespace dpipe

using namespace dpipe;
typedef __nv_bfloat16 bf16;

extern "C" int dpipe_row_chunk(void) { return ROW_CHUNK; }

extern "C" int dpipe_ln_modulate_fwd(const void* x, int64_t ldx, const void* scale, const void* shift, int64_t mod_stride,
                                     void* out, int64_t ldo, float* mean, float* rstd, int batch, int rows_per_batch, int D,
                                     float eps, void* stream) {
  return dpipe_ln_modulate_fwd_ex(x, ldx, scale, shift, mod_stride, out, ldo, mean, rstd, batch, rows_per_batch, D, eps, 0, stream);
}

extern "C" int dpipe_ln_modulate_fwd_ex(const void* x, int64_t ldx, const void* scale, const void* shift, int64_t mod_stride,
                                        void* out, int64_t ldo, float* mean, float* rstd, int batch, int rows_per_batch, int D,
                                        float eps, int flags, void* stream) {
  int rc = check_cols("dpipe_ln_modulate_fwd", D);
  if (rc) return rc;
  if (!x || !scale || !shift || !out) return fail(DPIPE_EINVAL, "dpipe_ln_modulate_fwd: null pointer");
  if (ldx % 8 || ldo % 8 || mod_stride % 8) return fail(DPIPE_EINVAL, "dpipe_ln_modulate_fwd: strides must be multiples of 8");
  if (D > 6144) return fail(DPIPE_EINVAL, "dpipe_ln_modulate_fwd: D=%d > 6144 (one CTA of D/8 threads at 79 registers must fit the register file)", D);
  dim3 grid((rows_per_batch + RG - 1) / RG, batch);
  ln_modulate_fwd_kernel<<<grid, D / 8, 0, (cudaStream_t)stream>>>((const bf16*)x, ldx, (const bf16*)scale, (const bf16*)shift,
                                                                    mod_stride, (bf16*)out, ldo, mean, rstd, rows_per_batch, D, eps, flags);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_ln_modulate_bwd(const void* dxn, int64_t lddxn, const void* x, int64_t ldx, const void* scale,
                                     int64_t mod_stride, const float* mean, const float* rstd, const void* dres,
                                     int64_t lddres, void* dx, int64_t lddx, float* partials, int batch, int rows_per_batch,
                                     int D, void* stream) {
  return dpipe_ln_modulate_bwd_ex(dxn, lddxn, x, ldx, scale, mod_stride, mean, rstd, dres, lddres, dx, lddx, partials, batch,
                                  rows_per_batch, D, 0, stream);
}

extern "C" int dpipe_ln_modulate_bwd_ex(const void* dxn, int64_t lddxn, const void* x, int64_t ldx, const void* scale,
                                        int64_t mod_stride, const float* mean, const float* rstd, const void* dres,
                                        int64_t lddres, void* dx, int64_t lddx, float* partials, int batch, int rows_per_batch,
                                        int D, int flags, void* stream) {
  int rc = check_cols("dpipe_ln_modulate_bwd", D);
  if (rc) return rc;
  if (!dxn || !x || !scale || !mean || !rstd || !dx || !partials) return fail(DPIPE_EINVAL, "dpipe_ln_modulate_bwd: null pointer");
  dim3 grid((rows_per_batch + ROW_CHUNK - 1) / ROW_CHUNK, batch);
#define DPIPE_LN_BWD_LAUNCH(RGT, MAXT, MINB)                                                                                     \
  ln_modulate_bwd_kernel<RGT, MAXT, MINB><<<grid, D / 8, 0, (cudaStream_t)stream>>>(                                             \
      (const bf16*)dxn, lddxn, (const bf16*)x, ldx, (const bf16*)scale, mod_stride, mean, rstd, (const bf16*)dres, lddres,       \
      (bf16*)dx, lddx, partials, rows_per_batch, D, flags)
  // block = D / 8 threads; the register cap follows the block size so that D = 3072 (Flux / Qwen) runs TWO 384-thread CTAs per
  // SM at <= 85 registers and D = 5120 (Wan) one 640-thread CTA at <= 102 (r2: 1 CTA / SM and 0.2 of the HBM peak under ncu)
  if (D <= 3072) DPIPE_LN_BWD_LAUNCH(2, 384, 2);
  else if (D <= 4096) DPIPE_LN_BWD_LAUNCH(2, 512, 1);
  else if (D <= 5120) DPIPE_LN_BWD_LAUNCH(2, 640, 1);
  else DPIPE_LN_BWD_LAUNCH(2, 1024, 1);
#undef DPIPE_LN_BWD_LAUNCH
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_gate_bwd(const void* dxo, int64_t lddx, const void* y, int64_t ldy, const void* gate, int64_t gate_stride,
                              void* dy, int64_t lddy, float* partials, int batch, int rows_per_batch, int D, void* stream) {
  int rc = check_cols("dpipe_gate_bwd", D);
  if (rc) return rc;
  if (!dxo || !y || !gate || !dy || !partials) return fail(DPIPE_EINVAL, "dpipe_gate_bwd: null pointer");
  dim3 grid((rows_per_batch + ROW_CHUNK - 1) / ROW_CHUNK, batch);
  gate_bwd_kernel<<<grid, D / 8, 0, (cudaStream_t)stream>>>((const bf16*)dxo, lddx, (const bf16*)y, ldy, (const bf16*)gate,
                                                             gate_stride, (bf16*)dy, lddy, partials, rows_per_batch, D);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_colreduce_finish(const float* partials, int batch, int nchunk, int nslot, int D, float* per_sample0,
                                      int64_t ld0, float* per_sample1, int64_t ld1, float* summed0, float* summed1,
                                      void* stream) {
  if (!partials || nslot < 1 || nslot > 2) return fail(DPIPE_EINVAL, "dpipe_colreduce_finish: bad arguments");
  FinishArgs fa;
  fa.per_sample[0] = per_sample0; fa.per_sample[1] = per_sample1;
  fa.ld[0] = ld0; fa.ld[1] = ld1;
  fa.summed[0] = summed0; fa.summed[1] = summed1;
  dim3 grid((D + 31) / 32, nslot);
  colreduce_finish_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(partials, batch, nchunk, nslot, D, fa);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// column sums of a bf16 [rows, N] matrix into fp32 out[N]; `partials` needs dpipe_colsum_chunks(rows) * N floats
extern "C" int dpipe_colsum_chunks(int rows) { return (rows + 63) / 64; }
extern "C" int dpipe_colsum(const void* x, int64_t ldx, int rows, int N, float* partials, float* out, void* stream) {
  if (!x || !partials || !out || N % 8 || ldx % 8) return fail(DPIPE_EINVAL, "dpipe_colsum: bad arguments");
  const int nchunk = dpipe_colsum_chunks(rows);
  const int threads = 128;
  dim3 grid(nchunk, (N / 8 + threads - 1) / threads);
  colsum_kernel<<<grid, threads, 0, (cudaStream_t)stream>>>((const bf16*)x, ldx, partials, rows, N, 64);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  FinishArgs fa = {};
  fa.summed[0] = out;
  colreduce_finish_kernel<<<dim3((N + 31) / 32, 1), 256, 0, (cudaStream_t)stream>>>(partials, 1, nchunk, 1, N, fa);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_qknorm_rope_bwd(const dpipe_qk_bwd_args* a, void* stream) {
  if (!a || !a->dq || !a->dk || !a->dv || !a->qhat || !a->khat || !a->q_rstd || !a->k_rstd || !a->q_norm_w || !a->k_norm_w ||
      !a->rope_cos || !a->rope_sin || !a->dqkv || !a->dbias || !a->dw)
    return fail(DPIPE_EINVAL, "dpipe_qknorm_rope_bwd: null pointer");
  if (a->ld % 8 || a->seq_offset + a->rows_per_batch > a->seq_total) return fail(DPIPE_EINVAL, "dpipe_qknorm_rope_bwd: bad geometry");
  QkBwdParams p;
  p.dq = (const bf16*)a->dq; p.dk = (const bf16*)a->dk; p.dv = (const bf16*)a->dv;
  p.qhat = (const bf16*)a->qhat; p.khat = (const bf16*)a->khat;
  p.q_rstd = a->q_rstd; p.k_rstd = a->k_rstd;
  p.wq = (const bf16*)a->q_norm_w; p.wk = (const bf16*)a->k_norm_w;
  p.cos = a->rope_cos; p.sin = a->rope_sin;
  p.dqkv = (bf16*)a->dqkv; p.ld = a->ld;
  p.dbias = a->dbias; p.dw = a->dw;
  p.heads = a->heads; p.seq_total = a->seq_total; p.seq_offset = a->seq_offset; p.rows_per_batch = a->rows_per_batch;
  const int warps_per_cta = 4;
  const int nwarp = (a->rows_per_batch + QK_TOK_PER_WARP - 1) / QK_TOK_PER_WARP;
  dim3 grid((nwarp + warps_per_cta - 1) / warps_per_cta, a->heads * 3, a->batch);
  qknorm_rope_bwd_kernel<<<grid, warps_per_cta * 32, 0, (cudaStream_t)stream>>>(p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// workspace: 1024 floats
extern "C" int dpipe_mse_loss(const void* out, const float* target, const float* mask, int64_t numel, float* workspace,
                              float* loss, void* dout, void* stream) {
  if (!out || !target || !workspace || !loss || numel <= 0) return fail(DPIPE_EINVAL, "dpipe_mse_loss: bad arguments");
  int blocks = (int)((numel + 256 * 8 - 1) / (256 * 8));
  if (blocks > 1024) blocks = 1024;
  mse_loss_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const bf16*)out, target, mask, numel, workspace, (bf16*)dout);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  mse_finish_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(workspace, blocks, numel, loss);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
