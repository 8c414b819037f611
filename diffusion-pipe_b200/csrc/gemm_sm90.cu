// Warp-specialised persistent bf16 GEMM for sm_90a, 128x256 output tiles:
//   TMA (128B-swizzled tiles) -> shared memory ring -> wgmma (two consumer warpgroups, 64 rows x 256 columns
//   each, fp32 accumulators in registers) -> fp32 tile staged, one 64-column quarter at a time, in a buffer of each
//   warpgroup's own -> coalesced fused epilogue.  One CTA per SM walks the tiles; the producer warp keeps loading the
//   next tile's k-blocks into the ring while the consumers run the epilogue of the last one.
//
//   D[M,N] = Aop[M,K] * Bop[N,K]^T.  Each operand may be K-major (reduction dim contiguous) or
//   MN-major (non-reduced dim contiguous), so forward (X*W^T), dgrad (dY*W) and wgrad (dY^T*X) all run
//   on the same kernel without a transpose pass.
//
//   The ABI keeps its cta_group field (1 or 2) for compatibility; sm_90a has no paired-CTA MMA, so both values run this
//   kernel and produce the same result.
//
// Replaces the cuBLASLt GEMMs behind nn.Linear in the reference's Flux blocks
// (reference: models/flux.py:502,525 and SURVEY.md section 2.3 shapes).
#include <stdlib.h>

#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int BM = 128;  // rows per tile (two consumer warpgroups of 64)
constexpr int BN = 256;  // columns per tile (wgmma N)
constexpr int BK = 64;   // K per pipeline stage = one 128-byte swizzle row of bf16
constexpr int UK = 16;   // K per wgmma
constexpr int A_TILE_BYTES = BM * BK * 2;  // 16 KiB
constexpr int B_TILE_BYTES = BN * BK * 2;  // 32 KiB
constexpr int SUB_BYTES = 64 * 64 * 2;     // one 64(mn) x 64(k) MN-major sub-tile = 8 KiB
constexpr int STAGE_BYTES = A_TILE_BYTES + B_TILE_BYTES;
constexpr int STAGES = 4;                  // 192 KiB of operand staging
constexpr int EPI_SMEM_BYTES = 2 * (64 * 64 * 4 + 64 * 4);  // each warpgroup: a fp32 64x64 quarter + 64 rstd
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_SMEM_BYTES + 256 /*barriers*/ + 1024 /*align slack*/;
constexpr int GEMM_THREADS = 384;  // warps 0-7: two consumer warpgroups; warpgroup 2: warp 8 is the TMA producer
// the producer warpgroup gives its registers to the consumers: 128 x 40 + 256 x 232 <= 64 Ki
constexpr int PRODUCER_REGS = 40;
constexpr int CONSUMER_REGS = 232;
static_assert(SMEM_BYTES <= 227 * 1024, "ring, epilogue buffers and barriers must fit one SM's shared memory");

struct GemmParams {
  int M, N, K;
  int num_m_tiles;  // tiles of BM rows
  int num_tiles;
  __nv_bfloat16* out;
  int64_t ldo;
  __nv_bfloat16* out2;
  int64_t ldo2;
  const __nv_bfloat16* bias;
  const __nv_bfloat16* aux;
  int64_t ldaux;
  const __nv_bfloat16* gate;
  int64_t gate_stride;
  int rows_per_batch;
  int accumulate;
  dpipe_qkv_epilogue qkv;
};

// ---------------------------------------------------------------------------------------------
// epilogue: each consumer warpgroup stages its 64 rows of the tile one 64-column quarter at a time in a buffer of its
// own (not the operand ring, so the producer keeps loading the next tile meanwhile) and drains the quarter row by row:
// a thread takes 8 consecutive columns of 4 rows, so 8 lanes cover one row's 64 columns and every global access of a
// warp touches 4 contiguous 128-byte row segments.  Each output element sees the same fp32 operations as when one
// thread walked a whole row.
// ---------------------------------------------------------------------------------------------
constexpr int EPI_COLS = 64;          // columns per staged quarter
constexpr int EPI_ROWS = 4;           // rows per thread and quarter
constexpr int STG_FLOATS = 64 * EPI_COLS;

// staged fp32 quarter [64 rows][64 columns]: the 16-byte chunk c of row r lives at chunk c ^ (r & 7), so both the
// fragment writes (8 rows x 32 B per instruction) and the drain reads (4 rows x 128 B) take the fewest wavefronts
__device__ __forceinline__ int stg_idx(int r, int c) { return r * EPI_COLS + ((((c >> 2) ^ r) & 7) << 2) + ((c >> 2) & 8) * 4 + (c & 3); }

template <int Q>
__device__ __forceinline__ void stage_q(const float* acc, float* stg, int r0, int c0) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int a = 4 * (8 * Q + j), c = 8 * j + c0;
    *reinterpret_cast<float2*>(stg + stg_idx(r0, c)) = make_float2(acc[a], acc[a + 1]);
    *reinterpret_cast<float2*>(stg + stg_idx(r0 + 8, c)) = make_float2(acc[a + 2], acc[a + 3]);
  }
}
// accumulator columns [64q, 64q + 64) of the warpgroup's fragment -> stg (a switch keeps every acc index constant)
__device__ __forceinline__ void stage_quarter(const float* acc, float* stg, int q, int w4, int lane) {
  const int r0 = w4 * 16 + (lane >> 2), c0 = 2 * (lane & 3);
  switch (q) {
    case 0: stage_q<0>(acc, stg, r0, c0); break;
    case 1: stage_q<1>(acc, stg, r0, c0); break;
    case 2: stage_q<2>(acc, stg, r0, c0); break;
    default: stage_q<3>(acc, stg, r0, c0); break;
  }
}

__device__ __forceinline__ void ld_stg8(const float* stg, int r, int c, float* f) {
  const float4 lo = *reinterpret_cast<const float4*>(stg + stg_idx(r, c));
  const float4 hi = *reinterpret_cast<const float4*>(stg + stg_idx(r, c + 4));
  f[0] = lo.x; f[1] = lo.y; f[2] = lo.z; f[3] = lo.w; f[4] = hi.x; f[5] = hi.y; f[6] = hi.z; f[7] = hi.w;
}
__device__ __forceinline__ uint4 ld_u4(const void* p) { return *reinterpret_cast<const uint4*>(p); }
__device__ __forceinline__ void unpack_bf16x8(uint4 q, float* f) {
  f[0] = bf16_lo(q.x); f[1] = bf16_hi(q.x); f[2] = bf16_lo(q.y); f[3] = bf16_hi(q.y);
  f[4] = bf16_lo(q.z); f[5] = bf16_hi(q.z); f[6] = bf16_lo(q.w); f[7] = bf16_hi(q.w);
}
__device__ __forceinline__ void load_bf16x8(const __nv_bfloat16* p, bool ok, float* f) {
  if (ok) {
    unpack_bf16x8(ld_u4(p), f);
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = 0.f;
  }
}
__device__ __forceinline__ void store_bf16x8(__nv_bfloat16* p, const float* f) {
  uint4 q;
  q.x = pack_bf16(f[0], f[1]); q.y = pack_bf16(f[2], f[3]); q.z = pack_bf16(f[4], f[5]); q.w = pack_bf16(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = q;
}

// one staged quarter of a non-QKV tile (and of the MLP half of the fused linear1); `col` is the global column of the
// thread's first element, rows row0 + rw + 4i
template <int EPI>
__device__ __forceinline__ void drain_quarter(const GemmParams& p, const float* stg, int row0, int rw, int cl, int col) {
  if (col >= p.N) return;  // N % 8 == 0: a thread's 8 columns are all in or all out
  float b[8];
  load_bf16x8(p.bias ? p.bias + col : nullptr, p.bias != nullptr, b);
  // every global input of the 4 rows is requested before the first is used
  uint4 in0[EPI_ROWS], in1[EPI_ROWS];
#pragma unroll
  for (int i = 0; i < EPI_ROWS; ++i) {
    const int row = row0 + rw + 4 * i;
    const bool ok = row < p.M;
    in0[i] = in1[i] = make_uint4(0, 0, 0, 0);
    if constexpr (EPI == DPIPE_EPI_STORE) {
      if (ok && p.accumulate) in0[i] = ld_u4(p.out + (int64_t)row * p.ldo + col);
    } else if constexpr (EPI == DPIPE_EPI_GATE_RES) {
      if (ok) {
        in0[i] = ld_u4(p.aux + (int64_t)row * p.ldaux + col);
        in1[i] = ld_u4(p.gate + (int64_t)(row / p.rows_per_batch) * p.gate_stride + col);
      }
    } else if constexpr (EPI == DPIPE_EPI_MUL_GELU_GRAD) {
      if (ok) in0[i] = ld_u4(p.aux + (int64_t)row * p.ldaux + col);
    }
  }
#pragma unroll
  for (int i = 0; i < EPI_ROWS; ++i) {
    const int rl = rw + 4 * i, row = row0 + rl;
    if (row >= p.M) continue;
    float acc[8];
    ld_stg8(stg, rl, cl, acc);
    if constexpr (EPI == DPIPE_EPI_STORE) {
      __nv_bfloat16* dst = p.out + (int64_t)row * p.ldo + col;
      float old[8];
      unpack_bf16x8(in0[i], old);
      if ((col & ~31) + 32 <= p.N) {
        if (p.accumulate) {
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += old[j];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += b[j];
        store_bf16x8(dst, acc);
      } else {
        // the partial 32-column group at the right edge (N % 32 != 0) adds the bias before the old value
        __nv_bfloat16 o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float v = acc[j] + b[j];
          if (p.accumulate) v += old[j];
          o[j] = __float2bfloat16_rn(v);
        }
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(o);
      }
    } else if constexpr (EPI == DPIPE_EPI_BIAS_GELU || EPI == DPIPE_EPI_QKV_ROPE) {
      // QKV_ROPE: columns past n_qkv are the MLP half of the fused linear1 of a single-stream block
      const int out_col = EPI == DPIPE_EPI_QKV_ROPE ? col - p.qkv.n_qkv : col;
      float u[8], h[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        u[j] = bf16_round(acc[j] + b[j]);
        h[j] = gelu_tanh(u[j]);
      }
      if (p.out2) store_bf16x8(p.out2 + (int64_t)row * p.ldo2 + out_col, u);
      store_bf16x8(p.out + (int64_t)row * p.ldo + out_col, h);
    } else if constexpr (EPI == DPIPE_EPI_GATE_RES) {
      float res[8], g[8], y[8], o[8];
      unpack_bf16x8(in0[i], res);
      unpack_bf16x8(in1[i], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        y[j] = bf16_round(acc[j] + b[j]);
        o[j] = res[j] + bf16_round(g[j] * y[j]);
      }
      if (p.out2) store_bf16x8(p.out2 + (int64_t)row * p.ldo2 + col, y);
      store_bf16x8(p.out + (int64_t)row * p.ldo + col, o);
    } else if constexpr (EPI == DPIPE_EPI_MUL_GELU_GRAD) {
      float u[8], o[8];
      unpack_bf16x8(in0[i], u);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = acc[j] * gelu_tanh_grad(u[j]);
      store_bf16x8(p.out + (int64_t)row * p.ldo + col, o);
    }
  }
}

// q / k / v columns of the fused QKV projection: the 256-wide tile holds two heads of one of q, k, v
// (the tile never straddles: heads * 128 % 256 == 0)
__device__ __forceinline__ void qkv_tile(const GemmParams& p, const float* acc, float* stg, float* rstd_s, int row0,
                                         int n0, int w4, int lane, int bar_id) {
  const dpipe_qkv_epilogue& e = p.qkv;
  const int hd = e.heads * 128;
  const int which = n0 / hd;  // 0 q, 1 k, 2 v
  const int t = w4 * 32 + lane;
  const int rw = w4 * 16 + (lane >> 3), cl = (lane & 7) * 8;
  const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(which == 0 ? e.q_norm_w : e.k_norm_w);
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(which == 0 ? e.q : which == 1 ? e.k : e.v);
  __nv_bfloat16* dst_hat = reinterpret_cast<__nv_bfloat16*>(which == 0 ? e.qhat : e.khat);
  float* dst_rstd = which == 0 ? e.q_rstd : e.k_rstd;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int col_h = n0 + hh * 128;  // global column of this head's first element
    const int head = (col_h - which * hd) >> 7;
    if (which == 2) {
#pragma unroll
      for (int qq = 0; qq < 2; ++qq) {
        named_bar_sync(bar_id, 128);
        stage_quarter(acc, stg, 2 * hh + qq, w4, lane);
        named_bar_sync(bar_id, 128);
        const int c = qq * 64 + cl;  // column inside the head
        float b[8];
        load_bf16x8(p.bias ? p.bias + col_h + c : nullptr, p.bias != nullptr, b);
#pragma unroll
        for (int i = 0; i < EPI_ROWS; ++i) {
          const int rl = rw + 4 * i, row = row0 + rl;
          if (row >= p.M) continue;
          const int batch = row / p.rows_per_batch;
          const int pos = e.seq_offset + row - batch * p.rows_per_batch;
          const int64_t o = (((int64_t)batch * e.heads + head) * e.seq_total + pos) * 128;
          float f[8];
          ld_stg8(stg, rl, cl, f);
#pragma unroll
          for (int j = 0; j < 8; ++j) f[j] += b[j];
          store_bf16x8(dst + o + c, f);
        }
      }
      continue;
    }
    // pass 1: thread t < 64 sums the squares of row t's 128 bf16-rounded projections in column order
    // (reference: RMSNorm on the bf16 Linear output)
    float ss = 0.f;
#pragma unroll
    for (int qq = 0; qq < 2; ++qq) {
      named_bar_sync(bar_id, 128);
      stage_quarter(acc, stg, 2 * hh + qq, w4, lane);
      named_bar_sync(bar_id, 128);
      if (t < 64) {
#pragma unroll 1
        for (int c = 0; c < EPI_COLS; c += 8) {
          float b[8], r[8];
          load_bf16x8(p.bias ? p.bias + col_h + qq * 64 + c : nullptr, p.bias != nullptr, b);
          ld_stg8(stg, t, c, r);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            float v = bf16_round(r[j] + b[j]);
            ss += v * v;
          }
        }
      }
    }
    if (t < 64) {
      const float rstd = rsqrtf(ss * (1.0f / 128.0f) + e.eps);
      rstd_s[t] = rstd;
      const int row = row0 + t;
      if (row < p.M && dst_rstd) {
        const int batch = row / p.rows_per_batch;
        const int pos = e.seq_offset + row - batch * p.rows_per_batch;
        dst_rstd[((int64_t)batch * e.heads + head) * e.seq_total + pos] = rstd;
      }
    }
    // pass 2: normalise, scale, rotate, store; the head's second quarter is still staged, the first is staged again
#pragma unroll
    for (int qq = 1; qq >= 0; --qq) {
      named_bar_sync(bar_id, 128);
      if (qq == 0) {
        stage_quarter(acc, stg, 2 * hh, w4, lane);
        named_bar_sync(bar_id, 128);
      }
      const int c = qq * 64 + cl;
      float b[8], wv[8];
      load_bf16x8(p.bias ? p.bias + col_h + c : nullptr, p.bias != nullptr, b);
      load_bf16x8(w + c, true, wv);
#pragma unroll
      for (int i = 0; i < EPI_ROWS; ++i) {
        const int rl = rw + 4 * i, row = row0 + rl;
        if (row >= p.M) continue;
        const int batch = row / p.rows_per_batch;
        const int pos = e.seq_offset + row - batch * p.rows_per_batch;
        const int64_t o = (((int64_t)batch * e.heads + head) * e.seq_total + pos) * 128;
        // the rope rows are requested first (registers allow one row's worth next to the live accumulators)
        const float4* pc = reinterpret_cast<const float4*>(e.rope_cos + (int64_t)pos * 128 + c);
        const float4* ps = reinterpret_cast<const float4*>(e.rope_sin + (int64_t)pos * 128 + c);
        const float4 c0 = pc[0], c1 = pc[1], s0 = ps[0], s1 = ps[1];
        const float rstd = rstd_s[rl];
        float r[8], xh[8], y[8], ro[8];
        ld_stg8(stg, rl, cl, r);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float v = bf16_round(r[j] + b[j]);
          xh[j] = bf16_round(v * rstd);
          y[j] = bf16_round(xh[j] * wv[j]);
        }
        if (dst_hat) store_bf16x8(dst_hat + o + c, xh);
        const float cs[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
        const float sn[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          ro[j] = y[j] * cs[j] - y[j + 1] * sn[j];
          ro[j + 1] = y[j + 1] * cs[j + 1] + y[j] * sn[j + 1];
        }
        store_bf16x8(dst + o + c, ro);
      }
    }
  }
}

// the fused epilogue of one tile for one consumer warpgroup: rows [row0, row0 + 64), columns [n0, n0 + 256)
template <int EPI>
__device__ __forceinline__ void epilogue_wg(const GemmParams& p, const float* acc, float* stg, float* rstd_s, int row0,
                                            int n0, int w4, int lane, int bar_id) {
  if constexpr (EPI == DPIPE_EPI_QKV_ROPE) {
    if (n0 < p.qkv.n_qkv) {
      qkv_tile(p, acc, stg, rstd_s, row0, n0, w4, lane, bar_id);
      return;
    }
  }
  const int rw = w4 * 16 + (lane >> 3), cl = (lane & 7) * 8;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (n0 + q * EPI_COLS >= p.N) break;  // uniform over the warpgroup: every thread meets the same barriers
    named_bar_sync(bar_id, 128);           // the previous quarter is drained
    stage_quarter(acc, stg, q, w4, lane);
    named_bar_sync(bar_id, 128);
    drain_quarter<EPI>(p, stg, row0, rw, cl, n0 + q * EPI_COLS + cl);
  }
}

// ---------------------------------------------------------------------------------------------
// the kernel: persistent, CTA b takes tiles b, b + gridDim.x, ... (M fastest)
// ---------------------------------------------------------------------------------------------
template <bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                 const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg_all = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);  // [2 warpgroups][STG_FLOATS]
  float* rstd_all = stg_all + 2 * STG_FLOATS;                               // [2 warpgroups][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(rstd_all + 2 * 64);
  uint64_t* full_bar = bars;             // [STAGES]
  uint64_t* empty_bar = bars + STAGES;   // [STAGES]

  const uint32_t warp = warp_id_uniform();
  const uint32_t lane = lane_id();
  const int num_kb = (p.K + BK - 1) / BK;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  // `it` counts k-blocks over all of this CTA's tiles: ring stage it % STAGES, barrier phase (it / STAGES) & 1
  if (warp >= 8) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp > 8) return;
    // ================= TMA producer: runs ahead into the next tile's k-blocks as stages free up =================
    if (elect_one()) {
      int it = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m0 = (tile % p.num_m_tiles) * BM, n0 = (tile / p.num_m_tiles) * BN;
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int stage = it % STAGES;
          mbar_wait(smem_u32(&empty_bar[stage]), ((it / STAGES) & 1) ^ 1);
          const uint32_t a_dst = smem_u32(smem + stage * STAGE_BYTES);
          const uint32_t b_dst = a_dst + A_TILE_BYTES;
          const int k0 = kb * BK;
          const uint32_t bar = smem_u32(&full_bar[stage]);
          mbar_expect_tx(bar, STAGE_BYTES);
          if constexpr (!A_MN) {
            tma_load_2d(&tma_a, bar, a_dst, k0, m0);
          } else {
            tma_load_2d(&tma_a, bar, a_dst, m0, k0);
            tma_load_2d(&tma_a, bar, a_dst + SUB_BYTES, m0 + 64, k0);
          }
          if constexpr (!B_MN) {
            tma_load_2d(&tma_b, bar, b_dst, k0, n0, kEvictLast);
          } else {
#pragma unroll
            for (int j = 0; j < BN / 64; ++j) tma_load_2d(&tma_b, bar, b_dst + j * SUB_BYTES, n0 + 64 * j, k0, kEvictLast);
          }
        }
      }
    }
    return;
  }

  // ================= consumer warpgroups: rows [64 wg, 64 wg + 64) of each tile =================
  setmaxnreg_inc<CONSUMER_REGS>();
  const int wg = warp >> 2, w4 = warp & 3;
  float* stg = stg_all + wg * STG_FLOATS;
  float* rstd_s = rstd_all + wg * 64;
  const int bar_id = 2 + wg;  // named barrier of this warpgroup's epilogue buffer (0 is __syncthreads)
  int it = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int m0 = (tile % p.num_m_tiles) * BM, n0 = (tile / p.num_m_tiles) * BN;
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < num_kb; ++kb) {
      const int stage = (it + kb) % STAGES;
      mbar_wait(smem_u32(&full_bar[stage]), ((it + kb) / STAGES) & 1);
      const uint32_t a_base = smem_u32(smem + stage * STAGE_BYTES);
      const uint32_t b_base = a_base + A_TILE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / UK; ++k) {
        // K-major: rows of this warpgroup start 64 rows (8 KiB) in; step 16 elements (32 B) inside the swizzle row.
        // MN-major: sub-tile `wg` holds this warpgroup's 64 rows; step 16 k-rows = two 1024 B swizzle atoms.
        const uint64_t adesc = A_MN ? make_smem_desc(a_base + wg * SUB_BYTES + k * 2048, SUB_BYTES, 1024)
                                    : make_smem_desc(a_base + wg * (64 * 128) + k * 32, 16, 1024);
        const uint64_t bdesc = B_MN ? make_smem_desc(b_base + k * 2048, SUB_BYTES, 1024)
                                    : make_smem_desc(b_base + k * 32, 16, 1024);
        wgmma_m64n256k16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, 1u);
      }
      wgmma_commit();
      // keep one k-block of wgmma in flight; the previous one has retired, so its stage can be refilled
      wgmma_wait<1>();
      reg_fence<128>(acc);
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&empty_bar[(it + kb - 1) % STAGES]));
      }
    }
    wgmma_wait<0>();
    reg_fence<128>(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&empty_bar[(it + num_kb - 1) % STAGES]));
    it += num_kb;
    epilogue_wg<EPI>(p, acc, stg, rstd_s, m0 + wg * 64, n0, w4, lane, bar_id);
  }
}

// ---------------------------------------------------------------------------------------------
// host launcher
// ---------------------------------------------------------------------------------------------
template <bool A_MN, bool B_MN, int EPI>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  auto kern = gemm_bf16_kernel<A_MN, B_MN, EPI>;
  static bool configured = false;
  if (!configured) {
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    configured = true;
  }
  const int grid = p.num_tiles < num_sms() ? p.num_tiles : num_sms();
  kern<<<grid, GEMM_THREADS, SMEM_BYTES, stream>>>(ta, tb, p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

static int dispatch(const dpipe_gemm_args* a, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                    cudaStream_t s) {
  const int layout = (a->a_mn ? 2 : 0) | (a->b_mn ? 1 : 0);
  switch (a->epilogue) {
    case DPIPE_EPI_STORE:
      if (layout == 0) return launch<false, false, DPIPE_EPI_STORE>(ta, tb, p, s);
      if (layout == 1) return launch<false, true, DPIPE_EPI_STORE>(ta, tb, p, s);
      if (layout == 3) return launch<true, true, DPIPE_EPI_STORE>(ta, tb, p, s);
      break;
    case DPIPE_EPI_BIAS_GELU:
      if (layout == 0) return launch<false, false, DPIPE_EPI_BIAS_GELU>(ta, tb, p, s);
      break;
    case DPIPE_EPI_GATE_RES:
      if (layout == 0) return launch<false, false, DPIPE_EPI_GATE_RES>(ta, tb, p, s);
      break;
    case DPIPE_EPI_QKV_ROPE:
      if (layout == 0) return launch<false, false, DPIPE_EPI_QKV_ROPE>(ta, tb, p, s);
      break;
    case DPIPE_EPI_MUL_GELU_GRAD:
      if (layout == 1) return launch<false, true, DPIPE_EPI_MUL_GELU_GRAD>(ta, tb, p, s);
      break;
    default:
      break;
  }
  return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: epilogue %d is not built for operand layout a_mn=%d b_mn=%d",
              a->epilogue, a->a_mn, a->b_mn);
}

}  // namespace dpipe

extern "C" int dpipe_gemm_bf16(const dpipe_gemm_args* a, void* stream) {
  using namespace dpipe;
  if (!a) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: null args");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: empty problem %dx%dx%d", a->M, a->N, a->K);
  if (a->cta_group != 1 && a->cta_group != 2) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: cta_group must be 1 or 2");
  if (!a->A || !a->B || !a->out) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: null operand");
  if (a->N % 8 != 0 || a->ldo % 8 != 0) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: N and ldo must be multiples of 8");
  if (a->rows_per_batch <= 0) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: rows_per_batch must be > 0");
  if (a->epilogue != DPIPE_EPI_STORE && a->N % 32 != 0)
    return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: fused epilogues need N %% 32 == 0");
  if ((a->epilogue == DPIPE_EPI_GATE_RES && (!a->gate || !a->aux)) ||
      (a->epilogue == DPIPE_EPI_MUL_GELU_GRAD && !a->aux))
    return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: epilogue %d needs aux/gate inputs", a->epilogue);

  GemmParams p = {};
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.num_m_tiles = (a->M + BM - 1) / BM;
  p.num_tiles = p.num_m_tiles * ((a->N + BN - 1) / BN);
  p.out = reinterpret_cast<__nv_bfloat16*>(a->out); p.ldo = a->ldo;
  p.out2 = reinterpret_cast<__nv_bfloat16*>(a->out2); p.ldo2 = a->ldo2;
  p.bias = reinterpret_cast<const __nv_bfloat16*>(a->bias);
  p.aux = reinterpret_cast<const __nv_bfloat16*>(a->aux); p.ldaux = a->ldaux;
  p.gate = reinterpret_cast<const __nv_bfloat16*>(a->gate); p.gate_stride = a->gate_stride;
  p.rows_per_batch = a->rows_per_batch;
  p.accumulate = a->accumulate;
  if (a->epilogue == DPIPE_EPI_QKV_ROPE) {
    if (!a->qkv) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: QKV_ROPE epilogue needs args->qkv");
    p.qkv = *a->qkv;
    const dpipe_qkv_epilogue& e = p.qkv;
    if (e.heads <= 0 || (e.heads * 128) % BN != 0 || e.n_qkv != 3 * e.heads * 128 || e.n_qkv > a->N)
      return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: bad qkv epilogue geometry (heads=%d n_qkv=%d N=%d)", e.heads, e.n_qkv, a->N);
    if (!e.q || !e.k || !e.v || !e.q_norm_w || !e.k_norm_w || !e.rope_cos || !e.rope_sin)
      return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: qkv epilogue has null pointers");
    if (e.seq_offset + a->rows_per_batch > e.seq_total)
      return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: qkv stream does not fit the joint sequence");
    if (e.n_qkv < a->N && !a->out) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: fused linear1 needs an MLP output");
  }
  // the epilogue moves 8 bf16 (16 bytes) per access through every pointer it uses except the fp32 rstd rows
  {
    const bool has_out2 = a->epilogue == DPIPE_EPI_BIAS_GELU || a->epilogue == DPIPE_EPI_GATE_RES ||
                          a->epilogue == DPIPE_EPI_QKV_ROPE;
    const bool has_aux = a->epilogue == DPIPE_EPI_GATE_RES || a->epilogue == DPIPE_EPI_MUL_GELU_GRAD;
    const char* bad = nullptr;
    if (misaligned(a->out, 16)) bad = "out";
    else if (has_out2 && a->out2 && (misaligned(a->out2, 16) || a->ldo2 % 8 != 0)) bad = "out2/ldo2";
    else if (a->bias && misaligned(a->bias, 16)) bad = "bias";
    else if (has_aux && (misaligned(a->aux, 16) || a->ldaux % 8 != 0)) bad = "aux/ldaux";
    else if (a->epilogue == DPIPE_EPI_GATE_RES && (misaligned(a->gate, 16) || a->gate_stride % 8 != 0)) bad = "gate/gate_stride";
    if (!bad && a->epilogue == DPIPE_EPI_QKV_ROPE) {
      const dpipe_qkv_epilogue& e = p.qkv;
      if (misaligned(e.q, 16)) bad = "qkv.q";
      else if (misaligned(e.k, 16)) bad = "qkv.k";
      else if (misaligned(e.v, 16)) bad = "qkv.v";
      else if (misaligned(e.qhat, 16)) bad = "qkv.qhat";
      else if (misaligned(e.khat, 16)) bad = "qkv.khat";
      else if (misaligned(e.q_norm_w, 16)) bad = "qkv.q_norm_w";
      else if (misaligned(e.k_norm_w, 16)) bad = "qkv.k_norm_w";
      else if (misaligned(e.rope_cos, 16)) bad = "qkv.rope_cos";
      else if (misaligned(e.rope_sin, 16)) bad = "qkv.rope_sin";
      else if (misaligned(e.q_rstd, 4)) bad = "qkv.q_rstd";
      else if (misaligned(e.k_rstd, 4)) bad = "qkv.k_rstd";
    }
    if (bad) return fail(DPIPE_EINVAL, "dpipe_gemm_bf16: %s misaligned (pointers 16-byte aligned, fp32 rstd 4-byte, "
                                       "leading dimensions multiples of 8 elements)", bad);
  }

  CUtensorMap ta, tb;
  int rc;
  // K-major operand X[R,K]: dims {K, R}, box {64, rows}.  MN-major operand stored [K,R]: dims {R, K}, box {64, 64}.
  if (!a->a_mn) rc = make_tmap_2d_bf16(&ta, a->A, (uint64_t)a->K, (uint64_t)a->M, (uint64_t)a->lda, BK, BM);
  else          rc = make_tmap_2d_bf16(&ta, a->A, (uint64_t)a->M, (uint64_t)a->K, (uint64_t)a->lda, 64, BK);
  if (rc) return rc;
  if (!a->b_mn) rc = make_tmap_2d_bf16(&tb, a->B, (uint64_t)a->K, (uint64_t)a->N, (uint64_t)a->ldb, BK, BN);
  else          rc = make_tmap_2d_bf16(&tb, a->B, (uint64_t)a->N, (uint64_t)a->K, (uint64_t)a->ldb, 64, BK);
  if (rc) return rc;

  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return dispatch(a, ta, tb, p, s);
}
