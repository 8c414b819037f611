// Warp-specialised bf16 GEMM for sm_90a, one 128x256 output tile per CTA:
//   TMA (128B-swizzled tiles) -> shared memory ring -> wgmma (two consumer warpgroups, 64 rows x 256 columns
//   each, fp32 accumulators in registers) -> fp32 tile staged in shared memory (over the drained ring) ->
//   one thread per row and column half runs the fused epilogue.
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
constexpr int STG_LD = BN + 4;             // fp32 staging row stride: rows read 16 B at a time land in distinct banks
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
constexpr int GEMM_THREADS = 288;  // warps 0-7: two consumer warpgroups; warp 8: TMA producer
static_assert(BM * STG_LD * 4 <= STAGES * STAGE_BYTES, "the fp32 staging tile must fit in the operand ring");

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
// epilogue helpers: every thread owns one staged row and walks it 32 columns at a time
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_bf16x32(const __nv_bfloat16* p, bool ok, float* f) {
  if (ok) {
    const uint4* v = reinterpret_cast<const uint4*>(p);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 q = v[j];
      f[j * 8 + 0] = bf16_lo(q.x); f[j * 8 + 1] = bf16_hi(q.x);
      f[j * 8 + 2] = bf16_lo(q.y); f[j * 8 + 3] = bf16_hi(q.y);
      f[j * 8 + 4] = bf16_lo(q.z); f[j * 8 + 5] = bf16_hi(q.z);
      f[j * 8 + 6] = bf16_lo(q.w); f[j * 8 + 7] = bf16_hi(q.w);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = 0.f;
  }
}
__device__ __forceinline__ void store_bf16x32(__nv_bfloat16* p, const float* f) {
  uint4* v = reinterpret_cast<uint4*>(p);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    uint4 q;
    q.x = pack_bf16(f[j * 8 + 0], f[j * 8 + 1]);
    q.y = pack_bf16(f[j * 8 + 2], f[j * 8 + 3]);
    q.z = pack_bf16(f[j * 8 + 4], f[j * 8 + 5]);
    q.w = pack_bf16(f[j * 8 + 6], f[j * 8 + 7]);
    v[j] = q;
  }
}
__device__ __forceinline__ void load_f32x32(const float* p, float* f) {
  const float4* v = reinterpret_cast<const float4*>(p);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float4 q = v[j];
    f[j * 4 + 0] = q.x; f[j * 4 + 1] = q.y; f[j * 4 + 2] = q.z; f[j * 4 + 3] = q.w;
  }
}

// bias + GELU(tanh) for one 32-column chunk; `col` is the global column of f[0]
__device__ __forceinline__ void epi_bias_gelu_chunk(const GemmParams& p, bool ok, int row, int col,
                                                    int out_col, float* acc) {
  float b[32];
  load_bf16x32(p.bias ? p.bias + col : nullptr, p.bias != nullptr, b);
  float u[32], h[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    u[j] = bf16_round(acc[j] + b[j]);
    h[j] = gelu_tanh(u[j]);
  }
  if (ok) {
    if (p.out2) store_bf16x32(p.out2 + (int64_t)row * p.ldo2 + out_col, u);
    store_bf16x32(p.out + (int64_t)row * p.ldo + out_col, h);
  }
}

__device__ __forceinline__ void ld_row32(const float* s, uint32_t* r) {
  const float4* v = reinterpret_cast<const float4*>(s);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float4 q = v[j];
    r[j * 4 + 0] = __float_as_uint(q.x); r[j * 4 + 1] = __float_as_uint(q.y);
    r[j * 4 + 2] = __float_as_uint(q.z); r[j * 4 + 3] = __float_as_uint(q.w);
  }
}

template <int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, int row, int n0, const float* srow, int half) {
  // `half` selects which 128 of the tile's 256 accumulator columns this thread drains; srow is its staged fp32 row
  const bool row_ok = row < p.M;
  const int batch = row_ok ? row / p.rows_per_batch : 0;

  if constexpr (EPI == DPIPE_EPI_QKV_ROPE) {
    if (n0 < p.qkv.n_qkv) {
      // ---- q / k / v columns: this 256-wide tile holds two heads of one of q, k, v ----
      const dpipe_qkv_epilogue& e = p.qkv;
      const int hd = e.heads * 128;
      const int which = n0 / hd;  // 0 q, 1 k, 2 v (tile never straddles: hd % 256 == 0)
      const int tok = row_ok ? row - batch * p.rows_per_batch : 0;
      const int pos = e.seq_offset + tok;
#pragma unroll 1
      for (int hh = half; hh <= half; ++hh) {
        const int col_h = n0 + hh * 128;  // global column of this head's first element
        if (col_h >= p.N) break;
        const int head = (col_h - which * hd) >> 7;
        const int64_t o = (((int64_t)batch * e.heads + head) * e.seq_total + pos) * 128;
        if (which == 2) {
#pragma unroll 1
          for (int c = 0; c < 4; ++c) {
            uint32_t r[32];
            ld_row32(srow + hh * 128 + c * 32, r);
            float b[32], f[32];
            load_bf16x32(p.bias ? p.bias + col_h + c * 32 : nullptr, p.bias != nullptr, b);
#pragma unroll
            for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(r[j]) + b[j];
            if (row_ok) store_bf16x32(reinterpret_cast<__nv_bfloat16*>(e.v) + o + c * 32, f);
          }
        } else {
          // pass 1: sum of squares of the bf16-rounded projection (reference: RMSNorm on the bf16 Linear output)
          float ss = 0.f;
#pragma unroll 1
          for (int c = 0; c < 4; ++c) {
            uint32_t r[32];
            ld_row32(srow + hh * 128 + c * 32, r);
            float b[32];
            load_bf16x32(p.bias ? p.bias + col_h + c * 32 : nullptr, p.bias != nullptr, b);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              float v = bf16_round(__uint_as_float(r[j]) + b[j]);
              ss += v * v;
            }
          }
          const float rstd = rsqrtf(ss * (1.0f / 128.0f) + e.eps);
          const __nv_bfloat16* w = reinterpret_cast<const __nv_bfloat16*>(which == 0 ? e.q_norm_w : e.k_norm_w);
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(which == 0 ? e.q : e.k);
          __nv_bfloat16* dst_hat = reinterpret_cast<__nv_bfloat16*>(which == 0 ? e.qhat : e.khat);
          float* dst_rstd = which == 0 ? e.q_rstd : e.k_rstd;
          if (row_ok && dst_rstd) dst_rstd[((int64_t)batch * e.heads + head) * e.seq_total + pos] = rstd;
          // pass 2: normalise, scale, rotate, store
#pragma unroll 1
          for (int c = 0; c < 4; ++c) {
            uint32_t r[32];
            ld_row32(srow + hh * 128 + c * 32, r);
            float b[32], wv[32], xh[32], y[32];
            load_bf16x32(p.bias ? p.bias + col_h + c * 32 : nullptr, p.bias != nullptr, b);
            load_bf16x32(w + c * 32, true, wv);
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              float v = bf16_round(__uint_as_float(r[j]) + b[j]);
              xh[j] = bf16_round(v * rstd);
              y[j] = bf16_round(xh[j] * wv[j]);
            }
            if (row_ok) {
              if (dst_hat) store_bf16x32(dst_hat + o + c * 32, xh);
              float cs[32], sn[32], ro[32];
              load_f32x32(e.rope_cos + (int64_t)pos * 128 + c * 32, cs);
              load_f32x32(e.rope_sin + (int64_t)pos * 128 + c * 32, sn);
#pragma unroll
              for (int j = 0; j < 32; j += 2) {
                ro[j] = y[j] * cs[j] - y[j + 1] * sn[j];
                ro[j + 1] = y[j + 1] * cs[j + 1] + y[j] * sn[j + 1];
              }
              store_bf16x32(dst + o + c * 32, ro);
            }
          }
        }
      }
      return;
    }
  }

#pragma unroll 1
  for (int c = half * 4; c < half * 4 + 4; ++c) {
    const int col = n0 + c * 32;
    if (col >= p.N) break;  // warp-uniform
    uint32_t r[32];
    ld_row32(srow + c * 32, r);
    float acc[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[j] = __uint_as_float(r[j]);
    const bool ok = row_ok && (col + 32 <= p.N);
    const bool tail = row_ok && !ok;  // partial chunk at the right edge (N % 32 != 0)

    if constexpr (EPI == DPIPE_EPI_STORE) {
      float b[32];
      load_bf16x32(p.bias ? p.bias + col : nullptr, p.bias != nullptr && col + 32 <= p.N, b);
      if (p.bias && col + 32 > p.N) {
        for (int j = 0; j < 32 && col + j < p.N; ++j) b[j] = __bfloat162float(p.bias[col + j]);
      }
      __nv_bfloat16* dst = p.out + (int64_t)row * p.ldo + col;
      if (ok) {
        if (p.accumulate) {
          float old[32];
          load_bf16x32(dst, true, old);
#pragma unroll
          for (int j = 0; j < 32; ++j) acc[j] += old[j];
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] += b[j];
        store_bf16x32(dst, acc);
      } else if (tail) {
        for (int j = 0; j < 32 && col + j < p.N; ++j) {
          float v = acc[j] + b[j];
          if (p.accumulate) v += __bfloat162float(dst[j]);
          dst[j] = __float2bfloat16_rn(v);
        }
      }
    } else if constexpr (EPI == DPIPE_EPI_BIAS_GELU) {
      epi_bias_gelu_chunk(p, ok, row, col, col, acc);
    } else if constexpr (EPI == DPIPE_EPI_QKV_ROPE) {
      // columns beyond n_qkv: the MLP half of the fused linear1 of a single-stream block
      epi_bias_gelu_chunk(p, ok, row, col, col - p.qkv.n_qkv, acc);
    } else if constexpr (EPI == DPIPE_EPI_GATE_RES) {
      float b[32], g[32], res[32], y[32], o[32];
      load_bf16x32(p.bias ? p.bias + col : nullptr, p.bias != nullptr, b);
      load_bf16x32(p.gate + (int64_t)batch * p.gate_stride + col, ok, g);
      load_bf16x32(p.aux + (int64_t)row * p.ldaux + col, ok, res);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        y[j] = bf16_round(acc[j] + b[j]);
        o[j] = res[j] + bf16_round(g[j] * y[j]);
      }
      if (ok) {
        if (p.out2) store_bf16x32(p.out2 + (int64_t)row * p.ldo2 + col, y);
        store_bf16x32(p.out + (int64_t)row * p.ldo + col, o);
      }
    } else if constexpr (EPI == DPIPE_EPI_MUL_GELU_GRAD) {
      float u[32], o[32];
      load_bf16x32(p.aux + (int64_t)row * p.ldaux + col, ok, u);
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] = acc[j] * gelu_tanh_grad(u[j]);
      if (ok) store_bf16x32(p.out + (int64_t)row * p.ldo + col, o);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------------------------
template <bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
                 const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;             // [STAGES]
  uint64_t* empty_bar = bars + STAGES;   // [STAGES]

  const uint32_t warp = warp_id_uniform();
  const uint32_t lane = lane_id();
  const int mt = blockIdx.x % p.num_m_tiles, nt = blockIdx.x / p.num_m_tiles;
  const int m0 = mt * BM, n0 = nt * BN;
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

  if (warp == 8) {
    // ================= TMA producer =================
    if (elect_one()) {
      for (int kb = 0; kb < num_kb; ++kb) {
        const int stage = kb % STAGES;
        mbar_wait(smem_u32(&empty_bar[stage]), ((kb / STAGES) & 1) ^ 1);
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
    return;
  }

  // ================= consumer warpgroups: rows [64 wg, 64 wg + 64) of the tile =================
  const int wg = warp >> 2;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int stage = kb % STAGES;
    mbar_wait(smem_u32(&full_bar[stage]), (kb / STAGES) & 1);
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
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[(kb - 1) % STAGES]));
    }
  }
  wgmma_wait<0>();
  reg_fence<128>(acc);

  // every TMA write has landed (all full barriers were waited on) and both warpgroups have retired their wgmma:
  // the ring is free and holds the fp32 tile from here on
  named_bar_sync(1, 256);
  float* stg = reinterpret_cast<float*>(smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      *reinterpret_cast<float2*>(stg + r0 * STG_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(stg + (r0 + 8) * STG_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_bar_sync(1, 256);
  const int r = threadIdx.x & (BM - 1);
  const int half = threadIdx.x >> 7;
  epilogue_tile<EPI>(p, m0 + r, n0, stg + r * STG_LD, half);
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
  kern<<<p.num_tiles, GEMM_THREADS, SMEM_BYTES, stream>>>(ta, tb, p);
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
