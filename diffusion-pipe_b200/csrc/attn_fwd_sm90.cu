// FlashAttention-style fused attention forward for sm_90a (head_dim 128, non-causal, bf16 in / fp32 softmax).
//
// One CTA owns a 128-row query tile of one (batch, head) and streams K/V tiles of 128 keys:
//   warp 8      : TMA producer (Q once, K ring, V ring)
//   warps 0-7   : two consumer warpgroups, 64 query rows each.  S = Q K^T by wgmma (both operands K-major in
//                 shared memory) into registers; online softmax in registers; O += P V by wgmma with P taken
//                 straight from the S registers as the bf16 A fragment and V MN-major in shared memory.
// The two warpgroups run independently, so one exponentiates while the other's wgmma occupies the tensor core.
//
// Replaces torch SDPA / flash_attn as dispatched by the reference's Flux blocks
// (reference: diffusers attention inside models/flux.py:502,525; Wan: models/wan/attention.py:108-122).
#include <stdlib.h>

#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int ATT_THREADS = 288;
constexpr int TQ = 128;   // query rows per CTA (64 per consumer warpgroup)
constexpr int TK = 128;   // keys per tile
constexpr int HD = 128;   // head dim
constexpr int HALF_TILE_BYTES = 128 * 64 * 2;   // one [128 rows][64 cols] swizzled sub-tile = 16 KiB
constexpr int TILE_BYTES = 2 * HALF_TILE_BYTES; // 32 KiB
constexpr int KV_STAGES = 2;
constexpr int ATT_SMEM_BYTES = TILE_BYTES + 2 * KV_STAGES * TILE_BYTES + 1024 + 256;

struct AttnFwdParams {
  __nv_bfloat16* o;
  int64_t ldo;
  float* lse;
  int batch, heads, seq_q, seq_k;
  float scale_log2;  // softmax scale * log2(e)
};

// POLY: of every 8 column pairs of a score row, this many take their exponential from the FMA-pipe polynomial instead of
// MUFU (0 = all MUFU).
template <int POLY>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                const __grid_constant__ CUtensorMap tma_v, const AttnFwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* q_smem = smem;                                   // 1 tile
  uint8_t* k_smem = smem + TILE_BYTES;                      // KV_STAGES tiles
  uint8_t* v_smem = k_smem + KV_STAGES * TILE_BYTES;        // KV_STAGES tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(v_smem + KV_STAGES * TILE_BYTES);
  uint64_t* q_full = bars;            // [1]
  uint64_t* k_full = bars + 1;        // [KV_STAGES]
  uint64_t* k_empty = k_full + KV_STAGES;
  uint64_t* v_full = k_empty + KV_STAGES;
  uint64_t* v_empty = v_full + KV_STAGES;

  const uint32_t warp = warp_id_uniform();
  const uint32_t lane = lane_id();
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int bh = b * p.heads + head;
  const int q0 = blockIdx.x * TQ;
  const int nkv = (p.seq_k + TK - 1) / TK;

  if (warp == 8 && elect_one()) {
    tma_prefetch_desc(&tma_q);
    tma_prefetch_desc(&tma_k);
    tma_prefetch_desc(&tma_v);
    mbar_init(smem_u32(q_full), 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(smem_u32(&k_full[s]), 1);
      mbar_init(smem_u32(&k_empty[s]), 8);  // one arrival per consumer warp
      mbar_init(smem_u32(&v_full[s]), 1);
      mbar_init(smem_u32(&v_empty[s]), 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================= TMA producer =================
    if (elect_one()) {
      const uint32_t qb = smem_u32(q_full);
      mbar_expect_tx(qb, TILE_BYTES);
      for (int h = 0; h < 2; ++h)
        tma_load_3d(&tma_q, qb, smem_u32(q_smem + h * HALF_TILE_BYTES), h * 64, q0, bh, kEvictFirst);
      for (int j = 0; j < nkv; ++j) {
        const int kv0 = j * TK, stage = j % KV_STAGES;
        const uint32_t ph = ((j / KV_STAGES) & 1) ^ 1;
        mbar_wait(smem_u32(&k_empty[stage]), ph);
        const uint32_t kb = smem_u32(&k_full[stage]);
        mbar_expect_tx(kb, TILE_BYTES);
        for (int h = 0; h < 2; ++h)
          tma_load_3d(&tma_k, kb, smem_u32(k_smem + stage * TILE_BYTES + h * HALF_TILE_BYTES), h * 64, kv0, bh,
                      kEvictLast);
        mbar_wait(smem_u32(&v_empty[stage]), ph);
        const uint32_t vb = smem_u32(&v_full[stage]);
        mbar_expect_tx(vb, TILE_BYTES);
        for (int h = 0; h < 2; ++h)
          tma_load_3d(&tma_v, vb, smem_u32(v_smem + stage * TILE_BYTES + h * HALF_TILE_BYTES), h * 64, kv0, bh,
                      kEvictLast);
      }
    }
    return;
  }

  // ================= consumer warpgroup `wg`: query rows [q0 + 64 wg, q0 + 64 wg + 64) =================
  const int wg = warp >> 2;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: rloc and rloc + 8
  const int cq = 2 * (lane & 3);                               // first of this thread's column pair in each 8-block
  const float c = p.scale_log2;
  float m[2] = {-INFINITY, -INFINITY};   // running max, scaled-log2 units
  float l[2] = {0.f, 0.f};               // this thread's share of the row sums
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  const uint32_t qa = smem_u32(q_smem) + wg * (64 * 128);
  mbar_wait(smem_u32(q_full), 0);

  for (int j = 0; j < nkv; ++j) {
    const int stage = j % KV_STAGES;
    const uint32_t ph = (j / KV_STAGES) & 1;
    float s[64];
    mbar_wait(smem_u32(&k_full[stage]), ph);
    {
      const uint32_t kb = smem_u32(k_smem + stage * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k) {
        const uint32_t off = (k >> 2) * HALF_TILE_BYTES + (k & 3) * 32;
        wgmma_m64n128k16_ss<0, 0>(s, make_smem_desc(qa + off, 16, 1024), make_smem_desc(kb + off, 16, 1024),
                                  k != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<64>(s);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&k_empty[stage]));

    const int valid = p.seq_k - j * TK;   // keys of this tile that exist (>= TK except on the last tile)
    if (valid < TK) {
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
    }
    // ---- row maxima (a row is spread over the 4 threads of a quad) and the online rescale ----
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jb = 0; jb < 16; ++jb) mx = fmaxf(mx, fmaxf(s[4 * jb + 2 * h], s[4 * jb + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx * c);
      alpha[h] = (j == 0) ? 0.f : fast_exp2(m[h] - m_new);
      m[h] = m_new;
      l[h] *= alpha[h];
    }
    if (j > 0) {
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] *= alpha[(i >> 1) & 1];
    }
    // ---- P = exp2(S*c - m) (fp32 row sums), packed to the bf16 A fragments of the PV wgmma ----
    uint32_t pa[32];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int h = (i >> 1) & 1;
      const f32x2 x = f2_fma(f2_pack(s[i], s[i + 1]), f2_pack(c, c), f2_pack(-m[h], -m[h]));
      const f32x2 e = (((i >> 1) & 7) < POLY) ? f2_exp2_poly(x) : f2_exp2_mufu(x);
      float p0, p1;
      f2_unpack(e, p0, p1);
      l[h] += p0 + p1;
      pa[i >> 1] = pack_bf16(p0, p1);
    }
    mbar_wait(smem_u32(&v_full[stage]), ph);
    {
      const uint32_t vb = smem_u32(v_smem + stage * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TK / 16; ++k) {
        // V sub-tile h holds d in [64h, 64h+64): LBO = distance between the two halves, SBO = 8 keys, 16 keys per step
        wgmma_m64n128k16_rs<1>(o, pa + 4 * k, make_smem_desc(vb + k * 2048, HALF_TILE_BYTES, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<64>(o);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&v_empty[stage]));
  }

  // ---- epilogue: O / l -> bf16 -> global ; LSE ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qrow = q0 + rloc + 8 * h;
    if (qrow >= p.seq_q) continue;
    const float inv_l = 1.0f / l[h];
    __nv_bfloat16* orow = p.o + ((int64_t)b * p.seq_q + qrow) * p.ldo + head * HD;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
      *reinterpret_cast<uint32_t*>(orow + 8 * jb + cq) = pack_bf16(o[4 * jb + 2 * h] * inv_l, o[4 * jb + 2 * h + 1] * inv_l);
    if (p.lse && (lane & 3) == 0) p.lse[(int64_t)bh * p.seq_q + qrow] = m[h] + log2f(l[h]);
  }
}

}  // namespace dpipe

extern "C" int dpipe_attn_fwd(const dpipe_attn_args* a, void* stream) {
  using namespace dpipe;
  if (!a || !a->q || !a->k || !a->v || !a->o) return fail(DPIPE_EINVAL, "dpipe_attn_fwd: null argument");
  if (a->batch <= 0 || a->heads <= 0 || a->seq_q <= 0 || a->seq_k <= 0)
    return fail(DPIPE_EINVAL, "dpipe_attn_fwd: empty problem");
  if (a->ldo % 8 != 0 || a->ldo < (int64_t)a->heads * HD) return fail(DPIPE_EINVAL, "dpipe_attn_fwd: bad ldo");
  CUtensorMap tq, tk, tv;
  const uint64_t bh = (uint64_t)a->batch * a->heads;
  int rc;
  if ((rc = make_tmap_3d_bf16(&tq, a->q, HD, a->seq_q, bh, HD, (uint64_t)a->seq_q * HD, 64, TQ, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tk, a->k, HD, a->seq_k, bh, HD, (uint64_t)a->seq_k * HD, 64, TK, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tv, a->v, HD, a->seq_k, bh, HD, (uint64_t)a->seq_k * HD, 64, TK, 1))) return rc;
  static bool configured = false;
  // DPIPE_ATTN_FWD_POLY = 0 | 2 | 4: column pairs out of 8 exponentiated on the FMA pipe.  H100's dense bf16 wgmma
  // needs 0.25 clk/SM per score at head_dim 128 against 0.0625 for MUFU's 16 exponentials/clk, so MUFU alone is
  // the default here.
  static int poly = 0;
  if (!configured) {
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM_BYTES));
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM_BYTES));
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATT_SMEM_BYTES));
    const char* e = getenv("DPIPE_ATTN_FWD_POLY");
    if (e && (e[0] == '0' || e[0] == '2' || e[0] == '4') && e[1] == 0) poly = e[0] - '0';
    configured = true;
  }
  AttnFwdParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(a->o);
  p.ldo = a->ldo;
  p.lse = a->lse;
  p.batch = a->batch; p.heads = a->heads; p.seq_q = a->seq_q; p.seq_k = a->seq_k;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  dim3 grid((a->seq_q + TQ - 1) / TQ, a->heads, a->batch);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (poly == 0) attn_fwd_kernel<0><<<grid, ATT_THREADS, ATT_SMEM_BYTES, st>>>(tq, tk, tv, p);
  else if (poly == 4) attn_fwd_kernel<4><<<grid, ATT_THREADS, ATT_SMEM_BYTES, st>>>(tq, tk, tv, p);
  else attn_fwd_kernel<2><<<grid, ATT_THREADS, ATT_SMEM_BYTES, st>>>(tq, tk, tv, p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
