// Fused attention backward for sm_90a (head_dim 128, non-causal), three kernels:
//
//   attn_bwd_delta    D[b,h,q] = sum_d O*dO                       (HBM-bound, one warp per (token, head))
//   attn_bwd_dkv      one CTA per 128-key tile (64 keys per consumer warpgroup), loops over 64-query chunks:
//                        St  = K Q^T          (wgmma, both operands K-major in shared memory)
//                        dPt = V dO^T                                  Pt  = exp2(St*c - LSE[q])
//                                                                      dSt = Pt * (dPt - D[q])
//                        dV += Pt  dO         (wgmma, Pt / dSt straight from registers as the A fragment,
//                        dK += dSt Q           dO / Q chunks re-used MN-major)
//   attn_bwd_dq       one CTA per 128-query tile (64 queries per consumer warpgroup), loops over 64-key chunks:
//                        S = Q K^T, dP = dO V^T ; dS = P*(dP - D) ; dQ += dS K (K chunk re-used MN-major)
//
// Splitting dQ from dK/dV recomputes S and dP once more (7 instead of 5 tile GEMMs) but needs no atomics and no fp32
// dQ staging buffer.  The transposed formulation in dkv puts P^T / dS^T in the accumulator layout that wgmma takes
// as its register A operand, so neither goes through shared memory.
//
// LSE is the log2-domain logsumexp written by attn_fwd.  Outputs dQ/dK/dV are head-major [B,H,L,128] bf16.
// Replaces flash-attn / SDPA backward reached through autograd from models/flux.py:502,525.
#include <stdlib.h>

#include "host_util.h"
#include "sm90_common.cuh"

namespace dpipe {

constexpr int AB_THREADS = 288;          // dq: warps 0-7 two consumer warpgroups, warp 8 TMA producer
constexpr int DKV_THREADS = 256;         // dkv: the two consumer warpgroups only
constexpr int BT = 128;                  // rows of the tile a CTA owns (keys in dkv, queries in dq)
constexpr int BC = 64;                   // rows of the streamed chunks (queries in dkv, keys in dq)
constexpr int BHALF = BT * 64 * 2;       // [128 rows][64 d] swizzled half tile = 16 KiB
constexpr int BTILE = 2 * BHALF;         // 32 KiB
constexpr int CHALF = BC * 64 * 2;       // [64 rows][64 d] = 8 KiB
constexpr int CTILE = 2 * CHALF;         // 16 KiB
constexpr int AB_STAGES = 2;
constexpr int AB_SMEM_BYTES = 2 * BTILE + 2 * AB_STAGES * CTILE + 1024 + 256;

struct AttnBwdParams {
  const float* lse;    // [B,H,Lq] log2 domain
  const float* delta;  // [B,H,Lq]
  __nv_bfloat16* dq;   // [B,H,Lq,128]
  __nv_bfloat16* dk;   // [B,H,Lk,128]
  __nv_bfloat16* dv;   // [B,H,Lk,128]
  int batch, heads, seq_q, seq_k;
  float scale_log2, scale;
};

// K-major operand tile of `half_bytes` per 64-wide d half: byte offset of k-step `k` (16 d per step)
__device__ __forceinline__ uint32_t kmajor_off(int k, int half_bytes) { return (k >> 2) * half_bytes + (k & 3) * 32; }

// ---------------------------------------------------------------------------------------------
__global__ void attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ o, int64_t ldo,
                                      const __nv_bfloat16* __restrict__ d_o, int64_t lddo, float* __restrict__ delta,
                                      int batch, int heads, int seq) {
  const int64_t gw = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int64_t total = (int64_t)batch * seq * heads;
  if (gw >= total) return;
  const int h = gw % heads;
  const int64_t tok = gw / heads;  // b*seq + q
  const uint2 a = *reinterpret_cast<const uint2*>(o + tok * ldo + h * 128 + lane * 4);
  const uint2 b = *reinterpret_cast<const uint2*>(d_o + tok * lddo + h * 128 + lane * 4);
  float s = bf16_lo(a.x) * bf16_lo(b.x) + bf16_hi(a.x) * bf16_hi(b.x) + bf16_lo(a.y) * bf16_lo(b.y) +
            bf16_hi(a.y) * bf16_hi(b.y);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) {
    const int bb = tok / seq, q = tok % seq;
    delta[((int64_t)bb * heads + h) * seq + q] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// dK / dV
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(DKV_THREADS, 1)
attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tma_q64, const __grid_constant__ CUtensorMap tma_k,
                    const __grid_constant__ CUtensorMap tma_v, const __grid_constant__ CUtensorMap tma_do64,
                    const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_smem = smem;                       // the CTA's own 128-row tiles: 2 x BTILE
  uint8_t* b_smem = smem + 2 * BTILE;           // streamed chunks: [AB_STAGES][2] x CTILE
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * BTILE + 2 * AB_STAGES * CTILE);
  uint64_t* own_full = bars;                    // [1]
  uint64_t* c_full = bars + 1;                  // [AB_STAGES]
  uint64_t* c_empty = c_full + AB_STAGES;       // [AB_STAGES]

  const uint32_t warp = warp_id_uniform();
  const uint32_t lane = lane_id();
  const int r0 = blockIdx.x * BT;
  const int head = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.heads + head;

  if (threadIdx.x == 0) {
    mbar_init(smem_u32(own_full), 1);
    for (int s = 0; s < AB_STAGES; ++s) {
      mbar_init(smem_u32(&c_full[s]), 1);
      mbar_init(smem_u32(&c_empty[s]), 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int wg = warp >> 2;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's tile rows: rloc and rloc + 8
  const int cq = 2 * (lane & 3);                               // first of its column pair in each 8-column block
  const int nq = (p.seq_q + BC - 1) / BC;

  // no producer warp here: a ninth warp would cap every thread at 168 registers (three warps on one SM sub-partition)
  // and the four accumulators below need more, so thread 0 issues the loads between its own wgmma
  auto load_chunk = [&](int j) {
    const int stage = j % AB_STAGES;
    const uint32_t cb = smem_u32(&c_full[stage]);
    mbar_expect_tx(cb, 2 * CTILE);
    uint8_t* qd = b_smem + stage * 2 * CTILE;
    for (int h = 0; h < 2; ++h) {
      tma_load_3d(&tma_q64, cb, smem_u32(qd + h * CHALF), h * 64, j * BC, bh, kEvictLast);
      tma_load_4d(&tma_do64, cb, smem_u32(qd + CTILE + h * CHALF), h * 64, j * BC, head, b, kEvictLast);
    }
  };
  if (threadIdx.x == 0) {
    const uint32_t ob = smem_u32(own_full);
    mbar_expect_tx(ob, 2 * BTILE);
    for (int h = 0; h < 2; ++h) {
      tma_load_3d(&tma_k, ob, smem_u32(a_smem + h * BHALF), h * 64, r0, bh, kEvictFirst);
      tma_load_3d(&tma_v, ob, smem_u32(a_smem + BTILE + h * BHALF), h * 64, r0, bh, kEvictFirst);
    }
    for (int j = 0; j < AB_STAGES && j < nq; ++j) load_chunk(j);
  }

  // ================= consumer warpgroup `wg`: keys [r0 + 64 wg, r0 + 64 wg + 64) =================
  const float c = p.scale_log2;
  const float* lse_bh = p.lse + (int64_t)bh * p.seq_q;
  const float* dl_bh = p.delta + (int64_t)bh * p.seq_q;
  const uint32_t ka = smem_u32(a_smem) + wg * (64 * 128);
  const uint32_t va = ka + BTILE;
  float dv[64], dk[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) { dv[i] = 0.f; dk[i] = 0.f; }
  mbar_wait(smem_u32(own_full), 0);

  for (int j = 0; j < nq; ++j) {
    const int stage = j % AB_STAGES;
    mbar_wait(smem_u32(&c_full[stage]), (j / AB_STAGES) & 1);
    const uint32_t qb = smem_u32(b_smem + stage * 2 * CTILE);
    const uint32_t dob = qb + CTILE;
    float st[32], dpt[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)   // St[kv, 64 q] = K Q^T
      wgmma_m64n64k16_ss<0, 0>(st, make_smem_desc(ka + kmajor_off(k, BHALF), 16, 1024),
                               make_smem_desc(qb + kmajor_off(k, CHALF), 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < 8; ++k)   // dPt[kv, 64 q] = V dO^T
      wgmma_m64n64k16_ss<0, 0>(dpt, make_smem_desc(va + kmajor_off(k, BHALF), 16, 1024),
                               make_smem_desc(dob + kmajor_off(k, CHALF), 16, 1024), k != 0);
    wgmma_commit();
    // this thread's 16 query columns: their LSE and D (queries past seq_q get P = 0)
    float nl[16], dl[16];
#pragma unroll
    for (int x = 0; x < 16; ++x) {
      const int q = j * BC + 8 * (x >> 1) + cq + (x & 1);
      nl[x] = q < p.seq_q ? -__ldg(lse_bh + q) : -INFINITY;
      dl[x] = q < p.seq_q ? __ldg(dl_bh + q) : 0.f;
    }
    wgmma_wait<0>();
    reg_fence<32>(st);
    reg_fence<32>(dpt);
    uint32_t pa[16], da[16];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int x = 2 * (i >> 2);   // column pair index of st[i], st[i + 1]
      const f32x2 e = f2_exp2_mufu(f2_fma(f2_pack(st[i], st[i + 1]), f2_pack(c, c), f2_pack(nl[x], nl[x + 1])));
      const f32x2 d = f2_mul(e, f2_sub(f2_pack(dpt[i], dpt[i + 1]), f2_pack(dl[x], dl[x + 1])));
      float p0, p1, d0, d1;
      f2_unpack(e, p0, p1);
      f2_unpack(d, d0, d1);
      pa[i >> 1] = pack_bf16(p0, p1);
      da[i >> 1] = pack_bf16(d0, d1);
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BC / 16; ++k) {   // dV[kv, d] += Pt[kv, 64 q] dO[64 q, d]; dK[kv, d] += dSt Q
      wgmma_m64n128k16_rs<1>(dv, pa + 4 * k, make_smem_desc(dob + k * 2048, CHALF, 1024), 1u);
      wgmma_m64n128k16_rs<1>(dk, da + 4 * k, make_smem_desc(qb + k * 2048, CHALF, 1024), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(dv);
    reg_fence<64>(dk);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&c_empty[stage]));
    if (threadIdx.x == 0 && j + AB_STAGES < nq) {
      mbar_wait(smem_u32(&c_empty[stage]), (j / AB_STAGES) & 1);
      load_chunk(j + AB_STAGES);
    }
    __syncwarp();   // warp 0 reconverges before the next (warp-aligned) wgmma
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int kv = r0 + rloc + 8 * h;
    if (kv >= p.seq_k) continue;
    const int64_t o = ((int64_t)bh * p.seq_k + kv) * 128;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb) {
      *reinterpret_cast<uint32_t*>(p.dv + o + 8 * jb + cq) = pack_bf16(dv[4 * jb + 2 * h], dv[4 * jb + 2 * h + 1]);
      *reinterpret_cast<uint32_t*>(p.dk + o + 8 * jb + cq) =
          pack_bf16(dk[4 * jb + 2 * h] * p.scale, dk[4 * jb + 2 * h + 1] * p.scale);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// dQ
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k64,
                   const __grid_constant__ CUtensorMap tma_v64, const __grid_constant__ CUtensorMap tma_do,
                   const AttnBwdParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_smem = smem;                       // the CTA's own 128-row tiles: 2 x BTILE
  uint8_t* b_smem = smem + 2 * BTILE;           // streamed chunks: [AB_STAGES][2] x CTILE
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * BTILE + 2 * AB_STAGES * CTILE);
  uint64_t* own_full = bars;                    // [1]
  uint64_t* c_full = bars + 1;                  // [AB_STAGES]
  uint64_t* c_empty = c_full + AB_STAGES;       // [AB_STAGES]

  const uint32_t warp = warp_id_uniform();
  const uint32_t lane = lane_id();
  const int r0 = blockIdx.x * BT;
  const int head = blockIdx.y, b = blockIdx.z;
  const int bh = b * p.heads + head;

  if (warp == 8 && elect_one()) {
    mbar_init(smem_u32(own_full), 1);
    for (int s = 0; s < AB_STAGES; ++s) {
      mbar_init(smem_u32(&c_full[s]), 1);
      mbar_init(smem_u32(&c_empty[s]), 8);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  const int wg = warp >> 2;
  const int rloc = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's tile rows: rloc and rloc + 8
  const int cq = 2 * (lane & 3);                               // first of its column pair in each 8-column block
  const int nk = (p.seq_k + BC - 1) / BC;

  if (warp == 8) {
    // ================= TMA producer: Q and dO once, then (K, V) chunks of 64 keys =================
    if (elect_one()) {
      const uint32_t ob = smem_u32(own_full);
      mbar_expect_tx(ob, 2 * BTILE);
      for (int h = 0; h < 2; ++h) {
        tma_load_3d(&tma_q, ob, smem_u32(a_smem + h * BHALF), h * 64, r0, bh, kEvictFirst);
        tma_load_4d(&tma_do, ob, smem_u32(a_smem + BTILE + h * BHALF), h * 64, r0, head, b, kEvictFirst);
      }
      for (int j = 0; j < nk; ++j) {
        const int stage = j % AB_STAGES;
        mbar_wait(smem_u32(&c_empty[stage]), ((j / AB_STAGES) & 1) ^ 1);
        const uint32_t cb = smem_u32(&c_full[stage]);
        mbar_expect_tx(cb, 2 * CTILE);
        uint8_t* kv = b_smem + stage * 2 * CTILE;
        for (int h = 0; h < 2; ++h) {
          tma_load_3d(&tma_k64, cb, smem_u32(kv + h * CHALF), h * 64, j * BC, bh, kEvictLast);
          tma_load_3d(&tma_v64, cb, smem_u32(kv + CTILE + h * CHALF), h * 64, j * BC, bh, kEvictLast);
        }
      }
    }
    return;
  }

  // ================= consumer warpgroup `wg`: queries [r0 + 64 wg, r0 + 64 wg + 64) =================
  const float c = p.scale_log2;
  float nl[2], dl[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = r0 + rloc + 8 * h;
    nl[h] = q < p.seq_q ? -__ldg(p.lse + (int64_t)bh * p.seq_q + q) : 0.f;
    dl[h] = q < p.seq_q ? __ldg(p.delta + (int64_t)bh * p.seq_q + q) : 0.f;
  }
  const uint32_t qa = smem_u32(a_smem) + wg * (64 * 128);
  const uint32_t doa = qa + BTILE;
  float dq[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) dq[i] = 0.f;
  mbar_wait(smem_u32(own_full), 0);

  for (int j = 0; j < nk; ++j) {
    const int stage = j % AB_STAGES;
    mbar_wait(smem_u32(&c_full[stage]), (j / AB_STAGES) & 1);
    const uint32_t kb = smem_u32(b_smem + stage * 2 * CTILE);
    const uint32_t vb = kb + CTILE;
    float sc[32], dp[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k)   // S[q, 64 kv] = Q K^T
      wgmma_m64n64k16_ss<0, 0>(sc, make_smem_desc(qa + kmajor_off(k, BHALF), 16, 1024),
                               make_smem_desc(kb + kmajor_off(k, CHALF), 16, 1024), k != 0);
#pragma unroll
    for (int k = 0; k < 8; ++k)   // dP[q, 64 kv] = dO V^T
      wgmma_m64n64k16_ss<0, 0>(dp, make_smem_desc(doa + kmajor_off(k, BHALF), 16, 1024),
                               make_smem_desc(vb + kmajor_off(k, CHALF), 16, 1024), k != 0);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<32>(sc);
    reg_fence<32>(dp);
    const int valid = p.seq_k - j * BC;   // keys of this chunk that exist
    uint32_t da[16];
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      const int h = (i >> 1) & 1;
      const int col = 8 * (i >> 2) + cq;
      const f32x2 e = f2_exp2_mufu(f2_fma(f2_pack(sc[i], sc[i + 1]), f2_pack(c, c), f2_pack(nl[h], nl[h])));
      float p0, p1;
      f2_unpack(e, p0, p1);
      if (col >= valid) p0 = 0.f;
      if (col + 1 >= valid) p1 = 0.f;
      const f32x2 d = f2_mul(f2_pack(p0, p1), f2_sub(f2_pack(dp[i], dp[i + 1]), f2_pack(dl[h], dl[h])));
      float d0, d1;
      f2_unpack(d, d0, d1);
      da[i >> 1] = pack_bf16(d0, d1);
    }
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BC / 16; ++k)   // dQ[q, d] += dS[q, 64 kv] K[64 kv, d]
      wgmma_m64n128k16_rs<1>(dq, da + 4 * k, make_smem_desc(kb + k * 2048, CHALF, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<64>(dq);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&c_empty[stage]));
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = r0 + rloc + 8 * h;
    if (q >= p.seq_q) continue;
    const int64_t o = ((int64_t)bh * p.seq_q + q) * 128;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
      *reinterpret_cast<uint32_t*>(p.dq + o + 8 * jb + cq) =
          pack_bf16(dq[4 * jb + 2 * h] * p.scale, dq[4 * jb + 2 * h + 1] * p.scale);
  }
}

}  // namespace dpipe

extern "C" int dpipe_attn_bwd(const dpipe_attn_bwd_args* a, void* stream) {
  using namespace dpipe;
  if (!a || !a->q || !a->k || !a->v || !a->o || !a->d_o || !a->lse || !a->delta || !a->dq || !a->dk || !a->dv)
    return fail(DPIPE_EINVAL, "dpipe_attn_bwd: null argument");
  if (a->batch <= 0 || a->heads <= 0 || a->seq_q <= 0 || a->seq_k <= 0) return fail(DPIPE_EINVAL, "dpipe_attn_bwd: empty problem");
  if (a->ldo % 8 || a->lddo % 8) return fail(DPIPE_EINVAL, "dpipe_attn_bwd: ldo/lddo must be multiples of 8");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int B = a->batch, H = a->heads, Lq = a->seq_q, Lk = a->seq_k;
  {
    const int64_t warps = (int64_t)B * Lq * H;
    const int wpb = 8;
    attn_bwd_delta_kernel<<<(unsigned)((warps + wpb - 1) / wpb), wpb * 32, 0, s>>>(
        reinterpret_cast<const __nv_bfloat16*>(a->o), a->ldo, reinterpret_cast<const __nv_bfloat16*>(a->d_o), a->lddo,
        a->delta, B, H, Lq);
  }
  // 128-row boxes for the tile a CTA owns, 64-row boxes for the chunks it streams
  CUtensorMap tq, tk, tv, tdo, tq64, tk64, tv64, tdo64;
  const uint64_t bh = (uint64_t)B * H;
  int rc;
  if ((rc = make_tmap_3d_bf16(&tq, a->q, 128, Lq, bh, 128, (uint64_t)Lq * 128, 64, BT, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tk, a->k, 128, Lk, bh, 128, (uint64_t)Lk * 128, 64, BT, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tv, a->v, 128, Lk, bh, 128, (uint64_t)Lk * 128, 64, BT, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tq64, a->q, 128, Lq, bh, 128, (uint64_t)Lq * 128, 64, BC, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tk64, a->k, 128, Lk, bh, 128, (uint64_t)Lk * 128, 64, BC, 1))) return rc;
  if ((rc = make_tmap_3d_bf16(&tv64, a->v, 128, Lk, bh, 128, (uint64_t)Lk * 128, 64, BC, 1))) return rc;
  {
    const uint64_t dims[4] = {128, (uint64_t)Lq, (uint64_t)H, (uint64_t)B};
    const uint64_t strides[3] = {(uint64_t)a->lddo, 128, (uint64_t)Lq * a->lddo};
    const uint32_t box[4] = {64, BT, 1, 1};
    const uint32_t box64[4] = {64, BC, 1, 1};
    if ((rc = make_tmap_4d_bf16(&tdo, a->d_o, dims, strides, box))) return rc;
    if ((rc = make_tmap_4d_bf16(&tdo64, a->d_o, dims, strides, box64))) return rc;
  }
  static bool configured = false;
  if (!configured) {
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dkv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM_BYTES));
    DPIPE_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_dq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM_BYTES));
    configured = true;
  }
  AttnBwdParams p;
  p.lse = a->lse; p.delta = a->delta;
  p.dq = reinterpret_cast<__nv_bfloat16*>(a->dq);
  p.dk = reinterpret_cast<__nv_bfloat16*>(a->dk);
  p.dv = reinterpret_cast<__nv_bfloat16*>(a->dv);
  p.batch = B; p.heads = H; p.seq_q = Lq; p.seq_k = Lk;
  p.scale = a->scale; p.scale_log2 = a->scale * 1.4426950408889634f;
  attn_bwd_dkv_kernel<<<dim3((Lk + BT - 1) / BT, H, B), DKV_THREADS, AB_SMEM_BYTES, s>>>(tq64, tk, tv, tdo64, p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  attn_bwd_dq_kernel<<<dim3((Lq + BT - 1) / BT, H, B), AB_THREADS, AB_SMEM_BYTES, s>>>(tq, tk64, tv64, tdo, p);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}
