// Device code shared by the optimizer step kernels (step_tail.cu, automagic.cu, prodigy.cu, adamw8bit.cu, came.cu):
// rounding and element access, the tensor of a CTA, fixed-order fp64 sums, the 16-byte layout of a per-element pass,
// and the row / column sums of the factored (Adafactor) second-moment statistics.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace dpipe {

// ---------------------------------------------------------------------------------------------------------------------
// rounding and element access; bf16 tensors are dtype 0, fp32 tensors dtype 1
// ---------------------------------------------------------------------------------------------------------------------
template <bool BF16>
__device__ __forceinline__ float R(float x) { return BF16 ? __bfloat162float(__float2bfloat16_rn(x)) : x; }
__device__ __forceinline__ float rnd(float x, bool r) { return r ? __bfloat162float(__float2bfloat16_rn(x)) : x; }
__device__ __forceinline__ float rsqrt_rn(float x) { return __fdiv_rn(1.0f, __fsqrt_rn(x)); }   // torch: 1 / sqrt(x)

template <bool BF16>
__device__ __forceinline__ float ld1(const void* __restrict__ a, long long j) {
  return BF16 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a)[j]) : reinterpret_cast<const float*>(a)[j];
}
template <bool BF16>
__device__ __forceinline__ void st1(void* __restrict__ a, long long j, float x) {   // x is a value of the dtype
  if (BF16) reinterpret_cast<__nv_bfloat16*>(a)[j] = __float2bfloat16_rn(x);
  else reinterpret_cast<float*>(a)[j] = x;
}
// (spelled out rather than through ld1: its __restrict__ parameter changes the code of Automagic's per-element kernels)
__device__ __forceinline__ float ld_dt(const void* a, long long j, int dt) {
  return dt == 0 ? __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(a)[j]) : reinterpret_cast<const float*>(a)[j];
}
__device__ __forceinline__ void st_dt(void* a, long long j, float x, int dt) {
  if (dt == 0) st1<true>(a, j, x);
  else st1<false>(a, j, x);
}

// element k of a 16-byte vector (8 bf16 or 4 fp32), and its replacement by a value of the dtype
template <bool BF16>
__device__ __forceinline__ float lane(const uint4& q, int k) {
  const uint32_t w = (&q.x)[BF16 ? k >> 1 : k];
  return BF16 ? __uint_as_float((k & 1) ? (w & 0xffff0000u) : (w << 16)) : __uint_as_float(w);
}
template <bool BF16>
__device__ __forceinline__ void set_lane(uint4& q, int k, float x) {
  uint32_t& w = (&q.x)[BF16 ? k >> 1 : k];
  if (BF16) {
    const uint32_t b = __float_as_uint(x) >> 16;
    w = (k & 1) ? ((w & 0xffffu) | (b << 16)) : ((w & 0xffff0000u) | b);
  } else {
    w = __float_as_uint(x);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// multi-tensor launches and fixed-order sums
// ---------------------------------------------------------------------------------------------------------------------
// the tensor of CTA b, from the prefix sums pre[0..n] of the CTAs per tensor
__device__ __forceinline__ int find(const long long* pre, int n, long long b) {
  int lo = 0, hi = n - 1;                                   // last i with pre[i] <= b
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (pre[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// deterministic sum over a CTA of THREADS threads (fixed tree); red holds THREADS / 32 doubles; valid in every thread
template <int THREADS>
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < THREADS / 32; ++w) s += red[w];
  return s;
}

// ---------------------------------------------------------------------------------------------------------------------
// per-element passes in CTAs of ELEMS elements of one tensor T (any record with p, numel and dtype).  When every pointer
// the pass reads or writes shares p's offset mod 16 B (vec), the elements before p's first 16-byte boundary (the head)
// go one by one in CTA 0, the rest in 16-byte vectors and an element-wise tail per CTA; otherwise every element goes
// one by one.
// ---------------------------------------------------------------------------------------------------------------------
template <class Tensor>
__host__ __device__ __forceinline__ long long head_of(const Tensor& T, bool vec) {
  if (!vec) return 0;
  const long long esz = T.dtype == 0 ? 2 : 4;
  const long long h = (long long)((16 - (reinterpret_cast<uintptr_t>(T.p) & 15)) & 15) / esz;
  return h < T.numel ? h : T.numel;
}
template <long long ELEMS, class Tensor>
__host__ __device__ __forceinline__ long long ctas_of(const Tensor& T, bool vec) {
  const long long body = T.numel - head_of(T, vec);
  return body > ELEMS ? (body + ELEMS - 1) / ELEMS : 1;
}

// ---------------------------------------------------------------------------------------------------------------------
// factored statistics of a [L, R, C] tensor: the row sums over C and the column sums over R of an element x, in fp64.
// One CTA per FM_TILE x FM_TILE tile writes the row sums of its column strip and the column partials of its row block
// to scratch; a fold kernel adds those in a fixed order, one thread per row (then per column).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int FM_TILE = 128;            // tile: 128 rows (16 per warp of 256 threads) x 128 columns (4 per lane)

struct FmGeom {
  long long L, R, C;
  __host__ __device__ long long nstrip() const { return (C + FM_TILE - 1) / FM_TILE; }   // column strips
  __host__ __device__ long long nrb() const { return (R + FM_TILE - 1) / FM_TILE; }      // row blocks
  __host__ __device__ long long tiles() const { return L * nrb() * nstrip(); }
  __host__ __device__ long long row_partials() const { return nstrip() * L * R; }        // doubles of scratch
  __host__ __device__ long long col_partials() const { return nrb() * L * C; }
  __host__ __device__ long long row_ctas(int threads) const { return (L * R + threads - 1) / threads; }
  __host__ __device__ long long fold_ctas(int threads) const { return row_ctas(threads) + (L * C + threads - 1) / threads; }
};

// tile b of the tensor: row sums to scratch[rp + strip * L*R + l * R + r], column partials to
// scratch[cp + rb * L*C + l * C + c].  x = e(j, e.row(l, r), e.col(l, c)) for flat element j at (l, r, c); e.row is read
// once per row and e.col once per column of the tile.  colred: THREADS / 32 * FM_TILE doubles of shared memory.
template <int THREADS, class E>
__device__ __forceinline__ void fm_tile(const FmGeom& f, long long b, double* __restrict__ scratch, long long rp,
                                        long long cp, double* colred, const E& e) {
  const long long R_ = f.R, C = f.C, LR = f.L * R_, LC = f.L * C;
  const long long nstrip = f.nstrip(), nrb = f.nrb();
  const long long strip = b % nstrip;
  b /= nstrip;
  const long long rb = b % nrb, l = b / nrb;
  const int warp = threadIdx.x >> 5, ln = threadIdx.x & 31;
  double cacc[4] = {0.0, 0.0, 0.0, 0.0};
  const long long c0 = strip * FM_TILE + ln;
  float cv[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) cv[j] = c0 + 32 * j < C ? e.col(l, c0 + 32 * j) : 0.f;
#pragma unroll 1                                                             // unrolled, the u0 pass spills
  for (int kk = 0; kk < FM_TILE / (THREADS / 32); ++kk) {
    const long long r = rb * FM_TILE + warp + (THREADS / 32) * kk;
    if (r >= R_) break;                                                      // warp-uniform
    const long long base = (l * R_ + r) * C;
    const float rv = e.row(l, r);
    double rs = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c0 + 32 * j < C) {
        const double x = e(base + c0 + 32 * j, rv, cv[j]);
        rs += x;
        cacc[j] += x;
      }
    }
    rs = warp_sum(rs);
    if (ln == 0) scratch[rp + strip * LR + l * R_ + r] = rs;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) colred[warp * FM_TILE + ln + 32 * j] = cacc[j];
  __syncthreads();
  if (threadIdx.x < FM_TILE) {
    const long long c = strip * FM_TILE + threadIdx.x;
    if (c < C) {
      double a = 0.0;
      for (int w = 0; w < THREADS / 32; ++w) a += colred[w * FM_TILE + threadIdx.x];
      scratch[cp + rb * LC + l * C + c] = a;
    }
  }
}

}  // namespace dpipe
