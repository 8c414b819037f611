// Prodigy optimizer step (pytorch_optimizer.Prodigy, built for `type = 'Prodigy'`) as multi-tensor kernels over up to
// 64 tensors per launch, in two phases with no host synchronisation; the step size d lives in a device block from one
// step to the next:
//
//   statistics  pg_stats_kernel   per element: m, v, s; per CTA (8192 elements of one tensor): fp64 sums of
//                                 g * (p0 - p) and |s_new|                                       18 B / bf16 parameter
//               pg_fold_kernel    one CTA per tensor: folds its CTA partials in a fixed order into scratch[2i..2i+1]
//               pg_finish_kernel  one thread, after every chunk: d_numerator, d_denom, d_hat, d, d_max, step, skip
//   apply       pg_apply_kernel   per element: denom = sqrt(v) + d * eps, decoupled weight decay, p -= d_lr * m / denom;
//                                 returns at once when the statistics phase set the skip flag      8 B / bf16 parameter
//
// Every float operation is an IEEE round-to-nearest intrinsic in the order of oracle/prodigy_ref.py (bit-identical to
// prodigy_stats_emulated / prodigy_fold / prodigy_apply_emulated); bf16 tensors round to bf16 after every op.  The
// scalars are computed in fp64 from the device block by every thread, with explicit _rn intrinsics (no contraction).
// 16-byte vectors when the tensors of a set share their offset mod 16 B, element-wise access otherwise.
//                                                                     replaces Prodigy.step (train.py:698-700).
#include <cuda_bf16.h>

#include "host_util.h"
#include "optim_common.cuh"

namespace dpipe {
namespace {

constexpr int PG_MAX = 64;
constexpr int PG_THREADS = 256;
constexpr long long PG_ELEMS = 8192;    // elements of one tensor per CTA

struct PgList {
  dpipe_prodigy_tensor t[PG_MAX];
  long long cta0[PG_MAX + 1];           // prefix sums of the CTAs per tensor
  int slot[PG_MAX];                     // index of t[i] in the caller's array (its sums slot)
  int n;
};

struct PgScal {
  double lr, omb1, omb2, beta1, beta2, d0, d_coef, growth_rate;
  float b1, b2, b3;
  double beta3;
  int bias_correction, safeguard_warmup;
};

// the per-step doubles every kernel derives from the device block in the same way
struct PgStep {
  double t, d, d_lr;
};

__device__ __forceinline__ double powi(double b, long long n) {     // oracle powi: b**n by squaring
  double r = 1.0, x = b;
  while (n) {
    if (n & 1) r = __dmul_rn(r, x);
    x = __dmul_rn(x, x);
    n >>= 1;
  }
  return r;
}

__device__ __forceinline__ PgStep step_of(const double* __restrict__ blk, const PgScal& s) {
  PgStep o;
  o.t = __dadd_rn(blk[DPIPE_PRODIGY_STEP], 1.0);
  o.d = blk[DPIPE_PRODIGY_D];
  double bc = 1.0;
  if (s.bias_correction) {
    const long long t = (long long)o.t;
    bc = __ddiv_rn(__dsub_rn(1.0, powi(s.beta1, t)), __dsqrt_rn(__dsub_rn(1.0, powi(s.beta2, t))));
  }
  o.d_lr = __ddiv_rn(__dmul_rn(o.d, s.lr), bc);
  return o;
}

// a tensor set goes through 16-byte vectors when all six tensors share their offset mod 16 B
__host__ __device__ __forceinline__ bool vectorised(const dpipe_prodigy_tensor& T) {
  const uintptr_t mis = reinterpret_cast<uintptr_t>(T.p) & 15;
  return (reinterpret_cast<uintptr_t>(T.g) & 15) == mis && (reinterpret_cast<uintptr_t>(T.p0) & 15) == mis &&
         (reinterpret_cast<uintptr_t>(T.s) & 15) == mis && (reinterpret_cast<uintptr_t>(T.m) & 15) == mis &&
         (reinterpret_cast<uintptr_t>(T.v) & 15) == mis;
}
struct StatCoef {
  float b1, b2, b3, am, av, as;
};

// statistics of one element (oracle prodigy_stats_emulated)
template <bool BF16>
__device__ __forceinline__ void stat_elem(float g, float p, float p0, float& s, float& m, float& v, const StatCoef& c,
                                          double& dot, double& asum) {
  const float diff = R<BF16>(__fsub_rn(p0, p));
  dot += (double)g * (double)diff;
  m = R<BF16>(__fmaf_rn(g, c.am, R<BF16>(__fmul_rn(m, c.b1))));
  v = R<BF16>(__fmaf_rn(c.av, __fmul_rn(g, g), R<BF16>(__fmul_rn(v, c.b2))));
  s = R<BF16>(__fmaf_rn(g, c.as, R<BF16>(__fmul_rn(s, c.b3))));
  asum += fabs((double)s);
}

template <bool BF16>
__device__ __forceinline__ void stat_at(const dpipe_prodigy_tensor& T, long long j, const StatCoef& c, double& dot,
                                        double& asum) {
  float s = ld1<BF16>(T.s, j), m = ld1<BF16>(T.m, j), v = ld1<BF16>(T.v, j);
  stat_elem<BF16>(ld1<BF16>(T.g, j), ld1<BF16>(T.p, j), ld1<BF16>(T.p0, j), s, m, v, c, dot, asum);
  st1<BF16>(T.s, j, s);
  st1<BF16>(T.m, j, m);
  st1<BF16>(T.v, j, v);
}

template <bool BF16>
__device__ __forceinline__ void stats_range(const dpipe_prodigy_tensor& T, long long b, const StatCoef& c, double& dot,
                                            double& asum) {
  constexpr int VEC = BF16 ? 8 : 4;
  const long long h = head_of(T, vectorised(T)), lo = h + b * PG_ELEMS;
  const long long hi = lo + PG_ELEMS < T.numel ? lo + PG_ELEMS : T.numel;
  if (!vectorised(T)) {
    for (long long j = lo + threadIdx.x; j < hi; j += PG_THREADS) stat_at<BF16>(T, j, c, dot, asum);
    return;
  }
  if (b == 0 && threadIdx.x < h) stat_at<BF16>(T, threadIdx.x, c, dot, asum);
  const long long nv = (hi - lo) / VEC;
  const uint4* __restrict__ g4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.g) + lo * (BF16 ? 2 : 4));
  const uint4* __restrict__ p4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.p) + lo * (BF16 ? 2 : 4));
  const uint4* __restrict__ q4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.p0) + lo * (BF16 ? 2 : 4));
  uint4* __restrict__ s4 = reinterpret_cast<uint4*>(static_cast<char*>(T.s) + lo * (BF16 ? 2 : 4));
  uint4* __restrict__ m4 = reinterpret_cast<uint4*>(static_cast<char*>(T.m) + lo * (BF16 ? 2 : 4));
  uint4* __restrict__ v4 = reinterpret_cast<uint4*>(static_cast<char*>(T.v) + lo * (BF16 ? 2 : 4));
  for (long long j = threadIdx.x; j < nv; j += PG_THREADS) {
    const uint4 G = __ldg(g4 + j), P = __ldg(p4 + j), Q = __ldg(q4 + j);
    uint4 S = s4[j], M = m4[j], V = v4[j];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      float s = lane<BF16>(S, k), m = lane<BF16>(M, k), v = lane<BF16>(V, k);
      stat_elem<BF16>(lane<BF16>(G, k), lane<BF16>(P, k), lane<BF16>(Q, k), s, m, v, c, dot, asum);
      set_lane<BF16>(S, k, s);
      set_lane<BF16>(M, k, m);
      set_lane<BF16>(V, k, v);
    }
    s4[j] = S;
    m4[j] = M;
    v4[j] = V;
  }
  const long long tail = lo + nv * VEC + threadIdx.x;
  if (tail < hi) stat_at<BF16>(T, tail, c, dot, asum);
}

__global__ void __launch_bounds__(PG_THREADS) pg_stats_kernel(const __grid_constant__ PgList tl, const PgScal sc,
                                                             const double* __restrict__ blk,
                                                             double* __restrict__ partials) {
  __shared__ double red[PG_THREADS / 32];
  long long b = blockIdx.x;
  const int i = find(tl.cta0, tl.n, b);
  const dpipe_prodigy_tensor& T = tl.t[i];
  b -= tl.cta0[i];
  const PgStep st = step_of(blk, sc);
  StatCoef c;
  c.b1 = sc.b1;
  c.b2 = sc.b2;
  c.b3 = sc.b3;
  c.am = __double2float_rn(__dmul_rn(st.d, sc.omb1));                                   // d * (1 - beta1)
  c.av = __double2float_rn(__dmul_rn(__dmul_rn(st.d, st.d), sc.omb2));                  // d * d * (1 - beta2)
  c.as = __double2float_rn(__dmul_rn(__ddiv_rn(st.d, sc.d0), sc.safeguard_warmup ? st.d : st.d_lr));
  double dot = 0.0, asum = 0.0;
  if (T.dtype == 0) stats_range<true>(T, b, c, dot, asum);
  else stats_range<false>(T, b, c, dot, asum);
  dot = block_sum<PG_THREADS>(dot, red);
  asum = block_sum<PG_THREADS>(asum, red);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = dot;
    partials[2 * blockIdx.x + 1] = asum;
  }
}

// one CTA per tensor of the chunk: its partials in a fixed order -> sums[2 * slot[i]]
__global__ void __launch_bounds__(PG_THREADS) pg_fold_kernel(const __grid_constant__ PgList tl,
                                                            const double* __restrict__ partials,
                                                            double* __restrict__ sums) {
  __shared__ double red[PG_THREADS / 32];
  const int i = blockIdx.x;
  double dot = 0.0, asum = 0.0;
  for (long long k = tl.cta0[i] + threadIdx.x; k < tl.cta0[i + 1]; k += PG_THREADS) {
    dot += partials[2 * k];
    asum += partials[2 * k + 1];
  }
  dot = block_sum<PG_THREADS>(dot, red);
  asum = block_sum<PG_THREADS>(asum, red);
  if (threadIdx.x == 0) {
    sums[2 * tl.slot[i]] = dot;
    sums[2 * tl.slot[i] + 1] = asum;
  }
}

// oracle prodigy_fold, in tensor order, in fp64 (Python's max(a, b) keeps a unless b > a; min(a, b) unless b < a)
__global__ void pg_finish_kernel(const PgScal sc, double* __restrict__ blk, const double* __restrict__ sums, int n) {
  if (threadIdx.x != 0) return;
  const PgStep st = step_of(blk, sc);
  const double k = __dmul_rn(__ddiv_rn(st.d, sc.d0), st.d_lr);
  double num = __dmul_rn(blk[DPIPE_PRODIGY_D_NUMERATOR], sc.beta3);
  for (int i = 0; i < n; ++i) num = __dadd_rn(num, __dmul_rn(k, sums[2 * i]));
  double den = 0.0;
  for (int i = 0; i < n; ++i) den = __dadd_rn(den, sums[2 * i + 1]);
  blk[DPIPE_PRODIGY_D_NUMERATOR] = num;
  blk[DPIPE_PRODIGY_D_LR] = st.d_lr;
  if (den == 0.0) {
    blk[DPIPE_PRODIGY_SKIP] = 1.0;
    return;
  }
  double d = st.d;
  const double d_hat = __ddiv_rn(__dmul_rn(sc.d_coef, num), den);
  if (d == sc.d0) d = d_hat > d ? d_hat : d;
  const double d_max = d_hat > blk[DPIPE_PRODIGY_D_MAX] ? d_hat : blk[DPIPE_PRODIGY_D_MAX];
  const double dg = __dmul_rn(d, sc.growth_rate);
  blk[DPIPE_PRODIGY_D] = dg < d_max ? dg : d_max;
  blk[DPIPE_PRODIGY_D_MAX] = d_max;
  blk[DPIPE_PRODIGY_D_HAT] = d_hat;
  blk[DPIPE_PRODIGY_D_DENOM] = den;
  blk[DPIPE_PRODIGY_STEP] = st.t;
  blk[DPIPE_PRODIGY_SKIP] = 0.0;
}

struct ApplyCoef {
  float decay, deps, ndlr;
};

template <bool BF16>
__device__ __forceinline__ float apply_elem(float p, float m, float v, const ApplyCoef& c) {
  const float den = R<BF16>(__fadd_rn(R<BF16>(__fsqrt_rn(v)), c.deps));       // exp_avg_sq.sqrt().add_(d * eps)
  p = R<BF16>(__fmul_rn(p, c.decay));                                          // p.mul_(1 - wd * d_lr)
  return R<BF16>(__fmaf_rn(c.ndlr, __fdiv_rn(m, den), p));                     // p.addcdiv_(m, den, value=-d_lr)
}

template <bool BF16>
__device__ __forceinline__ void apply_range(const dpipe_prodigy_tensor& T, long long b, const ApplyCoef& c) {
  constexpr int VEC = BF16 ? 8 : 4;
  const long long h = head_of(T, vectorised(T)), lo = h + b * PG_ELEMS;
  const long long hi = lo + PG_ELEMS < T.numel ? lo + PG_ELEMS : T.numel;
  if (!vectorised(T)) {
    for (long long j = lo + threadIdx.x; j < hi; j += PG_THREADS)
      st1<BF16>(T.p, j, apply_elem<BF16>(ld1<BF16>(T.p, j), ld1<BF16>(T.m, j), ld1<BF16>(T.v, j), c));
    return;
  }
  if (b == 0 && threadIdx.x < h) {
    const long long j = threadIdx.x;
    st1<BF16>(T.p, j, apply_elem<BF16>(ld1<BF16>(T.p, j), ld1<BF16>(T.m, j), ld1<BF16>(T.v, j), c));
  }
  const long long nv = (hi - lo) / VEC;
  uint4* __restrict__ p4 = reinterpret_cast<uint4*>(static_cast<char*>(T.p) + lo * (BF16 ? 2 : 4));
  const uint4* __restrict__ m4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.m) + lo * (BF16 ? 2 : 4));
  const uint4* __restrict__ v4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.v) + lo * (BF16 ? 2 : 4));
  for (long long j = threadIdx.x; j < nv; j += PG_THREADS) {
    uint4 P = p4[j];
    const uint4 M = __ldg(m4 + j), V = __ldg(v4 + j);
#pragma unroll
    for (int k = 0; k < VEC; ++k) set_lane<BF16>(P, k, apply_elem<BF16>(lane<BF16>(P, k), lane<BF16>(M, k), lane<BF16>(V, k), c));
    p4[j] = P;
  }
  const long long j = lo + nv * VEC + threadIdx.x;
  if (j < hi) st1<BF16>(T.p, j, apply_elem<BF16>(ld1<BF16>(T.p, j), ld1<BF16>(T.m, j), ld1<BF16>(T.v, j), c));
}

__global__ void __launch_bounds__(PG_THREADS) pg_apply_kernel(const __grid_constant__ PgList tl,
                                                             const double* __restrict__ blk) {
  if (blk[DPIPE_PRODIGY_SKIP] != 0.0) return;
  long long b = blockIdx.x;
  const int i = find(tl.cta0, tl.n, b);
  const dpipe_prodigy_tensor& T = tl.t[i];
  b -= tl.cta0[i];
  const double d_lr = blk[DPIPE_PRODIGY_D_LR], d = blk[DPIPE_PRODIGY_D];
  ApplyCoef c;
  c.decay = __double2float_rn(__dsub_rn(1.0, __dmul_rn(T.weight_decay, T.fixed_decay ? 1.0 : d_lr)));
  c.deps = __double2float_rn(__dmul_rn(d, T.eps));
  c.ndlr = __double2float_rn(-d_lr);
  if (T.dtype == 0) apply_range<true>(T, b, c);
  else apply_range<false>(T, b, c);
}

int check_tensors(const char* fn, const dpipe_prodigy_tensor* t, int n) {
  if (n < 0) return fail(DPIPE_EINVAL, "%s: n < 0", fn);
  if (n > 0 && !t) return fail(DPIPE_EINVAL, "%s: null argument", fn);
  for (int i = 0; i < n; ++i) {
    const dpipe_prodigy_tensor& T = t[i];
    if (T.dtype != 0 && T.dtype != 1) return fail(DPIPE_EINVAL, "%s: tensor %d has dtype %d (0 = bf16, 1 = fp32)", fn, i, T.dtype);
    if (T.numel < 0) return fail(DPIPE_EINVAL, "%s: tensor %d has numel < 0", fn, i);
    if (T.numel == 0) continue;
    if (!T.p || !T.g || !T.p0 || !T.s || !T.m || !T.v) return fail(DPIPE_EINVAL, "%s: tensor %d has a null pointer", fn, i);
    const uintptr_t esz = T.dtype == 0 ? 2 : 4;
    for (const void* q : {(const void*)T.p, T.g, T.p0, (const void*)T.s, (const void*)T.m, (const void*)T.v})
      if (reinterpret_cast<uintptr_t>(q) % esz) return fail(DPIPE_EINVAL, "%s: tensor %d is not aligned to its dtype", fn, i);
  }
  return 0;
}

PgScal make_scalars(const dpipe_prodigy_scalars* s) {
  PgScal a;
  a.lr = s->lr;
  a.beta1 = s->beta1;
  a.beta2 = s->beta2;
  a.omb1 = 1.0 - s->beta1;
  a.omb2 = 1.0 - s->beta2;
  a.beta3 = s->beta3;
  a.d0 = s->d0;
  a.d_coef = s->d_coef;
  a.growth_rate = s->growth_rate;
  a.b1 = (float)s->beta1;
  a.b2 = (float)s->beta2;
  a.b3 = (float)s->beta3;
  a.bias_correction = s->bias_correction;
  a.safeguard_warmup = s->safeguard_warmup;
  return a;
}

// the next chunk of up to 64 non-empty tensors from *pos (empty ones are skipped: their sums stay 0); returns its CTA
// count
long long fill(PgList& tl, const dpipe_prodigy_tensor* t, int n, int* pos) {
  tl.n = 0;
  tl.cta0[0] = 0;
  for (; *pos < n && tl.n < PG_MAX; ++*pos) {
    if (t[*pos].numel == 0) continue;
    tl.t[tl.n] = t[*pos];
    tl.slot[tl.n] = *pos;
    tl.cta0[tl.n + 1] = tl.cta0[tl.n] + ctas_of<PG_ELEMS>(t[*pos], vectorised(t[*pos]));
    ++tl.n;
  }
  return tl.cta0[tl.n];
}

long long partials_needed(const dpipe_prodigy_tensor* t, int n) {
  long long need = 0;
  for (int pos = 0; pos < n;) {
    PgList tl;
    const long long k = fill(tl, t, n, &pos);
    need = k > need ? k : need;
  }
  return 2 * need;
}

}  // namespace
}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_prodigy_scratch_doubles(const dpipe_prodigy_tensor* t, int n, int64_t* out) {
  if (!out) return fail(DPIPE_EINVAL, "dpipe_prodigy_scratch_doubles: null argument");
  if (int e = check_tensors("dpipe_prodigy_scratch_doubles", t, n)) return e;
  *out = 2LL * n + partials_needed(t, n);
  return 0;
}

extern "C" int dpipe_prodigy_stats(const dpipe_prodigy_tensor* t, int n, const dpipe_prodigy_scalars* s, double* state,
                                   double* scratch, int64_t scratch_len, void* stream) {
  if (int e = check_tensors("dpipe_prodigy_stats", t, n)) return e;
  if (!s || !state) return fail(DPIPE_EINVAL, "dpipe_prodigy_stats: null scalars or state block");
  if (!(s->d0 > 0.0)) return fail(DPIPE_EINVAL, "dpipe_prodigy_stats: d0 must be > 0");
  if (!(s->beta1 >= 0.0 && s->beta1 < 1.0 && s->beta2 >= 0.0 && s->beta2 < 1.0))
    return fail(DPIPE_EINVAL, "dpipe_prodigy_stats: betas must lie in [0, 1)");
  const long long need = 2LL * n + partials_needed(t, n);
  if (!scratch || scratch_len < need)
    return fail(DPIPE_EINVAL, "dpipe_prodigy_stats: scratch holds %lld doubles, needs %lld", (long long)scratch_len, need);
  const PgScal sc = make_scalars(s);
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0) DPIPE_CUDA_CHECK(cudaMemsetAsync(scratch, 0, sizeof(double) * 2 * (size_t)n, st));   // empty tensors: 0, 0
  for (int pos = 0; pos < n;) {
    PgList tl;
    const long long ctas = fill(tl, t, n, &pos);
    if (tl.n == 0) continue;
    pg_stats_kernel<<<(unsigned)ctas, PG_THREADS, 0, st>>>(tl, sc, state, scratch + 2LL * n);
    DPIPE_CUDA_CHECK(cudaGetLastError());
    pg_fold_kernel<<<tl.n, PG_THREADS, 0, st>>>(tl, scratch + 2LL * n, scratch);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  pg_finish_kernel<<<1, 32, 0, st>>>(sc, state, scratch, n);
  DPIPE_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" int dpipe_prodigy_apply(const dpipe_prodigy_tensor* t, int n, const double* state, void* stream) {
  if (int e = check_tensors("dpipe_prodigy_apply", t, n)) return e;
  if (!state) return fail(DPIPE_EINVAL, "dpipe_prodigy_apply: null state block");
  for (int pos = 0; pos < n;) {
    PgList tl;
    const long long ctas = fill(tl, t, n, &pos);
    if (tl.n == 0) continue;
    pg_apply_kernel<<<(unsigned)ctas, PG_THREADS, 0, (cudaStream_t)stream>>>(tl, state);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}
