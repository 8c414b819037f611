// CAME optimizer step (pytorch_optimizer.CAME, built for `type = 'CAME'`) as multi-tensor kernels over up to 64
// tensors per launch, with no host synchronisation:
//
//   second moment   cm_tile_kernel<false>  row sums over C and column partials over 128-row blocks of
//                                          u0 = g*g + eps1, fp64, one 128 x 128 tile per CTA (factored)   2 B / bf16 param
//                   cm_fold_kernel         folds the partials in a fixed order, beta2 EMA of exp_avg_sq_row / _col,
//                                          column factors rsqrt(col)
//                   cm_rowmean_kernel      row.mean(-1) per leading index and the row factors rsqrt(row / mean)
//   update RMS      cm_sumsq_kernel        per element u = r * c * g (1-D / 0-D: the beta2 EMA of exp_avg_sq and
//                                          u = rsqrt(v) * g); fp64 sum u^2 per CTA (8192 elements)         2 B / bf16 param
//                   cm_clip_kernel         one CTA per tensor: folds the CTA partials, clip divisor
//   residual        cm_tile_kernel<true>   u again, / clip divisor, m = beta1 m + (1 - beta1) u (written),
//                                          res = (u - m)^2 + eps2, its row sums and column partials       6 B / bf16 param
//                   cm_fold_kernel, cm_rowmean_kernel   as above with beta3 on exp_avg_res_row / _col
//   apply           cm_apply_kernel        p *= decay; p -= lr * (r_res * c_res * m)  (1-D / 0-D: m's update here,
//                                          and p -= lr * m)                                                6 B / bf16 param
//
// Every float operation is an IEEE round-to-nearest intrinsic in the order of oracle/came_ref.py came_param_emulated
// (bit-identical to it, fed with the sums these kernels write); tensors of a bf16 parameter round to bf16 after every
// op, as the text's bf16 torch ops do.  Reductions accumulate in fp64 in a fixed order and fold in a fixed order: no
// float atomics, bitwise repeatable.  The per-element kernels use 16-byte vectors when p, g, m (and v) share their
// offset mod 16 B, element-wise access otherwise; the tile kernels read one element per lane, coalesced along rows.
//                                                                     replaces CAME.step (train.py:698-700).
#include <cuda_bf16.h>

#include "host_util.h"
#include "optim_common.cuh"

namespace dpipe {
namespace {

constexpr int CM_MAX = 64;
constexpr int CM_THREADS = 256;
constexpr long long CM_ELEMS = 8192;    // elements of one tensor per CTA of the per-element kernels

struct CmList {
  dpipe_came_tensor t[CM_MAX];
  long long tile0[CM_MAX + 1];          // prefix sums: tiles, fold CTAs, (tensor, l) pairs (factored), element CTAs
  long long fold0[CM_MAX + 1];
  long long lrow0[CM_MAX + 1];
  long long cta0[CM_MAX + 1];
  long long rp[CM_MAX], cp[CM_MAX];     // scratch offsets (doubles) of the row / column partials
  long long pp;                         // scratch offset of the per-CTA sums of u^2
  int n;
};

// fp32 coefficients of one tensor's group, rounded from the doubles once per CTA
struct Coef {
  float b1, a1, b2, a2, b3, a3, eps1, eps2, lr, decay;
};

__device__ __forceinline__ Coef coef_of(const dpipe_came_tensor& T) {
  Coef c;
  c.b1 = __double2float_rn(T.beta1);
  c.a1 = __double2float_rn(__dsub_rn(1.0, T.beta1));
  c.b2 = __double2float_rn(T.beta2);
  c.a2 = __double2float_rn(__dsub_rn(1.0, T.beta2));
  c.b3 = __double2float_rn(T.beta3);
  c.a3 = __double2float_rn(__dsub_rn(1.0, T.beta3));
  c.eps1 = __double2float_rn(T.eps1);
  c.eps2 = __double2float_rn(T.eps2);
  c.lr = __double2float_rn(T.lr);
  c.decay = __double2float_rn(__dsub_rn(1.0, __dmul_rn(T.weight_decay, T.fixed_decay ? 1.0 : T.lr)));
  return c;
}

// per-tensor workspace layouts (include/dpipe.h): fac = [clip divisor, r_sq, c_sq, r_res, c_res],
// sums = [sum u^2, sq rows, sq columns, sq row-state sums, res rows, res columns, res row-state sums]
__device__ __forceinline__ float* rfac(const dpipe_came_tensor& T, bool res) {
  return T.fac + 1 + (res ? T.L * (T.R + T.C) : 0);
}
__device__ __forceinline__ float* cfac(const dpipe_came_tensor& T, bool res) { return rfac(T, res) + T.L * T.R; }
__device__ __forceinline__ double* sums_of(const dpipe_came_tensor& T, bool res) {
  return T.sums + 1 + (res ? T.L * (T.R + T.C + 1) : 0);
}

// ---------------------------------------------------------------------------------------------------------------------
// factored statistics
// ---------------------------------------------------------------------------------------------------------------------
// one element of a tile: u0 = g*g + eps1 (second moment), or the momentum update and res = (u - m)^2 + eps2, from the
// second moment's row and column factors
template <bool BF16, bool RES>
struct TileElem {
  const dpipe_came_tensor& T;
  const Coef& k;
  float clipdiv;
  __device__ __forceinline__ float row(long long l, long long r) const { return RES ? rfac(T, false)[l * T.R + r] : 0.f; }
  __device__ __forceinline__ float col(long long l, long long c) const { return RES ? cfac(T, false)[l * T.C + c] : 0.f; }
  __device__ __forceinline__ float operator()(long long j, float rf, float cf) const {
    const float g = ld1<BF16>(T.g, j);
    if (!RES) return R<BF16>(__fadd_rn(R<BF16>(__fmul_rn(g, g)), k.eps1));
    float u = R<BF16>(__fmul_rn(R<BF16>(__fmul_rn(rf, cf)), g));
    u = R<BF16>(__fdiv_rn(u, clipdiv));
    const float m = R<BF16>(__fmaf_rn(u, k.a1, R<BF16>(__fmul_rn(ld1<BF16>(T.m, j), k.b1))));
    st1<BF16>(T.m, j, m);
    const float d = R<BF16>(__fsub_rn(u, m));
    return R<BF16>(__fadd_rn(R<BF16>(__fmul_rn(d, d)), k.eps2));
  }
};

template <bool RES>
__global__ void __launch_bounds__(CM_THREADS) cm_tile_kernel(const __grid_constant__ CmList tl,
                                                            double* __restrict__ scratch) {
  __shared__ double colred[CM_THREADS / 32 * FM_TILE];
  long long b = blockIdx.x;
  const int i = find(tl.tile0, tl.n, b);
  const dpipe_came_tensor& T = tl.t[i];
  b -= tl.tile0[i];
  const FmGeom f{T.L, T.R, T.C};
  const Coef k = coef_of(T);
  const float clipdiv = RES ? T.fac[0] : 1.0f;
  if (T.dtype == 0) fm_tile<CM_THREADS>(f, b, scratch, tl.rp[i], tl.cp[i], colred, TileElem<true, RES>{T, k, clipdiv});
  else fm_tile<CM_THREADS>(f, b, scratch, tl.rp[i], tl.cp[i], colred, TileElem<false, RES>{T, k, clipdiv});
}

// one thread per row (then per column): fold the partials in a fixed order, EMA with beta (beta2 / beta3), column
// factors; the folded sums go to the tensor's `sums`
__global__ void __launch_bounds__(CM_THREADS) cm_fold_kernel(const __grid_constant__ CmList tl,
                                                            const double* __restrict__ scratch, int res) {
  long long b = blockIdx.x;
  const int i = find(tl.fold0, tl.n, b);
  const dpipe_came_tensor& T = tl.t[i];
  b -= tl.fold0[i];
  const Coef k = coef_of(T);
  const float beta = res ? k.b3 : k.b2, alpha = res ? k.a3 : k.a2;
  const bool bf = T.dtype == 0;
  const long long R_ = T.R, C = T.C, LR = T.L * R_, LC = T.L * C;
  const FmGeom f{T.L, R_, C};
  double* sums = sums_of(T, res);
  const long long nrowcta = f.row_ctas(CM_THREADS);
  if (b < nrowcta) {
    const long long q = b * CM_THREADS + threadIdx.x;
    if (q >= LR) return;
    const long long nstrip = f.nstrip();
    double a = 0.0;
    for (long long st = 0; st < nstrip; ++st) a += scratch[tl.rp[i] + st * LR + q];
    sums[q] = a;
    void* row = res ? T.res_row : T.row;
    const float mean = __double2float_rn(a / (double)C);                     // x.mean(dim=-1)
    // row.mul_(beta).add_(mean, alpha=1-beta): torch's add with alpha is one fma; every op rounds to the dtype
    float r;
    if (bf) r = R<true>(__fmaf_rn(R<true>(mean), alpha, R<true>(__fmul_rn(ld_dt(row, q, 0), beta))));
    else r = __fmaf_rn(mean, alpha, __fmul_rn(ld_dt(row, q, 1), beta));
    st_dt(row, q, r, T.dtype);
  } else {
    const long long q = (b - nrowcta) * CM_THREADS + threadIdx.x;
    if (q >= LC) return;
    const long long nrb = f.nrb();
    double a = 0.0;
    for (long long kk = 0; kk < nrb; ++kk) a += scratch[tl.cp[i] + kk * LC + q];
    sums[LR + q] = a;
    void* col = res ? T.res_col : T.col;
    const float mean = __double2float_rn(a / (double)R_);                    // x.mean(dim=-2)
    float c;
    if (bf) c = R<true>(__fmaf_rn(R<true>(mean), alpha, R<true>(__fmul_rn(ld_dt(col, q, 0), beta))));
    else c = __fmaf_rn(mean, alpha, __fmul_rn(ld_dt(col, q, 1), beta));
    st_dt(col, q, c, T.dtype);
    cfac(T, res)[q] = bf ? R<true>(rsqrt_rn(c)) : rsqrt_rn(c);                // col.rsqrt()
  }
}

// one CTA per (tensor, leading index l): row.mean(-1) and the row factors rsqrt(row / row.mean(-1))
__global__ void __launch_bounds__(CM_THREADS) cm_rowmean_kernel(const __grid_constant__ CmList tl, int res) {
  __shared__ double red[CM_THREADS / 32];
  long long b = blockIdx.x;
  const int i = find(tl.lrow0, tl.n, b);
  const dpipe_came_tensor& T = tl.t[i];
  const long long l = b - tl.lrow0[i];
  const bool bf = T.dtype == 0;
  const long long R_ = T.R;
  const void* row = res ? T.res_row : T.row;
  double a = 0.0;
  for (long long kk = threadIdx.x; kk < R_; kk += CM_THREADS) a += ld_dt(row, l * R_ + kk, T.dtype);
  a = block_sum<CM_THREADS>(a, red);
  if (threadIdx.x == 0) sums_of(T, res)[T.L * (R_ + T.C) + l] = a;
  float rm = __double2float_rn(a / (double)R_);
  if (bf) rm = R<true>(rm);
  float* rf = rfac(T, res) + l * R_;
  for (long long kk = threadIdx.x; kk < R_; kk += CM_THREADS) {
    const float x = ld_dt(row, l * R_ + kk, T.dtype);
    rf[kk] = bf ? R<true>(rsqrt_rn(R<true>(__fdiv_rn(x, rm)))) : rsqrt_rn(__fdiv_rn(x, rm));
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// per-element kernels: one CTA per CM_ELEMS elements of one tensor
// ---------------------------------------------------------------------------------------------------------------------
// p, g, m (and v of an unfactored tensor) go through 16-byte vectors when they share their offset mod 16 B
__host__ __device__ __forceinline__ bool vectorised(const dpipe_came_tensor& T) {
  const uintptr_t mis = reinterpret_cast<uintptr_t>(T.p) & 15;
  return (reinterpret_cast<uintptr_t>(T.g) & 15) == mis && (reinterpret_cast<uintptr_t>(T.m) & 15) == mis &&
         (T.factored || (reinterpret_cast<uintptr_t>(T.v) & 15) == mis);
}
// the factor pair of flat element j of a factored tensor [L, R, C]: rf[q] with q = j / C and cf[l * C + j % C]
struct Pos {
  long long q, c;
  __device__ __forceinline__ Pos(long long j, long long C) : q(j / C), c(j - (j / C) * C) {}
  __device__ __forceinline__ void next(long long C) {
    if (++c == C) { c = 0; ++q; }
  }
  __device__ __forceinline__ long long col(const dpipe_came_tensor& T) const { return (T.L == 1 ? 0 : q / T.R) * T.C + c; }
};

// u before clipping (second-moment factors), for factored tensors
template <bool BF16>
__device__ __forceinline__ float u_fact(const dpipe_came_tensor& T, const Pos& x, float g) {
  return R<BF16>(__fmul_rn(R<BF16>(__fmul_rn(rfac(T, false)[x.q], cfac(T, false)[x.col(T)])), g));
}
// 1-D / 0-D: v = beta2 v + (1 - beta2) u0, then u = rsqrt(v) * g
template <bool BF16>
__device__ __forceinline__ float u_plain(float g, float& v, const Coef& k) {
  const float u0 = R<BF16>(__fadd_rn(R<BF16>(__fmul_rn(g, g)), k.eps1));
  v = R<BF16>(__fmaf_rn(u0, k.a2, R<BF16>(__fmul_rn(v, k.b2))));
  return R<BF16>(__fmul_rn(R<BF16>(rsqrt_rn(v)), g));
}

template <bool BF16>
__device__ __forceinline__ float sumsq_at(const dpipe_came_tensor& T, const Coef& k, long long j) {
  const float g = ld1<BF16>(T.g, j);
  if (T.factored) return u_fact<BF16>(T, Pos(j, T.C), g);
  float v = ld1<BF16>(T.v, j);
  const float u = u_plain<BF16>(g, v, k);
  st1<BF16>(T.v, j, v);
  return u;
}

template <bool BF16>
__device__ __forceinline__ double sumsq_range(const dpipe_came_tensor& T, const Coef& k, long long b) {
  constexpr int VEC = BF16 ? 8 : 4;
  const long long h = head_of(T, vectorised(T)), lo = h + b * CM_ELEMS;
  const long long hi = lo + CM_ELEMS < T.numel ? lo + CM_ELEMS : T.numel;
  double s = 0.0;
  if (!vectorised(T)) {
    for (long long j = lo + threadIdx.x; j < hi; j += CM_THREADS) {
      const float u = sumsq_at<BF16>(T, k, j);
      s += (double)u * (double)u;
    }
    return s;
  }
  if (b == 0 && threadIdx.x < h) {
    const float u = sumsq_at<BF16>(T, k, threadIdx.x);
    s += (double)u * (double)u;
  }
  const long long nv = (hi - lo) / VEC;
  const long long esz = BF16 ? 2 : 4;
  const uint4* __restrict__ g4 = reinterpret_cast<const uint4*>(static_cast<const char*>(T.g) + lo * esz);
  for (long long j = threadIdx.x; j < nv; j += CM_THREADS) {
    const uint4 G = __ldg(g4 + j);
    if (T.factored) {
      Pos x(lo + j * VEC, T.C);
#pragma unroll
      for (int e = 0; e < VEC; ++e, x.next(T.C)) {
        const float u = u_fact<BF16>(T, x, lane<BF16>(G, e));
        s += (double)u * (double)u;
      }
    } else {
      uint4* __restrict__ v4 = reinterpret_cast<uint4*>(static_cast<char*>(T.v) + lo * esz);
      uint4 V = v4[j];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        float v = lane<BF16>(V, e);
        const float u = u_plain<BF16>(lane<BF16>(G, e), v, k);
        set_lane<BF16>(V, e, v);
        s += (double)u * (double)u;
      }
      v4[j] = V;
    }
  }
  const long long tail = lo + nv * VEC + threadIdx.x;
  if (tail < hi) {
    const float u = sumsq_at<BF16>(T, k, tail);
    s += (double)u * (double)u;
  }
  return s;
}

__global__ void __launch_bounds__(CM_THREADS) cm_sumsq_kernel(const __grid_constant__ CmList tl,
                                                             double* __restrict__ scratch) {
  __shared__ double red[CM_THREADS / 32];
  long long b = blockIdx.x;
  const int i = find(tl.cta0, tl.n, b);
  const dpipe_came_tensor& T = tl.t[i];
  b -= tl.cta0[i];
  const Coef k = coef_of(T);
  double s = T.dtype == 0 ? sumsq_range<true>(T, k, b) : sumsq_range<false>(T, k, b);
  s = block_sum<CM_THREADS>(s, red);
  if (threadIdx.x == 0) scratch[tl.pp + blockIdx.x] = s;
}

// one CTA per tensor: sum u^2 from its CTA partials in a fixed order; clip divisor
// max(fp32(sqrt(sum)) / fp32(sqrt(numel)) / clip_threshold, 1), each quotient rounded to the dtype
__global__ void __launch_bounds__(CM_THREADS) cm_clip_kernel(const __grid_constant__ CmList tl,
                                                            const double* __restrict__ scratch, double clip) {
  __shared__ double red[CM_THREADS / 32];
  const int i = blockIdx.x;
  const dpipe_came_tensor& T = tl.t[i];
  double s = 0.0;
  for (long long kk = tl.cta0[i] + threadIdx.x; kk < tl.cta0[i + 1]; kk += CM_THREADS) s += scratch[tl.pp + kk];
  s = block_sum<CM_THREADS>(s, red);
  if (threadIdx.x != 0) return;
  T.sums[0] = s;
  const bool bf = T.dtype == 0;
  float norm = __double2float_rn(sqrt(s));                                     // update.norm(2)
  if (bf) norm = R<true>(norm);
  float rms = __fdiv_rn(norm, __double2float_rn(sqrt((double)T.numel)));      // / math.sqrt(numel)
  if (bf) rms = R<true>(rms);
  float q = __fdiv_rn(rms, __double2float_rn(clip));                          // / clip_threshold
  if (bf) q = R<true>(q);
  T.fac[0] = fmaxf(q, 1.0f);                                                   // .clamp_(min=1.0)
}

// p *= decay; p -= lr * upd, with upd = r_res * c_res * m (factored) or m after its update here (1-D / 0-D)
template <bool BF16>
__device__ __forceinline__ float apply_elem(const dpipe_came_tensor& T, const Coef& k, const Pos& x, float p, float m) {
  const float upd = R<BF16>(__fmul_rn(R<BF16>(__fmul_rn(rfac(T, true)[x.q], cfac(T, true)[x.col(T)])), m));
  p = R<BF16>(__fmul_rn(p, k.decay));
  return R<BF16>(__fsub_rn(p, R<BF16>(__fmul_rn(upd, k.lr))));
}
template <bool BF16>
__device__ __forceinline__ float apply_plain(const Coef& k, float clipdiv, float p, float g, float v, float& m) {
  const float u = R<BF16>(__fdiv_rn(R<BF16>(__fmul_rn(R<BF16>(rsqrt_rn(v)), g)), clipdiv));
  m = R<BF16>(__fmaf_rn(u, k.a1, R<BF16>(__fmul_rn(m, k.b1))));
  p = R<BF16>(__fmul_rn(p, k.decay));
  return R<BF16>(__fsub_rn(p, R<BF16>(__fmul_rn(m, k.lr))));
}

template <bool BF16>
__device__ __forceinline__ void apply_at(const dpipe_came_tensor& T, const Coef& k, float clipdiv, long long j) {
  if (T.factored) {
    st1<BF16>(T.p, j, apply_elem<BF16>(T, k, Pos(j, T.C), ld1<BF16>(T.p, j), ld1<BF16>(T.m, j)));
  } else {
    float m = ld1<BF16>(T.m, j);
    st1<BF16>(T.p, j, apply_plain<BF16>(k, clipdiv, ld1<BF16>(T.p, j), ld1<BF16>(T.g, j), ld1<BF16>(T.v, j), m));
    st1<BF16>(T.m, j, m);
  }
}

template <bool BF16>
__device__ __forceinline__ void apply_range(const dpipe_came_tensor& T, const Coef& k, long long b) {
  constexpr int VEC = BF16 ? 8 : 4;
  const float clipdiv = T.fac[0];
  const long long h = head_of(T, vectorised(T)), lo = h + b * CM_ELEMS;
  const long long hi = lo + CM_ELEMS < T.numel ? lo + CM_ELEMS : T.numel;
  if (!vectorised(T)) {
    for (long long j = lo + threadIdx.x; j < hi; j += CM_THREADS) apply_at<BF16>(T, k, clipdiv, j);
    return;
  }
  if (b == 0 && threadIdx.x < h) apply_at<BF16>(T, k, clipdiv, threadIdx.x);
  const long long nv = (hi - lo) / VEC;
  const long long esz = BF16 ? 2 : 4;
  uint4* __restrict__ p4 = reinterpret_cast<uint4*>(static_cast<char*>(T.p) + lo * esz);
  uint4* __restrict__ m4 = reinterpret_cast<uint4*>(static_cast<char*>(T.m) + lo * esz);
  for (long long j = threadIdx.x; j < nv; j += CM_THREADS) {
    uint4 P = p4[j], M = m4[j];
    if (T.factored) {
      Pos x(lo + j * VEC, T.C);
#pragma unroll
      for (int e = 0; e < VEC; ++e, x.next(T.C)) set_lane<BF16>(P, e, apply_elem<BF16>(T, k, x, lane<BF16>(P, e), lane<BF16>(M, e)));
    } else {
      const uint4 G = __ldg(reinterpret_cast<const uint4*>(static_cast<const char*>(T.g) + lo * esz) + j);
      const uint4 V = __ldg(reinterpret_cast<const uint4*>(static_cast<const char*>(T.v) + lo * esz) + j);
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        float m = lane<BF16>(M, e);
        set_lane<BF16>(P, e, apply_plain<BF16>(k, clipdiv, lane<BF16>(P, e), lane<BF16>(G, e), lane<BF16>(V, e), m));
        set_lane<BF16>(M, e, m);
      }
      m4[j] = M;
    }
    p4[j] = P;
  }
  const long long tail = lo + nv * VEC + threadIdx.x;
  if (tail < hi) apply_at<BF16>(T, k, clipdiv, tail);
}

__global__ void __launch_bounds__(CM_THREADS) cm_apply_kernel(const __grid_constant__ CmList tl) {
  long long b = blockIdx.x;
  const int i = find(tl.cta0, tl.n, b);
  const dpipe_came_tensor& T = tl.t[i];
  b -= tl.cta0[i];
  const Coef k = coef_of(T);
  if (T.dtype == 0) apply_range<true>(T, k, b);
  else apply_range<false>(T, k, b);
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
bool beta_ok(double b) { return b >= 0.0 && b < 1.0; }

int check_tensors(const char* fn, const dpipe_came_tensor* t, int n) {
  if (n < 0) return fail(DPIPE_EINVAL, "%s: n < 0", fn);
  if (n > 0 && !t) return fail(DPIPE_EINVAL, "%s: null argument", fn);
  for (int i = 0; i < n; ++i) {
    const dpipe_came_tensor& T = t[i];
    if (T.dtype != 0 && T.dtype != 1) return fail(DPIPE_EINVAL, "%s: tensor %d has dtype %d (0 = bf16, 1 = fp32)", fn, i, T.dtype);
    if (T.numel < 0) return fail(DPIPE_EINVAL, "%s: tensor %d has numel < 0", fn, i);
    if (T.numel == 0) continue;
    if (!T.p || !T.g || !T.m || !T.fac || !T.sums) return fail(DPIPE_EINVAL, "%s: tensor %d has a null pointer", fn, i);
    if (!beta_ok(T.beta1) || !beta_ok(T.beta2) || !beta_ok(T.beta3))
      return fail(DPIPE_EINVAL, "%s: tensor %d: betas must lie in [0, 1)", fn, i);
    if (!(T.eps1 >= 0.0) || !(T.eps2 >= 0.0) || !(T.lr >= 0.0) || !(T.weight_decay >= 0.0))
      return fail(DPIPE_EINVAL, "%s: tensor %d: lr, weight_decay, eps1 and eps2 must be >= 0", fn, i);
    const int esz = T.dtype == 0 ? 2 : 4;
    if (T.factored) {
      if (T.L < 1 || T.R < 1 || T.C < 1 || T.L * T.R * T.C != T.numel)
        return fail(DPIPE_EINVAL, "%s: tensor %d: L * R * C = %lld * %lld * %lld is not numel %lld", fn, i, (long long)T.L,
                    (long long)T.R, (long long)T.C, (long long)T.numel);
      if (!T.row || !T.col || !T.res_row || !T.res_col)
        return fail(DPIPE_EINVAL, "%s: tensor %d: factored tensor without its row / column statistics", fn, i);
      for (const void* q : {(const void*)T.row, (const void*)T.col, (const void*)T.res_row, (const void*)T.res_col})
        if (misaligned(q, esz)) return fail(DPIPE_EINVAL, "%s: tensor %d is not aligned to its dtype", fn, i);
    } else if (!T.v) {
      return fail(DPIPE_EINVAL, "%s: tensor %d: unfactored tensor without exp_avg_sq", fn, i);
    } else if (misaligned(T.v, esz)) {
      return fail(DPIPE_EINVAL, "%s: tensor %d is not aligned to its dtype", fn, i);
    }
    for (const void* q : {(const void*)T.p, T.g, (const void*)T.m})
      if (misaligned(q, esz)) return fail(DPIPE_EINVAL, "%s: tensor %d is not aligned to its dtype", fn, i);
    if (misaligned(T.fac, 4) || misaligned(T.sums, 8))
      return fail(DPIPE_EINVAL, "%s: tensor %d: workspace not aligned", fn, i);
  }
  return 0;
}

// the next chunk of up to 64 non-empty tensors from *pos; fills the prefix sums and scratch offsets, returns the
// doubles of scratch the chunk needs
long long fill(CmList& tl, const dpipe_came_tensor* t, int n, int* pos) {
  tl.n = 0;
  tl.tile0[0] = tl.fold0[0] = tl.lrow0[0] = tl.cta0[0] = 0;
  long long off = 0;
  for (; *pos < n && tl.n < CM_MAX; ++*pos) {
    const dpipe_came_tensor& T = t[*pos];
    if (T.numel == 0) continue;
    const int k = tl.n++;
    tl.t[k] = T;
    long long tiles = 0, fold = 0, lrow = 0;
    tl.rp[k] = tl.cp[k] = off;
    if (T.factored) {
      const FmGeom f{T.L, T.R, T.C};
      tiles = f.tiles();
      fold = f.fold_ctas(CM_THREADS);
      lrow = T.L;
      tl.cp[k] = off + f.row_partials();
      off = tl.cp[k] + f.col_partials();
    }
    tl.tile0[k + 1] = tl.tile0[k] + tiles;
    tl.fold0[k + 1] = tl.fold0[k] + fold;
    tl.lrow0[k + 1] = tl.lrow0[k] + lrow;
    tl.cta0[k + 1] = tl.cta0[k] + ctas_of<CM_ELEMS>(T, vectorised(T));
  }
  tl.pp = off;
  return off + tl.cta0[tl.n];
}

long long scratch_needed(const dpipe_came_tensor* t, int n) {
  long long need = 0;
  for (int pos = 0; pos < n;) {
    CmList tl;
    const long long k = fill(tl, t, n, &pos);
    need = k > need ? k : need;
  }
  return need;
}

}  // namespace
}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_came_scratch_doubles(const dpipe_came_tensor* t, int n, int64_t* out) {
  if (!out) return fail(DPIPE_EINVAL, "dpipe_came_scratch_doubles: null argument");
  if (int e = check_tensors("dpipe_came_scratch_doubles", t, n)) return e;
  *out = scratch_needed(t, n);
  return 0;
}

extern "C" int dpipe_came_step(const dpipe_came_tensor* t, int n, double clip_threshold, double* scratch,
                               int64_t scratch_len, void* stream) {
  if (int e = check_tensors("dpipe_came_step", t, n)) return e;
  if (!(clip_threshold > 0.0)) return fail(DPIPE_EINVAL, "dpipe_came_step: clip_threshold must be > 0");
  const long long need = scratch_needed(t, n);
  if (need > 0 && (!scratch || scratch_len < need))
    return fail(DPIPE_EINVAL, "dpipe_came_step: scratch holds %lld doubles, needs %lld", (long long)scratch_len, need);
  cudaStream_t st = (cudaStream_t)stream;
  for (int pos = 0; pos < n;) {
    CmList tl;
    fill(tl, t, n, &pos);
    if (tl.n == 0) continue;
    const bool fact = tl.tile0[tl.n] > 0;
    if (fact) {
      cm_tile_kernel<false><<<(unsigned)tl.tile0[tl.n], CM_THREADS, 0, st>>>(tl, scratch);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      cm_fold_kernel<<<(unsigned)tl.fold0[tl.n], CM_THREADS, 0, st>>>(tl, scratch, 0);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      cm_rowmean_kernel<<<(unsigned)tl.lrow0[tl.n], CM_THREADS, 0, st>>>(tl, 0);
      DPIPE_CUDA_CHECK(cudaGetLastError());
    }
    cm_sumsq_kernel<<<(unsigned)tl.cta0[tl.n], CM_THREADS, 0, st>>>(tl, scratch);
    DPIPE_CUDA_CHECK(cudaGetLastError());
    cm_clip_kernel<<<tl.n, CM_THREADS, 0, st>>>(tl, scratch, clip_threshold);
    DPIPE_CUDA_CHECK(cudaGetLastError());
    if (fact) {
      cm_tile_kernel<true><<<(unsigned)tl.tile0[tl.n], CM_THREADS, 0, st>>>(tl, scratch);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      cm_fold_kernel<<<(unsigned)tl.fold0[tl.n], CM_THREADS, 0, st>>>(tl, scratch, 1);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      cm_rowmean_kernel<<<(unsigned)tl.lrow0[tl.n], CM_THREADS, 0, st>>>(tl, 1);
      DPIPE_CUDA_CHECK(cudaGetLastError());
    }
    cm_apply_kernel<<<(unsigned)tl.cta0[tl.n], CM_THREADS, 0, st>>>(tl);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}
