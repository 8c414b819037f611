// Automagic optimizer step (the reference's optimizers/automagic.py, built for `type = 'automagic'`) as multi-tensor
// kernels over up to 64 tensors per launch, in two phases with no host synchronisation:
//
//   statistics  am_reduce_kernel   row sums over C and column partials over 128-row blocks of u0 = g*g + eps, fp64,
//                                  one 128 x 128 tile per CTA (factored tensors)
//               am_fold_kernel     folds the partials in a fixed order, EMA of exp_avg_sq_row / exp_avg_sq_col and
//                                  the column factors rsqrt(col)
//               am_rowmean_kernel  row.mean(-1) per leading index and the row factors rsqrt(row / row.mean(-1))
//               am_lr_kernel       per element: u (EMA of exp_avg_sq for 1-D / 0-D tensors), new_lr; per CTA:
//                                  sum u^2, sum new_lr, max |new_lr| (fp64 / fp32, one partial per CTA)
//               am_finish_kernel   folds the partials (fixed order): clip divisor, avg_lr, lr code scale
//   apply       am_apply_kernel    per element: u again, / clip divisor, new polarity, new lr codes, weight decay,
//                                  Kahan-summed bf16 (or plain fp32) weight update
//
// Every float operation is an IEEE round-to-nearest intrinsic in the order of the reference's torch ops; at step 1 of
// a bf16 parameter every op on the statistics and on u rounds to bf16, because the reference's state tensors are bf16
// then.  Reductions accumulate in fp64 per thread in a fixed order and fold in a fixed order: no float atomics, bitwise
// repeatable.  Bit-identical (apply phase) to oracle/automagic_ref.py automagic_apply_emulated.
//                                                                     replaces Automagic.step (optimizers/automagic.py
//                                                                     :175-344, train.py:692-694).
#include <cuda_bf16.h>

#include "host_util.h"
#include "optim_common.cuh"

namespace dpipe {
namespace {

constexpr int AM_MAX = 64;
constexpr int AM_THREADS = 256;
constexpr int AM_WS_HEAD = 4;           // ws[0] clip divisor, ws[1] lr absmax, ws[2] avg_lr, ws[3] fp32(previous scale)

struct AmList {
  dpipe_automagic_tensor t[AM_MAX];
  long long tiles0[AM_MAX + 1];         // prefix sums: reduce tiles, fold CTAs, (tensor, l) pairs
  long long fold0[AM_MAX + 1];
  long long lrow0[AM_MAX + 1];
  long long rp[AM_MAX], cp[AM_MAX];     // scratch offsets (doubles) of the row / column partials
  long long pp;                         // scratch offset of the am_lr_kernel partials: [n][grid][3]
  int n;
};

struct AmScal {
  float beta2, alpha, eps, bump, min_lr, max_lr, clip, neg_wd;
  int has_wd;
};

__device__ __forceinline__ float new_lr(float u, signed char code, unsigned char pol, float scale, const AmScal& s) {
  const float mask = __fmul_rn((float)code, scale);                          // lr_mask = q.float() * scale
  const float nl = ((u > 0.f) == (pol != 0)) ? __fadd_rn(mask, s.bump) : __fsub_rn(mask, s.bump);
  return fminf(fmaxf(nl, s.min_lr), s.max_lr);                               // clamp(min_lr, max_lr)
}

// u before clipping for a factored tensor: (r_factor * c_factor) * g
__device__ __forceinline__ float u_factored(float rf, float cf, float g, bool r) {
  return rnd(__fmul_rn(rnd(__fmul_rn(rf, cf), r), g), r);
}

// walks the flat index j of an [L*R, C] tensor in steps of `stride` without a division per element
struct RowCol {
  long long q, c, sq, sc;
  __device__ RowCol(long long j, long long stride, long long C) : q(j / C), c(j % C), sq(stride / C), sc(stride % C) {}
  __device__ __forceinline__ void next(long long C) {
    c += sc;
    q += sq;
    if (c >= C) { c -= C; ++q; }
  }
};

// u0 = grad**2 + eps of a tile element, in fp32 at every step
struct U0 {
  const dpipe_automagic_tensor& T;
  float eps;
  __device__ __forceinline__ float row(long long, long long) const { return 0.f; }
  __device__ __forceinline__ float col(long long, long long) const { return 0.f; }
  __device__ __forceinline__ float operator()(long long j, float, float) const {
    const float g = ld_dt(T.g, j, T.dtype);
    return __fadd_rn(__fmul_rn(g, g), eps);
  }
};

__global__ void __launch_bounds__(AM_THREADS) am_reduce_kernel(const __grid_constant__ AmList tl, const AmScal s,
                                                              double* __restrict__ scratch) {
  __shared__ double colred[AM_THREADS / 32 * FM_TILE];
  long long b = blockIdx.x;
  const int i = find(tl.tiles0, tl.n, b);
  const dpipe_automagic_tensor& T = tl.t[i];
  b -= tl.tiles0[i];
  fm_tile<AM_THREADS>(FmGeom{T.L, T.R, T.C}, b, scratch, tl.rp[i], tl.cp[i], colred, U0{T, s.eps});
}

// one thread per row (then per column) of a factored tensor: fold the partials, EMA, column factors
__global__ void __launch_bounds__(AM_THREADS) am_fold_kernel(const __grid_constant__ AmList tl, const AmScal s,
                                                            const double* __restrict__ scratch) {
  long long b = blockIdx.x;
  const int i = find(tl.fold0, tl.n, b);
  const dpipe_automagic_tensor& T = tl.t[i];
  b -= tl.fold0[i];
  const bool r = T.flags & DPIPE_AUTOMAGIC_ROUND_BF16;
  const long long R = T.R, C = T.C, LR = T.L * R, LC = T.L * C;
  const FmGeom f{T.L, R, C};
  const long long nrowcta = f.row_ctas(AM_THREADS);
  if (b < nrowcta) {
    const long long q = b * AM_THREADS + threadIdx.x;
    if (q >= LR) return;
    const long long nstrip = f.nstrip();
    double a = 0.0;
    for (long long st = 0; st < nstrip; ++st) a += scratch[tl.rp[i] + st * LR + q];
    const float mean = __double2float_rn(a / (double)C);                     // update.mean(dim=-1)
    // row.mul_(beta2).add_(mean, alpha=1-beta2): torch's vectorised add with alpha is one fused multiply-add
    T.row[q] = rnd(__fmaf_rn(mean, s.alpha, rnd(__fmul_rn(T.row[q], s.beta2), r)), r);
  } else {
    const long long q = (b - nrowcta) * AM_THREADS + threadIdx.x;
    if (q >= LC) return;
    const long long nrb = f.nrb();
    double a = 0.0;
    for (long long k = 0; k < nrb; ++k) a += scratch[tl.cp[i] + k * LC + q];
    const float mean = __double2float_rn(a / (double)R);                     // update.mean(dim=-2)
    const float col = rnd(__fmaf_rn(mean, s.alpha, rnd(__fmul_rn(T.col[q], s.beta2), r)), r);
    T.col[q] = col;
    T.ws[AM_WS_HEAD + T.L + LR + q] = rnd(rsqrt_rn(col), r);                  // c_factor
  }
}

// one CTA per (tensor, leading index l): row.mean(-1) and the row factors rsqrt(row / row.mean(-1))
__global__ void __launch_bounds__(AM_THREADS) am_rowmean_kernel(const __grid_constant__ AmList tl) {
  __shared__ double red[AM_THREADS / 32];
  long long b = blockIdx.x;
  const int i = find(tl.lrow0, tl.n, b);
  const dpipe_automagic_tensor& T = tl.t[i];
  const long long l = b - tl.lrow0[i];
  const bool r = T.flags & DPIPE_AUTOMAGIC_ROUND_BF16;
  const long long R = T.R;
  const float* row = T.row + l * R;
  double a = 0.0;
  for (long long k = threadIdx.x; k < R; k += AM_THREADS) a += row[k];
  a = block_sum<AM_THREADS>(a, red);
  const float rm = rnd(__double2float_rn(a / (double)R), r);
  if (threadIdx.x == 0) T.ws[AM_WS_HEAD + l] = rm;
  float* rf = T.ws + AM_WS_HEAD + T.L + l * R;
  for (long long k = threadIdx.x; k < R; k += AM_THREADS) rf[k] = rnd(rsqrt_rn(rnd(__fdiv_rn(row[k], rm), r)), r);
}

// per element: u (unclipped; 1-D / 0-D tensors update exp_avg_sq here) and new_lr; per CTA and tensor: partials
__global__ void __launch_bounds__(AM_THREADS) am_lr_kernel(const __grid_constant__ AmList tl, const AmScal s,
                                                          double* __restrict__ scratch) {
  __shared__ double red[AM_THREADS / 32];
  __shared__ float mx[AM_THREADS / 32];
  const long long tid = (long long)blockIdx.x * AM_THREADS + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * AM_THREADS;
  for (int i = 0; i < tl.n; ++i) {
    const dpipe_automagic_tensor& T = tl.t[i];
    const bool r = T.flags & DPIPE_AUTOMAGIC_ROUND_BF16;
    const float scale = (float)*T.scale;
    double sumsq = 0.0, lrsum = 0.0;
    float amax = 0.f;
    if (T.flags & DPIPE_AUTOMAGIC_FACTORED) {
      const float* rf = T.ws + AM_WS_HEAD + T.L;
      const float* cf = rf + T.L * T.R;
      const long long C = T.C;
      RowCol rc(tid, nthreads, C);
      for (long long j = tid; j < T.numel; j += nthreads, rc.next(C)) {
        const long long l = T.L == 1 ? 0 : rc.q / T.R;
        const float u = u_factored(rf[rc.q], cf[l * C + rc.c], ld_dt(T.g, j, T.dtype), r);
        sumsq += (double)u * (double)u;
        const float nl = new_lr(u, T.code[j], T.pol[j], scale, s);
        lrsum += nl;
        amax = fmaxf(amax, fabsf(nl));
      }
    } else {
      for (long long j = tid; j < T.numel; j += nthreads) {
        const float g = ld_dt(T.g, j, T.dtype);
        const float v = rnd(__fmaf_rn(__fadd_rn(__fmul_rn(g, g), s.eps), s.alpha, rnd(__fmul_rn(T.v[j], s.beta2), r)), r);
        T.v[j] = v;
        const float u = rnd(__fmul_rn(rnd(rsqrt_rn(v), r), g), r);           // exp_avg_sq.rsqrt().mul_(grad)
        sumsq += (double)u * (double)u;
        const float nl = new_lr(u, T.code[j], T.pol[j], scale, s);
        lrsum += nl;
        amax = fmaxf(amax, fabsf(nl));
      }
    }
    sumsq = block_sum<AM_THREADS>(sumsq, red);
    lrsum = block_sum<AM_THREADS>(lrsum, red);
    float w = amax;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) w = fmaxf(w, __shfl_xor_sync(0xffffffffu, w, off));
    if ((threadIdx.x & 31) == 0) mx[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x == 0) {
      float mm = 0.f;
      for (int k = 0; k < AM_THREADS / 32; ++k) mm = fmaxf(mm, mx[k]);
      double* out = scratch + tl.pp + ((long long)i * gridDim.x + blockIdx.x) * 3;
      out[0] = sumsq;
      out[1] = lrsum;
      out[2] = mm;
    }
    __syncthreads();
  }
}

// one CTA per tensor: folds the am_lr_kernel partials in a fixed order
__global__ void __launch_bounds__(AM_THREADS) am_finish_kernel(const __grid_constant__ AmList tl, const AmScal s,
                                                              const double* __restrict__ scratch, int grid) {
  __shared__ double red[AM_THREADS / 32];
  __shared__ float mx[AM_THREADS / 32];
  const int i = blockIdx.x;
  const dpipe_automagic_tensor& T = tl.t[i];
  const bool r = T.flags & DPIPE_AUTOMAGIC_ROUND_BF16;
  const double* part = scratch + tl.pp + (long long)i * grid * 3;
  double sumsq = 0.0, lrsum = 0.0;
  float amax = 0.f;
  for (int k = threadIdx.x; k < grid; k += AM_THREADS) {
    sumsq += part[3 * k];
    lrsum += part[3 * k + 1];
    amax = fmaxf(amax, (float)part[3 * k + 2]);
  }
  sumsq = block_sum<AM_THREADS>(sumsq, red);
  lrsum = block_sum<AM_THREADS>(lrsum, red);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if ((threadIdx.x & 31) == 0) mx[threadIdx.x >> 5] = amax;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int k = 0; k < AM_THREADS / 32; ++k) amax = fmaxf(amax, mx[k]);
  // _rms(update) = update.norm(2) / numel ** 0.5, then / clip_threshold, clamp_(min=1)
  const float norm = rnd(__double2float_rn(sqrt(sumsq)), r);
  const float rms = rnd(__fdiv_rn(norm, __double2float_rn(sqrt((double)T.numel))), r);
  const float clipdiv = fmaxf(rnd(__fdiv_rn(rms, s.clip), r), 1.0f);
  const float avg = __double2float_rn(lrsum / (double)T.numel);               // torch.mean(new_lr)
  const double old = *T.scale;
  T.ws[0] = clipdiv;
  T.ws[1] = amax;
  T.ws[2] = avg;
  T.ws[3] = (float)old;
  *T.avg_lr = avg;
  *T.scale = amax > 0.f ? (double)amax / 127.0 : 1.0;                         // Auto8bitTensor: absmax / 127
}

__global__ void __launch_bounds__(AM_THREADS) am_apply_kernel(const __grid_constant__ AmList tl, const AmScal s) {
  const long long tid = (long long)blockIdx.x * AM_THREADS + threadIdx.x;
  const long long nthreads = (long long)gridDim.x * AM_THREADS;
  for (int i = 0; i < tl.n; ++i) {
    const dpipe_automagic_tensor& T = tl.t[i];
    const bool r = T.flags & DPIPE_AUTOMAGIC_ROUND_BF16, fact = T.flags & DPIPE_AUTOMAGIC_FACTORED;
    const float clipdiv = T.ws[0], oscale = T.ws[3], nscale = (float)*T.scale;
    const float* rf = T.ws + AM_WS_HEAD + T.L;
    const float* cf = rf + T.L * T.R;
    const long long C = fact ? T.C : 1;
    RowCol rc(tid, nthreads, C);
    for (long long j = tid; j < T.numel; j += nthreads, rc.next(C)) {
      const float g = ld_dt(T.g, j, T.dtype);
      float u;
      if (fact) {
        const long long l = T.L == 1 ? 0 : rc.q / T.R;
        u = u_factored(rf[rc.q], cf[l * C + rc.c], g, r);
      } else {
        u = rnd(__fmul_rn(rnd(rsqrt_rn(T.v[j]), r), g), r);
      }
      u = rnd(__fdiv_rn(u, clipdiv), r);                                       // update.div_(clip divisor)
      const float nl = new_lr(u, T.code[j], T.pol[j], oscale, s);
      T.pol[j] = u > 0.f;
      const float qv = fminf(fmaxf(rintf(__fdiv_rn(nl, nscale)), -127.f), 127.f);
      T.code[j] = (signed char)(int)qv;
      u = rnd(__fmul_rn(u, nl), r);                                            // update.mul_(new_lr)
      if (T.dtype == 0) {
        const float p = ld_dt(T.p, j, 0);
        float upd = -u;
        if (s.has_wd) upd = rnd(__fadd_rn(upd, __fmul_rn(__fmul_rn(p, s.neg_wd), nl)), r);
        __nv_bfloat16* sh = reinterpret_cast<__nv_bfloat16*>(T.shift) + j;
        float shift = R<true>(__fadd_rn(__bfloat162float(*sh), upd));               // shift.add_(update)
        const float pn = R<true>(__fadd_rn(p, shift));                              // p.add_(shift)
        shift = R<true>(__fadd_rn(shift, __fsub_rn(p, pn)));                        // shift.add_(old - p)
        *sh = __float2bfloat16_rn(shift);
        reinterpret_cast<__nv_bfloat16*>(T.p)[j] = __float2bfloat16_rn(pn);
      } else {
        float* pp = reinterpret_cast<float*>(T.p) + j;
        float p = *pp;
        if (s.has_wd) p = __fadd_rn(p, __fmul_rn(__fmul_rn(p, s.neg_wd), nl));
        *pp = __fadd_rn(p, -u);
      }
    }
  }
}

int check_tensors(const char* fn, const dpipe_automagic_tensor* t, int n, const dpipe_automagic_scalars* s) {
  if (n < 0) return fail(DPIPE_EINVAL, "%s: n < 0", fn);
  if (n > 0 && !t) return fail(DPIPE_EINVAL, "%s: null argument", fn);
  for (int i = 0; i < n; ++i) {
    const dpipe_automagic_tensor& T = t[i];
    if (T.dtype != 0 && T.dtype != 1) return fail(DPIPE_EINVAL, "%s: tensor %d has dtype %d (0 = bf16, 1 = fp32)", fn, i, T.dtype);
    if (T.numel < 0) return fail(DPIPE_EINVAL, "%s: tensor %d has numel < 0", fn, i);
    if (T.flags & ~(DPIPE_AUTOMAGIC_FACTORED | DPIPE_AUTOMAGIC_ROUND_BF16))
      return fail(DPIPE_EINVAL, "%s: tensor %d has unknown flags %d", fn, i, T.flags);
    if ((T.flags & DPIPE_AUTOMAGIC_ROUND_BF16) && T.dtype != 0)
      return fail(DPIPE_EINVAL, "%s: tensor %d: bf16 rounding of the statistics is for bf16 weights only", fn, i);
    if (T.numel == 0) continue;
    if (!T.p || !T.g || !T.code || !T.pol || !T.scale || !T.avg_lr || !T.ws)
      return fail(DPIPE_EINVAL, "%s: tensor %d has a null pointer", fn, i);
    if ((T.dtype == 0) != (T.shift != nullptr))
      return fail(DPIPE_EINVAL, "%s: tensor %d: a bf16 tensor needs its Kahan shift, an fp32 tensor has none", fn, i);
    if (T.flags & DPIPE_AUTOMAGIC_FACTORED) {
      if (T.L < 1 || T.R < 1 || T.C < 1 || T.L * T.R * T.C != T.numel)
        return fail(DPIPE_EINVAL, "%s: tensor %d: L * R * C = %lld * %lld * %lld is not numel %lld", fn, i, (long long)T.L,
                    (long long)T.R, (long long)T.C, (long long)T.numel);
      if (!T.row || !T.col) return fail(DPIPE_EINVAL, "%s: tensor %d: factored tensor without row / col statistics", fn, i);
    } else if (!T.v) {
      return fail(DPIPE_EINVAL, "%s: tensor %d: unfactored tensor without exp_avg_sq", fn, i);
    }
  }
  if (n > 0 && s && !(s->clip_threshold > 0.0)) return fail(DPIPE_EINVAL, "%s: clip_threshold must be > 0", fn);
  return 0;
}

AmScal make_scalars(const dpipe_automagic_scalars* s) {
  AmScal a;
  a.beta2 = (float)s->beta2;
  a.alpha = (float)(1.0 - s->beta2);
  a.eps = (float)s->eps;
  a.bump = (float)s->lr_bump;
  a.min_lr = (float)s->min_lr;
  a.max_lr = (float)s->max_lr;
  a.clip = (float)s->clip_threshold;
  a.neg_wd = (float)(-s->weight_decay);
  a.has_wd = s->weight_decay != 0.0;
  return a;
}

int grid_blocks() { return 4 * num_sms(); }

// the next chunk of up to 64 non-empty tensors starting at *pos; fills the prefix sums and scratch offsets
void fill(AmList& tl, const dpipe_automagic_tensor* t, int n, int* pos, long long* scratch_need, int grid) {
  tl.n = 0;
  tl.tiles0[0] = tl.fold0[0] = tl.lrow0[0] = 0;
  long long off = 0;
  for (; *pos < n && tl.n < AM_MAX; ++*pos) {
    const dpipe_automagic_tensor& T = t[*pos];
    if (T.numel == 0) continue;
    const int k = tl.n++;
    tl.t[k] = T;
    long long tiles = 0, fold = 0, lrow = 0;
    tl.rp[k] = tl.cp[k] = off;
    if (T.flags & DPIPE_AUTOMAGIC_FACTORED) {
      const FmGeom f{T.L, T.R, T.C};
      tiles = f.tiles();
      fold = f.fold_ctas(AM_THREADS);
      lrow = T.L;
      tl.cp[k] = off + f.row_partials();
      off = tl.cp[k] + f.col_partials();
    }
    tl.tiles0[k + 1] = tl.tiles0[k] + tiles;
    tl.fold0[k + 1] = tl.fold0[k] + fold;
    tl.lrow0[k + 1] = tl.lrow0[k] + lrow;
  }
  tl.pp = off;
  *scratch_need = off + (long long)tl.n * grid * 3;
}

}  // namespace
}  // namespace dpipe

using namespace dpipe;

extern "C" int dpipe_automagic_scratch_doubles(const dpipe_automagic_tensor* t, int n, int64_t* out) {
  if (!out) return fail(DPIPE_EINVAL, "dpipe_automagic_scratch_doubles: null argument");
  if (int e = check_tensors("dpipe_automagic_scratch_doubles", t, n, nullptr)) return e;
  const int grid = grid_blocks();
  long long need = 0;
  int pos = 0;
  while (pos < n) {
    AmList tl;
    long long k = 0;
    fill(tl, t, n, &pos, &k, grid);
    need = k > need ? k : need;
  }
  *out = need;
  return 0;
}

extern "C" int dpipe_automagic_stats(const dpipe_automagic_tensor* t, int n, const dpipe_automagic_scalars* s,
                                     double* scratch, int64_t scratch_len, void* stream) {
  if (n > 0 && !s) return fail(DPIPE_EINVAL, "dpipe_automagic_stats: null scalars");
  if (int e = check_tensors("dpipe_automagic_stats", t, n, s)) return e;
  if (n == 0) return 0;
  const int grid = grid_blocks();
  long long need = 0;
  for (int pos = 0; pos < n;) {
    AmList tl;
    long long k = 0;
    fill(tl, t, n, &pos, &k, grid);
    need = k > need ? k : need;
  }
  if (!scratch || scratch_len < need)
    return fail(DPIPE_EINVAL, "dpipe_automagic_stats: scratch holds %lld doubles, needs %lld", (long long)scratch_len, need);
  const AmScal sc = make_scalars(s);
  cudaStream_t st = (cudaStream_t)stream;
  for (int pos = 0; pos < n;) {
    AmList tl;
    long long k = 0;
    fill(tl, t, n, &pos, &k, grid);
    if (tl.n == 0) continue;
    if (tl.tiles0[tl.n] > 0) {
      am_reduce_kernel<<<(unsigned)tl.tiles0[tl.n], AM_THREADS, 0, st>>>(tl, sc, scratch);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      am_fold_kernel<<<(unsigned)tl.fold0[tl.n], AM_THREADS, 0, st>>>(tl, sc, scratch);
      DPIPE_CUDA_CHECK(cudaGetLastError());
      am_rowmean_kernel<<<(unsigned)tl.lrow0[tl.n], AM_THREADS, 0, st>>>(tl);
      DPIPE_CUDA_CHECK(cudaGetLastError());
    }
    am_lr_kernel<<<grid, AM_THREADS, 0, st>>>(tl, sc, scratch);
    DPIPE_CUDA_CHECK(cudaGetLastError());
    am_finish_kernel<<<tl.n, AM_THREADS, 0, st>>>(tl, sc, scratch, grid);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}

extern "C" int dpipe_automagic_apply(const dpipe_automagic_tensor* t, int n, const dpipe_automagic_scalars* s, void* stream) {
  if (n > 0 && !s) return fail(DPIPE_EINVAL, "dpipe_automagic_apply: null scalars");
  if (int e = check_tensors("dpipe_automagic_apply", t, n, s)) return e;
  if (n == 0) return 0;
  const int grid = grid_blocks();
  const AmScal sc = make_scalars(s);
  for (int pos = 0; pos < n;) {
    AmList tl;
    long long k = 0;
    fill(tl, t, n, &pos, &k, grid);
    if (tl.n == 0) continue;
    am_apply_kernel<<<grid, AM_THREADS, 0, (cudaStream_t)stream>>>(tl, sc);
    DPIPE_CUDA_CHECK(cudaGetLastError());
  }
  return 0;
}
