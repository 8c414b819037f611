/*
 * dpipe.h — C ABI of libdpipe_b200.so: the sm_90a kernels and the 1F1B stage executor behind the
 * reference's Flux training hot path.
 *
 * The reference (tdrussell/diffusion-pipe) has no native code and no FFI of its own: every entry
 * point here replaces a *library call site* of the reference, cited per function as
 * "replaces: <reference file:line>" (paths relative to the reference repo root).
 *
 * Conventions
 *   - every function returns 0 on success or a negative DPIPE_E* code; dpipe_last_error() gives a
 *     thread-local human readable message.  Nothing throws across this boundary.
 *   - the caller owns all memory; pointers are raw CUDA device pointers unless a parameter says
 *     "host".  bf16 tensors are row-major with explicit leading dimensions in ELEMENTS.
 *   - all kernels are enqueued asynchronously on `stream` (a cudaStream_t passed as void*).
 *   - no hidden allocation: scratch space is passed in by the caller where needed.
 */
#ifndef DPIPE_H_
#define DPIPE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DPIPE_OK 0
#define DPIPE_EINVAL (-1)   /* bad argument (shape/alignment/enum) */
#define DPIPE_ECUDA (-2)    /* a CUDA runtime/driver call failed */
#define DPIPE_ENOTSUP (-3)  /* device is not sm_90 / feature not compiled */
#define DPIPE_ESTATE (-4)   /* executor used out of order */

const char* dpipe_last_error(void);
/* returns the ABI version (bumped on any signature change) */
int dpipe_abi_version(void);
/* 0 if device `dev` is an sm_90 part this library can run on */
int dpipe_check_device(int dev);

/* ------------------------------------------------------------------------------------------ */
/* Dense bf16 GEMM on wgmma tensor cores (TMA -> smem -> wgmma -> registers -> epilogue).      */
/*   D[M,N] (fp32 accumulators) = Aop[M,K] * Bop[N,K]^T, then a fused epilogue.                  */
/* replaces: cuBLASLt via nn.Linear inside the diffusers blocks invoked from                     */
/*           models/flux.py:502,525 (forward) and their autograd backward (dgrad/wgrad).         */
/* ------------------------------------------------------------------------------------------ */
enum {
  DPIPE_EPI_STORE = 0,     /* out = acc (+bias) (+out if accumulate)                                   */
  DPIPE_EPI_BIAS_GELU = 1, /* u = bf16(acc+bias); out2 = u (optional); out = gelu_tanh(u)               */
  DPIPE_EPI_GATE_RES = 2,  /* y = bf16(acc+bias); out2 = y (optional); out = aux + gate[b,:]*y          */
  DPIPE_EPI_QKV_ROPE = 3,  /* cols < n_qkv: bias -> per-head RMSNorm(q,k) -> RoPE -> head-major scatter; */
                           /* cols >= n_qkv: BIAS_GELU into (out,out2)                                  */
  DPIPE_EPI_MUL_GELU_GRAD = 4 /* out = acc * gelu_tanh'(aux)   (dgrad through GELU)                      */
};

typedef struct dpipe_qkv_epilogue {
  void* q;            /* bf16 [batch, heads, seq_total, 128]  (post norm + rope) */
  void* k;            /* bf16 same layout */
  void* v;            /* bf16 same layout (bias only) */
  void* qhat;         /* bf16 same layout: x * rstd before the norm weight (saved for backward), may be NULL */
  void* khat;         /* bf16 same layout, may be NULL */
  float* q_rstd;      /* fp32 [batch, heads, seq_total], may be NULL */
  float* k_rstd;      /* fp32 [batch, heads, seq_total], may be NULL */
  const void* q_norm_w; /* bf16 [128] */
  const void* k_norm_w; /* bf16 [128] */
  const float* rope_cos; /* fp32 [seq_total, 128] (interleaved-repeat layout of diffusers FluxPosEmbed) */
  const float* rope_sin; /* fp32 [seq_total, 128] */
  int heads;          /* H; the q, k, v column blocks are H*128 wide each */
  int seq_total;      /* joint sequence length (text + image) */
  int seq_offset;     /* position of this stream's first token in the joint sequence */
  int n_qkv;          /* 3*H*128; columns beyond it take the BIAS_GELU path */
  float eps;          /* RMSNorm epsilon (1e-6 in Flux) */
} dpipe_qkv_epilogue;

typedef struct dpipe_gemm_args {
  const void* A; int64_t lda; int a_mn; /* a_mn=0: A stored [M,K] (K contiguous); 1: stored [K,M] */
  const void* B; int64_t ldb; int b_mn; /* b_mn=0: B stored [N,K] (K contiguous); 1: stored [K,N] */
  int M, N, K;
  int epilogue;                 /* DPIPE_EPI_* */
  void* out; int64_t ldo;       /* bf16 [M, >=N] */
  void* out2; int64_t ldo2;     /* bf16, optional second output (see epilogue) */
  const void* bias;             /* bf16 [N] or NULL */
  const void* aux; int64_t ldaux;   /* bf16 [M,N] epilogue input (residual / pre-activation) */
  const void* gate; int64_t gate_stride; /* bf16 [batch, gate_stride], column n of batch b at gate[b*gate_stride+n] */
  int rows_per_batch;           /* rows of A that belong to one sample (for gate / qkv batch index) */
  int accumulate;               /* STORE only: out = bf16(float(out) + acc) */
  int cta_group;                /* 1 or 2; accepted for ABI compatibility: sm_90a runs one CTA per 128x256 tile either way */
  const dpipe_qkv_epilogue* qkv; /* required for DPIPE_EPI_QKV_ROPE */
} dpipe_gemm_args;

/* Alignment (refused with DPIPE_EINVAL before any launch): A and B are TMA operands, 16-byte aligned with lda / ldb
 * multiples of 8.  The epilogue accesses 16 bytes at a time, so out, bias and every out2 / aux / gate the epilogue uses
 * are 16-byte aligned and ldo / ldo2 / ldaux / gate_stride multiples of 8; so are qkv->q, k, v, qhat, khat, q_norm_w,
 * k_norm_w, rope_cos and rope_sin, while q_rstd / k_rstd need 4 bytes. */
int dpipe_gemm_bf16(const dpipe_gemm_args* args, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* Fused attention (FlashAttention-style, head_dim 128, non-causal) on wgmma + TMA.           */
/* replaces: torch SDPA dispatched by the diffusers Flux attention processor invoked from        */
/*           models/flux.py:502,525; flash_attn_varlen_func at models/wan/attention.py:108-122.  */
/* ------------------------------------------------------------------------------------------ */
typedef struct dpipe_attn_args {
  const void* q;   /* bf16 [batch, heads, seq_q, 128] contiguous */
  const void* k;   /* bf16 [batch, heads, seq_k, 128] */
  const void* v;   /* bf16 [batch, heads, seq_k, 128] */
  void* o;         /* bf16 token-major [batch*seq_q, ldo]; head h occupies columns [128h, 128h+128) */
  int64_t ldo;
  float* lse;      /* fp32 [batch, heads, seq_q]: log2-domain logsumexp = max*scale*log2(e) + log2(sum); may be NULL (fwd) */
  int batch, heads, seq_q, seq_k;
  float scale;     /* softmax scale, 1/sqrt(128) for Flux */
} dpipe_attn_args;

int dpipe_attn_fwd(const dpipe_attn_args* args, void* stream);

typedef struct dpipe_attn_bwd_args {
  const void* q;   /* bf16 [batch, heads, seq_q, 128] (as given to the forward) */
  const void* k;   /* bf16 [batch, heads, seq_k, 128] */
  const void* v;   /* bf16 [batch, heads, seq_k, 128] */
  const void* o;   /* bf16 token-major forward output [batch*seq_q, ldo] */
  int64_t ldo;
  const void* d_o; /* bf16 token-major gradient of o [batch*seq_q, lddo] */
  int64_t lddo;
  const float* lse; /* fp32 [batch, heads, seq_q] from dpipe_attn_fwd (log2 domain) */
  float* delta;     /* fp32 [batch, heads, seq_q] scratch: rowsum(o * d_o), written by this call */
  void* dq;        /* bf16 [batch, heads, seq_q, 128] */
  void* dk;        /* bf16 [batch, heads, seq_k, 128] */
  void* dv;        /* bf16 [batch, heads, seq_k, 128] */
  int batch, heads, seq_q, seq_k;
  float scale;
} dpipe_attn_bwd_args;

/* Alignment (refused with DPIPE_EINVAL before any launch): q, k, v and d_o are TMA operands, 16-byte aligned; ldo and
 * lddo multiples of 8.  The forward writes o in 4-byte pairs and lse as fp32: both 4-byte aligned.  The backward reads
 * o and d_o 8 bytes at a time (8-byte aligned) and writes dq / dk / dv in 4-byte pairs and lse / delta as fp32 (4-byte
 * aligned). */
/* backward of dpipe_attn_fwd; replaces flash-attn / SDPA backward reached via autograd from models/flux.py:502,525 */
int dpipe_attn_bwd(const dpipe_attn_bwd_args* args, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* HBM-bound kernels around the GEMMs (LayerNorm+modulation, gated residual, q/k norm + RoPE     */
/* backward, bias-gradient column sums, masked MSE loss).                                        */
/* replaces: the unfused ATen kernels behind diffusers AdaLayerNormZero{,Single}/Continuous,     */
/*           gate*out + residual, RMSNorm(q,k), apply_rotary_emb (call sites models/flux.py:     */
/*           502,525,546-548) and F.mse_loss in models/base.py:418-436.                          */
/* Row reductions are two-stage and atomics-free: kernels taking `partials` write                */
/* partials[batch][nchunk][2][D] fp32 with nchunk = ceil(rows_per_batch / dpipe_row_chunk());    */
/* dpipe_colreduce_finish folds them.  D must be a multiple of 256.                              */
/* ------------------------------------------------------------------------------------------ */
int dpipe_row_chunk(void);

/* out = LayerNorm(x, eps, no affine) * bf16(1 + scale[b]) + shift[b]; saves mean/rstd (fp32 [batch*rows]) */
int dpipe_ln_modulate_fwd(const void* x, int64_t ldx, const void* scale, const void* shift, int64_t mod_stride,
                          void* out, int64_t ldo, float* mean, float* rstd, int batch, int rows_per_batch, int D,
                          float eps, void* stream);
/* flags for the _ex forms below */
#define DPIPE_LN_MULT_DIRECT 1 /* `scale` is the multiplier itself (LayerNorm with affine weight: Wan norm3, models/wan/model.py:266-268) */
#define DPIPE_LN_ROUND_STEPS 2 /* round x_hat and x_hat*mult to bf16 before the next op: Wan's `norm(x) * (1 + e1) + e0` on bf16 tensors (models/wan/model.py:301-302) */
int dpipe_ln_modulate_fwd_ex(const void* x, int64_t ldx, const void* scale, const void* shift, int64_t mod_stride,
                             void* out, int64_t ldo, float* mean, float* rstd, int batch, int rows_per_batch, int D,
                             float eps, int flags, void* stream);
int dpipe_ln_modulate_bwd_ex(const void* dxn, int64_t lddxn, const void* x, int64_t ldx, const void* scale,
                             int64_t mod_stride, const float* mean, const float* rstd, const void* dres, int64_t lddres,
                             void* dx, int64_t lddx, float* partials, int batch, int rows_per_batch, int D, int flags,
                             void* stream);
/* dx = LN'(dxn * bf16(1+scale)) (+ dres);  partial slot 0 = d scale, slot 1 = d shift (per sample) */
int dpipe_ln_modulate_bwd(const void* dxn, int64_t lddxn, const void* x, int64_t ldx, const void* scale,
                          int64_t mod_stride, const float* mean, const float* rstd, const void* dres, int64_t lddres,
                          void* dx, int64_t lddx, float* partials, int batch, int rows_per_batch, int D, void* stream);
/* x_new = res + gate[b]*y:  dy = bf16(gate*dx);  partial slot 0 = sum dx*y (d gate, per sample), slot 1 = sum dy (d bias) */
int dpipe_gate_bwd(const void* dx, int64_t lddx, const void* y, int64_t ldy, const void* gate, int64_t gate_stride,
                   void* dy, int64_t lddy, float* partials, int batch, int rows_per_batch, int D, void* stream);
/* slot s of partials -> per_sample{s}[b*ld{s} + d] and/or summed{s}[d] (sum over samples); NULL outputs are skipped */
int dpipe_colreduce_finish(const float* partials, int batch, int nchunk, int nslot, int D, float* per_sample0,
                           int64_t ld0, float* per_sample1, int64_t ld1, float* summed0, float* summed1, void* stream);
/* out[n] = sum_rows x[r,n] (bias gradients); partials needs dpipe_colsum_chunks(rows)*N floats */
int dpipe_colsum_chunks(int rows);
int dpipe_colsum(const void* x, int64_t ldx, int rows, int N, float* partials, float* out, void* stream);

typedef struct dpipe_qk_bwd_args {
  const void* dq; const void* dk; const void* dv;  /* bf16 [batch, heads, seq_total, 128] from dpipe_attn_bwd */
  const void* qhat; const void* khat;              /* bf16, saved by the QKV_ROPE epilogue */
  const float* q_rstd; const float* k_rstd;        /* fp32 [batch, heads, seq_total] */
  const void* q_norm_w; const void* k_norm_w;      /* bf16 [128] */
  const float* rope_cos; const float* rope_sin;    /* fp32 [seq_total, 128] */
  void* dqkv; int64_t ld;                          /* bf16 token-major [batch*rows_per_batch, >= 3*heads*128] */
  float* dbias;                                    /* fp32 [3*heads*128]: += column sums of dqkv (caller zeroes) */
  float* dw;                                       /* fp32 [2][128]: += d q_norm_w, d k_norm_w (caller zeroes) */
  int batch, heads, seq_total, seq_offset, rows_per_batch;
} dpipe_qk_bwd_args;
/* backward of the DPIPE_EPI_QKV_ROPE epilogue for one stream */
int dpipe_qknorm_rope_bwd(const dpipe_qk_bwd_args* args, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* Wan attention pre-processing (csrc/wan_norm.cu): RMSNorm over the full model width + RoPE +  */
/* token-major -> head-major scatter.  Replaces WanRMSNorm / rope_apply / the .view(b, s, n, d) */
/* of models/wan/model.py:41-68,71-87,137-156,171-183.  Up to three projections per launch.    */
/* ------------------------------------------------------------------------------------------ */
typedef struct dpipe_wan_norm_proj {
  const void* src; int64_t ld;   /* bf16 [batch*seq, ld]: projection output (bias added), width heads*128 used */
  const void* weight;            /* bf16 [heads*128] RMSNorm scale, or NULL: no normalisation (v) */
  void* dst;                     /* bf16 [batch, heads, seq, 128] */
  void* xhat;                    /* bf16 [batch*seq, heads*128]: normalised rows before the scale (for backward), or NULL */
  float* rstd;                   /* fp32 [batch*seq], or NULL */
  int rope;                      /* rotate with the tables below */
} dpipe_wan_norm_proj;
typedef struct dpipe_wan_norm_fwd_args {
  dpipe_wan_norm_proj proj[3];
  int nproj;
  const float* cos; const float* sin;   /* fp32 [seq, 128], every frequency repeated twice (NULL if no projection ropes) */
  int batch, seq, heads;
  float eps;
} dpipe_wan_norm_fwd_args;
int dpipe_wan_norm_rope_fwd(const dpipe_wan_norm_fwd_args* args, void* stream);

typedef struct dpipe_wan_norm_bwd_proj {
  const void* dy;                /* bf16 [batch, heads, seq, 128]: gradient of dst */
  const void* xhat; const float* rstd; const void* weight;   /* as saved / passed in the forward (NULL for v) */
  void* dx; int64_t ld;          /* bf16 [batch*seq, ld]: gradient of src */
  float* dw_partials;            /* fp32 [ceil(batch*seq / dpipe_wan_norm_rows()), heads*128]; fold with dpipe_colreduce_finish */
  int rope;
} dpipe_wan_norm_bwd_proj;
typedef struct dpipe_wan_norm_bwd_args {
  dpipe_wan_norm_bwd_proj proj[3];
  int nproj;
  const float* cos; const float* sin;
  int batch, seq, heads;
} dpipe_wan_norm_bwd_args;
int dpipe_wan_norm_rows(void);
int dpipe_wan_norm_rope_bwd(const dpipe_wan_norm_bwd_args* args, void* stream);

/* AdaLayerNorm modulation linear for a micro-batch of B <= 8 samples (HBM-bound, rank-B):
 *   out[b,:] = W * bf16(silu(temb[b,:])) + bias.   replaces nn.Linear(SiLU(temb)) of AdaLayerNormZero{,Single}/Continuous
 *   (models/flux.py:502,525,547). */
int dpipe_mod_fwd(const void* temb, const void* W, const void* bias, void* out, int B, int N, int K, void* stream);
/* its backward in one pass over W/dW: dW (+)= bf16(dmod)^T silu(temb); dbias[n] = sum_b dmod[b,n] (overwritten);
 * dtemb[b,:] += silu'(temb) * bf16(bf16(dmod) W).  partials: dpipe_mod_bwd_chunks(N) * B * K floats.  dW and dbias may be
 * NULL.  1 <= B <= 8 and K a multiple of 256 up to 8192, every B at every such K (fixed-size CTAs over 64-row chunks x
 * 1024-column blocks). */
int dpipe_mod_bwd_chunks(int N);
int dpipe_mod_bwd(const float* dmod, int64_t ldd, const void* temb, const void* W, void* dW, int accumulate, float* dbias,
                  float* partials, float* dtemb, int B, int N, int K, void* stream);

/* loss = mean((out - target)^2 * mask); dout (bf16, optional) = 2 (out-target) mask / numel.  workspace: 1024 floats */
int dpipe_mse_loss(const void* out, const float* target, const float* mask, int64_t numel, float* workspace,
                   float* loss, void* dout, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* Optimizer-step tail and micro-batch preparation (HBM-bound).                                   */
/* ------------------------------------------------------------------------------------------ */
/* out[0] (device fp32) = sum over the n tensors of sum(g^2), fp32 accumulation per thread, per-CTA partials folded in
 * double in a fixed order.  dtypes[i]: 0 = bf16, 1 = fp32; every tensor contiguous.  partials: at least
 * dpipe_grad_sumsq_blocks() * ceil(n / 64) floats.
 * replaces: the per-parameter `p.grad.data.float().norm(2)` loop of clip_grad_norm_ (utils/patches.py:204-224). */
int dpipe_grad_sumsq_blocks(void);
int dpipe_grad_sumsq(const void* const* ptrs, const int64_t* numels, const int* dtypes, int n, float* partials,
                     int64_t partials_len, float* out, void* stream);
/* g *= *coef (device fp32 scalar) for the same tensor lists; returns without touching memory when *coef >= 1.
 * replaces: `p.grad.data.mul_(clip_coef)` (utils/patches.py:238-243). */
int dpipe_grad_scale(const void* const* ptrs, const int64_t* numels, const int* dtypes, int n, const float* coef,
                     void* stream);
/* One AdamW step with optimi's update rule over n tensor sets (p, g, m, v, c) of numels[i] elements each, all five of
 * dtypes[i] (0 = bf16, 1 = fp32), contiguous, at any element offset.  kahan_comps (the array, or any entry) may be NULL:
 * no Kahan compensation for that tensor; a non-NULL c needs bf16.  With t the step count, on the host in double and
 * rounded to fp32: debias(b, t) = (b^t - b) / (b^t - 1), beta1_comp = 1 - debias(beta1, t), beta2_hat = debias(beta2, t),
 * one_minus_beta2_hat = 1 - beta2_hat, decay = 1 - lr * weight_decay (fully decoupled: 1 - lr / max_lr * weight_decay).
 *   p *= decay;  m = lerp(m, g, beta1_comp);  v = v * beta2_hat + one_minus_beta2_hat * g * g;
 *   u = -lr * m / (sqrt(v) + eps);  with c: c += u; old = p; p += c; c += old - p   without: p += u
 * Each operation is IEEE round-to-nearest fp32 in this order (no FMA), rounded to bf16 where a bf16 torch op rounds;
 * elementwise, so bitwise repeatable.  Up to 64 tensors per launch.
 * replaces: optimi.AdamW (Kahan summation for bf16 weights) built for `type = 'adamw_optimi'` (train.py:676-678). */
int dpipe_adamw_step(void* const* params, const void* const* grads, void* const* exp_avgs, void* const* exp_avg_sqs,
                     void* const* kahan_comps, const int64_t* numels, const int* dtypes, int n, float lr, float beta1_comp,
                     float beta2_hat, float one_minus_beta2_hat, float eps, float decay, void* stream);
/* One parameter of an Automagic step (the reference's optimizers/automagic.py).  All tensors contiguous, at any element
 * offset.  p / g / shift: dtype (0 = bf16, 1 = fp32), numel elements; shift (Kahan) for bf16 weights only, NULL for fp32.
 * flags & DPIPE_AUTOMAGIC_FACTORED (ndim >= 2): shape = [L (= prod(shape[:-2]), 1 for 2-D), R, C], row = exp_avg_sq_row
 * [L*R] and col = exp_avg_sq_col [L*C] fp32; otherwise v = exp_avg_sq [numel] fp32.  flags & DPIPE_AUTOMAGIC_ROUND_BF16:
 * step 1 of a bf16 parameter, where the reference's statistics are bf16 tensors: every op on them and on u rounds to bf16.
 * code: int8 lr codes, pol: last polarity (bool bytes), scale: the codes' scale (fp64 scalar), avg_lr: fp32 scalar.
 * ws (fp32, per tensor, written by dpipe_automagic_stats, read by dpipe_automagic_apply):
 *   ws[0] clip divisor max(rms(u) / clip_threshold, 1)   ws[1] max |new_lr|   ws[2] avg_lr   ws[3] fp32(previous scale)
 *   factored only: ws[4 .. 4+L) row.mean(-1), then L*R row factors rsqrt(row / row.mean(-1)), then L*C column factors
 *   rsqrt(col): 4 + L + L*R + L*C floats; unfactored: 4 floats. */
#define DPIPE_AUTOMAGIC_FACTORED 1
#define DPIPE_AUTOMAGIC_ROUND_BF16 2
typedef struct dpipe_automagic_tensor {
    void* p;
    const void* g;
    float* row;
    float* col;
    float* v;
    signed char* code;
    unsigned char* pol;
    void* shift;
    double* scale;
    float* avg_lr;
    float* ws;
    int64_t numel, L, R, C;
    int dtype;
    int flags;
} dpipe_automagic_tensor;
/* the group's hyper-parameters, as the Python floats the reference passes; the kernels use their fp32 roundings
 * (alpha = fp32(1 - beta2), -weight_decay), and eps is eps[0] of the reference's tuple */
typedef struct dpipe_automagic_scalars {
    double beta2, eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay;
} dpipe_automagic_scalars;
/* doubles of fp64 scratch dpipe_automagic_stats needs for these tensors (row / column partials and per-CTA sums of
 * the largest chunk of 64) */
int dpipe_automagic_scratch_doubles(const dpipe_automagic_tensor* t, int n, int64_t* out);
/* Automagic statistics phase over n parameters, up to 64 per launch group (5 launches per group, none per tensor):
 *   u0 = g*g + eps;  factored: row = EMA_beta2(u0.mean(-1)), col = EMA_beta2(u0.mean(-2)),
 *                    u = (rsqrt(row / row.mean(-1)) * rsqrt(col)) * g;   unfactored: v = EMA_beta2(u0), u = rsqrt(v) * g
 *   (EMA: x = x * beta2 + (1 - beta2) * mean, torch's fused add with alpha)
 *   new_lr = clamp(q * scale +- lr_bump, min_lr, max_lr), + where (u > 0) == last polarity
 *   clip divisor = max(fp32(sqrt(sum u^2)) / fp32(sqrt(numel)) / clip_threshold, 1); avg_lr = mean(new_lr);
 *   scale = max|new_lr| / 127 (fp64; 1 when 0).  Row means, factors and the per-tensor scalars go to ws (above).
 * Reductions accumulate in fp64 in a fixed order (bitwise repeatable), no float atomics, no host synchronisation.
 * replaces: the statistics half of Automagic.step (optimizers/automagic.py:240-300, optimizer_utils.py:222-232). */
int dpipe_automagic_stats(const dpipe_automagic_tensor* t, int n, const dpipe_automagic_scalars* s, double* scratch,
                          int64_t scratch_len, void* stream);
/* Automagic apply phase, one launch per group of 64, after dpipe_automagic_stats on the same tensors: u as above,
 * u /= clip divisor, new polarity, codes = clamp(round(new_lr / fp32(scale)), -127, 127), u *= new_lr, then
 *   bf16: upd = -u + p * (-weight_decay) * new_lr; shift += upd; old = p; p += shift; shift += old - p
 *   fp32: p += p * (-weight_decay) * new_lr; p -= u            (the weight-decay term only when weight_decay != 0)
 * Each operation is IEEE round-to-nearest fp32 in the reference's op order (no FMA), rounded to bf16 where a bf16
 * torch op rounds: bit-identical to oracle/automagic_ref.py automagic_apply_emulated.
 * replaces: the update half of Automagic.step (optimizers/automagic.py:300-344). */
int dpipe_automagic_apply(const dpipe_automagic_tensor* t, int n, const dpipe_automagic_scalars* s, void* stream);
/* One parameter of a Prodigy step (pytorch_optimizer.Prodigy, built for `type = 'Prodigy'`).  p, g and the state s, p0,
 * m = exp_avg, v = exp_avg_sq: numel elements each of dtype (0 = bf16, 1 = fp32), contiguous, at any element offset
 * (16-byte vectors when all six share their offset mod 16 B).  weight_decay (decoupled), fixed_decay and eps are the
 * parameter's group's. */
typedef struct dpipe_prodigy_tensor {
    void* p;
    const void* g;
    const void* p0;
    void* s;
    void* m;
    void* v;
    int64_t numel;
    double weight_decay;
    double eps;
    int dtype;
    int fixed_decay;
} dpipe_prodigy_tensor;
/* group 0's hyper-parameters, as the Python floats the reference passes (beta3: sqrt(beta2) when it is None) */
typedef struct dpipe_prodigy_scalars {
    double lr, beta1, beta2, beta3, d0, d_coef, growth_rate;
    int bias_correction, safeguard_warmup;
} dpipe_prodigy_scalars;
/* the optimizer's device scalar block (fp64), shared by all its param groups, read and written only by the kernels */
#define DPIPE_PRODIGY_D 0
#define DPIPE_PRODIGY_D_MAX 1
#define DPIPE_PRODIGY_D_HAT 2
#define DPIPE_PRODIGY_D_NUMERATOR 3
#define DPIPE_PRODIGY_D_DENOM 4
#define DPIPE_PRODIGY_STEP 5
#define DPIPE_PRODIGY_D_LR 6 /* d * lr / bias_correction of the last statistics phase (its old d) */
#define DPIPE_PRODIGY_SKIP 7 /* 1 when the last statistics phase found d_denom == 0 */
#define DPIPE_PRODIGY_STATE_DOUBLES 8
/* doubles of fp64 scratch dpipe_prodigy_stats needs: 2 * n per-tensor sums, then the per-CTA partials of the largest
 * chunk of 64 */
int dpipe_prodigy_scratch_doubles(const dpipe_prodigy_tensor* t, int n, int64_t* out);
/* Prodigy statistics phase over the n parameters of ALL param groups in group order, 64 per launch (2 launches per 64,
 * then 1), no host synchronisation.  From the device block (old d, step) and the host scalars, in double:
 *   t = step + 1, bc = (1 - beta1^t) / sqrt(1 - beta2^t) (powers by squaring; 1 without bias_correction),
 *   d_lr = d * lr / bc, k = (d / d0) * d_lr; per element in fp32 (coefficients rounded to fp32):
 *   m = fma(g, d * (1 - beta1), m * beta1);  v = fma(d * d * (1 - beta2), g * g, v * beta2);
 *   s = fma(g, (d / d0) * (safeguard_warmup ? d : d_lr), s * beta3)      (rounded to bf16 after each op for bf16)
 *   per tensor in fp64: dot_i = sum g * (p0 - p), abs_i = sum |s| (per-CTA partials, fixed-order folds: bitwise
 *   repeatable, no float atomics), written to scratch[2i], scratch[2i + 1];
 *   then one CTA, in tensor order: d_numerator = beta3 * d_numerator + k * dot_0 + k * dot_1 ..., d_denom = sum abs_i;
 *   d_denom == 0: SKIP = 1 (d, d_max, d_hat and step unchanged); otherwise d_hat = d_coef * d_numerator / d_denom,
 *   d = max(d, d_hat) if d == d0, d_max = max(d_max, d_hat), d = min(d_max, d * growth_rate), step = t, SKIP = 0.
 * Empty tensors are skipped (their sums are 0).  Bit-identical to oracle/prodigy_ref.py prodigy_stats_emulated /
 * prodigy_fold, whose elementwise order is that of torch's CUDA kernels.
 * replaces: the first loop of Prodigy.step and its d_denom / d_hat host syncs (train.py:698-700). */
int dpipe_prodigy_stats(const dpipe_prodigy_tensor* t, int n, const dpipe_prodigy_scalars* s, double* state,
                        double* scratch, int64_t scratch_len, void* stream);
/* Prodigy apply phase after dpipe_prodigy_stats (any subset of its tensors), one launch per 64; returns at once on
 * the device when SKIP is set.  With the old d_lr and the new d from the block, per element in fp32:
 *   denom = sqrt(v) + d * eps;  p = p * (1 - weight_decay * (fixed_decay ? 1 : d_lr));  p = fma(-d_lr, m / denom, p)
 * (rounded to bf16 after each op for bf16).  Bit-identical to oracle/prodigy_ref.py prodigy_apply_emulated.
 * replaces: the second loop of Prodigy.step (train.py:698-700). */
int dpipe_prodigy_apply(const dpipe_prodigy_tensor* t, int n, const double* state, void* stream);
/* One parameter of an AdamW8bit step (bitsandbytes.optim.AdamW8bit, built for `type = 'adamw8bit'`).  p, g: numel
 * elements of dtype (0 = bf16, 1 = fp32), contiguous, at any element offset (16-byte vectors where aligned).
 * absmax1 == absmax2 == NULL: state1 = m, state2 = v are fp32 [numel] (bnb's 32-bit path, numel < min_8bit_size);
 * otherwise state1 / state2 are uint8 codes [numel] of the signed / unsigned dynamic map and absmax1 / absmax2 fp32
 * [ceil(numel / 256)].  The scalars of the parameter's step t and group, in double on the host, rounded to fp32:
 * step_size = -lr * sqrt(1 - beta2^t) / (1 - beta1^t), eps_c2 = fp32(sqrt(1 - beta2^t)) * eps,
 * decay = 1 - lr * weight_decay (fp32 ops). */
typedef struct dpipe_adamw8bit_tensor {
    void* p;
    const void* g;
    void* state1;
    void* state2;
    float* absmax1;
    float* absmax2;
    int64_t numel;
    float step_size;
    float beta1;
    float beta2;
    float eps_c2;
    float decay;
    int dtype;
} dpipe_adamw8bit_tensor;
/* One AdamW8bit step over n parameters, up to 64 non-empty ones per launch (one warp per 256-element block), no host
 * synchronisation.  qmap1 / qmap2: the 256 sorted fp32 entries of the signed / unsigned map (may be NULL when no
 * tensor has 8-bit states).  Per element, fp32 IEEE round-to-nearest ops in this order (no FMA):
 *   8-bit: m = qmap1[state1] * absmax1[blk], v = qmap2[state2] * absmax2[blk]  (a non-finite g: m = v = 0, p kept)
 *   m = m * beta1 + (1 - beta1) * g;  v = v * beta2 + ((1 - beta2) * g) * g
 *   p = p + step_size * (m / (sqrt(v) + eps_c2));  p = p * decay        (each rounded to bf16 for bf16)
 *   8-bit: absmax1[blk] = max |m|, absmax2[blk] = max v (warp max: order-free);  state1 = the nearest qmap1 entry to
 *   m / absmax1 (counted in fp32 midpoints (q[k] + q[k+1]) * 0.5, ties down; 0 when absmax1 == 0), moved one code
 *   towards m's sign when the entry's sign bit differs from m's;  state2 = the nearest qmap2 entry to v / absmax2.
 * Bit-identical to oracle/adamw8bit_ref.py adamw8bit_emulated.
 * replaces: bitsandbytes.optim.AdamW8bit.step (train.py:650-700). */
int dpipe_adamw8bit_step(const dpipe_adamw8bit_tensor* t, int n, const float* qmap1, const float* qmap2, void* stream);
/* One parameter of a CAME step (pytorch_optimizer.CAME, built for `type = 'CAME'`).  p, g and the state m = exp_avg:
 * numel elements of dtype (0 = bf16, 1 = fp32), contiguous, at any element offset.  factored != 0 (ndim >= 2): shape
 * [L = prod(shape[:-2]), R, C]; row / res_row = exp_avg_sq_row / exp_avg_res_row [L*R], col / res_col =
 * exp_avg_sq_col / exp_avg_res_col [L*C], all of dtype; otherwise v = exp_avg_sq [numel] of dtype.  The group's
 * hyper-parameters as the Python floats the reference passes (the kernels use their fp32 roundings).
 * fac (fp32) and sums (fp64), per tensor, written by the step:
 *   fac  = [clip divisor]  factored: then r_sq [L*R], c_sq [L*C], r_res [L*R], c_res [L*C]   (1 + 2 (L*R + L*C))
 *   sums = [sum u^2]       factored: then for sq, then for res: row sums [L*R], column sums [L*C], sums over R of
 *          the new row statistics [L]                                                          (1 + 2 (L*R + L*C + L)) */
typedef struct dpipe_came_tensor {
    void* p;
    const void* g;
    void* m;
    void* row;
    void* col;
    void* res_row;
    void* res_col;
    void* v;
    float* fac;
    double* sums;
    int64_t numel, L, R, C;
    double lr, weight_decay, beta1, beta2, beta3, eps1, eps2;
    int dtype;
    int factored;
    int fixed_decay;
} dpipe_came_tensor;
/* doubles of fp64 scratch dpipe_came_step needs for these tensors (row / column partials and per-CTA sums of u^2 of
 * the largest chunk of 64) */
int dpipe_came_scratch_doubles(const dpipe_came_tensor* t, int n, int64_t* out);
/* One CAME step over n parameters, up to 64 non-empty ones per launch group (10 launches per group with a factored
 * tensor, 3 without), no host synchronisation.  Per tensor, in fp32 ops rounded to the dtype after each op:
 *   u0 = g*g + eps1;  factored: row = fma(mean_C(u0), 1 - beta2, row * beta2), col likewise over R,
 *                     u = (rsqrt(row / mean_R(row)) * rsqrt(col)) * g;   else: v = fma(u0, 1 - beta2, v * beta2),
 *                     u = rsqrt(v) * g
 *   clip divisor = max(fp32(sqrt(sum u^2)) / fp32(sqrt(numel)) / clip_threshold, 1);  u /= clip divisor
 *   m = fma(u, 1 - beta1, m * beta1);  res = (u - m)^2 + eps2
 *   factored: res_row / res_col as row / col with beta3 over res, upd = (rsqrt(res_row / mean) * rsqrt(res_col)) * m;
 *   else: upd = m
 *   p = p * (1 - weight_decay * (fixed_decay ? 1 : lr));  p = p - upd * lr
 * rsqrt(x) = 1 / sqrt(x), both correctly rounded.  Means are fp64 sums (fixed-order folds: bitwise repeatable, no
 * float atomics) divided in fp64 and rounded to fp32.  Empty tensors are skipped.  Bit-identical to
 * oracle/came_ref.py came_param_emulated fed with the sums written here.
 * replaces: CAME.step (train.py:698-700). */
int dpipe_came_step(const dpipe_came_tensor* t, int n, double clip_threshold, double* scratch, int64_t scratch_len,
                    void* stream);
/* flow-matching noising of one batch on the device, fp32, IEEE-rounded multiplies and adds (bit-identical to the host ops):
 *   xt = (1 - t[b]) * x1 + t[b] * x0,   target = x0 - x1      x1, x0: [bs, c, frames, h, w] contiguous; t: [bs]
 * pack != 0 (frames == 1): both outputs in diffusers' packed layout [bs, (h/2)(w/2), 4c] (2x2 patches, channel-major).
 * replaces: models/flux.py:368-378, models/qwen_image.py:447-455 (pack) and models/wan/wan.py:400-404 (plain). */
int dpipe_noise_pack(const float* x1, const float* x0, const float* t, float* xt, float* target, int bs, int c,
                     int64_t frames, int h, int w, int pack, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* 1F1B pipeline schedule planner (host only).                                                   */
/* replaces: utils/patches.py:113-160 (train_schedule_steps) driven by deepspeed==0.18.4          */
/*           runtime/pipe/schedule.py TrainSchedule / InferenceSchedule helpers.                  */
/* ------------------------------------------------------------------------------------------ */
enum {
  DPIPE_OP_TICK_END = 0, /* closes one schedule tick (one `yield cmds` of the reference) */
  DPIPE_OP_LOAD_MICRO_BATCH = 1,
  DPIPE_OP_SEND_ACTIVATION = 2,
  DPIPE_OP_RECV_ACTIVATION = 3,
  DPIPE_OP_SEND_GRAD = 4,
  DPIPE_OP_RECV_GRAD = 5,
  DPIPE_OP_FORWARD_PASS = 6,
  DPIPE_OP_BACKWARD_PASS = 7,
  DPIPE_OP_REDUCE_TIED_GRADS = 8,
  DPIPE_OP_REDUCE_GRADS = 9,
  DPIPE_OP_OPTIMIZER_STEP = 10,
  DPIPE_OP_BACKWARD_INPUT = 11,  /* split backward: input gradients only (zero-bubble schedule) */
  DPIPE_OP_BACKWARD_WEIGHT = 12  /* split backward: the deferred weight gradients of one micro-batch */
};
typedef struct dpipe_instr {
  int32_t op;          /* DPIPE_OP_* */
  int32_t buffer;      /* pipe buffer index (-1 when not applicable) */
  int32_t micro_batch; /* micro-batch id the instruction belongs to (-1 when not applicable) */
} dpipe_instr;

/* number of activation buffers of a stage: max(2, min(stages - stage_id, micro_batches)) */
int dpipe_sched_num_pipe_buffers(int micro_batches, int stages, int stage_id);
/* writes the instruction stream of one train_batch into out[0..capacity); returns the count (call with capacity 0 to size) */
int dpipe_sched_train(int micro_batches, int stages, int stage_id, dpipe_instr* out, int capacity);
/* forward-only schedule of eval_batch */
int dpipe_sched_infer(int micro_batches, int stages, int stage_id, dpipe_instr* out, int capacity);
/* split-backward ("zero-bubble") order for one stage from a deterministic list-scheduling simulation of all stages with
 * relative costs tf / tb / tw (forward, input-gradient, weight-gradient) and at most max_inflight micro-batches held
 * per stage (forward done, weight-gradient pass pending).  Not in the reference; loss-equivalent to 1F1B.  Same calling
 * convention as dpipe_sched_train.  The _ex form charges stage s (tf, tb, tw) * stage_weight[s] (e.g. its number of
 * transformer blocks; NULL = all 1) and keeps, among a few candidate list schedules, the one with the smallest
 * simulated makespan under those costs. */
int dpipe_sched_zb(int micro_batches, int stages, int stage_id, int tf, int tb, int tw, int max_inflight,
                   dpipe_instr* out, int capacity);
int dpipe_sched_zb_ex(int micro_batches, int stages, int stage_id, int tf, int tb, int tw, int max_inflight,
                      const int* stage_weight, dpipe_instr* out, int capacity);
long long dpipe_sched_zb_makespan(int micro_batches, int stages, int tf, int tb, int tw, int max_inflight);
long long dpipe_sched_zb_makespan_ex(int micro_batches, int stages, int tf, int tb, int tw, int max_inflight,
                                      const int* stage_weight);
/* contiguous min-max partition of n layer weights into `parts` stages; bounds has parts+1 entries
 * (replaces DeepSpeed partition_balanced behind partition_method='parameters', train.py:81-90,606) */
int dpipe_partition_balanced(const int64_t* weights, int n, int parts, int* bounds);

/* ------------------------------------------------------------------------------------------ */
/* fp8 storage of a frozen base (LoRA runs with `transformer_dtype = 'float8'`).                  */
/* replaces: autocast widening the float8 weight to bf16 inside every nn.Linear of the blocks      */
/*           (models/flux.py:172,203-205; models/qwen_image.py:249-262; utils/common.py:18-20).    */
/* ------------------------------------------------------------------------------------------ */
#define DPIPE_FP8_E4M3 0 /* torch.float8_e4m3fn */
#define DPIPE_FP8_E5M2 1 /* torch.float8_e5m2 */
/* dst[r*ld_dst + c] (bf16) = widen(src[r*ld_src + c]) for a rows x cols matrix of fp8 codes (exact: every fp8 value is a
 * bf16 value).  cols and ld_src multiples of 16, ld_dst a multiple of 8, both pointers 16-byte aligned. */
int dpipe_fp8_to_bf16(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int64_t rows, int64_t cols, int format,
                      void* stream);
/* the 256 bf16 bit patterns the kernel maps the fp8 codes to (host function; used by the CPU-side table test) */
int dpipe_fp8_code_table(int format, uint16_t* bf16_bits_256);

/* ------------------------------------------------------------------------------------------ */
/* Stage-boundary transport: CUDA-IPC mailboxes, peer copies over NVLink, device-side flags.     */
/* replaces: DeepSpeed _exec_send/recv_activations/_grads over NCCL p2p, as emitted by the       */
/*           schedule at utils/patches.py:134-143 (SURVEY.md 8a E6).                             */
/* ------------------------------------------------------------------------------------------ */
/* cudaMalloc `bytes` (zero-filled) on the current device and export a 64-byte IPC handle */
int dpipe_ipc_alloc(int64_t bytes, void** dev_ptr, unsigned char* handle64);
/* map a peer process' allocation; the returned pointer is valid in this process */
int dpipe_ipc_open(const unsigned char* handle64, void** dev_ptr);
int dpipe_ipc_close(void* dev_ptr);
int dpipe_ipc_free(void* dev_ptr);
/* cudaMemcpyPeerAsync(dst on dst_device <- src on src_device) on `stream` */
int dpipe_peer_copy(void* dst, int dst_device, const void* src, int src_device, int64_t bytes, void* stream);
/* *flag = value with system-scope release semantics, ordered after all prior work on `stream` */
int dpipe_flag_write(void* flag, uint64_t value, void* stream);
/* blocks `stream` (not the host) until *flag >= value; traps after timeout_s seconds (0 = never) */
int dpipe_flag_wait_geq(const void* flag, uint64_t value, double timeout_s, void* stream);

/* ------------------------------------------------------------------------------------------ */
/* Pipeline-schedule executor: walks one stage's instruction stream; C++ owns the order, the copy stream, the events */
/* and the stage-boundary copies, the host runs only the instructions that need autograd.                           */
/* replaces: deepspeed PipelineEngine._exec_schedule / _exec_send_* / _exec_recv_* over the instruction stream of   */
/*           utils/patches.py:113-160, called from train.py:918 (train_batch) and train.py:181 (eval_batch).        */
/* ------------------------------------------------------------------------------------------ */
typedef struct dpipe_exec dpipe_exec;
enum { DPIPE_CH_ACT_OUT = 0, DPIPE_CH_ACT_IN = 1, DPIPE_CH_GRAD_OUT = 2, DPIPE_CH_GRAD_IN = 3 };
#define DPIPE_OP_NEED_HANDSHAKE 100 /* dpipe_exec_next pseudo-instruction: op = 100 + DPIPE_CH_* of the channel to handshake */
/* copy stream + event pool on the current device; nslots mailbox slots per channel; timeout of the device-side flag waits */
int dpipe_exec_create(int device, int nslots, double timeout_s, dpipe_exec** out);
int dpipe_exec_destroy(dpipe_exec* x);
void* dpipe_exec_copy_stream(dpipe_exec* x); /* cudaStream_t the boundary copies run on */
/* after the host handshake of a channel: sender: flags_local = own `free` flags, remote = the peer's mailbox (mapped);
 * receiver: flags_local = own mailbox, remote = the peer's `free` flags (mapped).  reset_counts when a mailbox was re-made. */
int dpipe_exec_bind(dpipe_exec* x, int channel, void* flags_local, void* remote, int peer_device, int64_t flag_bytes,
                    int64_t slot_bytes, int reset_counts);
/* byte offset and size of every tensor of the boundary tuple inside a slot */
int dpipe_exec_set_layout(dpipe_exec* x, int channel, int n, const int64_t* offsets, const int64_t* nbytes);
int dpipe_exec_forget_layouts(dpipe_exec* x); /* reset_activation_shape(): train.py:916 */
/* the instruction array of dpipe_sched_train / _infer / _zb_ex for this stage */
int dpipe_exec_load_plan(dpipe_exec* x, const dpipe_instr* instrs, int n, int train, int is_first_stage, int is_last_stage,
                         int num_buffers);
/* device pointers of the tuple a coming SendActivation / SendGrad of pipe buffer `buffer` copies (same order as the layout) */
int dpipe_exec_stage_send(dpipe_exec* x, int channel, int buffer, int n, const void* const* ptrs);
/* slot that holds (or will hold) the tuple received for micro_batch on DPIPE_CH_ACT_IN / DPIPE_CH_GRAD_IN */
int dpipe_exec_recv_base(dpipe_exec* x, int channel, int micro_batch, void** base);
/* runs Send* / Recv* instructions itself; returns 1 with *out = the next instruction the host must execute (or a
 * DPIPE_OP_NEED_HANDSHAKE pseudo-instruction), 0 when the plan is finished, < 0 on error */
int dpipe_exec_next(dpipe_exec* x, void* compute_stream, dpipe_instr* out);

#ifdef __cplusplus
}
#endif
#endif /* DPIPE_H_ */
