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
 * dtemb[b,:] += silu'(temb) * (dmod W).  partials: dpipe_mod_bwd_chunks(N) * B * K floats.  dW may be NULL. */
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
