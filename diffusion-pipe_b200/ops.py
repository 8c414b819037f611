"""Tensor-level wrappers over the C ABI (include/dpipe.h).  torch is used only for device memory and streams;
every compute call goes to libdpipe_b200.so, and a missing library raises (no fallback)."""
import ctypes
import math

import torch

from . import _abi, _lib
from ._abi import AttnArgs, AttnBwdArgs, QkBwdArgs, WanNormBwdArgs, WanNormFwdArgs
from ._lib import GemmArgs, QkvEpilogue, check, lib

EPI_STORE = _lib.EPI_STORE
EPI_BIAS_GELU = _lib.EPI_BIAS_GELU
EPI_GATE_RES = _lib.EPI_GATE_RES
EPI_QKV_ROPE = _lib.EPI_QKV_ROPE
EPI_MUL_GELU_GRAD = _lib.EPI_MUL_GELU_GRAD

# kernel-launch counter (bench.py reports it as gpu_launches)
LAUNCHES = 0
# when a list, tensor-core kernels append (start_event, end_event, algorithmic_flops, kind) — bench.py's roofline
PROFILE = None


# when a list, weight-gradient work is queued instead of launched (split-backward / zero-bubble schedule): the engine
# sets it around a BackwardInput pass and runs the queued closures in the matching BackwardWeight pass
WGRAD_DEFER = None


def deferring():
    return WGRAD_DEFER is not None


def defer(fn):
    """run `fn` now, or queue it when a split-backward pass is active"""
    if WGRAD_DEFER is not None:
        WGRAD_DEFER.append(fn)
    else:
        fn()


def _prof_begin():
    if PROFILE is None:
        return None
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def _prof_end(e0, flops, kind, tag=None):
    if e0 is None:
        return
    e1 = torch.cuda.Event(enable_timing=True)
    e1.record()
    PROFILE.append((e0, e1, flops, kind, tag))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _req_bf16(t, name):
    if t.dtype != torch.bfloat16 or not t.is_cuda:
        raise TypeError(f'{name} must be a CUDA bf16 tensor, got {t.dtype} on {t.device}')
    if t.stride(-1) != 1:
        raise ValueError(f'{name} must be contiguous in its last dimension')


def _req_f32(t, name):
    if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
        raise TypeError(f'{name} must be a contiguous CUDA fp32 tensor')


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
def gemm(a, b, *, a_mn=False, b_mn=False, out=None, epilogue=EPI_STORE, bias=None, out2=None, aux=None, gate=None,
         rows_per_batch=None, accumulate=False, cta_group=2, qkv=None, M=None, N=None, K=None):
    """D[M,N] = Aop[M,K] @ Bop[N,K]^T with a fused epilogue (see include/dpipe.h).

    a: [M,K] (a_mn=False) or [K,M] (a_mn=True); b: [N,K] (b_mn=False) or [K,N] (b_mn=True).
    """
    global LAUNCHES
    _req_bf16(a, 'a')
    _req_bf16(b, 'b')
    assert a.dim() == 2 and b.dim() == 2
    if M is None:
        M = a.shape[1] if a_mn else a.shape[0]
    if K is None:
        K = a.shape[0] if a_mn else a.shape[1]
    if N is None:
        N = b.shape[1] if b_mn else b.shape[0]
    kb = b.shape[0] if b_mn else b.shape[1]
    if kb != K:
        raise ValueError(f'reduction dims differ: {K} vs {kb}')
    if out is None:
        out = torch.empty((M, N), dtype=torch.bfloat16, device=a.device)
    _req_bf16(out, 'out')
    args = GemmArgs()
    args.A, args.lda, args.a_mn = _ptr(a), a.stride(0), int(a_mn)
    args.B, args.ldb, args.b_mn = _ptr(b), b.stride(0), int(b_mn)
    args.M, args.N, args.K = M, N, K
    args.epilogue = epilogue
    args.out, args.ldo = _ptr(out), out.stride(0)
    if out2 is not None:
        _req_bf16(out2, 'out2')
        args.out2, args.ldo2 = _ptr(out2), out2.stride(0)
    if bias is not None:
        _req_bf16(bias, 'bias')
        args.bias = _ptr(bias)
    if aux is not None:
        _req_bf16(aux, 'aux')
        args.aux, args.ldaux = _ptr(aux), aux.stride(0)
    if gate is not None:
        _req_bf16(gate, 'gate')
        args.gate, args.gate_stride = _ptr(gate), gate.stride(0)
    args.rows_per_batch = int(rows_per_batch) if rows_per_batch else M
    args.accumulate = int(bool(accumulate))
    args.cta_group = cta_group
    if qkv is not None:
        args.qkv = ctypes.pointer(qkv)
    _e = _prof_begin()
    check(lib().dpipe_gemm_bf16(ctypes.byref(args), _stream()), 'dpipe_gemm_bf16')
    _prof_end(_e, 2.0 * M * N * K, 'gemm', (M, N, K, int(a_mn), int(b_mn), epilogue, int(bool(accumulate))))
    LAUNCHES += 1
    return out


def make_qkv_epilogue(q, k, v, q_norm_w, k_norm_w, rope_cos, rope_sin, heads, seq_total, seq_offset, qhat=None,
                      khat=None, q_rstd=None, k_rstd=None, eps=1e-6):
    e = QkvEpilogue()
    e.q, e.k, e.v = _ptr(q), _ptr(k), _ptr(v)
    e.qhat, e.khat = _ptr(qhat), _ptr(khat)
    e.q_rstd, e.k_rstd = _ptr(q_rstd), _ptr(k_rstd)
    _req_bf16(q_norm_w, 'q_norm_w')
    _req_bf16(k_norm_w, 'k_norm_w')
    e.q_norm_w, e.k_norm_w = _ptr(q_norm_w), _ptr(k_norm_w)
    _req_f32(rope_cos, 'rope_cos')
    _req_f32(rope_sin, 'rope_sin')
    e.rope_cos, e.rope_sin = _ptr(rope_cos), _ptr(rope_sin)
    e.heads, e.seq_total, e.seq_offset = heads, seq_total, seq_offset
    e.n_qkv = 3 * heads * 128
    e.eps = eps
    return e


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
def attn_fwd(q, k, v, out=None, lse=None, scale=None):
    """softmax(q k^T * scale) v.  q: [B,H,Lq,128], k/v: [B,H,Lk,128] (bf16, contiguous).
    Returns (o [B*Lq, >=H*128] token-major, lse [B,H,Lq] fp32 in the log2 domain)."""
    global LAUNCHES
    for t, n in ((q, 'q'), (k, 'k'), (v, 'v')):
        _req_bf16(t, n)
        if not t.is_contiguous() or t.shape[-1] != 128:
            raise ValueError(f'{n} must be contiguous [B,H,L,128]')
    B, H, Lq, _ = q.shape
    Lk = k.shape[2]
    if out is None:
        out = torch.empty((B * Lq, H * 128), dtype=torch.bfloat16, device=q.device)
    if lse is None:
        lse = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
    a = AttnArgs()
    a.q, a.k, a.v = _ptr(q), _ptr(k), _ptr(v)
    a.o, a.ldo = _ptr(out), out.stride(0)
    a.lse = _ptr(lse)
    a.batch, a.heads, a.seq_q, a.seq_k = B, H, Lq, Lk
    a.scale = float(scale if scale is not None else 128 ** -0.5)
    _e = _prof_begin()
    check(lib().dpipe_attn_fwd(ctypes.byref(a), _stream()), 'dpipe_attn_fwd')
    _prof_end(_e, 4.0 * B * H * Lq * Lk * 128, 'attn_fwd')
    LAUNCHES += 1
    return out, lse


def attn_bwd(q, k, v, o, d_o, lse, scale=None, dq=None, dk=None, dv=None, delta=None):
    """Backward of attn_fwd.  o / d_o are token-major [B*Lq, >=H*128]; returns head-major (dq, dk, dv)."""
    global LAUNCHES
    B, H, Lq, _ = q.shape
    Lk = k.shape[2]
    for t, n in ((q, 'q'), (k, 'k'), (v, 'v')):
        _req_bf16(t, n)
        if not t.is_contiguous():
            raise ValueError(f'{n} must be contiguous')
    _req_bf16(o, 'o')
    _req_bf16(d_o, 'd_o')
    dq = torch.empty_like(q) if dq is None else dq
    dk = torch.empty_like(k) if dk is None else dk
    dv = torch.empty_like(v) if dv is None else dv
    delta = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device) if delta is None else delta
    a = AttnBwdArgs()
    a.q, a.k, a.v = _ptr(q), _ptr(k), _ptr(v)
    a.o, a.ldo = _ptr(o), o.stride(0)
    a.d_o, a.lddo = _ptr(d_o), d_o.stride(0)
    a.lse, a.delta = _ptr(lse), _ptr(delta)
    a.dq, a.dk, a.dv = _ptr(dq), _ptr(dk), _ptr(dv)
    a.batch, a.heads, a.seq_q, a.seq_k = B, H, Lq, Lk
    a.scale = float(scale if scale is not None else 128 ** -0.5)
    _e = _prof_begin()
    check(lib().dpipe_attn_bwd(ctypes.byref(a), _stream()), 'dpipe_attn_bwd')
    _prof_end(_e, 10.0 * B * H * Lq * Lk * 128, 'attn_bwd')
    LAUNCHES += 3
    return dq, dk, dv


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm + modulation, gated residual, reductions
# ---------------------------------------------------------------------------------------------------------------
_ROW_CHUNK = None


def row_chunk():
    global _ROW_CHUNK
    if _ROW_CHUNK is None:
        _ROW_CHUNK = lib().dpipe_row_chunk()
    return _ROW_CHUNK


def nchunks(rows_per_batch):
    rc = row_chunk()
    return (rows_per_batch + rc - 1) // rc


LN_MULT_DIRECT = 1   # include/dpipe.h DPIPE_LN_MULT_DIRECT: `scale` is the multiplier itself (affine LayerNorm)
LN_ROUND_STEPS = 2   # DPIPE_LN_ROUND_STEPS: bf16 rounding after every elementwise op (Wan modulation on bf16 tensors)


def ln_modulate_fwd(x, scale, shift, batch, rows_per_batch, eps=1e-6, out=None, save_stats=True, flags=0):
    """out = LN(x) * bf16(1+scale[b]) + shift[b].  x: [batch*rows, D]; scale/shift: [batch, D] views (bf16)."""
    global LAUNCHES
    _req_bf16(x, 'x')
    _req_bf16(scale, 'scale')
    _req_bf16(shift, 'shift')
    D = x.shape[1]
    assert scale.stride(0) == shift.stride(0)
    if out is None:
        out = torch.empty((x.shape[0], D), dtype=torch.bfloat16, device=x.device)
    mean = rstd = None
    if save_stats:
        mean = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
        rstd = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    _e = _prof_begin()
    check(lib().dpipe_ln_modulate_fwd_ex(_ptr(x), x.stride(0), _ptr(scale), _ptr(shift), scale.stride(0), _ptr(out),
                                         out.stride(0), _ptr(mean), _ptr(rstd), batch, rows_per_batch, D, eps, flags,
                                         _stream()), 'dpipe_ln_modulate_fwd')
    _prof_end(_e, 0.0, 'ln_fwd')
    LAUNCHES += 1
    return out, mean, rstd


def ln_modulate_bwd(dxn, x, scale, mean, rstd, batch, rows_per_batch, dres=None, dx=None, partials=None, flags=0):
    """Returns (dx, partials) with partials[batch][nchunk][2][D]: slot 0 = d scale, slot 1 = d shift."""
    global LAUNCHES
    _req_bf16(dxn, 'dxn')
    _req_bf16(x, 'x')
    _req_bf16(scale, 'scale')
    D = x.shape[1]
    nc = nchunks(rows_per_batch)
    if dx is None:
        dx = torch.empty((x.shape[0], D), dtype=torch.bfloat16, device=x.device)
    if partials is None:
        partials = torch.empty((batch, nc, 2, D), dtype=torch.float32, device=x.device)
    if dres is not None:
        _req_bf16(dres, 'dres')
    _e = _prof_begin()
    check(lib().dpipe_ln_modulate_bwd_ex(_ptr(dxn), dxn.stride(0), _ptr(x), x.stride(0), _ptr(scale), scale.stride(0),
                                         _ptr(mean), _ptr(rstd), _ptr(dres), dres.stride(0) if dres is not None else 0,
                                         _ptr(dx), dx.stride(0), _ptr(partials), batch, rows_per_batch, D, flags,
                                         _stream()), 'dpipe_ln_modulate_bwd')
    _prof_end(_e, 0.0, 'ln_bwd')
    LAUNCHES += 1
    return dx, partials


def gate_bwd(dx, y, gate, batch, rows_per_batch, dy=None, partials=None):
    """dy = bf16(gate*dx); partial slot 0 = sum dx*y (d gate per sample), slot 1 = sum dy (d bias)."""
    global LAUNCHES
    _req_bf16(dx, 'dx')
    _req_bf16(y, 'y')
    _req_bf16(gate, 'gate')
    D = y.shape[1]
    nc = nchunks(rows_per_batch)
    if dy is None:
        dy = torch.empty((y.shape[0], D), dtype=torch.bfloat16, device=y.device)
    if partials is None:
        partials = torch.empty((batch, nc, 2, D), dtype=torch.float32, device=y.device)
    _e = _prof_begin()
    check(lib().dpipe_gate_bwd(_ptr(dx), dx.stride(0), _ptr(y), y.stride(0), _ptr(gate), gate.stride(0), _ptr(dy),
                               dy.stride(0), _ptr(partials), batch, rows_per_batch, D, _stream()), 'dpipe_gate_bwd')
    _prof_end(_e, 0.0, 'gate_bwd')
    LAUNCHES += 1
    return dy, partials


def colreduce_finish(partials, per_sample0=None, per_sample1=None, summed0=None, summed1=None):
    """partials [batch, nchunk, nslot, D] fp32.  per_sample*: fp32 [batch, D] views (row stride = stride(0));
    summed*: fp32 [D]."""
    global LAUNCHES
    batch, nc, nslot, D = partials.shape
    ld0 = per_sample0.stride(0) if per_sample0 is not None else 0
    ld1 = per_sample1.stride(0) if per_sample1 is not None else 0
    _e = _prof_begin()
    check(lib().dpipe_colreduce_finish(_ptr(partials), batch, nc, nslot, D, _ptr(per_sample0), ld0, _ptr(per_sample1),
                                       ld1, _ptr(summed0), _ptr(summed1), _stream()), 'dpipe_colreduce_finish')
    _prof_end(_e, 0.0, 'finish')
    LAUNCHES += 1


def colsum(x, out=None):
    """fp32 column sums of a bf16 [rows, N] matrix."""
    global LAUNCHES
    _req_bf16(x, 'x')
    rows, N = x.shape
    nc = lib().dpipe_colsum_chunks(rows)
    partials = torch.empty((nc, N), dtype=torch.float32, device=x.device)
    if out is None:
        out = torch.empty(N, dtype=torch.float32, device=x.device)
    _e = _prof_begin()
    check(lib().dpipe_colsum(_ptr(x), x.stride(0), rows, N, _ptr(partials), _ptr(out), _stream()), 'dpipe_colsum')
    _prof_end(_e, 0.0, 'colsum')
    LAUNCHES += 2
    return out


FP8_FORMATS = {torch.float8_e4m3fn: 0, torch.float8_e5m2: 1}      # DPIPE_FP8_E4M3 / DPIPE_FP8_E5M2


def fp8_to_bf16(src, dst):
    """dst (bf16 [rows, cols] view, last dimension contiguous) = widen(src) for a 2-D fp8 matrix (float8_e4m3fn or
    float8_e5m2; exact).  The frozen base of a LoRA run stored in fp8 is expanded into a GEMM operand buffer with this
    before each GEMM that reads it (reference: autocast widens the float8 weight inside nn.Linear)."""
    global LAUNCHES
    if src.dtype not in FP8_FORMATS or not src.is_cuda or src.dim() != 2 or src.stride(1) != 1:
        raise TypeError(f'src must be a 2-D CUDA float8 tensor with a contiguous last dimension, got {src.dtype} {tuple(src.shape)}')
    _req_bf16(dst, 'dst')
    if dst.dim() != 2 or tuple(dst.shape) != tuple(src.shape):
        raise ValueError(f'dst {tuple(dst.shape)} must have the shape of src {tuple(src.shape)}')
    _e = _prof_begin()
    check(lib().dpipe_fp8_to_bf16(_ptr(src), src.stride(0), _ptr(dst), dst.stride(0), src.shape[0], src.shape[1],
                                  FP8_FORMATS[src.dtype], _stream()), 'dpipe_fp8_to_bf16')
    _prof_end(_e, 0.0, 'fp8_widen')
    LAUNCHES += 1
    return dst


def qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, q_norm_w, k_norm_w, rope_cos, rope_sin, dqkv, dbias, dw,
                    batch, heads, seq_total, seq_offset, rows_per_batch):
    """Backward of the QKV_ROPE epilogue for one stream: writes token-major dqkv [batch*rows, 3*H*128] and
    accumulates dbias (fp32 [3*H*128]) and dw (fp32 [2,128]) — both must be zero-initialised by the caller."""
    global LAUNCHES
    a = QkBwdArgs()
    a.dq, a.dk, a.dv = _ptr(dq), _ptr(dk), _ptr(dv)
    a.qhat, a.khat = _ptr(qhat), _ptr(khat)
    a.q_rstd, a.k_rstd = _ptr(q_rstd), _ptr(k_rstd)
    a.q_norm_w, a.k_norm_w = _ptr(q_norm_w), _ptr(k_norm_w)
    a.rope_cos, a.rope_sin = _ptr(rope_cos), _ptr(rope_sin)
    _req_bf16(dqkv, 'dqkv')
    a.dqkv, a.ld = _ptr(dqkv), dqkv.stride(0)
    _req_f32(dbias, 'dbias')
    _req_f32(dw, 'dw')
    a.dbias, a.dw = _ptr(dbias), _ptr(dw)
    a.batch, a.heads, a.seq_total, a.seq_offset, a.rows_per_batch = batch, heads, seq_total, seq_offset, rows_per_batch
    _e = _prof_begin()
    check(lib().dpipe_qknorm_rope_bwd(ctypes.byref(a), _stream()), 'dpipe_qknorm_rope_bwd')
    _prof_end(_e, 0.0, 'qknorm_bwd')
    LAUNCHES += 1


def wan_norm_rope_fwd(projs, batch, seq, heads, cos=None, sin=None, eps=1e-6):
    """Wan q/k/v pre-processing (csrc/wan_norm.cu).  projs: up to three dicts {src [batch*seq, >=C] bf16 view, weight
    [C] bf16 or None, rope bool}.  Returns per projection (dst [batch, heads, seq, 128], xhat [batch*seq, C] or None,
    rstd [batch*seq] or None)."""
    global LAUNCHES
    a = WanNormFwdArgs()
    C = heads * 128
    outs = []
    for i, pj in enumerate(projs):
        src = pj['src']
        _req_bf16(src, 'src')
        dev = src.device
        dst = torch.empty((batch, heads, seq, 128), dtype=torch.bfloat16, device=dev)
        w = pj.get('weight')
        xhat = rstd = None
        if w is not None:
            _req_bf16(w, 'weight')
            xhat = torch.empty((batch * seq, C), dtype=torch.bfloat16, device=dev)
            rstd = torch.empty(batch * seq, dtype=torch.float32, device=dev)
        e = a.proj[i]
        e.src, e.ld, e.weight, e.dst, e.xhat, e.rstd = _ptr(src), src.stride(0), _ptr(w), _ptr(dst), _ptr(xhat), _ptr(rstd)
        e.rope = 1 if pj.get('rope') else 0
        outs.append((dst, xhat, rstd))
    a.nproj = len(projs)
    if cos is not None:
        _req_f32(cos, 'cos')
        _req_f32(sin, 'sin')
    a.cos, a.sin = _ptr(cos), _ptr(sin)
    a.batch, a.seq, a.heads, a.eps = batch, seq, heads, eps
    _e = _prof_begin()
    check(lib().dpipe_wan_norm_rope_fwd(ctypes.byref(a), _stream()), 'dpipe_wan_norm_rope_fwd')
    _prof_end(_e, 0.0, 'wan_norm_fwd')
    LAUNCHES += 1
    return outs


def wan_norm_rope_bwd(projs, batch, seq, heads, cos=None, sin=None):
    """Backward of wan_norm_rope_fwd.  projs: dicts {dy [batch, heads, seq, 128], dx [batch*seq, >=C] bf16 view (written),
    weight, xhat, rstd (None for v), rope}.  Returns, per projection, the fp32 d weight [C] (or None)."""
    global LAUNCHES
    a = WanNormBwdArgs()
    C = heads * 128
    rows = batch * seq
    nchunk = (rows + lib().dpipe_wan_norm_rows() - 1) // lib().dpipe_wan_norm_rows()
    parts = []
    for i, pj in enumerate(projs):
        dy, dx = pj['dy'], pj['dx']
        _req_bf16(dy, 'dy')
        _req_bf16(dx, 'dx')
        if not dy.is_contiguous():
            raise ValueError('dy must be a contiguous [batch, heads, seq, 128] tensor')
        w = pj.get('weight')
        part = torch.empty((1, nchunk, 1, C), dtype=torch.float32, device=dy.device) if w is not None else None
        e = a.proj[i]
        e.dy, e.xhat, e.rstd, e.weight = _ptr(dy), _ptr(pj.get('xhat')), _ptr(pj.get('rstd')), _ptr(w)
        e.dx, e.ld, e.dw_partials = _ptr(dx), dx.stride(0), _ptr(part)
        e.rope = 1 if pj.get('rope') else 0
        parts.append(part)
    a.nproj = len(projs)
    a.cos, a.sin = _ptr(cos), _ptr(sin)
    a.batch, a.seq, a.heads = batch, seq, heads
    _e = _prof_begin()
    check(lib().dpipe_wan_norm_rope_bwd(ctypes.byref(a), _stream()), 'dpipe_wan_norm_rope_bwd')
    _prof_end(_e, 0.0, 'wan_norm_bwd')
    LAUNCHES += 1
    dws = []
    for part in parts:
        if part is None:
            dws.append(None)
            continue
        dw = torch.empty(C, dtype=torch.float32, device=part.device)
        colreduce_finish(part, summed0=dw)
        dws.append(dw)
    return dws


def mod_fwd(temb, weight, bias):
    """mod[B, N] = W @ bf16(silu(temb)) + bias  (rank-B, HBM-bound kernel; temb [B, K] bf16)."""
    global LAUNCHES
    _req_bf16(temb, 'temb')
    _req_bf16(weight, 'weight')
    assert temb.is_contiguous() and weight.is_contiguous()
    B, K = temb.shape
    N = weight.shape[0]
    out = torch.empty((B, N), dtype=torch.bfloat16, device=temb.device)
    _e = _prof_begin()
    check(lib().dpipe_mod_fwd(_ptr(temb), _ptr(weight), _ptr(bias), _ptr(out), B, N, K, _stream()), 'dpipe_mod_fwd')
    _prof_end(_e, 0.0, 'mod_fwd')
    LAUNCHES += 1
    return out


def mod_bwd(dmod32, temb, weight, wgrad, accumulate, dtemb32):
    """Backward of mod_fwd.  dmod32 fp32 [B, N]; wgrad bf16 [N, K] or None; dtemb32 fp32 [B, K] is accumulated into.
    Returns dbias fp32 [N]."""
    global LAUNCHES
    _req_f32(dmod32, 'dmod32')
    _req_f32(dtemb32, 'dtemb32')
    B, K = temb.shape
    N = weight.shape[0]
    nc = lib().dpipe_mod_bwd_chunks(N)
    partials = torch.empty((nc, B, K), dtype=torch.float32, device=temb.device)
    dbias = torch.empty(N, dtype=torch.float32, device=temb.device)
    _e = _prof_begin()
    check(lib().dpipe_mod_bwd(_ptr(dmod32), dmod32.stride(0), _ptr(temb), _ptr(weight), _ptr(wgrad), int(bool(accumulate)),
                              _ptr(dbias), _ptr(partials), _ptr(dtemb32), B, N, K, _stream()), 'dpipe_mod_bwd')
    _prof_end(_e, 0.0, 'mod_bwd')
    LAUNCHES += 2
    return dbias


def mse_loss(out, target, mask=None, want_grad=True):
    """(loss fp32 scalar tensor, dout bf16 or None) for loss = mean((out-target)^2 * mask)."""
    global LAUNCHES
    _req_bf16(out, 'out')
    assert out.is_contiguous()
    target = target.to(torch.float32).contiguous()
    if mask is not None:
        mask = mask.to(torch.float32).expand_as(target).contiguous()
    ws = torch.empty(1024, dtype=torch.float32, device=out.device)
    loss = torch.empty((), dtype=torch.float32, device=out.device)
    dout = torch.empty_like(out) if want_grad else None
    _e = _prof_begin()
    check(lib().dpipe_mse_loss(_ptr(out), _ptr(target), _ptr(mask), out.numel(), _ptr(ws), _ptr(loss), _ptr(dout),
                               _stream()), 'dpipe_mse_loss')
    _prof_end(_e, 0.0, 'mse')
    LAUNCHES += 2
    return loss, dout


# ---------------------------------------------------------------------------------------------------------------
# optimizer-step tail (gradient norm / clipping, AdamW step) and micro-batch preparation
# ---------------------------------------------------------------------------------------------------------------
_GRAD_DTYPES = {torch.bfloat16: 0, torch.float32: 1}


def _tensor_lists(tensors):
    n = len(tensors)
    ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tensors])
    numels = (ctypes.c_int64 * n)(*[t.numel() for t in tensors])
    dtypes = (ctypes.c_int * n)(*[_GRAD_DTYPES[t.dtype] for t in tensors])
    return ptrs, numels, dtypes


def grads_supported(tensors):
    return all(t.is_cuda and t.dtype in _GRAD_DTYPES and t.is_contiguous() for t in tensors)


def grad_sumsq(tensors):
    """fp32 device scalar: sum over `tensors` (contiguous CUDA bf16 / fp32) of sum(g^2) — one pass, no fp32 copies"""
    global LAUNCHES
    dev = tensors[0].device
    nl = max(1, (len(tensors) + 63) // 64)
    blocks = lib().dpipe_grad_sumsq_blocks()
    partials = torch.empty(blocks * nl, dtype=torch.float32, device=dev)
    out = torch.empty((), dtype=torch.float32, device=dev)
    ptrs, numels, dtypes = _tensor_lists(tensors)
    _e = _prof_begin()
    check(lib().dpipe_grad_sumsq(ptrs, numels, dtypes, len(tensors), _ptr(partials), partials.numel(), _ptr(out), _stream()),
          'dpipe_grad_sumsq')
    _prof_end(_e, 0.0, 'grad_sumsq')
    LAUNCHES += nl + 1
    return out


def grad_scale(tensors, coef):
    """g *= coef (fp32 device scalar) in place; the kernels return immediately when coef >= 1"""
    global LAUNCHES
    _req_f32(coef, 'coef')
    ptrs, numels, dtypes = _tensor_lists(tensors)
    _e = _prof_begin()
    check(lib().dpipe_grad_scale(ptrs, numels, dtypes, len(tensors), _ptr(coef), _stream()), 'dpipe_grad_scale')
    _prof_end(_e, 0.0, 'grad_scale')
    LAUNCHES += max(1, (len(tensors) + 63) // 64)


def adamw_step(params, grads, exp_avgs, exp_avg_sqs, kahan_comps, *, lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps,
               decay):
    """One AdamW step (optimi's update rule, include/dpipe.h dpipe_adamw_step) in place over the tensor sets
    (p, g, m, v, c): contiguous CUDA tensors of one shape and dtype (bf16 or fp32) per set; kahan_comps[i] is None for no
    Kahan compensation and must be None for fp32.  The scalars are the fp32 values the kernel uses (optim.step_scalars)."""
    global LAUNCHES
    n = len(params)
    if not (len(grads) == len(exp_avgs) == len(exp_avg_sqs) == len(kahan_comps) == n):
        raise ValueError('adamw_step: the five tensor lists differ in length')
    for i, (p, g, m, v, c) in enumerate(zip(params, grads, exp_avgs, exp_avg_sqs, kahan_comps)):
        if p.dtype not in _GRAD_DTYPES:
            raise TypeError(f'adamw_step: tensor {i} is {p.dtype}; the kernel takes bf16 or fp32')
        for t, name in ((p, 'param'), (g, 'grad'), (m, 'exp_avg'), (v, 'exp_avg_sq'), (c, 'kahan_comp')):
            if t is None and name == 'kahan_comp':
                continue
            if not t.is_cuda or t.dtype != p.dtype or t.shape != p.shape or not t.is_contiguous():
                raise TypeError(f'adamw_step: {name} {i} must be a contiguous CUDA {p.dtype} tensor of shape '
                                f'{tuple(p.shape)}, got {t.dtype} {tuple(t.shape)} on {t.device}')
        if c is not None and p.dtype != torch.bfloat16:
            raise TypeError(f'adamw_step: tensor {i}: Kahan compensation is for bf16 tensors only')
    if n == 0:
        return

    def ptrs(ts):
        return (ctypes.c_void_p * n)(*[t.data_ptr() if t is not None else None for t in ts])
    numels = (ctypes.c_int64 * n)(*[p.numel() for p in params])
    dtypes = (ctypes.c_int * n)(*[_GRAD_DTYPES[p.dtype] for p in params])
    _e = _prof_begin()
    check(lib().dpipe_adamw_step(ptrs(params), ptrs(grads), ptrs(exp_avgs), ptrs(exp_avg_sqs), ptrs(kahan_comps), numels,
                                 dtypes, n, lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps, decay, _stream()),
          'dpipe_adamw_step')
    _prof_end(_e, 0.0, 'adamw_step')
    LAUNCHES += (n + 63) // 64


def automagic_dims(shape):
    """(factored, L, R, C) of a parameter shape: ndim >= 2 is factored over [L = prod(shape[:-2]), R, C]"""
    if len(shape) < 2:
        return False, 1, 1, 1
    lead = 1
    for s in shape[:-2]:
        lead *= int(s)
    return True, lead, int(shape[-2]), int(shape[-1])


def automagic_workspace(params):
    """one fp32 buffer on the params' device, returned as per-tensor views: [clip divisor, max |new_lr|, avg_lr,
    fp32(previous scale)] and, for factored tensors, L row means, L*R row factors, L*C column factors (include/dpipe.h)"""
    sizes = []
    for p in params:
        f, L, R, C = automagic_dims(p.shape)
        sizes.append(4 + (L + L * R + L * C if f else 0))
    flat = torch.empty(max(1, sum(sizes)), dtype=torch.float32, device=params[0].device if params else 'cpu')
    return list(torch.split(flat[:sum(sizes)], sizes)) if params else []


def _automagic_args(name, params, grads, rows, cols, vs, codes, scales, polarities, shifts, avg_lrs, ws, round_bf16,
                    beta2, eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay):
    n = len(params)
    lists = (grads, rows, cols, vs, codes, scales, polarities, shifts, avg_lrs, ws, round_bf16)
    if any(len(x) != n for x in lists):
        raise ValueError(f'{name}: the tensor lists differ in length')
    arr = (_abi.AutomagicTensor * max(1, n))()

    def need(t, what, i, dtype, numel):
        if t is None or not t.is_cuda or t.dtype != dtype or t.numel() != numel or not t.is_contiguous():
            got = 'None' if t is None else f'{t.dtype} {tuple(t.shape)} on {t.device}'
            raise TypeError(f'{name}: {what} {i} must be a contiguous CUDA {dtype} tensor of {numel} elements, got {got}')
        return t.data_ptr()
    for i, p in enumerate(params):
        if p.dtype not in _GRAD_DTYPES:
            raise TypeError(f'{name}: tensor {i} is {p.dtype}; the kernels take bf16 or fp32 weights')
        f, L, R, C = automagic_dims(p.shape)
        n_el = p.numel()
        a = arr[i]
        a.p = need(p, 'param', i, p.dtype, n_el)
        a.g = need(grads[i], 'grad', i, p.dtype, n_el)
        if f:
            a.row = need(rows[i], 'exp_avg_sq_row', i, torch.float32, L * R)
            a.col = need(cols[i], 'exp_avg_sq_col', i, torch.float32, L * C)
        else:
            a.v = need(vs[i], 'exp_avg_sq', i, torch.float32, n_el)
        a.code = need(codes[i], 'lr codes', i, torch.int8, n_el)
        a.pol = need(polarities[i], 'last_polarity', i, torch.bool, n_el)
        if p.dtype == torch.bfloat16:
            a.shift = need(shifts[i], 'shift', i, torch.bfloat16, n_el)
        elif shifts[i] is not None:
            raise TypeError(f'{name}: tensor {i}: the Kahan shift is for bf16 weights only')
        a.scale = need(scales[i], 'lr code scale', i, torch.float64, 1)
        a.avg_lr = need(avg_lrs[i], 'avg_lr', i, torch.float32, 1)
        a.ws = need(ws[i], 'workspace', i, torch.float32, 4 + (L + L * R + L * C if f else 0))
        a.numel, a.L, a.R, a.C = n_el, L, R, C
        a.dtype = _GRAD_DTYPES[p.dtype]
        a.flags = (1 if f else 0) | (2 if round_bf16[i] else 0)
    sc = _abi.AutomagicScalars(beta2, eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay)
    return arr, n, sc


def automagic_stats(params, grads, rows, cols, vs, codes, scales, polarities, shifts, avg_lrs, ws, round_bf16, *, beta2,
                    eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay):
    """Automagic statistics phase (include/dpipe.h dpipe_automagic_stats) over parameter i with its state: rows / cols
    (factored) or vs (1-D / 0-D) fp32 EMA statistics, updated in place; int8 lr codes, bool last polarity, fp64 0-dim
    code scale (replaced by the new scale), fp32 0-dim avg_lr (written); ws[i] from automagic_workspace (written);
    round_bf16[i] for step 1 of a bf16 parameter.  No host synchronisation."""
    global LAUNCHES
    arr, n, sc = _automagic_args('automagic_stats', params, grads, rows, cols, vs, codes, scales, polarities, shifts,
                                 avg_lrs, ws, round_bf16, beta2, eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay)
    if n == 0:
        return
    need = ctypes.c_int64()
    check(lib().dpipe_automagic_scratch_doubles(arr, n, ctypes.byref(need)), 'dpipe_automagic_scratch_doubles')
    scratch = torch.empty(max(1, need.value), dtype=torch.float64, device=params[0].device)
    _e = _prof_begin()
    check(lib().dpipe_automagic_stats(arr, n, ctypes.byref(sc), scratch.data_ptr(), scratch.numel(), _stream()),
          'dpipe_automagic_stats')
    _prof_end(_e, 0.0, 'automagic_stats')
    LAUNCHES += 5 * ((n + 63) // 64)


def automagic_apply(params, grads, rows, cols, vs, codes, scales, polarities, shifts, avg_lrs, ws, round_bf16, *, beta2,
                    eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay):
    """Automagic apply phase (include/dpipe.h dpipe_automagic_apply) after automagic_stats on the same arguments: new
    polarity and lr codes, weight decay, Kahan-summed bf16 (plain fp32) weight update, in place; the weights' version
    counters move."""
    global LAUNCHES
    arr, n, sc = _automagic_args('automagic_apply', params, grads, rows, cols, vs, codes, scales, polarities, shifts,
                                 avg_lrs, ws, round_bf16, beta2, eps, lr_bump, min_lr, max_lr, clip_threshold, weight_decay)
    if n == 0:
        return
    _e = _prof_begin()
    check(lib().dpipe_automagic_apply(arr, n, ctypes.byref(sc), _stream()), 'dpipe_automagic_apply')
    _prof_end(_e, 0.0, 'automagic_apply')
    LAUNCHES += (n + 63) // 64
    # the kernel wrote the weights behind autograd's back: move their version counters as an in-place op would, so
    # that caches keyed on them (lora.py's fused factor buffers) see the new values
    for p in params:
        torch.autograd.graph.increment_version(p)


class ProdigyArgs:
    """The packed per-tensor arguments of Prodigy steps (include/dpipe.h dpipe_prodigy_tensor) and their fp64 scratch,
    built once by `prodigy_pack` and reused while the parameters, their state and the group options stay the same:
    filling the ctypes array costs host time per tensor.  It holds no gradients: `prodigy_stats` writes the gradient
    pointers of each step into the packed array with one tensor copy and keeps no reference to them.
    scratch[2i], scratch[2i + 1] hold tensor i's dot(g, p0 - p) and sum(|s|) after `prodigy_stats`."""

    def __init__(self, arr, params, s, p0, m, v, scratch):
        self.arr, self.n = arr, len(params)
        self.params, self.s, self.p0, self.m, self.v = params, s, p0, m, v
        self.scratch = scratch
        self.chunks = (sum(1 for p in params if p.numel()) + 63) // 64      # launches per phase (empty tensors skipped)
        words = torch.frombuffer(arr, dtype=torch.int64).view(-1, ctypes.sizeof(_abi.ProdigyTensor) // 8)
        self._g = words[:self.n, _abi.ProdigyTensor.g.offset // 8]          # the `g` field of every entry

    def set_grads(self, grads):
        """point the packed entries at this step's gradients (same shape, dtype, device and contiguity as the
        parameters)"""
        if len(grads) != self.n:
            raise ValueError(f'prodigy: {len(grads)} gradients for {self.n} parameters')
        for i, (p, g) in enumerate(zip(self.params, grads)):
            if g is None or g.dtype != p.dtype or g.shape != p.shape or g.get_device() != p.get_device() \
                    or not g.is_contiguous():
                got = 'None' if g is None else f'{g.dtype} {tuple(g.shape)} on {g.device}'
                raise TypeError(f'prodigy: grad {i} must be a contiguous {p.dtype} tensor of shape {tuple(p.shape)} '
                                f'on {p.device}, got {got}')
        if self.n:
            self._g.copy_(torch.tensor([g.data_ptr() for g in grads], dtype=torch.int64))


def prodigy_pack(params, s, p0, m, v, weight_decay, eps, fixed_decay, device=None):
    """ProdigyArgs for the parameters of every param group in group order: per parameter its state tensors s, p0,
    exp_avg (m), exp_avg_sq (v) (contiguous CUDA tensors of its shape and dtype, bf16 or fp32) and its group's
    weight_decay, eps, fixed_decay.  device: where the scratch goes (the parameters' device by default)."""
    n = len(params)
    if any(len(x) != n for x in (s, p0, m, v, weight_decay, eps, fixed_decay)):
        raise ValueError('prodigy_pack: the argument lists differ in length')
    arr = (_abi.ProdigyTensor * max(1, n))()
    for i, p in enumerate(params):
        if p.dtype not in _GRAD_DTYPES:
            raise TypeError(f'prodigy: tensor {i} is {p.dtype}; the kernels take bf16 or fp32 weights')
        for t, name in ((p, 'param'), (s[i], 's'), (p0[i], 'p0'), (m[i], 'exp_avg'), (v[i], 'exp_avg_sq')):
            if t is None or not t.is_cuda or t.dtype != p.dtype or t.shape != p.shape or not t.is_contiguous():
                got = 'None' if t is None else f'{t.dtype} {tuple(t.shape)} on {t.device}'
                raise TypeError(f'prodigy: {name} {i} must be a contiguous CUDA {p.dtype} tensor of shape '
                                f'{tuple(p.shape)}, got {got}')
        a = arr[i]
        a.p, a.p0, a.s, a.m, a.v = (t.data_ptr() for t in (p, p0[i], s[i], m[i], v[i]))
        a.g = a.p                   # a valid pointer until prodigy_stats writes the step's gradient
        a.numel, a.weight_decay, a.eps = p.numel(), weight_decay[i], eps[i]
        a.dtype, a.fixed_decay = _GRAD_DTYPES[p.dtype], int(bool(fixed_decay[i]))
    need = ctypes.c_int64()
    check(lib().dpipe_prodigy_scratch_doubles(arr, n, ctypes.byref(need)), 'dpipe_prodigy_scratch_doubles')
    scratch = torch.empty(max(1, need.value), dtype=torch.float64, device=device if device is not None else params[0].device)
    return ProdigyArgs(arr, list(params), list(s), list(p0), list(m), list(v), scratch)


def prodigy_stats(args, grads, state, *, lr, betas, beta3, d0, d_coef, growth_rate, bias_correction, safeguard_warmup):
    """Prodigy statistics phase (include/dpipe.h dpipe_prodigy_stats) over every tensor of `args` with this step's
    gradients `grads` (one per parameter): s, exp_avg, exp_avg_sq in place; then d_numerator, d_denom, d_hat, d,
    d_max, step and the skip flag in `state`, the optimizer's fp64 device block of _abi.PRODIGY_STATE_DOUBLES (read for
    the old d and step).  Host scalars are group 0's hyper-parameters (beta3 None: sqrt(beta2)).  No host
    synchronisation."""
    global LAUNCHES
    if state.dtype != torch.float64 or not state.is_cuda or state.numel() != _abi.PRODIGY_STATE_DOUBLES:
        raise TypeError('prodigy_stats: state must be a CUDA fp64 tensor of '
                        f'{_abi.PRODIGY_STATE_DOUBLES} elements')
    args.set_grads(grads)
    b1, b2 = betas
    sc = _abi.ProdigyScalars(lr, b1, b2, beta3 if beta3 is not None else math.sqrt(b2), d0, d_coef, growth_rate,
                             int(bool(bias_correction)), int(bool(safeguard_warmup)))
    _e = _prof_begin()
    check(lib().dpipe_prodigy_stats(args.arr, args.n, ctypes.byref(sc), state.data_ptr(), args.scratch.data_ptr(),
                                    args.scratch.numel(), _stream()), 'dpipe_prodigy_stats')
    _prof_end(_e, 0.0, 'prodigy_stats')
    LAUNCHES += (1 if args.n else 0) + 2 * args.chunks + 1          # memset of the sums, stats + fold per chunk, finish


def prodigy_apply(args, state):
    """Prodigy apply phase (include/dpipe.h dpipe_prodigy_apply) after prodigy_stats: the weights in place, unless the
    statistics phase set the skip flag; the weights' version counters move."""
    global LAUNCHES
    _e = _prof_begin()
    check(lib().dpipe_prodigy_apply(args.arr, args.n, state.data_ptr(), _stream()), 'dpipe_prodigy_apply')
    _prof_end(_e, 0.0, 'prodigy_apply')
    LAUNCHES += args.chunks
    for p in args.params:           # as automagic_apply: caches keyed on the version see the new weights
        torch.autograd.graph.increment_version(p)


class CameArgs:
    """The packed per-tensor arguments of CAME steps (include/dpipe.h dpipe_came_tensor), their workspaces and fp64
    scratch, built once by `came_pack` and reused while the parameters, their state and the group options other than
    lr stay the same.  It holds no gradients: `came_step` writes each step's gradient pointers and learning rates into
    the packed array with one tensor copy each.  fac[i] / sums[i] are tensor i's views of the fp32 / fp64 workspaces
    (clip divisor and factors / the fp64 sums of the last step)."""

    def __init__(self, arr, params, state, fac, sums, scratch, launches):
        self.arr, self.n = arr, len(params)
        self.params, self.state = params, state             # the state tensors the array points at, kept alive
        self.fac, self.sums, self.scratch = fac, sums, scratch
        self.launches = launches
        cols = ctypes.sizeof(_abi.CameTensor) // 8
        self._g = torch.frombuffer(arr, dtype=torch.int64).view(-1, cols)[:self.n, _abi.CameTensor.g.offset // 8]
        self._lr = torch.frombuffer(arr, dtype=torch.float64).view(-1, cols)[:self.n, _abi.CameTensor.lr.offset // 8]

    def set_step(self, grads, lrs):
        """point the packed entries at this step's gradients (same shape, dtype, device and contiguity as the
        parameters) and learning rates"""
        if len(grads) != self.n or len(lrs) != self.n:
            raise ValueError(f'came: {len(grads)} gradients and {len(lrs)} learning rates for {self.n} parameters')
        for i, (p, g) in enumerate(zip(self.params, grads)):
            if g is None or g.dtype != p.dtype or g.shape != p.shape or g.get_device() != p.get_device() \
                    or not g.is_contiguous():
                got = 'None' if g is None else f'{g.dtype} {tuple(g.shape)} on {g.device}'
                raise TypeError(f'came: grad {i} must be a contiguous {p.dtype} tensor of shape {tuple(p.shape)} '
                                f'on {p.device}, got {got}')
        if self.n:
            self._g.copy_(torch.tensor([g.data_ptr() for g in grads], dtype=torch.int64))
            self._lr.copy_(torch.tensor([float(x) for x in lrs], dtype=torch.float64))


def came_workspace_sizes(shape):
    """(fp32, fp64) workspace elements of one tensor (include/dpipe.h dpipe_came_tensor fac / sums)"""
    f, L, R, C = automagic_dims(shape)
    return (1 + 2 * (L * R + L * C), 1 + 2 * (L * R + L * C + L)) if f else (1, 1)


def came_pack(params, m, row, col, res_row, res_col, v, weight_decay, betas, eps1, eps2, fixed_decay):
    """CameArgs for the parameters of every param group in group order: per parameter its state exp_avg (m), and
    exp_avg_sq_row / _col, exp_avg_res_row / _col (ndim >= 2: row / col / res_row / res_col, None otherwise) or
    exp_avg_sq (v, None for ndim >= 2), contiguous CUDA tensors of its dtype (bf16 or fp32), and its group's
    weight_decay, betas (beta1, beta2, beta3), eps1, eps2, fixed_decay."""
    n = len(params)
    if any(len(x) != n for x in (m, row, col, res_row, res_col, v, weight_decay, betas, eps1, eps2, fixed_decay)):
        raise ValueError('came_pack: the argument lists differ in length')
    arr = (_abi.CameTensor * max(1, n))()
    sizes = [came_workspace_sizes(p.shape) for p in params]
    dev = params[0].device if params else 'cpu'
    fac_flat = torch.empty(max(1, sum(s[0] for s in sizes)), dtype=torch.float32, device=dev)
    sums_flat = torch.zeros(max(1, sum(s[1] for s in sizes)), dtype=torch.float64, device=dev)
    fac = list(torch.split(fac_flat[:sum(s[0] for s in sizes)], [s[0] for s in sizes])) if n else []
    sums = list(torch.split(sums_flat[:sum(s[1] for s in sizes)], [s[1] for s in sizes])) if n else []

    def need(t, what, i, p, shape):
        if t is None or not t.is_cuda or t.dtype != p.dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
            got = 'None' if t is None else f'{t.dtype} {tuple(t.shape)} on {t.device}'
            raise TypeError(f'came: {what} {i} must be a contiguous CUDA {p.dtype} tensor of shape {tuple(shape)}, '
                            f'got {got}')
        return t.data_ptr()
    for i, p in enumerate(params):
        if p.dtype not in _GRAD_DTYPES:
            raise TypeError(f'came: tensor {i} is {p.dtype}; the kernels take bf16 or fp32 weights')
        f, L, R, C = automagic_dims(p.shape)
        a = arr[i]
        a.p = need(p, 'param', i, p, p.shape)
        a.g = a.p                   # a valid pointer until came_step writes the step's gradient
        a.m = need(m[i], 'exp_avg', i, p, p.shape)
        if f:
            a.row = need(row[i], 'exp_avg_sq_row', i, p, p.shape[:-1])
            a.col = need(col[i], 'exp_avg_sq_col', i, p, p.shape[:-2] + p.shape[-1:])
            a.res_row = need(res_row[i], 'exp_avg_res_row', i, p, p.shape[:-1])
            a.res_col = need(res_col[i], 'exp_avg_res_col', i, p, p.shape[:-2] + p.shape[-1:])
        else:
            a.v = need(v[i], 'exp_avg_sq', i, p, p.shape)
        a.fac, a.sums = fac[i].data_ptr(), sums[i].data_ptr()
        a.numel, a.L, a.R, a.C = p.numel(), L, R, C
        a.weight_decay, (a.beta1, a.beta2, a.beta3) = weight_decay[i], betas[i]
        a.eps1, a.eps2 = eps1[i], eps2[i]
        a.dtype, a.factored, a.fixed_decay = _GRAD_DTYPES[p.dtype], int(f), int(bool(fixed_decay[i]))
    need_d = ctypes.c_int64()
    check(lib().dpipe_came_scratch_doubles(arr, n, ctypes.byref(need_d)), 'dpipe_came_scratch_doubles')
    scratch = torch.empty(max(1, need_d.value), dtype=torch.float64, device=dev)
    nonempty = [p.ndim >= 2 for p in params if p.numel()]
    launches = sum(10 if any(nonempty[k:k + 64]) else 3 for k in range(0, len(nonempty), 64))
    return CameArgs(arr, list(params), (list(m), list(row), list(col), list(res_row), list(res_col), list(v)), fac,
                    sums, scratch, launches)


def came_step(args, grads, lrs, clip_threshold):
    """One CAME step (include/dpipe.h dpipe_came_step) over every tensor of `args` with this step's gradients and
    per-parameter learning rates: the state and the weights in place, no host synchronisation; the weights' version
    counters move."""
    global LAUNCHES
    args.set_step(grads, lrs)
    _e = _prof_begin()
    check(lib().dpipe_came_step(args.arr, args.n, float(clip_threshold), args.scratch.data_ptr(), args.scratch.numel(),
                                _stream()), 'dpipe_came_step')
    _prof_end(_e, 0.0, 'came_step')
    LAUNCHES += args.launches
    for p in args.params:           # as automagic_apply: caches keyed on the version see the new weights
        torch.autograd.graph.increment_version(p)


_A8_DTYPE = None


def _a8_dtype():
    global _A8_DTYPE
    if _A8_DTYPE is None:
        import numpy as np
        _A8_DTYPE = np.dtype(_abi.Adamw8bitTensor)
    return _A8_DTYPE


def adamw8bit_step(params, grads, state1, state2, absmax1, absmax2, scalars, qmap1=None, qmap2=None):
    """One AdamW8bit step (include/dpipe.h dpipe_adamw8bit_step) over parameter i with its gradient and state, in
    place: state1 / state2 fp32 m / v like the parameter with absmax1[i] = absmax2[i] = None, or uint8 codes like the
    parameter with fp32 absmax of ceil(numel / 256) blocks; scalars[i] the dict of oracle/adamw8bit_ref.py step_scalars
    (step_size, beta1, beta2, eps_c2, decay) for its group and step.  qmap1 / qmap2: the 256-entry fp32 maps of every
    8-bit tensor of the call.  Parameters and gradients are contiguous CUDA bf16 / fp32 tensors.  No host
    synchronisation; the weights' version counters move."""
    global LAUNCHES
    n = len(params)
    if any(len(x) != n for x in (grads, state1, state2, absmax1, absmax2, scalars)):
        raise ValueError('adamw8bit_step: the argument lists differ in length')

    def bad(what, i, t, want):
        got = 'None' if t is None else f'{t.dtype} {tuple(t.shape)} on {t.device}'
        return TypeError(f'adamw8bit_step: {what} {i} must be {want}, got {got}')
    q8 = False
    for i, p in enumerate(params):
        if p.dtype not in _GRAD_DTYPES:
            raise TypeError(f'adamw8bit_step: tensor {i} is {p.dtype}; the kernel takes bf16 or fp32 weights')
        if not p.is_cuda or not p.is_contiguous():
            raise bad('param', i, p, 'a contiguous CUDA tensor')
        g = grads[i]
        if g is None or g.dtype != p.dtype or g.shape != p.shape or g.device != p.device or not g.is_contiguous():
            raise bad('grad', i, g, f'a contiguous {p.dtype} tensor of shape {tuple(p.shape)} on {p.device}')
        a1, a2 = absmax1[i], absmax2[i]
        sdt = torch.float32 if a1 is None else torch.uint8
        for t, what in ((state1[i], 'state1'), (state2[i], 'state2')):
            if t is None or t.dtype != sdt or t.numel() != p.numel() or t.device != p.device or not t.is_contiguous():
                raise bad(what, i, t, f'a contiguous {sdt} tensor of {p.numel()} elements on {p.device}')
        if (a1 is None) != (a2 is None):
            raise TypeError(f'adamw8bit_step: tensor {i}: absmax1 and absmax2 are both given or both None')
        if a1 is not None:
            q8 = True
            nb = (p.numel() + 255) // 256
            for t, what in ((a1, 'absmax1'), (a2, 'absmax2')):
                if t.dtype != torch.float32 or t.numel() != nb or t.device != p.device or not t.is_contiguous():
                    raise bad(what, i, t, f'a contiguous fp32 tensor of {nb} elements on {p.device}')
    if q8:
        for t, what in ((qmap1, 'qmap1'), (qmap2, 'qmap2')):
            if t is None or t.dtype != torch.float32 or t.numel() != 256 or t.device != params[0].device \
                    or not t.is_contiguous():
                raise bad(what, 0, t, f'a contiguous fp32 tensor of 256 elements on {params[0].device}')
    if n == 0:
        return
    import numpy as np
    arr = np.zeros(n, dtype=_a8_dtype())
    for f, ts in (('p', params), ('g', grads), ('state1', state1), ('state2', state2), ('absmax1', absmax1),
                  ('absmax2', absmax2)):
        arr[f] = [0 if t is None else t.data_ptr() for t in ts]
    arr['numel'] = [p.numel() for p in params]
    for f in ('step_size', 'beta1', 'beta2', 'eps_c2', 'decay'):
        arr[f] = [s[f] for s in scalars]
    arr['dtype'] = [_GRAD_DTYPES[p.dtype] for p in params]
    _e = _prof_begin()
    check(lib().dpipe_adamw8bit_step(arr.ctypes.data, n, qmap1.data_ptr() if q8 else None,
                                     qmap2.data_ptr() if q8 else None, _stream()), 'dpipe_adamw8bit_step')
    _prof_end(_e, 0.0, 'adamw8bit_step')
    LAUNCHES += (sum(1 for p in params if p.numel()) + 63) // 64
    for p in params:                # as automagic_apply: caches keyed on the version see the new weights
        torch.autograd.graph.increment_version(p)


def noise_pack(x1, x0, t, pack):
    """(x_t, target) = ((1-t) x1 + t x0, x0 - x1) on the device, fp32, bit-identical to the separate host ops; x1/x0 any
    [bs, ...] shape; pack=True ([bs, c, h, w]) writes diffusers' 2x2-packed [bs, (h/2)(w/2), 4c] layout."""
    global LAUNCHES
    for a, n in ((x1, 'x1'), (x0, 'x0'), (t, 't')):
        _req_f32(a, n)
    assert x1.shape == x0.shape and x1.dim() >= 2 and t.numel() == x1.shape[0]
    bs = x1.shape[0]
    if pack:
        assert x1.dim() == 4, 'packing takes [bs, c, h, w] latents'
        c, frames, h, w = x1.shape[1], 1, x1.shape[2], x1.shape[3]
        shape = (bs, (h // 2) * (w // 2), 4 * c)
    else:
        c, frames, h, w = 1, 1, 1, x1.numel() // bs
        shape = tuple(x1.shape)
    xt = torch.empty(shape, dtype=torch.float32, device=x1.device)
    target = torch.empty(shape, dtype=torch.float32, device=x1.device)
    check(lib().dpipe_noise_pack(_ptr(x1), _ptr(x0), _ptr(t), _ptr(xt), _ptr(target), bs, c, frames, h, w, int(bool(pack)),
                                 _stream()), 'dpipe_noise_pack')
    LAUNCHES += 1
    return xt, target


def noise_on_device(x1, x0, t, pack, device):
    """`device_prepare_inputs`: the clean latents, the noise and the timesteps drawn on the host (same RNG stream and order
    as the reference's prepare_inputs) go to the device through pinned memory, asynchronously; the flow-matching mix, the
    target and the packing run there in one kernel.  Returns device tensors with the host path's bits."""
    def up(a):
        a = a.float().contiguous()
        if a.device.type == 'cpu':
            a = a.pin_memory() if not a.is_pinned() else a
        return a.to(device, non_blocking=True)
    return noise_pack(up(x1), up(x0), up(t), pack)
