"""Flux transformer blocks on the sm_90a kernels.

Each block is ONE torch.autograd.Function whose forward and backward are sequences of C-ABI kernel launches
(ops.py): wgmma GEMMs with fused epilogues, the fused attention kernels and the HBM-bound LayerNorm /
modulation / gate kernels.  Nothing here computes with torch ops except [batch, D]-sized vector glue
(SiLU of the timestep embedding, dtype casts of reduced gradients) and tensor allocation.

Parameter names follow diffusers' FluxTransformerBlock / FluxSingleTransformerBlock (the classes the reference wraps
at models/flux.py:490-533), so `p.original_name`, checkpoints and optimizers see the same model.  Projections that the
kernels consume as one matrix (q,k,v[,proj_mlp]) are allocated fused and exposed through per-projection *views*.

The arithmetic (including where bf16 roundings happen under the reference's autocast) is the one restated in
oracle/flux_ref.py; tests/test_flux_blocks_gpu.py checks both directions against it.

Memory policy (H100, 80 GB): no activation recompute at all — a block saves its bf16 intermediates, including the
LayerNorm+modulation outputs that feed its GEMMs (~0.54 GB per block per sample at 1024^2; round 1 recomputed those two
HBM passes per stream in backward: 1.5 % of the step for 2 GB per sample).
"""
import torch
from torch import nn

from . import ops

HD = 128  # head dim


def _silu_bf16(temb):
    # reference: nn.SiLU on the bf16 conditioning vector inside AdaLayerNormZero (bf16 in, bf16 out)
    return torch.nn.functional.silu(temb.float()).to(torch.bfloat16)


class _Lin(nn.Module):
    """weight/bias holder named like an nn.Linear (parameters may be views of a fused allocation)."""

    def __init__(self, weight, bias):
        super().__init__()
        self.weight = weight
        self.bias = bias


class FusedParam:
    """One contiguous (weight, bias) allocation exposed as several row-slices (diffusers' separate projections).
    Gradients are produced into one contiguous buffer whose slices are the views' .grad."""

    def __init__(self, out_features_list, in_features, dtype, device, std=0.02):
        total = sum(out_features_list)
        self.weight = torch.empty(total, in_features, dtype=dtype, device=device).normal_(0, std)
        self.bias = torch.zeros(total, dtype=dtype, device=device)
        self.w_views, self.b_views = [], []
        r = 0
        for n in out_features_list:
            self.w_views.append(nn.Parameter(self.weight[r:r + n]))
            self.b_views.append(nn.Parameter(self.bias[r:r + n]))
            r += n
        self.sizes = list(out_features_list)
        self.wgrad = None
        self.bgrad = None

    def lin(self, i):
        return _Lin(self.w_views[i], self.b_views[i])

    def _views_ok(self):
        """True if the per-projection parameters still alias the fused storage (e.g. not after a .to())."""
        return self.w_views[0].data_ptr() == self.weight.data_ptr()

    def grads(self):
        """Returns (wgrad, bgrad, accumulate).  accumulate=False means the buffers hold no gradient yet (first
        micro-batch after zero_grad(set_to_none=True)) and the kernels may overwrite them."""
        if self.wgrad is None:
            self.wgrad = torch.empty_like(self.weight)
            self.bgrad = torch.empty_like(self.bias)
        fresh = any(p.grad is None or p.grad.data_ptr() != self._slice_ptr(i)
                    for i, p in enumerate(self.w_views))
        if fresh:
            r = 0
            for i, n in enumerate(self.sizes):
                self.w_views[i].grad = self.wgrad[r:r + n]
                self.b_views[i].grad = self.bgrad[r:r + n]
                r += n
        return self.wgrad, self.bgrad, not fresh

    def _slice_ptr(self, i):
        return self.wgrad.data_ptr() + sum(self.sizes[:i]) * self.wgrad.stride(0) * self.wgrad.element_size()

    def requires_grad(self):
        return any(p.requires_grad for p in self.w_views)


def _plain(out_f, in_f, dtype, device, std=0.02):
    return _Lin(nn.Parameter(torch.empty(out_f, in_f, dtype=dtype, device=device).normal_(0, std)),
                nn.Parameter(torch.zeros(out_f, dtype=dtype, device=device)))


def _grad_buf(p):
    """(.grad buffer, accumulate) for a plain parameter."""
    if p.grad is None:
        p.grad = torch.empty_like(p)
        return p.grad, False
    return p.grad, True


def _acc_vec(p, g32):
    """p.grad (+)= g32 (fp32 reduced vector) for bias / norm-weight parameters."""
    if not p.requires_grad:
        return
    if p.grad is None:
        p.grad = g32.to(p.dtype).view_as(p)
    else:
        p.grad.add_(g32.view_as(p))


def _acc_fused_bias(fp, bgrad, acc, g32):
    if acc:
        bgrad.add_(g32)
    else:
        bgrad.copy_(g32)


# =====================================================================================================================
# modulation linear: mod[B, n*D] = silu(temb) @ W^T + b      (AdaLayerNormZero{,Single}.linear)
# =====================================================================================================================
def _mod_fwd(temb, lin):
    """mod = Linear(SiLU(temb)) on the rank-batch kernel (csrc/modulation.cu)."""
    return ops.mod_fwd(temb if temb.is_contiguous() else temb.contiguous(), lin.weight, lin.bias)


def _mod_bwd(dmod32, temb, lin, d_temb32):
    """dmod32: fp32 [B, n*D] gradient of the modulation vector; accumulates d temb into d_temb32 (fp32 [B, D])."""
    wg, acc = (None, False)
    if lin.weight.requires_grad:
        wg, acc = _grad_buf(lin.weight)
    dbias = ops.mod_bwd(dmod32, temb if temb.is_contiguous() else temb.contiguous(), lin.weight, wg, acc, d_temb32)
    if lin.weight.requires_grad:
        _acc_vec(lin.bias, dbias)


# =====================================================================================================================
# double-stream block
# =====================================================================================================================
def _valid_rows(n_txt, Lt, Ltot, device):
    """rows of the joint [text; image] sequence that exist for a sample with n_txt real prompt tokens"""
    return torch.cat([torch.arange(n_txt, device=device), torch.arange(Lt, Ltot, device=device)])


def _ragged_attn_fwd(q, k, v, Lt, txt_lens):
    """Joint attention for a micro-batch whose prompts have different lengths (key-padding mask of
    models/qwen_image.py:472-476): every sample attends over its own valid rows only — gathered into a dense
    [1, H, L_b, 128] problem for the same kernels.  Padded text rows are neither keys nor (meaningful) queries; their
    output is zero, which no loss term can see (they are masked out of the keys of every later block)."""
    B, H, Ltot, _ = q.shape
    o = torch.zeros((B * Ltot, H * HD), dtype=q.dtype, device=q.device)
    o3 = o.view(B, Ltot, H * HD)
    saved = []
    for b, n in enumerate(txt_lens):
        idx = _valid_rows(int(n), Lt, Ltot, q.device)
        qb, kb, vb = (t[b:b + 1].index_select(2, idx) for t in (q, k, v))
        ob, lse_b = ops.attn_fwd(qb, kb, vb)
        o3[b].index_copy_(0, idx, ob)
        saved.append((idx, qb, kb, vb, ob, lse_b))
    return o, saved


def _ragged_attn_bwd(saved, d_o, shape):
    B, H, Ltot, _ = shape
    d_o3 = d_o.view(B, Ltot, H * HD)
    dq, dk, dv = (torch.zeros(shape, dtype=d_o.dtype, device=d_o.device) for _ in range(3))
    for b, (idx, qb, kb, vb, ob, lse_b) in enumerate(saved):
        dqb, dkb, dvb = ops.attn_bwd(qb, kb, vb, ob, d_o3[b].index_select(0, idx), lse_b)
        dq[b].index_copy_(1, idx, dqb[0])
        dk[b].index_copy_(1, idx, dkb[0])
        dv[b].index_copy_(1, idx, dvb[0])
    return dq, dk, dv


class _Stream:
    """Per-stream (image or text) state saved by the double block forward."""
    __slots__ = ('x', 'mod', 'mean1', 'rstd1', 'xn', 'y_attn', 'x1', 'mean2', 'rstd2', 'xn2', 'u', 'h', 'y_mlp', 'L', 'off')


class FluxDoubleBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin, txt_lens=None):
        """txt_lens: None (every text row is a real token) or one prompt length per sample (Qwen-Image key mask)"""
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        Ltot = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        shp = (B, H, Ltot, HD)
        q = torch.empty(shp, dtype=bf, device=dev)
        k = torch.empty(shp, dtype=bf, device=dev)
        v = torch.empty(shp, dtype=bf, device=dev)
        qhat = torch.empty(shp, dtype=bf, device=dev)
        khat = torch.empty(shp, dtype=bf, device=dev)
        q_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        streams = []
        # (input, rows, seq offset, modulation linear, fused qkv, q/k norm weights)
        spec = ((hidden, Li, Lt, blk.norm1.linear, blk.qkv, blk.attn.norm_q, blk.attn.norm_k),
                (enc, Lt, 0, blk.norm1_context.linear, blk.add_qkv, blk.attn.norm_added_q, blk.attn.norm_added_k))
        for x3, L, off, modlin, fq, nq, nk in spec:
            st = _Stream()
            st.L, st.off = L, off
            st.x = x3.reshape(B * L, D)
            st.mod = _mod_fwd(temb, modlin)                               # [B, 6D]: shift,scale,gate (msa), shift,scale,gate (mlp)
            m = st.mod
            xn, st.mean1, st.rstd1 = ops.ln_modulate_fwd(st.x, m[:, D:2 * D], m[:, 0:D], B, L)
            e = ops.make_qkv_epilogue(q, k, v, nq.weight, nk.weight, cos, sin, H, Ltot, off, qhat, khat, q_rstd, k_rstd)
            ops.gemm(xn, fq.weight, bias=fq.bias, epilogue=ops.EPI_QKV_ROPE, out=xn, rows_per_batch=L, qkv=e)   # (no token-major output: `out` is not written)
            st.xn = xn
            streams.append(st)
        if txt_lens is None:
            o, lse = ops.attn_fwd(q, k, v)                                # o: [B*Ltot, H*HD] token-major
        else:
            o, lse = _ragged_attn_fwd(q, k, v, Lt, txt_lens)              # lse: per-sample saved state
        ctx.ragged = txt_lens is not None
        o3 = o.view(B, Ltot, H * HD)
        outs = []
        tail = ((blk.attn.to_out[0], blk.ff), (blk.attn.to_add_out, blk.ff_context))
        for st, (wo, ff) in zip(streams, tail):
            L, off, m = st.L, st.off, st.mod
            st.y_attn = torch.empty((B * L, D), dtype=bf, device=dev)
            st.x1 = torch.empty((B * L, D), dtype=bf, device=dev)
            for b in range(B):                                            # rows of one sample are contiguous in o
                rs = slice(b * L, (b + 1) * L)
                ops.gemm(o3[b, off:off + L], wo.weight, bias=wo.bias, epilogue=ops.EPI_GATE_RES, aux=st.x[rs],
                         gate=m[b:b + 1, 2 * D:3 * D], out=st.x1[rs], out2=st.y_attn[rs], rows_per_batch=L)
            xn2, st.mean2, st.rstd2 = ops.ln_modulate_fwd(st.x1, m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L)
            st.xn2 = xn2
            w1, w2 = ff.net[0].proj, ff.net[2]
            st.u = torch.empty((B * L, w1.weight.shape[0]), dtype=bf, device=dev)
            st.h = ops.gemm(xn2, w1.weight, bias=w1.bias, epilogue=ops.EPI_BIAS_GELU, out2=st.u)
            st.y_mlp = torch.empty((B * L, D), dtype=bf, device=dev)
            x2 = ops.gemm(st.h, w2.weight, bias=w2.bias, epilogue=ops.EPI_GATE_RES, aux=st.x1,
                          gate=m[:, 5 * D:6 * D], out2=st.y_mlp, rows_per_batch=L)
            outs.append(x2.view(B, L, D))
        ctx.blk = blk
        ctx.streams = streams
        ctx.attn = (q, k, v, qhat, khat, q_rstd, k_rstd, o, lse)
        ctx.save_for_backward(temb, cos, sin)
        ctx.dims = (B, Li, Lt, D, H)
        return outs[0], outs[1]

    @staticmethod
    def backward(ctx, d_hidden, d_enc):
        blk = ctx.blk
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        Ltot = Li + Lt
        dev = temb.device
        bf = torch.bfloat16
        q, k, v, qhat, khat, q_rstd, k_rstd, o, lse = ctx.attn
        o3 = o.view(B, Ltot, H * HD)
        d_o = torch.empty((B * Ltot, H * HD), dtype=bf, device=dev)
        d_o3 = d_o.view(B, Ltot, H * HD)
        tail = ((blk.attn.to_out[0], blk.ff), (blk.attn.to_add_out, blk.ff_context))
        dmods, dx1s = [], []
        for st, (wo, ff), dxo in zip(ctx.streams, tail, (d_hidden, d_enc)):
            L, off, m = st.L, st.off, st.mod
            dx2 = dxo.reshape(B * L, D)
            if dx2.dtype != bf:
                dx2 = dx2.to(bf)
            dmod = torch.empty((B, 6 * D), dtype=torch.float32, device=dev)
            w1, w2 = ff.net[0].proj, ff.net[2]
            # ---- MLP branch: x2 = x1 + gate_mlp * (h W2^T + b2) ----
            dy2, part = ops.gate_bwd(dx2, st.y_mlp, m[:, 5 * D:6 * D], B, L)
            db2 = torch.empty(D, dtype=torch.float32, device=dev)
            ops.colreduce_finish(part, per_sample0=dmod[:, 5 * D:6 * D], summed1=db2)
            du = ops.gemm(dy2, w2.weight, b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=st.u)        # [BL, 4D]
            if w2.weight.requires_grad:
                def wgrad_w2(w2=w2, dy2=dy2, h=st.h, db2=db2):
                    g, acc = _grad_buf(w2.weight)
                    ops.gemm(dy2, h, a_mn=True, b_mn=True, out=g, accumulate=acc)                      # dW2 = dy2^T h
                    _acc_vec(w2.bias, db2)
                ops.defer(wgrad_w2)
            xn2 = st.xn2
            if w1.weight.requires_grad:
                db1 = ops.colsum(du)

                def wgrad_w1(w1=w1, du=du, xn2=xn2, db1=db1):
                    g, acc = _grad_buf(w1.weight)
                    ops.gemm(du, xn2, a_mn=True, b_mn=True, out=g, accumulate=acc)                     # dW1 = du^T xn2
                    _acc_vec(w1.bias, db1)
                ops.defer(wgrad_w1)
            # (the xn2 storage is recycled for the result unless a deferred weight-gradient still needs xn2)
            dxn2 = ops.gemm(du, w1.weight, b_mn=True, out=None if ops.deferring() else xn2)
            dx1, part = ops.ln_modulate_bwd(dxn2, st.x1, m[:, 4 * D:5 * D], st.mean2, st.rstd2, B, L, dres=dx2)
            ops.colreduce_finish(part, per_sample0=dmod[:, 4 * D:5 * D], per_sample1=dmod[:, 3 * D:4 * D])
            # ---- attention branch: x1 = x + gate_msa * (o W_o^T + b_o) ----
            dy1, part = ops.gate_bwd(dx1, st.y_attn, m[:, 2 * D:3 * D], B, L, dy=dxn2)
            dbo = torch.empty(D, dtype=torch.float32, device=dev)
            ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D], summed1=dbo)
            for b in range(B):
                rs = slice(b * L, (b + 1) * L)
                ops.gemm(dy1[rs], wo.weight, b_mn=True, out=d_o3[b, off:off + L])                      # d o (this stream's rows)
            if wo.weight.requires_grad:
                def wgrad_wo(wo=wo, dy1=dy1, o3=o3, dbo=dbo, L=L, off=off):
                    wg, acc = _grad_buf(wo.weight)
                    for b in range(B):
                        ops.gemm(dy1[b * L:(b + 1) * L], o3[b, off:off + L], a_mn=True, b_mn=True, out=wg,
                                 accumulate=acc or b > 0)                                              # dWo = dy1^T o
                    _acc_vec(wo.bias, dbo)
                ops.defer(wgrad_wo)
            dmods.append(dmod)
            dx1s.append(dx1)
        if ctx.ragged:
            dq, dk, dv = _ragged_attn_bwd(lse, d_o, q.shape)
        else:
            dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse)
        d_temb = torch.zeros_like(temb, dtype=torch.float32)
        grads = []
        spec = ((blk.norm1.linear, blk.qkv, blk.attn.norm_q, blk.attn.norm_k),
                (blk.norm1_context.linear, blk.add_qkv, blk.attn.norm_added_q, blk.attn.norm_added_k))
        for st, dmod, dx1, (modlin, fq, nq, nk) in zip(ctx.streams, dmods, dx1s, spec):
            L, off, m = st.L, st.off, st.mod
            dqkv = torch.empty((B * L, 3 * H * HD), dtype=bf, device=dev)
            dbias = torch.zeros(3 * H * HD, dtype=torch.float32, device=dev)
            dw = torch.zeros((2, HD), dtype=torch.float32, device=dev)
            ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, nq.weight, nk.weight, cos, sin, dqkv, dbias, dw,
                                B, H, Ltot, off, L)
            xn = st.xn
            if fq.requires_grad():
                def wgrad_qkv(fq=fq, nq=nq, nk=nk, dqkv=dqkv, xn=xn, dbias=dbias, dw=dw):
                    wgrad, bgrad, acc = fq.grads()
                    ops.gemm(dqkv, xn, a_mn=True, b_mn=True, out=wgrad, accumulate=acc)                # dWqkv = dqkv^T xn
                    _acc_fused_bias(fq, bgrad, acc, dbias)
                    _acc_vec(nq.weight, dw[0])
                    _acc_vec(nk.weight, dw[1])
                ops.defer(wgrad_qkv)
            dxn = ops.gemm(dqkv, fq.weight, b_mn=True, out=None if ops.deferring() else xn)
            dx, part = ops.ln_modulate_bwd(dxn, st.x, m[:, D:2 * D], st.mean1, st.rstd1, B, L, dres=dx1)
            ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
            _mod_bwd(dmod, temb, modlin, d_temb)
            grads.append(dx.view(B, L, D))
        ctx.streams = None
        ctx.attn = None
        return None, grads[0], grads[1], d_temb.to(temb.dtype), None, None, None


class _Attn(nn.Module):
    pass


class _FF(nn.Module):
    def __init__(self, dim, inner, dtype, device):
        super().__init__()
        g = nn.Module()
        g.proj = _plain(inner, dim, dtype, device)
        self.net = nn.ModuleList([g, nn.Identity(), _plain(dim, inner, dtype, device)])


class _AdaNorm(nn.Module):
    def __init__(self, dim, chunks, dtype, device):
        super().__init__()
        self.linear = _plain(chunks * dim, dim, dtype, device)


def _norm_w(dtype, device):
    m = nn.Module()
    m.weight = nn.Parameter(torch.ones(HD, dtype=dtype, device=device))
    return m


class FluxTransformerBlock(nn.Module):
    """Drop-in for diffusers.models.transformers.transformer_flux.FluxTransformerBlock (same parameter names and
    call signature as used at models/flux.py:502); returns (encoder_hidden_states, hidden_states)."""

    def __init__(self, dim=3072, heads=24, mlp_ratio=4, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        assert dim == heads * HD
        self.dim, self.heads = dim, heads
        self.norm1 = _AdaNorm(dim, 6, dtype, device)
        self.norm1_context = _AdaNorm(dim, 6, dtype, device)
        self.qkv = FusedParam([dim] * 3, dim, dtype, device)
        self.add_qkv = FusedParam([dim] * 3, dim, dtype, device)
        a = _Attn()
        a.to_q, a.to_k, a.to_v = self.qkv.lin(0), self.qkv.lin(1), self.qkv.lin(2)
        a.add_q_proj, a.add_k_proj, a.add_v_proj = self.add_qkv.lin(0), self.add_qkv.lin(1), self.add_qkv.lin(2)
        a.norm_q, a.norm_k = _norm_w(dtype, device), _norm_w(dtype, device)
        a.norm_added_q, a.norm_added_k = _norm_w(dtype, device), _norm_w(dtype, device)
        a.to_out = nn.ModuleList([_plain(dim, dim, dtype, device), nn.Identity()])
        a.to_add_out = _plain(dim, dim, dtype, device)
        self.attn = a
        self.ff = _FF(dim, dim * mlp_ratio, dtype, device)
        self.ff_context = _FF(dim, dim * mlp_ratio, dtype, device)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, joint_attention_kwargs=None):
        cos, sin = image_rotary_emb
        if 'lora' in self.__dict__:          # adapters attached (lora.py): frozen base, K-extended GEMMs
            from .lora import FluxDoubleBlockLoraFn
            h, e = FluxDoubleBlockLoraFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin, None)
            return e, h
        h, e = FluxDoubleBlockFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin, None)
        return e, h


# =====================================================================================================================
# single-stream block
# =====================================================================================================================
def _joint(enc, hidden):
    """[enc; hidden] along the sequence.  The layer protocol hands the two streams over separately (models/flux.py:520-533),
    but between two single blocks they are the two halves of ONE buffer (the previous block's output / the next block's
    input gradient): then the joint tensor is a view, not a copy (batch 1: rows of the same [L, D] matrix)."""
    B, Lt, D = enc.shape
    Li = hidden.shape[1]
    if (B == 1 and enc.dtype == hidden.dtype and enc.is_contiguous() and hidden.is_contiguous()
            and enc.untyped_storage().data_ptr() == hidden.untyped_storage().data_ptr()
            and hidden.storage_offset() == enc.storage_offset() + Lt * D):
        return enc.as_strided((B, Lt + Li, D), ((Lt + Li) * D, D, 1))
    return torch.cat([enc, hidden], dim=1)


class FluxSingleBlockFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin):
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        L = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        x = _joint(enc, hidden).reshape(B * L, D)
        mod = _mod_fwd(temb, blk.norm.linear)                               # [B, 3D]: shift, scale, gate
        xn, mean, rstd = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], B, L)
        shp = (B, H, L, HD)
        q = torch.empty(shp, dtype=bf, device=dev)
        k = torch.empty(shp, dtype=bf, device=dev)
        v = torch.empty(shp, dtype=bf, device=dev)
        qhat = torch.empty(shp, dtype=bf, device=dev)
        khat = torch.empty(shp, dtype=bf, device=dev)
        q_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        inner = blk.mlp_dim
        cat = torch.empty((B * L, D + inner), dtype=bf, device=dev)      # [attn | gelu(mlp)]: the operand of proj_out
        u = torch.empty((B * L, inner), dtype=bf, device=dev)
        f1 = blk.lin1
        e = ops.make_qkv_epilogue(q, k, v, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos, sin, H, L, 0, qhat, khat,
                                  q_rstd, k_rstd)
        ops.gemm(xn, f1.weight, bias=f1.bias, epilogue=ops.EPI_QKV_ROPE, out=cat[:, D:], out2=u, rows_per_batch=L, qkv=e)
        _, lse = ops.attn_fwd(q, k, v, out=cat)
        y = torch.empty((B * L, D), dtype=bf, device=dev)
        po = blk.proj_out
        xo = ops.gemm(cat, po.weight, bias=po.bias, epilogue=ops.EPI_GATE_RES, aux=x, gate=mod[:, 2 * D:3 * D], out2=y,
                      rows_per_batch=L)
        xo3 = xo.view(B, L, D)
        ctx.blk = blk
        ctx.saved = (x, mod, mean, rstd, q, k, v, qhat, khat, q_rstd, k_rstd, cat, u, lse, y, xn)
        ctx.save_for_backward(temb, cos, sin)
        ctx.dims = (B, Li, Lt, D, H)
        return xo3[:, Lt:], xo3[:, :Lt]

    @staticmethod
    def backward(ctx, d_hidden, d_enc):
        blk = ctx.blk
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        L = Li + Lt
        dev = temb.device
        bf = torch.bfloat16
        x, mod, mean, rstd, q, k, v, qhat, khat, q_rstd, k_rstd, cat, u, lse, y, xn = ctx.saved
        inner = blk.mlp_dim
        dxo = _joint(d_enc, d_hidden).reshape(B * L, D)
        if dxo.dtype != bf:
            dxo = dxo.to(bf)
        dmod = torch.empty((B, 3 * D), dtype=torch.float32, device=dev)
        po, f1 = blk.proj_out, blk.lin1
        dy, part = ops.gate_bwd(dxo, y, mod[:, 2 * D:3 * D], B, L)
        dbo = torch.empty(D, dtype=torch.float32, device=dev)
        ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D], summed1=dbo)
        n1 = 3 * H * HD + inner
        dlin1 = torch.empty((B * L, n1), dtype=bf, device=dev)           # [dq | dk | dv | d mlp_pre]
        d_o = torch.empty((B * L, D), dtype=bf, device=dev)
        ops.gemm(dy, po.weight[:, :D], b_mn=True, out=d_o)                                              # d attn
        ops.gemm(dy, po.weight[:, D:], b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=u, out=dlin1[:, 3 * H * HD:])
        if po.weight.requires_grad:
            def wgrad_po(po=po, dy=dy, cat=cat, dbo=dbo):
                g, acc = _grad_buf(po.weight)
                ops.gemm(dy, cat, a_mn=True, b_mn=True, out=g, accumulate=acc)
                _acc_vec(po.bias, dbo)
            ops.defer(wgrad_po)
        dq, dk, dv = ops.attn_bwd(q, k, v, cat, d_o, lse)
        dbias = torch.zeros(n1, dtype=torch.float32, device=dev)
        dw = torch.zeros((2, HD), dtype=torch.float32, device=dev)
        ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos,
                            sin, dlin1, dbias[:3 * H * HD], dw, B, H, L, 0, L)
        if f1.requires_grad():
            ops.colsum(dlin1[:, 3 * H * HD:], out=dbias[3 * H * HD:])

            def wgrad_lin1(f1=f1, blk=blk, dlin1=dlin1, xn=xn, dbias=dbias, dw=dw):
                wgrad, bgrad, acc = f1.grads()
                ops.gemm(dlin1, xn, a_mn=True, b_mn=True, out=wgrad, accumulate=acc)
                _acc_fused_bias(f1, bgrad, acc, dbias)
                _acc_vec(blk.attn.norm_q.weight, dw[0])
                _acc_vec(blk.attn.norm_k.weight, dw[1])
            ops.defer(wgrad_lin1)
        dxn = ops.gemm(dlin1, f1.weight, b_mn=True, out=None if ops.deferring() else xn)
        dx, part = ops.ln_modulate_bwd(dxn, x, mod[:, D:2 * D], mean, rstd, B, L, dres=dxo)
        ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
        d_temb = torch.zeros((B, D), dtype=torch.float32, device=dev)
        _mod_bwd(dmod, temb, blk.norm.linear, d_temb)
        dx3 = dx.view(B, L, D)
        ctx.saved = None
        return None, dx3[:, Lt:], dx3[:, :Lt], d_temb.to(temb.dtype), None, None


class FluxSingleTransformerBlock(nn.Module):
    """Drop-in for diffusers' FluxSingleTransformerBlock (>=0.35 signature used at models/flux.py:525): takes and
    returns separate text / image streams."""

    def __init__(self, dim=3072, heads=24, mlp_ratio=4, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        assert dim == heads * HD
        self.dim, self.heads, self.mlp_dim = dim, heads, dim * mlp_ratio
        self.norm = _AdaNorm(dim, 3, dtype, device)
        self.lin1 = FusedParam([dim, dim, dim, self.mlp_dim], dim, dtype, device)   # rows [q; k; v; proj_mlp] (models/flux.py:66)
        a = _Attn()
        a.to_q, a.to_k, a.to_v = self.lin1.lin(0), self.lin1.lin(1), self.lin1.lin(2)
        a.norm_q, a.norm_k = _norm_w(dtype, device), _norm_w(dtype, device)
        self.attn = a
        self.proj_mlp = self.lin1.lin(3)
        self.proj_out = _plain(dim, dim + self.mlp_dim, dtype, device)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, joint_attention_kwargs=None):
        cos, sin = image_rotary_emb
        if 'lora' in self.__dict__:
            from .lora import FluxSingleBlockLoraFn
            h, e = FluxSingleBlockLoraFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin)
            return e, h
        h, e = FluxSingleBlockFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin)
        return e, h
