"""Flux transformer blocks on the sm_90a kernels.

Each block is ONE torch.autograd.Function whose forward and backward are sequences of C-ABI kernel launches
(ops.py): wgmma GEMMs with fused epilogues, the fused attention kernels and the HBM-bound LayerNorm /
modulation / gate kernels.  Nothing here computes with torch ops except [batch, D]-sized vector glue
(SiLU of the timestep embedding, dtype casts of reduced gradients) and tensor allocation.

Parameter names follow diffusers' FluxTransformerBlock / FluxSingleTransformerBlock (the classes the reference wraps
at models/flux.py:490-533), so `p.original_name`, checkpoints and optimizers see the same model.  Projections that the
kernels consume as one matrix (q,k,v[,proj_mlp]) are allocated fused and exposed through per-projection *views*.

**GEMM sites.**  The block functions never touch a linear's weight directly: they read the block's `sites`, one object
per GEMM (`DenseSite` here, `lora.LoraSite` once adapters are attached) and one per modulation linear (`DenseMod` /
`lora.ModLora`).  A dense site is the LoRA site's interface with R = 0 adapter columns: the same operands, buffers and
weight-gradient queueing, so one function serves dense and LoRA training and the two never drift apart.  The sites
also hold the policy for the LayerNorm+modulation outputs that feed a GEMM (`keep` / `rebuild`, see DESIGN.md §3).

The arithmetic (including where bf16 roundings happen under the reference's autocast) is the one restated in
oracle/flux_ref.py; tests/test_flux_blocks_gpu.py checks both directions against it.

Memory policy (H100, 80 GB): dense training recomputes nothing — a block saves its bf16 intermediates, including the
LayerNorm+modulation outputs that feed its GEMMs (~0.54 GB per block per sample at 1024^2; round 1 recomputed those two
HBM passes per stream in backward: 1.5 % of the step for 2 GB per sample).  With adapters only their R columns are
kept and the LayerNorm is recomputed in backward (lora.py).
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


def _defer_acc(*pairs):
    """queues p.grad (+)= g32 for the (vector parameter, fp32 gradient) pairs whose parameter is trained"""
    pairs = [(p, g) for p, g in pairs if p.requires_grad]
    if pairs:
        ops.defer(lambda: [_acc_vec(p, g) for p, g in pairs])


# =====================================================================================================================
# GEMM sites without an adapter (the R = 0 form of lora.LoraSite)
# =====================================================================================================================
class DenseSite:
    """One GEMM `y = x W^T + b` of a block over a `_Lin` or a `FusedParam`.  Operands are the weight itself, activation
    buffers are plain `[rows, K]` / `[rows, N]`, and the weight gradient dW (+)= dy^T x plus the bias gradient are queued
    when the weight is trained."""
    R = 0

    def __init__(self, lin):
        self.lin = lin

    @property
    def w_fwd(self):
        return self.lin.weight

    w_dgrad = w_fwd

    @property
    def bias(self):
        return self.lin.bias

    @property
    def K(self):
        return self.lin.weight.shape[1]

    @property
    def N(self):
        return self.lin.weight.shape[0]

    @property
    def bias_grad(self):
        """True when queue_grads also needs the fp32 bias gradient (i.e. the site's weight is trained)"""
        lin = self.lin
        return lin.requires_grad() if isinstance(lin, FusedParam) else lin.weight.requires_grad

    def refresh(self):
        pass

    def alloc_in(self, rows, device):
        return torch.empty((rows, self.K), dtype=torch.bfloat16, device=device)

    def alloc_dy(self, rows, device, spare=None):
        """[rows, N] dy buffer; `spare`, a dead [rows, N] buffer of the caller, is used instead of a new one"""
        return torch.empty((rows, self.N), dtype=torch.bfloat16, device=device) if spare is None else spare

    def input_operand(self, x):
        return x

    def project(self, xa):
        pass

    def backproject(self, dya):
        pass

    def keep(self, xa, recompute=False):
        """what backward keeps of the LayerNorm output `xa` feeding this site: the buffer itself, or nothing when the
        caller recomputes it (Wan: its storage is recycled in forward)"""
        return None if recompute else xa

    def spare(self, xa):
        """xa's storage for the caller to reuse as a [rows, K] output once xa is dead"""
        return xa

    def rebuild(self, kept, rows, device, ln):
        """the input operand again in backward; `ln(out)` recomputes the LayerNorm into `out`"""
        if kept is not None:
            return kept
        xa = self.alloc_in(rows, device)
        ln(xa)
        return xa

    def dgrad_out(self, xa):
        """output buffer of the input-gradient GEMM: xa's storage, unless a deferred weight gradient still reads xa"""
        return None if ops.deferring() else xa

    def queue_grads(self, x, dy, db=None):
        """dW (+)= dy^T x and b (+)= db as deferred weight-gradient work.  x, dy may be lists of row blocks (one per
        sample): their products are accumulated into one gradient and the bias is added once."""
        if not self.bias_grad:
            return
        xs, dys = (x, dy) if isinstance(x, list) else ([x], [dy])

        def wgrad(lin=self.lin, xs=xs, dys=dys, db=db):
            fused = isinstance(lin, FusedParam)
            if fused:
                g, bg, acc = lin.grads()
            else:
                g, acc = _grad_buf(lin.weight)
            for i, (x, dy) in enumerate(zip(xs, dys)):
                ops.gemm(dy, x, a_mn=True, b_mn=True, out=g, accumulate=acc or i > 0)
            if not fused:
                _acc_vec(lin.bias, db)
            elif acc:
                bg.add_(db)
            else:
                bg.copy_(db)
        ops.defer(wgrad)


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


class DenseMod:
    """modulation linear without an adapter (the interface of lora.ModLora)"""

    def __init__(self, lin):
        self.lin = lin

    def refresh(self):
        pass

    def fwd(self, temb):
        return _mod_fwd(temb, self.lin), None

    def bwd(self, dmod32, temb, saved, d_temb32):
        _mod_bwd(dmod32, temb, self.lin, d_temb32)


def _refresh(sites):
    for s in sites.values():
        s.refresh()


# =====================================================================================================================
# double-stream block
# =====================================================================================================================
def _valid_rows(n_txt, Lt, Ltot, device):
    """rows of the joint [text; image] sequence that exist for a sample with n_txt real prompt tokens"""
    return torch.cat([torch.arange(n_txt, device=device), torch.arange(Lt, Ltot, device=device)])


def _ragged_attn_fwd(q, k, v, Lt, txt_lens, out):
    """Joint attention for a micro-batch whose prompts have different lengths (key-padding mask of
    models/qwen_image.py:472-476): every sample attends over its own valid rows only — gathered into a dense
    [1, H, L_b, 128] problem for the same kernels — and its output lands in the first H*128 columns of `out`
    [B*Ltot, >= H*128].  Padded text rows are neither keys nor (meaningful) queries; their output is zero, which no loss
    term can see (they are masked out of the keys of every later block)."""
    B, H, Ltot, _ = q.shape
    out[:, :H * HD].zero_()
    o3 = out.view(B, Ltot, out.shape[1])[:, :, :H * HD]
    saved = []
    for b, n in enumerate(txt_lens):
        idx = _valid_rows(int(n), Lt, Ltot, q.device)
        qb, kb, vb = (t[b:b + 1].index_select(2, idx) for t in (q, k, v))
        ob, lse_b = ops.attn_fwd(qb, kb, vb)
        o3[b].index_copy_(0, idx, ob)
        saved.append((idx, qb, kb, vb, ob, lse_b))
    return saved


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
    __slots__ = ('x', 'mod', 'mod_saved', 'mean1', 'rstd1', 'xn', 'y_attn', 'x1', 'mean2', 'rstd2', 'xn2', 'u', 'h',
                 'y_mlp', 'L', 'off')


class FluxDoubleBlockFn(torch.autograd.Function):
    """Flux / Qwen-Image double-stream block over `blk.sites` (keys: mod, mod_c, qkv, add_qkv, to_out, to_add_out, ff1,
    ff2, ffc1, ffc2; the *_c / add_* / ffc* sites serve the text stream)."""

    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin, txt_lens=None):
        """txt_lens: None (every text row is a real token) or one prompt length per sample (Qwen-Image key mask)"""
        S = blk.sites
        _refresh(S)
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        Ltot = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        shp = (B, H, Ltot, HD)
        q, k, v, qhat, khat = (torch.empty(shp, dtype=bf, device=dev) for _ in range(5))
        q_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        streams = []
        # (input, rows, seq offset, modulation, qkv site, q/k norm weights)
        spec = ((hidden, Li, Lt, S['mod'], S['qkv'], blk.attn.norm_q, blk.attn.norm_k),
                (enc, Lt, 0, S['mod_c'], S['add_qkv'], blk.attn.norm_added_q, blk.attn.norm_added_k))
        for x3, L, off, ml, sq, nq, nk in spec:
            st = _Stream()
            st.L, st.off = L, off
            st.x = x3.reshape(B * L, D)
            st.mod, st.mod_saved = ml.fwd(temb)                             # [B, 6D]: shift,scale,gate (msa), shift,scale,gate (mlp)
            m = st.mod
            xa = sq.alloc_in(B * L, dev)
            _, st.mean1, st.rstd1 = ops.ln_modulate_fwd(st.x, m[:, D:2 * D], m[:, 0:D], B, L, out=xa[:, :D])
            sq.project(xa)
            e = ops.make_qkv_epilogue(q, k, v, nq.weight, nk.weight, cos, sin, H, Ltot, off, qhat, khat, q_rstd, k_rstd)
            ops.gemm(xa, sq.w_fwd, bias=sq.bias, epilogue=ops.EPI_QKV_ROPE, out=xa, rows_per_batch=L, qkv=e)   # (no token-major output: `out` is not written)
            st.xn = sq.keep(xa)
            streams.append(st)
        so, sao = S['to_out'], S['to_add_out']
        assert so.R == sao.R
        oa = so.alloc_in(B * Ltot, dev)                                     # attention output (+ adapter columns), token-major
        if txt_lens is None:
            _, lse = ops.attn_fwd(q, k, v, out=oa)
        else:
            lse = _ragged_attn_fwd(q, k, v, Lt, txt_lens, oa)               # lse: per-sample saved state
        ctx.ragged = txt_lens is not None
        oa3 = oa.view(B, Ltot, oa.shape[1])
        outs = []
        tail = ((so, S['ff1'], S['ff2']), (sao, S['ffc1'], S['ffc2']))
        for st, (swo, s1, s2) in zip(streams, tail):
            L, off, m = st.L, st.off, st.mod
            st.y_attn = torch.empty((B * L, D), dtype=bf, device=dev)
            st.x1 = torch.empty((B * L, D), dtype=bf, device=dev)
            for b in range(B):                                              # rows of one sample are contiguous in o
                rs = slice(b * L, (b + 1) * L)
                rows = oa3[b, off:off + L]
                swo.project(rows)
                ops.gemm(rows, swo.w_fwd, bias=swo.bias, epilogue=ops.EPI_GATE_RES, aux=st.x[rs],
                         gate=m[b:b + 1, 2 * D:3 * D], out=st.x1[rs], out2=st.y_attn[rs], rows_per_batch=L)
            x2a = s1.alloc_in(B * L, dev)
            _, st.mean2, st.rstd2 = ops.ln_modulate_fwd(st.x1, m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L, out=x2a[:, :D])
            s1.project(x2a)
            st.xn2 = s1.keep(x2a)
            st.u = torch.empty((B * L, s1.N), dtype=bf, device=dev)
            st.h = s2.alloc_in(B * L, dev)
            ops.gemm(x2a, s1.w_fwd, bias=s1.bias, epilogue=ops.EPI_BIAS_GELU, out=st.h[:, :s1.N], out2=st.u)
            s2.project(st.h)
            st.y_mlp = torch.empty((B * L, D), dtype=bf, device=dev)
            x2 = ops.gemm(st.h, s2.w_fwd, bias=s2.bias, epilogue=ops.EPI_GATE_RES, aux=st.x1,
                          gate=m[:, 5 * D:6 * D], out2=st.y_mlp, rows_per_batch=L)
            outs.append(x2.view(B, L, D))
        ctx.blk = blk
        ctx.streams = streams
        ctx.attn = (q, k, v, qhat, khat, q_rstd, k_rstd, oa, lse)
        ctx.save_for_backward(temb, cos, sin)
        ctx.dims = (B, Li, Lt, D, H)
        return outs[0], outs[1]

    @staticmethod
    def backward(ctx, d_hidden, d_enc):
        blk = ctx.blk
        S = blk.sites
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        Ltot = Li + Lt
        C = H * HD
        dev = temb.device
        bf = torch.bfloat16
        f32 = torch.float32
        q, k, v, qhat, khat, q_rstd, k_rstd, oa, lse = ctx.attn
        oa3 = oa.view(B, Ltot, oa.shape[1])
        d_o = torch.empty((B * Ltot, C), dtype=bf, device=dev)
        d_o3 = d_o.view(B, Ltot, C)
        tail = ((S['to_out'], S['ff1'], S['ff2']), (S['to_add_out'], S['ffc1'], S['ffc2']))
        dmods, dx1s = [], []
        for st, (swo, s1, s2), dxo in zip(ctx.streams, tail, (d_hidden, d_enc)):
            L, off, m = st.L, st.off, st.mod
            dx2 = dxo.reshape(B * L, D)
            if dx2.dtype != bf:
                dx2 = dx2.to(bf)
            dmod = torch.empty((B, 6 * D), dtype=f32, device=dev)
            # ---- MLP branch: x2 = x1 + gate_mlp * (h W2^T + b2) ----
            dy2a = s2.alloc_dy(B * L, dev)
            _, part = ops.gate_bwd(dx2, st.y_mlp, m[:, 5 * D:6 * D], B, L, dy=dy2a[:, :D])
            db2 = torch.empty(D, dtype=f32, device=dev) if s2.bias_grad else None
            ops.colreduce_finish(part, per_sample0=dmod[:, 5 * D:6 * D], summed1=db2)
            s2.backproject(dy2a)
            dua = s1.alloc_dy(B * L, dev)
            ops.gemm(dy2a, s2.w_dgrad, b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=st.u, out=dua[:, :s1.N])   # [BL, 4D]
            s2.queue_grads(st.h, dy2a, db2)                                                                   # dW2 = dy2^T h
            s1.backproject(dua)
            x2a = s1.rebuild(st.xn2, B * L, dev, lambda out: ops.ln_modulate_fwd(
                st.x1, m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L, out=out, save_stats=False))
            s1.queue_grads(x2a, dua, ops.colsum(dua) if s1.bias_grad else None)                             # dW1 = du^T xn2
            dxn2 = ops.gemm(dua, s1.w_dgrad, b_mn=True, out=s1.dgrad_out(x2a))
            dx1, part = ops.ln_modulate_bwd(dxn2, st.x1, m[:, 4 * D:5 * D], st.mean2, st.rstd2, B, L, dres=dx2)
            ops.colreduce_finish(part, per_sample0=dmod[:, 4 * D:5 * D], per_sample1=dmod[:, 3 * D:4 * D])
            # ---- attention branch: x1 = x + gate_msa * (o W_o^T + b_o) ----
            dy1a = swo.alloc_dy(B * L, dev, spare=dxn2)
            _, part = ops.gate_bwd(dx1, st.y_attn, m[:, 2 * D:3 * D], B, L, dy=dy1a[:, :D])
            dbo = torch.empty(D, dtype=f32, device=dev) if swo.bias_grad else None
            ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D], summed1=dbo)
            swo.backproject(dy1a)
            for b in range(B):
                ops.gemm(dy1a[b * L:(b + 1) * L], swo.w_dgrad, b_mn=True, out=d_o3[b, off:off + L])       # d o (this stream's rows)
            swo.queue_grads([oa3[b, off:off + L] for b in range(B)], [dy1a[b * L:(b + 1) * L] for b in range(B)], dbo)
            dmods.append(dmod)
            dx1s.append(dx1)
        if ctx.ragged:
            dq, dk, dv = _ragged_attn_bwd(lse, d_o, q.shape)
        else:
            dq, dk, dv = ops.attn_bwd(q, k, v, oa, d_o, lse)
        d_temb = torch.zeros_like(temb, dtype=f32)
        grads = []
        spec = ((S['mod'], S['qkv'], blk.attn.norm_q, blk.attn.norm_k),
                (S['mod_c'], S['add_qkv'], blk.attn.norm_added_q, blk.attn.norm_added_k))
        for st, dmod, dx1, (ml, sq, nq, nk) in zip(ctx.streams, dmods, dx1s, spec):
            L, off, m = st.L, st.off, st.mod
            dqa = sq.alloc_dy(B * L, dev)
            dbias = torch.zeros(3 * C, dtype=f32, device=dev)
            dw = torch.zeros((2, HD), dtype=f32, device=dev)
            ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, nq.weight, nk.weight, cos, sin, dqa, dbias, dw,
                                B, H, Ltot, off, L)
            _defer_acc((nq.weight, dw[0]), (nk.weight, dw[1]))
            sq.backproject(dqa)
            xa = sq.rebuild(st.xn, B * L, dev, lambda out: ops.ln_modulate_fwd(
                st.x, m[:, D:2 * D], m[:, 0:D], B, L, out=out, save_stats=False))
            sq.queue_grads(xa, dqa, dbias)                                                                    # dWqkv = dqkv^T xn
            dxn = ops.gemm(dqa, sq.w_dgrad, b_mn=True, out=sq.dgrad_out(xa))
            dx, part = ops.ln_modulate_bwd(dxn, st.x, m[:, D:2 * D], st.mean1, st.rstd1, B, L, dres=dx1)
            ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
            ml.bwd(dmod, temb, st.mod_saved, d_temb)
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


def double_block_sites(mod, mod_c, qkv, add_qkv, attn, ff, ff_context):
    """the dense `sites` of a double-stream block (FluxDoubleBlockFn); lora.attach_double_block replaces them"""
    return {'mod': DenseMod(mod), 'mod_c': DenseMod(mod_c), 'qkv': DenseSite(qkv), 'add_qkv': DenseSite(add_qkv),
            'to_out': DenseSite(attn.to_out[0]), 'to_add_out': DenseSite(attn.to_add_out),
            'ff1': DenseSite(ff.net[0].proj), 'ff2': DenseSite(ff.net[2]),
            'ffc1': DenseSite(ff_context.net[0].proj), 'ffc2': DenseSite(ff_context.net[2])}


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
        self.sites = double_block_sites(self.norm1.linear, self.norm1_context.linear, self.qkv, self.add_qkv, a, self.ff,
                                        self.ff_context)

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, joint_attention_kwargs=None):
        cos, sin = image_rotary_emb
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
    """Flux single-stream block over `blk.sites` (keys: mod, lin1 = [q; k; v; proj_mlp], proj_out)."""

    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin):
        S = blk.sites
        _refresh(S)
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        L = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        s1, s2 = S['lin1'], S['proj_out']
        x = _joint(enc, hidden).reshape(B * L, D)
        mod, mod_saved = S['mod'].fwd(temb)                                 # [B, 3D]: shift, scale, gate
        xa = s1.alloc_in(B * L, dev)
        _, mean, rstd = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], B, L, out=xa[:, :D])
        s1.project(xa)
        xn = s1.keep(xa)
        shp = (B, H, L, HD)
        q, k, v, qhat, khat = (torch.empty(shp, dtype=bf, device=dev) for _ in range(5))
        q_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        inner = blk.mlp_dim
        cata = s2.alloc_in(B * L, dev)              # [attn | gelu(mlp) (| adapter columns)]: the operand of proj_out
        u = torch.empty((B * L, inner), dtype=bf, device=dev)
        e = ops.make_qkv_epilogue(q, k, v, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos, sin, H, L, 0, qhat, khat,
                                  q_rstd, k_rstd)
        ops.gemm(xa, s1.w_fwd, bias=s1.bias, epilogue=ops.EPI_QKV_ROPE, out=cata[:, D:D + inner], out2=u, rows_per_batch=L,
                 qkv=e)
        _, lse = ops.attn_fwd(q, k, v, out=cata)
        s2.project(cata)
        y = torch.empty((B * L, D), dtype=bf, device=dev)
        xo = ops.gemm(cata, s2.w_fwd, bias=s2.bias, epilogue=ops.EPI_GATE_RES, aux=x, gate=mod[:, 2 * D:3 * D], out2=y,
                      rows_per_batch=L)
        xo3 = xo.view(B, L, D)
        ctx.blk = blk
        ctx.saved = (x, mod, mod_saved, mean, rstd, xn, q, k, v, qhat, khat, q_rstd, k_rstd, cata, u, lse, y)
        ctx.save_for_backward(temb, cos, sin)
        ctx.dims = (B, Li, Lt, D, H)
        return xo3[:, Lt:], xo3[:, :Lt]

    @staticmethod
    def backward(ctx, d_hidden, d_enc):
        blk = ctx.blk
        S = blk.sites
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        L = Li + Lt
        C = H * HD
        dev = temb.device
        bf = torch.bfloat16
        f32 = torch.float32
        x, mod, mod_saved, mean, rstd, xn, q, k, v, qhat, khat, q_rstd, k_rstd, cata, u, lse, y = ctx.saved
        s1, s2 = S['lin1'], S['proj_out']
        inner = blk.mlp_dim
        dxo = _joint(d_enc, d_hidden).reshape(B * L, D)
        if dxo.dtype != bf:
            dxo = dxo.to(bf)
        dmod = torch.empty((B, 3 * D), dtype=f32, device=dev)
        dya = s2.alloc_dy(B * L, dev)
        _, part = ops.gate_bwd(dxo, y, mod[:, 2 * D:3 * D], B, L, dy=dya[:, :D])
        dbo = torch.empty(D, dtype=f32, device=dev) if s2.bias_grad else None
        ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D], summed1=dbo)
        s2.backproject(dya)
        dl1a = s1.alloc_dy(B * L, dev)                                   # [dq | dk | dv | d mlp_pre (| adapter columns)]
        d_o = torch.empty((B * L, D), dtype=bf, device=dev)
        wd = s2.w_dgrad                                                  # [D (+ R), D + inner]
        ops.gemm(dya, wd[:, :D], b_mn=True, out=d_o)                                                     # d attn
        ops.gemm(dya, wd[:, D:], b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=u, out=dl1a[:, 3 * C:3 * C + inner])
        s2.queue_grads(cata, dya, dbo)
        dq, dk, dv = ops.attn_bwd(q, k, v, cata, d_o, lse)
        dbias = torch.zeros(3 * C + inner, dtype=f32, device=dev)
        dw = torch.zeros((2, HD), dtype=f32, device=dev)
        ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos,
                            sin, dl1a, dbias[:3 * C], dw, B, H, L, 0, L)
        _defer_acc((blk.attn.norm_q.weight, dw[0]), (blk.attn.norm_k.weight, dw[1]))
        if s1.bias_grad:
            ops.colsum(dl1a[:, 3 * C:3 * C + inner], out=dbias[3 * C:])
        s1.backproject(dl1a)
        xa = s1.rebuild(xn, B * L, dev, lambda out: ops.ln_modulate_fwd(
            x, mod[:, D:2 * D], mod[:, 0:D], B, L, out=out, save_stats=False))
        s1.queue_grads(xa, dl1a, dbias)
        dxn = ops.gemm(dl1a, s1.w_dgrad, b_mn=True, out=s1.dgrad_out(xa))
        dx, part = ops.ln_modulate_bwd(dxn, x, mod[:, D:2 * D], mean, rstd, B, L, dres=dxo)
        ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
        d_temb = torch.zeros((B, D), dtype=f32, device=dev)
        S['mod'].bwd(dmod, temb, mod_saved, d_temb)
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
        self.sites = {'mod': DenseMod(self.norm.linear), 'lin1': DenseSite(self.lin1), 'proj_out': DenseSite(self.proj_out)}

    def forward(self, hidden_states, encoder_hidden_states, temb, image_rotary_emb, joint_attention_kwargs=None):
        cos, sin = image_rotary_emb
        h, e = FluxSingleBlockFn.apply(self, hidden_states, encoder_hidden_states, temb, cos, sin)
        return e, h
