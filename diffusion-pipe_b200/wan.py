"""Wan (t2v) on the sm_90a kernels — the drop-in for the reference's models/wan/wan.py + models/wan/model.py
(SURVEY.md rows W1-W3).

Same plugin surface as the reference's WanPipeline (models/wan/wan.py:67-411): `name`, `checkpointable_layers`,
`prepare_inputs(batch, timestep_quantile)`, `to_layers()`, `get_loss_fn()`, and layers that speak its tuple protocol
`(x, e, e0, seq_lens, grid_sizes, freqs, context)` (models/wan/wan.py:414-546).  Parameter names are the reference's
(`blocks.N.self_attn.q.weight`, `blocks.N.modulation`, `head.head.weight`, ...), so checkpoints and `original_name`
match.

A WanAttentionBlock (models/wan/model.py:242-318) is ONE torch.autograd.Function here: wgmma GEMMs with fused bias /
GELU / gated-residual epilogues, the fused attention kernels (self-attention over the video tokens with RoPE,
cross-attention over the 512 text slots), the LayerNorm+modulation kernels in their "bf16 after every op" mode (the
block's operands are all bf16 tensors in the reference) and the full-width RMSNorm+RoPE kernels of csrc/wan_norm.cu.
Like the Flux blocks it reads its GEMMs through `blk.sites` (flux_blocks.DenseSite, or lora.LoraSite once adapters are
attached), so dense and LoRA training run the same function.  Its three LayerNorm+modulation outputs are recomputed in
backward (DESIGN.md §3).
Scope: model_type 't2v' (Wan2.1 / Wan2.2 T2V) and 'i2v_v2' (Wan2.2 I2V: first-frame mask + conditioning latents as extra
input channels), both cross_attn_type 'default', with cached text embeddings; Wan2.1 i2v / flf2v (CLIP image context)
and ti2v (per-token timesteps) raise NotImplementedError.

Differences from the reference's tuple contents (internal to these layers): `freqs` travels as real fp32
`[2, L, 128]` (cos, sin of the per-token multipliers rope_apply builds from `grid_sizes`, models/wan/model.py:41-68)
instead of the complex64 `[1024, 64]` base table; all samples of a micro-batch must share one latent shape (the
reference's size-bucketed batches always do), so `seq_lens` masks nothing.
"""
import json
import math

import torch
from torch import nn

from . import ops
from .flux import linear, make_contiguous
from .flux_blocks import HD, DenseSite, FusedParam, _acc_vec, _defer_acc, _grad_buf, _mod_bwd, _mod_fwd, _plain, _refresh
from .plugin import PluginSurface

WAN_T2V_14B_CONFIG = {   # reference: models/wan/configs.py:60-75 (t2v_14B)
    'model_type': 't2v', 'dim': 5120, 'ffn_dim': 13824, 'num_heads': 40, 'num_layers': 40, 'in_dim': 16, 'out_dim': 16,
    'text_dim': 4096, 'text_len': 512, 'freq_dim': 256, 'patch_size': [1, 2, 2], 'eps': 1e-6,
}
WAN_T2V_1_3B_CONFIG = dict(WAN_T2V_14B_CONFIG, dim=1536, ffn_dim=8960, num_heads=12, num_layers=30)


# =====================================================================================================================
# small autograd pieces
# =====================================================================================================================
class SiluLinearFn(torch.autograd.Function):
    """Linear(SiLU(e)) on the rank-batch kernel (time_projection, models/wan/model.py:465)."""

    @staticmethod
    def forward(ctx, e, lin):
        shp = e.shape
        e2 = e.reshape(-1, shp[-1]).to(torch.bfloat16).contiguous()
        ctx.lin, ctx.shp, ctx.dtype = lin, shp, e.dtype
        ctx.save_for_backward(e2)
        return _mod_fwd(e2, lin).view(*shp[:-1], lin.weight.shape[0])

    @staticmethod
    def backward(ctx, dy):
        (e2,) = ctx.saved_tensors
        d = torch.zeros(e2.shape, dtype=torch.float32, device=e2.device)
        _mod_bwd(dy.reshape(e2.shape[0], -1).float().contiguous(), e2, ctx.lin, d)
        return d.to(ctx.dtype).view(ctx.shp), None


class PatchEmbedFn(torch.autograd.Function):
    """Conv3d with kernel == stride (models/wan/model.py:458-459) as a GEMM over unfolded patches; the parameter keeps
    the reference's 5-D shape, the kernels see it as [dim, C*pt*ph*pw]."""

    @staticmethod
    def forward(ctx, cols, conv):
        shp = cols.shape
        c2 = cols.reshape(-1, shp[-1]).to(torch.bfloat16).contiguous()
        dim = conv.weight.shape[0]
        y = ops.gemm(c2, conv.weight.view(dim, -1), bias=conv.bias)
        ctx.conv, ctx.shp, ctx.dtype = conv, shp, cols.dtype
        ctx.save_for_backward(c2)
        return y.view(*shp[:-1], dim)

    @staticmethod
    def backward(ctx, dy):
        conv = ctx.conv
        (c2,) = ctx.saved_tensors
        dim = conv.weight.shape[0]
        dy2 = dy.reshape(-1, dim)
        if dy2.dtype != torch.bfloat16:
            dy2 = dy2.to(torch.bfloat16)
        dy2 = dy2.contiguous()
        if conv.weight.requires_grad:
            def wgrad(conv=conv, dy2=dy2, c2=c2, dim=dim):
                g, acc = _grad_buf(conv.weight)
                ops.gemm(dy2, c2, a_mn=True, b_mn=True, out=g.view(dim, -1), accumulate=acc)
                _acc_vec(conv.bias, ops.colsum(dy2))
            ops.defer(wgrad)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = ops.gemm(dy2, conv.weight.view(dim, -1), b_mn=True).view(ctx.shp).to(ctx.dtype)
        return dx, None


class LnModFn(torch.autograd.Function):
    """out = LayerNorm(x) * (1 + scale[b]) + shift[b] with the reference's bf16 rounding after every op (Head,
    models/wan/model.py:338-343)."""

    @staticmethod
    def forward(ctx, x, scale, shift):
        B, L, D = x.shape
        x2 = x.reshape(B * L, D)
        scale, shift = scale.contiguous(), shift.contiguous()
        out, mean, rstd = ops.ln_modulate_fwd(x2, scale, shift, B, L, flags=ops.LN_ROUND_STEPS)
        ctx.save_for_backward(x2, scale, mean, rstd)
        ctx.dims = (B, L, D)
        return out.view(B, L, D)

    @staticmethod
    def backward(ctx, dout):
        x2, scale, mean, rstd = ctx.saved_tensors
        B, L, D = ctx.dims
        d2 = dout.reshape(B * L, D)
        if d2.dtype != torch.bfloat16:
            d2 = d2.to(torch.bfloat16)
        dx, part = ops.ln_modulate_bwd(d2.contiguous(), x2, scale, mean, rstd, B, L, flags=ops.LN_ROUND_STEPS)
        dmod = torch.empty((2, B, D), dtype=torch.float32, device=x2.device)
        ops.colreduce_finish(part, per_sample0=dmod[0], per_sample1=dmod[1])
        return dx.view(B, L, D), dmod[0].to(scale.dtype), dmod[1].to(scale.dtype)


# =====================================================================================================================
# the block
# =====================================================================================================================
class WanBlockFn(torch.autograd.Function):
    """Wan attention block over `blk.sites` (keys: sa_qkv, sa_o, ca_q, ca_kv, ca_o, ffn1, ffn2)."""

    @staticmethod
    def forward(ctx, blk, x, e0, context, cos, sin):
        S = blk.sites
        _refresh(S)
        B, L, D = x.shape
        Lc = context.shape[1]
        H = blk.num_heads
        dev = x.device
        bf = torch.bfloat16
        LN_STEPS, LN_MULT = ops.LN_ROUND_STEPS, ops.LN_MULT_DIRECT
        x2 = x.reshape(B * L, D)
        c2 = context.reshape(B * Lc, D)
        if c2.dtype != bf:
            c2 = c2.to(bf)
        mod = (blk.modulation.unsqueeze(0) + e0).reshape(B, 6, D)      # bf16 + bf16 -> bf16, as the reference (:298)
        sa, ca = blk.self_attn, blk.cross_attn
        s_qkv, s_o, s_cq, s_ckv, s_co, s_f1, s_f2 = (S[k] for k in ('sa_qkv', 'sa_o', 'ca_q', 'ca_kv', 'ca_o', 'ffn1', 'ffn2'))
        # the LayerNorm outputs that feed the sites are recomputed in backward (keep(recompute=True)); a dense site's
        # buffer is recycled as the output of the next residual GEMM (x1, x3)
        # ---- self-attention ----
        xa = s_qkv.alloc_in(B * L, dev)
        _, mean1, rstd1 = ops.ln_modulate_fwd(x2, mod[:, 1], mod[:, 0], B, L, eps=blk.eps, out=xa[:, :D], flags=LN_STEPS)
        s_qkv.project(xa)
        kept1 = s_qkv.keep(xa, recompute=True)
        qkv = ops.gemm(xa, s_qkv.w_fwd, bias=s_qkv.bias)
        (q, xhq, rq), (k, xhk, rk), (v, _, _) = ops.wan_norm_rope_fwd(
            [{'src': qkv[:, 0:D], 'weight': sa.norm_q.weight, 'rope': True},
             {'src': qkv[:, D:2 * D], 'weight': sa.norm_k.weight, 'rope': True},
             {'src': qkv[:, 2 * D:3 * D]}], B, L, H, cos, sin, eps=blk.eps)
        spare = s_qkv.spare(xa)
        del qkv, xa
        oa = s_o.alloc_in(B * L, dev)
        _, lse = ops.attn_fwd(q, k, v, out=oa)
        s_o.project(oa)
        y_attn = torch.empty((B * L, D), dtype=bf, device=dev)
        x1 = ops.gemm(oa, s_o.w_fwd, bias=s_o.bias, epilogue=ops.EPI_GATE_RES, aux=x2, gate=mod[:, 2], out2=y_attn,
                      rows_per_batch=L, out=spare)
        # ---- cross-attention (text context; all text_len slots attended: context_lens=None at models/wan/wan.py:526) ----
        n3w = blk.norm3.weight.view(1, D).expand(B, D)
        n3b = blk.norm3.bias.view(1, D).expand(B, D)
        x3a = s_cq.alloc_in(B * L, dev)
        _, mean3, rstd3 = ops.ln_modulate_fwd(x1, n3w, n3b, B, L, eps=blk.eps, out=x3a[:, :D], flags=LN_MULT)
        s_cq.project(x3a)
        kept3 = s_cq.keep(x3a, recompute=True)
        qc_lin = ops.gemm(x3a, s_cq.w_fwd, bias=s_cq.bias)
        ((qc, xhqc, rqc),) = ops.wan_norm_rope_fwd([{'src': qc_lin, 'weight': ca.norm_q.weight}], B, L, H, eps=blk.eps)
        del qc_lin, x3a
        ca_in = s_ckv.input_operand(c2)
        kv_lin = ops.gemm(ca_in, s_ckv.w_fwd, bias=s_ckv.bias)
        (kc, xhkc, rkc), (vc, _, _) = ops.wan_norm_rope_fwd(
            [{'src': kv_lin[:, 0:D], 'weight': ca.norm_k.weight}, {'src': kv_lin[:, D:2 * D]}], B, Lc, H, eps=blk.eps)
        del kv_lin
        oca = s_co.alloc_in(B * L, dev)
        _, lse_c = ops.attn_fwd(qc, kc, vc, out=oca)
        s_co.project(oca)
        x2_ = ops.gemm(oca, s_co.w_fwd, bias=s_co.bias, epilogue=ops.EPI_GATE_RES, aux=x1, gate=blk._ones(B, D, dev),
                       rows_per_batch=L)
        # ---- feed-forward ----
        x2a = s_f1.alloc_in(B * L, dev)
        _, mean2, rstd2 = ops.ln_modulate_fwd(x2_, mod[:, 4], mod[:, 3], B, L, eps=blk.eps, out=x2a[:, :D], flags=LN_STEPS)
        s_f1.project(x2a)
        kept2 = s_f1.keep(x2a, recompute=True)
        F = s_f1.N
        u = torch.empty((B * L, F), dtype=bf, device=dev)
        ha = s_f2.alloc_in(B * L, dev)
        ops.gemm(x2a, s_f1.w_fwd, bias=s_f1.bias, epilogue=ops.EPI_BIAS_GELU, out=ha[:, :F], out2=u)
        spare = s_f1.spare(x2a)
        del x2a
        s_f2.project(ha)
        y_mlp = torch.empty((B * L, D), dtype=bf, device=dev)
        x3 = ops.gemm(ha, s_f2.w_fwd, bias=s_f2.bias, epilogue=ops.EPI_GATE_RES, aux=x2_, gate=mod[:, 5], out2=y_mlp,
                      rows_per_batch=L, out=spare)
        ctx.blk = blk
        ctx.saved = (x2, c2, mod, mean1, rstd1, kept1, q, k, v, xhq, rq, xhk, rk, oa, lse, y_attn, x1, mean3, rstd3, kept3,
                     qc, xhqc, rqc, ca_in, kc, xhkc, rkc, vc, oca, lse_c, x2_, mean2, rstd2, kept2, u, ha, y_mlp)
        ctx.save_for_backward(cos, sin)
        ctx.dims = (B, L, Lc, D, H)
        ctx.in_dtypes = (x.dtype, e0.dtype, context.dtype)
        return x3.view(B, L, D)

    @staticmethod
    def backward(ctx, dx3):
        blk = ctx.blk
        S = blk.sites
        cos, sin = ctx.saved_tensors
        B, L, Lc, D, H = ctx.dims
        (x2, c2, mod, mean1, rstd1, kept1, q, k, v, xhq, rq, xhk, rk, oa, lse, y_attn, x1, mean3, rstd3, kept3,
         qc, xhqc, rqc, ca_in, kc, xhkc, rkc, vc, oca, lse_c, x2_, mean2, rstd2, kept2, u, ha, y_mlp) = ctx.saved
        ctx.saved = None
        dev = x2.device
        bf = torch.bfloat16
        f32 = torch.float32
        LN_STEPS, LN_MULT = ops.LN_ROUND_STEPS, ops.LN_MULT_DIRECT
        sa, ca = blk.self_attn, blk.cross_attn
        s_qkv, s_o, s_cq, s_ckv, s_co, s_f1, s_f2 = (S[k] for k in ('sa_qkv', 'sa_o', 'ca_q', 'ca_kv', 'ca_o', 'ffn1', 'ffn2'))
        F = s_f1.N
        dmod = torch.zeros((B, 6, D), dtype=f32, device=dev)
        d3 = dx3.reshape(B * L, D)
        if d3.dtype != bf:
            d3 = d3.to(bf)
        d3 = d3.contiguous()
        # ---- feed-forward: x3 = x2 + gate5 * (h W2^T + b2) ----
        dy2a = s_f2.alloc_dy(B * L, dev)
        _, part = ops.gate_bwd(d3, y_mlp, mod[:, 5], B, L, dy=dy2a[:, :D])
        db2 = torch.empty(D, dtype=f32, device=dev) if s_f2.bias_grad else None
        ops.colreduce_finish(part, per_sample0=dmod[:, 5], summed1=db2)
        s_f2.backproject(dy2a)
        dua = s_f1.alloc_dy(B * L, dev)
        ops.gemm(dy2a, s_f2.w_dgrad, b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=u, out=dua[:, :F])
        s_f2.queue_grads(ha, dy2a, db2)
        s_f1.backproject(dua)
        x2a = s_f1.rebuild(kept2, B * L, dev, lambda out: ops.ln_modulate_fwd(
            x2_, mod[:, 4], mod[:, 3], B, L, eps=blk.eps, out=out, save_stats=False, flags=LN_STEPS))
        s_f1.queue_grads(x2a, dua, ops.colsum(dua) if s_f1.bias_grad else None)
        dxn2 = ops.gemm(dua, s_f1.w_dgrad, b_mn=True, out=s_f1.dgrad_out(x2a))
        # d x2 lands directly in the dy operand of the cross-attention output projection (x2 = x1 + o_c W^T: no gate)
        dca = s_co.alloc_dy(B * L, dev)
        _, part = ops.ln_modulate_bwd(dxn2, x2_, mod[:, 4], mean2, rstd2, B, L, dres=d3, dx=dca[:, :D], flags=LN_STEPS)
        ops.colreduce_finish(part, per_sample0=dmod[:, 4], per_sample1=dmod[:, 3])
        dx2 = dca[:, :D]
        # ---- cross-attention: x2 = x1 + (oc Wo^T + bo) ----
        s_co.backproject(dca)
        d_oc = ops.gemm(dca, s_co.w_dgrad, b_mn=True)
        s_co.queue_grads(oca, dca, ops.colsum(dca) if s_co.bias_grad else None)
        dqc, dkc, dvc = ops.attn_bwd(qc, kc, vc, oca, d_oc, lse_c)
        dqca = s_cq.alloc_dy(B * L, dev)
        (dw_nqc,) = ops.wan_norm_rope_bwd([{'dy': dqc, 'dx': dqca[:, :D], 'weight': ca.norm_q.weight, 'xhat': xhqc, 'rstd': rqc}],
                                          B, L, H)
        s_cq.backproject(dqca)
        dkva = s_ckv.alloc_dy(B * Lc, dev)
        dw_nkc, _ = ops.wan_norm_rope_bwd([{'dy': dkc, 'dx': dkva[:, 0:D], 'weight': ca.norm_k.weight, 'xhat': xhkc, 'rstd': rkc},
                                           {'dy': dvc, 'dx': dkva[:, D:2 * D]}], B, Lc, H)
        s_ckv.backproject(dkva)
        n3w = blk.norm3.weight.view(1, D).expand(B, D)
        n3b = blk.norm3.bias.view(1, D).expand(B, D)
        x3a = s_cq.rebuild(kept3, B * L, dev, lambda out: ops.ln_modulate_fwd(
            x1, n3w, n3b, B, L, eps=blk.eps, out=out, save_stats=False, flags=LN_MULT))
        dbq_c = ops.colsum(dqca) if s_cq.bias_grad else None
        dbkv_c = ops.colsum(dkva) if s_ckv.bias_grad else None
        if ca_in is c2 and ops.deferring():
            # `context` arrives from the previous stage as a view of a stage-link mailbox slot, which is handed back
            # to the sender once this input-gradient pass has been enqueued: a weight-gradient closure that runs
            # later must own its copy (5 MB).  Nothing else a closure captures is a boundary tensor.
            ca_in = ca_in.clone()
        s_cq.queue_grads(x3a, dqca, dbq_c)
        s_ckv.queue_grads(ca_in, dkva, dbkv_c)
        _defer_acc((ca.norm_q.weight, dw_nqc), (ca.norm_k.weight, dw_nkc))
        d_ctx = ops.gemm(dkva, s_ckv.w_dgrad, b_mn=True)
        dxn3 = ops.gemm(dqca, s_cq.w_dgrad, b_mn=True, out=s_cq.dgrad_out(x3a))
        dx1, part = ops.ln_modulate_bwd(dxn3, x1, n3w, mean3, rstd3, B, L, dres=dx2, flags=LN_MULT)
        if blk.norm3.weight.requires_grad:
            dn3 = torch.empty((2, D), dtype=f32, device=dev)
            ops.colreduce_finish(part, summed0=dn3[0], summed1=dn3[1])
            _acc_vec(blk.norm3.weight, dn3[0])
            _acc_vec(blk.norm3.bias, dn3[1])
        # ---- self-attention: x1 = x + gate2 * (o Wo^T + bo) ----
        dy1a = s_o.alloc_dy(B * L, dev, spare=dxn3)
        _, part = ops.gate_bwd(dx1, y_attn, mod[:, 2], B, L, dy=dy1a[:, :D])
        dbo = torch.empty(D, dtype=f32, device=dev) if s_o.bias_grad else None
        ops.colreduce_finish(part, per_sample0=dmod[:, 2], summed1=dbo)
        s_o.backproject(dy1a)
        d_o = ops.gemm(dy1a, s_o.w_dgrad, b_mn=True)
        s_o.queue_grads(oa, dy1a, dbo)
        dq, dk, dv = ops.attn_bwd(q, k, v, oa, d_o, lse)
        dqkva = s_qkv.alloc_dy(B * L, dev)
        dw_nq, dw_nk, _ = ops.wan_norm_rope_bwd(
            [{'dy': dq, 'dx': dqkva[:, 0:D], 'weight': sa.norm_q.weight, 'xhat': xhq, 'rstd': rq, 'rope': True},
             {'dy': dk, 'dx': dqkva[:, D:2 * D], 'weight': sa.norm_k.weight, 'xhat': xhk, 'rstd': rk, 'rope': True},
             {'dy': dv, 'dx': dqkva[:, 2 * D:3 * D]}], B, L, H, cos, sin)
        _defer_acc((sa.norm_q.weight, dw_nq), (sa.norm_k.weight, dw_nk))
        s_qkv.backproject(dqkva)
        xa = s_qkv.rebuild(kept1, B * L, dev, lambda out: ops.ln_modulate_fwd(
            x2, mod[:, 1], mod[:, 0], B, L, eps=blk.eps, out=out, save_stats=False, flags=LN_STEPS))
        s_qkv.queue_grads(xa, dqkva, ops.colsum(dqkva) if s_qkv.bias_grad else None)
        dxn1 = ops.gemm(dqkva, s_qkv.w_dgrad, b_mn=True, out=s_qkv.dgrad_out(xa))
        dx, part = ops.ln_modulate_bwd(dxn1, x2, mod[:, 1], mean1, rstd1, B, L, dres=dx1, flags=LN_STEPS)
        ops.colreduce_finish(part, per_sample0=dmod[:, 1], per_sample1=dmod[:, 0])
        # ---- modulation: e = modulation + e0 ----
        if blk.modulation.requires_grad:
            _acc_vec(blk.modulation, dmod.sum(0))
        xdt, edt, cdt = ctx.in_dtypes
        return (None, dx.view(B, L, D).to(xdt), dmod.view(B, 1, 6, D).to(edt), d_ctx.view(B, Lc, D).to(cdt), None, None)


class _WanNormW(nn.Module):
    def __init__(self, dim, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype, device=device))


class _WanSelfAttn(nn.Module):
    """parameter holder named like WanSelfAttention (q, k, v, o, norm_q, norm_k); q/k/v share one fused allocation"""

    def __init__(self, dim, dtype, device):
        super().__init__()
        qkv = FusedParam([dim] * 3, dim, dtype, device)
        self.q, self.k, self.v = qkv.lin(0), qkv.lin(1), qkv.lin(2)
        self.o = _plain(dim, dim, dtype, device)
        self.norm_q, self.norm_k = _WanNormW(dim, dtype, device), _WanNormW(dim, dtype, device)
        self.__dict__['qkv'] = qkv


class _WanCrossAttn(nn.Module):
    """WanCrossAttention: q from the video tokens, k / v (one fused allocation) from the text context"""

    def __init__(self, dim, dtype, device):
        super().__init__()
        kv = FusedParam([dim] * 2, dim, dtype, device)
        self.q = _plain(dim, dim, dtype, device)
        self.k, self.v = kv.lin(0), kv.lin(1)
        self.o = _plain(dim, dim, dtype, device)
        self.norm_q, self.norm_k = _WanNormW(dim, dtype, device), _WanNormW(dim, dtype, device)
        self.__dict__['kv'] = kv


class _Affine(nn.Module):
    def __init__(self, dim, dtype, device):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(dim, dtype=dtype, device=device))


class WanAttentionBlock(nn.Module):
    """Drop-in for models/wan/model.py:242-318 (cross_attn_type 'default', qk_norm=True, cross_attn_norm=True)."""

    def __init__(self, dim=5120, ffn_dim=13824, num_heads=40, eps=1e-6, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        assert dim == num_heads * HD, 'kernels are specialised for head_dim 128'
        self.dim, self.ffn_dim, self.num_heads, self.eps = dim, ffn_dim, num_heads, eps
        self.self_attn = _WanSelfAttn(dim, dtype, device)
        self.norm3 = _Affine(dim, dtype, device)
        self.cross_attn = _WanCrossAttn(dim, dtype, device)
        self.ffn = nn.ModuleList([_plain(ffn_dim, dim, dtype, device), nn.Identity(), _plain(dim, ffn_dim, dtype, device)])
        self.modulation = nn.Parameter(torch.randn(1, 6, dim, device=device).to(dtype) / dim ** 0.5)
        self.__dict__['_ones_cache'] = {}
        sa, ca = self.self_attn, self.cross_attn
        self.sites = {'sa_qkv': DenseSite(sa.qkv), 'sa_o': DenseSite(sa.o), 'ca_q': DenseSite(ca.q), 'ca_kv': DenseSite(ca.kv),
                      'ca_o': DenseSite(ca.o), 'ffn1': DenseSite(self.ffn[0]), 'ffn2': DenseSite(self.ffn[2])}

    def _ones(self, B, D, device):
        key = (B, D, str(device))
        t = self._ones_cache.get(key)
        if t is None:
            t = self._ones_cache[key] = torch.ones((B, D), dtype=torch.bfloat16, device=device)
        return t

    def forward(self, x, e, seq_lens, grid_sizes, freqs, context, context_lens=None):
        assert context_lens is None, 'the reference passes context_lens=None (models/wan/wan.py:526)'
        return WanBlockFn.apply(self, x, e, context, freqs[0], freqs[1])


# =====================================================================================================================
# model + pipeline layers
# =====================================================================================================================
def sinusoidal_embedding_1d(dim, position):
    """models/wan/model.py:14-25."""
    half = dim // 2
    position = position.type(torch.float32)
    sinusoid = torch.outer(position, torch.pow(10000, -torch.arange(half, device=position.device).to(position).div(half)))
    return torch.cat([torch.cos(sinusoid), torch.sin(sinusoid)], dim=1)


def wan_rope_tables(grid, head_dim=HD, device=None, theta=10000):
    """the per-token multipliers rope_apply builds (models/wan/model.py:41-68, base table :478-484) as real fp32
    [2, f*h*w, head_dim]: cos and sin, every frequency repeated twice."""
    f, h, w = grid
    d, c = head_dim, head_dim // 2

    def angles(n, dim):
        return torch.outer(torch.arange(n, device=device),
                           1.0 / torch.pow(theta, torch.arange(0, dim, 2, device=device).to(torch.float32).div(dim)))
    af, ah, aw = angles(f, d - 4 * (d // 6)), angles(h, 2 * (d // 6)), angles(w, 2 * (d // 6))
    assert af.shape[1] == c - 2 * (c // 3) and ah.shape[1] == c // 3
    ang = torch.cat([af.view(f, 1, 1, -1).expand(f, h, w, -1), ah.view(1, h, 1, -1).expand(f, h, w, -1),
                     aw.view(1, 1, w, -1).expand(f, h, w, -1)], dim=-1).reshape(f * h * w, -1)
    return torch.stack([ang.cos().repeat_interleave(2, dim=1), ang.sin().repeat_interleave(2, dim=1)]).contiguous()


class _Seq(nn.ModuleList):
    """nn.Sequential-style indices (text_embedding.0 / .2, time_embedding.0 / .2, time_projection.1)."""


class WanHead(nn.Module):
    """models/wan/model.py:321-349: LN + modulation on bf16 tensors, then the projection under fp32 autocast."""

    def __init__(self, dim, out_dim, patch_size, eps, dtype, device):
        super().__init__()
        self.eps = eps
        self.head = _plain(math.prod(patch_size) * out_dim, dim, dtype, device)
        self.modulation = nn.Parameter(torch.randn(1, 2, dim, device=device).to(dtype) / dim ** 0.5)

    def forward(self, x, e):
        B, L, D = x.shape
        m = (self.modulation.unsqueeze(0) + e.unsqueeze(2)).reshape(B, 2, D)          # e: [B, 1, D]
        xm = LnModFn.apply(x, m[:, 1], m[:, 0])
        # fp32 autocast region of the reference: bf16 values, fp32 arithmetic and result (cuBLAS sgemm; 0.002% of the FLOPs)
        return torch.nn.functional.linear(xm.float(), self.head.weight.float(), self.head.bias.float())


class WanModel(nn.Module):
    """Parameter tree with the reference's names (models/wan/model.py:368-489, model_type 't2v')."""

    def __init__(self, cfg=None, dtype=torch.bfloat16, device='cuda'):
        super().__init__()
        cfg = dict(WAN_T2V_14B_CONFIG, **(cfg or {}))
        if cfg['model_type'] not in ('t2v', 'i2v_v2'):
            raise NotImplementedError(f"Wan model_type {cfg['model_type']!r}: 't2v' and 'i2v_v2' (Wan2.2 I2V) run on the sm_90a path")
        if cfg['model_type'] == 'i2v_v2' and cfg['in_dim'] == 16:
            cfg['in_dim'] = 36           # models/wan/configs.py (i2v_A14B): x + mask + y channels
        self.config = cfg
        dim = cfg['dim']
        self.dim, self.num_heads, self.freq_dim, self.text_len = dim, cfg['num_heads'], cfg['freq_dim'], cfg['text_len']
        self.patch_size, self.out_dim, self.in_dim = tuple(cfg['patch_size']), cfg['out_dim'], cfg['in_dim']
        assert dim // self.num_heads == HD, 'kernels are specialised for head_dim 128'
        assert self.patch_size[0] == 1, 'patchify as a GEMM assumes temporal patch 1'
        self.patch_embedding = nn.Module()
        self.patch_embedding.weight = nn.Parameter(torch.empty(dim, self.in_dim, *self.patch_size, dtype=dtype, device=device).normal_(0, 0.02))
        self.patch_embedding.bias = nn.Parameter(torch.zeros(dim, dtype=dtype, device=device))
        self.text_embedding = _Seq([_plain(dim, cfg['text_dim'], dtype, device), nn.Identity(), _plain(dim, dim, dtype, device)])
        self.time_embedding = _Seq([_plain(dim, self.freq_dim, dtype, device), nn.Identity(), _plain(dim, dim, dtype, device)])
        self.time_projection = _Seq([nn.Identity(), _plain(dim * 6, dim, dtype, device)])
        self.blocks = nn.ModuleList([WanAttentionBlock(dim, cfg['ffn_dim'], self.num_heads, cfg['eps'], dtype, device)
                                     for _ in range(cfg['num_layers'])])
        self.head = WanHead(dim, self.out_dim, self.patch_size, cfg['eps'], dtype, device)
        for name, p in self.named_parameters():
            p.original_name = name


def unpatchify(x, grid, patch_size, out_dim):
    """models/wan/model.py:492-517 for a batch whose samples share one grid: [B, L, prod(patch)*C] -> [B, C, F, H, W]."""
    B = x.shape[0]
    f, h, w = grid
    pt, ph, pw = patch_size
    u = x[:, :f * h * w].view(B, f, h, w, pt, ph, pw, out_dim)
    u = torch.einsum('bfhwpqrc->bcfphqwr', u)
    return u.reshape(B, out_dim, f * pt, h * ph, w * pw)


class InitialLayer(nn.Module):
    """models/wan/wan.py:414-511 (t2v, cached text embeddings)."""

    def __init__(self, patch_embedding, time_embedding, text_embedding, time_projection, cfg):
        super().__init__()
        self.patch_embedding, self.time_embedding = patch_embedding, time_embedding
        self.text_embedding, self.time_projection = text_embedding, time_projection
        self.dim, self.num_heads, self.freq_dim, self.text_len = cfg['dim'], cfg['num_heads'], cfg['freq_dim'], cfg['text_len']
        self.patch_size = tuple(cfg['patch_size'])
        self.model_type = cfg.get('model_type', 't2v')

    def forward(self, inputs):
        for item in inputs:
            if torch.is_floating_point(item) and item.numel() > 0:
                item.requires_grad_(True)
        x, y, t, text_embeddings, text_seq_lens, clip_fea = inputs
        if clip_fea.numel() > 0 or (y.numel() > 0) != (self.model_type == 'i2v_v2'):
            raise NotImplementedError('Wan2.1 i2v / flf2v conditioning (CLIP image context) is not on the sm_90a path; '
                                      "model_type 'i2v_v2' expects `y`, 't2v' must not get it")
        if torch.is_floating_point(text_seq_lens) or not torch.is_floating_point(text_embeddings):
            raise NotImplementedError('uncached text encoder (token ids in the pipeline tuple) is not supported: cache_text_embeddings must be true')
        if self.model_type == 'i2v_v2':
            # Wan2.2 I2V (models/wan/wan.py:459-465): first-frame mask (4 channels, 1 on frame 0) and the conditioning
            # latents y ride as extra input channels of the patch embedding: [x | mask | y] = 16 + 4 + 16
            bs_, _, f_, h_, w_ = x.shape
            fmask = torch.zeros((bs_, 4, f_, h_, w_), device=x.device, dtype=x.dtype)
            fmask[:, :, 0, ...] = 1
            x = torch.cat([x, fmask, y.to(x.dtype)], dim=1)
        bs, c, f, h, w = x.shape
        pt, ph, pw = self.patch_size
        dev = x.device
        # patch_embedding: Conv3d with kernel == stride == (1, 2, 2)  ==  a GEMM over unfolded patches (K = c*pt*ph*pw)
        cols = x.view(bs, c, f // pt, pt, h // ph, ph, w // pw, pw).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(bs, -1, c * pt * ph * pw)
        xe = PatchEmbedFn.apply(cols, self.patch_embedding)                       # [bs, L, dim] bf16
        grid = (f // pt, h // ph, w // pw)
        L = grid[0] * grid[1] * grid[2]
        grid_sizes = torch.tensor([grid] * bs, dtype=torch.long, device=dev)
        seq_lens = torch.full((bs,), L, dtype=torch.long, device=dev)
        if t.dim() != 1:
            raise NotImplementedError('per-token timesteps (Wan2.2 ti2v) are not on the sm_90a path')
        emb = sinusoidal_embedding_1d(self.freq_dim, t.flatten()).unflatten(0, (bs, 1))
        e = linear(emb, self.time_embedding[0])
        e = linear(torch.nn.functional.silu(e), self.time_embedding[2])           # [bs, 1, dim] bf16
        e0 = SiluLinearFn.apply(e, self.time_projection[1]).unflatten(2, (6, self.dim))
        # text: zero the slots beyond each prompt's length, pad to text_len (models/wan/wan.py:453,491-497)
        T = text_embeddings.shape[1]
        keep = (torch.arange(T, device=dev)[None, :] < text_seq_lens.to(dev)[:, None]).unsqueeze(-1)
        ctx_in = text_embeddings * keep.to(text_embeddings.dtype)
        if T < self.text_len:
            ctx_in = torch.cat([ctx_in, ctx_in.new_zeros(bs, self.text_len - T, ctx_in.shape[2])], dim=1)
        elif T > self.text_len:
            raise ValueError(f'text embeddings have {T} slots, model text_len is {self.text_len}')
        context = linear(ctx_in, self.text_embedding[0])
        context = linear(torch.nn.functional.gelu(context, approximate='tanh'), self.text_embedding[2])
        freqs = wan_rope_tables(grid, self.dim // self.num_heads, device=dev)
        return make_contiguous(xe, e, e0, seq_lens, grid_sizes, freqs, context)


class TransformerLayer(nn.Module):
    def __init__(self, block, block_idx):
        super().__init__()
        self.block = block
        self.block_idx = block_idx

    def forward(self, inputs):
        x, e, e0, seq_lens, grid_sizes, freqs, context = inputs
        x = self.block(x, e0, seq_lens, grid_sizes, freqs, context, None)
        return make_contiguous(x, e, e0, seq_lens, grid_sizes, freqs, context)


class FinalLayer(nn.Module):
    def __init__(self, head, patch_size, out_dim):
        super().__init__()
        self.head = head
        self.patch_size, self.out_dim = tuple(patch_size), out_dim

    def forward(self, inputs):
        x, e, e0, seq_lens, grid_sizes, freqs, context = inputs
        y = self.head(x, e)
        # grid from shape metadata of the rope table would lose (f, h, w); grid_sizes is identical for all samples, and
        # reading one row is the same host sync the reference does (`grid_sizes.tolist()`, models/wan/model.py:509)
        grid = tuple(int(v) for v in grid_sizes[0].tolist())
        return unpatchify(y, grid, self.patch_size, self.out_dim)


def get_t_distribution(model_config):
    """utils/common.py:124-146."""
    method = model_config.get('timestep_sample_method', 'logit_normal')
    if method == 'logit_normal':
        dist = torch.distributions.normal.Normal(0, 1)
    elif method == 'uniform':
        dist = torch.distributions.uniform.Uniform(0, 1)
    else:
        raise NotImplementedError()
    n_buckets = 10_000
    delta = 1 / n_buckets
    t = dist.icdf(torch.linspace(delta, 1 - delta, n_buckets))
    if method == 'logit_normal':
        t = torch.sigmoid(t * model_config.get('sigmoid_scale', 1.0))
    return t


def slice_t_distribution(t, min_t=0.0, max_t=1.0):
    start = torch.searchsorted(t, min_t).item()
    end = torch.searchsorted(t, max_t).item()
    return t[start:end]


def sample_t(t, batch_size, quantile=None):
    if quantile is not None:
        i = (torch.full((batch_size,), quantile) * len(t)).to(torch.int32)
    else:
        i = torch.randint(0, len(t), size=(batch_size,))
    return t[i]


class WanPipeline(PluginSurface):
    """Mirror of the reference WanPipeline's training-side surface (models/wan/wan.py:67-411).  VAE, UMT5, CLIP and
    latent caching are outside the hot path (SURVEY.md section 8); `prepare_inputs` consumes the same cached tensors
    (`latents`, `text_embeddings`, `seq_lens`, `mask`)."""
    name = 'wan'
    framerate = 16
    checkpointable_layers = ['TransformerLayer']
    adapter_target_modules = ['WanAttentionBlock']
    pixels_round_to_multiple = 16

    def __init__(self, config, device='cuda'):
        from .flux import get_lin_function, time_shift
        self._get_lin_function, self._time_shift = get_lin_function, time_shift
        self.config = config
        self.model_config = config['model']
        self.cache_text_embeddings = self.model_config.get('cache_text_embeddings', True)
        if not self.cache_text_embeddings:
            raise NotImplementedError('cache_text_embeddings = false (text encoder inside the pipeline) is not supported')
        dtype = self.model_config.get('dtype', torch.bfloat16)
        if isinstance(dtype, str):
            dtype = {'bfloat16': torch.bfloat16, 'float16': torch.float16, 'float32': torch.float32}[dtype]
        if dtype != torch.bfloat16:
            raise NotImplementedError('the sm_90a Wan path computes in bf16 (model.dtype must be bfloat16)')
        tcfg = self.model_config.get('transformer_config', None)
        if tcfg is None:
            tcfg = self._find_checkpoint_config()
        if isinstance(tcfg, str):
            with open(tcfg) as f:
                tcfg = {k: v for k, v in json.load(f).items() if k in WAN_T2V_14B_CONFIG}
            if tcfg.get('model_type') == 'i2v' and not self._checkpoint_has('blocks.0.cross_attn.k_img.weight'):
                tcfg['model_type'] = 'i2v_v2'            # Wan2.2 I2V ships model_type 'i2v' without the CLIP branch (wan.py:131-135)
        self.tcfg = dict(WAN_T2V_14B_CONFIG, **(tcfg or {}))
        self.model_type = self.tcfg['model_type']
        if self.model_type == 'i2v_v2' and 'in_dim' not in (tcfg or {}):
            self.tcfg['in_dim'] = 36
        device = self.model_config.get("device", device)      # (tests: "cpu" with the kernel test doubles)
        self.dtype, self.device = dtype, device
        self.t_dist = get_t_distribution(self.model_config)
        self.pipeline_model = None
        self.model_engine = None
        self.adapter_config = None
        self.transformer = None
        if not self.model_config.get('lazy_layers', False):
            self.transformer = WanModel(self.tcfg, dtype=dtype, device=device)
            if path := self.model_config.get('transformer_path', None):
                self.load_transformer_weights(path)
            self.transformer.train()

    def _find_checkpoint_config(self):
        """models/wan/wan.py:80-97: `transformer_path` is a directory holding config.json next to its shards, or a single
        file whose config.json sits in `ckpt_path` (Wan2.2: `ckpt_path/low_noise_model`).  None when no checkpoint is named
        (synthetic runs: the 14B t2v defaults)."""
        import os
        mc = self.model_config
        ckpt, tp = mc.get('ckpt_path', None), mc.get('transformer_path', None)
        tp = tp or ckpt
        if tp is None:
            return None
        if tp == ckpt and os.path.isdir(tp):
            mc.setdefault('transformer_path', tp)
        cands = [os.path.join(tp, 'config.json')] if os.path.isdir(tp) else \
            ([os.path.join(ckpt, 'config.json'), os.path.join(ckpt, 'low_noise_model', 'config.json')] if ckpt else [])
        for c in cands:
            if os.path.exists(c):
                return c
        return None

    def _checkpoint_has(self, key):
        from .flux import FluxPipeline
        path = self.model_config.get('transformer_path', None)
        return bool(path) and key in FluxPipeline._weight_index(path)

    def load_transformer_weights(self, path):
        from .flux import FluxPipeline
        FluxPipeline.load_transformer_weights(self, path)

    def load_diffusion_model(self):
        pass

    def save_model(self, save_dir, state_dict):
        """models/wan/wan.py:264-265"""
        from .flux import FluxPipeline
        FluxPipeline.write_model_file(save_dir, state_dict)

    def configure_adapter(self, adapter_config):
        from .flux import FluxPipeline
        FluxPipeline.configure_adapter(self, adapter_config)

    def _adapt(self, module, dev):
        from .flux import FluxPipeline
        return FluxPipeline._adapt(self, module, dev)

    def load_adapter_weights(self, adapter_path):
        """models/base.py:367-388 (`[adapter] init_from_existing`)"""
        from .flux import FluxPipeline
        FluxPipeline.load_adapter_weights(self, adapter_path)

    def save_adapter(self, save_dir, peft_state_dict):
        """models/wan/wan.py:258-262 (ComfyUI format: keys prefixed with diffusion_model.)"""
        from .flux import FluxPipeline
        FluxPipeline.write_peft_config(self, save_dir, peft_state_dict)
        FluxPipeline.write_adapter_file(save_dir, {'diffusion_model.' + k: v for k, v in peft_state_dict.items()})

    def get_param_groups(self, parameters):
        return [{'params': parameters}]

    def model_specific_dataset_config_validation(self, dataset_config):
        pass

    # ---- data -> model inputs (models/wan/wan.py:332-373) ----
    def prepare_inputs(self, inputs, timestep_quantile=None):
        latents = inputs['latents'].float()
        mask = inputs['mask']
        text_embeddings = inputs['text_embeddings']
        seq_lens = inputs['seq_lens']
        bs, channels, num_frames, h, w = latents.shape
        if mask is not None:
            mask = mask.unsqueeze(1)
            mask = torch.nn.functional.interpolate(mask, size=(h, w), mode='nearest-exact')
            mask = mask.unsqueeze(2)
        t = self.t_dist
        if shift := self.model_config.get('shift', None):
            t = (t * shift) / (1 + (shift - 1) * t)
        elif self.model_config.get('flux_shift', False):
            mu = self._get_lin_function(y1=0.5, y2=1.15)((h // 2) * (w // 2))
            t = self._time_shift(mu, 1.0, t)
        t = slice_t_distribution(t, min_t=self.model_config.get('min_t', 0.0), max_t=self.model_config.get('max_t', 1.0))
        t = sample_t(t, bs, quantile=timestep_quantile).to(latents.device)
        x_1 = latents
        x_0 = torch.randn_like(x_1)
        if self._noise_on_device(x_1):
            x_t, target = ops.noise_on_device(x_1, x_0, t, False, self.device)
        else:
            te = t.view(-1, 1, 1, 1, 1)
            x_t = (1 - te) * x_1 + te * x_0
            target = x_0 - x_1
        t = t * 1000
        y = inputs['y'] if self.model_type == 'i2v_v2' else None          # models/wan/wan.py:335
        return (x_t, y, t, text_embeddings, seq_lens, None), (target, mask)

    # ---- layers / loss ----
    def to_layers(self):
        from .flux import base_storage_dtype
        base_storage_dtype(self.model_config, self.adapter_config is not None)    # float8 base: LoRA runs only
        if self.transformer is None:
            return self._lazy_layers()
        m = self.transformer
        layers = [InitialLayer(m.patch_embedding, m.time_embedding, m.text_embedding, m.time_projection, self.tcfg)]
        layers += [TransformerLayer(block, i) for i, block in enumerate(m.blocks)]
        layers.append(FinalLayer(m.head, m.patch_size, m.out_dim))
        return layers

    def _lazy_layers(self):
        from .pipe.module import LayerSpec
        cfg, dtype, device = self.tcfg, self.dtype, self.device
        dim = cfg['dim']

        def name_params(module, prefix_map):
            for n, p in module.named_parameters():
                for local, glob in prefix_map.items():
                    if n.startswith(local):
                        p.original_name = glob + n[len(local):]
                        break
            return module

        def build_first(dev=None):
            d = dev or device
            pe = nn.Module()
            pe.weight = nn.Parameter(torch.empty(dim, cfg['in_dim'], *cfg['patch_size'], dtype=dtype, device=d).normal_(0, 0.02))
            pe.bias = nn.Parameter(torch.zeros(dim, dtype=dtype, device=d))
            w = InitialLayer(pe, _Seq([_plain(dim, cfg['freq_dim'], dtype, d), nn.Identity(), _plain(dim, dim, dtype, d)]),
                             _Seq([_plain(dim, cfg['text_dim'], dtype, d), nn.Identity(), _plain(dim, dim, dtype, d)]),
                             _Seq([nn.Identity(), _plain(dim * 6, dim, dtype, d)]), cfg)
            return self._adapt(name_params(w, {'': ''}), dev)

        def build_block(i, dev=None):
            w = TransformerLayer(WanAttentionBlock(dim, cfg['ffn_dim'], cfg['num_heads'], cfg['eps'], dtype, dev or device), i)
            return self._adapt(name_params(w, {'block.': f'blocks.{i}.'}), dev)

        def build_last(dev=None):
            w = FinalLayer(WanHead(dim, cfg['out_dim'], cfg['patch_size'], cfg['eps'], dtype, dev or device), cfg['patch_size'], cfg['out_dim'])
            return self._adapt(name_params(w, {'': ''}), dev)

        def count(fn, *a):
            return sum(p.numel() for p in fn(*a, dev='meta').parameters())

        def spec(cls, fn, *a, n):
            s = LayerSpec(cls, *a)
            s.build = lambda fn=fn, a=a: fn(*a)
            s.param_count = n
            return s
        n_block = count(build_block, 0)
        layers = [spec(InitialLayer, build_first, n=count(build_first))]
        layers += [spec(TransformerLayer, build_block, i, n=n_block) for i in range(cfg['num_layers'])]
        layers.append(spec(FinalLayer, build_last, n=count(build_last)))
        return layers

    def get_loss_fn(self):
        """models/base.py:418-436 on the fp32 prediction [B, C, F, H, W] (590 k elements: ATen elementwise on the device)."""
        cfg = self.config

        def loss_fn(output, label):
            target, mask = label
            o, t = output.float(), target.to(output.device, torch.float32)
            if 'huber_delta' in cfg:
                loss = torch.nn.functional.huber_loss(o, t, reduction='none', delta=cfg['huber_delta'])
            elif 'smooth_l1_beta' in cfg:
                loss = torch.nn.functional.smooth_l1_loss(o, t, reduction='none', beta=cfg['smooth_l1_beta'])
            else:
                loss = torch.nn.functional.mse_loss(o, t, reduction='none')
            if mask.numel() > 0:
                loss = loss * mask.to(o.device, torch.float32)
            return loss.mean()
        return loss_fn
