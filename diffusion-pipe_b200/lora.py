"""LoRA on the fused Flux / Qwen-Image blocks — the adapter path of the reference (models/base.py:263-303:
`peft.LoraConfig(r=rank, lora_alpha=rank, lora_dropout=dropout, bias='none', target_modules=<every nn.Linear inside the
blocks named in adapter_target_modules>)`; train.py:115-133 forces alpha = rank, i.e. scaling 1; SURVEY.md 8(f) item 3).

    y = x W^T + b + (x A^T) B^T          W, b frozen;  A [r, K], B [N, r] trained

**LoRA as a K-extension.**  Both terms are contractions feeding one accumulator, so the adapter rides the SAME wgmma
GEMM — and therefore every fused epilogue (QKV->RMSNorm->RoPE scatter, bias+GELU, gate*y+residual, x GELU') — instead
of a second GEMM plus an elementwise add:

    forward   [x | t] . [W | B]^T        t = x A^T   (r extra K columns; one small GEMM produces t in place)
    backward  [dy | dt] . [W ; A]        dt = dy B   (r extra reduction rows; same epilogues as the dense dgrad)
    grads     dB = dy^T t,  dA = dt^T x  (two skinny GEMMs, queued with the other weight-gradient work)

Each site owns ONE buffer `[(N + R) x (K + R)]` holding `[[W | B], [A | 0]]`: the forward operand is its first N rows,
the dgrad operand its first K columns, so W is stored once and no transposes or copies of W exist.  Projections that the
kernels consume fused (q, k, v of a stream) keep per-projection adapters: A's are stacked, B's are block-diagonal.
The trained factors are ordinary contiguous Parameters (`<linear>.lora_A.weight`, `<linear>.lora_B.weight`, PEFT's
state-dict names); they are copied into the site buffer when their version counter moves (after an optimizer step).
The frozen base produces no weight gradient: a LoRA step runs 2/3 of the dense-training FLOPs.

Supported: rank % 8 == 0 (16-byte rows for TMA), dropout 0, Flux double / single blocks, Qwen-Image and Wan blocks.
Modulation linears (AdaLayerNormZero.linear, batch-row) get their adapter through a [batch, r] torch matmul.

**fp8 base** (`transformer_dtype = 'float8'` / `'float8_e5m2'`: models/flux.py:172,203-205, models/qwen_image.py:249-263,
models/wan/wan.py:216-235).  The reference stores the frozen 2-D weights of the blocks as unscaled float8 and lets
autocast widen them to bf16 inside every nn.Linear.  Here a site then keeps W ONLY as an `[N, K]` fp8 matrix (half the
bytes of the bf16 buffer; the linears' `.weight` are views of it) plus two small bf16 matrices (stacked A's, block-diagonal
B's); `w_fwd` / `w_dgrad` expand `[[W | B], [A | .]]` into ONE per-device operand scratch (the size of the largest site)
with the widening kernel of csrc/fp8_dequant.cu right before the GEMM that reads it — stream order makes the single
buffer safe, and the weight-gradient closures of the zero-bubble order never read W.  Every fp8 value is a bf16 value, so
the GEMMs see exactly what the reference's autocast produces.  Cost: 3 bytes of HBM traffic per weight element per GEMM
(≈6 % of the GEMM's own time at Flux shapes), for half the weight memory.
"""
import math

import torch
from torch import nn

from . import ops
from .flux_blocks import HD, _acc_vec, _grad_buf, _mod_bwd, _mod_fwd


class _LoraW(nn.Module):
    def __init__(self, weight):
        super().__init__()
        self.weight = weight


def _kaiming_a(r, k, dtype, device):
    w = torch.empty(r, k, dtype=torch.float32, device=device)
    nn.init.kaiming_uniform_(w, a=math.sqrt(5))              # peft LoraLayer.reset_lora_parameters (default init)
    return nn.Parameter(w.to(dtype))


# ---- fp8 storage of the frozen base (`transformer_dtype = 'float8'`; module docstring, last paragraph) ----------------
FP8_DTYPES = (torch.float8_e4m3fn, torch.float8_e5m2)
_SCRATCH = {}        # device -> flat bf16 operand buffer shared by every fp8 site of that device (grown on demand)
_SCRATCH_OWNER = {}  # device -> key of what the buffer currently holds
_UIDS = [0]
_EPOCH = [0]         # bumped at the start of every block forward: the scratch is trusted only within one pass over a block


def _uid():
    _UIDS[0] += 1
    return _UIDS[0]


def _widened(device, key, shape, fill):
    """bf16 [rows, cols] view of the device's operand scratch holding whatever `fill(view)` writes; the fill is skipped
    when the scratch still holds `key`.  Everything that reads the view is enqueued on the current stream before the next
    call can overwrite it, so ONE buffer (the size of the largest site) serves all sites."""
    n = shape[0] * shape[1]
    flat = _SCRATCH.get(device)
    if flat is None or flat.numel() < n:
        flat = torch.empty(n, dtype=torch.bfloat16, device=device)
        _SCRATCH[device] = flat
        _SCRATCH_OWNER.pop(device, None)
    view = flat[:n].view(shape)
    if _SCRATCH_OWNER.get(device) != key:
        with torch.no_grad():
            fill(view)
        _SCRATCH_OWNER[device] = key
    return view


class LoraSite:
    """One GEMM site = one or several nn.Linear-like holders (weight [n_i, K], bias) that the kernels consume as one
    [N, K] matrix, plus their LoRA factors.  See the module docstring for the buffer layout."""

    def __init__(self, lins, rank, dtype=torch.bfloat16, base_dtype=None):
        if rank % 8:
            raise ValueError(f'LoRA rank must be a multiple of 8 on the sm_90a path (got {rank})')
        self.lins, self.r = list(lins), rank
        w0 = self.lins[0].weight
        dev = w0.device
        self.K = w0.shape[1]
        self.sizes = [l.weight.shape[0] for l in self.lins]
        self.N = sum(self.sizes)
        self.R = rank * len(self.lins)
        self.fp8 = base_dtype in FP8_DTYPES
        self.uid = _uid()
        if self.fp8:
            if self.K % 16:
                raise ValueError(f'fp8 base storage needs in_features % 16 == 0 (got {self.K})')
            self.buf = None
            self.w8 = torch.empty((self.N, self.K), dtype=base_dtype, device=dev)       # the only copy of W
            self.ab = torch.zeros((self.R, self.K), dtype=torch.bfloat16, device=dev)   # stacked A's
            self.bb = torch.zeros((self.N, self.R), dtype=torch.bfloat16, device=dev)   # block-diagonal B's
        else:
            self.buf = torch.zeros((self.N + self.R, self.K + self.R), dtype=w0.dtype, device=dev)
        self.bias = torch.zeros(self.N, dtype=torch.bfloat16 if self.fp8 else w0.dtype, device=dev)
        row = 0
        self.A, self.B = [], []
        for i, l in enumerate(self.lins):
            n = self.sizes[i]
            base = self.w8[row:row + n] if self.fp8 else self.buf[row:row + n, :self.K]
            base.copy_(l.weight.detach().to(base.dtype))
            if l.bias is not None:
                self.bias[row:row + n].copy_(l.bias.detach())
            # the base parameters now live inside the site buffer (frozen): checkpoints load straight into it
            l.weight.data = base
            l.weight.requires_grad_(False)
            if l.bias is not None:
                l.bias.data = self.bias[row:row + n]
                l.bias.requires_grad_(False)
            a = _kaiming_a(rank, self.K, dtype, dev)
            b = nn.Parameter(torch.zeros(n, rank, dtype=dtype, device=dev))
            l.lora_A, l.lora_B = _LoraW(a), _LoraW(b)
            self.A.append(a)
            self.B.append(b)
            row += n
        self._versions = None
        self.refresh()

    # ---- operand views -------------------------------------------------------------------------------------------
    def _operand(self):
        """[(N + R) x (K + R)] bf16 `[[W | B], [A | .]]`: the site's own buffer, or (fp8 base) the device's operand scratch
        with W widened into it by the dequant kernel (csrc/fp8_dequant.cu) — re-expanded unless this site was the last
        user of the scratch within the same pass (per-sample loops over one site)"""
        if not self.fp8:
            return self.buf

        def fill(view):
            ops.fp8_to_bf16(self.w8, view[:self.N, :self.K])
            view[self.N:, :self.K].copy_(self.ab)
            view[:self.N, self.K:].copy_(self.bb)
        return _widened(self.w8.device, (self.uid, self._versions, _EPOCH[0]), (self.N + self.R, self.K + self.R), fill)

    @property
    def base_weight(self):  # [N, K] storage of the frozen W (bf16 view of the site buffer, or the fp8 matrix)
        return self.w8 if self.fp8 else self.buf[:self.N, :self.K]

    @property
    def w_fwd(self):        # [N, K + R]   ([W | B]),  K-major B operand of the forward GEMM
        return self._operand()[:self.N]

    @property
    def w_dgrad(self):      # [N + R, K]   ([W ; A]),  MN-major (b_mn) operand of the input-gradient GEMM
        return self._operand()[:, :self.K]

    @property
    def a_all(self):        # [R, K]       stacked A's
        return self.ab if self.fp8 else self.buf[self.N:, :self.K]

    @property
    def b_blk(self):        # [N, R]       block-diagonal B's
        return self.bb if self.fp8 else self.buf[:self.N, self.K:]

    def refresh(self):
        """copies the trained factors into the site buffer if an optimizer step (or a load) changed them"""
        if self.fp8:
            _EPOCH[0] += 1      # (called at the start of every block forward) W may have been reloaded since the last pass
        v = tuple(p._version for p in self.A + self.B)
        if v == self._versions:
            return
        row = 0
        a_dst, b_dst = self.a_all, self.b_blk
        with torch.no_grad():
            for i, (a, b) in enumerate(zip(self.A, self.B)):
                n = self.sizes[i]
                a_dst[i * self.r:(i + 1) * self.r].copy_(a)
                b_dst[row:row + n, i * self.r:(i + 1) * self.r].copy_(b)
                row += n
        self._versions = tuple(p._version for p in self.A + self.B)

    # ---- the three small GEMMs ---------------------------------------------------------------------------------------
    def alloc_in(self, rows, device):
        """[rows, K + R] activation buffer: the producing kernel writes x into [:, :K], project() fills the tail"""
        return torch.empty((rows, self.K + self.R), dtype=torch.bfloat16, device=device)

    def alloc_dy(self, rows, device):
        return torch.empty((rows, self.N + self.R), dtype=torch.bfloat16, device=device)

    def project(self, xa):
        """t = x A^T into the tail columns of xa (rows of xa may be a slice of a larger buffer)"""
        ops.gemm(xa[:, :self.K], self.a_all, out=xa[:, self.K:])

    def backproject(self, dya):
        """dt = dy B into the tail columns of dya"""
        ops.gemm(dya[:, :self.N], self.b_blk, b_mn=True, out=dya[:, self.N:])

    def queue_grads(self, xa, dya):
        """dA_i = dt_i^T x,  dB_i = dy_i^T t_i   (weight-gradient work: deferred in the zero-bubble order)"""
        def wgrad(self=self, xa=xa, dya=dya):
            K, N, r = self.K, self.N, self.r
            row = 0
            for i, (a, b) in enumerate(zip(self.A, self.B)):
                n = self.sizes[i]
                if a.requires_grad:
                    g, acc = _grad_buf(a)
                    ops.gemm(dya[:, N + i * r:N + (i + 1) * r], xa[:, :K], a_mn=True, b_mn=True, out=g, accumulate=acc)
                if b.requires_grad:
                    g, acc = _grad_buf(b)
                    ops.gemm(dya[:, row:row + n], xa[:, K + i * r:K + (i + 1) * r], a_mn=True, b_mn=True, out=g, accumulate=acc)
                row += n
        ops.defer(wgrad)


class _WidenedLin:
    """what _mod_fwd / _mod_bwd read of a frozen linear: its (widened) weight and its bias"""
    __slots__ = ('weight', 'bias')

    def __init__(self, weight, bias):
        self.weight, self.bias = weight, bias


class ModLora:
    """adapter of a batch-row modulation linear (AdaLayerNormZero.linear): mod += (silu(temb) A^T) B^T on [batch, r]"""

    def __init__(self, lin, rank, dtype=torch.bfloat16, base_dtype=None):
        self.lin = lin
        dev = lin.weight.device
        lin.weight.requires_grad_(False)
        if lin.bias is not None:
            lin.bias.requires_grad_(False)
        self.fp8 = base_dtype in FP8_DTYPES
        self.uid = _uid()
        if self.fp8:
            if lin.weight.shape[1] % 16:
                raise ValueError(f'fp8 base storage needs in_features % 16 == 0 (got {lin.weight.shape[1]})')
            lin.weight.data = lin.weight.detach().to(base_dtype)
        self.a = _kaiming_a(rank, lin.weight.shape[1], dtype, dev)
        self.b = nn.Parameter(torch.zeros(lin.weight.shape[0], rank, dtype=dtype, device=dev))
        lin.lora_A, lin.lora_B = _LoraW(self.a), _LoraW(self.b)

    def _base(self):
        """the linear as the modulation kernels read it: itself, or (fp8 base) its weight widened into the operand scratch"""
        if not self.fp8:
            return self.lin
        w8 = self.lin.weight.detach()
        w = _widened(w8.device, (self.uid, _EPOCH[0]), tuple(w8.shape), lambda view: ops.fp8_to_bf16(w8, view))
        return _WidenedLin(w, self.lin.bias)

    def fwd(self, temb):
        if self.fp8:
            _EPOCH[0] += 1
        s = torch.nn.functional.silu(temb.float()).to(torch.bfloat16)
        t = (s.float() @ self.a.float().t()).to(torch.bfloat16)                    # lora_A output (bf16)
        mod = _mod_fwd(temb, self._base())
        return (mod.float() + (t.float() @ self.b.float().t()).to(torch.bfloat16).float()).to(torch.bfloat16), (s, t)

    def bwd(self, dmod32, temb, saved, d_temb32):
        """accumulates d temb (fp32) and the factor gradients"""
        s, t = saved
        d = dmod32.to(torch.bfloat16).float()
        _mod_bwd(dmod32, temb, self._base(), d_temb32)                            # frozen base: only the d temb part
        dt = d @ self.b.float()
        _acc_vec(self.b, d.t() @ t.float())
        _acc_vec(self.a, dt.t() @ s.float())
        ds = dt @ self.a.float()
        tf = temb.float()
        sg = torch.sigmoid(tf)
        d_temb32.add_(ds.to(torch.bfloat16).float() * (sg * (1 + tf * (1 - sg))))


def _needs(p):
    return p is not None and p.requires_grad


# =====================================================================================================================
# double-stream block (Flux, Qwen-Image)
# =====================================================================================================================
class FluxDoubleBlockLoraFn(torch.autograd.Function):
    """FluxDoubleBlockFn (flux_blocks.py) with every Linear of the block carrying a LoRA adapter and the base frozen."""

    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin, txt_lens=None):
        lo = blk.lora
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        Ltot = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        for s in lo['sites']:
            s.refresh()
        shp = (B, H, Ltot, HD)
        q, k, v, qhat, khat = (torch.empty(shp, dtype=bf, device=dev) for _ in range(5))
        q_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, Ltot), dtype=torch.float32, device=dev)
        spec = ((hidden, Li, Lt, lo['mod'], lo['qkv'], blk.attn.norm_q, blk.attn.norm_k),
                (enc, Lt, 0, lo['mod_c'], lo['add_qkv'], blk.attn.norm_added_q, blk.attn.norm_added_k))
        streams = []
        for x3, L, off, ml, sq, nq, nk in spec:
            st = {'L': L, 'off': off, 'x': x3.reshape(B * L, D)}
            st['mod'], st['mod_saved'] = ml.fwd(temb)
            m = st['mod']
            xa = sq.alloc_in(B * L, dev)
            _, st['mean1'], st['rstd1'] = ops.ln_modulate_fwd(st['x'], m[:, D:2 * D], m[:, 0:D], B, L, out=xa[:, :D])
            sq.project(xa)
            e = ops.make_qkv_epilogue(q, k, v, nq.weight, nk.weight, cos, sin, H, Ltot, off, qhat, khat, q_rstd, k_rstd)
            ops.gemm(xa, sq.w_fwd, bias=sq.bias, epilogue=ops.EPI_QKV_ROPE, out=xa, rows_per_batch=L, qkv=e)
            st['t_qkv'] = xa[:, D:].clone()          # [rows, R]: what the factor gradients need (x itself is recomputed)
            streams.append(st)
        so, sao = lo['to_out'], lo['to_add_out']
        assert so.R == sao.R
        oa = torch.empty((B * Ltot, H * HD + so.R), dtype=bf, device=dev)      # attention output + adapter columns
        if txt_lens is None:
            _, lse = ops.attn_fwd(q, k, v, out=oa)
        else:                                  # prompts of different lengths in one micro-batch (flux_blocks._ragged_attn_fwd)
            from .flux_blocks import _ragged_attn_fwd
            o_dense, lse = _ragged_attn_fwd(q, k, v, Lt, txt_lens)
            oa[:, :H * HD].copy_(o_dense)
        ctx.ragged = txt_lens is not None
        oa3 = oa.view(B, Ltot, H * HD + so.R)
        outs = []
        tail = ((so, lo['ff1'], lo['ff2']), (sao, lo['ffc1'], lo['ffc2']))
        for st, (swo, s1, s2) in zip(streams, tail):
            L, off, m = st['L'], st['off'], st['mod']
            st['y_attn'] = torch.empty((B * L, D), dtype=bf, device=dev)
            st['x1'] = torch.empty((B * L, D), dtype=bf, device=dev)
            for b in range(B):
                rs = slice(b * L, (b + 1) * L)
                rows = oa3[b, off:off + L]
                swo.project(rows)
                ops.gemm(rows, swo.w_fwd, bias=swo.bias, epilogue=ops.EPI_GATE_RES, aux=st['x'][rs], gate=m[b:b + 1, 2 * D:3 * D],
                         out=st['x1'][rs], out2=st['y_attn'][rs], rows_per_batch=L)
            x2a = s1.alloc_in(B * L, dev)
            _, st['mean2'], st['rstd2'] = ops.ln_modulate_fwd(st['x1'], m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L, out=x2a[:, :D])
            s1.project(x2a)
            st['t_ff1'] = x2a[:, D:].clone()
            st['u'] = torch.empty((B * L, s1.N), dtype=bf, device=dev)
            ha = s2.alloc_in(B * L, dev)
            ops.gemm(x2a, s1.w_fwd, bias=s1.bias, epilogue=ops.EPI_BIAS_GELU, out=ha[:, :s1.N], out2=st['u'])
            s2.project(ha)
            st['ha'] = ha
            st['y_mlp'] = torch.empty((B * L, D), dtype=bf, device=dev)
            x2 = ops.gemm(ha, s2.w_fwd, bias=s2.bias, epilogue=ops.EPI_GATE_RES, aux=st['x1'], gate=m[:, 5 * D:6 * D],
                          out2=st['y_mlp'], rows_per_batch=L)
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
        lo = blk.lora
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        Ltot = Li + Lt
        C = H * HD
        dev = temb.device
        bf = torch.bfloat16
        q, k, v, qhat, khat, q_rstd, k_rstd, oa, lse = ctx.attn
        so, sao = lo['to_out'], lo['to_add_out']
        oa3 = oa.view(B, Ltot, C + so.R)
        d_o = torch.empty((B * Ltot, C), dtype=bf, device=dev)
        d_o3 = d_o.view(B, Ltot, C)
        tail = ((so, lo['ff1'], lo['ff2']), (sao, lo['ffc1'], lo['ffc2']))
        dmods, dx1s = [], []
        for st, (swo, s1, s2), dxo in zip(ctx.streams, tail, (d_hidden, d_enc)):
            L, off, m = st['L'], st['off'], st['mod']
            dx2 = dxo.reshape(B * L, D)
            if dx2.dtype != bf:
                dx2 = dx2.to(bf)
            dmod = torch.empty((B, 6 * D), dtype=torch.float32, device=dev)
            # ---- MLP branch ----
            dy2a = s2.alloc_dy(B * L, dev)
            _, part = ops.gate_bwd(dx2, st['y_mlp'], m[:, 5 * D:6 * D], B, L, dy=dy2a[:, :D])
            ops.colreduce_finish(part, per_sample0=dmod[:, 5 * D:6 * D])
            s2.backproject(dy2a)
            s2.queue_grads(st['ha'], dy2a)
            dua = s1.alloc_dy(B * L, dev)
            ops.gemm(dy2a, s2.w_dgrad, b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=st['u'], out=dua[:, :s1.N])
            s1.backproject(dua)
            x2a = s1.alloc_in(B * L, dev)
            ops.ln_modulate_fwd(st['x1'], m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L, out=x2a[:, :D], save_stats=False)
            x2a[:, D:].copy_(st['t_ff1'])
            s1.queue_grads(x2a, dua)
            dxn2 = ops.gemm(dua, s1.w_dgrad, b_mn=True)
            dx1, part = ops.ln_modulate_bwd(dxn2, st['x1'], m[:, 4 * D:5 * D], st['mean2'], st['rstd2'], B, L, dres=dx2)
            ops.colreduce_finish(part, per_sample0=dmod[:, 4 * D:5 * D], per_sample1=dmod[:, 3 * D:4 * D])
            # ---- attention branch ----
            dy1a = swo.alloc_dy(B * L, dev)
            _, part = ops.gate_bwd(dx1, st['y_attn'], m[:, 2 * D:3 * D], B, L, dy=dy1a[:, :D])
            ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D])
            swo.backproject(dy1a)
            for b in range(B):
                rs = slice(b * L, (b + 1) * L)
                ops.gemm(dy1a[rs], swo.w_dgrad, b_mn=True, out=d_o3[b, off:off + L])
                swo.queue_grads(oa3[b, off:off + L], dy1a[rs])
            dmods.append(dmod)
            dx1s.append(dx1)
        if ctx.ragged:
            from .flux_blocks import _ragged_attn_bwd
            dq, dk, dv = _ragged_attn_bwd(lse, d_o, q.shape)
        else:
            dq, dk, dv = ops.attn_bwd(q, k, v, oa, d_o, lse)
        d_temb = torch.zeros_like(temb, dtype=torch.float32)
        grads = []
        spec = ((lo['mod'], lo['qkv'], blk.attn.norm_q, blk.attn.norm_k), (lo['mod_c'], lo['add_qkv'], blk.attn.norm_added_q, blk.attn.norm_added_k))
        for st, dmod, dx1, (ml, sq, nq, nk) in zip(ctx.streams, dmods, dx1s, spec):
            L, off, m = st['L'], st['off'], st['mod']
            dqa = sq.alloc_dy(B * L, dev)
            dbias = torch.zeros(3 * C, dtype=torch.float32, device=dev)
            dw = torch.zeros((2, HD), dtype=torch.float32, device=dev)
            ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, nq.weight, nk.weight, cos, sin, dqa, dbias, dw,
                                B, H, Ltot, off, L)
            if _needs(nq.weight):
                _acc_vec(nq.weight, dw[0])
                _acc_vec(nk.weight, dw[1])
            sq.backproject(dqa)
            xa = sq.alloc_in(B * L, dev)
            ops.ln_modulate_fwd(st['x'], m[:, D:2 * D], m[:, 0:D], B, L, out=xa[:, :D], save_stats=False)
            xa[:, D:].copy_(st['t_qkv'])
            sq.queue_grads(xa, dqa)
            dxn = ops.gemm(dqa, sq.w_dgrad, b_mn=True)
            dx, part = ops.ln_modulate_bwd(dxn, st['x'], m[:, D:2 * D], st['mean1'], st['rstd1'], B, L, dres=dx1)
            ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
            ml.bwd(dmod, temb, st['mod_saved'], d_temb)
            grads.append(dx.view(B, L, D))
        ctx.streams = None
        ctx.attn = None
        return None, grads[0], grads[1], d_temb.to(temb.dtype), None, None, None


# =====================================================================================================================
# single-stream block (Flux)
# =====================================================================================================================
class FluxSingleBlockLoraFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, blk, hidden, enc, temb, cos, sin):
        lo = blk.lora
        B, Li, D = hidden.shape
        Lt = enc.shape[1]
        L = Li + Lt
        H = blk.heads
        dev = hidden.device
        bf = torch.bfloat16
        for s in lo['sites']:
            s.refresh()
        s1, s2 = lo['lin1'], lo['proj_out']
        inner = blk.mlp_dim
        x = torch.cat([enc, hidden], dim=1).reshape(B * L, D)
        mod, mod_saved = lo['mod'].fwd(temb)
        xa = s1.alloc_in(B * L, dev)
        _, mean, rstd = ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], B, L, out=xa[:, :D])
        s1.project(xa)
        t1 = xa[:, D:].clone()
        shp = (B, H, L, HD)
        q, k, v, qhat, khat = (torch.empty(shp, dtype=bf, device=dev) for _ in range(5))
        q_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        k_rstd = torch.empty((B, H, L), dtype=torch.float32, device=dev)
        cata = s2.alloc_in(B * L, dev)              # [attn | gelu(mlp) | adapter columns]: the operand of proj_out
        u = torch.empty((B * L, inner), dtype=bf, device=dev)
        e = ops.make_qkv_epilogue(q, k, v, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos, sin, H, L, 0, qhat, khat,
                                  q_rstd, k_rstd)
        ops.gemm(xa, s1.w_fwd, bias=s1.bias, epilogue=ops.EPI_QKV_ROPE, out=cata[:, D:D + inner], out2=u, rows_per_batch=L, qkv=e)
        _, lse = ops.attn_fwd(q, k, v, out=cata)
        s2.project(cata)
        y = torch.empty((B * L, D), dtype=bf, device=dev)
        xo = ops.gemm(cata, s2.w_fwd, bias=s2.bias, epilogue=ops.EPI_GATE_RES, aux=x, gate=mod[:, 2 * D:3 * D], out2=y,
                      rows_per_batch=L)
        xo3 = xo.view(B, L, D)
        ctx.blk = blk
        ctx.saved = (x, mod, mod_saved, mean, rstd, t1, q, k, v, qhat, khat, q_rstd, k_rstd, cata, u, lse, y)
        ctx.save_for_backward(temb, cos, sin)
        ctx.dims = (B, Li, Lt, D, H)
        return xo3[:, Lt:], xo3[:, :Lt]

    @staticmethod
    def backward(ctx, d_hidden, d_enc):
        blk = ctx.blk
        lo = blk.lora
        temb, cos, sin = ctx.saved_tensors
        B, Li, Lt, D, H = ctx.dims
        L = Li + Lt
        C = H * HD
        dev = temb.device
        bf = torch.bfloat16
        x, mod, mod_saved, mean, rstd, t1, q, k, v, qhat, khat, q_rstd, k_rstd, cata, u, lse, y = ctx.saved
        s1, s2 = lo['lin1'], lo['proj_out']
        inner = blk.mlp_dim
        dxo = torch.cat([d_enc, d_hidden], dim=1).reshape(B * L, D)
        if dxo.dtype != bf:
            dxo = dxo.to(bf)
        dmod = torch.empty((B, 3 * D), dtype=torch.float32, device=dev)
        dya = s2.alloc_dy(B * L, dev)
        _, part = ops.gate_bwd(dxo, y, mod[:, 2 * D:3 * D], B, L, dy=dya[:, :D])
        ops.colreduce_finish(part, per_sample0=dmod[:, 2 * D:3 * D])
        s2.backproject(dya)
        s2.queue_grads(cata, dya)
        dl1a = s1.alloc_dy(B * L, dev)                                   # [dq | dk | dv | d mlp_pre | adapter columns]
        d_o = torch.empty((B * L, D), dtype=bf, device=dev)
        wd = s2.w_dgrad                                                  # [D + R, D + inner]
        ops.gemm(dya, wd[:, :D], b_mn=True, out=d_o)
        ops.gemm(dya, wd[:, D:], b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=u, out=dl1a[:, 3 * C:3 * C + inner])
        dq, dk, dv = ops.attn_bwd(q, k, v, cata, d_o, lse)
        dbias = torch.zeros(3 * C, dtype=torch.float32, device=dev)
        dw = torch.zeros((2, HD), dtype=torch.float32, device=dev)
        ops.qknorm_rope_bwd(dq, dk, dv, qhat, khat, q_rstd, k_rstd, blk.attn.norm_q.weight, blk.attn.norm_k.weight, cos, sin,
                            dl1a, dbias, dw, B, H, L, 0, L)
        if _needs(blk.attn.norm_q.weight):
            _acc_vec(blk.attn.norm_q.weight, dw[0])
            _acc_vec(blk.attn.norm_k.weight, dw[1])
        s1.backproject(dl1a)
        xa = s1.alloc_in(B * L, dev)
        ops.ln_modulate_fwd(x, mod[:, D:2 * D], mod[:, 0:D], B, L, out=xa[:, :D], save_stats=False)
        xa[:, D:].copy_(t1)
        s1.queue_grads(xa, dl1a)
        dxn = ops.gemm(dl1a, s1.w_dgrad, b_mn=True)
        dx, part = ops.ln_modulate_bwd(dxn, x, mod[:, D:2 * D], mean, rstd, B, L, dres=dxo)
        ops.colreduce_finish(part, per_sample0=dmod[:, D:2 * D], per_sample1=dmod[:, 0:D])
        d_temb = torch.zeros((B, D), dtype=torch.float32, device=dev)
        lo['mod'].bwd(dmod, temb, mod_saved, d_temb)
        dx3 = dx.view(B, L, D)
        ctx.saved = None
        return None, dx3[:, Lt:], dx3[:, :Lt], d_temb.to(temb.dtype), None, None


# =====================================================================================================================
# attaching adapters
# =====================================================================================================================
def _name_factors(blk):
    """original_name of a new factor = the block's prefix (taken from an already named parameter) + its local name"""
    prefix = None
    for n, p in blk.named_parameters():
        on = getattr(p, 'original_name', None)
        if on is not None and on.endswith(n):
            prefix = on[:len(on) - len(n)]
            break
    if prefix is None:
        return
    for n, p in blk.named_parameters():
        if '.lora_A.' in n or '.lora_B.' in n:
            p.original_name = prefix + n


def attach(module, rank, dtype=torch.bfloat16, base_dtype=None):
    """attaches adapters to every supported block found under `module`; returns the number of blocks adapted.
    base_dtype = torch.float8_e4m3fn / float8_e5m2 stores the frozen 2-D weights of the blocks in fp8 (the reference's
    `transformer_dtype`); None keeps them in the compute dtype."""
    n = 0
    for m in module.modules():
        if 'lora' in m.__dict__:
            continue
        cls = type(m).__name__
        if cls in ('FluxTransformerBlock', 'QwenImageTransformerBlock'):
            attach_double_block(m, rank, dtype, base_dtype)
            n += 1
        elif cls == 'FluxSingleTransformerBlock':
            attach_single_block(m, rank, dtype, base_dtype)
            n += 1
        elif cls == 'WanAttentionBlock':
            attach_wan_block(m, rank, dtype, base_dtype)
            n += 1
    return n


def attach_double_block(blk, rank, dtype=torch.bfloat16, base_dtype=None):
    """every nn.Linear of a FluxTransformerBlock / QwenImageTransformerBlock gets an adapter (models/base.py:263-271)"""
    a = blk.attn
    lo = {
        'mod': ModLora(blk.norm1.linear, rank, dtype, base_dtype), 'mod_c': ModLora(blk.norm1_context.linear, rank, dtype, base_dtype),
        'qkv': LoraSite([a.to_q, a.to_k, a.to_v], rank, dtype, base_dtype),
        'add_qkv': LoraSite([a.add_q_proj, a.add_k_proj, a.add_v_proj], rank, dtype, base_dtype),
        'to_out': LoraSite([a.to_out[0]], rank, dtype, base_dtype), 'to_add_out': LoraSite([a.to_add_out], rank, dtype, base_dtype),
        'ff1': LoraSite([blk.ff.net[0].proj], rank, dtype, base_dtype), 'ff2': LoraSite([blk.ff.net[2]], rank, dtype, base_dtype),
        'ffc1': LoraSite([blk.ff_context.net[0].proj], rank, dtype, base_dtype), 'ffc2': LoraSite([blk.ff_context.net[2]], rank, dtype, base_dtype),
    }
    lo['sites'] = [v for v in lo.values() if isinstance(v, LoraSite)]
    for n in (a.norm_q, a.norm_k, a.norm_added_q, a.norm_added_k):
        n.weight.requires_grad_(False)                       # bias='none', no modules_to_save: only the factors train
    for fp, site in ((blk.qkv, lo['qkv']), (blk.add_qkv, lo['add_qkv'])):
        fp.weight, fp.bias = site.base_weight, site.bias   # drop the old fused storage (the site owns W now)
    blk.__dict__['lora'] = lo
    _name_factors(blk)
    return lo


def attach_single_block(blk, rank, dtype=torch.bfloat16, base_dtype=None):
    a = blk.attn
    lo = {
        'mod': ModLora(blk.norm.linear, rank, dtype, base_dtype),
        'lin1': LoraSite([a.to_q, a.to_k, a.to_v, blk.proj_mlp], rank, dtype, base_dtype),
        'proj_out': LoraSite([blk.proj_out], rank, dtype, base_dtype),
    }
    lo['sites'] = [v for v in lo.values() if isinstance(v, LoraSite)]
    for n in (a.norm_q, a.norm_k):
        n.weight.requires_grad_(False)
    blk.lin1.weight, blk.lin1.bias = lo['lin1'].base_weight, lo['lin1'].bias
    blk.__dict__['lora'] = lo
    _name_factors(blk)
    return lo


def lora_state_dict(module):
    """{original_name: tensor} of the adapter factors only (what the reference's save_adapter receives)"""
    return {n: p.detach() for n, p in module.named_parameters() if '.lora_A.' in n or '.lora_B.' in n}


# =====================================================================================================================
# Wan attention block (adapter_target_modules = ['WanAttentionBlock'], models/wan/wan.py:71: its ten nn.Linear)
# =====================================================================================================================
class WanBlockLoraFn(torch.autograd.Function):
    """WanBlockFn (wan.py) with adapters on q/k/v/o of both attentions and on the two FFN linears; base, norms and the
    modulation table frozen."""

    @staticmethod
    def forward(ctx, blk, x, e0, context, cos, sin):
        lo = blk.lora
        B, L, D = x.shape
        Lc = context.shape[1]
        H = blk.num_heads
        dev = x.device
        bf = torch.bfloat16
        for s in lo['sites']:
            s.refresh()
        LN_STEPS, LN_MULT = ops.LN_ROUND_STEPS, ops.LN_MULT_DIRECT
        x2 = x.reshape(B * L, D)
        mod = (blk.modulation.unsqueeze(0) + e0).reshape(B, 6, D)
        sa, ca = blk.self_attn, blk.cross_attn
        s_qkv, s_o, s_cq, s_ckv, s_co, s_f1, s_f2 = (lo[k] for k in ('sa_qkv', 'sa_o', 'ca_q', 'ca_kv', 'ca_o', 'ffn1', 'ffn2'))
        # ---- self-attention ----
        xa = s_qkv.alloc_in(B * L, dev)
        _, mean1, rstd1 = ops.ln_modulate_fwd(x2, mod[:, 1], mod[:, 0], B, L, eps=blk.eps, out=xa[:, :D], flags=LN_STEPS)
        s_qkv.project(xa)
        t_qkv = xa[:, D:].clone()
        qkv = ops.gemm(xa, s_qkv.w_fwd, bias=s_qkv.bias)
        (q, xhq, rq), (k, xhk, rk), (v, _, _) = ops.wan_norm_rope_fwd(
            [{'src': qkv[:, 0:D], 'weight': sa.norm_q.weight, 'rope': True},
             {'src': qkv[:, D:2 * D], 'weight': sa.norm_k.weight, 'rope': True},
             {'src': qkv[:, 2 * D:3 * D]}], B, L, H, cos, sin, eps=blk.eps)
        del qkv, xa
        oa = s_o.alloc_in(B * L, dev)
        _, lse = ops.attn_fwd(q, k, v, out=oa)
        s_o.project(oa)
        y_attn = torch.empty((B * L, D), dtype=bf, device=dev)
        x1 = ops.gemm(oa, s_o.w_fwd, bias=s_o.bias, epilogue=ops.EPI_GATE_RES, aux=x2, gate=mod[:, 2], out2=y_attn, rows_per_batch=L)
        # ---- cross-attention ----
        n3w = blk.norm3.weight.view(1, D).expand(B, D)
        n3b = blk.norm3.bias.view(1, D).expand(B, D)
        x3a = s_cq.alloc_in(B * L, dev)
        _, mean3, rstd3 = ops.ln_modulate_fwd(x1, n3w, n3b, B, L, eps=blk.eps, out=x3a[:, :D], flags=LN_MULT)
        s_cq.project(x3a)
        t_cq = x3a[:, D:].clone()
        qc_lin = ops.gemm(x3a, s_cq.w_fwd, bias=s_cq.bias)
        ((qc, xhqc, rqc),) = ops.wan_norm_rope_fwd([{'src': qc_lin, 'weight': ca.norm_q.weight}], B, L, H, eps=blk.eps)
        del qc_lin, x3a
        ca_in = s_ckv.alloc_in(B * Lc, dev)
        ca_in[:, :D].copy_(context.reshape(B * Lc, D))
        s_ckv.project(ca_in)
        kv_lin = ops.gemm(ca_in, s_ckv.w_fwd, bias=s_ckv.bias)
        (kc, xhkc, rkc), (vc, _, _) = ops.wan_norm_rope_fwd(
            [{'src': kv_lin[:, 0:D], 'weight': ca.norm_k.weight}, {'src': kv_lin[:, D:2 * D]}], B, Lc, H, eps=blk.eps)
        del kv_lin
        oca = s_co.alloc_in(B * L, dev)
        _, lse_c = ops.attn_fwd(qc, kc, vc, out=oca)
        s_co.project(oca)
        x2_ = ops.gemm(oca, s_co.w_fwd, bias=s_co.bias, epilogue=ops.EPI_GATE_RES, aux=x1, gate=blk._ones(B, D, dev), rows_per_batch=L)
        # ---- feed-forward ----
        x2a = s_f1.alloc_in(B * L, dev)
        _, mean2, rstd2 = ops.ln_modulate_fwd(x2_, mod[:, 4], mod[:, 3], B, L, eps=blk.eps, out=x2a[:, :D], flags=LN_STEPS)
        s_f1.project(x2a)
        t_f1 = x2a[:, D:].clone()
        F = s_f1.N
        u = torch.empty((B * L, F), dtype=bf, device=dev)
        ha = s_f2.alloc_in(B * L, dev)
        ops.gemm(x2a, s_f1.w_fwd, bias=s_f1.bias, epilogue=ops.EPI_BIAS_GELU, out=ha[:, :F], out2=u)
        del x2a
        s_f2.project(ha)
        y_mlp = torch.empty((B * L, D), dtype=bf, device=dev)
        x3 = ops.gemm(ha, s_f2.w_fwd, bias=s_f2.bias, epilogue=ops.EPI_GATE_RES, aux=x2_, gate=mod[:, 5], out2=y_mlp, rows_per_batch=L)
        ctx.blk = blk
        ctx.saved = (x2, mod, mean1, rstd1, t_qkv, q, k, v, xhq, rq, xhk, rk, oa, lse, y_attn, x1, mean3, rstd3, t_cq, qc, xhqc,
                     rqc, ca_in, kc, xhkc, rkc, vc, oca, lse_c, x2_, mean2, rstd2, t_f1, u, ha, y_mlp)
        ctx.save_for_backward(cos, sin)
        ctx.dims = (B, L, Lc, D, H)
        ctx.in_dtypes = (x.dtype, e0.dtype, context.dtype)
        return x3.view(B, L, D)

    @staticmethod
    def backward(ctx, dx3):
        blk = ctx.blk
        lo = blk.lora
        cos, sin = ctx.saved_tensors
        B, L, Lc, D, H = ctx.dims
        (x2, mod, mean1, rstd1, t_qkv, q, k, v, xhq, rq, xhk, rk, oa, lse, y_attn, x1, mean3, rstd3, t_cq, qc, xhqc,
         rqc, ca_in, kc, xhkc, rkc, vc, oca, lse_c, x2_, mean2, rstd2, t_f1, u, ha, y_mlp) = ctx.saved
        ctx.saved = None
        dev = x2.device
        bf = torch.bfloat16
        LN_STEPS, LN_MULT = ops.LN_ROUND_STEPS, ops.LN_MULT_DIRECT
        sa, ca = blk.self_attn, blk.cross_attn
        s_qkv, s_o, s_cq, s_ckv, s_co, s_f1, s_f2 = (lo[k] for k in ('sa_qkv', 'sa_o', 'ca_q', 'ca_kv', 'ca_o', 'ffn1', 'ffn2'))
        F = s_f1.N
        dmod = torch.zeros((B, 6, D), dtype=torch.float32, device=dev)
        d3 = dx3.reshape(B * L, D)
        if d3.dtype != bf:
            d3 = d3.to(bf)
        d3 = d3.contiguous()
        # ---- feed-forward ----
        dy2a = s_f2.alloc_dy(B * L, dev)
        _, part = ops.gate_bwd(d3, y_mlp, mod[:, 5], B, L, dy=dy2a[:, :D])
        ops.colreduce_finish(part, per_sample0=dmod[:, 5])
        s_f2.backproject(dy2a)
        s_f2.queue_grads(ha, dy2a)
        dua = s_f1.alloc_dy(B * L, dev)
        ops.gemm(dy2a, s_f2.w_dgrad, b_mn=True, epilogue=ops.EPI_MUL_GELU_GRAD, aux=u, out=dua[:, :F])
        s_f1.backproject(dua)
        x2a = s_f1.alloc_in(B * L, dev)
        ops.ln_modulate_fwd(x2_, mod[:, 4], mod[:, 3], B, L, eps=blk.eps, out=x2a[:, :D], save_stats=False, flags=LN_STEPS)
        x2a[:, D:].copy_(t_f1)
        s_f1.queue_grads(x2a, dua)
        dxn2 = ops.gemm(dua, s_f1.w_dgrad, b_mn=True)
        # d x2 lands directly in the dy operand of the cross-attention output projection (x2 = x1 + o_c W^T: no gate)
        dca = s_co.alloc_dy(B * L, dev)
        _, part = ops.ln_modulate_bwd(dxn2, x2_, mod[:, 4], mean2, rstd2, B, L, dres=d3, dx=dca[:, :D], flags=LN_STEPS)
        ops.colreduce_finish(part, per_sample0=dmod[:, 4], per_sample1=dmod[:, 3])
        dx2 = dca[:, :D]
        # ---- cross-attention ----
        s_co.backproject(dca)
        s_co.queue_grads(oca, dca)
        d_oc = ops.gemm(dca, s_co.w_dgrad, b_mn=True)
        dqc, dkc, dvc = ops.attn_bwd(qc, kc, vc, oca, d_oc, lse_c)
        dqca = s_cq.alloc_dy(B * L, dev)
        ops.wan_norm_rope_bwd([{'dy': dqc, 'dx': dqca[:, :D], 'weight': ca.norm_q.weight, 'xhat': xhqc, 'rstd': rqc}], B, L, H)
        s_cq.backproject(dqca)
        dkva = s_ckv.alloc_dy(B * Lc, dev)
        ops.wan_norm_rope_bwd([{'dy': dkc, 'dx': dkva[:, 0:D], 'weight': ca.norm_k.weight, 'xhat': xhkc, 'rstd': rkc},
                               {'dy': dvc, 'dx': dkva[:, D:2 * D]}], B, Lc, H)
        s_ckv.backproject(dkva)
        s_ckv.queue_grads(ca_in, dkva)
        n3w = blk.norm3.weight.view(1, D).expand(B, D)
        n3b = blk.norm3.bias.view(1, D).expand(B, D)
        x3a = s_cq.alloc_in(B * L, dev)
        ops.ln_modulate_fwd(x1, n3w, n3b, B, L, eps=blk.eps, out=x3a[:, :D], save_stats=False, flags=LN_MULT)
        x3a[:, D:].copy_(t_cq)
        s_cq.queue_grads(x3a, dqca)
        d_ctx = ops.gemm(dkva, s_ckv.w_dgrad, b_mn=True)
        dxn3 = ops.gemm(dqca, s_cq.w_dgrad, b_mn=True)
        dx1, _ = ops.ln_modulate_bwd(dxn3, x1, n3w, mean3, rstd3, B, L, dres=dx2, flags=LN_MULT)      # norm3 is frozen
        # ---- self-attention ----
        dy1a = s_o.alloc_dy(B * L, dev)
        _, part = ops.gate_bwd(dx1, y_attn, mod[:, 2], B, L, dy=dy1a[:, :D])
        ops.colreduce_finish(part, per_sample0=dmod[:, 2])
        s_o.backproject(dy1a)
        s_o.queue_grads(oa, dy1a)
        d_o = ops.gemm(dy1a, s_o.w_dgrad, b_mn=True)
        dq, dk, dv = ops.attn_bwd(q, k, v, oa, d_o, lse)
        dqkva = s_qkv.alloc_dy(B * L, dev)
        ops.wan_norm_rope_bwd(
            [{'dy': dq, 'dx': dqkva[:, 0:D], 'weight': sa.norm_q.weight, 'xhat': xhq, 'rstd': rq, 'rope': True},
             {'dy': dk, 'dx': dqkva[:, D:2 * D], 'weight': sa.norm_k.weight, 'xhat': xhk, 'rstd': rk, 'rope': True},
             {'dy': dv, 'dx': dqkva[:, 2 * D:3 * D]}], B, L, H, cos, sin)
        s_qkv.backproject(dqkva)
        xa = s_qkv.alloc_in(B * L, dev)
        ops.ln_modulate_fwd(x2, mod[:, 1], mod[:, 0], B, L, eps=blk.eps, out=xa[:, :D], save_stats=False, flags=LN_STEPS)
        xa[:, D:].copy_(t_qkv)
        s_qkv.queue_grads(xa, dqkva)
        dxn1 = ops.gemm(dqkva, s_qkv.w_dgrad, b_mn=True)
        dx, part = ops.ln_modulate_bwd(dxn1, x2, mod[:, 1], mean1, rstd1, B, L, dres=dx1, flags=LN_STEPS)
        ops.colreduce_finish(part, per_sample0=dmod[:, 1], per_sample1=dmod[:, 0])
        xdt, edt, cdt = ctx.in_dtypes
        return (None, dx.view(B, L, D).to(xdt), dmod.view(B, 1, 6, D).to(edt), d_ctx.view(B, Lc, D).to(cdt), None, None)


def attach_wan_block(blk, rank, dtype=torch.bfloat16, base_dtype=None):
    sa, ca = blk.self_attn, blk.cross_attn
    lo = {
        'sa_qkv': LoraSite([sa.q, sa.k, sa.v], rank, dtype, base_dtype), 'sa_o': LoraSite([sa.o], rank, dtype, base_dtype),
        'ca_q': LoraSite([ca.q], rank, dtype, base_dtype), 'ca_kv': LoraSite([ca.k, ca.v], rank, dtype, base_dtype), 'ca_o': LoraSite([ca.o], rank, dtype, base_dtype),
        'ffn1': LoraSite([blk.ffn[0]], rank, dtype, base_dtype), 'ffn2': LoraSite([blk.ffn[2]], rank, dtype, base_dtype),
    }
    lo['sites'] = [v for v in lo.values() if isinstance(v, LoraSite)]
    for p in (sa.norm_q.weight, sa.norm_k.weight, ca.norm_q.weight, ca.norm_k.weight, blk.norm3.weight, blk.norm3.bias, blk.modulation):
        p.requires_grad_(False)
    sa.qkv.weight, sa.qkv.bias = lo['sa_qkv'].base_weight, lo['sa_qkv'].bias
    ca.kv.weight, ca.kv.bias = lo['ca_kv'].base_weight, lo['ca_kv'].bias
    blk.__dict__['lora'] = lo
    _name_factors(blk)
    return lo
