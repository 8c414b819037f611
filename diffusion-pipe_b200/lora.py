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

**Sites.**  `LoraSite` and `ModLora` implement the site interface that the block functions (flux_blocks.py, wan.py) are
written against; `attach_*` replaces a block's dense sites (flux_blocks.DenseSite / DenseMod, the same interface with R = 0)
by adapted ones, and the same autograd Function then trains the factors.  An adapted site keeps only the R adapter columns
of a LayerNorm+modulation output it consumes and recomputes the LayerNorm in backward (memory; DESIGN.md §3).

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
from .flux_blocks import _acc_vec, _grad_buf, _mod_bwd, _mod_fwd


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

    # ---- the site interface of the block functions (flux_blocks.DenseSite is its R = 0 form) ---------------------------
    bias_grad = False       # the base (bias included) is frozen

    def alloc_in(self, rows, device):
        """[rows, K + R] activation buffer: the producing kernel writes x into [:, :K], project() fills the tail"""
        return torch.empty((rows, self.K + self.R), dtype=torch.bfloat16, device=device)

    def alloc_dy(self, rows, device, spare=None):
        """[rows, N + R] dy buffer (a dense site's `spare` is too narrow to hold the adapter columns)"""
        return torch.empty((rows, self.N + self.R), dtype=torch.bfloat16, device=device)

    def input_operand(self, x):
        """[x | x A^T] in a new buffer, for an input x [rows, K] produced outside the block"""
        xa = self.alloc_in(x.shape[0], x.device)
        xa[:, :self.K].copy_(x)
        self.project(xa)
        return xa

    def keep(self, xa, recompute=False):
        """backward keeps only the adapter columns t of a LayerNorm output xa = [x | t]; x is recomputed (memory)"""
        return xa[:, self.K:].clone()

    def spare(self, xa):
        return None

    def rebuild(self, t, rows, device, ln):
        """[x | t] again in backward; `ln(out)` recomputes the LayerNorm output x into `out`"""
        xa = self.alloc_in(rows, device)
        ln(xa[:, :self.K])
        xa[:, self.K:].copy_(t)
        return xa

    def dgrad_out(self, xa):
        return None

    def project(self, xa):
        """t = x A^T into the tail columns of xa (rows of xa may be a slice of a larger buffer)"""
        ops.gemm(xa[:, :self.K], self.a_all, out=xa[:, self.K:])

    def backproject(self, dya):
        """dt = dy B into the tail columns of dya"""
        ops.gemm(dya[:, :self.N], self.b_blk, b_mn=True, out=dya[:, self.N:])

    def queue_grads(self, xa, dya, db=None):
        """dA_i = dt_i^T x,  dB_i = dy_i^T t_i   (weight-gradient work: deferred in the zero-bubble order).  xa, dya may
        be lists of row blocks (one per sample); `db`, the gradient of the frozen bias, is not used."""
        xas, dyas = (xa, dya) if isinstance(xa, list) else ([xa], [dya])

        def wgrad(self=self, xas=xas, dyas=dyas):
            K, N, r = self.K, self.N, self.r
            for xa, dya in zip(xas, dyas):
                row = 0
                for i, (a, b) in enumerate(zip(self.A, self.B)):
                    n = self.sizes[i]
                    if a.requires_grad:
                        g, acc = _grad_buf(a)
                        ops.gemm(dya[:, N + i * r:N + (i + 1) * r], xa[:, :K], a_mn=True, b_mn=True, out=g, accumulate=acc)
                    if b.requires_grad:
                        g, acc = _grad_buf(b)
                        ops.gemm(dya[:, row:row + n], xa[:, K + i * r:K + (i + 1) * r], a_mn=True, b_mn=True, out=g,
                                 accumulate=acc)
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

    def refresh(self):
        if self.fp8:
            _EPOCH[0] += 1

    def fwd(self, temb):
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


def _install(blk, lo):
    """the adapted sites replace the block's dense ones (`blk.sites`, read by the block functions); `blk.lora` keeps
    them, with the list of GEMM sites under 'sites', and marks the block as adapted"""
    blk.sites = dict(lo)
    lo['sites'] = [v for v in lo.values() if isinstance(v, LoraSite)]
    blk.__dict__['lora'] = lo
    _name_factors(blk)
    return lo


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
    for n in (a.norm_q, a.norm_k, a.norm_added_q, a.norm_added_k):
        n.weight.requires_grad_(False)                       # bias='none', no modules_to_save: only the factors train
    for fp, site in ((blk.qkv, lo['qkv']), (blk.add_qkv, lo['add_qkv'])):
        fp.weight, fp.bias = site.base_weight, site.bias   # drop the old fused storage (the site owns W now)
    return _install(blk, lo)


def attach_single_block(blk, rank, dtype=torch.bfloat16, base_dtype=None):
    a = blk.attn
    lo = {
        'mod': ModLora(blk.norm.linear, rank, dtype, base_dtype),
        'lin1': LoraSite([a.to_q, a.to_k, a.to_v, blk.proj_mlp], rank, dtype, base_dtype),
        'proj_out': LoraSite([blk.proj_out], rank, dtype, base_dtype),
    }
    for n in (a.norm_q, a.norm_k):
        n.weight.requires_grad_(False)
    blk.lin1.weight, blk.lin1.bias = lo['lin1'].base_weight, lo['lin1'].bias
    return _install(blk, lo)


def lora_state_dict(module):
    """{original_name: tensor} of the adapter factors only (what the reference's save_adapter receives)"""
    return {n: p.detach() for n, p in module.named_parameters() if '.lora_A.' in n or '.lora_B.' in n}


def attach_wan_block(blk, rank, dtype=torch.bfloat16, base_dtype=None):
    sa, ca = blk.self_attn, blk.cross_attn
    lo = {
        'sa_qkv': LoraSite([sa.q, sa.k, sa.v], rank, dtype, base_dtype), 'sa_o': LoraSite([sa.o], rank, dtype, base_dtype),
        'ca_q': LoraSite([ca.q], rank, dtype, base_dtype), 'ca_kv': LoraSite([ca.k, ca.v], rank, dtype, base_dtype), 'ca_o': LoraSite([ca.o], rank, dtype, base_dtype),
        'ffn1': LoraSite([blk.ffn[0]], rank, dtype, base_dtype), 'ffn2': LoraSite([blk.ffn[2]], rank, dtype, base_dtype),
    }
    for p in (sa.norm_q.weight, sa.norm_k.weight, ca.norm_q.weight, ca.norm_k.weight, blk.norm3.weight, blk.norm3.bias, blk.modulation):
        p.requires_grad_(False)
    sa.qkv.weight, sa.qkv.bias = lo['sa_qkv'].base_weight, lo['sa_qkv'].bias
    ca.kv.weight, ca.kv.bias = lo['ca_kv'].base_weight, lo['ca_kv'].bias
    return _install(blk, lo)
