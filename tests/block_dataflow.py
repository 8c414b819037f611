"""Launch recorder and dataflow specs of the block autograd Functions (FluxDoubleBlockFn, FluxSingleBlockFn, WanBlockFn).

**Recorder.**  `Recorder.install(monkeypatch, ops)` wraps every kernel wrapper a block calls, on top of whatever
implementation is installed (the real kernels, or tests/kernel_doubles.py).  For each call it keeps the op, its scalar
arguments, a clone of every tensor argument taken before the call (`pre`) and after it (`post`), the returned tensors
(`ret`), and the number of bytes of every argument's storage that the call changed outside its documented outputs
(`stray`, evaluated lazily on the device).  `make_qkv_epilogue` is wrapped too, so the tensors behind a QKV epilogue
struct appear as `qkv.<field>` arguments of the GEMM that uses it.  Clones are taken on the current stream: no
synchronisation, and no matching by data pointer.

**Specs.**  `spec_flux_double`, `spec_flux_single` and `spec_wan` restate, from the oracle's math (oracle/flux_ref.py,
oracle/qwen_ref.py, oracle/wan_ref.py, oracle/lora_ref.py), the launches one forward plus backward must make: op and
scalars, where every operand it reads comes from (a block input, a parameter, an operand built from the parameters,
or an earlier call's output), and the torch glue between calls, recomputed on the recorded values.  `Replay.take`
matches the next recorded call against that statement, bit for bit; the weight-gradient GEMMs may instead come after
the queue of deferred weight-gradient work drains (`ops.WGRAD_DEFER`), and nothing else may move.  At the end the
block's outputs, the input gradients and every trained parameter's `.grad` must equal the value the spec assembled.

Operand names: `W` / `b` a linear's weight and bias; LoRA (oracle/lora_ref.py: y = x W^T + b + (x A^T) B^T) runs as a
K-extension, [x | x A^T] [W | B]^T forward and [dy | dy B] [W ; A] backward, with the A's of the projections a site
consumes fused stacked and their B's block-diagonal.  An fp8 base is widened exactly to bf16 (the reference's
autocast) into one operand buffer shared by every site, so the spec expects a widening launch whenever a site's
operand is needed and the buffer last held another site's (or an earlier forward's).
"""
import inspect

import torch

WRAPPED = ('gemm', 'attn_fwd', 'attn_bwd', 'ln_modulate_fwd', 'ln_modulate_bwd', 'gate_bwd', 'colreduce_finish', 'colsum',
           'qknorm_rope_bwd', 'wan_norm_rope_fwd', 'wan_norm_rope_bwd', 'mod_fwd', 'mod_bwd', 'fp8_to_bf16')
EPI_STORE, EPI_BIAS_GELU, EPI_GATE_RES, EPI_QKV_ROPE, EPI_MUL_GELU_GRAD = 0, 1, 2, 3, 4
HD = 128
_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits(t):
    return t.detach().contiguous().view(_INT[t.element_size()])


def same_bits(a, b):
    return a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and torch.equal(bits(a), bits(b))


# =====================================================================================================================
# recorder
# =====================================================================================================================
class Call:
    __slots__ = ('index', 'op', 'scalars', 'defaults', 'live', 'pre', 'post', 'ret', 'stray', 'phase')

    def __repr__(self):
        return f'call {self.index} ({self.op})'


def _flatten(op, bound, epis):
    """named tensors and scalars of one call (nested: QKV epilogue fields, the projection dicts of the Wan kernels)"""
    tensors, scalars = {}, {}
    for name, v in bound.items():
        if torch.is_tensor(v):
            tensors[name] = v
        elif name == 'qkv' and v is not None:
            for k, x in epis[id(v)].items():
                (tensors if torch.is_tensor(x) or x is None else scalars)[f'qkv.{k}'] = x
            tensors = {k: x for k, x in tensors.items() if x is not None}
        elif name == 'projs':
            for i, pj in enumerate(v):
                for k, x in pj.items():
                    (tensors if torch.is_tensor(x) else scalars)[f'projs[{i}].{k}'] = x
        elif v is None or isinstance(v, (bool, int, float)):
            scalars[name] = v
    return tensors, scalars


def _outputs(op, t, s, ret):
    """the tensor views a call may write: its documented outputs"""
    g = t.get
    if op == 'gemm':
        outs = [ret]
        if s['epilogue'] == EPI_QKV_ROPE:
            b = t['b']
            n = b.shape[1] if s['b_mn'] else b.shape[0]
            if n <= s['qkv.n_qkv']:
                outs = []
            elif 'out2' in t:
                outs.append(t['out2'])
            L = t['a'].shape[1] if s['a_mn'] else t['a'].shape[0]
            L = s['rows_per_batch'] or L
            sl = slice(s['qkv.seq_offset'], s['qkv.seq_offset'] + L)
            outs += [t[f'qkv.{k}'][:, :, sl] for k in ('q', 'k', 'v', 'qhat', 'khat', 'q_rstd', 'k_rstd') if f'qkv.{k}' in t]
        elif 'out2' in t:
            outs.append(t['out2'])
        return outs
    if op == 'attn_fwd':
        return [ret[0][:, :t['q'].shape[1] * HD], ret[1]]
    if op == 'attn_bwd':
        return [x for x in (g('dq'), g('dk'), g('dv'), g('delta')) if x is not None]
    if op in ('ln_modulate_bwd', 'gate_bwd'):
        return [ret[0], ret[1]]
    if op == 'ln_modulate_fwd':
        return [ret[0]]
    if op == 'colreduce_finish':
        return [x for x in (g('per_sample0'), g('per_sample1'), g('summed0'), g('summed1')) if x is not None]
    if op == 'colsum':
        return [ret]
    if op == 'qknorm_rope_bwd':
        C = 3 * s['heads'] * HD
        return [t['dqkv'][:, :C], t['dbias'][:C], t['dw']]
    if op == 'wan_norm_rope_bwd':
        C = s['heads'] * HD
        return [v[:, :C] for k, v in t.items() if k.endswith('.dx')]
    if op == 'mod_bwd':
        return [x for x in (g('wgrad'), t['dtemb32']) if x is not None]
    if op == 'fp8_to_bf16':
        return [t['dst']]
    return []      # wan_norm_rope_fwd, mod_fwd: every output is a new tensor


def _storage_bytes(t):
    return torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage())


def _mark(mask, t):
    """sets the bytes of view t in `mask` (a uint8 vector over t's storage)"""
    es = t.element_size()
    idx = torch.arange(mask.numel() // es, device=mask.device).as_strided(t.shape, t.stride(), t.storage_offset())
    for k in range(es):
        mask[idx.reshape(-1) * es + k] = 1


class Recorder:
    def __init__(self):
        self.calls = []
        self.epis = {}
        self.phase = None
        self._depth = 0

    def install(self, monkeypatch, ops):
        for name in WRAPPED:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))
        real = ops.make_qkv_epilogue
        sig = inspect.signature(real)

        def make_qkv_epilogue(*a, **k):
            e = real(*a, **k)
            b = sig.bind(*a, **k)
            b.apply_defaults()
            d = dict(b.arguments)
            d['n_qkv'] = 3 * d['heads'] * HD
            self.epis[id(e)] = d
            self.epis.setdefault('_keep', []).append(e)
            return e
        monkeypatch.setattr(ops, 'make_qkv_epilogue', make_qkv_epilogue)
        return self

    def _wrap(self, op, real):
        sig = inspect.signature(real)

        def wrapper(*a, **k):
            if self._depth:                       # a wrapper calling another one (wan_norm_rope_bwd -> colreduce_finish)
                return real(*a, **k)
            b = sig.bind(*a, **k)
            b.apply_defaults()
            tensors, scalars = _flatten(op, b.arguments, self.epis)
            c = Call()
            c.index, c.op, c.scalars, c.live, c.phase = len(self.calls), op, scalars, tensors, self.phase
            c.defaults = {n: p.default for n, p in sig.parameters.items() if p.default is not inspect.Parameter.empty}
            c.pre = {n: x.clone() for n, x in tensors.items()}
            storages = {}
            for x in tensors.values():
                storages.setdefault(x.untyped_storage().data_ptr(), x)
            before = {p: _storage_bytes(x).clone() for p, x in storages.items()}
            self._depth += 1
            try:
                r = real(*a, **k)
            finally:
                self._depth -= 1
            c.post = {n: x.clone() for n, x in tensors.items()}
            c.ret = tuple(x.clone() if torch.is_tensor(x) else x for x in r) if isinstance(r, (tuple, list)) else (
                r.clone() if torch.is_tensor(r) else r)
            if op == 'wan_norm_rope_fwd':
                c.ret = [tuple(x.clone() if x is not None else None for x in o) for o in r]
            c.stray = []
            outs = [o for o in _outputs(op, tensors, scalars, r) if torch.is_tensor(o)]
            for p, x in storages.items():
                now = _storage_bytes(x)
                mask = torch.zeros_like(now)
                for o in outs:
                    if o.untyped_storage().data_ptr() == p:
                        _mark(mask, o)
                c.stray.append(((before[p] != now) & (mask == 0)).sum())
            self.calls.append(c)
            return r
        return wrapper


# =====================================================================================================================
# replay: matching recorded calls against a spec
# =====================================================================================================================
class SpecError(AssertionError):
    pass


def _reads(c):
    """name -> (pre-call value) of every operand the call reads"""
    t, s = c.pre, c.scalars
    op = c.op
    keep = lambda *names: {n: t[n] for n in names if n in t}
    if op == 'gemm':
        r = keep('a', 'b', 'bias')
        if s['epilogue'] in (EPI_GATE_RES, EPI_MUL_GELU_GRAD):
            r.update(keep('aux'))
        if s['epilogue'] == EPI_GATE_RES:
            r.update(keep('gate'))
        if s['accumulate']:
            r['out'] = t['out']
        if s['epilogue'] == EPI_QKV_ROPE:
            r.update(keep('qkv.q_norm_w', 'qkv.k_norm_w', 'qkv.rope_cos', 'qkv.rope_sin'))
        return r
    if op == 'attn_fwd':
        return keep('q', 'k', 'v')
    if op == 'attn_bwd':
        C = t['q'].shape[1] * HD
        return {'q': t['q'], 'k': t['k'], 'v': t['v'], 'o': t['o'][:, :C], 'd_o': t['d_o'][:, :C], 'lse': t['lse']}
    if op == 'ln_modulate_fwd':
        return keep('x', 'scale', 'shift')
    if op == 'ln_modulate_bwd':
        return keep('dxn', 'x', 'scale', 'mean', 'rstd', 'dres')
    if op == 'gate_bwd':
        return keep('dx', 'y', 'gate')
    if op == 'colreduce_finish':
        return keep('partials')
    if op == 'colsum':
        return keep('x')
    if op == 'qknorm_rope_bwd':
        return keep('dq', 'dk', 'dv', 'qhat', 'khat', 'q_rstd', 'k_rstd', 'q_norm_w', 'k_norm_w', 'rope_cos', 'rope_sin',
                    'dbias', 'dw')
    if op == 'wan_norm_rope_fwd':
        C = s['heads'] * HD
        r = {n: (v[:, :C] if n.endswith('.src') else v) for n, v in t.items()}
        return r
    if op == 'wan_norm_rope_bwd':
        return {n: v for n, v in t.items() if not n.endswith('.dx')}
    if op == 'mod_fwd':
        return keep('temb', 'weight', 'bias')
    if op == 'mod_bwd':
        r = keep('dmod32', 'temb', 'weight', 'dtemb32')
        if s['accumulate']:
            r['wgrad'] = t['wgrad']
        return r
    if op == 'fp8_to_bf16':
        return keep('src')
    raise KeyError(op)


SCALAR_OPERAND = {   # the operand a scalar decides about, named in a mismatch message
    'accumulate': "out (the gradient it adds to)", 'qkv.seq_offset': 'qkv.q/k/v/qhat/khat/q_rstd/k_rstd (rows written)',
    'rows_per_batch': 'gate (the row each sample reads)', 'seq_offset': 'dq/dk/dv (rows read)',
    'M': 'a / out (rows)', 'N': 'b / out (columns)', 'K': 'a / b (reduction length)', 'cta_group': 'b (tile sharing)'}


class Replay:
    """walks one micro-batch's recorded calls: `main` (forward and input-gradient pass) and `drained` (the deferred
    weight-gradient queue, empty when weight gradients run immediately)"""

    def __init__(self, main, drained, deferred):
        self.main, self.drained, self.deferred = list(main), list(drained), deferred
        self.i = self.j = 0
        self.matched = []

    def take(self, op, operands, wgrad=False, present=None, why=None, **scalars):
        """the next recorded call, checked against `op`, its `scalars` (every top-level scalar the spec does not name
        must keep the wrapper's default), the outputs it must be given (`present`) and its operands.  `why` names
        what the call provides, for the message when it is missing."""
        lst, pos = (self.drained, self.j) if (wgrad and self.deferred) else (self.main, self.i)
        where = 'the drained weight-gradient queue' if lst is self.drained else 'the block pass'
        want = f'{op} (operand {next(iter(operands), "-")}: {why})' if why else op
        if pos >= len(lst):
            raise SpecError(f'{want}: spec expects one more call in {where}, none was made')
        c = lst[pos]
        if lst is self.drained:
            self.j += 1
        else:
            self.i += 1
        if c.op != op:
            raise SpecError(f'{c!r}: spec expects {want} here')
        for k, v in scalars.items():
            if c.scalars.get(k, None) != v:
                raise SpecError(f'{c!r}: scalar {k} = {c.scalars.get(k)!r}, spec {v!r}'
                                + (f' (operand {SCALAR_OPERAND[k]})' if k in SCALAR_OPERAND else ''))
        for k, v in c.scalars.items():
            if k not in scalars and k in c.defaults and v != c.defaults[k]:
                raise SpecError(f'{c!r}: scalar {k} = {v!r}, spec keeps the default {c.defaults[k]!r}'
                                + (f' (operand {SCALAR_OPERAND[k]})' if k in SCALAR_OPERAND else ''))
        if present is not None:
            got = {n for n in ('per_sample0', 'per_sample1', 'summed0', 'summed1', 'wgrad') if n in c.live}
            for n in sorted(set(present) - got):
                raise SpecError(f'{c!r}: output operand {n} missing (given: {sorted(got)})')
            for n in sorted(got - set(present)):
                raise SpecError(f'{c!r}: output operand {n} given, the spec has none')
        reads = _reads(c)
        for n, src in operands.items():
            if src is None:
                if n in reads:
                    raise SpecError(f'{c!r}: operand {n} given, the spec has none')
                continue
            if n not in reads:
                raise SpecError(f'{c!r}: operand {n} missing')
            if not same_bits(reads[n], src):
                got = reads[n]
                detail = (f'shape {tuple(got.shape)} vs {tuple(src.shape)}' if tuple(got.shape) != tuple(src.shape) else
                          f'dtype {got.dtype} vs {src.dtype}' if got.dtype != src.dtype else
                          f'{int((bits(got) != bits(src)).sum())} of {src.numel()} elements differ')
                raise SpecError(f'{c!r}: operand {n} differs from its source ({detail})')
        for n in reads:
            if n not in operands:
                raise SpecError(f'{c!r}: operand {n} has no source in the spec')
        stray = [int(n) for n in c.stray]
        if any(stray):
            raise SpecError(f'{c!r}: {sum(stray)} bytes written outside its documented outputs')
        self.matched.append(c)
        return c

    def done(self):
        for lst, pos, where in ((self.main, self.i, 'block pass'), (self.drained, self.j, 'drained queue')):
            if pos < len(lst):
                raise SpecError(f'{lst[pos]!r}: extra call in the {where}, the spec expects none')


def expect_equal(got, want, what):
    if got is None or want is None:
        if got is not None or want is not None:
            raise SpecError(f'{what}: {"None" if got is None else "a tensor"}, spec {"None" if want is None else "a tensor"}')
        return
    if not same_bits(got, want):
        n = int((bits(got) != bits(want)).sum()) if tuple(got.shape) == tuple(want.shape) and got.dtype == want.dtype else -1
        raise SpecError(f'{what}: differs from the value assembled from the recorded calls ({n} elements, '
                        f'{got.dtype} {tuple(got.shape)} vs {want.dtype} {tuple(want.shape)})')


# =====================================================================================================================
# operands built from the parameters, and the spec's state
# =====================================================================================================================
FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)
BF = torch.bfloat16
F32 = torch.float32


def _cat8(ts, dim=0):
    """torch.cat for fp8 tensors too (through their bytes)"""
    if ts[0].dtype in FP8:
        return torch.cat([t.detach().view(torch.uint8) for t in ts], dim).view(ts[0].dtype)
    return torch.cat([t.detach() for t in ts], dim)


class Spec:
    """one micro-batch's replay plus the state that outlives it: `grads` (id(param) -> (param, expected .grad)) and
    `snap` (id(param) -> the parameter's value when this micro-batch ran)"""

    def __init__(self, rp, grads, snap):
        self.rp, self.grads, self.snap = rp, grads, snap
        self.owner = None           # what the shared fp8 operand buffer holds

    def P(self, p):
        return self.snap[id(p)]

    def take(self, op, operands, **kw):
        return self.rp.take(op, operands, **kw)

    def new_forward(self):
        self.owner = None           # every block forward starts a new epoch of the operand buffer

    def widen(self, key, w8):
        """fp8 base: the operand buffer is refilled unless it still holds `key` from this pass"""
        if self.owner != key:
            self.take('fp8_to_bf16', {'src': w8}, why=f'fp8 base of {key}, widened into the operand buffer')
            self.owner = key

    def prev_grad(self, p):
        """expected gradient so far of a parameter, or of a fused matrix (a string key)"""
        g = self.grads.get(p if isinstance(p, str) else id(p))
        return None if g is None else g[1]

    def set_grad(self, p, g):
        if isinstance(p, str):
            self.grads[p] = (None, g)
        else:
            self.grads[id(p)] = (p, g)

    def acc_vec(self, p, g32):
        """a bias / norm weight / modulation factor gradient: bf16(g) the first time, then .grad += g (fp32 operand)"""
        if not p.requires_grad:
            return
        prev = self.prev_grad(p)
        self.set_grad(p, g32.to(p.dtype).view_as(p) if prev is None else prev.clone().add_(g32.view_as(p)))

    def wgrad_gemm(self, p, a, b, view=None):
        """dW (+)= a^T b (both MN-major) into p's gradient (`view`: the rows of a fused gradient it fills)"""
        prev = self.prev_grad(p)
        acc = prev is not None
        c = self.take('gemm', {'a': a, 'b': b, 'bias': None, 'out': prev}, wgrad=True, epilogue=EPI_STORE, a_mn=True,
                      b_mn=True, accumulate=acc, rows_per_batch=None)
        self.set_grad(p, c.ret)
        return c


class Site:
    """a GEMM over one or several linears consumed as one [N, K] matrix (q, k, v fused), with their LoRA factors when
    adapted.  Everything here is built from the parameters' values of the current micro-batch."""

    def __init__(self, sp, name, lins):
        self.sp, self.name, self.lins = sp, name, list(lins)
        w = self.lins[0].weight
        self.fp8 = w.dtype in FP8
        self.lora = hasattr(self.lins[0], 'lora_A')
        self.K = w.shape[1]
        self.sizes = [l.weight.shape[0] for l in self.lins]
        self.N = sum(self.sizes)
        self.r = self.lins[0].lora_A.weight.shape[0] if self.lora else 0
        self.R = self.r * len(self.lins)

    @property
    def trained(self):
        return not self.lora and self.lins[0].weight.requires_grad

    def W(self):
        return _cat8([self.sp.P(l.weight) for l in self.lins]).to(BF)

    def bias(self):
        return _cat8([self.sp.P(l.bias) for l in self.lins]).to(BF)

    def A(self):              # stacked A's [R, K]
        return torch.cat([self.sp.P(l.lora_A.weight) for l in self.lins])

    def Bblk(self):           # block-diagonal B's [N, R]
        return torch.block_diag(*[self.sp.P(l.lora_B.weight) for l in self.lins])

    def _widen(self):
        if self.fp8:
            self.sp.widen(self.name, _cat8([self.sp.P(l.weight) for l in self.lins]))

    def fwd_operand(self):    # [W | B]
        self._widen()
        return torch.cat([self.W(), self.Bblk()], 1) if self.lora else self.W()

    def dgrad_operand(self):  # [W ; A]
        self._widen()
        return torch.cat([self.W(), self.A()], 0) if self.lora else self.W()

    def project(self, x):
        """[x | x A^T]"""
        if not self.lora:
            return x
        c = self.sp.take('gemm', {'a': x, 'b': self.A(), 'bias': None}, epilogue=EPI_STORE, a_mn=False, b_mn=False,
                         accumulate=False, rows_per_batch=None)
        return torch.cat([x, c.ret], 1)

    def backproject(self, dy):
        """[dy | dy B]"""
        if not self.lora:
            return dy
        c = self.sp.take('gemm', {'a': dy, 'b': self.Bblk(), 'bias': None}, epilogue=EPI_STORE, a_mn=False, b_mn=True,
                         accumulate=False, rows_per_batch=None)
        return torch.cat([dy, c.ret], 1)

    def fwd(self, xa, epilogue=EPI_STORE, rows_per_batch=None, extra=None, **scalars):
        b = self.fwd_operand()
        ops_ = {'a': xa, 'b': b, 'bias': self.bias()}
        ops_.update(extra or {})
        return self.sp.take('gemm', ops_, epilogue=epilogue, a_mn=False, b_mn=False, accumulate=False,
                            rows_per_batch=rows_per_batch, **scalars)

    def dgrad(self, dya, epilogue=EPI_STORE, extra=None, cols=None):
        w = self.dgrad_operand()
        ops_ = {'a': dya, 'b': w if cols is None else w[:, cols], 'bias': None}
        ops_.update(extra or {})
        return self.sp.take('gemm', ops_, epilogue=epilogue, a_mn=False, b_mn=True, accumulate=False, rows_per_batch=None)

    def rebuild(self, kept, ln, recompute=False):
        """the operand [x | t] again in backward: dense sites keep x unless the block recomputes it (Wan); adapted ones
        recompute the LayerNorm (`ln()` takes that call and returns its output) and keep only the adapter columns t"""
        if not self.lora:
            return ln() if recompute else kept
        return torch.cat([ln(), kept[:, self.K:]], 1)

    def wgrad(self, xs, dys, db):
        """dense: dW (+)= sum_i dy_i^T x_i, b (+)= db.  LoRA: dA_j (+)= dt_j^T x, dB_j (+)= dy_j^T t_j per sample"""
        sp = self.sp
        if self.lora:
            K, N, r = self.K, self.N, self.r
            for xa, dya in zip(xs, dys):
                row = 0
                for j, l in enumerate(self.lins):
                    n = self.sizes[j]
                    sp.wgrad_gemm(l.lora_A.weight, dya[:, N + j * r:N + (j + 1) * r], xa[:, :K])
                    sp.wgrad_gemm(l.lora_B.weight, dya[:, row:row + n], xa[:, K + j * r:K + (j + 1) * r])
                    row += n
            return
        if not self.trained:
            return
        wkey, bkey = 'W ' + self.name, 'b ' + self.name
        for x, dy in zip(xs, dys):
            sp.wgrad_gemm(wkey, dy, x)
        g = sp.prev_grad(wkey)
        bprev = sp.prev_grad(bkey)
        bnew = db.to(BF) if bprev is None else bprev.clone().add_(db)
        sp.set_grad(bkey, bnew)
        row = 0
        for j, l in enumerate(self.lins):      # the per-projection parameters' .grad are row blocks of the fused one
            n = self.sizes[j]
            sp.set_grad(l.weight, g[row:row + n])
            sp.set_grad(l.bias, bnew[row:row + n])
            row += n


class Mod:
    """a modulation linear mod = W silu(temb) + b (oracle RefAdaLayerNormZero / AdaLayerNormZeroSingle), LoRA on [B, r]"""

    def __init__(self, sp, name, lin):
        self.sp, self.name, self.lin = sp, name, lin
        self.fp8 = lin.weight.dtype in FP8
        self.lora = hasattr(lin, 'lora_A')

    def W(self):
        w = self.sp.P(self.lin.weight)
        if self.fp8:
            self.sp.widen(self.name, w)
        return w.to(BF)

    def fwd(self, temb):
        sp = self.sp
        if self.lora:
            A, B = sp.P(self.lin.lora_A.weight), sp.P(self.lin.lora_B.weight)
            self.s = torch.nn.functional.silu(temb.float()).to(BF)                  # bf16 conditioning vector
            self.t = (self.s.float() @ A.float().t()).to(BF)                          # lora_A output
        c = sp.take('mod_fwd', {'temb': temb, 'weight': self.W(), 'bias': sp.P(self.lin.bias)})
        if not self.lora:
            return c.ret
        return (c.ret.float() + (self.t.float() @ B.float().t()).to(BF).float()).to(BF)

    def bwd(self, dmod, temb, dtemb):
        sp = self.sp
        trained = self.lin.weight.requires_grad
        prev = sp.prev_grad(self.lin.weight) if trained else None
        c = sp.take('mod_bwd', {'dmod32': dmod, 'temb': temb, 'weight': self.W(), 'dtemb32': dtemb, 'wgrad': prev},
                    accumulate=prev is not None, present=['wgrad'] if trained else [])
        dtemb = c.post['dtemb32']
        if trained:
            sp.set_grad(self.lin.weight, c.post['wgrad'])
            sp.acc_vec(self.lin.bias, c.ret)
        if self.lora:
            A, B = sp.P(self.lin.lora_A.weight), sp.P(self.lin.lora_B.weight)
            d = dmod.to(BF).float()                                                  # the bf16 gradient of mod
            dt = d @ B.float()
            sp.acc_vec(self.lin.lora_B.weight, d.t() @ self.t.float())
            sp.acc_vec(self.lin.lora_A.weight, dt.t() @ self.s.float())
            ds = dt @ A.float()
            tf = temb.float()
            sg = torch.sigmoid(tf)
            dtemb = dtemb.clone()
            dtemb.add_(ds.to(BF).float() * (sg * (1 + tf * (1 - sg))))
        return dtemb


def _finish(sp, part, present):
    c = sp.take('colreduce_finish', {'partials': part}, present=present)
    return c.post


def _ln_fwd(sp, x, scale, shift, B, L, save_stats=True, eps=1e-6, flags=0):
    c = sp.take('ln_modulate_fwd', {'x': x, 'scale': scale, 'shift': shift}, batch=B, rows_per_batch=L, eps=eps,
                save_stats=save_stats, flags=flags)
    return c.ret


def _qkv_scalars(H, Ltot, off):
    return {'qkv.heads': H, 'qkv.seq_total': Ltot, 'qkv.seq_offset': off, 'qkv.eps': 1e-6}


# =====================================================================================================================
# Flux / Qwen-Image double-stream block  (oracle/flux_ref.py RefFluxTransformerBlock, oracle/qwen_ref.py
# RefQwenImageTransformerBlock with its key mask)
# =====================================================================================================================
class _S:
    pass


def spec_flux_double(sp, blk, hidden, enc, temb, cos, sin, d_hidden, d_enc, txt_lens=None):
    """returns (image output, text output, d hidden, d enc, d temb) assembled from the recorded calls"""
    B, Li, D = hidden.shape
    Lt = enc.shape[1]
    Ltot = Li + Lt
    H = blk.heads
    C = H * HD
    a = blk.attn
    img, txt = _S(), _S()
    for s, x3, L, off, lin_mod, qkv, nq, nk, to_out, ff, dout, nm in (
            (img, hidden, Li, Lt, blk.norm1.linear, [a.to_q, a.to_k, a.to_v], a.norm_q, a.norm_k, a.to_out[0], blk.ff,
             d_hidden, 'img'),
            (txt, enc, Lt, 0, blk.norm1_context.linear, [a.add_q_proj, a.add_k_proj, a.add_v_proj], a.norm_added_q,
             a.norm_added_k, a.to_add_out, blk.ff_context, d_enc, 'txt')):
        s.x, s.L, s.off, s.nq, s.nk, s.dout = x3.reshape(B * L, D), L, off, nq, nk, dout.reshape(B * L, D)
        s.mod = Mod(sp, nm + '.mod', lin_mod)
        s.qkv, s.o = Site(sp, nm + '.qkv', qkv), Site(sp, nm + '.o', [to_out])
        s.f1, s.f2 = Site(sp, nm + '.ff1', [ff.net[0].proj]), Site(sp, nm + '.ff2', [ff.net[2]])
    streams = (img, txt)
    sp.new_forward()
    # ---- forward: norm1 / norm1_context, joint q k v (text rows first), RMSNorm(q, k), RoPE ----
    for s in streams:
        s.m = m = s.mod.fwd(temb)         # [B, 6D] = shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp
        xn, s.mean1, s.rstd1 = _ln_fwd(sp, s.x, m[:, D:2 * D], m[:, 0:D], B, s.L)
        s.xa = s.qkv.project(xn)
        s.cq = s.qkv.fwd(s.xa, EPI_QKV_ROPE, s.L, extra={'qkv.q_norm_w': sp.P(s.nq.weight), 'qkv.k_norm_w': sp.P(s.nk.weight),
                                                       'qkv.rope_cos': cos, 'qkv.rope_sin': sin}, **_qkv_scalars(H, Ltot, s.off))

    def joint(f):
        return torch.cat([txt.cq.post[f'qkv.{f}'][:, :, :Lt], img.cq.post[f'qkv.{f}'][:, :, Lt:]], 2)
    q, k, v, qhat, khat, q_rstd, k_rstd = (joint(f) for f in ('q', 'k', 'v', 'qhat', 'khat', 'q_rstd', 'k_rstd'))
    if txt_lens is None:
        c = sp.take('attn_fwd', {'q': q, 'k': k, 'v': v}, scale=None)
        o, lse = c.post['out'][:, :C], c.ret[1]
    else:
        # key mask: sample b attends over its n_b real prompt tokens and every image token; padded rows output 0
        o = torch.zeros((B * Ltot, C), dtype=BF, device=q.device)
        o3, ragged = o.view(B, Ltot, C), []
        for b, n in enumerate(txt_lens):
            idx = torch.cat([torch.arange(int(n)), torch.arange(Lt, Ltot)]).to(q.device)
            qb, kb, vb = (t[b:b + 1].index_select(2, idx) for t in (q, k, v))
            c = sp.take('attn_fwd', {'q': qb, 'k': kb, 'v': vb}, scale=None)
            o3[b].index_copy_(0, idx, c.ret[0][:, :C])
            ragged.append((idx, qb, kb, vb, c.ret[0], c.ret[1]))
    o3 = o.view(B, Ltot, C)
    outs = []
    for s in streams:
        L, off, m = s.L, s.off, s.m
        s.oa, x1, y = [], [], []
        for b in range(B):                # to_out / to_add_out over this stream's rows of sample b: x1 = x + gate_msa y
            ra = s.o.project(o3[b, off:off + L])
            c = s.o.fwd(ra, EPI_GATE_RES, L, extra={'aux': s.x[b * L:(b + 1) * L], 'gate': m[b:b + 1, 2 * D:3 * D]})
            s.oa.append(ra)
            x1.append(c.ret)
            y.append(c.post['out2'])
        s.x1, s.y_attn = torch.cat(x1), torch.cat(y)
        xn2, s.mean2, s.rstd2 = _ln_fwd(sp, s.x1, m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L)
        s.x2a = s.f1.project(xn2)
        c = s.f1.fwd(s.x2a, EPI_BIAS_GELU)
        s.u = c.post['out2']
        s.ha = s.f2.project(c.ret)
        c = s.f2.fwd(s.ha, EPI_GATE_RES, L, extra={'aux': s.x1, 'gate': m[:, 5 * D:6 * D]})
        s.y_mlp = c.post['out2']
        outs.append(c.ret.view(B, L, D))
    # ---- backward ----
    d_o = torch.full((B * Ltot, C), float('nan'), dtype=BF, device=q.device)
    d_o3 = d_o.view(B, Ltot, C)
    for s in streams:
        L, off, m = s.L, s.off, s.m
        s.dmod = torch.full((B, 6 * D), float('nan'), dtype=F32, device=q.device)
        dy2, part = sp.take('gate_bwd', {'dx': s.dout, 'y': s.y_mlp, 'gate': m[:, 5 * D:6 * D]}, batch=B,
                            rows_per_batch=L).ret
        f = _finish(sp, part, ['per_sample0'] + (['summed1'] if s.f2.trained else []))
        s.dmod[:, 5 * D:6 * D] = f['per_sample0']
        dy2a = s.f2.backproject(dy2)
        du = s.f2.dgrad(dy2a, EPI_MUL_GELU_GRAD, extra={'aux': s.u}).ret
        s.f2.wgrad([s.ha], [dy2a], f.get('summed1'))
        dua = s.f1.backproject(du)
        x2a = s.f1.rebuild(s.x2a, lambda: _ln_fwd(sp, s.x1, m[:, 4 * D:5 * D], m[:, 3 * D:4 * D], B, L, save_stats=False)[0])
        db1 = sp.take('colsum', {'x': dua}).ret if s.f1.trained else None
        s.f1.wgrad([x2a], [dua], db1)
        dxn2 = s.f1.dgrad(dua).ret
        s.dx1, part = sp.take('ln_modulate_bwd', {'dxn': dxn2, 'x': s.x1, 'scale': m[:, 4 * D:5 * D], 'mean': s.mean2,
                                                  'rstd': s.rstd2, 'dres': s.dout}, batch=B, rows_per_batch=L, flags=0).ret
        f = _finish(sp, part, ['per_sample0', 'per_sample1'])
        s.dmod[:, 4 * D:5 * D], s.dmod[:, 3 * D:4 * D] = f['per_sample0'], f['per_sample1']
        dy1, part = sp.take('gate_bwd', {'dx': s.dx1, 'y': s.y_attn, 'gate': m[:, 2 * D:3 * D]}, batch=B,
                            rows_per_batch=L).ret
        f = _finish(sp, part, ['per_sample0'] + (['summed1'] if s.o.trained else []))
        s.dmod[:, 2 * D:3 * D] = f['per_sample0']
        dy1a = s.o.backproject(dy1)
        for b in range(B):
            d_o3[b, off:off + L] = s.o.dgrad(dy1a[b * L:(b + 1) * L]).ret
        s.o.wgrad(s.oa, [dy1a[b * L:(b + 1) * L] for b in range(B)], f.get('summed1'))
    if txt_lens is None:
        dq, dk, dv = sp.take('attn_bwd', {'q': q, 'k': k, 'v': v, 'o': o, 'd_o': d_o, 'lse': lse}, scale=None).ret
    else:
        dq, dk, dv = (torch.zeros_like(q) for _ in range(3))
        for b, (idx, qb, kb, vb, ob, lse_b) in enumerate(ragged):
            g = sp.take('attn_bwd', {'q': qb, 'k': kb, 'v': vb, 'o': ob[:, :C], 'd_o': d_o3[b].index_select(0, idx),
                                     'lse': lse_b}, scale=None).ret
            for t, gb in zip((dq, dk, dv), g):
                t[b].index_copy_(1, idx, gb[0])
    dtemb = torch.zeros(temb.shape, dtype=F32, device=q.device)
    grads = []
    for s in streams:
        L, off, m = s.L, s.off, s.m
        c = sp.take('qknorm_rope_bwd', {'dq': dq, 'dk': dk, 'dv': dv, 'qhat': qhat, 'khat': khat, 'q_rstd': q_rstd,
                                        'k_rstd': k_rstd, 'q_norm_w': sp.P(s.nq.weight), 'k_norm_w': sp.P(s.nk.weight),
                                        'rope_cos': cos, 'rope_sin': sin,
                                        'dbias': torch.zeros(3 * C, dtype=F32, device=q.device),
                                        'dw': torch.zeros((2, HD), dtype=F32, device=q.device)},
                    batch=B, heads=H, seq_total=Ltot, seq_offset=off, rows_per_batch=L)
        sp.acc_vec(s.nq.weight, c.post['dw'][0])
        sp.acc_vec(s.nk.weight, c.post['dw'][1])
        dqa = s.qkv.backproject(c.post['dqkv'][:, :3 * C])
        xa = s.qkv.rebuild(s.xa, lambda: _ln_fwd(sp, s.x, m[:, D:2 * D], m[:, 0:D], B, L, save_stats=False)[0])
        s.qkv.wgrad([xa], [dqa], c.post['dbias'])
        dxn = s.qkv.dgrad(dqa).ret
        dx, part = sp.take('ln_modulate_bwd', {'dxn': dxn, 'x': s.x, 'scale': m[:, D:2 * D], 'mean': s.mean1,
                                               'rstd': s.rstd1, 'dres': s.dx1}, batch=B, rows_per_batch=L, flags=0).ret
        f = _finish(sp, part, ['per_sample0', 'per_sample1'])
        s.dmod[:, D:2 * D], s.dmod[:, 0:D] = f['per_sample0'], f['per_sample1']
        dtemb = s.mod.bwd(s.dmod, temb, dtemb)
        grads.append(dx.view(B, L, D))
    return outs[0], outs[1], grads[0], grads[1], dtemb.to(temb.dtype)


# =====================================================================================================================
# Flux single-stream block  (oracle/flux_ref.py RefFluxSingleTransformerBlock: [text; image] one sequence)
# =====================================================================================================================
def spec_flux_single(sp, blk, hidden, enc, temb, cos, sin, d_hidden, d_enc):
    B, Li, D = hidden.shape
    Lt = enc.shape[1]
    L = Li + Lt
    H = blk.heads
    C = H * HD
    a = blk.attn
    inner = blk.mlp_dim
    mod = Mod(sp, 'mod', blk.norm.linear)
    s1 = Site(sp, 'lin1', [a.to_q, a.to_k, a.to_v, blk.proj_mlp])
    s2 = Site(sp, 'proj_out', [blk.proj_out])
    sp.new_forward()
    x = torch.cat([enc, hidden], 1).reshape(B * L, D)
    m = mod.fwd(temb)                         # [B, 3D] = shift, scale, gate
    xn, mean, rstd = _ln_fwd(sp, x, m[:, D:2 * D], m[:, 0:D], B, L)
    xa = s1.project(xn)
    c = s1.fwd(xa, EPI_QKV_ROPE, L, extra={'qkv.q_norm_w': sp.P(a.norm_q.weight), 'qkv.k_norm_w': sp.P(a.norm_k.weight),
                                           'qkv.rope_cos': cos, 'qkv.rope_sin': sin}, **_qkv_scalars(H, L, 0))
    q, k, v, qhat, khat, q_rstd, k_rstd = (c.post[f'qkv.{f}'] for f in ('q', 'k', 'v', 'qhat', 'khat', 'q_rstd', 'k_rstd'))
    h_mlp, u = c.post['out'], c.post['out2']                 # gelu(proj_mlp(xn)) and its pre-activation
    c = sp.take('attn_fwd', {'q': q, 'k': k, 'v': v}, scale=None)
    attn, lse = c.post['out'][:, :C], c.ret[1]
    cata = s2.project(torch.cat([attn, h_mlp], 1))           # proj_out(cat(attn, mlp))
    c = s2.fwd(cata, EPI_GATE_RES, L, extra={'aux': x, 'gate': m[:, 2 * D:3 * D]})
    xo3, y = c.ret.view(B, L, D), c.post['out2']
    dxo = torch.cat([d_enc, d_hidden], 1).reshape(B * L, D)
    dmod = torch.full((B, 3 * D), float('nan'), dtype=F32, device=x.device)
    dy, part = sp.take('gate_bwd', {'dx': dxo, 'y': y, 'gate': m[:, 2 * D:3 * D]}, batch=B, rows_per_batch=L).ret
    f = _finish(sp, part, ['per_sample0'] + (['summed1'] if s2.trained else []))
    dmod[:, 2 * D:3 * D] = f['per_sample0']
    dya = s2.backproject(dy)
    d_o = s2.dgrad(dya, cols=slice(0, D)).ret
    dmlp = s2.dgrad(dya, EPI_MUL_GELU_GRAD, extra={'aux': u}, cols=slice(D, None)).ret
    s2.wgrad([cata], [dya], f.get('summed1'))
    dq, dk, dv = sp.take('attn_bwd', {'q': q, 'k': k, 'v': v, 'o': attn, 'd_o': d_o, 'lse': lse}, scale=None).ret
    c = sp.take('qknorm_rope_bwd', {'dq': dq, 'dk': dk, 'dv': dv, 'qhat': qhat, 'khat': khat, 'q_rstd': q_rstd,
                                    'k_rstd': k_rstd, 'q_norm_w': sp.P(a.norm_q.weight), 'k_norm_w': sp.P(a.norm_k.weight),
                                    'rope_cos': cos, 'rope_sin': sin,
                                    'dbias': torch.zeros(3 * C, dtype=F32, device=x.device),
                                    'dw': torch.zeros((2, HD), dtype=F32, device=x.device)},
                batch=B, heads=H, seq_total=L, seq_offset=0, rows_per_batch=L)
    sp.acc_vec(a.norm_q.weight, c.post['dw'][0])
    sp.acc_vec(a.norm_k.weight, c.post['dw'][1])
    dbias = c.post['dbias']
    if s1.trained:
        dbias = torch.cat([dbias, sp.take('colsum', {'x': dmlp}).ret])
    dl1a = s1.backproject(torch.cat([c.post['dqkv'][:, :3 * C], dmlp], 1))
    xa_b = s1.rebuild(xa, lambda: _ln_fwd(sp, x, m[:, D:2 * D], m[:, 0:D], B, L, save_stats=False)[0])
    s1.wgrad([xa_b], [dl1a], dbias)
    dxn = s1.dgrad(dl1a).ret
    dx, part = sp.take('ln_modulate_bwd', {'dxn': dxn, 'x': x, 'scale': m[:, D:2 * D], 'mean': mean, 'rstd': rstd,
                                           'dres': dxo}, batch=B, rows_per_batch=L, flags=0).ret
    f = _finish(sp, part, ['per_sample0', 'per_sample1'])
    dmod[:, D:2 * D], dmod[:, 0:D] = f['per_sample0'], f['per_sample1']
    dtemb = mod.bwd(dmod, temb, torch.zeros((B, D), dtype=F32, device=x.device))
    dx3 = dx.view(B, L, D)
    return xo3[:, Lt:], xo3[:, :Lt], dx3[:, Lt:], dx3[:, :Lt], dtemb.to(temb.dtype)


# =====================================================================================================================
# running a block under the recorder and checking it against its spec
# =====================================================================================================================
def build_block(kind, D, rank=0, base_dtype=None, device='cpu', seed=0):
    """a block with every parameter random (norm weights around 1), adapters attached when rank > 0"""
    from diffusion_pipe_b200 import flux_blocks as FB, lora, qwen_image as Q, wan as W
    torch.manual_seed(seed)
    H = D // HD
    blk = {'double': lambda: FB.FluxTransformerBlock(D, H, device=device),
           'qwen': lambda: Q.QwenImageTransformerBlock(D, H, device=device),
           'single': lambda: FB.FluxSingleTransformerBlock(D, H, device=device),
           'wan': lambda: W.WanAttentionBlock(D, 2 * D, H, device=device)}[kind]()
    g = torch.Generator().manual_seed(seed)

    def rnd(shape, std):
        return torch.randn(shape, generator=g) * std

    with torch.no_grad():
        for n, p in blk.named_parameters():
            norm = p.dim() == 1 and 'norm' in n and 'linear' not in n
            p.copy_((1 + rnd(p.shape, 0.1) if norm else rnd(p.shape, 0.1 if 'modulation' in n else 0.05)).to(p.dtype))
        if rank:
            lora.attach(blk, rank, base_dtype=base_dtype)
            for n, p in blk.named_parameters():
                if '.lora_A.' in n or '.lora_B.' in n:
                    p.copy_(rnd(p.shape, 0.05).to(p.dtype))
    return blk


def _tables(L, device, g):
    ang = (torch.rand((L, HD // 2), generator=g) * 6.2831853).repeat_interleave(2, -1)
    return torch.cos(ang).to(device), torch.sin(ang).to(device)


def _wan_norm(sp, projs, B, L, H, cos=None, sin=None, eps=None, bwd=False):
    """wan_norm_rope_fwd / _bwd over projection dicts of operands (`rope` a scalar, `dx` an output)"""
    operands, scalars = {}, {'batch': B, 'seq': L, 'heads': H}
    for i, pj in enumerate(projs):
        for k, v in pj.items():
            if k == 'rope':
                scalars[f'projs[{i}].rope'] = v
            else:
                operands[f'projs[{i}].{k}'] = v
    if cos is not None:
        operands.update({'cos': cos, 'sin': sin})
    if eps is not None:
        scalars['eps'] = eps
    return sp.take('wan_norm_rope_bwd' if bwd else 'wan_norm_rope_fwd', operands, **scalars)


# =====================================================================================================================
# Wan attention block  (oracle/wan_ref.py RefWanAttentionBlock: bf16 after every op of the modulation)
# =====================================================================================================================
def spec_wan(sp, blk, x, e0, context, cos, sin, dx3):
    B, L, D = x.shape
    Lc = context.shape[1]
    H = blk.num_heads
    C = H * HD
    eps = blk.eps
    STEPS, MULT = 2, 1
    sa, ca = blk.self_attn, blk.cross_attn
    s_qkv, s_o = Site(sp, 'sa_qkv', [sa.q, sa.k, sa.v]), Site(sp, 'sa_o', [sa.o])
    s_cq, s_ckv, s_co = Site(sp, 'ca_q', [ca.q]), Site(sp, 'ca_kv', [ca.k, ca.v]), Site(sp, 'ca_o', [ca.o])
    s_f1, s_f2 = Site(sp, 'ffn1', [blk.ffn[0]]), Site(sp, 'ffn2', [blk.ffn[2]])
    sp.new_forward()
    dev = x.device
    x2, c2 = x.reshape(B * L, D), context.reshape(B * Lc, D)
    mod = (sp.P(blk.modulation).unsqueeze(0) + e0).reshape(B, 6, D)     # e = modulation + e0 (bf16), chunks 0..5
    # ---- self-attention: y = self_attn(norm1(x) (1 + e1) + e0); x = x + y e2 ----
    xn1, mean1, rstd1 = _ln_fwd(sp, x2, mod[:, 1], mod[:, 0], B, L, eps=eps, flags=STEPS)
    xa = s_qkv.project(xn1)
    qkv = s_qkv.fwd(xa).ret
    (q, xhq, rq), (k, xhk, rk), (v, _, _) = _wan_norm(sp, [
        {'src': qkv[:, 0:D], 'weight': sp.P(sa.norm_q.weight), 'rope': True},
        {'src': qkv[:, D:2 * D], 'weight': sp.P(sa.norm_k.weight), 'rope': True},
        {'src': qkv[:, 2 * D:3 * D]}], B, L, H, cos, sin, eps).ret
    c = sp.take('attn_fwd', {'q': q, 'k': k, 'v': v}, scale=None)
    oa, lse = s_o.project(c.post['out'][:, :C]), c.ret[1]
    c = s_o.fwd(oa, EPI_GATE_RES, L, extra={'aux': x2, 'gate': mod[:, 2]})
    x1, y_attn = c.ret, c.post['out2']
    # ---- cross-attention: x = x + cross_attn(norm3(x), context) ----
    n3w = sp.P(blk.norm3.weight).view(1, D).expand(B, D)
    n3b = sp.P(blk.norm3.bias).view(1, D).expand(B, D)
    xn3, mean3, rstd3 = _ln_fwd(sp, x1, n3w, n3b, B, L, eps=eps, flags=MULT)
    x3a = s_cq.project(xn3)
    ((qc, xhqc, rqc),) = _wan_norm(sp, [{'src': s_cq.fwd(x3a).ret, 'weight': sp.P(ca.norm_q.weight)}], B, L, H, eps=eps).ret
    ca_in = s_ckv.project(c2)
    kv = s_ckv.fwd(ca_in).ret
    (kc, xhkc, rkc), (vc, _, _) = _wan_norm(sp, [{'src': kv[:, 0:D], 'weight': sp.P(ca.norm_k.weight)},
                                                 {'src': kv[:, D:2 * D]}], B, Lc, H, eps=eps).ret
    c = sp.take('attn_fwd', {'q': qc, 'k': kc, 'v': vc}, scale=None)
    oca, lse_c = s_co.project(c.post['out'][:, :C]), c.ret[1]
    x2_ = s_co.fwd(oca, EPI_GATE_RES, L, extra={'aux': x1, 'gate': torch.ones((B, D), dtype=BF, device=dev)}).ret
    # ---- ffn: x = x + ffn(norm2(x) (1 + e4) + e3) e5 ----
    xn2, mean2, rstd2 = _ln_fwd(sp, x2_, mod[:, 4], mod[:, 3], B, L, eps=eps, flags=STEPS)
    x2a = s_f1.project(xn2)
    c = s_f1.fwd(x2a, EPI_BIAS_GELU)
    u = c.post['out2']
    ha = s_f2.project(c.ret)
    c = s_f2.fwd(ha, EPI_GATE_RES, L, extra={'aux': x2_, 'gate': mod[:, 5]})
    x3, y_mlp = c.ret, c.post['out2']
    # ---- backward ----
    dmod = torch.full((B, 6, D), float('nan'), dtype=F32, device=dev)
    d3 = dx3.reshape(B * L, D)
    dy2, part = sp.take('gate_bwd', {'dx': d3, 'y': y_mlp, 'gate': mod[:, 5]}, batch=B, rows_per_batch=L).ret
    f = _finish(sp, part, ['per_sample0'] + (['summed1'] if s_f2.trained else []))
    dmod[:, 5] = f['per_sample0']
    dy2a = s_f2.backproject(dy2)
    du = s_f2.dgrad(dy2a, EPI_MUL_GELU_GRAD, extra={'aux': u}).ret
    s_f2.wgrad([ha], [dy2a], f.get('summed1'))
    dua = s_f1.backproject(du)
    x2a_b = s_f1.rebuild(x2a, lambda: _ln_fwd(sp, x2_, mod[:, 4], mod[:, 3], B, L, save_stats=False, eps=eps,
                                               flags=STEPS)[0], recompute=True)
    db = sp.take('colsum', {'x': dua}).ret if s_f1.trained else None
    s_f1.wgrad([x2a_b], [dua], db)
    dxn2 = s_f1.dgrad(dua).ret
    dx2, part = sp.take('ln_modulate_bwd', {'dxn': dxn2, 'x': x2_, 'scale': mod[:, 4], 'mean': mean2, 'rstd': rstd2,
                                            'dres': d3}, batch=B, rows_per_batch=L, flags=STEPS).ret
    f = _finish(sp, part, ['per_sample0', 'per_sample1'])
    dmod[:, 4], dmod[:, 3] = f['per_sample0'], f['per_sample1']
    dca = s_co.backproject(dx2)
    d_oc = s_co.dgrad(dca).ret
    db = sp.take('colsum', {'x': dca}).ret if s_co.trained else None
    s_co.wgrad([oca], [dca], db)
    dqc, dkc, dvc = sp.take('attn_bwd', {'q': qc, 'k': kc, 'v': vc, 'o': oca[:, :C], 'd_o': d_oc, 'lse': lse_c},
                            scale=None).ret
    c = _wan_norm(sp, [{'dy': dqc, 'weight': sp.P(ca.norm_q.weight), 'xhat': xhqc, 'rstd': rqc}], B, L, H, bwd=True)
    dw_nqc = c.ret[0]
    dqca = s_cq.backproject(c.post['projs[0].dx'][:, :C])
    c = _wan_norm(sp, [{'dy': dkc, 'weight': sp.P(ca.norm_k.weight), 'xhat': xhkc, 'rstd': rkc}, {'dy': dvc}], B, Lc, H,
                  bwd=True)
    dw_nkc = c.ret[0]
    dkva = s_ckv.backproject(torch.cat([c.post['projs[0].dx'][:, :C], c.post['projs[1].dx'][:, :C]], 1))
    x3a_b = s_cq.rebuild(x3a, lambda: _ln_fwd(sp, x1, n3w, n3b, B, L, save_stats=False, eps=eps, flags=MULT)[0],
                         recompute=True)
    dbq = sp.take('colsum', {'x': dqca}).ret if s_cq.trained else None
    dbkv = sp.take('colsum', {'x': dkva}).ret if s_ckv.trained else None
    s_cq.wgrad([x3a_b], [dqca], dbq)
    s_ckv.wgrad([ca_in], [dkva], dbkv)
    sp.acc_vec(ca.norm_q.weight, dw_nqc)
    sp.acc_vec(ca.norm_k.weight, dw_nkc)
    d_ctx = s_ckv.dgrad(dkva).ret
    dxn3 = s_cq.dgrad(dqca).ret
    dx1, part = sp.take('ln_modulate_bwd', {'dxn': dxn3, 'x': x1, 'scale': n3w, 'mean': mean3, 'rstd': rstd3,
                                            'dres': dx2}, batch=B, rows_per_batch=L, flags=MULT).ret
    if blk.norm3.weight.requires_grad:
        f = _finish(sp, part, ['summed0', 'summed1'])
        sp.acc_vec(blk.norm3.weight, f['summed0'])
        sp.acc_vec(blk.norm3.bias, f['summed1'])
    dy1, part = sp.take('gate_bwd', {'dx': dx1, 'y': y_attn, 'gate': mod[:, 2]}, batch=B, rows_per_batch=L).ret
    f = _finish(sp, part, ['per_sample0'] + (['summed1'] if s_o.trained else []))
    dmod[:, 2] = f['per_sample0']
    dy1a = s_o.backproject(dy1)
    d_o = s_o.dgrad(dy1a).ret
    s_o.wgrad([oa], [dy1a], f.get('summed1'))
    dq, dk, dv = sp.take('attn_bwd', {'q': q, 'k': k, 'v': v, 'o': oa[:, :C], 'd_o': d_o, 'lse': lse}, scale=None).ret
    c = _wan_norm(sp, [{'dy': dq, 'weight': sp.P(sa.norm_q.weight), 'xhat': xhq, 'rstd': rq, 'rope': True},
                       {'dy': dk, 'weight': sp.P(sa.norm_k.weight), 'xhat': xhk, 'rstd': rk, 'rope': True},
                       {'dy': dv}], B, L, H, cos, sin, bwd=True)
    sp.acc_vec(sa.norm_q.weight, c.ret[0])
    sp.acc_vec(sa.norm_k.weight, c.ret[1])
    dqkva = s_qkv.backproject(torch.cat([c.post[f'projs[{i}].dx'][:, :C] for i in range(3)], 1))
    xa_b = s_qkv.rebuild(xa, lambda: _ln_fwd(sp, x2, mod[:, 1], mod[:, 0], B, L, save_stats=False, eps=eps,
                                             flags=STEPS)[0], recompute=True)
    db = sp.take('colsum', {'x': dqkva}).ret if s_qkv.trained else None
    s_qkv.wgrad([xa_b], [dqkva], db)
    dxn1 = s_qkv.dgrad(dqkva).ret
    dx, part = sp.take('ln_modulate_bwd', {'dxn': dxn1, 'x': x2, 'scale': mod[:, 1], 'mean': mean1, 'rstd': rstd1,
                                           'dres': dx1}, batch=B, rows_per_batch=L, flags=STEPS).ret
    f = _finish(sp, part, ['per_sample0', 'per_sample1'])
    dmod[:, 1], dmod[:, 0] = f['per_sample0'], f['per_sample1']
    sp.acc_vec(blk.modulation, dmod.sum(0))
    return x3.view(B, L, D), dx.view(B, L, D), dmod.view(B, 1, 6, D).to(e0.dtype), d_ctx.view(B, Lc, D)


SPECS = {'double': spec_flux_double, 'qwen': spec_flux_double, 'single': spec_flux_single}


def run_and_check(monkeypatch, ops, kind, blk, B, Li, Lt, Lc=None, deferred=False, n_mb=1, txt_lens=None, device='cpu',
                  mutate=None, clobber=False, step_between=False, seed=1):
    """runs n_mb micro-batches of forward + backward (weight gradients immediate or deferred and drained after each
    input-gradient pass) under the recorder, then replays every micro-batch against the block's spec.  `mutate(mp, ops)`
    is installed after the recorder, i.e. between the block and the recorder.  Returns the recorder."""
    rec = Recorder().install(monkeypatch, ops)
    if mutate is not None:
        mutate(monkeypatch, ops)
    g = torch.Generator().manual_seed(seed)
    D = blk.dim
    L = Li + (Lt if kind != 'wan' else 0)
    cos, sin = _tables(L, device, g)
    runs = []

    def inp(*shape):
        return torch.randn(shape, generator=g).to(BF).to(device).requires_grad_(True)

    for mb in range(n_mb):
        snap = {id(p): p.detach().clone() for p in blk.parameters()}
        if kind == 'wan':
            ins = (inp(B, Li, D), inp(B, 1, 6, D) * 0.1, inp(B, Lc, D))
            ins = tuple(t.detach().requires_grad_(True) for t in ins)
        else:
            ins = (inp(B, Li, D), inp(B, Lt, D), inp(B, D))
        saved = tuple(t.detach().clone() for t in ins)
        rec.phase = ('fwd', mb)
        if kind == 'wan':
            outs = (blk(ins[0], ins[1], None, None, (cos, sin), ins[2]),)
        elif kind == 'qwen':
            e, h = blk(ins[0], ins[1], ins[2], (cos, sin), txt_lens=txt_lens)
            outs = (h, e)
        else:
            e, h = blk(ins[0], ins[1], ins[2], (cos, sin))
            outs = (h, e)
        douts = tuple(torch.randn(o.shape, generator=g).to(BF).to(device) for o in outs)
        out_vals = tuple(o.detach().clone() for o in outs)
        if deferred:
            ops.WGRAD_DEFER = []
        rec.phase = ('bwd', mb)
        try:
            torch.autograd.backward(outs, douts)
        finally:
            queue, ops.WGRAD_DEFER = ops.WGRAD_DEFER, None
        in_grads = tuple(t.grad.detach().clone() for t in ins)
        if deferred:
            if clobber:        # a stage link hands the input mailbox slots back before the weight-gradient pass
                with torch.no_grad():
                    for t in ins:
                        t.fill_(float('nan'))
            rec.phase = ('drain', mb)
            for fn in queue:
                fn()
        runs.append((snap, saved, douts, out_vals, in_grads))
        if step_between and mb + 1 < n_mb:          # an optimizer step between micro-batches changes the trained values
            with torch.no_grad():
                for p in blk.parameters():
                    if p.requires_grad:
                        p.add_((torch.randn(p.shape, generator=g) * 0.01).to(p.dtype).to(device))
    rec.phase = None
    grads = {}
    spec = SPECS[kind] if kind != 'wan' else spec_wan
    for mb, (snap, saved, douts, out_vals, in_grads) in enumerate(runs):
        rp = Replay([c for c in rec.calls if c.phase in (('fwd', mb), ('bwd', mb))],
                    [c for c in rec.calls if c.phase == ('drain', mb)], deferred)
        sp = Spec(rp, grads, snap)
        if kind == 'wan':
            res = spec(sp, blk, saved[0], saved[1], saved[2], cos, sin, douts[0])
            names = ('output', 'd x', 'd e', 'd context')
            got = out_vals + in_grads
        else:
            kw = {'txt_lens': txt_lens} if kind == 'qwen' else {}
            res = spec(sp, blk, saved[0], saved[1], saved[2], cos, sin, douts[0], douts[1], **kw)
            names = ('image output', 'text output', 'd hidden', 'd enc', 'd temb')
            got = out_vals + in_grads
        rp.done()
        for n, a, w in zip(names, got, res):
            expect_equal(a, w.reshape(a.shape) if w is not None else None, f'micro-batch {mb}: {n}')
    for n, p in blk.named_parameters():
        want = grads.get(id(p))
        if p.requires_grad:
            if want is None:
                raise SpecError(f'{n}: trained, but the spec produced no gradient for it')
            expect_equal(p.grad, want[1].view_as(p), f'{n}.grad')
        elif p.grad is not None:
            raise SpecError(f'{n}: frozen, but .grad is set')
    return rec


def grads_immediate_vs_deferred(monkeypatch, ops, kind, D, rank, base, B, Li, Lt, Lc, txt_lens=None, device='cpu'):
    """runs two micro-batches with immediate, then with deferred weight gradients, each on a fresh block built from
    the same seed, and requires bit-identical .grad of every parameter"""
    grads = []
    for deferred in (False, True):
        blk = build_block(kind, D, rank, base, device=device)
        with monkeypatch.context() as mp:
            run_and_check(mp, ops, kind, blk, B, Li, Lt, Lc, deferred=deferred, n_mb=2, txt_lens=txt_lens, device=device,
                          step_between=True)
        grads.append({n: p.grad for n, p in blk.named_parameters() if p.grad is not None})
    if grads[0].keys() != grads[1].keys():
        raise SpecError(f'parameters with a .grad differ: {sorted(grads[0].keys() ^ grads[1].keys())}')
    for n, g in grads[0].items():
        expect_equal(grads[1][n], g, f'{n}.grad, deferred against immediate')
    return len(grads[0])
