"""CPU: the launch sequence and dataflow of the block autograd Functions (FluxDoubleBlockFn for Flux and Qwen-Image,
FluxSingleBlockFn, WanBlockFn) on the kernel test doubles, against the specs of tests/block_dataflow.py: every operand
bit for bit against its named source, no byte written outside a call's outputs, the exact call sequence, and the block's
outputs, input gradients and parameter gradients assembled from the recorded calls.  Each mutation below injects one
wiring error between the block and the recorder and must be rejected.  tests/test_block_dataflow_gpu.py runs the same
specs on the real kernels and checks every call per element against the fp64 references."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import block_dataflow as BD  # noqa: E402

D = 256
LI, LT, LC = 88, 40, 24


@pytest.fixture
def ops(monkeypatch):
    import kernel_doubles
    from diffusion_pipe_b200 import lora, ops
    kernel_doubles.install(monkeypatch, ops)
    monkeypatch.setattr(ops, 'WGRAD_DEFER', None)
    monkeypatch.setattr(lora, '_SCRATCH', {})
    monkeypatch.setattr(lora, '_SCRATCH_OWNER', {})
    return ops


VARIANTS = {   # name: (kind, rank, fp8 base, micro-batch, txt_lens)
    'double': ('double', 0, None, 1, None),
    'double-lora': ('double', 16, None, 1, None),
    'double-lora-fp8': ('double', 16, torch.float8_e4m3fn, 1, None),
    'qwen': ('qwen', 0, None, 1, None),
    'qwen-ragged': ('qwen', 0, None, 3, (40, 1, 23)),
    'single': ('single', 0, None, 1, None),
    'single-lora': ('single', 16, None, 1, None),
    'single-lora-fp8': ('single', 16, torch.float8_e4m3fn, 1, None),
    'wan': ('wan', 0, None, 1, None),
    'wan-lora': ('wan', 16, None, 1, None),
    'wan-lora-fp8': ('wan', 16, torch.float8_e5m2, 1, None),
}


def run(monkeypatch, ops, variant, deferred=False, n_mb=1, B=None, **kw):
    kind, rank, base, b, txt_lens = VARIANTS[variant]
    blk = BD.build_block(kind, D, rank, base)
    return BD.run_and_check(monkeypatch, ops, kind, blk, B or b, LI, LT, LC, deferred=deferred, n_mb=n_mb,
                            txt_lens=txt_lens, step_between=n_mb > 1, **kw)


@pytest.mark.parametrize('n_mb', [1, 2])
@pytest.mark.parametrize('deferred', [False, True], ids=['immediate', 'deferred'])
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_block_dataflow(monkeypatch, ops, variant, deferred, n_mb):
    rec = run(monkeypatch, ops, variant, deferred, n_mb)
    print(f'{variant}: {len(rec.calls)} calls checked')


@pytest.mark.parametrize('variant', list(VARIANTS))
def test_immediate_and_deferred_grads_identical(monkeypatch, ops, variant):
    kind, rank, base, b, txt_lens = VARIANTS[variant]
    assert BD.grads_immediate_vs_deferred(monkeypatch, ops, kind, D, rank, base, b, LI, LT, LC, txt_lens) > 0


@pytest.mark.parametrize('variant', ['double', 'qwen-ragged', 'single', 'wan', 'wan-lora'])
def test_deferred_weight_gradients_survive_recycled_inputs(monkeypatch, ops, variant):
    """the weight-gradient closures own every operand they read: the block's input storage can be handed back (and
    overwritten) after the input-gradient pass, as a stage link hands back a mailbox slot, before the queue drains"""
    run(monkeypatch, ops, variant, deferred=True, clobber=True)


# ---- mutations: each injects one wiring error between the block and the recorder ------------------------------------
def _wrap(mp, ops, name, fn):
    real = getattr(ops, name)
    mp.setattr(ops, name, lambda *a, **k: fn(real, *a, **k))


def _row0(t):
    return torch.as_strided(t, t.shape, t.stride(), t.storage_offset() % t.stride(0))


def m_gate_row0(mp, ops):                  # 1: every sample's attention residual reads sample 0's gate row
    def f(real, *a, **k):
        if k.get('epilogue') == BD.EPI_GATE_RES and k['gate'].shape[0] == 1:
            k['gate'] = _row0(k['gate'])
        return real(*a, **k)
    _wrap(mp, ops, 'gemm', f)


def m_mlp_aux_is_input(mp, ops):           # 2: the MLP residual adds the block input instead of x1
    inputs = {}

    def ln(real, x, *a, **k):                # a stream's first LayerNorm reads the block input
        inputs.setdefault(x.shape[0], x)
        return real(x, *a, **k)

    def f(real, *a, **k):
        if k.get('epilogue') == BD.EPI_GATE_RES and 'out' not in k:
            k['aux'] = inputs[k['aux'].shape[0]]
        return real(*a, **k)
    _wrap(mp, ops, 'ln_modulate_fwd', ln)
    _wrap(mp, ops, 'gemm', f)


def m_text_offset(mp, ops):                # 3: the text stream's QKV epilogue gets the image stream's seq_offset
    def f(real, *a, **k):
        a = list(a)
        if a[9] == 0:
            a[9] = LT
        return real(*a, **k)
    _wrap(mp, ops, 'make_qkv_epilogue', f)


def m_swap_ln2(mp, ops):                   # 4: scale and shift swapped in the second LayerNorm modulation
    def f(real, x, scale, shift, *a, **k):
        if scale.storage_offset() % scale.stride(0) == 4 * D:
            scale, shift = shift, scale
        return real(x, scale, shift, *a, **k)
    _wrap(mp, ops, 'ln_modulate_fwd', f)


def m_drop_dres(mp, ops):                  # 5: one stream's ln_modulate_bwd drops dres
    def f(real, *a, **k):
        if a[0].shape[0] == LT:
            k['dres'] = None
        return real(*a, **k)
    _wrap(mp, ops, 'ln_modulate_bwd', f)


def m_swap_finish(mp, ops):                # 6: colreduce_finish gets per_sample0 and per_sample1 swapped
    def f(real, part, per_sample0=None, per_sample1=None, **k):
        return real(part, per_sample0=per_sample1, per_sample1=per_sample0, **k)
    _wrap(mp, ops, 'colreduce_finish', f)


def m_dgrad_over_xa(mp, ops):              # 7: DenseSite.dgrad_out returns xa while weight gradients are deferred
    from diffusion_pipe_b200 import flux_blocks
    mp.setattr(flux_blocks.DenseSite, 'dgrad_out', lambda self, xa: xa)


def m_no_refresh(mp, ops):                 # 8: LoraSite.refresh skipped after an optimizer step changed the factors
    from diffusion_pipe_b200 import lora
    mp.setattr(lora.LoraSite, 'refresh', lambda self: None)


def m_no_refill(mp, ops):                  # 9: _widened never refills the fp8 operand buffer
    from diffusion_pipe_b200 import lora
    real = lora._widened

    def f(device, key, shape, fill):
        if lora._SCRATCH.get(device) is not None and lora._SCRATCH[device].numel() >= shape[0] * shape[1]:
            return lora._SCRATCH[device][:shape[0] * shape[1]].view(shape)
        return real(device, key, shape, fill)
    mp.setattr(lora, '_widened', f)


def m_padded_key(mp, ops):                 # 10: one padded text row among sample b's key rows
    from diffusion_pipe_b200 import flux_blocks
    real = flux_blocks._valid_rows
    mp.setattr(flux_blocks, '_valid_rows', lambda n, Lt, Ltot, dev: real(min(n + 1, Lt), Lt, Ltot, dev))


def m_explicit_rows(mp, ops):              # a GEMM given an explicit row count one short of its operand's
    def f(real, a, b, **k):
        if k.get('epilogue') == BD.EPI_BIAS_GELU:
            k['M'] = a.shape[0] - 1
        return real(a, b, **k)
    _wrap(mp, ops, 'gemm', f)


def m_second_mb_overwrites(mp, ops):       # 11: the second micro-batch's weight-gradient GEMM overwrites .grad
    def f(real, *a, **k):
        if k.get('a_mn') and k.get('b_mn'):
            k['accumulate'] = False
        return real(*a, **k)
    _wrap(mp, ops, 'gemm', f)


def m_unrounded_dmod(mp, ops):             # 12: ModLora.bwd uses the fp32 dmod where the reference rounds it to bf16
    from diffusion_pipe_b200 import flux_blocks, lora

    def bwd(self, dmod32, temb, saved, d_temb32):
        s, t = saved
        d = dmod32.float()
        flux_blocks._mod_bwd(dmod32, temb, self._base(), d_temb32)
        dt = d @ self.b.float()
        flux_blocks._acc_vec(self.b, d.t() @ t.float())
        flux_blocks._acc_vec(self.a, dt.t() @ s.float())
        ds = dt @ self.a.float()
        tf = temb.float()
        sg = torch.sigmoid(tf)
        d_temb32.add_(ds.to(torch.bfloat16).float() * (sg * (1 + tf * (1 - sg))))
    mp.setattr(lora.ModLora, 'bwd', bwd)


MUTATIONS = {   # name: (variant, deferred, micro-batches, mutation, expected message)
    'gate_row0': ('qwen-ragged', False, 1, m_gate_row0, 'operand gate'),
    'mlp_aux_is_input': ('double', False, 1, m_mlp_aux_is_input, 'operand aux'),
    'text_offset': ('double', False, 1, m_text_offset, 'qkv.seq_offset'),
    'swap_ln2': ('double', False, 1, m_swap_ln2, 'operand scale'),
    'drop_dres': ('double', False, 1, m_drop_dres, 'operand dres'),
    'swap_finish': ('single', False, 1, m_swap_finish, 'colreduce_finish'),
    'dgrad_over_xa': ('double', True, 1, m_dgrad_over_xa, 'gemm'),
    'no_refresh': ('double-lora', False, 2, m_no_refresh, 'operand b'),
    'no_refill': ('wan-lora-fp8', False, 1, m_no_refill, 'fp8_to_bf16'),
    'padded_key': ('qwen-ragged', False, 1, m_padded_key, 'attn_fwd'),
    'second_mb_overwrites': ('single', True, 2, m_second_mb_overwrites, 'accumulate'),
    'explicit_rows': ('double', False, 1, m_explicit_rows, 'scalar M'),
    'unrounded_dmod': ('double-lora', False, 1, m_unrounded_dmod, 'dtemb32'),
}


@pytest.mark.parametrize('name', list(MUTATIONS))
def test_mutation_rejected(monkeypatch, ops, name):
    variant, deferred, n_mb, mut, msg = MUTATIONS[name]
    with pytest.raises(BD.SpecError, match=msg) as ei:
        run(monkeypatch, ops, variant, deferred, n_mb, mutate=mut)
    print(name, '->', ei.value)
    assert str(ei.value).startswith('call ') and 'operand' in str(ei.value)
