"""GPU: the dataflow specs of tests/block_dataflow.py on the real kernels (every operand bit for bit against its source,
no stray writes, the exact call sequence, outputs and gradients assembled from the recorded calls), and every recorded
call checked per element against the fp64 references of tests/gemm_attn_refs.py and tests/block_kernel_refs.py, applied
to that call's own operands: the kernels at the strided views, row blocks and offsets the blocks really pass."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import block_dataflow as BD  # noqa: E402
import block_kernel_refs as KR  # noqa: E402
import gemm_attn_refs as GR  # noqa: E402

pytestmark = pytest.mark.gpu

SHAPES = {'d256': (256, 1, 88, 40, 24), 'd512-tail': (512, 3, 130, 77, 77)}   # D, micro-batch, Li, Lt, Lc
VARIANTS = {   # name: (kind, rank, fp8 base)
    'double': ('double', 0, None), 'double-lora': ('double', 16, None),
    'double-lora-fp8': ('double', 16, torch.float8_e4m3fn),
    'single': ('single', 0, None), 'single-lora': ('single', 16, None),
    'single-lora-fp8': ('single', 16, torch.float8_e4m3fn),
    'qwen': ('qwen', 0, None), 'qwen-ragged': ('qwen', 0, None),
    'wan': ('wan', 0, None), 'wan-lora': ('wan', 16, None), 'wan-lora-fp8': ('wan', 16, torch.float8_e5m2),
}
WORST = {}      # op family -> worst err / bound over the module
FAMILY = {0: 'STORE', 1: 'BIAS_GELU', 2: 'GATE_RES', 3: 'QKV_ROPE', 4: 'MUL_GELU_GRAD'}


@pytest.fixture(scope='module', autouse=True)
def _report():
    """prints, after the module, the worst err / bound of every op family and the peak CUDA memory"""
    import time
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f'\nblock dataflow on {torch.cuda.get_device_name()}: {time.time() - t0:.0f} s, peak CUDA memory '
          f'{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB; worst err / bound: '
          + ', '.join(f'{k} {v:.3f}' for k, v in sorted(WORST.items())))


@pytest.fixture
def ops(monkeypatch):
    """the real kernels, with CUDA torch.empty / empty_like / new_empty NaN-filled: an element no launch wrote shows up"""
    from diffusion_pipe_b200 import lora, ops
    monkeypatch.setattr(ops, 'WGRAD_DEFER', None)
    monkeypatch.setattr(lora, '_SCRATCH', {})
    monkeypatch.setattr(lora, '_SCRATCH_OWNER', {})
    real_empty, real_like, real_new = torch.empty, torch.empty_like, torch.Tensor.new_empty

    def poison(t):
        if t.is_cuda and t.is_floating_point() and t.numel() and t.dtype not in BD.FP8:
            t.fill_(float('nan'))
        return t
    monkeypatch.setattr(torch, 'empty', lambda *a, **k: poison(real_empty(*a, **k)))
    monkeypatch.setattr(torch, 'empty_like', lambda *a, **k: poison(real_like(*a, **k)))
    monkeypatch.setattr(torch.Tensor, 'new_empty', lambda self, *a, **k: poison(real_new(self, *a, **k)))
    return ops


def _check(family, out, ref, what, bf16_out=None):
    KR.check(out, ref, what, bf16_out)
    if bf16_out is None:
        bf16_out = out.dtype == torch.bfloat16
    err, allowed = KR.violations(out, ref, bf16_out)
    r = float((err / allowed.clamp_min(1e-300)).max()) if err.numel() else 0.0
    WORST[family] = max(WORST.get(family, 0.0), r)


def _logical(t, mn):
    return t.t() if mn else t


def check_call(c, prev):
    """per-element check of one recorded call on its own pre-call operands; returns the reference a following
    colreduce_finish is checked against"""
    t, s, op, w = c.pre, c.scalars, c.op, f'{c!r}'
    if op == 'gemm':
        A, B = _logical(t['a'], s['a_mn']), _logical(t['b'], s['b_mn'])
        acc = GR.gemm_acc(A, B)
        e = s['epilogue']
        fam = f'gemm {FAMILY[e]}'
        rpb = s['rows_per_batch'] or A.shape[0]
        if e == BD.EPI_STORE:
            _check(fam, c.ret, GR.gemm_store_ref(acc, t.get('bias'), t['out'] if s['accumulate'] else None)['out'], w)
        elif e == BD.EPI_BIAS_GELU:
            r = GR.gemm_bias_gelu_ref(acc, t.get('bias'))
            _check(fam, c.ret, r['out'], w)
            _check(fam, c.post['out2'], r['out2'], w + ' out2')
        elif e == BD.EPI_GATE_RES:
            r = GR.gemm_gate_res_ref(acc, t['aux'], t['gate'], rpb, t.get('bias'))
            _check(fam, c.ret, r['out'], w)
            if 'out2' in t:
                _check(fam, c.post['out2'], r['out2'], w + ' out2')
        elif e == BD.EPI_MUL_GELU_GRAD:
            _check(fam, c.ret, GR.gemm_mul_gelu_grad_ref(acc, t['aux'])['out'], w)
        else:
            off, L = s['qkv.seq_offset'], rpb
            r = GR.gemm_qkv_ref(acc, t.get('bias'), t['qkv.q_norm_w'], t['qkv.k_norm_w'], t['qkv.rope_cos'],
                                t['qkv.rope_sin'], s['qkv.heads'], L, off, s['qkv.n_qkv'], s['qkv.eps'])
            for k in ('q', 'k', 'v', 'qhat', 'khat', 'q_rstd', 'k_rstd'):
                _check(fam, c.post[f'qkv.{k}'][:, :, off:off + L], r[k], f'{w} {k}')
            if 'out' in r:
                _check(fam, c.post['out'], r['out'], w + ' out')
                _check(fam, c.post['out2'], r['out2'], w + ' out2')
        return None
    if op == 'attn_fwd':
        q, k, v = t['q'], t['k'], t['v']
        B, H, Lq, _ = q.shape
        o = c.ret[0][:, :H * BD.HD].view(B, Lq, H, BD.HD)
        for b in range(B):
            for h in range(H):
                r = GR.attn_fwd_ref(q[b, h], k[b, h], v[b, h], BD.HD ** -0.5)
                _check('attn_fwd', o[b, :, h], r['o'], f'{w} o[{b},{h}]')
                _check('attn_fwd', c.ret[1][b, h], r['lse'], f'{w} lse[{b},{h}]')
        return None
    if op == 'attn_bwd':
        q, k, v = t['q'], t['k'], t['v']
        B, H, Lq, _ = q.shape
        o, do = (x[:, :H * BD.HD].reshape(B, Lq, H, BD.HD) for x in (t['o'], t['d_o']))
        for b in range(B):
            for h in range(H):
                r = GR.attn_bwd_ref(q[b, h], k[b, h], v[b, h], o[b, :, h], do[b, :, h], t['lse'][b, h], BD.HD ** -0.5)
                for i, n in enumerate(('dq', 'dk', 'dv')):
                    _check('attn_bwd', c.ret[i][b, h], r[n], f'{w} {n}[{b},{h}]')
        return None
    if op == 'ln_modulate_fwd':
        r = KR.ln_modulate_fwd_ref(t['x'], t['scale'], t['shift'], s['batch'], s['rows_per_batch'], s['eps'], s['flags'])
        _check('ln_modulate_fwd', c.ret[0], r['out'], w)
        if s['save_stats']:
            _check('ln_modulate_fwd', c.ret[1], r['mean'], w + ' mean')
            _check('ln_modulate_fwd', c.ret[2], r['rstd'], w + ' rstd')
        return None
    if op == 'ln_modulate_bwd':
        r = KR.ln_modulate_bwd_ref(t['dxn'], t['x'], t['scale'], t['mean'], t['rstd'], s['batch'], s['rows_per_batch'],
                                   t.get('dres'), s['flags'])
        _check('ln_modulate_bwd', c.ret[0], r['dx'], w)
        return {'per_sample0': r['dscale'], 'per_sample1': r['dshift'], 'summed0': r['dscale_sum'],
                'summed1': r['dshift_sum']}
    if op == 'gate_bwd':
        r = KR.gate_bwd_ref(t['dx'], t['y'], t['gate'], s['batch'], s['rows_per_batch'])
        _check('gate_bwd', c.ret[0], KR.E(r['dy']), w)
        return {'per_sample0': r['dgate'], 'summed1': r['dbias']}
    if op == 'colreduce_finish':
        for n in ('per_sample0', 'per_sample1', 'summed0', 'summed1'):
            if n in c.post:
                _check('colreduce_finish', c.post[n], prev[n], f'{w} {n}')
        return None
    if op == 'colsum':
        _check('colsum', c.ret, KR.colsum_ref(t['x']), w)
        return None
    if op == 'qknorm_rope_bwd':
        C3 = 3 * s['heads'] * BD.HD
        r = KR.qknorm_rope_bwd_ref(t['dq'], t['dk'], t['dv'], t['qhat'], t['khat'], t['q_rstd'], t['k_rstd'],
                                   t['q_norm_w'], t['k_norm_w'], t['rope_cos'], t['rope_sin'], s['batch'], s['heads'],
                                   s['seq_offset'], s['rows_per_batch'])
        _check('qknorm_rope_bwd', c.post['dqkv'][:, :C3], r['dqkv'], w + ' dqkv')
        _check('qknorm_rope_bwd', c.post['dw'], r['dw'], w + ' dw')
        _check('qknorm_rope_bwd', c.post['dbias'][:C3], KR.summed_rows_ref(c.post['dqkv'][:, :C3], t['dbias'][:C3]),
               w + ' dbias')
        return None
    if op in ('wan_norm_rope_fwd', 'wan_norm_rope_bwd'):
        B, L, H = s['batch'], s['seq'], s['heads']
        i = 0
        while f'projs[{i}].{"src" if op.endswith("fwd") else "dy"}' in t:
            g = lambda n: t.get(f'projs[{i}].{n}')
            rope = bool(s.get(f'projs[{i}].rope'))
            if op.endswith('fwd'):
                r = KR.wan_norm_rope_fwd_ref(g('src'), g('weight'), rope, t.get('cos'), t.get('sin'), B, L, H, s['eps'])
                _check('wan_norm_rope_fwd', c.ret[i][0], r['dst'], f'{w} dst[{i}]')
                if g('weight') is not None:
                    _check('wan_norm_rope_fwd', c.ret[i][1], r['xhat'], f'{w} xhat[{i}]')
                    _check('wan_norm_rope_fwd', c.ret[i][2], r['rstd'], f'{w} rstd[{i}]')
            else:
                r = KR.wan_norm_rope_bwd_ref(g('dy'), g('xhat'), g('rstd'), g('weight'), rope, t.get('cos'), t.get('sin'),
                                             B, L, H)
                _check('wan_norm_rope_bwd', c.post[f'projs[{i}].dx'][:, :H * BD.HD], r['dx'], f'{w} dx[{i}]')
                if g('weight') is not None:
                    _check('wan_norm_rope_bwd', c.ret[i], r['dw'], f'{w} dw[{i}]')
            i += 1
        return None
    if op == 'mod_fwd':
        _check('mod_fwd', c.ret, KR.mod_fwd_ref(t['temb'], t['weight'], t.get('bias')), w)
        return None
    if op == 'mod_bwd':
        r = KR.mod_bwd_ref(t['dmod32'], t['temb'], t['weight'], t.get('wgrad') if s['accumulate'] else None, t['dtemb32'])
        _check('mod_bwd', c.ret, r['dbias'], w + ' dbias')
        _check('mod_bwd', c.post['dtemb32'], r['dtemb'], w + ' dtemb')
        if 'wgrad' in c.post:
            _check('mod_bwd', c.post['wgrad'], r['dW'](), w + ' dW')
        return None
    if op == 'fp8_to_bf16':
        assert BD.same_bits(c.post['dst'], t['src'].to(torch.bfloat16)), w
        WORST['fp8_to_bf16'] = WORST.get('fp8_to_bf16', 0.0)
        return None
    raise KeyError(op)


@pytest.mark.parametrize('n_mb', [1, 2])
@pytest.mark.parametrize('deferred', [False, True], ids=['immediate', 'deferred'])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_block_dataflow_gpu(monkeypatch, ops, variant, shape, deferred, n_mb):
    kind, rank, base = VARIANTS[variant]
    D, B, Li, Lt, Lc = SHAPES[shape]
    txt_lens = None
    if variant == 'qwen-ragged':
        B = 3
        txt_lens = (Lt, 1, Lt // 2 + 1)
    blk = BD.build_block(kind, D, rank, base, device='cuda')
    rec = BD.run_and_check(monkeypatch, ops, kind, blk, B, Li, Lt, Lc, deferred=deferred, n_mb=n_mb, txt_lens=txt_lens,
                           device='cuda', step_between=n_mb > 1)
    prev = None
    for c in rec.calls:
        prev = check_call(c, prev)
    print(f'{variant} {shape} {"deferred" if deferred else "immediate"} x{n_mb}: {len(rec.calls)} calls')


@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_immediate_and_deferred_grads_identical_gpu(monkeypatch, ops, variant, shape):
    kind, rank, base = VARIANTS[variant]
    D, B, Li, Lt, Lc = SHAPES[shape]
    txt_lens = None
    if variant == 'qwen-ragged':
        B, txt_lens = 3, (Lt, 1, Lt // 2 + 1)
    assert BD.grads_immediate_vs_deferred(monkeypatch, ops, kind, D, rank, base, B, Li, Lt, Lc, txt_lens, 'cuda') > 0
