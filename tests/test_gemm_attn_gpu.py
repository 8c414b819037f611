"""GPU: the wgmma GEMM (every operand layout and epilogue it is built for) and the attention forward and backward,
element by element against the fp64 references of tests/gemm_attn_refs.py, at every tile tail and at the real shapes.

Two tiers.  Small-integer inputs make every fp32 partial sum exact in any order, so each output must be the rounding of
the exact value (bit for bit where no transcendental follows): that checks the indexing independently of the
accumulation model.  Random inputs with per-row magnitudes log-uniform over 1e-3 .. 1e2 (q and k over 1e-3 .. 10^0.5,
so that softmax keeps more than one key) are then held to the per-element bound.  Every output lives inside a
sentinel-filled buffer (Canvas / Flat of tests/test_block_kernels_gpu.py) with a row stride above its width, operands
are views whose padding is NaN, and each sample has its own gate row.

The worst err / bound of each kernel family, and of an all-positive K = 32768 GEMM where a truncating accumulator would
show its bias, is printed at the end of the module (pytest -s).  DPIPE_ATTN_FWD_POLY = 2 / 4 select the FMA-pipe
exponential of the attention forward once per process, so those run in a child process of this file."""
import os
import subprocess
import sys
import zlib

import pytest
import torch

import block_kernel_refs as R
import gemm_attn_refs as G
from test_block_kernels_gpu import SENTINEL, Canvas, Flat

pytestmark = pytest.mark.gpu

POLY = int(os.environ.get('DPIPE_ATTN_FWD_POLY', '0') or 0)
WORST = {}


@pytest.fixture(scope='module')
def ops():
    from diffusion_pipe_b200 import ops as o
    return o


@pytest.fixture(scope='module', autouse=True)
def _report():
    torch.cuda.reset_peak_memory_stats()
    yield
    for k in sorted(WORST):
        print(f'worst err / bound  {k:<28s} {WORST[k][0]:.3e}  ({WORST[k][1]})')
    print(f'peak CUDA memory of the module: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB')


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _rows(n, cols, g, lo=-3.0, hi=2.0):
    mag = 10 ** (lo + (hi - lo) * torch.rand(n, 1, generator=g, device='cuda'))
    return torch.randn(n, cols, generator=g, device='cuda') * mag


def _ints(shape, g, lim=3):
    return torch.randint(-lim, lim + 1, shape, generator=g, device='cuda').float()


def check(out, ref, family, what, bf16_out=None):
    """R.check, recording the worst err / bound of the family"""
    if bf16_out is None:
        bf16_out = out.dtype == torch.bfloat16
    err, allowed = R.violations(out, ref, bf16_out)
    ratio = torch.where(allowed > 0, err / allowed, torch.where(err > 0, torch.full_like(err, float('inf')), 0 * err))
    r = float(ratio.max()) if ratio.numel() else 0.0
    if r > WORST.get(family, (-1.0,))[0]:
        WORST[family] = (r, what)
    R.check(out, ref, what, bf16_out)


def _operand(t, mn):
    """a logical [R, K] bf16 operand stored K-major ([R, K] view) or MN-major ([K, R] view), each inside a NaN-padded
    buffer whose row stride exceeds the width"""
    r, k = t.shape
    if mn:
        buf = torch.full((k, (r + 7) // 8 * 8 + 8), float('nan'), device='cuda', dtype=torch.bfloat16)
        buf[:, :r] = t.t()
        return buf[:, :r]
    buf = torch.full((r, (k + 7) // 8 * 8 + 8), float('nan'), device='cuda', dtype=torch.bfloat16)
    buf[:, :k] = t
    return buf[:, :k]


def _vec(t):
    """a bf16 vector at a 16-byte offset inside a NaN buffer"""
    buf = torch.full((t.numel() + 16,), float('nan'), device='cuda', dtype=torch.bfloat16)
    buf[8:8 + t.numel()] = t
    return buf[8:8 + t.numel()]


def _wide(t, extra=16):
    buf = torch.full((t.shape[0], t.shape[1] + extra), float('nan'), device='cuda', dtype=torch.bfloat16)
    buf[:, :t.shape[1]] = t
    return buf[:, :t.shape[1]]


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
EPI = {'store': 0, 'bias_gelu': 1, 'gate_res': 2, 'qkv': 3, 'mul_gelu_grad': 4}
LAYOUTS = {'store': [(0, 0), (0, 1), (1, 1)], 'bias_gelu': [(0, 0)], 'gate_res': [(0, 0)], 'mul_gelu_grad': [(0, 1)]}


def gemm_case(ops, M, N, K, epi, layout=(0, 0), bias=True, out2=True, accumulate=False, rpb=None, ints=False,
              chunk=4096, twice=False):
    """one dpipe_gemm_bf16 call of a non-QKV epilogue into sentinel buffers, checked element by element"""
    g = _gen('gemm', M, N, K, epi, layout, bias, out2, accumulate, rpb, ints)
    what = f'{epi} {M}x{N}x{K} layout={layout} bias={bias} out2={out2} acc={accumulate} rpb={rpb} ints={ints}'
    if ints:
        A, Bw = _ints((M, K), g).bfloat16(), _ints((N, K), g).bfloat16()
        b = _ints((N,), g, 8).bfloat16() if bias else None
    else:
        A, Bw = _rows(M, K, g).bfloat16(), _rows(N, K, g, -3, 0).bfloat16()
        b = (torch.randn(N, generator=g, device='cuda') * 2).bfloat16() if bias else None
    rpb = rpb or M
    nsamp = -(-M // rpb)
    out = Canvas(M, N, torch.bfloat16)
    o2 = Canvas(M, N, torch.bfloat16) if out2 and epi in ('bias_gelu', 'gate_res') else None
    old = res = gate = aux = None
    if accumulate:
        old = (_ints((M, N), g, 40) if ints else _rows(M, N, g)).bfloat16()
        out.view.copy_(old)
    if epi == 'gate_res':
        res = _wide((_ints((M, N), g, 40) if ints else _rows(M, N, g)).bfloat16())
        mod = (torch.randn(nsamp, 3 * N, generator=g, device='cuda') * 0.5
               + torch.arange(nsamp, device='cuda')[:, None] * (1.0 if ints else 0.37) + 1).bfloat16()   # one row per sample
        if ints:
            mod = mod.float().round().bfloat16()
        gate = mod[:, N:2 * N]
    if epi == 'mul_gelu_grad':
        aux = _wide((torch.randn(M, N, generator=g, device='cuda') * 2).bfloat16())
    a_op, b_op = _operand(A, layout[0]), _operand(Bw, layout[1])
    kw = dict(a_mn=bool(layout[0]), b_mn=bool(layout[1]), out=out.view, epilogue=EPI[epi], bias=_vec(b) if bias else None,
              out2=o2.view if o2 is not None else None, aux=res if res is not None else aux, gate=gate, rows_per_batch=rpb,
              accumulate=accumulate)
    ops.gemm(a_op, b_op, **kw)
    torch.cuda.synchronize()
    assert out.intact() and (o2 is None or o2.intact()), what + ': sentinel overwritten'
    if twice:
        first = out.view.clone()
        if accumulate:
            out.view.copy_(old)
        ops.gemm(a_op, b_op, **kw)
        torch.cuda.synchronize()
        assert torch.equal(first.view(torch.int16), out.view.view(torch.int16)), what + ': not repeatable'
    fam = f'gemm {epi} {layout[0]}{layout[1]}'
    for c0 in range(0, N, chunk):
        cs = slice(c0, min(N, c0 + chunk))
        acc = R.exact(A.double() @ Bw[cs].double().t()) if ints else G.gemm_acc(A, Bw[cs])
        bc = b[cs] if bias else None
        if epi == 'store':
            ref = G.gemm_store_ref(acc, bc, old[:, cs] if accumulate else None)
        elif epi == 'bias_gelu':
            ref = G.gemm_bias_gelu_ref(acc, bc)
        elif epi == 'gate_res':
            ref = G.gemm_gate_res_ref(acc, res[:, cs], gate[:, cs], rpb, bc)
        else:
            ref = G.gemm_mul_gelu_grad_ref(acc, aux[:, cs])
        w = f'{what} cols {c0}'
        check(out.view[:, cs], ref['out'], fam, w + ' out')
        if o2 is not None:
            check(o2.view[:, cs], ref['out2'], fam, w + ' out2')
        if ints and epi in ('store', 'gate_res'):   # no transcendental: the rounding of the exact value, bit for bit
            assert torch.equal(out.view[:, cs].double(), R.bf(ref['out'].v)), w + ' out not bit-exact'
        if ints and o2 is not None:
            assert torch.equal(o2.view[:, cs].double(), R.bf(ref['out2'].v)), w + ' out2 not bit-exact'
        del acc, ref


MS = [1, 63, 64, 65, 127, 128, 129, 1029]
KS = [8, 56, 64, 144, 192, 256, 320]


@pytest.mark.parametrize('ints', [True, False])
@pytest.mark.parametrize('layout', LAYOUTS['store'])
@pytest.mark.parametrize('M', MS)
def test_gemm_store(M, layout, ints, ops):
    """N tails 8 / 40 / 264 (one partial 32-column chunk, one partial tile) and K below, at and above the 4 k-block
    ring; bias present and absent; accumulate onto the output at the N tails"""
    for N in (8, 40, 264):
        for i, K in enumerate(KS):
            gemm_case(ops, M, N, K, 'store', layout, bias=bool(i % 2), accumulate=(i % 3 == 0), ints=ints)


@pytest.mark.parametrize('ints', [True, False])
@pytest.mark.parametrize('epi', ['bias_gelu', 'gate_res', 'mul_gelu_grad'])
@pytest.mark.parametrize('M', MS)
def test_gemm_fused_epilogues(M, epi, ints, ops):
    layout = LAYOUTS[epi][0]
    for N in (32, 256, 288):
        for i, K in enumerate((8, 64, 144, 320)):
            gemm_case(ops, M, N, K, epi, layout, bias=bool(i % 2), out2=(i // 2 == 0), ints=ints)


@pytest.mark.parametrize('rpb', [1, 77, 192])
def test_gemm_gate_res_samples(rpb, ops):
    """8 samples, each with its own gate row; 77 and 192 put sample boundaries inside 128-row tiles"""
    for ints in (True, False):
        gemm_case(ops, 8 * rpb, 288, 144, 'gate_res', rpb=rpb, ints=ints)


def test_gemm_long_k_and_repeatability(ops):
    """K = 3072 in every layout and epilogue, run twice for identical bits; a wgrad-like K of 36 k (a long sequence)"""
    for epi, layouts in LAYOUTS.items():
        for layout in layouts:
            gemm_case(ops, 300, 264 if epi == 'store' else 288, 3072, epi, layout, twice=True)
    gemm_case(ops, 256, 264, 36864, 'store', (1, 1))
    gemm_case(ops, 200, 3072, 36864, 'store', (1, 1), bias=False, accumulate=True)


def test_gemm_calibration_all_positive_k32768(ops):
    """all products positive: a truncating or biased accumulator adds its error up over 2048 k16 steps"""
    g = _gen('calib')
    M, N, K = 256, 512, 32768
    A = torch.rand(M, K, generator=g, device='cuda').bfloat16()
    Bw = torch.rand(N, K, generator=g, device='cuda').bfloat16()
    out = ops.gemm(A, Bw)
    torch.cuda.synchronize()
    ref = G.gemm_acc(A, Bw)
    err = (out.double() - ref.v).abs()
    # the bf16 output rounding averages out over the tile; what remains of the mean is the accumulator's own bias
    print(f'calibration K={K}: worst err / (bound + half ulp) {float((err / (ref.e + 0.5 * R.ulp(ref.v))).max()):.3e}, '
          f'mean signed error / mean accumulation bound {float((out.double() - ref.v).mean() / ref.e.mean()):.3e}')
    check(out, ref, 'gemm calibration K=32768', 'calibration')


# ---------------------------------------------------------------------------------------------------------------
# QKV epilogue
# ---------------------------------------------------------------------------------------------------------------
def _rope(L, g):
    ang = torch.rand(L, 64, generator=g, device='cuda') * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous()


def qkv_case(ops, B, L, H, mlp, off, hats, K=96, ints=False, twice=False):
    g = _gen('qkv', B, L, H, mlp, off, hats, K, ints)
    what = f'qkv B={B} L={L} H={H} mlp={mlp} off={off} hats={hats} K={K} ints={ints}'
    n_qkv = 3 * H * 128
    N, M = n_qkv + mlp, B * L
    if ints:
        A, Bw = _ints((M, K), g).bfloat16(), _ints((N, K), g).bfloat16()
        b = _ints((N,), g, 8).bfloat16()
    else:
        A, Bw = _rows(M, K, g, -2, 1).bfloat16(), (torch.randn(N, K, generator=g, device='cuda') * K ** -0.5).bfloat16()
        b = (torch.randn(N, generator=g, device='cuda') * 0.3).bfloat16()
    wq, wk = ((1 + 0.3 * torch.randn(128, generator=g, device='cuda')).bfloat16() for _ in range(2))
    T = off + L + 7
    cos, sin = _rope(T, g)
    shp = (B, H, T, 128)
    bufs = {n: Flat(shp, torch.bfloat16) for n in (('q', 'k', 'v', 'qhat', 'khat') if hats else ('q', 'k', 'v'))}
    rstd = {n: Flat((B, H, T), torch.float32) for n in (('q_rstd', 'k_rstd') if hats else ())}
    out = Canvas(M, max(mlp, 8), torch.bfloat16)
    o2 = Canvas(M, mlp, torch.bfloat16) if mlp else None
    wq_v, wk_v = _vec(wq), _vec(wk)   # the epilogue struct holds raw pointers: keep the buffers alive
    e = ops.make_qkv_epilogue(bufs['q'].view, bufs['k'].view, bufs['v'].view, wq_v, wk_v, cos, sin, H, T, off,
                              qhat=bufs['qhat'].view if hats else None, khat=bufs['khat'].view if hats else None,
                              q_rstd=rstd['q_rstd'].view if hats else None, k_rstd=rstd['k_rstd'].view if hats else None)
    a_op, b_op = _operand(A, 0), _operand(Bw, 0)
    kw = dict(out=out.view, epilogue=3, bias=_vec(b), out2=o2.view if o2 is not None else None, rows_per_batch=L, qkv=e,
              N=N)
    ops.gemm(a_op, b_op, **kw)
    torch.cuda.synchronize()
    for n, f in list(bufs.items()) + list(rstd.items()):
        assert f.intact(), f'{what}: {n} sentinel overwritten'
        outside = torch.cat([f.view[:, :, :off].flatten(), f.view[:, :, off + L:].flatten()])
        assert bool((outside == SENTINEL).all()), f'{what}: {n} written outside rows [off, off + L)'
    assert out.intact() and (o2 is None or o2.intact())
    if not mlp:
        assert bool((out.view == SENTINEL).all()), what + ': out written without MLP columns'
    if twice:
        first = {n: f.buf.clone() for n, f in bufs.items()}
        ops.gemm(a_op, b_op, **kw)
        torch.cuda.synchronize()
        assert all(torch.equal(first[n].view(torch.int16), f.buf.view(torch.int16)) for n, f in bufs.items()), what
    acc = R.exact(A.double() @ Bw.double().t()) if ints else G.gemm_acc(A, Bw)
    ref = G.gemm_qkv_ref(acc, b, wq, wk, cos, sin, H, L, off, n_qkv)
    del acc
    rows = slice(off, off + L)
    for n, f in bufs.items():
        check(f.view[:, :, rows], ref[n], 'gemm qkv_rope', f'{what} {n}')
    for n, f in rstd.items():
        check(f.view[:, :, rows], ref[n], 'gemm qkv_rope', f'{what} {n}', bf16_out=False)
    if ints:   # v is one rounding of an exact sum
        assert torch.equal(bufs['v'].view[:, :, rows].double(), R.bf(ref['v'].v)), what + ' v not bit-exact'
    if mlp:
        check(out.view, ref['out'], 'gemm qkv_rope', what + ' mlp out')
        check(o2.view, ref['out2'], 'gemm qkv_rope', what + ' mlp out2')


@pytest.mark.parametrize('ints', [True, False])
@pytest.mark.parametrize('H', [2, 24])
def test_gemm_qkv_rope(H, ints, ops):
    """n_qkv == N and the fused linear1 (MLP columns past n_qkv, at col - n_qkv); seq_offset 0 and > 0; qhat / rstd
    present and NULL; a sample boundary inside a 128-row tile (77 rows per sample)"""
    for mlp in (0, 512 if H == 2 else 1024):
        for off, hats in ((0, True), (13, False), (512, True)):
            qkv_case(ops, 3 if H == 2 else 2, 77, H, mlp, off, hats, ints=ints)
    qkv_case(ops, 1, 129, H, 288, 5, True, K=3072 if not ints else 200, ints=ints, twice=not ints)


# ---------------------------------------------------------------------------------------------------------------
# GEMM real shapes (Flux / Qwen: D 3072, MLP 12288, linear1 N 21504, linear2 K 15360; Wan-14B: D 5120, FFN 13824)
# ---------------------------------------------------------------------------------------------------------------
REAL = [('flux qkv', 4608, 9216, 3072, 'store', (0, 0)), ('flux mlp up', 4608, 12288, 3072, 'bias_gelu', (0, 0)),
        ('flux linear2', 4608, 3072, 15360, 'gate_res', (0, 0)), ('flux mlp dgrad', 4608, 12288, 3072, 'mul_gelu_grad', (0, 1)),
        ('flux dgrad', 4608, 3072, 12288, 'store', (0, 1)), ('flux wgrad', 3072, 3072, 4608, 'store', (1, 1)),
        ('wan ffn up', 2048, 13824, 5120, 'bias_gelu', (0, 0)), ('wan ffn down', 2048, 5120, 13824, 'gate_res', (0, 0)),
        ('wan wgrad', 5120, 13824, 2048, 'store', (1, 1))]


@pytest.mark.parametrize('case', REAL, ids=[c[0] for c in REAL])
def test_gemm_real_shapes(case, ops):
    _, M, N, K, epi, layout = case
    gemm_case(ops, M, N, K, epi, layout, rpb=M // 2 if epi == 'gate_res' else None)


def test_gemm_flux_single_block_linear1(ops):
    """QKV_ROPE at the fused linear1 of a Flux single block: N = 21504 = 3 x 3072 + 12288, 24 heads, 4608 tokens"""
    qkv_case(ops, 1, 4608, 24, 12288, 0, True, K=3072)


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
def attn_case(ops, B, H, Lq, Lk, scale, heads=None, bwd=True, growing=False, twice=False):
    g = _gen('attn', B, H, Lq, Lk, scale, growing)
    what = f'attn B={B} H={H} Lq={Lq} Lk={Lk} scale={scale:.4g} growing={growing} poly={POLY}'
    q = _rows(B * H * Lq, 128, g, -3, 0.5).view(B, H, Lq, 128)
    k = _rows(B * H * Lk, 128, g, -3, 0.5).view(B, H, Lk, 128)
    if growing:   # logits that grow along the keys: the running maximum moves at every key tile
        u = torch.randn(B, H, 1, 128, generator=g, device='cuda')
        q = u.expand(B, H, Lq, 128) * (0.5 + torch.rand(B, H, Lq, 1, generator=g, device='cuda'))
        k = u * torch.linspace(0, 4, Lk, device='cuda')[:, None] + 0.1 * torch.randn(B, H, Lk, 128, generator=g, device='cuda')
    q, k = q.bfloat16().contiguous(), k.bfloat16().contiguous()
    v = _rows(B * H * Lk, 128, g).view(B, H, Lk, 128).bfloat16()
    o = Canvas(B * Lq, H * 128, torch.bfloat16)
    lse = Flat((B, H, Lq), torch.float32)
    ops.attn_fwd(q, k, v, out=o.view, lse=lse.view, scale=scale)
    torch.cuda.synchronize()
    assert o.intact() and lse.intact(), what + ': sentinel overwritten'
    assert bool(torch.isfinite(o.view).all()) and bool(torch.isfinite(lse.view).all()), what + ': non-finite output'
    heads = heads or [(b, h) for b in range(B) for h in range(H)]
    for b, h in heads:
        ref = G.attn_fwd_ref(q[b, h], k[b, h], v[b, h], scale, poly=POLY)
        check(o.view[b * Lq:(b + 1) * Lq, h * 128:(h + 1) * 128], ref['o'], f'attn fwd poly={POLY}', f'{what} o {b},{h}')
        check(lse.view[b, h], ref['lse'], f'attn fwd poly={POLY}', f'{what} lse {b},{h}', bf16_out=False)
        del ref
    if not bwd:
        return
    dbuf = torch.full((B * Lq, H * 128 + 40), float('nan'), device='cuda', dtype=torch.bfloat16)
    d_o = dbuf[:, 8:8 + H * 128]
    d_o.copy_(_rows(B * Lq, H * 128, g))
    dq, dk, dv = Flat((B, H, Lq, 128), torch.bfloat16), Flat((B, H, Lk, 128), torch.bfloat16), Flat((B, H, Lk, 128), torch.bfloat16)
    delta = Flat((B, H, Lq), torch.float32)
    args = (q, k, v, o.view, d_o, lse.view)
    kw = dict(scale=scale, dq=dq.view, dk=dk.view, dv=dv.view, delta=delta.view)
    ops.attn_bwd(*args, **kw)
    torch.cuda.synchronize()
    assert all(t.intact() for t in (dq, dk, dv, delta)), what + ': backward sentinel overwritten'
    assert all(bool(torch.isfinite(t.view).all()) for t in (dq, dk, dv)), what + ': non-finite gradient'
    if twice:
        first = [t.view.clone() for t in (dq, dk, dv)]
        ops.attn_bwd(*args, **kw)
        torch.cuda.synchronize()
        assert all(torch.equal(a.view(torch.int16), t.view.view(torch.int16)) for a, t in zip(first, (dq, dk, dv))), \
            what + ': backward not repeatable'
    for b, h in heads:
        rows = slice(b * Lq, (b + 1) * Lq)
        cols = slice(h * 128, (h + 1) * 128)
        ref = G.attn_bwd_ref(q[b, h], k[b, h], v[b, h], o.view[rows, cols], d_o[rows, cols], lse.view[b, h], scale)
        w = f'{what} {b},{h}'
        check(delta.view[b, h][:, None], ref['delta'], 'attn bwd', w + ' delta', bf16_out=False)
        check(dv.view[b, h], ref['dv'], 'attn bwd', w + ' dv')
        check(dk.view[b, h], ref['dk'], 'attn bwd', w + ' dk')
        check(dq.view[b, h], ref['dq'], 'attn bwd', w + ' dq')
        del ref


PAIRS = [(1, 1), (63, 129), (64, 64), (65, 127), (127, 65), (128, 257), (129, 1), (257, 63), (1, 4101), (4101, 129),
         (129, 4101), (65, 65)]
SCALES = [128 ** -0.5, 1.0, 0.05]


@pytest.mark.parametrize('pair', PAIRS, ids=[f'{a}x{b}' for a, b in PAIRS])
def test_attention(pair, ops):
    Lq, Lk = pair
    for i, scale in enumerate(SCALES):
        attn_case(ops, 1 + (i == 1), 2, Lq, Lk, scale, bwd=not POLY)


def test_attention_many_heads_and_rescales(ops):
    """B x H = 3 x 24 with every head checked; large logits growing along the keys (the running max moves at every key
    tile); the backward twice for identical bits"""
    attn_case(ops, 3, 24, 129, 257, 128 ** -0.5, bwd=not POLY, twice=True)
    for scale in SCALES:
        attn_case(ops, 1, 2, 200, 1000, scale, growing=True, bwd=not POLY)


def test_attention_exact_cases(ops):
    """q = 0: every valid key has P = 1 and LSE = log2(seq_k), so O is the mean of exactly the valid keys' V rows
    (small integers: exact sums); seq_k = 1: O = v bit for bit"""
    for Lq, Lk in ((63, 1), (129, 1), (65, 63), (64, 129), (130, 4101)):
        g = _gen('attn0', Lq, Lk)
        q = torch.zeros(2, 3, Lq, 128, device='cuda', dtype=torch.bfloat16)
        k = _rows(2 * 3 * Lk, 128, g).view(2, 3, Lk, 128).bfloat16()
        v = _ints((2, 3, Lk, 128), g, 4).bfloat16()
        o = Canvas(2 * Lq, 3 * 128, torch.bfloat16)
        lse = Flat((2, 3, Lq), torch.float32)
        ops.attn_fwd(q, k, v, out=o.view, lse=lse.view)
        torch.cuda.synchronize()
        assert o.intact() and lse.intact()
        got = o.view.view(2, Lq, 3, 128).permute(0, 2, 1, 3)
        mean = v.double().mean(2, keepdim=True).expand(2, 3, Lq, 128)
        check(got, R.E(mean, 4 * R.U * mean.abs()), 'attn exact', f'q=0 Lq={Lq} Lk={Lk} o')
        assert torch.allclose(lse.view.double(), torch.full_like(lse.view.double(), float(torch.log2(torch.tensor(float(Lk))))),
                              rtol=4 * R.U, atol=4 * R.U), (Lq, Lk)
        if Lk == 1:
            assert torch.equal(got, v.expand(2, 3, Lq, 128)), f'seq_k = 1: o != v (Lq={Lq})'


ATT_REAL = [('flux', 1, 24, 4608, 4608), ('qwen', 1, 24, 4608, 4608), ('wan self', 1, 40, 1560, 1560),
            ('wan cross', 1, 40, 1560, 512)]


@pytest.mark.parametrize('case', ATT_REAL, ids=[c[0] for c in ATT_REAL])
def test_attention_real_shapes(case, ops):
    """every element of the first, middle and last head; NaN and sentinels everywhere"""
    name, B, H, Lq, Lk = case
    if name == 'qwen':   # same geometry as Flux, on 4096 image + 512 text tokens with a different head split checked
        heads = [(0, 1), (0, 11), (0, 22)]
    else:
        heads = [(b, h) for b in range(B) for h in (0, H // 2, H - 1)]
    attn_case(ops, B, H, Lq, Lk, 128 ** -0.5, heads=heads, bwd=not POLY)


@pytest.mark.parametrize('poly', [2, 4])
def test_attention_forward_poly_exponential(poly):
    """attn_fwd_kernel<2> / <4>: the forward checks of this file in a child process that selects the polynomial"""
    if POLY:
        pytest.skip('already inside a polynomial run')
    env = dict(os.environ, DPIPE_ATTN_FWD_POLY=str(poly))
    r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-x', '-s', '-m', 'gpu', '-p', 'no:cacheprovider',
                        os.path.abspath(__file__), '-k', 'test_attention and not poly and not exact'],
                       env=env, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), capture_output=True,
                       text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-6000:] + r.stderr[-3000:]
