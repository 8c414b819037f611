"""CPU: the fp64 references of the wgmma GEMM and the attention kernels (tests/gemm_attn_refs.py).

With every rounding point off each reference is the plain operation, so it must agree with torch in float64.  The check
must accept each reference's own rounded output and reject each mutation tests/test_gemm_attn_gpu.py is there to catch:
a dropped k-block, a shifted bias or accumulation row, a sample reading the wrong gate row, a skipped rounding point, a
flipped rope sign or position, the fused MLP half written at the wrong column, a dropped or leaked key, the LSE in the
wrong base, a missing scale, a padded query row that is not masked, and D taken from the exact output instead of the
given one."""
import math

import pytest
import torch

import block_kernel_refs as R
import gemm_attn_refs as G

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, what):
    assert torch.allclose(a, b, rtol=1e-10, atol=1e-12 * max(1.0, b.abs().max().item())), (what, (a - b).abs().max().item())


def _as_kernel(ref, bf16_out=True):
    """what a kernel that computes the reference value exactly would write"""
    return R.bf(ref.v).bfloat16() if bf16_out else ref.v.float()


def _rejects(mutated, ref, bf16_out=True):
    assert R.accepts(_as_kernel(ref, bf16_out), ref, bf16_out), 'the check refuses the reference itself'
    assert not R.accepts(_as_kernel(mutated, bf16_out), ref, bf16_out), 'the check accepts a mutated output'


def _rows(n, cols, g, lo=-3.0, hi=2.0):
    mag = 10 ** (lo + (hi - lo) * torch.rand(n, 1, generator=g))
    return torch.randn(n, cols, generator=g) * mag


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
M, N, K = 200, 64, 200      # rows across two 128-row tiles; k-blocks 64, 64, 64 and a partial 8


def _gemm_inputs(seed=0, m=M, n=N, k=K):
    g = _g(seed)
    A = _rows(m, k, g).bfloat16()
    Bw = _rows(n, k, g, -1, 0.5).bfloat16()
    bias = torch.randn(n, generator=g).bfloat16()
    return A, Bw, bias, g


def test_gemm_references_match_plain_fp64():
    A, Bw, bias, g = _gemm_inputs()
    acc = G.gemm_acc(A, Bw)
    ex = A.double() @ Bw.double().t()
    _close(acc.v, ex, 'acc')
    old = _rows(M, N, g).bfloat16()
    _close(G.gemm_store_ref(acc, bias, old)['out'].v, ex + old.double() + bias.double(), 'store')
    ref = G.gemm_bias_gelu_ref(acc, bias, off='all')
    _close(ref['out2'].v, ex + bias.double(), 'bias_gelu u')
    _close(ref['out'].v, torch.nn.functional.gelu(ex + bias.double(), approximate='tanh'), 'bias_gelu')
    res, gate = _rows(M, N, g).bfloat16(), torch.randn(4, N, generator=g).bfloat16()
    ref = G.gemm_gate_res_ref(acc, res, gate, 50, bias, off='all')
    want = res.double() + gate.double().repeat_interleave(50, 0) * (ex + bias.double())
    _close(ref['out'].v, want, 'gate_res')
    aux = torch.randn(M, N, generator=g).bfloat16()
    u = aux.double().requires_grad_(True)
    grad, = torch.autograd.grad(torch.nn.functional.gelu(u, approximate='tanh'), u, ex)
    _close(G.gemm_mul_gelu_grad_ref(acc, aux, off='all')['out'].v, grad, 'mul_gelu_grad')


def _mut_gemm(A, Bw, bias):
    acc = G.gemm_acc(A, Bw)
    return G.gemm_store_ref(acc, bias)['out']


@pytest.mark.parametrize('mutation', ['interior_kblock', 'last_partial_kblock', 'bias_next_column'])
def test_gemm_check_rejects(mutation):
    A, Bw, bias, _ = _gemm_inputs(1)
    ref = _mut_gemm(A, Bw, bias)
    if mutation == 'interior_kblock':
        A2 = A.clone()
        A2[:, 64:128] = 0
        bad = _mut_gemm(A2, Bw, bias)
    elif mutation == 'last_partial_kblock':
        A2 = A.clone()
        A2[:, 192:] = 0
        bad = _mut_gemm(A2, Bw, bias)
    else:
        bad = _mut_gemm(A, Bw, torch.roll(bias, -1))
    _rejects(bad, ref)


def test_store_check_rejects_accumulate_reading_the_next_row():
    A, Bw, bias, g = _gemm_inputs(2)
    old = _rows(M, N, g).bfloat16()
    acc = G.gemm_acc(A, Bw)
    ref = G.gemm_store_ref(acc, bias, old)['out']
    _rejects(G.gemm_store_ref(acc, bias, torch.roll(old, -1, 0))['out'], ref)


RPB = 77   # 77 rows per sample: the boundary between samples 0 and 1 lies inside the first 128-row tile


@pytest.mark.parametrize('mutation', ['gate_of_sample_0', 'sample_off_by_one_at_a_boundary', 'y_not_rounded'])
def test_gate_res_check_rejects(mutation):
    A, Bw, bias, g = _gemm_inputs(3, m=4 * RPB)
    acc = G.gemm_acc(A, Bw)
    res = _rows(4 * RPB, N, g).bfloat16()
    gate = (torch.randn(4, N, generator=g) + torch.arange(4)[:, None]).bfloat16()   # a different row per sample
    ref = G.gemm_gate_res_ref(acc, res, gate, RPB, bias)
    if mutation == 'gate_of_sample_0':
        bad = G.gemm_gate_res_ref(acc, res, gate[:1].expand(4, -1), RPB, bias)
    elif mutation == 'sample_off_by_one_at_a_boundary':
        sample = G.sample_of_rows(4 * RPB, RPB, 'cpu').clone()
        sample[RPB] = 0        # the first row of sample 1 (row 77 of tile 0) takes sample 0's gate
        bad = G.gemm_gate_res_ref(acc, res, gate, RPB, bias, sample=sample)
    else:
        bad = G.gemm_gate_res_ref(acc, res, gate, RPB, bias, off={'y'})
    _rejects(bad['out'], ref['out'])


def test_fused_epilogues_accept_their_own_outputs():
    A, Bw, bias, g = _gemm_inputs(4)
    acc = G.gemm_acc(A, Bw)
    for ref in (G.gemm_bias_gelu_ref(acc, bias), G.gemm_bias_gelu_ref(acc, None),
                G.gemm_gate_res_ref(acc, _rows(M, N, g).bfloat16(), torch.randn(4, N, generator=g).bfloat16(), 50, bias),
                G.gemm_mul_gelu_grad_ref(acc, torch.randn(M, N, generator=g).bfloat16())):
        for name, e in ref.items():
            assert R.accepts(_as_kernel(e), e), name


def test_bias_gelu_accepts_either_neighbour_at_a_rounding_tie():
    """u = bf16(acc + bias) at an exact tie may round to either neighbour, and the kernel's gelu of that neighbour must
    pass: a bound that carries the one-ulp flip through gelu' alone misses gelu's curvature over that ulp (at u = 2.859
    the kernel's value is 1.00008 bounds away).  Found in place on an H100: the BIAS_GELU GEMM of a Qwen-Image block
    (M = 390, N = 2048, K = 512), element (370, 1293), got -0.0038300 want -0.0036374 bound 1.924e-4.  Every tie
    between adjacent bf16 values in [2^-20, 8) of either sign."""
    pos = torch.arange(0x3580, 0x4100, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).double()   # 2^-20 .. 8
    for vals in (pos, -pos):
        lo, hi = vals[:-1], vals[1:]
        acc = R.E(((lo + hi) / 2)[:, None], torch.full((lo.numel(), 1), 1e-30, dtype=torch.float64))
        ref = G.gemm_bias_gelu_ref(acc)
        for nb in (lo, hi):
            R.check(torch.nn.functional.gelu(nb.float(), approximate='tanh')[:, None], ref['out'], 'gelu of a neighbour',
                    bf16_out=False)


# ---------------------------------------------------------------------------------------------------------------
# QKV epilogue
# ---------------------------------------------------------------------------------------------------------------
H, QB, QL, QOFF = 2, 2, 40, 9


def _qkv_inputs(seed=5, mlp=256):
    g = _g(seed)
    n_qkv = 3 * H * 128
    A = _rows(QB * QL, 96, g, -1, 1).bfloat16()
    Bw = (torch.randn(n_qkv + mlp, 96, generator=g) * 0.2).bfloat16()
    bias = (torch.randn(n_qkv + mlp, generator=g) * 0.3).bfloat16()
    wq, wk = ((1 + 0.3 * torch.randn(128, generator=g)).bfloat16() for _ in range(2))
    ang = torch.rand(QOFF + QL + 5, 64, generator=g) * 6.28
    cos, sin = torch.cos(ang).repeat_interleave(2, 1), torch.sin(ang).repeat_interleave(2, 1)
    return A, Bw, bias, wq, wk, cos, sin, n_qkv


def _qkv(A, Bw, bias, wq, wk, cos, sin, n_qkv, off=()):
    return G.gemm_qkv_ref(G.gemm_acc(A, Bw), bias, wq, wk, cos, sin, H, QL, QOFF, n_qkv, off=off)


def test_qkv_reference_matches_plain_fp64():
    A, Bw, bias, wq, wk, cos, sin, n_qkv = _qkv_inputs()
    ref = _qkv(A, Bw, bias, wq, wk, cos, sin, n_qkv, off='all')
    x = A.double() @ Bw.double().t() + bias.double()
    hd = H * 128
    c = cos[QOFF:QOFF + QL].double()[:, 0::2]
    s = sin[QOFF:QOFF + QL].double()[:, 0::2]
    for which, name, w in ((0, 'q', wq), (1, 'k', wk)):
        t = x[:, which * hd:(which + 1) * hd].reshape(QB, QL, H, 128).transpose(1, 2)
        rstd = torch.rsqrt((t * t).mean(-1, keepdim=True) + 1e-6)
        y = t * rstd * w.double()
        rot = torch.view_as_real(torch.view_as_complex(y.reshape(QB, H, QL, 64, 2).contiguous()) * torch.complex(c, s))
        _close(ref[name].v, rot.reshape(QB, H, QL, 128), name)
        _close(ref[name + 'hat'].v, t * rstd, name + 'hat')
        _close(ref[name + '_rstd'].v, rstd[..., 0], name + '_rstd')
    _close(ref['v'].v, x[:, 2 * hd:3 * hd].reshape(QB, QL, H, 128).transpose(1, 2), 'v')
    _close(ref['out'].v, torch.nn.functional.gelu(x[:, n_qkv:], approximate='tanh'), 'mlp')
    ref = _qkv(A, Bw, bias, wq, wk, cos, sin, n_qkv)
    for name, e in ref.items():
        assert R.accepts(_as_kernel(e, name not in ('q_rstd', 'k_rstd')), e, name not in ('q_rstd', 'k_rstd')), name


@pytest.mark.parametrize('mutation', ['rope_sign', 'seq_offset_ignored', 'rstd_from_unrounded_pre', 'mlp_at_col'])
def test_qkv_check_rejects(mutation):
    A, Bw, bias, wq, wk, cos, sin, n_qkv = _qkv_inputs(6, mlp=1024)
    ref = _qkv(A, Bw, bias, wq, wk, cos, sin, n_qkv)
    if mutation == 'rope_sign':
        _rejects(_qkv(A, Bw, bias, wq, wk, cos, -sin, n_qkv)['q'], ref['q'])
    elif mutation == 'seq_offset_ignored':   # rows rotated by the angles of positions 0.. instead of QOFF..
        bad = _qkv(A, Bw, bias, wq, wk, torch.roll(cos, QOFF, 0), torch.roll(sin, QOFF, 0), n_qkv)
        _rejects(bad['k'], ref['k'])
    elif mutation == 'rstd_from_unrounded_pre':
        bad = _qkv(A, Bw, bias, wq, wk, cos, sin, n_qkv, off={'pre_ss'})
        assert not R.accepts(_as_kernel(bad['q_rstd'], False), ref['q_rstd'], False)
    else:
        # the MLP half written at `col` lands n_qkv columns to the right of where it belongs; what the view holds
        # from column 0 is the kernel's sentinel (here: zeros) up to n_qkv, then columns shifted by n_qkv
        mlp = _as_kernel(ref['out'])
        bad = torch.zeros_like(mlp)
        bad[:, n_qkv:] = mlp[:, :mlp.shape[1] - n_qkv]
        assert R.accepts(mlp, ref['out']) and not R.accepts(bad, ref['out'])


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
def _attn_inputs(Lq, Lk, seed=7, qmag=1.0):
    g = _g(seed)
    q = (_rows(Lq, 128, g, -1, 0.3) * qmag).bfloat16()
    k = _rows(Lk, 128, g, -1, 0.3).bfloat16()
    v = _rows(Lk, 128, g).bfloat16()
    return q, k, v, g


def _attn_plain(q, k, v, scale):
    s = (q.double() @ k.double().t()) * scale
    return torch.softmax(s, -1) @ v.double(), torch.logsumexp(s, -1) / math.log(2)


@pytest.mark.parametrize('scale', [128 ** -0.5, 1.0, 0.05])
def test_attention_references_match_plain_fp64(scale):
    q, k, v, g = _attn_inputs(70, 300)
    o, lse = _attn_plain(q, k, v, scale)
    ref = G.attn_fwd_ref(q, k, v, scale, off='all')
    _close(ref['o'].v, o, 'o')
    _close(ref['lse'].v, lse, 'lse')
    do = _rows(70, 128, g).bfloat16()
    Q, Kt, V = (t.double().requires_grad_(True) for t in (q, k, v))
    out = torch.softmax((Q @ Kt.t()) * scale, -1) @ V
    dq, dk, dv = torch.autograd.grad(out, (Q, Kt, V), do.double())
    b = G.attn_bwd_ref(q, k, v, o, do, lse, scale, off='all')
    _close(b['dq'].v, dq, 'dq')
    _close(b['dk'].v, dk, 'dk')
    _close(b['dv'].v, dv, 'dv')
    # with its rounding points on, the check accepts each reference's own output
    ref = G.attn_fwd_ref(q, k, v, scale)
    assert R.accepts(_as_kernel(ref['o']), ref['o']) and R.accepts(_as_kernel(ref['lse'], False), ref['lse'], False)
    for poly in (2, 4):
        rp = G.attn_fwd_ref(q, k, v, scale, poly=poly)
        assert (rp['o'].e >= ref['o'].e).all() and R.accepts(_as_kernel(rp['o']), rp['o'])
    b = G.attn_bwd_ref(q, k, v, _as_kernel(ref['o']), do, ref['lse'].v.float(), scale)
    for name in ('dq', 'dk', 'dv'):
        assert R.accepts(_as_kernel(b[name]), b[name]), name


def test_poly_columns_follow_the_score_fragment_layout():
    """attn_fwd_kernel<POLY>: register pair i of a thread holds columns 8 (i >> 2) + 2 (lane & 3) + {0, 1} of row half
    (i >> 1) & 1; the pair takes the polynomial when ((i >> 1) & 7) < POLY"""
    for poly in (2, 4):
        want = torch.zeros(128, dtype=torch.bool)
        for i in range(0, 64, 2):
            for lane in range(4):
                for h in range(2):
                    if ((i >> 1) & 1) == h and ((i >> 1) & 7) < poly:
                        col = 8 * (i >> 2) + 2 * lane
                        want[col] = want[col + 1] = True
        assert torch.equal(G.poly_columns(128, poly, 'cpu'), want), poly


LQ, LK = 70, 300   # three key tiles, the last one partial (44 keys)


@pytest.mark.parametrize('mutation', ['last_partial_key_tile_dropped', 'masked_key_let_through', 'P_unrounded',
                                      'lse_natural_log'])
def test_attention_forward_check_rejects(mutation):
    q, k, v, _ = _attn_inputs(LQ, LK, 8, qmag=0.3)
    scale = 128 ** -0.5
    ref = G.attn_fwd_ref(q, k, v, scale)
    if mutation == 'last_partial_key_tile_dropped':
        _rejects(G.attn_fwd_ref(q, k[:256], v[:256], scale)['o'], ref['o'])
    elif mutation == 'masked_key_let_through':   # the first padded key: K and V zero-filled, score 0
        z = torch.zeros(1, 128, dtype=torch.bfloat16)
        bad = G.attn_fwd_ref(q, torch.cat([k, z]), torch.cat([v, z]), scale)
        _rejects(bad['o'], ref['o'])
        _rejects(bad['lse'], ref['lse'], False)
    elif mutation == 'P_unrounded':
        _rejects(G.attn_fwd_ref(q, k, v, scale, off={'P'})['o'], ref['o'])
    else:
        bad = R.E(ref['lse'].v * math.log(2), ref['lse'].e)
        _rejects(bad, ref['lse'], False)


@pytest.mark.parametrize('mutation', ['dk_missing_scale', 'padded_query_reads_next_sample', 'D_from_exact_o'])
def test_attention_backward_check_rejects(mutation):
    q, k, v, g = _attn_inputs(LQ, LK, 9)
    scale = 128 ** -0.5
    fwd = G.attn_fwd_ref(q, k, v, scale)
    o, lse = _as_kernel(fwd['o']), fwd['lse'].v.float()
    do = _rows(LQ, 128, g).bfloat16()
    ref = G.attn_bwd_ref(q, k, v, o, do, lse, scale)
    if mutation == 'dk_missing_scale':
        _rejects(R.E(ref['dk'].v / scale, ref['dk'].e), ref['dk'])
    elif mutation == 'padded_query_reads_next_sample':
        # query row LQ (inside the last 64-query chunk) is not masked: its Q is the zero fill, its dO the next
        # sample's first row
        do_next = _rows(1, 128, g).bfloat16()
        z = torch.zeros(1, 128, dtype=torch.bfloat16)
        bad = G.attn_bwd_ref(torch.cat([q, z]), k, v, torch.cat([o, z]), torch.cat([do, do_next]),
                             torch.cat([lse, torch.zeros(1)]), scale)
        _rejects(bad['dv'], ref['dv'])
    else:
        bad = G.attn_bwd_ref(q, k, v, G.attn_exact(q, k, v, scale), do, lse, scale)
        assert not (R.accepts(_as_kernel(bad['dq']), ref['dq']) and R.accepts(_as_kernel(bad['dk']), ref['dk']))
