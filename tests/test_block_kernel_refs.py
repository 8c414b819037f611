"""CPU: the fp64 references and the per-element check of tests/block_kernel_refs.py.

With their rounding points switched off the references are the plain operations, so they must agree with torch
autograd in float64.  The check must accept each reference's own output and reject each mutation the GPU tests are
there to catch: a sample reading sample 0's modulation row, a row missing from a partial sum, a skipped bf16 rounding
point, a flipped rope sign, and one element 2 ulps off in a row scaled by 1e-3 (which the whole-tensor 2 % bound of
test_kernels_gpu._check accepts)."""
import pytest
import torch

import block_kernel_refs as R

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _close(a, b, what):
    assert torch.allclose(a, b, rtol=1e-10, atol=1e-12 * max(1.0, b.abs().max().item())), (what, (a - b).abs().max().item())


def _as_kernel(ref, bf16_out):
    """what a kernel that computes the reference value exactly would write"""
    return R.bf(ref.v).bfloat16() if bf16_out else ref.v.float()


def _rejects(out, ref, bf16_out):
    assert R.accepts(_as_kernel(ref, bf16_out), ref, bf16_out), 'the check refuses the reference itself'
    assert not R.accepts(out, ref, bf16_out), 'the check accepts a mutated output'


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
B, L, D = 3, 40, 256


def _mod_inputs(N=64, K=256, seed=0):
    g = _g(seed)
    temb = (torch.randn(B, K, generator=g) + torch.randn(B, 1, generator=g)).bfloat16()
    W = (torch.randn(N, K, generator=g) * 0.05).bfloat16()
    bias = (torch.randn(N, generator=g) * 0.1).bfloat16()
    dmod = torch.randn(B, N, generator=g)
    dW0 = (torch.randn(N, K, generator=g) * 0.1).bfloat16()
    dtemb0 = torch.randn(B, K, generator=g)
    return temb, W, bias, dmod, dW0, dtemb0


def _ln_inputs(seed=1):
    g = _g(seed)
    x = (torch.randn(B * L, D, generator=g) * torch.logspace(-3, 2, B * L)[:, None] + 3).bfloat16()
    mod = (torch.randn(B, 3 * D, generator=g) * 0.3).bfloat16()
    dxn = (torch.randn(B * L, D, generator=g)).bfloat16()
    return x, mod[:, :D], mod[:, D:2 * D], mod[:, 2 * D:], dxn


def _stats(x):
    xd = x.double()
    mean = xd.mean(-1)
    rstd = torch.rsqrt(((xd - mean[:, None]) ** 2).mean(-1) + 1e-6)
    return mean.float(), rstd.float()


# ---------------------------------------------------------------------------------------------------------------
# references against autograd
# ---------------------------------------------------------------------------------------------------------------
def test_modulation_references_match_autograd():
    temb, W, bias, dmod, dW0, dtemb0 = _mod_inputs()
    t = temb.double().requires_grad_(True)
    w = W.double().requires_grad_(True)
    b = bias.double().requires_grad_(True)
    out = torch.nn.functional.silu(t) @ w.t() + b
    _close(R.mod_fwd_ref(temb, W, bias, off='all').v, out.detach(), 'mod_fwd')
    (out * dmod.double()).sum().backward()
    ref = R.mod_bwd_ref(dmod, temb, W, dW0, dtemb0, off='all')
    _close(ref['dbias'].v, b.grad, 'dbias')
    _close(ref['dW']().v, dW0.double() + w.grad, 'dW')
    _close(ref['dtemb'].v, dtemb0.double() + t.grad, 'dtemb')
    assert R.mod_bwd_ref(dmod, temb, W, None, dtemb0)['dW'](slice(5, 9)).v.shape == (4, 256)


@pytest.mark.parametrize('flags', [0, R.LN_MULT_DIRECT])
def test_layernorm_references_match_autograd(flags):
    x, shift, scale, gate, dxn = _ln_inputs()
    X = x.double().view(B, L, D).requires_grad_(True)
    sc = scale.double().requires_grad_(True)
    sh = shift.double().requires_grad_(True)
    mult = sc if flags & R.LN_MULT_DIRECT else 1 + sc
    xn = torch.nn.functional.layer_norm(X, (D,), eps=1e-6)
    out = xn * mult[:, None] + sh[:, None]
    ref = R.ln_modulate_fwd_ref(x, scale, shift, B, L, flags=flags, off='all')
    _close(ref['out'].v, out.detach().reshape(-1, D), 'out')
    _close(ref['mean'].v, X.detach().mean(-1).reshape(-1), 'mean')
    _close(ref['rstd'].v, torch.rsqrt(X.detach().var(-1, unbiased=False) + 1e-6).reshape(-1), 'rstd')
    dres = torch.randn(B * L, D, generator=_g(3)).bfloat16()
    (out * dxn.double().view(B, L, D)).sum().backward()
    mean, rstd = X.detach().mean(-1).reshape(-1), torch.rsqrt(X.detach().var(-1, unbiased=False) + 1e-6).reshape(-1)
    bref = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L, dres=dres, flags=flags, off='all')
    _close(bref['dx'].v, X.grad.reshape(-1, D) + dres.double(), 'dx')
    _close(bref['dscale'].v, sc.grad, 'dscale')
    _close(bref['dshift'].v, sh.grad, 'dshift')
    _close(bref['dscale_sum'].v, sc.grad.sum(0), 'dscale summed')
    _close(bref['dshift_sum'].v, sh.grad.sum(0), 'dshift summed')


def test_gate_and_colsum_references_match_autograd():
    x, shift, scale, gate, dxn = _ln_inputs()
    y = torch.randn(B * L, D, generator=_g(4)).bfloat16()
    gt = gate.double().requires_grad_(True)
    Y = y.double().view(B, L, D).requires_grad_(True)
    (dxn.double().view(B, L, D) * gt[:, None] * Y).sum().backward()
    ref = R.gate_bwd_ref(dxn, y, gate, B, L)
    _close(ref['dgate'].v, gt.grad, 'dgate')
    assert torch.equal(ref['dy'], Y.grad.reshape(-1, D).float().bfloat16().double())
    _close(ref['dbias'].v, ref['dy'].sum(0), 'dbias')
    _close(R.colsum_ref(y).v, y.double().sum(0), 'colsum')


def _norm_rope(x, w, c, s, full_width):
    """RMSNorm (per head, or over the full width) then the interleaved rotation, in fp64"""
    if full_width:   # x [B, L, C]
        xh = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
        y = (xh * w).view(x.shape[0], x.shape[1], -1, 128).permute(0, 2, 1, 3)
    else:            # x [B, H, L, 128]
        xh = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
        y = xh * w
    yr = torch.stack([-y[..., 1::2], y[..., 0::2]], -1).flatten(-2)
    return y * c + yr * s, xh


def _tables(Lt, seed):
    ang = torch.rand(Lt, 64, generator=_g(seed), dtype=F64) * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).float(), torch.sin(ang).repeat_interleave(2, 1).float()


def _qk_case(rope_sign=1.0, samples=None):
    g = _g(5)
    Bq, H, off, rows = 2, 2, 3, 9
    Lt = off + rows + 2
    x = [torch.randn(Bq, H, Lt, 128, generator=g, dtype=F64) for _ in range(2)]
    rstd = [torch.rsqrt(t.pow(2).mean(-1) + 1e-6) for t in x]
    hat = [t * r[..., None] for t, r in zip(x, rstd)]
    w = [(1 + 0.2 * torch.randn(128, generator=g, dtype=F64)) for _ in range(2)]
    d = [torch.randn(Bq, H, Lt, 128, generator=g, dtype=F64) for _ in range(3)]
    cos, sin = _tables(Lt, 6)
    ref = R.qknorm_rope_bwd_ref(d[0], d[1], d[2], hat[0], hat[1], rstd[0], rstd[1], w[0], w[1], cos, sin, Bq, H, off, rows,
                                rope_sign=rope_sign, samples=samples)
    return (Bq, H, off, rows, x, w, d, cos, sin), ref


def test_qknorm_rope_reference_matches_autograd():
    (Bq, H, off, rows, x, w, d, cos, sin), ref = _qk_case()
    sl = slice(off, off + rows)
    c, s = cos[sl].double(), sin[sl].double()
    grads, dws = [], []
    for i in range(2):
        xi = x[i][:, :, sl].clone().requires_grad_(True)
        wi = w[i].clone().requires_grad_(True)
        (_norm_rope(xi, wi, c, s, False)[0] * d[i][:, :, sl]).sum().backward()
        grads.append(xi.grad)
        dws.append(wi.grad)
    grads.append(d[2][:, :, sl])
    want = torch.stack(grads).permute(1, 3, 0, 2, 4).reshape(Bq * rows, 3 * H * 128)
    _close(ref['dqkv'].v, want, 'dqkv')
    _close(ref['dw'].v, torch.stack(dws), 'dw')
    _, one = _qk_case(samples=[1])                                 # one sample's rows, the same d weight
    assert torch.equal(one['dqkv'].v, ref['dqkv'].v[rows:]) and torch.equal(one['dqkv'].e, ref['dqkv'].e[rows:])
    assert torch.equal(one['dw'].v, ref['dw'].v) and torch.equal(one['dw'].e, ref['dw'].e)


@pytest.mark.parametrize('weight,rope', [(True, True), (True, False), (False, True)])
def test_wan_norm_rope_references_match_autograd(weight, rope):
    g = _g(7)
    Bw, Lw, H = 2, 5, 2
    Cw = H * 128
    src = torch.randn(Bw * Lw, Cw + 8, generator=g).bfloat16()
    w = (1 + 0.2 * torch.randn(Cw, generator=g)).bfloat16() if weight else None
    cos, sin = _tables(Lw, 8)
    ref = R.wan_norm_rope_fwd_ref(src, w, rope, cos, sin, Bw, Lw, H, off='all')
    x = src[:, :Cw].double().view(Bw, Lw, Cw).requires_grad_(True)
    wd = w.double().requires_grad_(True) if weight else None
    c, s = (cos.double(), sin.double()) if rope else (torch.ones(Lw, 128, dtype=F64), torch.zeros(Lw, 128, dtype=F64))
    if weight:
        y, xh = _norm_rope(x, wd, c, s, True)
        _close(ref['xhat'].v, xh.detach().reshape(-1, Cw), 'xhat')
    else:
        y = x.view(Bw, Lw, H, 128).permute(0, 2, 1, 3)
        y = y * c + torch.stack([-y[..., 1::2], y[..., 0::2]], -1).flatten(-2) * s
    _close(ref['dst'].v, y.detach(), 'dst')
    dy = torch.randn(Bw, H, Lw, 128, generator=g).bfloat16()
    (y * dy.double()).sum().backward()
    xh = ref['xhat'].v if weight else None
    rstd = ref['rstd'].v if weight else None
    bref = R.wan_norm_rope_bwd_ref(dy, xh, rstd, w, rope, cos, sin, Bw, Lw, H)
    _close(bref['dx'].v, x.grad.reshape(-1, Cw), 'dx')
    if weight:
        _close(bref['dw'].v, wd.grad, 'dw')
        parts = [R.wan_norm_rope_bwd_ref(dy[b:b + 1], xh[b * Lw:(b + 1) * Lw], rstd[b * Lw:(b + 1) * Lw], w, rope, cos, sin, 1,
                                         Lw, H, total_rows=Bw * Lw)['dw'] for b in range(Bw)]
        _close(sum(p.v for p in parts), bref['dw'].v, 'dw of the parts')
        _close(sum(p.e for p in parts), bref['dw'].e, 'dw bound of the parts')


def test_mse_reference_matches_autograd():
    g = _g(9)
    out = torch.randn(2, 3, 4, 5, generator=g).bfloat16()
    tgt = torch.randn(2, 3, 4, 5, generator=g)
    mask = torch.rand(2, 1, 4, 5, generator=g)
    o = out.double().requires_grad_(True)
    loss = ((o - tgt.double()) ** 2 * mask.double()).mean()
    loss.backward()
    ref = R.mse_loss_ref(out, tgt, mask)
    _close(ref['loss'].v, loss.detach(), 'loss')
    _close(ref['dout'].v, o.grad, 'dout')


# ---------------------------------------------------------------------------------------------------------------
# the check rejects what the kernels could get wrong
# ---------------------------------------------------------------------------------------------------------------
def test_rejects_a_sample_reading_sample_0s_modulation_row():
    x, shift, scale, gate, dxn = _ln_inputs()
    ref = R.ln_modulate_fwd_ref(x, scale, shift, B, L)['out']
    wrong = R.ln_modulate_fwd_ref(x, scale[:1].expand(B, D), shift, B, L)['out']
    _rejects(_as_kernel(wrong, True), ref, True)
    wrong = R.ln_modulate_fwd_ref(x, scale, shift[:1].expand(B, D), B, L)['out']
    _rejects(_as_kernel(wrong, True), ref, True)
    y = torch.randn(B * L, D, generator=_g(4)).bfloat16()
    dy = R.gate_bwd_ref(dxn, y, gate, B, L)['dy']
    assert not torch.equal(R.gate_bwd_ref(dxn, y, gate[:1].expand(B, D), B, L)['dy'], dy)
    temb, W, bias, dmod, dW0, dtemb0 = _mod_inputs()
    ref = R.mod_bwd_ref(dmod, temb, W, dW0, dtemb0)
    wrong = R.mod_bwd_ref(dmod, temb[:1].expand(B, -1), W, dW0, dtemb0)
    _rejects(_as_kernel(wrong['dtemb'], False), ref['dtemb'], False)
    _rejects(_as_kernel(wrong['dW'](), True), ref['dW'](), True)


@pytest.mark.parametrize('row', [R.ROW_CHUNK - 1, 3])
def test_rejects_a_row_missing_from_a_partial_sum(row):
    """the last row of a 16-row chunk, or of the first 4-row group of each chunk"""
    x, shift, scale, gate, dxn = _ln_inputs()
    mean, rstd = _stats(x)
    ref = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L)
    wrong = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L, drop_row=row)
    for k in ('dscale', 'dshift', 'dscale_sum', 'dshift_sum'):
        _rejects(_as_kernel(wrong[k], False), ref[k], False)


@pytest.mark.parametrize('flags,point', [(0, 'one_plus_scale'), (R.LN_ROUND_STEPS, 'steps')])
def test_rejects_a_skipped_layernorm_rounding_point(flags, point):
    x, shift, scale, gate, dxn = _ln_inputs()
    ref = R.ln_modulate_fwd_ref(x, scale, shift, B, L, flags=flags)['out']
    wrong = R.ln_modulate_fwd_ref(x, scale, shift, B, L, flags=flags, off={point})['out']
    _rejects(_as_kernel(wrong, True), ref, True)
    if point == 'one_plus_scale':
        mean, rstd = _stats(x)
        ref = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L)['dx']
        wrong = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L, off={point})['dx']
        _rejects(_as_kernel(wrong, True), ref, True)


def test_rejects_unrounded_silu_or_dmod():
    temb, W, bias, dmod, dW0, dtemb0 = _mod_inputs()
    ref = R.mod_fwd_ref(temb, W, bias)
    _rejects(_as_kernel(R.mod_fwd_ref(temb, W, bias, off={'silu'}), True), ref, True)
    ref = R.mod_bwd_ref(dmod, temb, W, None, dtemb0)
    for point in ('silu', 'dmod', 'partials'):
        wrong = R.mod_bwd_ref(dmod, temb, W, None, dtemb0, off={point})
        if point != 'partials':
            _rejects(_as_kernel(wrong['dW'](), True), ref['dW'](), True)
        if point == 'dmod':
            _rejects(_as_kernel(wrong['dbias'], False), ref['dbias'], False)
        if point != 'silu':   # d temb takes silu' of the bf16 temb, not the rounded silu
            _rejects(_as_kernel(wrong['dtemb'], False), ref['dtemb'], False)


def test_rejects_a_flipped_rope_transpose_sign():
    _, ref = _qk_case()
    _, wrong = _qk_case(rope_sign=-1.0)
    _rejects(_as_kernel(wrong['dqkv'], True), ref['dqkv'], True)
    g = _g(7)
    Bw, Lw, H = 2, 5, 2
    dy = torch.randn(Bw, H, Lw, 128, generator=g).bfloat16()
    cos, sin = _tables(Lw, 8)
    ref = R.wan_norm_rope_bwd_ref(dy, None, None, None, True, cos, sin, Bw, Lw, H)['dx']
    wrong = R.wan_norm_rope_bwd_ref(dy, None, None, None, True, cos, sin, Bw, Lw, H, rope_sign=-1.0)['dx']
    _rejects(_as_kernel(wrong, True), ref, True)


def test_rejects_two_ulps_in_a_small_row_that_the_old_bound_accepts():
    from test_kernels_gpu import _check
    x, shift, scale, gate, dxn = _ln_inputs()
    dxn = dxn.clone()
    dxn[7] = (dxn[7].float() * 1e-3).bfloat16()                 # row 7 is a thousand times smaller than the others
    mean, rstd = _stats(x)
    ref = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L)['dx']
    out = _as_kernel(ref, True)
    j = int(out[7].float().abs().argmax())
    bits = out.view(torch.int16).clone()
    bits[7, j] += 2                                                # two bf16 ulps
    wrong = bits.view(torch.bfloat16)
    _rejects(wrong, ref, True)
    _check(wrong, ref.v)


def test_exact_and_boundary_cases_of_the_rounding_model():
    """a value on a bf16 grid point with no error rounds to itself with no bound; one within its bound of a rounding
    boundary gets one ulp; the ulp of 1.0 is 2^-7"""
    assert R.ulp(torch.tensor([1.0], dtype=F64)).item() == 2.0 ** -7
    assert R.ulp(torch.tensor([1.5e-3], dtype=F64)).item() == 2.0 ** -17
    exact = R.rnd(R.E(torch.tensor([1.0, 3.0], dtype=F64)), 'p', ())
    assert exact.e.abs().max().item() == 0 and torch.equal(exact.v, torch.tensor([1.0, 3.0], dtype=F64))
    mid = 1.0 + 2.0 ** -8                                          # halfway between 1 and 1 + 2^-7
    near = R.rnd(R.E(torch.tensor([mid + 1e-9], dtype=F64), torch.tensor([1e-8], dtype=F64)), 'p', ())
    assert near.e.item() > 2.0 ** -7
    far = R.rnd(R.E(torch.tensor([mid + 1e-4], dtype=F64), torch.tensor([1e-8], dtype=F64)), 'p', ())
    assert far.e.item() == 0 and far.v.item() == 1.0 + 2.0 ** -7
