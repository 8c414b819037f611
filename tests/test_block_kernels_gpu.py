"""GPU: the HBM-bound block kernels (modulation linears, LayerNorm + modulation, gated residual, column sums, q/k
RMSNorm-RoPE backward, Wan RMSNorm-RoPE, masked MSE) element by element against the fp64 references of
tests/block_kernel_refs.py, at micro-batches 1-8, the real widths and every width the host checks accept.

Inputs have structure rather than plain randn: row magnitudes spread over 1e-3 .. 1e2, LayerNorm rows whose mean is far
larger than their spread, and a different modulation row per sample, so that a wrong element in a small row or a
sample reading its neighbour's modulation stands out.  Every output is written into a view of a larger buffer (row
stride above the width, rows before and after it) filled with a sentinel, and the sentinel must survive."""
import ctypes
import zlib

import pytest
import torch

import block_kernel_refs as R

pytestmark = pytest.mark.gpu

SENTINEL = -12288.0   # exact in bf16 and fp32, far outside every output


@pytest.fixture(scope='module')
def ops():
    from diffusion_pipe_b200 import ops as o
    return o


def _lib():
    from diffusion_pipe_b200 import _lib as L
    return L


def _call(fn, *args):
    from diffusion_pipe_b200 import ops as o
    L = _lib()
    L.check(getattr(L.lib(), fn)(*args, o._stream()), fn)


P = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731


class Canvas:
    """a [rows, cols] output view inside a sentinel-filled buffer with `pad` extra columns per row and rows around it"""

    def __init__(self, rows, cols, dtype, pad=24, col0=8):
        self.buf = torch.full((rows + 3, cols + pad), SENTINEL, dtype=dtype, device='cuda')
        self.view = self.buf[1:rows + 1, col0:col0 + cols]
        self.inside = torch.zeros(self.buf.shape, dtype=torch.bool, device='cuda')
        self.inside[1:rows + 1, col0:col0 + cols] = True

    def intact(self):
        return bool((self.buf[~self.inside] == SENTINEL).all())


class Flat:
    """a contiguous [n] (or [*shape]) output inside a sentinel-filled buffer"""

    def __init__(self, shape, dtype, margin=64):
        n = 1
        for s in (shape if isinstance(shape, tuple) else (shape,)):
            n *= s
        self.buf = torch.full((n + 2 * margin,), SENTINEL, dtype=dtype, device='cuda')
        self.view = self.buf[margin:margin + n].view(shape)
        self.m = margin
        self.n = n

    def intact(self):
        return bool((self.buf[:self.m] == SENTINEL).all() and (self.buf[self.m + self.n:] == SENTINEL).all())


def _rows(n, cols, gen, lo=-3.0, hi=2.0):
    """[n, cols] fp32 rows of randn, each scaled by a magnitude log-uniform in [10^lo, 10^hi]"""
    mag = 10 ** (lo + (hi - lo) * torch.rand(n, 1, generator=gen, device='cuda'))
    return torch.randn(n, cols, generator=gen, device='cuda') * mag


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


# ---------------------------------------------------------------------------------------------------------------
# modulation linears
# ---------------------------------------------------------------------------------------------------------------
_W = {}


def _weight(N, K):
    if (N, K) not in _W:
        _W.clear()
        g = _gen('W', N, K)
        _W[(N, K)] = ((torch.randn(N, K, generator=g, device='cuda') * 0.02).bfloat16(),
                      (torch.randn(N, generator=g, device='cuda') * 0.05).bfloat16())
    return _W[(N, K)]


def _temb(B, K, g):
    return (_rows(B, K, g, -1, 0.7) + torch.randn(B, 1, generator=g, device='cuda')).bfloat16()   # per-sample rows


def _mod_fwd_case(B, N, K, with_bias, W=None):
    g = _gen('mf', B, N, K, with_bias)
    if W is None:
        W, bias = _weight(N, K)
    else:
        bias = (torch.randn(N, generator=g, device='cuda') * 0.05).bfloat16()
    bias = bias if with_bias else None
    temb = _temb(B, K, g)
    out = Flat((B, N), torch.bfloat16)
    _call('dpipe_mod_fwd', P(temb), P(W), P(bias), P(out.view), B, N, K)
    torch.cuda.synchronize()
    assert out.intact()
    for i in range(0, N, 8192):
        rows = slice(i, min(N, i + 8192))
        R.check(out.view[:, rows], R.mod_fwd_ref(temb, W, bias, rows=rows), f'mod_fwd B={B} N={N} K={K} rows {i}')


@pytest.mark.parametrize('with_bias', [True, False])
@pytest.mark.parametrize('NK', [(18432, 3072), (9216, 3072), (30720, 5120), (1000, 264)])
@pytest.mark.parametrize('B', [1, 2, 3, 4, 5, 8])
def test_mod_fwd(B, NK, with_bias):
    _mod_fwd_case(B, *NK, with_bias)


def test_mod_fwd_at_the_largest_shared_memory_footprint():
    """B * K * 4 bytes of silu(temb) in shared memory: 8 x 6400 is the largest the 200 KB limit admits"""
    g = _gen('mfmax')
    W = (torch.randn(200, 6400, generator=g, device='cuda') * 0.02).bfloat16()
    _mod_fwd_case(8, 200, 6400, True, W=W)
    temb = torch.zeros(8, 6408, device='cuda', dtype=torch.bfloat16)
    L = _lib()
    assert L.lib().dpipe_mod_fwd(P(temb), P(temb), None, P(temb), 8, 1, 6408, None) < 0


def _mod_bwd_run(B, N, K, mode, dmod, temb, W, dW0, dtemb0):
    """one dpipe_mod_bwd call into sentinel buffers; mode in {'none', 'overwrite', 'accumulate'}"""
    dW = None
    if mode != 'none':
        dW = Flat((N, K), torch.bfloat16)
        if mode == 'accumulate':
            dW.view.copy_(dW0)
    dbias = Flat(N, torch.float32)
    dtemb = Flat((B, K), torch.float32)
    dtemb.view.copy_(dtemb0)
    nchunk = _lib().lib().dpipe_mod_bwd_chunks(N)
    partials = torch.empty(nchunk * B * K, device='cuda')
    _call('dpipe_mod_bwd', P(dmod), dmod.stride(0), P(temb), P(W), P(dW.view) if dW else None, int(mode == 'accumulate'),
          P(dbias.view), P(partials), P(dtemb.view), B, N, K)
    torch.cuda.synchronize()
    assert dbias.intact() and dtemb.intact() and (dW is None or dW.intact())
    return dW, dbias, dtemb


@pytest.mark.parametrize('NK', [(18432, 3072), (30720, 5120), (100, 256), (1000, 8192)])
@pytest.mark.parametrize('B', [1, 2, 3, 4, 5, 6, 7, 8])
def test_mod_bwd(B, NK):
    """every sample count (kernel variants <2>, <4>, <8>) at the Flux / Qwen (3072) and Wan-14B (5120) widths, a one-block
    width and the largest accepted width; dW absent, overwritten and accumulated onto non-zero values; dmod with a row
    stride above N; dtemb accumulated onto non-zero values"""
    N, K = NK
    W, _ = _weight(N, K)
    g = _gen('mb', B, N, K)
    dmod_buf = _rows(B, N + 40, g, -3, 1)
    dmod = dmod_buf[:, 8:8 + N]
    temb = _temb(B, K, g)
    dW0 = (torch.randn(N, K, generator=g, device='cuda') * 0.1).bfloat16()
    dtemb0 = torch.randn(B, K, generator=g, device='cuda')
    for mode in ('none', 'overwrite', 'accumulate'):
        ref = R.mod_bwd_ref(dmod, temb, W, dW0 if mode == 'accumulate' else None, dtemb0)
        dW, dbias, dtemb = _mod_bwd_run(B, N, K, mode, dmod, temb, W, dW0, dtemb0)
        what = f'mod_bwd B={B} N={N} K={K} dW {mode}'
        R.check(dbias.view, ref['dbias'], what + ' dbias')
        R.check(dtemb.view, ref['dtemb'], what + ' dtemb')
        if dW is not None:
            for i in range(0, N, 4096):
                rows = slice(i, min(N, i + 4096))
                R.check(dW.view[rows], ref['dW'](rows), f'{what} dW rows {i}')
        del dW


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm + modulation, gated residual, column sums
# ---------------------------------------------------------------------------------------------------------------
def _ln_inputs(B, L, D, g):
    """x rows of spread magnitude, a third of them with |mean| 30-100x their spread; scale / shift / gate as slices of a
    [B, 6D] modulation tensor that differs per sample"""
    x = _rows(B * L, D, g)
    far = torch.rand(B * L, 1, generator=g, device='cuda') < 0.33
    x = torch.where(far, x + x.std(-1, keepdim=True) * (30 + 70 * torch.rand(B * L, 1, generator=g, device='cuda')), x)
    mod = (_rows(B, 6 * D, g, -1.5, 0) + torch.randn(B, 1, generator=g, device='cuda') * 0.3).bfloat16()
    return x.bfloat16(), mod


def _ln_fwd_run(x, scale, shift, B, L, D, flags):
    out = Canvas(B * L, D, torch.bfloat16)
    mean, rstd = Flat(B * L, torch.float32), Flat(B * L, torch.float32)
    _call('dpipe_ln_modulate_fwd_ex', P(x), x.stride(0), P(scale), P(shift), scale.stride(0), P(out.view), out.view.stride(0),
          P(mean.view), P(rstd.view), B, L, D, ctypes.c_float(1e-6), flags)
    torch.cuda.synchronize()
    assert out.intact() and mean.intact() and rstd.intact()
    return out.view, mean.view, rstd.view


def _ln_bwd_run(dxn, x, scale, mean, rstd, dres, B, L, D, flags):
    dx = Canvas(B * L, D, torch.bfloat16)
    nchunk = (L + R.ROW_CHUNK - 1) // R.ROW_CHUNK
    partials = torch.empty(B, nchunk, 2, D, device='cuda')
    _call('dpipe_ln_modulate_bwd_ex', P(dxn), dxn.stride(0), P(x), x.stride(0), P(scale), scale.stride(0), P(mean), P(rstd),
          P(dres), dres.stride(0) if dres is not None else 0, P(dx.view), dx.view.stride(0), P(partials), B, L, D, flags)
    ps = [Canvas(B, D, torch.float32) for _ in range(2)]
    sm = [Flat(D, torch.float32) for _ in range(2)]
    _call('dpipe_colreduce_finish', P(partials), B, nchunk, 2, D, P(ps[0].view), ps[0].view.stride(0), P(ps[1].view),
          ps[1].view.stride(0), P(sm[0].view), P(sm[1].view))
    torch.cuda.synchronize()
    assert dx.intact() and all(c.intact() for c in ps + sm)
    return dx.view, ps[0].view, ps[1].view, sm[0].view, sm[1].view


def _ln_case(B, L, D, flags, fwd=True, bwd=True):
    g = _gen('ln', B, L, D, flags)
    x, mod = _ln_inputs(B, L, D, g)
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    what = f'ln B={B} L={L} D={D} flags={flags}'
    if fwd:
        out, mean, rstd = _ln_fwd_run(x, scale, shift, B, L, D, flags)
        ref = R.ln_modulate_fwd_ref(x, scale, shift, B, L, flags=flags)
        R.check(mean, ref['mean'], what + ' mean')
        R.check(rstd, ref['rstd'], what + ' rstd')
        R.check(out, ref['out'], what + ' out')
    else:   # widths the forward does not take: statistics from fp64
        xd = x.double()
        mean = xd.mean(-1).float()
        rstd = torch.rsqrt(((xd - mean.double()[:, None]) ** 2).mean(-1) + 1e-6).float()
    if bwd:
        dxn = _rows(B * L, D, g).bfloat16()
        for dres in (None, _rows(B * L, D, g).bfloat16()):
            dx, dsc, dsh, dsc_sum, dsh_sum = _ln_bwd_run(dxn, x, scale, mean, rstd, dres, B, L, D, flags)
            ref = R.ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, B, L, dres=dres, flags=flags)
            w = what + (' dres' if dres is not None else '')
            R.check(dx, ref['dx'], w + ' dx')
            R.check(dsc, ref['dscale'], w + ' dscale')
            R.check(dsh, ref['dshift'], w + ' dshift')
            R.check(dsc_sum, ref['dscale_sum'], w + ' dscale summed')
            R.check(dsh_sum, ref['dshift_sum'], w + ' dshift summed')


FLAG_SETS = [0, R.LN_MULT_DIRECT, R.LN_ROUND_STEPS, R.LN_MULT_DIRECT | R.LN_ROUND_STEPS]


@pytest.mark.parametrize('flags', FLAG_SETS)
@pytest.mark.parametrize('D', [256, 3072, 4096, 5120, 6144, 8192])
def test_ln_modulate(D, flags):
    """the four flag combinations at every backward launch variant (<2,384,2> D <= 3072, <2,512,1> <= 4096,
    <2,640,1> <= 5120, <2,1024,1> above); batch 1 / 3 / 8 and row counts that end mid row-group and mid chunk"""
    for B in (1, 3, 8):
        for L in (1, 5, 17, 333):
            if B * L * D > 8 * 333 * 3072:
                continue
            _ln_case(B, L, D, flags, fwd=D <= 6144)


@pytest.mark.parametrize('BLD', [(1, 4608, 3072), (2, 2048, 5120)])
def test_ln_modulate_real_shapes(BLD):
    _ln_case(*BLD, 0)


def _gate_case(B, L, D):
    g = _gen('gate', B, L, D)
    dxo, y = _rows(B * L, D, g).bfloat16(), _rows(B * L, D, g).bfloat16()
    mod = (_rows(B, 6 * D, g, -1.5, 0)).bfloat16()
    gate = mod[:, 2 * D:3 * D]
    dy = Canvas(B * L, D, torch.bfloat16)
    nchunk = (L + R.ROW_CHUNK - 1) // R.ROW_CHUNK
    partials = torch.empty(B, nchunk, 2, D, device='cuda')
    _call('dpipe_gate_bwd', P(dxo), dxo.stride(0), P(y), y.stride(0), P(gate), gate.stride(0), P(dy.view), dy.view.stride(0),
          P(partials), B, L, D)
    dg, db = Canvas(B, D, torch.float32), Flat(D, torch.float32)
    _call('dpipe_colreduce_finish', P(partials), B, nchunk, 2, D, P(dg.view), dg.view.stride(0), None, 0, None, P(db.view))
    torch.cuda.synchronize()
    assert dy.intact() and dg.intact() and db.intact()
    ref = R.gate_bwd_ref(dxo, y, gate, B, L)
    what = f'gate_bwd B={B} L={L} D={D}'
    assert torch.equal(dy.view.double(), ref['dy']), what + ' dy'   # one rounding of an exact fp32 product
    R.check(dg.view, ref['dgate'], what + ' dgate')
    R.check(db.view, ref['dbias'], what + ' dbias')


@pytest.mark.parametrize('D', [256, 3072, 4096, 5120, 6144, 8192])
def test_gate_bwd(D):
    for B in (1, 3, 8):
        for L in (1, 5, 17, 333):
            if B * L * D <= 8 * 333 * 3072:
                _gate_case(B, L, D)
    if D == 3072:
        _gate_case(1, 4608, 3072)
    if D == 5120:
        _gate_case(2, 2048, 5120)


@pytest.mark.parametrize('N', [8, 24, 1032, 21504, 30720])
@pytest.mark.parametrize('rows', [1, 63, 64, 65, 4608])
def test_colsum(rows, N):
    g = _gen('cs', rows, N)
    xb = torch.empty(rows, N + 16, device='cuda', dtype=torch.bfloat16)
    xb.copy_(_rows(rows, N + 16, g))
    x = xb[:, 8:8 + N]
    out = Flat(N, torch.float32)
    nchunk = _lib().lib().dpipe_colsum_chunks(rows)
    partials = torch.empty(nchunk * N, device='cuda')
    _call('dpipe_colsum', P(x), x.stride(0), rows, N, P(partials), P(out.view))
    torch.cuda.synchronize()
    assert out.intact()
    R.check(out.view, R.colsum_ref(x), f'colsum rows={rows} N={N}')


# ---------------------------------------------------------------------------------------------------------------
# q / k RMSNorm + RoPE backward
# ---------------------------------------------------------------------------------------------------------------
def _rope_tables(Ltot, g):
    ang = torch.rand(Ltot, 64, generator=g, device='cuda') * 6.28
    return torch.cos(ang).repeat_interleave(2, 1).contiguous(), torch.sin(ang).repeat_interleave(2, 1).contiguous()


@pytest.mark.parametrize('rows', [1, 33, 4096])
@pytest.mark.parametrize('off', [0, 512])
@pytest.mark.parametrize('H', [2, 24])
@pytest.mark.parametrize('B', [1, 3])
def test_qknorm_rope_bwd(B, H, off, rows, ops):
    g = _gen('qk', B, H, off, rows)
    Ltot = off + rows + 7
    shp = (B, H, Ltot, 128)
    dq, dk, dv = (_rows(B * H * Ltot, 128, g).view(shp).bfloat16() for _ in range(3))
    qh, kh = (torch.randn(shp, generator=g, device='cuda').bfloat16() for _ in range(2))
    qr, kr = (torch.rand(B, H, Ltot, generator=g, device='cuda') * 3 + 0.1 for _ in range(2))
    wq, wk = ((1 + 0.2 * torch.randn(128, generator=g, device='cuda')).bfloat16() for _ in range(2))
    cos, sin = _rope_tables(Ltot, g)
    N = 3 * H * 128
    dqkv = Canvas(B * rows, N, torch.bfloat16)
    dbias0, dw0 = torch.randn(N, generator=g, device='cuda'), torch.randn(2, 128, generator=g, device='cuda')
    dbias, dw = Flat(N, torch.float32), Flat((2, 128), torch.float32)
    dbias.view.copy_(dbias0)
    dw.view.copy_(dw0)
    ops.qknorm_rope_bwd(dq, dk, dv, qh, kh, qr, kr, wq, wk, cos, sin, dqkv.view, dbias.view, dw.view, B, H, Ltot, off, rows)
    torch.cuda.synchronize()
    assert dqkv.intact() and dbias.intact() and dw.intact()
    what = f'qknorm_rope_bwd B={B} H={H} off={off} rows={rows}'
    for b in range(B):   # one sample's reference at a time keeps the fp64 copies within a few GB
        ref = R.qknorm_rope_bwd_ref(dq, dk, dv, qh, kh, qr, kr, wq, wk, cos, sin, B, H, off, rows, samples=[b])
        R.check(dqkv.view[b * rows:(b + 1) * rows], ref['dqkv'], f'{what} dqkv sample {b}')
    v = dqkv.view[:, 2 * H * 128:].reshape(B, rows, H, 128).permute(0, 2, 1, 3)
    assert torch.equal(v, dv[:, :, off:off + rows]), what + ' v'
    R.check(dbias.view, R.summed_rows_ref(dqkv.view, dbias0), what + ' dbias')   # float atomics: the bound only
    R.check(dw.view, R.add(R.exact(dw0), ref['dw']), what + ' dw')


# ---------------------------------------------------------------------------------------------------------------
# Wan full-width RMSNorm + RoPE
# ---------------------------------------------------------------------------------------------------------------
MIXES = {'self': ((True, True), (True, True), (False, False)), 'cross_q': ((True, False),), 'rope_v': ((True, True), (False, True))}


def _wan_case(B, L, H, mix, ops):
    g = _gen('wan', B, L, H, mix)
    Cw = H * 128
    projs = MIXES[mix]
    fused = _rows(B * L, 3 * Cw + 64, g).bfloat16()   # [rows, 3C] projection output, plus columns past the last slice
    cos, sin = _rope_tables(L, g)
    weights = [(1 + 0.2 * torch.randn(Cw, generator=g, device='cuda')).bfloat16() if w else None for w, _ in projs]
    srcs = [fused[:, i * Cw:(i + 1) * Cw] for i in range(len(projs))]
    fwd = ops.wan_norm_rope_fwd([{'src': s, 'weight': w, 'rope': r} for s, w, (_, r) in zip(srcs, weights, projs)],
                                B, L, H, cos, sin)
    dys = [_rows(B * H * L, 128, g).view(B, H, L, 128).bfloat16() for _ in projs]
    dxs = [Canvas(B * L, Cw, torch.bfloat16) for _ in projs]
    bwd = ops.wan_norm_rope_bwd([{'dy': dy, 'dx': dx.view, 'weight': w, 'xhat': f[1], 'rstd': f[2], 'rope': r}
                                 for dy, dx, w, f, (_, r) in zip(dys, dxs, weights, fwd, projs)], B, L, H, cos, sin)
    torch.cuda.synchronize()
    assert all(d.intact() for d in dxs)
    for i, ((w, r), (dst, xhat, rstd)) in enumerate(zip(projs, fwd)):
        what = f'wan_norm_rope B={B} L={L} H={H} {mix} projection {i}'
        if not w and not r:
            assert torch.equal(dst, srcs[i].reshape(B, L, H, 128).permute(0, 2, 1, 3)), what + ' v copy'
            assert torch.equal(dxs[i].view, dys[i].permute(0, 2, 1, 3).reshape(B * L, Cw)), what + ' dv copy'
            continue
        dw = None
        for b in range(B):   # one sample's reference at a time keeps the fp64 copies within a few GB
            rows = slice(b * L, (b + 1) * L)
            ref = R.wan_norm_rope_fwd_ref(srcs[i][rows], weights[i], r, cos, sin, 1, L, H)
            R.check(dst[b:b + 1], ref['dst'], f'{what} sample {b} dst')
            if w:
                R.check(xhat[rows], ref['xhat'], f'{what} sample {b} xhat')
                R.check(rstd[rows], ref['rstd'], f'{what} sample {b} rstd')
            del ref
            bref = R.wan_norm_rope_bwd_ref(dys[i][b:b + 1], xhat[rows] if w else None, rstd[rows] if w else None, weights[i],
                                           r, cos, sin, 1, L, H, total_rows=B * L)
            R.check(dxs[i].view[rows], bref['dx'], f'{what} sample {b} dx')
            if w:   # the d weight bounds of the parts add up to the whole's
                dw = bref['dw'] if dw is None else R.E(dw.v + bref['dw'].v, dw.e + bref['dw'].e)
            del bref
        if w:
            R.check(bwd[i], dw, what + ' dw')


@pytest.mark.parametrize('mix', sorted(MIXES))
@pytest.mark.parametrize('L', [1, 17, 1560])
@pytest.mark.parametrize('H', [2, 12, 40, 56])
@pytest.mark.parametrize('B', [1, 3])
def test_wan_norm_rope(B, H, L, mix, ops):
    _wan_case(B, L, H, mix, ops)


# ---------------------------------------------------------------------------------------------------------------
# masked MSE
# ---------------------------------------------------------------------------------------------------------------
MSE_SHAPES = {1: (1, 1, 1, 1), 2047: (1, 23, 1, 89), 2049: (1, 3, 1, 683), 2048 * 1024 + 1: (1, 3, 1, 699051)}


@pytest.mark.parametrize('mask', ['none', 'fractional', 'broadcast'])
@pytest.mark.parametrize('numel', sorted(MSE_SHAPES))
def test_mse_loss(numel, mask):
    """past 2048 * 1024 elements the 1024 CTAs walk the tensor grid-stride"""
    shp = MSE_SHAPES[numel]
    g = _gen('mse', numel, mask)
    out = torch.randn(shp, generator=g, device='cuda').bfloat16()
    tgt = torch.randn(shp, generator=g, device='cuda')
    m = None
    if mask == 'fractional':
        m = torch.rand(shp, generator=g, device='cuda')
    elif mask == 'broadcast':
        m = torch.rand(shp[0], 1, shp[2], shp[3], generator=g, device='cuda')
    mfull = m.expand_as(tgt).contiguous() if m is not None else None
    loss = Flat(1, torch.float32)
    dout = Flat(shp, torch.bfloat16)
    ws = torch.empty(1024, device='cuda')
    _call('dpipe_mse_loss', P(out), P(tgt), P(mfull), numel, P(ws), P(loss.view), P(dout.view))
    torch.cuda.synchronize()
    assert loss.intact() and dout.intact()
    ref = R.mse_loss_ref(out, tgt, m)
    R.check(loss.view[0], ref['loss'], f'mse numel={numel} mask={mask} loss')
    R.check(dout.view, ref['dout'], f'mse numel={numel} mask={mask} dout')


# ---------------------------------------------------------------------------------------------------------------
# launch envelope: the largest width each host check accepts launches, computes right, and one step wider is refused
# ---------------------------------------------------------------------------------------------------------------
def test_largest_accepted_widths_launch_and_compute(ops):
    """CTA sizes follow the width in ln_modulate_* (D / 8 threads), gate_bwd (D / 8) and wan_norm_rope_* (16 H); the
    modulation backward's do not.  gate_bwd at D = 8192 is 1024 threads at 64 registers: the whole register file."""
    L = _lib().lib()
    for B in range(1, 9):
        g = _gen('env', B)
        N, K = 64, 8192
        W = (torch.randn(N, K, generator=g, device='cuda') * 0.02).bfloat16()
        dmod, temb = _rows(B, N, g), _temb(B, K, g)
        dW0, dtemb0 = torch.zeros(N, K, device='cuda', dtype=torch.bfloat16), torch.zeros(B, K, device='cuda')
        ref = R.mod_bwd_ref(dmod, temb, W, None, dtemb0)
        dW, dbias, dtemb = _mod_bwd_run(B, N, K, 'overwrite', dmod, temb, W, dW0, dtemb0)
        R.check(dW.view, ref['dW'](), f'mod_bwd B={B} K={K} dW')
        R.check(dtemb.view, ref['dtemb'], f'mod_bwd B={B} K={K} dtemb')
        buf = ctypes.c_void_p(dW.view.data_ptr())
        assert L.dpipe_mod_bwd(buf, 0, buf, buf, buf, 0, buf, buf, buf, B, N, K + 256, None) < 0
    _ln_case(2, 17, 6144, 0, fwd=True, bwd=False)
    _ln_case(2, 17, 8192, 0, fwd=False, bwd=True)
    _gate_case(2, 17, 8192)
    x = torch.zeros(1, 8448, device='cuda', dtype=torch.bfloat16)
    assert L.dpipe_ln_modulate_fwd_ex(P(x), 8448, P(x), P(x), 0, P(x), 8448, None, None, 1, 1, 6400, ctypes.c_float(1e-6), 0, None) < 0
    assert L.dpipe_gate_bwd(P(x), 8448, P(x), 8448, P(x), 0, P(x), 8448, P(x), 1, 1, 8448, None) < 0
    _wan_case(2, 17, 56, 'self', ops)
    with pytest.raises(Exception, match='geometry'):
        ops.wan_norm_rope_fwd([{'src': torch.zeros(2, 57 * 128, device='cuda', dtype=torch.bfloat16)}], 1, 2, 57)
