"""fp64 references of the HBM-bound kernels around the GEMMs of a block (csrc/modulation.cu, csrc/elementwise.cu,
csrc/wan_norm.cu), each with a per-element error bound, and the check that applies that bound to every element.

A reference is evaluated in float64 from the kernel's exact bf16 / fp32 inputs.  Every quantity is an `E`: its fp64
value and a bound on how far the kernel's fp32 value of it can lie from that value.  The bound is built from three terms:

* fp32 arithmetic: an accumulation of n terms adds C * n * 2^-24 * sum|terms|, where n is the longest fp32 chain that
  feeds the element in the kernel's summation order; an elementwise op adds C * 2^-24 * |result|.  C (below) is one
  headroom factor, the same for every kernel: it covers __expf (2 + 1.2|x| ulp), rsqrtf (2 ulp) and the choice between
  a fused and an unfused multiply-add.
* rounding flips: at each bf16 rounding point the kernel documents, the reference rounds its fp64 value.  Where that
  value lies within its bound of a bf16 rounding boundary the kernel may land on the other neighbour, so the bound there
  becomes one bf16 ulp (plus the incoming bound); it is carried to the output through the gains of the later ops.
  Everywhere else the kernel's rounded value is the reference's, exactly, and the bound collapses to zero.
* final rounding: a bf16 output is compared with the unrounded final value, plus half a bf16 ulp.

Each reference takes `off`, a set of rounding-point names to skip (or 'all'): with every point off it is the plain
operation, which the CPU tests compare with torch autograd; switching one point off is one of the mutations the check
must reject.  Nothing here needs a GPU: the references run on whatever device their inputs are on.
"""
import math

import torch

U = 2.0 ** -24   # fp32 unit roundoff
C = 4.0          # headroom on every fp32 error term (see the module docstring)

ROW_CHUNK = 16   # csrc/elementwise.cu ROW_CHUNK: rows per CTA in the two-stage column reductions
MOD_ROWS = 64    # csrc/modulation.cu MOD_ROWS: weight rows per CTA in the modulation backward
COLSUM_ROWS = 64
WN_ROWS = 16     # csrc/wan_norm.cu WN_ROWS


class E:
    """fp64 value `v` and a bound `e` on |kernel - v| (same shape)"""
    __slots__ = ('v', 'e')

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    def __getitem__(self, i):
        return E(self.v[i], self.e[i])


def exact(t):
    return E(t.double())


def _on(name, off):
    return not (off == 'all' or name in off)


def bf(v):
    """round an fp64 tensor to bf16 as the kernel rounds its fp32 value (round to nearest even), back in fp64"""
    return v.float().bfloat16().double()


def ulp(a):
    """bf16 ulp of |a| (8 significant bits), floored at the smallest normal"""
    _, ex = torch.frexp(a.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(a), (ex - 8).to(torch.int32)).to(a.dtype)


def rnd(x, name, off):
    """a bf16 rounding point of the kernel"""
    if not _on(name, off):
        return x
    a = x.v.abs()
    u = ulp(a + x.e)
    dist = ((a / u - torch.floor(a / u)) - 0.5).abs() * u
    return E(bf(x.v), torch.where(dist <= x.e, u + x.e, torch.zeros_like(x.e)))


def add(a, b):
    v = a.v + b.v
    return E(v, a.e + b.e + C * U * v.abs())


def sub(a, b):
    v = a.v - b.v
    return E(v, a.e + b.e + C * U * v.abs())


def mul(a, b):
    v = a.v * b.v
    return E(v, a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e + C * U * v.abs())


def ssum(x, dim, n, keepdim=False):
    """fp32 sum of x over `dim` along a chain of at most n additions"""
    return E(x.v.sum(dim, keepdim=keepdim), x.e.sum(dim, keepdim=keepdim) + C * n * U * x.v.abs().sum(dim, keepdim=keepdim))


def rsqrt(x):
    r = torch.rsqrt(x.v)
    return E(r, 0.5 * r * x.e / x.v + 2 * C * U * r)


def silu(t, off):
    """fp32 silu with __expf of an exact input; `off` drops the transcendental error for the autograd comparison"""
    v = t * torch.sigmoid(t)
    return E(v, (C * (4 + 1.2 * t.abs()) * U * v.abs()) if _on('silu', off) else torch.zeros_like(v))


def silu_grad(t):
    s = torch.sigmoid(t)
    v = s * (1 + t * (1 - s))
    return E(v, C * (6 + 1.2 * t.abs()) * U * s * (1 + t.abs()))


def _block_chain(width):
    """block_sum over a row of `width` columns, one thread per 8: 8 serial adds, a 5-level shuffle tree, one add per warp"""
    return 8 + 5 + width // 256


def _finish_chain(nchunk):
    """colreduce_finish / mod_bwd_finish: 8 threads each fold every 8th chunk, then the 8 partials are added"""
    return (nchunk + 7) // 8 + 8


# ---------------------------------------------------------------------------------------------------------------
# check
# ---------------------------------------------------------------------------------------------------------------
def violations(out, ref, bf16_out):
    """per-element (error, allowed) of a kernel output against a reference E"""
    got = out.double()
    v, e = ref.v.to(got.device), ref.e.to(got.device)
    allowed = e + (0.5 * ulp(v.abs() + e) if bf16_out else U * v.abs())
    err = (got - v).abs()
    err = torch.where(torch.isfinite(got), err, torch.full_like(err, math.inf))
    return err, allowed


def check(out, ref, what='', bf16_out=None):
    """assert every element of `out` within the bound of `ref` (bf16 outputs: plus half an ulp of the exact value)"""
    if bf16_out is None:
        bf16_out = out.dtype == torch.bfloat16
    assert out.shape == ref.v.shape, (what, tuple(out.shape), tuple(ref.v.shape))
    err, allowed = violations(out, ref, bf16_out)
    bad = err > allowed
    if bad.any():
        n = int(bad.sum())
        i = int(torch.argmax((err - allowed).flatten()))
        idx = tuple(int(k) for k in torch.unravel_index(torch.tensor(i), out.shape))
        raise AssertionError(f'{what}: {n} of {out.numel()} elements outside the bound; worst at {idx}: got '
                             f'{out.double()[idx].item()!r} want {ref.v[idx].item()!r} bound {allowed[idx].item():.3e}')


def accepts(out, ref, bf16_out=None):
    try:
        check(out, ref, bf16_out=bf16_out)
        return True
    except AssertionError:
        return False


# ---------------------------------------------------------------------------------------------------------------
# modulation linears (csrc/modulation.cu)
# ---------------------------------------------------------------------------------------------------------------
def _silu_rows(temb, off):
    return rnd(silu(temb.double(), off), 'silu', off)


def mod_fwd_ref(temb, W, bias, off=(), rows=None):
    """out[b, n] = sum_k W[n, k] bf16(silu(temb[b, k])) + bias[n]; one warp per row: K/32 serial fmas per lane, a
    5-level shuffle tree, the bias.  rows: a slice of n (the reference of a 30720-row W is built in pieces)"""
    rows = rows or slice(0, W.shape[0])
    K = temb.shape[1]
    s = _silu_rows(temb, off)
    Wd = W[rows].double()
    v = s.v @ Wd.t()
    a = s.v.abs() @ Wd.abs().t()
    e = s.e @ Wd.abs().t()
    if bias is not None:
        b = bias[rows].double()
        v, a = v + b, a + b.abs()
    return E(v, e + C * (K // 32 + 6) * U * a)


def mod_bwd_ref(dmod, temb, W, dW0, dtemb0, off=()):
    """backward of mod_fwd, as dpipe_mod_bwd forms it.  Returns dict: dbias [N], dtemb [B, K], and dW(rows) -> E for
    a slice of rows (dW0 = None: dW overwritten; else accumulated onto dW0)"""
    B, K = temb.shape
    N = W.shape[0]
    t = temb.double()
    dm = exact(dmod)
    if _on('dmod', off):
        dm = E(bf(dm.v))
    s = _silu_rows(temb, off)
    out = {'dbias': ssum(dm, 0, B)}
    nchunk = (N + MOD_ROWS - 1) // MOD_ROWS
    pv, pa = torch.zeros_like(t), torch.zeros_like(t)
    for i in range(0, N, 4096):   # W in fp64 a slice at a time
        Wc = W[i:i + 4096].double()
        pv += dm.v[:, i:i + 4096] @ Wc
        pa += dm.v[:, i:i + 4096].abs() @ Wc.abs()
    P = E(pv, C * (MOD_ROWS + _finish_chain(nchunk)) * U * pa)
    p = rnd(P, 'partials', off)
    g = silu_grad(t) if _on('silu', off) else E(silu_grad(t).v)
    old = exact(dtemb0)
    out['dtemb'] = add(old, mul(p, g))

    def dW(rows=slice(0, N)):
        d = dm.v[:, rows].t()
        v = d @ s.v
        e = d.abs() @ s.e
        a = d.abs() @ s.v.abs()
        if dW0 is not None:
            o = dW0[rows].double()
            v, a = v + o, a + o.abs()
        return E(v, e + C * (B + 1) * U * a)
    out['dW'] = dW
    return out


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm + modulation, gated residual, column sums (csrc/elementwise.cu)
# ---------------------------------------------------------------------------------------------------------------
LN_MULT_DIRECT = 1
LN_ROUND_STEPS = 2


def _multiplier(scale, flags, off):
    sc = exact(scale)
    if flags & LN_MULT_DIRECT:
        return sc
    one = E(1 + sc.v, U * (1 + sc.v).abs())   # fp32 1 + bf16: exact unless |scale| < 2^-16
    return rnd(one, 'one_plus_scale', off)


def ln_modulate_fwd_ref(x, scale, shift, batch, rows_per_batch, eps=1e-6, flags=0, off=()):
    """out = LN(x) * m + shift (m = bf16(1 + scale) or scale itself with LN_MULT_DIRECT); with LN_ROUND_STEPS
    out = bf16(bf16(LN(x)) * m) + shift.  x [batch * rows, D]; scale / shift [batch, D].  Returns dict out [rows, D]
    (unrounded), mean / rstd [rows]."""
    D = x.shape[1]
    X = x.double().view(batch, rows_per_batch, D)
    n = _block_chain(D)
    s = X.sum(-1)
    m = s / D
    dm = C * n * U * X.abs().sum(-1) / D + C * U * m.abs()
    d = X - m[..., None]
    var = (d * d).sum(-1)
    dvar = C * (n + 2) * U * var + 3 * D * dm * dm
    rstd = rsqrt(E(var / D + eps, dvar / D + C * U * (var / D + eps)))
    xn = mul(E(d, dm[..., None] + C * U * d.abs()), E(rstd.v[..., None], rstd.e[..., None]))
    sc = _multiplier(scale, flags, off)
    sc = E(sc.v[:, None], sc.e[:, None])
    sh = exact(shift)[:, None]
    if flags & LN_ROUND_STEPS:
        o = add(rnd(mul(rnd(xn, 'steps', off), sc), 'steps', off), sh)
    else:
        o = add(mul(xn, sc), sh)
    return {'out': E(o.v.reshape(-1, D), o.e.reshape(-1, D)), 'mean': E(m.reshape(-1), dm.reshape(-1)),
            'rstd': E(rstd.v.reshape(-1), rstd.e.reshape(-1))}


def ln_modulate_bwd_ref(dxn, x, scale, mean, rstd, batch, rows_per_batch, dres=None, flags=0, off=(), drop_row=None):
    """dx = rstd (g - mean(g) - xhat mean(g xhat)) (+ dres) with g = dxn * m; per-sample column sums dscale =
    sum_rows dxn xhat, dshift = sum_rows dxn, and their sums over samples.  mean / rstd are the kernel's fp32 inputs.
    drop_row: a row index within each ROW_CHUNK chunk to leave out of the column sums (a mutation for the tests)."""
    D = x.shape[1]
    X = x.double().view(batch, rows_per_batch, D)
    dv = dxn.double().view(batch, rows_per_batch, D)
    mu = mean.double().view(batch, rows_per_batch, 1)
    rs = rstd.double().view(batch, rows_per_batch, 1)
    xh = E((X - mu) * rs, 2 * C * U * ((X - mu) * rs).abs())
    sc = _multiplier(scale, flags, off)
    g = E(dv * sc.v[:, None], dv.abs() * sc.e[:, None])   # bf16 x bf16 is exact in fp32
    n = _block_chain(D)
    m1 = ssum(g, -1, n, keepdim=True)
    m1 = E(m1.v / D, m1.e / D)
    m2 = ssum(mul(g, xh), -1, n + 1, keepdim=True)
    m2 = E(m2.v / D, m2.e / D)
    inner = sub(sub(g, m1), mul(xh, m2))
    o = mul(E(rs), inner)
    if dres is not None:
        o = add(o, E(dres.double().view(batch, rows_per_batch, D)))
    nchunk = (rows_per_batch + ROW_CHUNK - 1) // ROW_CHUNK
    keep = torch.ones(rows_per_batch, dtype=torch.float64, device=X.device)
    if drop_row is not None:
        keep[drop_row::ROW_CHUNK] = 0
    keep = keep[None, :, None]
    nr = ROW_CHUNK + _finish_chain(nchunk)
    t_scale = E(dv * xh.v * keep, dv.abs() * xh.e * keep)
    t_shift = E(dv * keep)
    dscale, dshift = ssum(t_scale, 1, nr), ssum(t_shift, 1, nr)
    return {'dx': E(o.v.reshape(-1, D), o.e.reshape(-1, D)), 'dscale': dscale, 'dshift': dshift,
            'dscale_sum': ssum(dscale, 0, batch), 'dshift_sum': ssum(dshift, 0, batch)}


def gate_bwd_ref(dxo, y, gate, batch, rows_per_batch):
    """dy = bf16(gate[b] dx) (one rounding of an exact fp32 product), dgate[b] = sum_rows dx y, dbias = sum dy"""
    D = y.shape[1]
    dv = dxo.double().view(batch, rows_per_batch, D)
    dy = bf(gate.double()[:, None] * dv)
    nchunk = (rows_per_batch + ROW_CHUNK - 1) // ROW_CHUNK
    nr = ROW_CHUNK + _finish_chain(nchunk)
    dgate = ssum(E(dv * y.double().view(batch, rows_per_batch, D)), 1, nr)
    dbias = ssum(ssum(E(dy), 1, nr), 0, batch)
    return {'dy': dy.reshape(-1, D), 'dgate': dgate, 'dbias': dbias}


def colsum_ref(x):
    """fp32 column sums of a bf16 [rows, N] matrix (built 1024 rows at a time: fp64 copies of a 4608 x 30720 matrix
    would not fit a few GB)"""
    rows = x.shape[0]
    nchunk = (rows + COLSUM_ROWS - 1) // COLSUM_ROWS
    v = torch.zeros(x.shape[1], dtype=torch.float64, device=x.device)
    a = torch.zeros_like(v)
    for i in range(0, rows, 1024):
        xi = x[i:i + 1024].double()
        v += xi.sum(0)
        a += xi.abs().sum(0)
    return E(v, C * (COLSUM_ROWS + _finish_chain(nchunk)) * U * a)


# ---------------------------------------------------------------------------------------------------------------
# rope helpers (interleaved pairs, every frequency repeated twice in the [L, 128] fp32 tables)
# ---------------------------------------------------------------------------------------------------------------
def rope_fwd(y, c, s):
    """out[2i] = y[2i] c[2i] - y[2i+1] s[2i];  out[2i+1] = y[2i+1] c[2i+1] + y[2i] s[2i+1]"""
    ye, yo = y.v[..., 0::2], y.v[..., 1::2]
    ee, eo = y.e[..., 0::2], y.e[..., 1::2]
    ce, co, se, so = c[..., 0::2], c[..., 1::2], s[..., 0::2], s[..., 1::2]
    ve = ye * ce - yo * se
    vo = yo * co + ye * so
    err_e = ee * ce.abs() + eo * se.abs() + 2 * C * U * ((ye * ce).abs() + (yo * se).abs())
    err_o = eo * co.abs() + ee * so.abs() + 2 * C * U * ((yo * co).abs() + (ye * so).abs())
    return E(torch.stack([ve, vo], -1).flatten(-2), torch.stack([err_e, err_o], -1).flatten(-2))


def rope_bwd(g, c, s, sign=1.0):
    """transpose of rope_fwd:  dy[2i] = g[2i] c[2i] + g[2i+1] s[2i+1];  dy[2i+1] = g[2i+1] c[2i+1] - g[2i] s[2i]
    (sign = -1 flips the sign of the g[2i+1] s[2i+1] term: a mutation for the tests)"""
    ge, go = g[..., 0::2], g[..., 1::2]
    ce, co, se, so = c[..., 0::2], c[..., 1::2], s[..., 0::2], s[..., 1::2]
    ve = ge * ce + sign * go * so
    vo = go * co - ge * se
    err_e = 2 * C * U * ((ge * ce).abs() + (go * so).abs())
    err_o = 2 * C * U * ((go * co).abs() + (ge * se).abs())
    return E(torch.stack([ve, vo], -1).flatten(-2), torch.stack([err_e, err_o], -1).flatten(-2))


# ---------------------------------------------------------------------------------------------------------------
# q / k RMSNorm + RoPE backward of the QKV epilogue (csrc/elementwise.cu qknorm_rope_bwd)
# ---------------------------------------------------------------------------------------------------------------
def qknorm_rope_bwd_ref(dq, dk, dv, qhat, khat, q_rstd, k_rstd, wq, wk, cos, sin, batch, heads, seq_offset, rows_per_batch,
                        rope_sign=1.0, samples=None):
    """dqkv token-major [len(samples) * rows, 3 H 128] for the given samples (default: all): for q and k
    rstd (dxh - xhat mean(dxh xhat)) with dxh = w * rope^T(g), for v the gradient itself.  Also the fp32 d weight [2, 128],
    always summed over every sample, head and token.  One sample is built at a time."""
    H = heads
    sl = slice(seq_offset, seq_offset + rows_per_batch)
    c, s = cos[sl].double(), sin[sl].double()
    samples = range(batch) if samples is None else samples
    dev = dq.device
    dw_v, dw_e, dw_a = (torch.zeros(2, 128, dtype=torch.float64, device=dev) for _ in range(3))
    pieces = []
    for b in range(batch):
        outs = []
        for i, (g, hat, rstd, w) in enumerate(((dq, qhat, q_rstd, wq), (dk, khat, k_rstd, wk))):
            G = g[b, :, sl].double()
            xh = hat[b, :, sl].double()
            dy = rope_bwd(G, c, s, rope_sign)
            t = dy.v * xh
            dw_v[i] += t.sum((0, 1))
            dw_a[i] += t.abs().sum((0, 1))
            dw_e[i] += (dy.e * xh.abs()).sum((0, 1))
            if b not in samples:
                continue
            rs = rstd[b, :, sl].double()[..., None]
            dxh = mul(dy, E(w.double()))
            dot = ssum(E(dxh.v * xh, dxh.e * xh.abs()), -1, 4 + 5 + 1, keepdim=True)
            d = E(dot.v / 128, dot.e / 128)
            outs.append(mul(E(rs), sub(dxh, mul(E(xh), d))))
        if b in samples:
            outs.append(E(dv[b, :, sl].double()))
            # [3, H, L, 128] -> [L, 3, H, 128] -> [L, 3 H 128]
            pieces.append(E(torch.stack([o.v for o in outs]).permute(2, 0, 1, 3).reshape(rows_per_batch, 3 * H * 128),
                            torch.stack([o.e for o in outs]).permute(2, 0, 1, 3).reshape(rows_per_batch, 3 * H * 128)))
            del outs
    dqkv = E(torch.cat([p.v for p in pieces]), torch.cat([p.e for p in pieces])) if pieces else None
    return {'dqkv': dqkv, 'dw': E(dw_v, dw_e + C * batch * H * rows_per_batch * U * dw_a)}


def summed_rows_ref(dqkv_out, start):
    """d bias of qknorm_rope_bwd: start + the column sums of the bf16 rows the kernel wrote (float atomics in any order:
    a chain of at most rows + 1 additions)"""
    v, a = start.double().clone(), start.double().abs()
    for i in range(0, dqkv_out.shape[0], 1024):
        X = dqkv_out[i:i + 1024].double()
        v += X.sum(0)
        a += X.abs().sum(0)
    return E(v, C * (dqkv_out.shape[0] + 1) * U * a)


# ---------------------------------------------------------------------------------------------------------------
# Wan full-width RMSNorm + RoPE + head-major scatter (csrc/wan_norm.cu)
# ---------------------------------------------------------------------------------------------------------------
def _to_head_major(t, B, L, H):
    return t.view(B, L, H, 128).permute(0, 2, 1, 3)


def wan_norm_rope_fwd_ref(src, weight, rope, cos, sin, B, L, H, eps=1e-6, off=()):
    """dst [B, H, L, 128] = rope(bf16(bf16(x rstd) w)) (weight given) or rope(x); xhat = x rstd, rstd [rows].
    src [B * L, >= C] with C = 128 H.  dst / xhat are returned unrounded."""
    Cw = H * 128
    x = src[:, :Cw].double()
    out = {}
    if weight is not None:
        ss = ssum(E(x * x), -1, _block_chain(Cw) + 1, keepdim=True)
        rstd = rsqrt(E(ss.v / Cw + eps, ss.e / Cw + C * U * (ss.v / Cw + eps)))
        xh = mul(E(x), rstd)
        out['xhat'], out['rstd'] = xh, E(rstd.v[:, 0], rstd.e[:, 0])
        y = rnd(mul(rnd(xh, 'xhat', off), E(weight.double())), 'y', off)
    else:
        y = E(x)
    if rope:
        y = rope_fwd(E(_to_head_major(y.v, B, L, H), _to_head_major(y.e, B, L, H)), cos[:L].double(), sin[:L].double())
    else:
        y = E(_to_head_major(y.v, B, L, H), _to_head_major(y.e, B, L, H))
    out['dst'] = y
    return out


def wan_norm_rope_bwd_ref(dy, xhat, rstd, weight, rope, cos, sin, B, L, H, rope_sign=1.0, total_rows=None):
    """dx [B * L, C] = rstd (dxh - xhat mean(dxh xhat)) with dxh = w rope^T(dy) (weight given) or rope^T(dy) / dy;
    d weight [C] = sum_rows rope^T(dy) xhat.  total_rows: the rows the kernel's d weight sum spans, when this call covers
    a part of them (the sums of the parts' values and bounds are then the whole's)"""
    Cw = H * 128
    g = dy.double()
    if rope:
        g = rope_bwd(g, cos[:L].double(), sin[:L].double(), rope_sign)
    else:
        g = E(g)
    g = E(g.v.permute(0, 2, 1, 3).reshape(B * L, Cw), g.e.permute(0, 2, 1, 3).reshape(B * L, Cw))
    if weight is None:
        return {'dx': g}
    xh = xhat.double()
    dxh = mul(g, E(weight.double()))
    dot = ssum(E(dxh.v * xh, dxh.e * xh.abs()), -1, _block_chain(Cw) + 1, keepdim=True)
    d = E(dot.v / Cw, dot.e / Cw + C * U * (dot.v / Cw).abs())
    o = mul(E(rstd.double()[:, None]), sub(dxh, mul(E(xh), d)))
    nchunk = ((total_rows or B * L) + WN_ROWS - 1) // WN_ROWS
    dw = ssum(E(g.v * xh, g.e * xh.abs()), 0, WN_ROWS + _finish_chain(nchunk) + 1)
    return {'dx': o, 'dw': dw}


# ---------------------------------------------------------------------------------------------------------------
# masked MSE (csrc/elementwise.cu mse_loss)
# ---------------------------------------------------------------------------------------------------------------
def mse_loss_ref(out, target, mask=None):
    """loss = mean((out - target)^2 mask), dout = 2 (out - target) mask / numel (unrounded); the kernel's grid is
    min(ceil(numel / 2048), 1024) CTAs of 256 threads, grid-stride, then one CTA folds the per-CTA sums"""
    numel = out.numel()
    d = out.double().flatten() - target.double().flatten()
    m = mask.double().expand_as(target).flatten() if mask is not None else torch.ones_like(d)
    blocks = min((numel + 2047) // 2048, 1024)
    n = (numel + blocks * 256 - 1) // (blocks * 256) + 13 + (blocks + 255) // 256 + 13
    t = d * d * m
    loss = E(t.sum() / numel, C * (n + 3) * U * t.abs().sum() / numel)
    g = 2 * d * m / numel
    return {'loss': loss, 'dout': E(g.view(out.shape), (4 * C * U * g.abs()).view(out.shape))}
