"""fp64 references of the wgmma GEMM (csrc/gemm_sm90.cu, every epilogue) and of the attention forward and backward
(csrc/attn_fwd_sm90.cu, csrc/attn_bwd_sm90.cu), each with a per-element error bound, built on the `E` values, rounding
points and check of tests/block_kernel_refs.py (see its docstring for the three terms of every bound and for `off`).

Tensor-core accumulation.  A product of two bf16 values is exact in fp32, and wgmma adds one k16 step (16 products) to
the fp32 accumulator at a time.  The bound of a dot product over K is C * n * U * sum_k |a_k b_k| with
n = ceil(K / 16) + 16: one rounding per k16 step, plus 16 for the alignment or truncation of the 16 products inside a
step.  This model comes from published analyses of earlier tensor cores (Volta to Ampere: products aligned to the
largest exponent of the step and truncated, not rounded); it has not been measured on H100, which is why
tests/test_gemm_attn_gpu.py runs an all-positive K = 32768 GEMM, where any truncation bias adds up, and prints the
worst err / bound of every kernel family.

The references follow the kernels' operation order and name every bf16 rounding point:
  GEMM      STORE        (acc + old) + bias, one rounding
            BIAS_GELU    'u' = bf16(acc + bias), then gelu_tanh in fp32 (tanhf)
            GATE_RES     'y' = bf16(acc + bias), 'gy' = bf16(gate y), then res + gy
            MUL_GELU_GRAD acc * gelu_tanh'(aux), no intermediate rounding
            QKV_ROPE     'pre' = bf16(acc + bias) ('pre_ss' where the sum of squares reads it), rstd = rsqrtf(sum / 128 +
                         eps) over a serial chain of 128, 'xhat' = bf16(pre rstd), 'yw' = bf16(xhat w), RoPE; v =
                         bf16(acc + bias) once; columns >= n_qkv take BIAS_GELU into out / out2 at col - n_qkv
  attention forward      S over 128 / 16 k16 steps; p = ex2(fma(S, c, -m_j)) with m_j the running row maximum after key
                         tile j (128 keys), 'P' = bf16(p) relative to that maximum, earlier tiles rescaled by
                         ex2(m_old - m_new); l sums the unrounded p; O = sum bf16(P) V * (1 / l) over a chain of
                         nkv * 9; lse = m + log2f(l) (log2 domain).  'c': the fp32 scale * log2(e) the host passes.
  attention backward     from the kernel's own o and lse: D = sum o dO (4 products per lane, a 5-level shuffle);
                         P = ex2(fma(S, c, -lse)); 'P' = bf16(P) for dV; 'dS' = bf16(P (dP - D)) for dK and dQ, which are
                         multiplied by the fp32 scale before their output rounding.
The FMA-pipe exponential of attn_fwd_kernel<2> / <4> is within POLY_REL (read from csrc/sm90_common.cuh) of exp2 in the
column pairs it serves, and turns a masked key into 2^-125 instead of 0 (its V is the TMA zero fill).
"""
import math
import os
import re

import torch

from block_kernel_refs import C, E, U, add, bf, exact, mul, rnd, rope_fwd, ssum, _on

LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
BK = 64       # csrc/gemm_sm90.cu: K per pipeline stage
TK = 128      # csrc/attn_fwd_sm90.cu: keys per tile
BC = 64       # csrc/attn_bwd_sm90.cu: rows of a streamed chunk
FTZ = 2.0 ** -126   # ex2.approx.ftz flushes results below the smallest normal to zero


def _poly_rel():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'diffusion-pipe_b200', 'csrc',
                            'sm90_common.cuh')).read()
    return float(re.search(r'max relative error ([0-9.e-]+)', src).group(1))


POLY_REL = _poly_rel()


def wgmma_chain(K):
    """the n of the accumulation bound of a K-long wgmma dot product"""
    return -(-K // 16) + 16


def mm(a, b, n):
    """E of a @ b.T over fp32 tensor-core accumulation of chain n; a, b are E (or exact tensors)"""
    a = a if isinstance(a, E) else exact(a)
    b = b if isinstance(b, E) else exact(b)
    av, bv = a.v.abs(), b.v.abs()
    v = a.v @ b.v.t()
    e = C * n * U * (av @ bv.t())
    if a.e.any():
        e = e + a.e @ bv.t()
    if b.e.any():
        e = e + av @ b.e.t() + a.e @ b.e.t()
    return E(v, e)


def gemm_acc(A, B):
    """the kernel's fp32 accumulator of A[M, K] @ B[N, K]^T (logical layouts: transpose MN-major operands first)"""
    return mm(A.double(), B.double(), wgmma_chain(A.shape[1]))


# ---------------------------------------------------------------------------------------------------------------
# GELU(tanh) and its derivative in fp32 (csrc/sm90_common.cuh)
# ---------------------------------------------------------------------------------------------------------------
K0, K1 = 0.7978845608028654, 0.044715


def gelu(u, off=()):
    """gelu_tanh of an E input: tanhf's 2 ulp and the rounding of inner are carried through 0.5 u (1 + t).  An input
    off by u.e moves the output by at most |gelu'(u)| u.e + K0 u.e^2 / 2 (Taylor: |gelu_tanh''| <= gelu_tanh''(0) = K0),
    so a u that the kernel rounded to the other bf16 neighbour (u.e one ulp) is within the bound where gelu curves."""
    x = u.v
    inner = K0 * (x + K1 * x ** 3)
    t = torch.tanh(inner)
    v = 0.5 * x * (1 + t)
    ai = K0 * (x.abs() + K1 * x.abs() ** 3)
    fn = C * U * (4 * v.abs() + 0.5 * x.abs() * (2 + 4 * ai * (1 - t * t)))
    d = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * K0 * (1 + 3 * K1 * x * x)
    return E(v, (fn if _on('gelu', off) else 0 * v) + d.abs() * u.e + 0.5 * K0 * u.e * u.e)


def gelu_grad(x, off=()):
    """gelu_tanh_grad of an exact bf16 input"""
    x = x.double()
    inner = K0 * (x + K1 * x ** 3)
    t = torch.tanh(inner)
    dinner = K0 * (1 + 3 * K1 * x * x)
    v = 0.5 * (1 + t) + 0.5 * x * (1 - t * t) * dinner
    ai = K0 * (x.abs() + K1 * x.abs() ** 3)
    fn = C * U * (8 * (0.5 * (1 + t).abs() + (0.5 * x * (1 - t * t) * dinner).abs())
                  + (0.5 - x * t * dinner).abs() * (2 + 4 * ai * (1 - t * t)))
    return E(v, fn if _on('gelu', off) else torch.zeros_like(v))


# ---------------------------------------------------------------------------------------------------------------
# GEMM epilogues
# ---------------------------------------------------------------------------------------------------------------
def _row_bcast(vec, M):
    return E(vec.double()[None, :].expand(M, -1))


def sample_of_rows(M, rows_per_batch, device):
    return torch.arange(M, device=device) // rows_per_batch


def gemm_store_ref(acc, bias=None, old=None):
    """DPIPE_EPI_STORE: bf16((acc + old) + bias)"""
    o = acc
    if old is not None:
        o = add(o, exact(old))
    if bias is not None:
        o = add(o, _row_bcast(bias, acc.v.shape[0]))
    return {'out': o}


def gemm_bias_gelu_ref(acc, bias=None, off=()):
    """DPIPE_EPI_BIAS_GELU: out2 = u = bf16(acc + bias), out = gelu_tanh(u)"""
    u = add(acc, _row_bcast(bias, acc.v.shape[0])) if bias is not None else acc
    u = rnd(u, 'u', off)
    return {'out': gelu(u, off), 'out2': u}


def gemm_gate_res_ref(acc, res, gate, rows_per_batch, bias=None, sample=None, off=()):
    """DPIPE_EPI_GATE_RES: out2 = y = bf16(acc + bias), out = res + bf16(gate[sample] y).  sample: the sample index of
    every row (default row // rows_per_batch)"""
    M = acc.v.shape[0]
    if sample is None:
        sample = sample_of_rows(M, rows_per_batch, acc.v.device)
    y = add(acc, _row_bcast(bias, M)) if bias is not None else acc
    y = rnd(y, 'y', off)
    gy = rnd(mul(exact(gate[sample]), y), 'gy', off)
    return {'out': add(exact(res), gy), 'out2': y}


def gemm_mul_gelu_grad_ref(acc, aux, off=()):
    """DPIPE_EPI_MUL_GELU_GRAD: acc * gelu_tanh'(aux)"""
    return {'out': mul(acc, gelu_grad(aux, off))}


def gemm_qkv_ref(acc, bias, wq, wk, cos, sin, heads, rows_per_batch, seq_offset, n_qkv, eps=1e-6, off=()):
    """DPIPE_EPI_QKV_ROPE.  Returns q / k / v / qhat / khat E [batch, heads, rows_per_batch, 128] (the rows
    [seq_offset, seq_offset + rows_per_batch) of the head-major outputs), q_rstd / k_rstd [batch, heads, rows_per_batch]
    and, when acc has columns past n_qkv, out / out2 [M, N - n_qkv] of the fused MLP half"""
    M, N = acc.v.shape
    H = heads
    B = M // rows_per_batch
    hd = H * 128
    if bias is not None:
        acc = add(acc, _row_bcast(bias, M))
    pos = slice(seq_offset, seq_offset + rows_per_batch)
    c, s = cos[pos].double(), sin[pos].double()

    def heads_of(x, which):   # [M, hd] columns of q / k / v -> [B, H, L, 128]
        sl = slice(which * hd, (which + 1) * hd)
        return E(x.v[:, sl].reshape(B, rows_per_batch, H, 128).transpose(1, 2),
                 x.e[:, sl].reshape(B, rows_per_batch, H, 128).transpose(1, 2))

    out = {'v': heads_of(acc, 2)}
    for which, name, w in ((0, 'q', wq), (1, 'k', wk)):
        x = heads_of(acc, which)
        pre = rnd(x, 'pre', off)
        pss = rnd(x, 'pre_ss', off) if _on('pre', off) else x
        ss = ssum(E(pss.v * pss.v, 2 * pss.v.abs() * pss.e), -1, 128)
        ms = E(ss.v / 128 + eps, ss.e / 128 + C * U * (ss.v / 128 + eps))
        r = torch.rsqrt(ms.v)
        rstd = E(r, 0.5 * r * ms.e / ms.v + 2 * C * U * r)
        rs = E(rstd.v[..., None], rstd.e[..., None])
        xhat = rnd(mul(pre, rs), 'xhat', off)
        y = rnd(mul(xhat, exact(w)), 'yw', off)
        out[name] = rope_fwd(y, c, s)
        out[name + 'hat'] = xhat
        out[name + '_rstd'] = rstd
    if N > n_qkv:
        mlp = gemm_bias_gelu_ref(E(acc.v[:, n_qkv:], acc.e[:, n_qkv:]), None, off)
        out['out'], out['out2'] = mlp['out'], mlp['out2']
    return out


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
def scale_log2(scale, off=()):
    """the c of ex2(S c - m): the host's fp32 product of fp32(scale) and fp32(log2 e)"""
    if not _on('c', off):
        return scale * LOG2E
    return float(torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32))


def _fp32(x, off=()):
    return float(torch.tensor(x, dtype=torch.float32)) if _on('c', off) else x


def poly_columns(Lk, poly, device):
    """keys whose exponential attn_fwd_kernel<POLY> takes from the polynomial: column pairs ((i >> 1) & 7) < POLY of
    the score fragment, i.e. 8-key blocks jb of a 128-key tile with 2 (jb % 4) + (row % 16 >= 8) < POLY"""
    jb = (torch.arange(Lk, device=device) % TK) // 8
    return (jb % 4) < (poly + 1) // 2


def attn_fwd_ref(q, k, v, scale, poly=0, off=()):
    """one (batch, head): q [Lq, 128], k / v [Lk, 128] bf16.  Returns o E [Lq, 128] (unrounded) and lse E [Lq]"""
    Lq, Lk = q.shape[0], k.shape[0]
    nkv = -(-Lk // TK)
    c = scale_log2(scale, off)
    S = mm(q.double(), k.double(), wgmma_chain(128))
    x = S.v * c
    # the running maximum each key's tile was exponentiated against, and the final one
    tmax = torch.stack([x[:, j * TK:(j + 1) * TK].max(1).values for j in range(nkv)], 1)
    run = torch.cummax(tmax, 1).values
    mk = run.repeat_interleave(TK, 1)[:, :Lk]
    m = run[:, -1:]
    dm = (c * S.e).max(1, keepdim=True).values + C * U * m.abs()   # the kernel's m against the reference's
    p = torch.exp2(x - mk)
    rel = LN2 * (c * S.e + C * U * (x.abs() + mk.abs()) + dm) + 2 * C * U
    if poly:
        rel = rel + POLY_REL * poly_columns(Lk, poly, q.device)[None, :]
    P = E(p, p * rel + (2.0 ** -125 if poly else FTZ))   # the polynomial clamps its argument at -125
    if not _on('exp', off):
        P = E(p)
    Pr = rnd(P, 'P', off)
    # rescale of tile j to the final maximum, with the error of the ex2(m_old - m_new) factors applied after it
    w = torch.exp2(mk - m)
    wrel = C * U * nkv * (2 + LN2 * (m - mk).abs())
    vd = v.double()
    n_o = nkv * 9 + 16
    pw = Pr.v * w
    num = E(pw @ vd, (Pr.e * w) @ vd.abs() + (C * n_o * U + wrel.max(1, keepdim=True).values) * (pw.abs() @ vd.abs()))
    lv = (P.v * w).sum(1, keepdim=True)
    le = (P.e * w).sum(1, keepdim=True) + (C * (nkv * 33 + 2) * U + wrel.max(1, keepdim=True).values) * lv
    if poly:
        le = le + (nkv * TK - Lk) * 2.0 ** -125
    o = num.v / lv
    oe = num.e / lv + o.abs() * le / lv + 2 * C * U * o.abs()
    lse = m[:, 0] + torch.log2(lv[:, 0])
    lse_e = dm[:, 0] + le[:, 0] / (lv[:, 0] * LN2) + C * U * (2 * lse.abs() + 4)
    return {'o': E(o, oe), 'lse': E(lse, lse_e)}


def attn_bwd_ref(q, k, v, o, do, lse, scale, off=()):
    """one (batch, head): q / o / do [Lq, 128], k / v [Lk, 128], lse [Lq] the forward's fp32 output.  o is the tensor the
    kernel is given (its D is formed from it).  Returns dq [Lq, 128], dk / dv [Lk, 128] E (unrounded)"""
    Lq, Lk = q.shape[0], k.shape[0]
    c = scale_log2(scale, off)
    sc = _fp32(scale, off)
    od, dod = o.double(), do.double()
    D = ssum(E(od * dod), -1, 4 + 5, keepdim=True)
    S = mm(q.double(), k.double(), wgmma_chain(128))
    ls = lse.double()[:, None]
    x = S.v * c - ls
    p = torch.exp2(x)
    P = E(p, p * (LN2 * (c * S.e + C * U * ((S.v * c).abs() + ls.abs())) + 2 * C * U) + FTZ)
    if not _on('exp', off):
        P = E(p)
    Pr = rnd(P, 'P', off)
    dP = mm(dod, v.double(), wgmma_chain(128))
    t = E(dP.v - D.v, dP.e + D.e + C * U * (dP.v - D.v).abs())
    dS = rnd(mul(P, t), 'dS', off)
    nq, nk = -(-Lq // BC) * 4 + 16, -(-Lk // BC) * 4 + 16
    dv = mm(E(Pr.v.t(), Pr.e.t()), dod.t(), nq)
    dkacc = mm(E(dS.v.t(), dS.e.t()), q.double().t(), nq)
    dqacc = mm(dS, k.double().t(), nk)
    dk = mul(dkacc, E(torch.full_like(dkacc.v, sc)))
    dq = mul(dqacc, E(torch.full_like(dqacc.v, sc)))
    return {'dq': dq, 'dk': dk, 'dv': dv, 'delta': D}


def attn_exact(q, k, v, scale):
    """softmax(q k^T scale) v in fp64: the O a mutated backward would take its D from"""
    s = (q.double() @ k.double().t()) * scale
    return torch.softmax(s, -1) @ v.double()
