"""CAME (pytorch_optimizer.CAME, the optimizer the reference builds for `type = 'CAME'` through its fallback
`getattr(pytorch_optimizer, optim_type)`, train.py:698-700), two ways.

RECALLED, not executed: pytorch_optimizer is neither installed in this image nor part of the reference tree, so its
step is restated here from memory of its source (pytorch_optimizer/optimizer/came.py, a port of Luo et al., 2023).  The
factor form is the in-tree `_approx_sq_grad` of the reference's optimizers/automagic.py:146-149:
r = rsqrt(row / row.mean(-1)), c = rsqrt(col).

Per parameter with a gradient, betas (beta1, beta2, beta3) and eps1, eps2 of its group, clip_threshold of the optimizer:

    u0  = g * g + eps1
    factored (ndim >= 2): row = beta2 row + (1 - beta2) u0.mean(-1);  col = beta2 col + (1 - beta2) u0.mean(-2)
                          u = (r(row) (x) c(col)) * g
    otherwise:            v = beta2 v + (1 - beta2) u0;  u = rsqrt(v) * g
    u  /= max(rms(u) / clip_threshold, 1)                     rms(x) = ||x||_2 / sqrt(numel)
    m   = beta1 m + (1 - beta1) u
    res = (u - m)**2 + eps2
    factored: res_row / res_col = EMA_beta3 of res.mean(-1) / res.mean(-2);  upd = (r(res_row) (x) c(res_col)) * m
    otherwise: upd = m
    p  *= 1 - lr * weight_decay  (weight_decouple; fixed_decay: 1 - weight_decay);   p -= lr * upd

Points where memory of the text is unsure, and what is assumed here:
  * Upcasting: the text is recalled to compute in the parameter's dtype, with no fp32 copy of a bf16 gradient or
    weight (the original CAME code upcasts both; pytorch_optimizer's port is recalled not to).  Every elementwise op
    on a bf16 parameter therefore rounds to bf16, as in oracle/prodigy_ref.py.
  * State dtypes: `exp_avg` is `zeros_like(p)`; `exp_avg_sq_row` / `_col`, `exp_avg_res_row` / `_col` and
    `exp_avg_sq` are created with the gradient's dtype.  For a bf16 parameter all of them are bf16.
  * Operation order: `update = grad * grad + eps1` (mul, then add), the EMAs as `x.mul_(beta).add_(y, alpha=1 - beta)`,
    the factors written into `update` by `torch.mul(r, c, out=update)` and then `update.mul_(grad)` (for the residual:
    `.mul_(exp_avg)`), `res = (update - exp_avg).pow_(2).add_(eps2)`, the weight decay before `update.mul_(lr)` and
    `p.add_(-update)`.  eps1 / eps2 are read from the group.
The text's `state['RMS']` (the weights' RMS, written every step and never read) is dropped, as optim.Automagic drops the
reference's: it would cost one more reduction over every weight.

`came_step_torch_ops` runs that text as torch ops (CPU or CUDA).  `came_step_emulated` is the specification of
csrc/came.cu, which must match it bit for bit: fp32, one IEEE rounding per torch op, rounded to bf16 where a bf16 torch
op rounds, in the order torch's CUDA kernels evaluate the text (add with alpha is fma(y, alpha, x); scalars and
coefficients are fp32).  Documented deviations from the text: (1) every reduction (row / column sums, the row mean of
the statistics, sum u^2) is an fp64 sum folded in a fixed order, rounded to fp32 (and then to the dtype) only for the
mean or norm, where torch sums in fp32 in its own order; (2) rsqrt is 1 / sqrt, both correctly rounded, where torch's
CUDA rsqrt is the approximate rsqrtf.  The emulation takes the kernels' own fp64 sums when given (`sums`), so the two
agree bit for bit whatever the order of the fp64 additions.
"""
import math
import struct

import torch

from oracle.prodigy_ref import _fma

BF16 = torch.bfloat16

DEFAULTS = dict(lr=2e-4, betas=(0.9, 0.999, 0.9999), weight_decay=0.0, weight_decouple=True, fixed_decay=False,
                ams_bound=False, eps1=1e-30, eps2=1e-16)
CLIP_THRESHOLD = 1.0


def f32(x):
    return struct.unpack('f', struct.pack('f', x))[0]


def factored(shape):
    return len(shape) >= 2


def init_state(p):
    """the text's state before the first step, without `RMS`"""
    st = {'step': 0, 'exp_avg': torch.zeros_like(p)}
    if factored(p.shape):
        for k in ('exp_avg_sq', 'exp_avg_res'):
            st[k + '_row'] = torch.zeros(p.shape[:-1], dtype=p.dtype, device=p.device)
            st[k + '_col'] = torch.zeros(p.shape[:-2] + p.shape[-1:], dtype=p.dtype, device=p.device)
    else:
        st['exp_avg_sq'] = torch.zeros_like(p)
    return st


# ---------------------------------------------------------------------------------------------------------------------
# the recalled text as torch ops
# ---------------------------------------------------------------------------------------------------------------------
def _approx_sq_grad(row, col, out):
    r = (row / row.mean(dim=-1, keepdim=True)).rsqrt_().unsqueeze(-1)
    c = col.unsqueeze(-2).rsqrt()
    torch.mul(r, c, out=out)


def _rms(x):
    return x.norm(2) / math.sqrt(x.numel())


def came_step_torch_ops(groups, grads, states, clip_threshold=CLIP_THRESHOLD):
    """One step in place.  groups: dicts with 'params' (tensors, updated in place) and the hyper-parameters of
    DEFAULTS; grads: the same nesting, None where a parameter has no gradient; states: {id(p): state}, created on the
    first step."""
    for group, gl in zip(groups, grads):
        beta1, beta2, beta3 = group['betas']
        for p, grad in zip(group['params'], gl):
            if grad is None:
                continue
            st = states.get(id(p))
            if st is None:
                st = states[id(p)] = init_state(p)
            st['step'] += 1
            fact = factored(grad.shape)
            update = torch.mul(grad, grad).add_(group['eps1'])
            if fact:
                row, col = st['exp_avg_sq_row'], st['exp_avg_sq_col']
                row.mul_(beta2).add_(update.mean(dim=-1), alpha=1.0 - beta2)
                col.mul_(beta2).add_(update.mean(dim=-2), alpha=1.0 - beta2)
                _approx_sq_grad(row, col, update)
            else:
                v = st['exp_avg_sq']
                v.mul_(beta2).add_(update, alpha=1.0 - beta2)
                torch.rsqrt(v, out=update)
            update.mul_(grad)
            update.div_((_rms(update) / clip_threshold).clamp_(min=1.0))
            exp_avg = st['exp_avg']
            exp_avg.mul_(beta1).add_(update, alpha=1.0 - beta1)
            res = update - exp_avg
            res.pow_(2).add_(group['eps2'])
            if fact:
                rrow, rcol = st['exp_avg_res_row'], st['exp_avg_res_col']
                rrow.mul_(beta3).add_(res.mean(dim=-1), alpha=1.0 - beta3)
                rcol.mul_(beta3).add_(res.mean(dim=-2), alpha=1.0 - beta3)
                _approx_sq_grad(rrow, rcol, update)
                update.mul_(exp_avg)
            else:
                update = exp_avg.clone()
            wd = group['weight_decay']
            if wd != 0.0:
                p.mul_(1.0 - wd * (1.0 if group['fixed_decay'] else group['lr']))
            update.mul_(group['lr'])
            p.add_(-update)


# ---------------------------------------------------------------------------------------------------------------------
# the kernels' specification
# ---------------------------------------------------------------------------------------------------------------------
def _t(x):
    return torch.tensor(f32(x), dtype=torch.float32)


def _rounder(dtype):
    if dtype == BF16:
        return lambda x: x.to(BF16).float()
    return lambda x: x


def _rsqrt(x):
    """1 / sqrt(x), each correctly rounded in fp32 (the fp64 root of an fp32 value rounds to the fp32 root)"""
    return torch.tensor(1.0, dtype=torch.float32) / torch.sqrt(x.double()).float()


def dims(shape):
    """(L, R, C) of a factored shape: [L = prod(shape[:-2]), R, C]"""
    return math.prod(shape[:-2]), int(shape[-2]), int(shape[-1])


def _moment(r, x3, row, col, beta, sums, key, own):
    """EMA of the row / column means of x3 [L, R, C] into row [L, R] / col [L, C] with the fp64 sums in `sums` (the
    kernels') or taken here; returns (row, col, rf, cf) and records the fp64 sums of its own values in `own`"""
    L, Rn, C = x3.shape
    own[key + '_row'], own[key + '_col'] = x3.double().sum(-1).flatten(), x3.double().sum(-2).flatten()
    rs = sums[key + '_row'].view(L, Rn) if sums else own[key + '_row'].view(L, Rn)
    cs = sums[key + '_col'].view(L, C) if sums else own[key + '_col'].view(L, C)
    a = _t(1.0 - beta)
    b = _t(beta)
    row = r(_fma(r((rs / C).float()), a, r(row * b)))
    col = r(_fma(r((cs / Rn).float()), a, r(col * b)))
    own[key + '_rm'] = row.double().sum(-1).flatten()
    ms = sums[key + '_rm'].view(L) if sums else own[key + '_rm']
    rm = r((ms / Rn).float())
    rf = r(_rsqrt(r(row / rm.unsqueeze(-1))))
    cf = r(_rsqrt(col))
    return row, col, rf, cf


def came_param_emulated(p, g, st, *, lr, betas, weight_decay, fixed_decay, eps1, eps2, clip_threshold, sums=None):
    """One parameter through the specification.  st: the state of init_state (not modified).  sums: the kernels' fp64
    sums of this tensor (keys sumsq and, factored, sq_row, sq_col, sq_rm, res_row, res_col, res_rm), or None
    for fp64 sums taken here.  Returns (new p, new state tensors dict, the fp64 sums of the values computed here in
    that layout, clip divisor).  An empty tensor is skipped, as the kernels skip it."""
    if p.numel() == 0:
        return p.detach().cpu().clone(), {}, {}, 1.0
    dt = p.dtype
    r = _rounder(dt)
    beta1, beta2, beta3 = betas
    shape = p.shape
    g = g.detach().cpu().float()
    pf = p.detach().cpu().float()
    new = {}
    own = {}
    u0 = r(r(g * g) + _t(eps1))
    fact = factored(shape)
    if fact:
        L, Rn, C = dims(shape)
        row, col, rf, cf = _moment(r, u0.reshape(L, Rn, C), st['exp_avg_sq_row'].cpu().float().reshape(L, Rn),
                                   st['exp_avg_sq_col'].cpu().float().reshape(L, C), beta2, sums, 'sq', own)
        new['exp_avg_sq_row'], new['exp_avg_sq_col'] = row, col
        u = r(r(rf.unsqueeze(-1) * cf.unsqueeze(-2)) * g.reshape(L, Rn, C)).reshape(shape)
    else:
        v = r(_fma(u0, _t(1.0 - beta2), r(st['exp_avg_sq'].cpu().float() * _t(beta2))))
        new['exp_avg_sq'] = v
        u = r(r(_rsqrt(v)) * g)
    own['sumsq'] = (u.double() ** 2).sum().reshape(1)
    ss = float(sums['sumsq']) if sums else float(own['sumsq'])
    norm = r(torch.tensor(math.sqrt(ss), dtype=torch.float64).float())
    rms = r(norm / _t(math.sqrt(u.numel())))
    clipdiv = torch.clamp(r(rms / _t(clip_threshold)), min=1.0)
    u = r(u / clipdiv)
    m = r(_fma(u, _t(1.0 - beta1), r(st['exp_avg'].cpu().float() * _t(beta1))))
    new['exp_avg'] = m
    d = r(u - m)
    res = r(r(d * d) + _t(eps2))
    if fact:
        rrow, rcol, rf2, cf2 = _moment(r, res.reshape(L, Rn, C), st['exp_avg_res_row'].cpu().float().reshape(L, Rn),
                                       st['exp_avg_res_col'].cpu().float().reshape(L, C), beta3, sums, 'res', own)
        new['exp_avg_res_row'], new['exp_avg_res_col'] = rrow, rcol
        upd = r(r(rf2.unsqueeze(-1) * cf2.unsqueeze(-2)) * m.reshape(L, Rn, C)).reshape(shape)
    else:
        upd = m
    if weight_decay != 0.0:
        pf = r(pf * _t(1.0 - weight_decay * (1.0 if fixed_decay else lr)))
    pf = r(pf - r(upd * _t(lr)))
    out = {k: v.reshape(st[k].shape).to(dt) for k, v in new.items()}
    return pf.to(dt), out, own, float(clipdiv)


def came_step_emulated(groups, grads, states, clip_threshold=CLIP_THRESHOLD):
    """One whole step through the specification, in place, with the arguments of came_step_torch_ops"""
    for group, gl in zip(groups, grads):
        for p, grad in zip(group['params'], gl):
            if grad is None:
                continue
            st = states.get(id(p))
            if st is None:
                st = states[id(p)] = init_state(p)
            pn, new, _, _ = came_param_emulated(p, grad, st, lr=group['lr'], betas=group['betas'],
                                                weight_decay=group['weight_decay'], fixed_decay=group['fixed_decay'],
                                                eps1=group['eps1'], eps2=group['eps2'], clip_threshold=clip_threshold)
            st['step'] += 1
            for k, v in new.items():
                st[k].copy_(v)
            p.copy_(pn)
