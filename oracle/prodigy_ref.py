"""Prodigy (pytorch_optimizer.Prodigy, the optimizer the reference builds for `type = 'Prodigy'` through its fallback
`getattr(pytorch_optimizer, optim_type)`, train.py:698-700), two ways.

RECALLED, not executed: pytorch_optimizer is neither installed in this image nor part of the reference tree, so its
step is restated here from memory of its source (pytorch_optimizer/optimizer/prodigy.py, itself a port of prodigyopt),
the way oracle/optim_ref.py restates optimi.  Where a detail of pytorch_optimizer could not be recalled, prodigyopt's
text is followed: `safeguard_warmup` (s accumulates with (d / d0) * d instead of (d / d0) * d_lr) and the group step
staying put when the step returns early.

One step over all param groups (d, d0, d_max, d_coef, growth_rate, lr, betas, beta3 and the bias correction from
param_groups[0]; weight_decay, fixed_decay and eps per group), host scalars in double:

    beta3 = beta3 or sqrt(beta2);  t = step + 1
    bias_correction = (1 - beta1**t) / sqrt(1 - beta2**t)  if bias_correction else 1
    d_lr = d * lr / bias_correction                                   (the OLD d)
    d_numerator *= beta3
    every parameter with a gradient, in group order:
        d_numerator += (d / d0) * d_lr * dot(g, p0 - p)
        m = m * beta1 + d * (1 - beta1) * g
        v = v * beta2 + d * d * (1 - beta2) * g * g
        s = s * beta3 + (d / d0) * d_lr * g
        d_denom += sum(|s|)
    d_denom == 0: return (m, v, s and d_numerator are updated; p, d, d_max, d_hat and the step are not)
    d_hat = d_coef * d_numerator / d_denom
    if d == d0: d = max(d, d_hat)
    d_max = max(d_max, d_hat);  d = min(d_max, d * growth_rate);  step = t
    every parameter with a gradient:
        denom = sqrt(v) + d * eps                                     (the NEW d)
        p *= 1 - weight_decay * (1 if fixed_decay else d_lr)          (weight_decouple=True)
        p -= d_lr * m / denom

The state is allocated like the parameter (s, p0, exp_avg, exp_avg_sq: 8 B per bf16 parameter), with no Kahan
summation: every elementwise op on a bf16 parameter rounds to bf16.

`prodigy_step_torch_ops` runs that text as torch ops.  Its per-tensor reductions are torch's: `torch.dot` and `.sum()`
of bf16 tensors return bf16, so each bf16 parameter's dot(g, p0 - p) and sum(|s|) is rounded to bf16 (2^-9 relative)
before it enters the fp32 d_numerator / d_denom, and d_hat is an fp32 quotient.

`prodigy_stats_emulated`, `prodigy_fold` and `prodigy_apply_emulated` are the specification of csrc/prodigy.cu, which
must match them bit for bit.  The elementwise ops are fp32, in the order torch's CUDA kernels (where the reference
trains) evaluate the text, each a single IEEE rounding, rounded to bf16 where a bf16 torch op rounds: x.mul_(beta) is
x * beta; add with alpha is fma(g, alpha, x); addcmul is fma(value, g * g, v); addcdiv is fma(value, m / denom, p); a
scalar added to a tensor and every coefficient are fp32; square roots and quotients correctly rounded.  On fp32 and bf16
CUDA tensors that is the text's result bit for bit (tests/test_prodigy_gpu.py).  torch's CPU kernels evaluate three of
these differently: addcmul as fma(value * g, g, v), addcdiv as (value * m) / denom + p, and a bf16 add rounds its alpha
or scalar to bf16 first; so on CPU the text can land one ulp away.  The per-tensor sums are fp64 (products of fp32
values are exact there); the scalar fold is fp64 in tensor order (d_numerator = d_numerator + k * dot_i, then
d_denom = d_denom + abs_i), so d_numerator, d_denom and d_hat keep fp64 precision where torch's are fp32 (and bf16 per
tensor); beta**t is taken by squaring, so the device computes the same bits as Python.
"""
import math
import struct

import torch

BF16 = torch.bfloat16

DEFAULTS = dict(lr=1.0, betas=(0.9, 0.999), beta3=None, d0=1e-6, d_coef=1.0, growth_rate=float('inf'),
                weight_decay=0.0, weight_decouple=True, fixed_decay=False, bias_correction=False,
                safeguard_warmup=False, eps=1e-8)


def f32(x):
    return struct.unpack('f', struct.pack('f', x))[0]


def init_group_state(d0):
    """the group scalars before the first step (d_numerator is an fp32 tensor in the text)"""
    return {'step': 0, 'd': d0, 'd_max': d0, 'd_hat': d0, 'd_numerator': 0.0, 'd_denom': 0.0}


def init_state(p):
    return {'s': torch.zeros_like(p), 'p0': p.clone(), 'exp_avg': torch.zeros_like(p),
            'exp_avg_sq': torch.zeros_like(p)}


def _beta3(h):
    return h['beta3'] if h['beta3'] is not None else math.sqrt(h['betas'][1])


# ---------------------------------------------------------------------------------------------------------------------
# the recalled text as torch ops
# ---------------------------------------------------------------------------------------------------------------------
def prodigy_step_torch_ops(groups, grads, states, gs):
    """One step in place.  groups: dicts with 'params' (tensors, updated in place) and the hyper-parameters of
    DEFAULTS; grads: the same nesting, None where a parameter has no gradient; states: {id(p): state}, created on the
    first step; gs: the group scalars of init_group_state (d_numerator becomes an fp32 tensor).  Returns False when the
    step returned early (d_denom == 0)."""
    g0 = groups[0]
    beta1, beta2 = g0['betas']
    beta3 = _beta3(g0)
    dev = g0['params'][0].device
    d_denom = torch.tensor([0.0], device=dev)
    if not torch.is_tensor(gs['d_numerator']):
        gs['d_numerator'] = torch.tensor([gs['d_numerator']], dtype=torch.float32, device=dev)
    d_numerator = gs['d_numerator']
    d_numerator.mul_(beta3)
    step = gs['step'] + 1
    bias_correction = ((1.0 - beta1 ** step) / math.sqrt(1.0 - beta2 ** step)) if g0['bias_correction'] else 1.0
    d, d0 = gs['d'], g0['d0']
    d_lr = d * g0['lr'] / bias_correction
    for group, gl in zip(groups, grads):
        for p, grad in zip(group['params'], gl):
            if grad is None:
                continue
            st = states.get(id(p))
            if st is None:
                st = states[id(p)] = init_state(p)
            p0, exp_avg, exp_avg_sq, s = st['p0'], st['exp_avg'], st['exp_avg_sq'], st['s']
            d_numerator.add_(torch.dot(grad.flatten(), (p0 - p).flatten()), alpha=(d / d0) * d_lr)
            exp_avg.mul_(beta1).add_(grad, alpha=d * (1.0 - beta1))
            exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=d * d * (1.0 - beta2))
            s.mul_(beta3).add_(grad, alpha=(d / d0) * (d if g0['safeguard_warmup'] else d_lr))
            d_denom.add_(s.abs().sum())
    if d_denom == 0:
        return False
    d_hat = (g0['d_coef'] * d_numerator / d_denom).item()
    if d == d0:
        d = max(d, d_hat)
    d_max = max(gs['d_max'], d_hat)
    d = min(d_max, d * g0['growth_rate'])
    gs.update(step=step, d=d, d_max=d_max, d_hat=d_hat, d_denom=d_denom.item())
    for group, gl in zip(groups, grads):
        for p, grad in zip(group['params'], gl):
            if grad is None:
                continue
            st = states[id(p)]
            de_nom = st['exp_avg_sq'].sqrt().add_(d * group['eps'])
            p.mul_(1.0 - group['weight_decay'] * (1.0 if group['fixed_decay'] else d_lr))
            p.addcdiv_(st['exp_avg'], de_nom, value=-d_lr)
    return True


# ---------------------------------------------------------------------------------------------------------------------
# the kernels' specification
# ---------------------------------------------------------------------------------------------------------------------
def powi(b, n):
    """b**n for an integer n >= 0 by squaring, in double (the device computes the same bits)"""
    r, x = 1.0, b
    while n:
        if n & 1:
            r = r * x
        x = x * x
        n >>= 1
    return r


def step_scalars(gs, h):
    """the doubles of one step from the group scalars and group 0's hyper-parameters: t, d_lr, the s coefficient k
    and the fp32 coefficients of the elementwise ops"""
    beta1, beta2 = h['betas']
    t = gs['step'] + 1
    bc = ((1.0 - powi(beta1, t)) / math.sqrt(1.0 - powi(beta2, t))) if h['bias_correction'] else 1.0
    d, d0 = gs['d'], h['d0']
    d_lr = d * h['lr'] / bc
    return dict(t=t, d=d, d_lr=d_lr, k=(d / d0) * d_lr, beta1=f32(beta1), beta2=f32(beta2), beta3=f32(_beta3(h)),
                a_m=f32(d * (1.0 - beta1)), a_v=f32(d * d * (1.0 - beta2)),
                a_s=f32((d / d0) * (d if h['safeguard_warmup'] else d_lr)))


def _t(x):
    return torch.tensor(x, dtype=torch.float32)


def _fma(a, b, c):
    """fp32 fused multiply-add, rounded once: the fp32 product is exact in fp64 and TwoSum gives the fp64 sum s with
    its exact error e; s rounds to the same fp32 value as the exact sum unless s lies exactly half-way between two fp32
    values and e != 0, where the exact sum lies on e's side"""
    a, b, c = a.double(), b.double(), c.double()
    prod = a * b
    s = prod + c
    bv = s - prod
    e = (prod - (s - bv)) + (c - bv)
    f = s.float()
    fd = f.double()
    inf = torch.full_like(f, float('inf'))
    other = torch.nextafter(f, torch.where(s > fd, inf, -inf)).double()     # the fp32 neighbour on s's side
    tie = (s != fd) & ((fd + other) / 2 == s) & (e != 0)
    fix = torch.where(e > 0, torch.maximum(fd, other), torch.minimum(fd, other)).float()
    return torch.where(tie, fix, f)


def _rounder(dtype):
    if dtype == BF16:
        return lambda x: x.to(BF16).float()
    return lambda x: x


def prodigy_stats_emulated(p, g, p0, s, m, v, sc):
    """the statistics phase of one parameter: returns (m, v, s) new in the parameter dtype, and the fp64 sums
    dot(g, p0 - p) and sum(|s_new|) (as Python floats; the kernel sums in its own fixed order)"""
    dt = p.dtype
    r = _rounder(dt)
    p, g, p0, s, m, v = (x.detach().cpu().float() for x in (p, g, p0, s, m, v))
    diff = r(p0 - p)
    dot = float((g.double() * diff.double()).sum())
    m = r(_fma(g, _t(sc['a_m']), r(m * _t(sc['beta1']))))
    v = r(_fma(_t(sc['a_v']), g * g, r(v * _t(sc['beta2']))))
    s = r(_fma(g, _t(sc['a_s']), r(s * _t(sc['beta3']))))
    return m.to(dt), v.to(dt), s.to(dt), dot, float(s.double().abs().sum())


def prodigy_fold(gs, h, sc, sums):
    """the finish kernel: the group scalars after the statistics phase from the per-tensor (dot, abs) sums in tensor
    order.  Returns (new group scalars, skipped)."""
    beta3 = _beta3(h)
    num = gs['d_numerator'] * beta3
    for dot, _ in sums:
        num = num + sc['k'] * dot
    den = 0.0
    for _, a in sums:
        den = den + a
    out = dict(gs, d_numerator=num)
    if den == 0.0:
        return out, True
    d = gs['d']
    d_hat = h['d_coef'] * num / den
    if d == h['d0']:
        d = d_hat if d_hat > d else d
    d_max = d_hat if d_hat > gs['d_max'] else gs['d_max']
    dg = d * h['growth_rate']
    d = dg if dg < d_max else d_max
    out.update(step=sc['t'], d=d, d_max=d_max, d_hat=d_hat, d_denom=den)
    return out, False


def prodigy_apply_emulated(p, m, v, *, d_lr, d, eps, weight_decay, fixed_decay):
    """the apply phase of one parameter with the old d_lr and the new d: returns the new p"""
    dt = p.dtype
    r = _rounder(dt)
    p, m, v = (x.detach().cpu().float() for x in (p, m, v))
    den = r(r(torch.sqrt(v.double()).float()) + _t(f32(d * eps)))
    p = r(p * _t(f32(1.0 - weight_decay * (1.0 if fixed_decay else d_lr))))
    p = r(_fma(_t(f32(-d_lr)), m / den, p))
    return p.to(dt)


def prodigy_step_emulated(groups, grads, states, gs):
    """One whole step through the specification, in place, with the arguments of prodigy_step_torch_ops (gs holds
    Python floats).  Returns (skipped, the per-tensor sums)."""
    h = groups[0]
    sc = step_scalars(gs, h)
    todo, sums = [], []
    for group, gl in zip(groups, grads):
        for p, grad in zip(group['params'], gl):
            if grad is None:
                continue
            st = states.get(id(p))
            if st is None:
                st = states[id(p)] = init_state(p)
            m, v, s, dot, a = prodigy_stats_emulated(p, grad, st['p0'], st['s'], st['exp_avg'], st['exp_avg_sq'], sc)
            st['exp_avg'].copy_(m)
            st['exp_avg_sq'].copy_(v)
            st['s'].copy_(s)
            sums.append((dot, a))
            todo.append((p, st, group))
    new, skipped = prodigy_fold(gs, h, sc, sums)
    gs.update(new)
    if not skipped:
        for p, st, group in todo:
            p.copy_(prodigy_apply_emulated(p, st['exp_avg'], st['exp_avg_sq'], d_lr=sc['d_lr'], d=gs['d'],
                                           eps=group['eps'], weight_decay=group['weight_decay'],
                                           fixed_decay=group['fixed_decay']))
    return skipped, sums
