"""optimi's AdamW update (the optimizer of the reference's `type = 'adamw_optimi'`, train.py:676-678), two ways.

RECALLED, not executed: optimi is neither installed in this image nor part of the reference tree, so its update rule is
restated here from memory of its source (optimi/adamw.py, the foreach-free `adamw` path), the way SURVEY.md marks
DeepSpeed's schedule helpers.  Per parameter group and step t (host, double):

    debias(b, t) = (b**t - b) / (b**t - 1)
    beta1_comp = 1 - debias(beta1, t);  beta2_hat = debias(beta2, t)
    wd = 1 - lr * weight_decay             (decouple_lr: 1 - (lr / max_lr) * weight_decay)
    if weight_decay != 0: p.mul_(wd)
    m.lerp_(g, beta1_comp)
    v.mul_(beta2_hat).addcmul_(g, g, value=1 - beta2_hat)
    if kahan and p is bf16:
        c.addcdiv_(m, v.sqrt().add_(eps), value=-lr)
        old = p.clone(); p.add_(c); c.add_(old.sub_(p))
    else:
        p.addcdiv_(m, v.sqrt().add_(eps), value=-lr)

`optimi_adamw_torch_ops` runs that text as torch ops on the state dtype.  `adamw_step_emulated` is the same arithmetic in
fp32, one IEEE-rounded operation per torch op (torch's own fused forms split: lerp as w < 0.5 ? m + w*(g-m) :
g - (g-m)*(1-w), addcmul as v + (value*g)*g, addcdiv as c + (value*m)/den) with an explicit round to the state dtype
wherever a bf16 torch op rounds.  It is the specification of csrc/step_tail.cu `adamw_step_multi_kernel`, which must
match it bit for bit.  The two differ on a small fraction of elements (under 0.1 %): where torch's CPU kernels contract
a multiply and an add (lerp, addcmul, addcdiv), and where torch's CPU bf16 `add_(eps)` rounds eps to bf16 first, so that
`v.sqrt().add_(eps)` may land one bf16 ulp away from the fp32-eps sum the kernel forms.

Both take the fp32 roundings of the host scalars, as the kernel does: lr, beta1_comp, beta2_hat, one_minus_beta2_hat
(= fp32(1 - beta2_hat)), eps, decay (= fp32(wd), 1.0 when weight_decay == 0).
"""
import struct

import torch


def f32(x):
    return struct.unpack('f', struct.pack('f', x))[0]


def _sqrt_rn(x):
    """correctly rounded fp32 square root.  torch's CPU fp32 sqrt goes through a vector math library that is off by one
    ulp on some inputs; the fp64 root rounded to fp32 is the IEEE result (53 >= 2 * 24 + 2 bits)"""
    return torch.sqrt(x.double()).float()


def optimi_scalars(lr, betas, weight_decay, eps, step, decouple_lr=False, max_lr=None):
    """the host scalars of one step, in double (recalled text above), rounded to fp32"""
    def debias(b):
        return (b ** step - b) / (b ** step - 1)
    beta2_hat = debias(betas[1])
    wd = 1 - ((lr / max_lr) if decouple_lr else lr) * weight_decay
    return dict(lr=f32(lr), beta1_comp=f32(1 - debias(betas[0])), beta2_hat=f32(beta2_hat),
                one_minus_beta2_hat=f32(1 - beta2_hat), eps=f32(eps), decay=f32(wd))


def optimi_adamw_torch_ops(p, g, m, v, c, *, lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps, decay):
    """the recalled optimi text on clones of the given tensors (CPU, their own dtype); returns (p, m, v, c)"""
    p, m, v = p.clone(), m.clone(), v.clone()
    c = c.clone() if c is not None else None
    if decay != 1.0:
        p.mul_(decay)
    m.lerp_(g, beta1_comp)
    v.mul_(beta2_hat).addcmul_(g, g, value=one_minus_beta2_hat)
    if c is not None and p.dtype == torch.bfloat16:
        c.addcdiv_(m, v.sqrt().add_(eps), value=-lr)
        old = p.clone()
        p.add_(c)
        c.add_(old.sub_(p))
    else:
        p.addcdiv_(m, v.sqrt().add_(eps), value=-lr)
    return p, m, v, c


def adamw_step_emulated(p, g, m, v, c, *, lr, beta1_comp, beta2_hat, one_minus_beta2_hat, eps, decay):
    """the kernel's specification (CPU): fp32, one rounding per operation, no FMA, rounded to the state dtype where a
    torch op on that dtype rounds.  Returns new (p, m, v, c) tensors in the input dtype (c None when not given)."""
    dt = p.dtype
    if dt == torch.bfloat16:
        def r(x):
            return x.to(torch.bfloat16).to(torch.float32)
    else:
        def r(x):
            return x
    s = {k: torch.tensor(val, dtype=torch.float32) for k, val in
         dict(lr=lr, w=beta1_comp, b2=beta2_hat, omb2=one_minus_beta2_hat, eps=eps, decay=decay).items()}
    p, g, m, v = (t.detach().to('cpu', torch.float32) for t in (p, g, m, v))
    c = c.detach().to('cpu', torch.float32) if c is not None else None
    p = r(p * s['decay'])
    d = g - m
    if abs(beta1_comp) < 0.5:
        m = r(m + s['w'] * d)
    else:
        m = r(g - d * (torch.tensor(1.0, dtype=torch.float32) - s['w']))
    v = r(v * s['b2'])
    v = r(v + (s['omb2'] * g) * g)
    den = r(r(_sqrt_rn(v)) + s['eps'])
    upd = (-s['lr'] * m) / den
    if c is not None:
        c = r(c + upd)
        old = p
        p = r(p + c)
        c = r(c + r(old - p))
    else:
        p = r(p + upd)
    out = [p.to(dt), m.to(dt), v.to(dt), c.to(dt) if c is not None else None]
    return tuple(out)


def update_fp32(m, v, *, lr, eps):
    """the per-step update u = fp32(fp32(-lr * m) / den) that adamw_step_emulated adds, from the already updated bf16 m
    and v (for the Kahan property test's fp64 reference sum)"""
    den = (_sqrt_rn(v.float()).to(v.dtype).float() + torch.tensor(eps, dtype=torch.float32)).to(v.dtype).float()
    return (-torch.tensor(lr, dtype=torch.float32) * m.float()) / den
