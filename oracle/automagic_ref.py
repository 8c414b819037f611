"""The Automagic optimizer step (the reference's optimizers/automagic.py, `type = 'automagic'` at train.py:692-694), two ways.

Per parameter with a gradient, in group order (g widened to fp32, eps = eps[0] of a tuple):

    u0 = g**2 + eps
    factored (ndim >= 2): row = EMA_beta2(u0.mean(-1)); col = EMA_beta2(u0.mean(-2))
                          u = (rsqrt(row / row.mean(-1)) (x) rsqrt(col)) * g
    otherwise:            v = EMA_beta2(u0); u = rsqrt(v) * g
    u /= max(rms(u) / clip_threshold, 1)
    new_lr = clamp(lr_mask + lr_bump where (u > 0) == last polarity else lr_mask - lr_bump, min_lr, max_lr)
    u *= new_lr; avg_lr = mean(new_lr); lr_mask stored as int8 codes with scale absmax(new_lr) / 127 (double)
    bf16 weights: shift += -u + p * (-wd) * new_lr; old = p; p += shift; shift += old - p
    fp32 weights: p += p * (-wd) * new_lr; p -= u

At step 1 of a bf16 parameter the statistics are bf16 tensors (they are created like the parameter), so every op on
them and on u rounds to bf16; from step 2 they are fp32.

`automagic_step_torch_ops` runs that rule as torch ops on CPU, on a state in the reference's `state_dict()` format
(`lr_mask` = {'quantized', 'scale', 'orig_dtype'}), and is pinned bit for bit to the reference's own code by
tests/golden/automagic_golden.pt.  `automagic_apply_emulated` is the apply phase in fp32, one IEEE-rounded operation per
torch op (rsqrt as 1 / sqrt, the square root correctly rounded), fed with given statistics: the specification of
csrc/automagic.cu am_apply_kernel, which must match it bit for bit.
"""
import struct

import torch

BF16 = torch.bfloat16


def f32(x):
    return struct.unpack('f', struct.pack('f', x))[0]


def _t32(x):
    return torch.tensor(f32(x), dtype=torch.float32)


def _eps0(eps):
    return eps[0] if isinstance(eps, (tuple, list)) else eps


def quantize_lr(lr):
    """int8 codes + double scale of an fp32 tensor, as the reference's Auto8bitTensor (CPU: a true fp32 division)"""
    amax = lr.abs().max().item()
    scale = amax / 127.0 if amax > 0 else 1.0
    return {'quantized': (lr / scale).round().clamp(-127, 127).to(torch.int8), 'scale': scale,
            'orig_dtype': torch.float32}


def dequantize_lr(mask):
    return mask['quantized'].to(torch.float32) * mask['scale']


def init_state(p, lr):
    """the state the reference creates before the first step (lr is the start lr after the > 1e-3 override)"""
    mask = quantize_lr(torch.ones(p.shape, dtype=torch.float32, device=p.device) * lr)
    st = {'step': 0, 'lr_mask': mask, 'avg_lr': torch.mean(dequantize_lr(mask)),
          'last_polarity': torch.zeros(p.shape, dtype=torch.bool, device=p.device)}
    if p.ndim >= 2:
        st['exp_avg_sq_row'] = torch.zeros(p.shape[:-1]).to(p)
        st['exp_avg_sq_col'] = torch.zeros(p.shape[:-2] + p.shape[-1:]).to(p)
    else:
        st['exp_avg_sq'] = torch.zeros_like(p)
    if p.dtype == BF16:
        st['shift'] = torch.zeros_like(p)
    return st


def automagic_step_torch_ops(p, g, st, *, beta2, eps, clip_threshold, weight_decay, lr_bump, min_lr, max_lr,
                             stats=None):
    """one step of one parameter, in place on CPU tensors p and st (reference state_dict format; st from init_state on the
    first step).  With `stats` a dict, records what the apply phase is fed: rf / cf (factored) or v, clip divisor,
    previous and new scale, the pre-step codes and polarity."""
    g32 = g.to(torch.float32)
    factored = g32.ndim >= 2
    if st['step'] > 0:                                   # after step 1 the statistics follow the fp32 gradient
        for k in ('exp_avg_sq_row', 'exp_avg_sq_col', 'exp_avg_sq'):
            if k in st:
                st[k] = st[k].to(g32)
    pw = p.clone().float() if p.dtype != torch.float32 else p
    st['step'] += 1
    if stats is not None:
        stats.update(codes=st['lr_mask']['quantized'].clone(), polarity=st['last_polarity'].clone(),
                     old_scale=st['lr_mask']['scale'])
    sq = g32 ** 2 + _eps0(eps)
    if factored:
        row, col = st['exp_avg_sq_row'], st['exp_avg_sq_col']
        row.mul_(beta2).add_(sq.mean(dim=-1), alpha=1.0 - beta2)
        col.mul_(beta2).add_(sq.mean(dim=-2), alpha=1.0 - beta2)
        rf = (row / row.mean(dim=-1, keepdim=True)).rsqrt_()
        cf = col.rsqrt()
        u = torch.mul(rf.unsqueeze(-1), cf.unsqueeze(-2)).mul_(g32)
        if stats is not None:
            stats.update(rf=rf.float().clone(), cf=cf.float().clone())
    else:
        v = st['exp_avg_sq']
        v.mul_(beta2).add_(sq, alpha=1.0 - beta2)
        u = v.rsqrt().mul_(g32)
        if stats is not None:
            stats.update(v=v.float().clone())
    clipdiv = (u.norm(2) / (u.numel() ** 0.5) / clip_threshold).clamp_(min=1.0)
    u.div_(clipdiv)
    cur = (u > 0).to(torch.bool)
    agree = torch.where(st['last_polarity'] == cur, 1, -1)
    st['last_polarity'] = cur
    mask = dequantize_lr(st['lr_mask'])
    new_lr = torch.clamp(torch.where(agree > 0, mask + lr_bump, mask - lr_bump), min=min_lr, max=max_lr)
    u.mul_(new_lr)
    st['lr_mask'] = quantize_lr(new_lr)
    st['avg_lr'] = torch.mean(new_lr)
    if stats is not None:
        stats.update(clipdiv=float(clipdiv), new_scale=st['lr_mask']['scale'], new_lr=new_lr.clone())
    wdu = pw * (-weight_decay) * new_lr if weight_decay != 0 else None
    if p.dtype == BF16:
        u.mul_(-1)
        if wdu is not None:
            u.add_(wdu)
        shift = st['shift']
        shift.add_(u)
        old = p.detach().float()
        p.add_(shift)
        shift.add_(old.sub_(p))
    else:
        if wdu is not None:
            pw.add_(wdu)
        pw.add_(-u)
    return p, st


def _sqrt_rn(x):
    """correctly rounded fp32 square root (fp64 root rounded once: 53 >= 2 * 24 + 2 bits)"""
    return torch.sqrt(x.double()).float()


def automagic_apply_emulated(p, g, *, codes, polarity, shift, old_scale, new_scale, clipdiv, round_bf16, weight_decay,
                             lr_bump, min_lr, max_lr, rf=None, cf=None, v=None):
    """the apply phase on CPU from given statistics: rf [.., R] / cf [.., C] (factored) or the updated v, the clip
    divisor, the previous and new code scales.  fp32, one rounding per op, no FMA, rounded to bf16 after every op on u
    when round_bf16.  Returns (p, shift, codes, polarity) as new tensors (shift None for fp32 weights)."""
    def r(x):
        return x.to(BF16).float() if round_bf16 else x
    one = torch.tensor(1.0, dtype=torch.float32)
    g = g.detach().cpu().float()
    if rf is not None:
        u = r(r(rf.float().unsqueeze(-1) * cf.float().unsqueeze(-2)) * g)
    else:
        u = r(r(one / _sqrt_rn(v.float())) * g)
    u = r(u / _t32(clipdiv))
    mask = codes.float() * _t32(old_scale)
    cur = u > 0
    nl = torch.where(cur == polarity, mask + _t32(lr_bump), mask - _t32(lr_bump))
    nl = torch.minimum(torch.maximum(nl, _t32(min_lr)), _t32(max_lr))
    new_codes = torch.round(nl / _t32(new_scale)).clamp(-127, 127).to(torch.int8)
    u = r(u * nl)
    p32 = p.detach().cpu().float()
    if p.dtype == BF16:
        upd = -u
        if weight_decay != 0:
            upd = r(upd + (p32 * _t32(-weight_decay)) * nl)
        sh = (shift.float() + upd).to(BF16).float()
        pn = (p32 + sh).to(BF16).float()
        sh = (sh + (p32 - pn)).to(BF16)
        return pn.to(BF16), sh, new_codes, cur
    pn = p32
    if weight_decay != 0:
        pn = pn + (p32 * _t32(-weight_decay)) * nl
    return pn + (-u), None, new_codes, cur
