"""optimi's AdamW, the optimizer the reference builds for `type = 'adamw_optimi'` (train.py:676-678), on the fused sm_90a
step kernel (csrc/step_tail.cu, `ops.adamw_step`).

bf16 weights updated by a plain optimizer lose most small steps: a weight near 0.02 has a bf16 ulp of 2^-13, so an update
of 2e-5 rounds back to the old value.  With Kahan summation (on by default for bf16 parameters, as in optimi) each bf16
weight carries a bf16 compensation buffer holding what the last rounding dropped, and the pair tracks the exact sum.

State per parameter, allocated like the parameter (bf16 for bf16 weights): `step` (host int), `exp_avg`, `exp_avg_sq` and,
with Kahan summation, `kahan_comp` — 6 B per bf16 parameter (4 B without Kahan), against 4 B for torch.optim.AdamW.
"""
import struct

import torch

from . import ops


def _f32(x):
    """the fp32 value nearest to the Python float x (what the kernel receives)"""
    return struct.unpack('f', struct.pack('f', x))[0]


def step_scalars(lr, betas, weight_decay, eps, step, decouple_lr=False, max_lr=None):
    """optimi's per-step scalars, computed in double on the host and rounded to fp32 (no device sync):
    debias(b, t) = (b^t - b) / (b^t - 1);  lerp weight beta1_comp = 1 - debias(beta1, t);  beta2_hat = debias(beta2, t);
    decay = 1 - lr * weight_decay, or with fully decoupled weight decay 1 - (lr / max_lr) * weight_decay"""
    beta1, beta2 = betas

    def debias(b):
        bt = b ** step
        return (bt - b) / (bt - 1.0)
    beta2_hat = debias(beta2)
    decay = 1.0 - (lr / max_lr if decouple_lr else lr) * weight_decay
    return dict(lr=_f32(lr), beta1_comp=_f32(1.0 - debias(beta1)), beta2_hat=_f32(beta2_hat),
                one_minus_beta2_hat=_f32(1.0 - beta2_hat), eps=_f32(eps), decay=_f32(decay))


class AdamW(torch.optim.Optimizer):
    """optimi.AdamW's constructor surface and update rule; every step is one multi-tensor kernel per param group.

    kahan_sum=None turns Kahan summation on for bf16 parameters and off for fp32 ones.  decouple_lr=True applies fully
    decoupled weight decay, scaled by lr / max_lr (max_lr defaults to the group's initial lr).  `group['lr']` is read on
    every step, so LR schedulers work as with any torch optimizer.  Parameters must be CUDA bf16 / fp32 tensors: there is
    no CPU path."""

    def __init__(self, params, lr, betas=(0.9, 0.99), weight_decay=1e-2, eps=1e-6, decouple_lr=False, max_lr=None,
                 kahan_sum=None, gradient_release=False):
        if gradient_release:
            raise NotImplementedError('adamw_optimi: gradient_release is not supported (the step runs once over all '
                                      'parameters after the backward pass)')
        if not 0.0 <= lr:
            raise ValueError(f'invalid learning rate {lr}')
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f'invalid betas {betas}')
        if not 0.0 <= weight_decay:
            raise ValueError(f'invalid weight_decay {weight_decay}')
        if not 0.0 <= eps:
            raise ValueError(f'invalid eps {eps}')
        defaults = dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay, eps=eps, decouple_lr=decouple_lr,
                        max_lr=max_lr, kahan_sum=kahan_sum)
        super().__init__(params, defaults)
        for group in self.param_groups:
            if group['decouple_lr'] and group['max_lr'] is None:
                group['max_lr'] = group['lr']

    def _init_state(self, p, group):
        state = self.state[p]
        state['step'] = 0
        state['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        state['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        kahan = group['kahan_sum']
        if (kahan is None or kahan) and p.dtype == torch.bfloat16:
            state['kahan_comp'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return state

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            by_step = {}            # parameters that missed a step (no gradient) carry a different bias correction
            for p in group['params']:
                if p.grad is None:
                    continue
                state = self.state[p] if self.state[p] else self._init_state(p, group)
                state['step'] += 1
                by_step.setdefault(state['step'], []).append(p)
            for t, ps in by_step.items():
                sc = step_scalars(group['lr'], group['betas'], group['weight_decay'], group['eps'], t, group['decouple_lr'],
                                  group['max_lr'])
                st = [self.state[p] for p in ps]
                ops.adamw_step(ps, [p.grad for p in ps], [s['exp_avg'] for s in st], [s['exp_avg_sq'] for s in st],
                               [s.get('kahan_comp') for s in st], **sc)
        return loss
