"""optimi's AdamW, the optimizer the reference builds for `type = 'adamw_optimi'` (train.py:676-678), on the fused sm_90a
step kernel (csrc/step_tail.cu, `ops.adamw_step`).

bf16 weights updated by a plain optimizer lose most small steps: a weight near 0.02 has a bf16 ulp of 2^-13, so an update
of 2e-5 rounds back to the old value.  With Kahan summation (on by default for bf16 parameters, as in optimi) each bf16
weight carries a bf16 compensation buffer holding what the last rounding dropped, and the pair tracks the exact sum.

State per parameter, allocated like the parameter (bf16 for bf16 weights): `step` (host int), `exp_avg`, `exp_avg_sq` and,
with Kahan summation, `kahan_comp` — 6 B per bf16 parameter (4 B without Kahan), against 4 B for torch.optim.AdamW.
"""
import math
import struct

import torch

from . import _abi, ops


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


_AUTOMAGIC_STATS = ('exp_avg_sq_row', 'exp_avg_sq_col', 'exp_avg_sq')


class Automagic(torch.optim.Optimizer):
    """The reference's Automagic (optimizers/automagic.py, `type = 'automagic'`): a per-element learning rate that grows
    by lr_bump while the sign of the update holds and shrinks when it flips, on Adafactor-style factored second moments,
    with Kahan-summed bf16 weights.  Each step is two fused phases per param group (`ops.automagic_stats`, then
    `ops.automagic_apply`; csrc/automagic.cu), with no host synchronisation.

    As in the reference: a start lr above 1e-3 is replaced by 1e-6 (with a warning) for the mask, `group['lr']` keeps the
    given value and nothing in the step reads it, so LR schedulers have no effect; lr_bump, min_lr and max_lr apply to the
    whole optimizer, beta2, eps, clip_threshold and weight_decay per group.  Parameters without a gradient are skipped
    and their step count does not advance.

    State per parameter: `step` (host int); `exp_avg_sq_row` / `exp_avg_sq_col` (factored, ndim >= 2) or `exp_avg_sq`,
    fp32 (at step 1 of a bf16 parameter they hold the bf16-rounded values the reference's bf16 state holds); the
    lr mask as int8 codes `lr_mask_q` with an fp64 0-dim `lr_mask_scale`; `last_polarity` (bool); `shift` (bf16 weights
    only); `avg_lr` (fp32 0-dim).  4 B per bf16 parameter plus the factored vectors (adamw_optimi: 6 B).  The reference's
    `RMS` entry (the weights' RMS, written and never read) is not kept.  state_dict() writes the lr mask in the
    reference's format {'quantized', 'scale', 'orig_dtype'} (one sync per tensor, at save time only), and
    load_state_dict() reads it, including a state dict written by the reference; one without any `lr_mask` is ignored,
    as in the reference.  Parameters must be bf16 / fp32 tensors (fp16 and fp8 are refused here) on a CUDA device: the
step kernels refuse CPU tensors, there is no CPU path."""

    def __init__(self, params, lr=1e-6, min_lr=1e-7, max_lr=1e-3, lr_bump=1e-6, eps=(1e-30, 1e-3), clip_threshold=1.0,
                 beta2=0.999, weight_decay=0.0, do_paramiter_swapping=False, paramiter_swapping_factor=0.1):
        if do_paramiter_swapping:
            raise NotImplementedError('automagic: do_paramiter_swapping is not supported (every parameter with a '
                                      'gradient steps)')
        self.lr = lr
        if self.lr > 1e-3:
            print(f'Warning! Start lr is very high: {self.lr}. Forcing to 1e-6. this does not work like prodigy')
            self.lr = 1e-6
        self.min_lr, self.max_lr, self.lr_bump = min_lr, max_lr, lr_bump
        defaults = dict(lr=lr, eps=eps, clip_threshold=clip_threshold, beta2=beta2, weight_decay=weight_decay)
        super().__init__(params, defaults)
        self.base_lrs = [lr for _ in self.param_groups]
        for group in self.param_groups:
            for p in group['params']:
                if p.dtype not in (torch.bfloat16, torch.float32):
                    raise TypeError(f'automagic: parameters must be bf16 or fp32 tensors, got {p.dtype}')

    def _mask_init(self, p):
        """codes and scale of the constant start mask, quantized on the host exactly as on CPU (no device sync)"""
        amax = _f32(self.lr)
        scale = amax / 127.0 if amax > 0 else 1.0
        q = torch.round(torch.tensor(amax, dtype=torch.float32) / torch.tensor(scale, dtype=torch.float32))
        q = int(q.clamp(-127, 127))
        return q, scale

    def _init_state(self, p):
        state = self.state[p]
        q, scale = self._mask_init(p)
        dev = p.device
        state['step'] = 0
        state['lr_mask_q'] = torch.full(p.shape, q, dtype=torch.int8, device=dev)
        state['lr_mask_scale'] = torch.full((), scale, dtype=torch.float64, device=dev)      # a fill: no host copy
        state['avg_lr'] = torch.full((), _f32(q * _f32(scale)), dtype=torch.float32, device=dev)
        state['last_polarity'] = torch.zeros(p.shape, dtype=torch.bool, device=dev)
        if p.ndim >= 2:
            state['exp_avg_sq_row'] = torch.zeros(p.shape[:-1], dtype=torch.float32, device=dev)
            state['exp_avg_sq_col'] = torch.zeros(p.shape[:-2] + p.shape[-1:], dtype=torch.float32, device=dev)
        else:
            state['exp_avg_sq'] = torch.zeros(p.shape, dtype=torch.float32, device=dev)
        if p.dtype == torch.bfloat16:
            state['shift'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return state

    @staticmethod
    def _get_lr(state):
        return state['avg_lr'] if 'avg_lr' in state else 0.0

    def _get_group_lr(self, group):
        lrs = [self._get_lr(self.state[p]) for p in group['params']]
        if not lrs:
            return self.lr
        return float(sum(lrs) / len(lrs))

    def get_learning_rates(self):
        """the mean avg_lr of each group's parameters (logging only: reads device scalars)"""
        lrs = [self._get_group_lr(group) for group in self.param_groups]
        return lrs if lrs else self.base_lrs

    def get_avg_learning_rate(self):
        lrs = self.get_learning_rates()
        return sum(lrs) / len(lrs)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            ps = [p for p in group['params'] if p.grad is not None and p.requires_grad]
            if not ps:
                continue
            sts = []
            for p in ps:
                st = self.state[p] if self.state[p] else self._init_state(p)
                st['step'] += 1
                sts.append(st)
            eps = group['eps']
            if isinstance(eps, (tuple, list)):
                eps = eps[0]
            args = ([p.grad for p in ps], [s.get('exp_avg_sq_row') for s in sts], [s.get('exp_avg_sq_col') for s in sts],
                    [s.get('exp_avg_sq') for s in sts], [s['lr_mask_q'] for s in sts], [s['lr_mask_scale'] for s in sts],
                    [s['last_polarity'] for s in sts], [s.get('shift') for s in sts], [s['avg_lr'] for s in sts],
                    ops.automagic_workspace(ps),
                    [p.dtype == torch.bfloat16 and s['step'] == 1 for p, s in zip(ps, sts)])
            sc = dict(beta2=group['beta2'], eps=eps, lr_bump=self.lr_bump, min_lr=self.min_lr, max_lr=self.max_lr,
                      clip_threshold=group['clip_threshold'], weight_decay=group['weight_decay'])
            ops.automagic_stats(ps, *args, **sc)
            ops.automagic_apply(ps, *args, **sc)
        return loss

    def state_dict(self):
        sd = super().state_dict()
        out = {}
        for k, st in sd['state'].items():
            s = {kk: v for kk, v in st.items() if kk not in ('lr_mask_q', 'lr_mask_scale')}
            if 'lr_mask_q' in st:
                s['lr_mask'] = {'quantized': st['lr_mask_q'], 'scale': float(st['lr_mask_scale'].item()),
                                'orig_dtype': torch.float32}
            out[k] = s
        sd['state'] = out
        return sd

    def load_state_dict(self, state_dict):
        saved = state_dict.get('state') if isinstance(state_dict, dict) else None
        if not isinstance(saved, dict) or not any(isinstance(s, dict) and 'lr_mask' in s for s in saved.values()):
            return                      # not an Automagic state: ignored, as in the reference
        groups, saved_groups = self.param_groups, state_dict['param_groups']
        if len(groups) != len(saved_groups) or any(len(g['params']) != len(s['params'])
                                                    for g, s in zip(groups, saved_groups)):
            raise ValueError('automagic: the loaded state dict has a different parameter group layout')
        for g, s in zip(groups, saved_groups):
            for k, v in s.items():
                if k != 'params':
                    g[k] = v
        self.state.clear()
        for g, s in zip(groups, saved_groups):
            for p, pid in zip(g['params'], s['params']):
                if pid in saved:
                    self.state[p] = self._state_from_saved(p, saved[pid])

    def _state_from_saved(self, p, s):
        """a saved (or reference) per-parameter state on p's device; statistics as fp32 (the reference's are bf16 after
        step 1 of a bf16 parameter), keeping their precision; copies, never views of the saved tensors"""
        dev = p.device
        st = {'step': int(s.get('step', 0))}
        if 'lr_mask' in s:
            m = s['lr_mask']
            st['lr_mask_q'] = m['quantized'].to(device=dev, dtype=torch.int8).clone(memory_format=torch.contiguous_format)
            st['lr_mask_scale'] = torch.tensor(float(m['scale']), dtype=torch.float64, device=dev)
        else:
            q, scale = self._mask_init(p)
            st['lr_mask_q'] = torch.full(p.shape, q, dtype=torch.int8, device=dev)
            st['lr_mask_scale'] = torch.tensor(scale, dtype=torch.float64, device=dev)
        avg = s.get('avg_lr', 0.0)
        st['avg_lr'] = torch.as_tensor(avg, dtype=torch.float32).to(dev).reshape(())
        pol = s.get('last_polarity')
        st['last_polarity'] = (pol.to(device=dev, dtype=torch.bool).clone(memory_format=torch.contiguous_format) if pol is not None else
                               torch.zeros(p.shape, dtype=torch.bool, device=dev))
        if p.ndim >= 2:
            for k, shape in (('exp_avg_sq_row', p.shape[:-1]), ('exp_avg_sq_col', p.shape[:-2] + p.shape[-1:])):
                st[k] = (s[k].to(device=dev, dtype=torch.float32).clone(memory_format=torch.contiguous_format) if k in s else
                         torch.zeros(shape, dtype=torch.float32, device=dev))
        else:
            st['exp_avg_sq'] = (s['exp_avg_sq'].to(device=dev, dtype=torch.float32).clone(memory_format=torch.contiguous_format) if 'exp_avg_sq' in s
                                else torch.zeros(p.shape, dtype=torch.float32, device=dev))
        if p.dtype == torch.bfloat16:
            st['shift'] = (s['shift'].to(device=dev, dtype=torch.bfloat16).clone(memory_format=torch.contiguous_format) if 'shift' in s else
                           torch.zeros_like(p, memory_format=torch.contiguous_format))
        return st


_PRODIGY_SCALARS = ('step', 'd', 'd_max', 'd_hat', 'd_numerator', 'd_denom')


class Prodigy(torch.optim.Optimizer):
    """pytorch_optimizer's Prodigy (`type = 'Prodigy'`, the reference's fallback `getattr(pytorch_optimizer, type)`,
    train.py:698-700): Adam whose step size d is estimated from the run itself, so `lr = 1` needs no tuning.  Each step
    is two fused phases over the parameters of all groups (`ops.prodigy_stats`, then `ops.prodigy_apply`;
    csrc/prodigy.cu), with no host synchronisation: d and its statistics live in one fp64 device block.

    As in the reference: d, d0, d_max, d_coef, growth_rate, lr, betas, beta3 and bias_correction come from
    param_groups[0], and the numerator and denominator of d sum over every group, so the factory's weight-decay / no-
    weight-decay groups share one d; weight_decay, fixed_decay and eps are read per group.  A step in which every
    gradient is zero (d_denom == 0) updates m, v, s and d_numerator and leaves the weights, d and the step count alone.
    `group['lr']` is read every step (LR schedulers work).

    The group entries `step`, `d`, `d_max`, `d_hat`, `d_numerator` and `d_denom` carry the reference's names; during
    training they are 0-dim views of the device block (the same in every group).  state_dict() writes them as Python
    numbers (one sync, at save time only); load_state_dict() takes numbers or tensors.  State per parameter, allocated
    like the parameter: `s`, `p0`, `exp_avg`, `exp_avg_sq` (8 B per bf16 parameter), no Kahan summation (the
    reference's optimizer has none).  Only decoupled weight decay; bf16 / fp32 parameters on a CUDA device (fp16, fp8
    and CPU tensors are refused)."""

    def __init__(self, params, lr=1.0, betas=(0.9, 0.999), beta3=None, d0=1e-6, d_coef=1.0, growth_rate=float('inf'),
                 weight_decay=0.0, weight_decouple=True, fixed_decay=False, bias_correction=False,
                 safeguard_warmup=False, eps=1e-8, gradient_release=False):
        if gradient_release:
            raise NotImplementedError('prodigy: gradient_release is not supported (d is estimated from every '
                                      'parameter before any weight moves)')
        if not weight_decouple:
            raise NotImplementedError('prodigy: weight_decouple=False (L2 weight decay added to the gradient) is not '
                                      'supported; decoupled weight decay is')
        if not 0.0 <= lr:
            raise ValueError(f'invalid learning rate {lr}')
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f'invalid betas {betas}')
        if not d0 > 0.0:
            raise ValueError(f'invalid d0 {d0}')
        if not 0.0 <= weight_decay:
            raise ValueError(f'invalid weight_decay {weight_decay}')
        if not 0.0 <= eps:
            raise ValueError(f'invalid eps {eps}')
        defaults = dict(lr=lr, betas=tuple(betas), beta3=beta3, d0=d0, d_coef=d_coef, growth_rate=growth_rate,
                        weight_decay=weight_decay, weight_decouple=True, fixed_decay=fixed_decay,
                        bias_correction=bias_correction, safeguard_warmup=safeguard_warmup, eps=eps)
        super().__init__(params, defaults)
        dev = None
        for group in self.param_groups:
            for p in group['params']:
                if p.dtype not in (torch.bfloat16, torch.float32):
                    raise TypeError(f'prodigy: parameters must be bf16 or fp32 tensors, got {p.dtype}')
                dev = dev or p.device
        self._block = torch.zeros(_abi.PRODIGY_STATE_DOUBLES, dtype=torch.float64, device=dev)
        self._set_block({})
        self._packed = (None, None)

    def _set_block(self, values):
        """write the group scalars (numbers or tensors) into the device block, and point every group's entries at it;
        d, d_max and d_hat default to d0, the others to 0"""
        d0 = self.param_groups[0]['d0']
        vals = [0.0] * _abi.PRODIGY_STATE_DOUBLES
        for k, v in dict({'d': d0, 'd_max': d0, 'd_hat': d0}, **values).items():
            vals[_abi.PRODIGY_SLOTS[k]] = float(v)
        self._block.copy_(torch.tensor(vals, dtype=torch.float64))
        for group in self.param_groups:
            for k in _PRODIGY_SCALARS:
                group[k] = self._block[_abi.PRODIGY_SLOTS[k]]

    def mean_d(self):
        """the mean of the groups' d as a device scalar (no sync), what the reference logs as train/prodigy_d"""
        return torch.stack([g['d'] for g in self.param_groups]).mean()

    def _init_state(self, p):
        state = self.state[p]
        state['s'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        state['p0'] = p.detach().clone(memory_format=torch.contiguous_format)
        state['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        state['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return state

    def _args(self, ps):
        """ops.ProdigyArgs for the (parameter, group) pairs ps, rebuilt only when that list, a parameter's storage or a
        group's weight_decay / eps / fixed_decay changes (the gradients are passed to each step, not packed)"""
        key = tuple((id(p), p.data_ptr(), g['weight_decay'], g['eps'], g['fixed_decay']) for p, g in ps)
        if self._packed[0] != key:
            sts = [self.state[p] if self.state[p] else self._init_state(p) for p, _ in ps]
            self._packed = (key, ops.prodigy_pack(
                [p for p, _ in ps], [s['s'] for s in sts], [s['p0'] for s in sts], [s['exp_avg'] for s in sts],
                [s['exp_avg_sq'] for s in sts], [g['weight_decay'] for _, g in ps], [g['eps'] for _, g in ps],
                [g['fixed_decay'] for _, g in ps], device=self._block.device))
        return self._packed[1]

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ps = [(p, group) for group in self.param_groups for p in group['params'] if p.grad is not None]
        args = self._args(ps)
        g0 = self.param_groups[0]
        ops.prodigy_stats(args, [p.grad for p, _ in ps], self._block, lr=g0['lr'], betas=g0['betas'],
                          beta3=g0['beta3'], d0=g0['d0'], d_coef=g0['d_coef'], growth_rate=g0['growth_rate'],
                          bias_correction=g0['bias_correction'], safeguard_warmup=g0['safeguard_warmup'])
        ops.prodigy_apply(args, self._block)
        return loss

    def state_dict(self):
        sd = super().state_dict()
        vals = self._block.tolist()                              # the one sync, at save time
        for g in sd['param_groups']:
            for k in _PRODIGY_SCALARS:
                g[k] = vals[_abi.PRODIGY_SLOTS[k]]
            g['step'] = int(g['step'])
        return sd

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        g0 = self.param_groups[0]
        self._set_block({k: g0[k] for k in _PRODIGY_SCALARS if k in g0})
        self._packed = (None, None)


_CAME_FACTORED = ('exp_avg_sq_row', 'exp_avg_sq_col', 'exp_avg_res_row', 'exp_avg_res_col')


class CAME(torch.optim.Optimizer):
    """pytorch_optimizer's CAME (`type = 'CAME'`, the reference's fallback `getattr(pytorch_optimizer, type)`,
    train.py:698-700): Adafactor's factored second moment, plus a factored "confidence" moment of the residual
    (u - m)^2 that scales the momentum update.  Each step is one call over the parameters of all groups
    (`ops.came_step`; csrc/came.cu), at most 10 launches per 64 parameters, with no host synchronisation.

    pytorch_optimizer's constructor surface and defaults; lr, betas, weight_decay, fixed_decay, eps1 and eps2 are read
    per group, `group['lr']` on every step (LR schedulers work); clip_threshold applies to the whole optimizer.
    ams_bound=True, maximize=True, weight_decouple=False (the text's L2 term is added to the gradient after the update
    is computed) and gradient_release are refused.  Parameters without a gradient are skipped and their step count
    does not advance.  State per parameter, pytorch_optimizer's keys, allocated in the parameter's dtype: `step` (host
    int), `exp_avg`, and `exp_avg_sq_row` / `exp_avg_sq_col` / `exp_avg_res_row` / `exp_avg_res_col` (ndim >= 2) or
    `exp_avg_sq`: about 2 B per bf16 parameter (adamw_optimi: 6 B).  The text's `RMS` entry (the weights' RMS, written
    every step and never read) is not kept, and dropped when a state dict that has it is loaded.  Parameters are bf16 /
    fp32 CUDA tensors (fp16 and fp8 are refused here, CPU tensors at the step)."""

    def __init__(self, params, lr=2e-4, betas=(0.9, 0.999, 0.9999), weight_decay=0.0, weight_decouple=True,
                 fixed_decay=False, clip_threshold=1.0, ams_bound=False, eps1=1e-30, eps2=1e-16, maximize=False,
                 gradient_release=False):
        for flag, what in ((ams_bound, 'ams_bound=True'), (maximize, 'maximize=True'),
                           (not weight_decouple, 'weight_decouple=False (L2 weight decay)'),
                           (gradient_release, 'gradient_release (the step runs once after the backward pass)')):
            if flag:
                raise NotImplementedError(f'came: {what} is not supported')
        if not 0.0 <= lr:
            raise ValueError(f'invalid learning rate {lr}')
        if len(betas) != 3 or not all(0.0 <= b < 1.0 for b in betas):
            raise ValueError(f'invalid betas {betas}')
        if not 0.0 <= weight_decay:
            raise ValueError(f'invalid weight_decay {weight_decay}')
        if not (0.0 <= eps1 and 0.0 <= eps2):
            raise ValueError(f'invalid eps1 / eps2 {eps1} / {eps2}')
        if not clip_threshold > 0.0:
            raise ValueError(f'invalid clip_threshold {clip_threshold}')
        self.clip_threshold = clip_threshold
        defaults = dict(lr=lr, betas=tuple(betas), weight_decay=weight_decay, weight_decouple=True,
                        fixed_decay=fixed_decay, ams_bound=False, eps1=eps1, eps2=eps2)
        super().__init__(params, defaults)
        for group in self.param_groups:
            for p in group['params']:
                if p.dtype not in (torch.bfloat16, torch.float32):
                    raise TypeError(f'came: parameters must be bf16 or fp32 tensors, got {p.dtype}')
        self._packed = (None, None)

    def _init_state(self, p):
        state = self.state[p]
        state['step'] = 0
        state['exp_avg'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        if p.ndim >= 2:
            for k in ('exp_avg_sq', 'exp_avg_res'):
                state[k + '_row'] = torch.zeros(p.shape[:-1], dtype=p.dtype, device=p.device)
                state[k + '_col'] = torch.zeros(p.shape[:-2] + p.shape[-1:], dtype=p.dtype, device=p.device)
        else:
            state['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.contiguous_format)
        return state

    def _args(self, ps):
        """ops.CameArgs for the (parameter, group) pairs ps, rebuilt only when that list, a parameter's storage or a
        group option other than lr changes (gradients and learning rates are passed to each step, not packed)"""
        key = tuple((id(p), p.data_ptr(), g['weight_decay'], g['betas'], g['eps1'], g['eps2'], g['fixed_decay'])
                    for p, g in ps)
        if self._packed[0] != key:
            sts = [self.state[p] if self.state[p] else self._init_state(p) for p, _ in ps]
            self._packed = (key, ops.came_pack(
                [p for p, _ in ps], [s['exp_avg'] for s in sts],
                *[[s.get(k) for s in sts] for k in _CAME_FACTORED], [s.get('exp_avg_sq') for s in sts],
                [g['weight_decay'] for _, g in ps], [tuple(g['betas']) for _, g in ps], [g['eps1'] for _, g in ps],
                [g['eps2'] for _, g in ps], [g['fixed_decay'] for _, g in ps]))
        return self._packed[1]

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        ps = [(p, group) for group in self.param_groups for p in group['params'] if p.grad is not None]
        args = self._args(ps)
        ops.came_step(args, [p.grad for p, _ in ps], [g['lr'] for _, g in ps], self.clip_threshold)
        for p, _ in ps:
            self.state[p]['step'] += 1
        return loss

    def load_state_dict(self, state_dict):
        """torch's load (state tensors cast to the parameter's dtype and device), made contiguous; `RMS` dropped"""
        super().load_state_dict(state_dict)
        for st in self.state.values():
            st.pop('RMS', None)
            for k, v in st.items():
                if torch.is_tensor(v) and k != 'step':
                    st[k] = v.contiguous()
            if torch.is_tensor(st.get('step')):
                st['step'] = int(st['step'])
        self._packed = (None, None)


def dynamic_map(signed):
    """bitsandbytes' create_dynamic_map(signed) (8 bits, 7 exponent bits): for each decade 10^(i-6), i = 0..6, the
    midpoints of linspace(0.1, 1, 2^i + 1) (signed, mirrored to negative values) or of linspace(0.1, 1, 2^(i+1) + 1)
    (unsigned), then 0 and 1.0; 256 sorted fp32 values"""
    data = []
    for i in range(7):
        b = torch.linspace(0.1, 1, (2 ** i if signed else 2 ** (i + 1)) + 1, dtype=torch.float32)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (i - 6)) * means).tolist()
        if signed:
            data += (-(10 ** (i - 6)) * means).tolist()
    data += [0.0, 1.0]
    return torch.tensor(sorted(data), dtype=torch.float32)


_A8_TENSORS = ('state1', 'state2', 'qmap1', 'qmap2', 'absmax1', 'absmax2')


class AdamW8bit(torch.optim.Optimizer):
    """bitsandbytes' AdamW8bit (`type = 'adamw8bit'`, train.py:650-700): Adam with decoupled weight decay whose moments
    are uint8 codes of bnb's dynamic maps with one fp32 absmax per 256 elements, about 2.03 B of state per parameter
    (adamw_optimi with Kahan: 6 B).  Parameters below `min_8bit_size` elements keep fp32 moments, as in bnb.  Every step
    is one multi-tensor kernel launch per 64 parameters over all groups (`ops.adamw8bit_step`, csrc/adamw8bit.cu), with
    no host synchronisation; its rule is oracle/adamw8bit_ref.py's.

    bnb's constructor surface and defaults; `optim_bits` is ignored, as in bnb.  block_wise=False, percentile_clipping
    other than 100, amsgrad, is_paged and gradient_release are refused.  `group['lr']`, betas, eps and weight_decay are
    read on every step (LR schedulers work).  Parameters without a gradient are skipped and their step count does not
    advance.  State per parameter, bnb's keys: `step` (int), `state1`, `state2` and, for 8-bit states, `qmap1`, `qmap2`
    (the maps, shared by the parameters of a device), `absmax1`, `absmax2`; load_state_dict() keeps every state tensor
    in its own dtype (torch's default would cast them to the parameter dtype).  Parameters are bf16 / fp32 CUDA tensors
    (fp16 and fp8 are refused here, CPU tensors at the step)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, is_paged=False, gradient_release=False):
        for flag, what in ((not block_wise, 'block_wise=False (one absmax per tensor)'),
                           (percentile_clipping != 100, 'percentile_clipping'), (amsgrad, 'amsgrad'),
                           (is_paged, 'is_paged (paged states)'),
                           (gradient_release, 'gradient_release (the step runs once after the backward pass)')):
            if flag:
                raise NotImplementedError(f'adamw8bit: {what} is not supported')
        if not 0.0 <= lr:
            raise ValueError(f'invalid learning rate {lr}')
        if not (0.0 <= betas[0] < 1.0 and 0.0 <= betas[1] < 1.0):
            raise ValueError(f'invalid betas {betas}')
        if not 0.0 <= weight_decay:
            raise ValueError(f'invalid weight_decay {weight_decay}')
        if not 0.0 <= eps:
            raise ValueError(f'invalid eps {eps}')
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))
        self.min_8bit_size = min_8bit_size
        self._maps = {}
        for group in self.param_groups:
            for p in group['params']:
                if p.dtype not in (torch.bfloat16, torch.float32):
                    raise TypeError(f'adamw8bit: parameters must be bf16 or fp32 tensors, got {p.dtype}')
                self._maps_on(p.device)         # copied to the device here, not in a step

    def _maps_on(self, device):
        if device not in self._maps:
            self._maps[device] = (dynamic_map(True).to(device), dynamic_map(False).to(device))
        return self._maps[device]

    def _init_state(self, p):
        state = self.state[p]
        state['step'] = 0
        if p.numel() < self.min_8bit_size:
            state['state1'] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
            state['state2'] = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
        else:
            nb = (p.numel() + 255) // 256
            state['state1'] = torch.zeros(p.shape, dtype=torch.uint8, device=p.device)
            state['qmap1'], state['qmap2'] = self._maps_on(p.device)
            state['state2'] = torch.zeros(p.shape, dtype=torch.uint8, device=p.device)
            state['absmax1'] = torch.zeros(nb, dtype=torch.float32, device=p.device)
            state['absmax2'] = torch.zeros(nb, dtype=torch.float32, device=p.device)
        return state

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        calls = {}                  # (qmap1, qmap2) -> the parameters stepped with those maps (fp32 states: any call)
        for group in self.param_groups:
            sc = {}
            for p in group['params']:
                if p.grad is None:
                    continue
                st = self.state[p] if self.state[p] else self._init_state(p)
                st['step'] += 1
                t = st['step']
                if t not in sc:
                    sc[t] = adamw8bit_scalars(group['lr'], group['betas'], group['eps'], group['weight_decay'], t)
                key = (id(st['qmap1']), id(st['qmap2'])) if 'qmap1' in st else None
                calls.setdefault(key, []).append((p, st, sc[t]))
        if None in calls and len(calls) > 1:
            plain = calls.pop(None)
            calls[next(iter(calls))] += plain
        for items in calls.values():
            st8 = next((st for _, st, _ in items if 'qmap1' in st), {})
            ops.adamw8bit_step([p for p, _, _ in items], [p.grad for p, _, _ in items],
                               [st['state1'] for _, st, _ in items], [st['state2'] for _, st, _ in items],
                               [st.get('absmax1') for _, st, _ in items], [st.get('absmax2') for _, st, _ in items],
                               [s for _, _, s in items], st8.get('qmap1'), st8.get('qmap2'))
        return loss

    def load_state_dict(self, state_dict):
        """torch's load, then every state tensor again from the saved one in its own dtype on the parameter's device;
        maps equal to this optimizer's are shared again (one launch per step; one comparison per tensor here)"""
        super().load_state_dict(state_dict)
        saved = state_dict['state']
        ids = [i for g in state_dict['param_groups'] for i in g['params']]
        params = [p for g in self.param_groups for p in g['params']]
        for pid, p in zip(ids, params):
            if pid not in saved:
                continue
            st = self.state[p]
            for k in _A8_TENSORS:
                if k in saved[pid]:
                    st[k] = saved[pid][k].to(device=p.device).clone(memory_format=torch.contiguous_format)
            st['step'] = int(saved[pid]['step'])
            if 'qmap1' in st:
                m1, m2 = self._maps_on(p.device)
                if torch.equal(st['qmap1'], m1) and torch.equal(st['qmap2'], m2):
                    st['qmap1'], st['qmap2'] = m1, m2


def adamw8bit_scalars(lr, betas, eps, weight_decay, step):
    """bnb's per-step scalars in double on the host, rounded to fp32 (bnb takes them with powf on the device):
    step_size = -lr * sqrt(1 - beta2^t) / (1 - beta1^t), eps_c2 = fp32(sqrt(1 - beta2^t)) * eps and
    decay = 1 - lr * weight_decay in fp32 arithmetic, as the kernel would compute them"""
    b1, b2 = betas
    c2 = math.sqrt(1.0 - b2 ** step)
    return dict(step_size=_f32(-lr * c2 / (1.0 - b1 ** step)), beta1=_f32(b1), beta2=_f32(b2),
                eps_c2=_f32(_f32(c2) * _f32(eps)), decay=_f32(1.0 - _f32(_f32(lr) * _f32(weight_decay))))
