"""bitsandbytes' AdamW8bit (`bitsandbytes.optim.AdamW8bit`, the optimizer the reference builds for `type = 'adamw8bit'`,
train.py:650-700): Adam with decoupled weight decay whose two moments are stored as 8-bit codes of a dynamic map with one
fp32 absmax per block of 256 elements.

RECALLED, not executed: bitsandbytes is neither installed in this image nor part of the reference tree (the reference
only imports it), so the update rule is restated here from memory of its `create_dynamic_map`, the blockwise 8-bit
kernel `kOptimizer8bit2StateBlockwise` and the 32-bit kernel `kOptimizer32bit2State` (ADAM), the way
oracle/optim_ref.py restates optimi.  The block size is 256, the size of current bitsandbytes releases; the reference
leaves bitsandbytes unpinned, and older releases used 2048.

One step of one parameter (step t, counted per parameter; scalars in double on the host, rounded to fp32, where bnb
computes them on the device with powf, a deviation of a few ulp at most):

    c1 = 1 - beta1**t;  c2 = sqrt(1 - beta2**t);  step_size = -lr * c2 / c1
    eps_c2 = fp32(c2) * fp32(eps);  decay = 1 - fp32(lr) * fp32(weight_decay)          (fp32 products)

  numel < min_8bit_size: fp32 state1 = m, state2 = v, per element (g of any value, NaN propagates):
    m = m * beta1 + (1 - beta1) * g
    v = v * beta2 + ((1 - beta2) * g) * g
    p = p + step_size * (m / (sqrt(v) + eps_c2))       rounded to the parameter dtype
    p = p * decay                                      rounded again (bnb applies it when weight_decay > 0; decay is
                                                       then 1 and p * 1 == p, so it is applied unconditionally)
  otherwise: uint8 codes state1 (signed map qmap1) and state2 (unsigned map qmap2), fp32 absmax1 / absmax2 of
  ceil(n / 256) blocks.  Per block of 256 elements:
    m = qmap1[state1] * absmax1[blk], v = qmap2[state2] * absmax2[blk]  (the stored absmax), then m, v as above;
    an element whose gradient is not finite gets m = v = 0 and keeps its p (no update, no weight decay);
    p as above from the new, unquantized m and v;
    absmax1[blk] = max |m|, absmax2[blk] = max v over the block (NaN ignored, as fmaxf does);
    state1 = quantize(qmap1, m / absmax1) and, when the code's map entry and m differ in sign bit, the code moves one
    step towards m's sign (bnb keeps the sign of the first moment: a small negative m maps to the smallest negative
    entry, not to 0); state2 = quantize(qmap2, v / absmax2).  A block whose new absmax is 0 quantizes 0 (every m of
    the block is +-0), so its codes dequantize to 0: an all-zero gradient block (a LoRA `A` at step 1) stays finite.

quantize(map, x) is the index of the nearest map entry, ties and all decided by the fp32 midpoints of adjacent
entries, mid[k] = (map[k] + map[k + 1]) * 0.5: the number of midpoints below x (NaN: 0).  bnb reaches a nearest entry
through a pivot search whose tie rule depends on the search path; this one is the same function away from ties.

Every operation is fp32 with one IEEE round-to-nearest rounding (no fused multiply-add); division and square root are
correctly rounded (bnb uses __fdividef), bf16 rounding is round-to-nearest-even.  `adamw8bit_emulated` is the
specification of csrc/adamw8bit.cu, which must match it bit for bit.
"""
import math

import numpy as np
import torch

BLOCK = 256
F32 = np.float32


def create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8):
    """bitsandbytes.functional.create_dynamic_map: for each decade 10^(i-6), i = 0..6, the midpoints of
    linspace(0.1, 1) (2^i of them signed, 2^(i+1) unsigned, mirrored to negative values when signed), then 0 and 1.0,
    sorted: 256 fp32 values"""
    data = []
    non_sign_bits = total_bits - 1
    additional_items = 2 ** (non_sign_bits - max_exponent_bits) - 1
    for i in range(max_exponent_bits):
        fraction_items = int(2 ** (i + non_sign_bits - max_exponent_bits) + 1 if signed
                             else 2 ** (i + non_sign_bits - max_exponent_bits + 1) + 1)
        boundaries = torch.linspace(0.1, 1, fraction_items, dtype=torch.float32)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    if additional_items > 0:
        boundaries = torch.linspace(0.1, 1, additional_items + 1, dtype=torch.float32)
        means = (boundaries[:-1] + boundaries[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    data.append(0)
    data.append(1.0)
    assert len(data) == 2 ** total_bits
    data.sort()
    return torch.tensor(data, dtype=torch.float32)


def midpoints(qmap):
    q = np.asarray(qmap, dtype=F32)
    return (q[:-1] + q[1:]) * F32(0.5)


def quantize(qmap, x):
    """index of the nearest entry of the sorted map for each fp32 x: the count of midpoints below x (NaN: 0)"""
    x = np.asarray(x, dtype=F32)
    code = np.searchsorted(midpoints(qmap), x, side='left')
    return np.where(np.isnan(x), 0, code).astype(np.uint8)


def step_scalars(lr, betas, eps, weight_decay, step):
    """the fp32 scalars of one step t = `step` (what ops.adamw8bit_step passes per tensor)"""
    b1, b2 = betas
    c1 = 1.0 - b1 ** step
    c2 = math.sqrt(1.0 - b2 ** step)
    return dict(step_size=float(F32(-lr * c2 / c1)), beta1=float(F32(b1)), beta2=float(F32(b2)),
                eps_c2=float(F32(c2) * F32(eps)), decay=float(F32(1.0) - F32(lr) * F32(weight_decay)))


def _np(t):
    return t.detach().cpu().float().numpy().astype(F32).reshape(-1)


def _round(x, dtype):
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=F32))
    return t.to(dtype) if dtype == torch.bfloat16 else t.clone()


def adamw8bit_emulated(p, g, state1, state2, absmax1=None, absmax2=None, qmap1=None, qmap2=None, *, step_size, beta1,
                       beta2, eps_c2, decay):
    """one step of one parameter, on copies; returns (p, state1, state2, absmax1, absmax2) as CPU tensors shaped like
    the inputs (absmax None for the fp32 path).  p and g share a dtype (bf16 or fp32); state1 / state2 are fp32 (the
    32-bit path, absmax None) or uint8 codes with their fp32 absmax and maps."""
    shape, dtype = p.shape, p.dtype
    b1, b2, ss, ec, dc = F32(beta1), F32(beta2), F32(step_size), F32(eps_c2), F32(decay)
    omb1, omb2 = F32(1.0) - b1, F32(1.0) - b2
    pf, gf = _np(p), _np(g)
    with np.errstate(all='ignore'):
        if absmax1 is None:
            m = _np(state1) * b1 + omb1 * gf
            v = _np(state2) * b2 + (omb2 * gf) * gf
            ok = np.ones(pf.shape, dtype=bool)
        else:
            q1, q2 = _np(qmap1), _np(qmap2)
            n = pf.size
            blk = np.arange(n) // BLOCK
            a1, a2 = _np(absmax1), _np(absmax2)
            c1 = state1.detach().cpu().reshape(-1).numpy().astype(np.int64)
            c2 = state2.detach().cpu().reshape(-1).numpy().astype(np.int64)
            ok = np.isfinite(gf)
            v = np.where(ok, (q2[c2] * a2[blk]) * b2 + (omb2 * gf) * gf, F32(0.0)).astype(F32)
            m = np.where(ok, (q1[c1] * a1[blk]) * b1 + omb1 * gf, F32(0.0)).astype(F32)
        upd = ss * (m / (np.sqrt(v) + ec))
        pn = _round(pf + upd, dtype).float().numpy()
        pn = _round(pn * dc, dtype).float().numpy()
        pn = np.where(ok, pn, pf).astype(F32)
        if absmax1 is None:
            return (_round(pn, dtype).view(shape), torch.from_numpy(m.copy()).view(shape),
                    torch.from_numpy(v.copy()).view(shape), None, None)
        nb = a1.size
        pad = nb * BLOCK - n
        am1 = np.fmax.reduce(np.pad(np.abs(m), (0, pad)).reshape(nb, BLOCK), axis=1).astype(F32)
        am2 = np.fmax.reduce(np.pad(np.abs(v), (0, pad)).reshape(nb, BLOCK), axis=1).astype(F32)
        x1 = np.where(am1[blk] > 0, m / np.where(am1[blk] > 0, am1[blk], F32(1.0)), F32(0.0)).astype(F32)
        x2 = np.where(am2[blk] > 0, v / np.where(am2[blk] > 0, am2[blk], F32(1.0)), F32(0.0)).astype(F32)
        k1 = quantize(q1, x1).astype(np.int64)
        flip = np.signbit(q1[k1]) != np.signbit(m)
        k1 = np.where(flip, np.where(m > 0, k1 + 1, k1 - 1), k1)
        k2 = quantize(q2, x2).astype(np.int64)
    return (_round(pn, dtype).view(shape), torch.from_numpy(k1.astype(np.uint8)).view(state1.shape),
            torch.from_numpy(k2.astype(np.uint8)).view(state2.shape), torch.from_numpy(am1), torch.from_numpy(am2))


def init_state(p, min_8bit_size=4096):
    """bnb's state of a parameter before its first step (CPU tensors)"""
    if p.numel() < min_8bit_size:
        return {'step': 0, 'state1': torch.zeros(p.shape, dtype=torch.float32),
                'state2': torch.zeros(p.shape, dtype=torch.float32)}
    nb = (p.numel() + BLOCK - 1) // BLOCK
    return {'step': 0, 'state1': torch.zeros(p.shape, dtype=torch.uint8), 'state2': torch.zeros(p.shape, dtype=torch.uint8),
            'qmap1': create_dynamic_map(True), 'qmap2': create_dynamic_map(False),
            'absmax1': torch.zeros(nb, dtype=torch.float32), 'absmax2': torch.zeros(nb, dtype=torch.float32)}


def step_emulated(p, g, state, *, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
    """one optimizer step of one parameter: advances state['step'] and returns the new p; the state is replaced"""
    state['step'] += 1
    sc = step_scalars(lr, betas, eps, weight_decay, state['step'])
    pn, s1, s2, a1, a2 = adamw8bit_emulated(p, g, state['state1'], state['state2'], state.get('absmax1'),
                                            state.get('absmax2'), state.get('qmap1'), state.get('qmap2'), **sc)
    state['state1'], state['state2'] = s1, s2
    if a1 is not None:
        state['absmax1'], state['absmax2'] = a1, a2
    return pn
