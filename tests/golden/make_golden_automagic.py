"""Generates tests/golden/automagic_golden.pt by running the REFERENCE TREE's own Automagic optimizer on CPU.

Run in the build container only (needs /root/reference):   python tests/golden/make_golden_automagic.py

optimizers/automagic.py imports `QBytesTensor` from optimum.quanto (absent from this image) and uses it only in an
isinstance check on the parameter; a stand-in module provides an unrelated class of that name.  Everything else —
optimizers/automagic.py and optimizer_utils.py's Auto8bitTensor — is the reference's code as it is.

Cases (4 steps each, torch.set_num_threads(1), gradients from synth.py seeds): bf16 and fp32 weights; 1-D, 2-D, 4-D and
5-D shapes; LoRA-like [16, 48] / [48, 16]; a weight-decay and a no-weight-decay group; one parameter without a gradient
at step 2; a start lr above 1e-3 (the reference falls back to 1e-6).  Stored per case and step: every parameter and its
full state (minus the never-read `RMS`), and the reference's state_dict() after step 2.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from synth import name_seed, synth_tensor  # noqa: E402

REF = '/root/reference'
OUT = os.path.join(HERE, 'automagic_golden.pt')
STEPS = 4

# (name, dtype, shape, group) per parameter; group 0 has weight decay (as train.py's split), group 1 none
CASES = {
    'bf16_mixed': dict(dtype='bfloat16', lr=1e-6, weight_decay=0.01, clip_threshold=1.0, params=[
        ('w2d', (24, 40), 0), ('lora_a', (16, 48), 0), ('lora_b', (48, 16), 0), ('w4d', (3, 5, 6, 7), 0),
        ('w5d', (2, 3, 2, 4, 5), 0), ('bias', (40,), 1), ('norm', (33,), 1), ('skip', (12, 20), 0)]),
    'fp32_mixed': dict(dtype='float32', lr=1e-6, weight_decay=0.01, clip_threshold=1.0, params=[
        ('w2d', (24, 40), 0), ('lora_a', (16, 48), 0), ('lora_b', (48, 16), 0), ('w4d', (3, 5, 6, 7), 0),
        ('w5d', (2, 3, 2, 4, 5), 0), ('bias', (40,), 1), ('skip', (7,), 1)]),
    'bf16_high_lr_clip': dict(dtype='bfloat16', lr=5e-3, weight_decay=0.1, clip_threshold=0.5, lr_bump=3e-6,
                              min_lr=2e-7, max_lr=5e-4, beta2=0.99, params=[
        ('w2d', (32, 64), 0), ('lora_b', (64, 16), 0), ('bias', (64,), 1), ('scalar', (), 1), ('skip', (8, 8), 0)]),
}
SKIP_AT_STEP = 2          # the parameter named 'skip' has no gradient at this step


def _import_reference():
    quanto = types.ModuleType('optimum.quanto')

    class QBytesTensor:      # only ever the second argument of isinstance
        pass
    quanto.QBytesTensor = QBytesTensor
    optimum = types.ModuleType('optimum')
    optimum.quanto = quanto
    sys.modules['optimum'] = optimum
    sys.modules['optimum.quanto'] = quanto
    sys.path.insert(0, REF)
    from optimizers import automagic
    return automagic.Automagic


def _grad(case, name, shape, step, dtype):
    return synth_tensor(shape, name_seed(f'{case}/{name}/grad/{step}'), 1e-2).to(dtype)


def _state_copy(st):
    out = {}
    for k, v in st.items():
        if k == 'RMS':
            continue
        if k == 'lr_mask':
            out[k] = {'quantized': v.quantized.clone(), 'scale': v.scale, 'orig_dtype': v.orig_dtype}
        elif torch.is_tensor(v):
            out[k] = v.clone()
        else:
            out[k] = v
    return out


def main():
    torch.set_num_threads(1)
    Automagic = _import_reference()
    golden = {'steps': STEPS, 'skip_at_step': SKIP_AT_STEP, 'cases': {}}
    for case, cfg in CASES.items():
        dtype = getattr(torch, cfg['dtype'])
        params, groups = [], [[], []]
        for name, shape, grp in cfg['params']:
            p = torch.nn.Parameter(synth_tensor(shape, name_seed(f'{case}/{name}'), 0.05).to(dtype))
            params.append(p)
            groups[grp].append(p)
        hyper = {k: cfg[k] for k in ('lr_bump', 'min_lr', 'max_lr', 'beta2') if k in cfg}
        opt = Automagic([{'params': groups[0]}, {'params': groups[1], 'weight_decay': 0.0}], lr=cfg['lr'],
                        weight_decay=cfg['weight_decay'], clip_threshold=cfg['clip_threshold'], **hyper)
        rec = {'config': {k: v for k, v in cfg.items() if k != 'params'}, 'params': cfg['params'],
               'init': [p.detach().clone() for p in params], 'grads': [], 'weights': [], 'states': []}
        for step in range(1, STEPS + 1):
            grads = []
            for (name, shape, _), p in zip(cfg['params'], params):
                if name == 'skip' and step == SKIP_AT_STEP:
                    p.grad = None
                    grads.append(None)
                else:
                    p.grad = _grad(case, name, shape, step, dtype)
                    grads.append(p.grad.clone())
            opt.step()
            rec['grads'].append(grads)
            rec['weights'].append([p.detach().clone() for p in params])
            rec['states'].append([_state_copy(opt.state[p]) if opt.state[p] else None for p in params])
            if step == 2:
                rec['state_dict_step2'] = {
                    'state': {k: _state_copy({kk: (vv if kk != 'lr_mask' else types.SimpleNamespace(**vv))
                                              for kk, vv in s.items()})
                              for k, s in opt.state_dict()['state'].items()},
                    'param_groups': opt.state_dict()['param_groups']}
        golden['cases'][case] = rec
    torch.save(golden, OUT)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
