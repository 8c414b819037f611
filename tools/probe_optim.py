"""Times one optimizer step over the parameters of 4 Flux double blocks (1.36 B bf16 parameters, D = 3072):

    python tools/probe_optim.py [--reps 20] [--warmup 3] [--out DIR]

Three variants, each on its own state, timed with CUDA events in alternating order (A B C, B C A, C A B, ...):
  torch_fused_adamw   torch.optim.AdamW(fused=True), bf16 state (what `type = 'adamw'` builds)
  optimi_foreach      optimi's AdamW text with Kahan summation as torch._foreach_* ops (the op-by-op form)
  adamw_step_kernel   ops.adamw_step, the fused sm_90a kernel, Kahan summation on
Prints one JSON line (also written to DIR/probe_optim.json, default: the temp directory) with the median step time, the
algorithmic bytes per step and GB/s against the H100 SXM's 3.35 TB/s, and the card's name and power limit read in this run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D = 3072
HBM_PEAK = 3.35e12


def double_block_shapes(d=D):
    """parameter shapes of one Flux double block (two streams: AdaLN modulation, q/k/v/out projections with biases,
    q/k RMSNorm weights, 4x MLP)"""
    stream = [(6 * d, d), (6 * d,)] + [(d, d), (d,)] * 4 + [(128,), (128,), (4 * d, d), (4 * d,), (d, 4 * d), (d,)]
    return stream * 2


# bytes per parameter read + written by each torch op of the op-by-op form (bf16: 2 B per tensor touched)
FOREACH_TOUCHES = {'p.mul_(wd)': 2, 'm.lerp_(g, w)': 3, 'v.mul_(b2)': 2, 'v.addcmul_(g, g)': 4, 'den = v.sqrt()': 2,
                   'den.add_(eps)': 2, 'c.addcdiv_(m, den)': 4, 'old = p.clone()': 2, 'p.add_(c)': 3,
                   'old.sub_(p)': 3, 'c.add_(old)': 3}


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--blocks', type=int, default=4)
    ap.add_argument('--out', default=tempfile.gettempdir())
    a = ap.parse_args()
    import torch
    from diffusion_pipe_b200 import optim
    assert torch.cuda.is_available(), 'probe_optim measures on the GPU'
    dev = 'cuda'
    bf = torch.bfloat16
    shapes = double_block_shapes() * a.blocks
    nparam = sum(torch.Size(s).numel() for s in shapes)
    torch.manual_seed(0)
    grads = [torch.randn(s, device=dev, dtype=bf) * 1e-3 for s in shapes]

    def params():
        return [torch.nn.Parameter(torch.randn(s, device=dev, dtype=bf) * 0.02) for s in shapes]

    # torch's fused AdamW (bf16 state)
    tp = params()
    for p, g in zip(tp, grads):
        p.grad = g
    topt = torch.optim.AdamW(tp, lr=2e-5, betas=(0.9, 0.99), eps=1e-6, weight_decay=1e-2, fused=True)

    # the kernel
    kp = params()
    for p, g in zip(kp, grads):
        p.grad = g
    kopt = optim.AdamW(kp, lr=2e-5)

    # optimi's text as foreach ops, Kahan on
    fp = [p.detach() for p in params()]
    fm = [torch.zeros_like(p) for p in fp]
    fv = [torch.zeros_like(p) for p in fp]
    fc = [torch.zeros_like(p) for p in fp]
    fstep = [0]

    def foreach_step():
        fstep[0] += 1
        sc = optim.step_scalars(2e-5, (0.9, 0.99), 1e-2, 1e-6, fstep[0])
        torch._foreach_mul_(fp, sc['decay'])
        torch._foreach_lerp_(fm, grads, sc['beta1_comp'])
        torch._foreach_mul_(fv, sc['beta2_hat'])
        torch._foreach_addcmul_(fv, grads, grads, value=sc['one_minus_beta2_hat'])
        den = torch._foreach_sqrt(fv)
        torch._foreach_add_(den, sc['eps'])
        torch._foreach_addcdiv_(fc, fm, den, value=-sc['lr'])
        del den
        old = torch._foreach_mul(fp, 1.0)
        torch._foreach_add_(fp, fc)
        torch._foreach_sub_(old, fp)
        torch._foreach_add_(fc, old)

    variants = {'torch_fused_adamw': topt.step, 'optimi_foreach': foreach_step, 'adamw_step_kernel': kopt.step}
    bytes_per_param = {'torch_fused_adamw': 14, 'optimi_foreach': 2 * sum(FOREACH_TOUCHES.values()),
                       'adamw_step_kernel': 18}
    names = list(variants)
    for _ in range(a.warmup):
        for n in names:
            variants[n]()
    torch.cuda.synchronize()
    times = {n: [] for n in names}
    for r in range(a.reps):
        order = names[r % 3:] + names[:r % 3]
        for n in order:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            variants[n]()
            e1.record()
            e1.synchronize()
            times[n].append(e0.elapsed_time(e1) * 1e-3)
    res = {'gpu': gpu_info(), 'params': nparam, 'blocks': a.blocks, 'reps': a.reps, 'hbm_peak_Bps': HBM_PEAK, 'variants': {}}
    for n in names:
        ts = sorted(times[n])
        med = ts[len(ts) // 2]
        nbytes = bytes_per_param[n] * nparam
        res['variants'][n] = {'median_ms': med * 1e3, 'min_ms': ts[0] * 1e3, 'max_ms': ts[-1] * 1e3,
                              'algorithmic_bytes': nbytes, 'bytes_per_param': bytes_per_param[n],
                              'GBps': nbytes / med / 1e9, 'share_of_hbm_peak': nbytes / med / HBM_PEAK}
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'probe_optim.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
