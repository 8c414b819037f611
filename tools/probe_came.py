"""Times one CAME step (`type = 'CAME'`) on the two bf16 workloads of tools/probe_automagic.py and tools/probe_prodigy.py:

    python tools/probe_came.py [--reps 10] [--warmup 2] [--out DIR]

  qwen_lora_r32   the rank-32 LoRA factors of 60 Qwen-Image blocks (1680 tensors)
  flux_4_double   a full fine-tune of 4 Flux double blocks (1.36 B parameters)

On each, two variants on their own copies of the weights and state, timed with CUDA events in alternating order:
  torch_ops       the recalled op sequence as torch ops on the GPU (oracle/came_ref.py came_step_torch_ops)
  kernels         optim.CAME.step(): ops.came_step (csrc/came.cu), with fresh gradient tensors every step and
                  zero_grad(set_to_none=True) after it, as in the engine
Prints one JSON line (also written to DIR/probe_came.json, default: the temp directory) with the median step time, the
host time of the step call, the kernels' algorithmic bytes (`kernel_bytes`), GB/s and the share of the H100 SXM's
3.35 TB/s, the card's name and power limit read in this run, and the time of each kernel (by name, summed over its
launches) in one more step under torch.profiler.
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from probe_automagic import qwen_lora_shapes  # noqa: E402
from probe_optim import HBM_PEAK, double_block_shapes, gpu_info  # noqa: E402


def kernel_bytes(shape, esz=2):
    """bytes the step must move for one parameter of this shape.  ndim >= 2: g read three times (u0 sums, sum u^2,
    the momentum / residual pass), exp_avg read and written, p read and written (8 per element), and the four row /
    column statistics read and written; otherwise g twice, exp_avg_sq read, written and read again, exp_avg and p read
    and written (9 per element)"""
    n = 1
    for s in shape:
        n *= s
    if len(shape) < 2:
        return 9 * esz * n
    lead = n // (shape[-2] * shape[-1])
    return 8 * esz * n + 2 * 2 * esz * lead * (shape[-2] + shape[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=tempfile.gettempdir())
    a = ap.parse_args()
    import torch
    from diffusion_pipe_b200 import optim
    from oracle import came_ref as CR
    assert torch.cuda.is_available(), 'probe_came measures on the GPU'
    bf = torch.bfloat16
    res = {'gpu': gpu_info(), 'reps': a.reps, 'hbm_peak_Bps': HBM_PEAK, 'workloads': {}}
    for wname, shapes in (('qwen_lora_r32', qwen_lora_shapes()), ('flux_4_double', double_block_shapes() * 4)):
        torch.manual_seed(0)
        grads = [torch.randn(s, device='cuda', dtype=bf) * 1e-3 for s in shapes]

        def params():
            return [torch.nn.Parameter(torch.randn(s, device='cuda', dtype=bf) * 0.02) for s in shapes]
        kp = params()
        kgrads = [grads, [g.clone() for g in grads]]     # fresh gradient tensors every step, as the engine gives them
        kopt = optim.CAME(kp, lr=1e-4, weight_decay=0.01)
        nk = [0]

        def kernel_step():
            for p, g in zip(kp, kgrads[nk[0] % 2]):
                p.grad = g
            nk[0] += 1
            kopt.step()
            kopt.zero_grad(set_to_none=True)
        tp = [p.detach() for p in params()]
        tgroups = [dict(CR.DEFAULTS, lr=1e-4, weight_decay=0.01, params=tp)]
        tstates = {}

        def torch_step():
            CR.came_step_torch_ops(tgroups, [grads], tstates)
        variants = {'torch_ops': torch_step, 'kernels': kernel_step}
        names = list(variants)
        for _ in range(a.warmup):
            for n in names:
                variants[n]()
        torch.cuda.synchronize()
        times = {n: [] for n in names}
        host = {n: [] for n in names}
        for r in range(a.reps):
            for n in (names if r % 2 == 0 else names[::-1]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                t0 = time.perf_counter()
                variants[n]()
                host[n].append(time.perf_counter() - t0)
                e1.record()
                e1.synchronize()
                times[n].append(e0.elapsed_time(e1) * 1e-3)
        nparam = sum(torch.Size(s).numel() for s in shapes)
        nbytes = sum(kernel_bytes(tuple(s)) for s in shapes)
        w = {'params': nparam, 'tensors': len(shapes), 'kernel_algorithmic_bytes': nbytes,
             'bytes_per_param': nbytes / nparam, 'variants': {}}
        for n in names:
            ts = sorted(times[n])
            med = ts[len(ts) // 2]
            v = {'median_ms': med * 1e3, 'min_ms': ts[0] * 1e3, 'max_ms': ts[-1] * 1e3,
                 'host_median_ms': sorted(host[n])[len(host[n]) // 2] * 1e3}
            if n == 'kernels':
                v.update(GBps=nbytes / med / 1e9, share_of_hbm_peak=nbytes / med / HBM_PEAK)
            w['variants'][n] = v
        w['speedup'] = w['variants']['torch_ops']['median_ms'] / w['variants']['kernels']['median_ms']
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            kernel_step()
            torch.cuda.synchronize()
        phases = {}
        for ev in prof.key_averages():
            m = re.search(r'cm_\w+(<(true|false)>)?', ev.key)
            if m:
                phases[m.group(0)] = phases.get(m.group(0), 0.0) + ev.device_time_total / 1e3
        w['kernel_ms'] = phases
        res['workloads'][wname] = w
        del kopt, kp, kgrads, tp, tstates, tgroups, grads
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'probe_came.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
