"""Times one AdamW8bit step (`type = 'adamw8bit'`) against the other AdamW steps on the two bf16 workloads of
tools/probe_prodigy.py:

    python tools/probe_adamw8bit.py [--reps 10] [--warmup 2] [--out DIR]

  qwen_lora_r32   the rank-32 LoRA factors of 60 Qwen-Image blocks (1680 tensors)
  flux_4_double   a full fine-tune of 4 Flux double blocks (1.36 B parameters)

On each, three optimizers on their own copies of the weights, with fresh gradient tensors every step and
zero_grad(set_to_none=True) after it, as in the engine, timed with CUDA events in alternating order:
  adamw8bit       optim.AdamW8bit: ops.adamw8bit_step (csrc/adamw8bit.cu)
  adamw_optimi    optim.AdamW with Kahan summation: ops.adamw_step (csrc/step_tail.cu)
  torch_adamw     torch.optim.AdamW(fused=True), bf16 states (`type = 'adamw'`)
Prints one JSON line (also written to DIR/probe_adamw8bit.json, default: the temp directory) with the card's name and
power limit read in this run, and per variant the median step time, the host time of the step call, the state bytes
the first step allocated, and for adamw8bit its algorithmic bytes (10 B per element of a tensor with 8-bit states:
read p, g and two codes, write p and two codes, plus 16 B of absmax per 256; 22 B with fp32 states), GB/s and the
share of the H100 SXM's 3.35 TB/s.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from probe_automagic import qwen_lora_shapes  # noqa: E402
from probe_optim import HBM_PEAK, double_block_shapes, gpu_info  # noqa: E402


def adamw8bit_bytes(n, min_8bit_size=4096):
    if n < min_8bit_size:
        return 22 * n
    return 10 * n + 16 * ((n + 255) // 256)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=tempfile.gettempdir())
    a = ap.parse_args()
    import torch
    from diffusion_pipe_b200 import optim
    assert torch.cuda.is_available(), 'probe_adamw8bit measures on the GPU'
    bf = torch.bfloat16
    res = {'gpu': gpu_info(), 'reps': a.reps, 'hbm_peak_Bps': HBM_PEAK, 'workloads': {}}
    makers = {'adamw8bit': lambda ps: optim.AdamW8bit(ps, lr=1e-4, weight_decay=0.01),
              'adamw_optimi': lambda ps: optim.AdamW(ps, lr=1e-4, weight_decay=0.01),
              'torch_adamw': lambda ps: torch.optim.AdamW(ps, lr=1e-4, weight_decay=0.01, fused=True)}
    for wname, shapes in (('qwen_lora_r32', qwen_lora_shapes()), ('flux_4_double', double_block_shapes() * 4)):
        torch.manual_seed(0)
        grads = [torch.randn(s, device='cuda', dtype=bf) * 1e-3 for s in shapes]
        gsets = [grads, [g.clone() for g in grads]]         # fresh gradient tensors every step, as the engine gives them
        variants, state_bytes = {}, {}
        for name, make in makers.items():
            ps = [torch.nn.Parameter(torch.randn(s, device='cuda', dtype=bf) * 0.02) for s in shapes]
            opt = make(ps)
            count = [0]

            def step(ps=ps, opt=opt, count=count):
                for p, g in zip(ps, gsets[count[0] % 2]):
                    p.grad = g
                count[0] += 1
                opt.step()
                opt.zero_grad(set_to_none=True)
            torch.cuda.synchronize()
            m0 = torch.cuda.memory_allocated()
            step()
            torch.cuda.synchronize()
            state_bytes[name] = torch.cuda.memory_allocated() - m0
            variants[name] = step
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
        nbytes = sum(adamw8bit_bytes(torch.Size(s).numel()) for s in shapes)
        w = {'params': nparam, 'tensors': len(shapes), 'adamw8bit_algorithmic_bytes': nbytes, 'variants': {}}
        for n in names:
            ts = sorted(times[n])
            med = ts[len(ts) // 2]
            v = {'median_ms': med * 1e3, 'min_ms': ts[0] * 1e3, 'max_ms': ts[-1] * 1e3,
                 'host_median_ms': sorted(host[n])[len(host[n]) // 2] * 1e3, 'state_bytes': state_bytes[n],
                 'state_bytes_per_param': state_bytes[n] / nparam}
            if n == 'adamw8bit':
                v.update(GBps=nbytes / med / 1e9, share_of_hbm_peak=nbytes / med / HBM_PEAK)
            w['variants'][n] = v
        res['workloads'][wname] = w
        del variants, gsets, grads
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'probe_adamw8bit.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
