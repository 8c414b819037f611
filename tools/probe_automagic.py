"""Times one Automagic step (`type = 'automagic'`) on two bf16 workloads:

    python tools/probe_automagic.py [--reps 10] [--warmup 2] [--out DIR]

  qwen_lora_r32   the rank-32 LoRA factors lora.py attaches to 60 Qwen-Image blocks (D = 3072): per block the A [32, in]
                  and B [out, 32] factors of the two modulation linears (3072 -> 18432), the eight attention projections
                  (3072 -> 3072) and the two MLPs of each stream (3072 -> 12288 -> 3072); 1440 tensors
  flux_4_double   a full fine-tune of 4 Flux double blocks (1.36 B parameters, tools/probe_optim.py's shapes)

On each, two variants on their own copies of the weights and state, timed with CUDA events in alternating order:
  torch_ops       the reference's op sequence as torch ops on the GPU (oracle/automagic_ref.py
                  automagic_step_torch_ops, including the per-tensor `.item()` of the lr-mask quantization)
  kernels         optim.Automagic.step(): ops.automagic_stats + ops.automagic_apply (csrc/automagic.cu)
Prints one JSON line (also written to DIR/probe_automagic.json, default: the temp directory) with the median step
time, the kernels' algorithmic bytes (derived per tensor below), GB/s and the share of the H100 SXM's 3.35 TB/s, and the
card's name and power limit read in this run, and the time of each kernel phase (statistics, apply) in one more step.
"""
import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from probe_optim import HBM_PEAK, double_block_shapes, gpu_info  # noqa: E402

D = 3072


def qwen_lora_shapes(rank=32, blocks=60, d=D):
    """(out, in) of every adapted linear of one Qwen-Image block, as LoRA factor shapes A [rank, in], B [out, rank]"""
    lins = [(6 * d, d)] * 2 + [(d, d)] * 8 + [(4 * d, d), (d, 4 * d)] * 2
    return [s for o, i in lins for s in ((rank, i), (o, rank))] * blocks


def kernel_bytes(shape, esz=2):
    """bytes the kernels move for one bf16 tensor (elementwise traffic; the O(R + C) statistics are left out):
    factored: reduce pass reads g; lr pass reads g, code, polarity; apply reads g, p, shift, code, polarity and writes
    p, shift, code, polarity.  Unfactored: no reduce pass, exp_avg_sq (fp32) read and written in the lr pass, read in
    apply."""
    n = 1
    for s in shape:
        n *= s
    lr_pass = esz + 1 + 1
    apply = (esz + esz + esz + 1 + 1) + (esz + esz + 1 + 1)
    if len(shape) >= 2:
        return n * (esz + lr_pass + apply)
    return n * (lr_pass + 8 + apply + 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=tempfile.gettempdir())
    a = ap.parse_args()
    import torch
    from diffusion_pipe_b200 import ops, optim
    from oracle import automagic_ref as A
    assert torch.cuda.is_available(), 'probe_automagic measures on the GPU'
    bf = torch.bfloat16
    hyper = dict(beta2=0.999, eps=(1e-30, 1e-3), clip_threshold=1.0, weight_decay=0.01, lr_bump=1e-6, min_lr=1e-7,
                 max_lr=1e-3)
    res = {'gpu': gpu_info(), 'reps': a.reps, 'hbm_peak_Bps': HBM_PEAK, 'workloads': {}}
    for wname, shapes in (('qwen_lora_r32', qwen_lora_shapes()), ('flux_4_double', double_block_shapes() * 4)):
        torch.manual_seed(0)
        grads = [torch.randn(s, device='cuda', dtype=bf) * 1e-3 for s in shapes]

        def params():
            return [torch.nn.Parameter(torch.randn(s, device='cuda', dtype=bf) * 0.02) for s in shapes]
        kp = params()
        for p, g in zip(kp, grads):
            p.grad = g
        kopt = optim.Automagic(kp, weight_decay=hyper['weight_decay'])
        tp = [p.detach() for p in params()]
        tst = [A.init_state(p, 1e-6) for p in tp]

        def torch_step():
            for p, g, st in zip(tp, grads, tst):
                A.automagic_step_torch_ops(p, g, st, **hyper)
        variants = {'torch_ops': torch_step, 'kernels': kopt.step}
        names = list(variants)
        for _ in range(a.warmup):
            for n in names:
                variants[n]()
        torch.cuda.synchronize()
        times = {n: [] for n in names}
        for r in range(a.reps):
            for n in (names if r % 2 == 0 else names[::-1]):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                variants[n]()
                e1.record()
                e1.synchronize()
                times[n].append(e0.elapsed_time(e1) * 1e-3)
        nparam = sum(torch.Size(s).numel() for s in shapes)
        nbytes = sum(kernel_bytes(s) for s in shapes)
        w = {'params': nparam, 'tensors': len(shapes), 'kernel_algorithmic_bytes': nbytes,
             'kernel_bytes_per_param': nbytes / nparam, 'variants': {}}
        for n in names:
            ts = sorted(times[n])
            med = ts[len(ts) // 2]
            v = {'median_ms': med * 1e3, 'min_ms': ts[0] * 1e3, 'max_ms': ts[-1] * 1e3}
            if n == 'kernels':
                v.update(GBps=nbytes / med / 1e9, share_of_hbm_peak=nbytes / med / HBM_PEAK)
            w['variants'][n] = v
        w['speedup'] = w['variants']['torch_ops']['median_ms'] / w['variants']['kernels']['median_ms']
        ops.PROFILE = []                    # one more kernel step with CUDA events around each phase
        kopt.step()
        torch.cuda.synchronize()
        phases = {}
        for e0, e1, _, kind, _ in ops.PROFILE:
            phases[kind] = phases.get(kind, 0.0) + e0.elapsed_time(e1)
        ops.PROFILE = None
        w['kernel_phase_ms'] = phases
        res['workloads'][wname] = w
        del kopt, kp, tp, tst, grads
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, 'probe_automagic.json'), 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
