#!/usr/bin/env python
"""bench.py — training samples/sec for Flux-dev 1024x1024 bf16 full fine-tune on N pipeline stages (N GPUs of one node).

    python bench.py --gpus 1 --steps 3 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the CPU restatement of the reference path, timed on host cores

One "step" = one optimizer step of the reference's hot path (train.py:915-918): GAS micro-batches of forward+backward
through all 59 pipeline layers, gradient clipping, AdamW, on synthetic latents / text embeddings of the named shape
(BASELINE.json configs[1..2]: Flux-dev full fine-tune, bf16, 1024x1024 -> 4096 image + 512 text tokens, micro-batch 1,
16 micro-batches).  Weights are random-initialised at the real architecture (19 double + 38 single blocks, 11.9 B
parameters).  Every stage keeps its bf16 activations (no recompute): 3x forward FLOPs per step, 223.2 TFLOP/sample.

Prints ONE JSON line (rank 0).  `value` = samples/s with the micro-batches resident in HBM; `e2e` = the same through
engine.train_batch with HOST (pinned) micro-batches and a device->host read of the loss inside the timed region.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FWD_TFLOP_PER_BLOCK = 1.3046          # SURVEY.md section 8(d): 1.0437 GEMM + 0.2609 attention, L=4608, D=3072
TRAIN_TFLOP_PER_SAMPLE = 223.2        # 57 blocks x 1.305 x 3 (forward + backward, no recompute)
METRIC = 'training samples/sec (device-timed, max over stages) Flux-dev 1024^2 bf16'   # BASELINE.json:metric
GEMM_FRACTION = 0.80
# the other BASELINE.json configurations (`--family wan|qwen`): full model blocks, algorithmic training TFLOP / sample (SURVEY 8d)
FAMILIES = {
    'flux': {'blocks': 57, 'train_tflop': 223.2, 'metric': METRIC},
    'wan': {'blocks': 40, 'train_tflop': 887.8,
            'metric': 'training samples/sec (device-timed, max over ranks) Wan2.1-14B t2v 33f 512^2 bf16'},
    'qwen': {'blocks': 60, 'train_tflop': 219.4,
             'metric': 'training samples/sec (device-timed, max over ranks) Qwen-Image 1024^2 bf16, 256 text tokens'},
}
WEIGHT_SEED = 1234                    # layer i of the model is initialised from WEIGHT_SEED + i on whatever rank builds it


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument('--gpus', type=int, default=1)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--impl', default='dpipe', choices=['dpipe', 'reference'])
    ap.add_argument('--micro-batches', type=int, default=16)
    ap.add_argument('--micro-batch-size', type=int, default=1)
    ap.add_argument('--res', type=int, default=1024)
    ap.add_argument('--text-len', type=int, default=512)
    ap.add_argument('--layers', type=str, default=None,
                    help='double,single block counts (default: Flux-dev 19,38 from 4 pipeline stages up; 10,20 on 1 or 2 stages, '
                         'where the full model with AdamW state, 8 bytes per parameter = 95 GB, does not fit 80 GB GPUs). '
                         'Scaling comparisons across stage counts must pass the same value everywhere')
    ap.add_argument('--no-optimizer', action='store_true', help='diagnostic: skip the optimizer step (INVALID as a bench value)')
    ap.add_argument('--no-cpu-baseline', action='store_true')
    ap.add_argument('--no-library-baseline', action='store_true',
                    help='skip the cuBLAS + SDPA timing of the restated reference blocks on the GPU (context only, N=1)')
    ap.add_argument('--schedule', default='auto', choices=['auto', '1f1b', 'zb'],
                    help="pipeline order: the reference's 1F1B or the split-backward zero-bubble order (auto: zb whenever there is more than one stage and the stage link is one-sided; the engine itself falls back to 1F1B on torch.distributed p2p links)")
    ap.add_argument('--profile-kernels', action='store_true', default=True)
    ap.add_argument('--family', default='flux', choices=['flux', 'wan', 'qwen'],
                    help='flux = the BASELINE.json metric (configs[1]/[2]); wan = configs[3] (Wan2.1-14B t2v, 33 frames 512^2); '
                         'qwen = configs[4] (Qwen-Image 1024^2, 256 text tokens)')
    ap.add_argument('--pp', type=int, default=0, help='pipeline stages (default: every GPU is a stage)')
    ap.add_argument('--blocks', type=int, default=0, help='wan / qwen: transformer blocks (default: the full model, 40 / 60)')
    ap.add_argument('--frames', type=int, default=33)
    ap.add_argument('--max-inflight', type=int, default=0, help='zero-bubble order: micro-batches a stage may hold (activation memory bound)')
    ap.add_argument('--partition', default='time', choices=['time', 'blocks'],
                    help='flux stage split: balanced by MEASURED block times (double vs single block, probed before the model is built) or by block count')
    ap.add_argument('--instrumented-steps', type=int, default=2,
                    help='extra steps, after the timed region, with a CUDA event pair around every kernel launch (roofline, shares)')
    ap.add_argument('--dump-outputs', metavar='DIR', default=None,
                    help='after the timed steps, write what the last timed step computed (loss, and a fixed seeded sample of the '
                         'updated parameters of this stage) as DIR/<name>.npy, float32/float64, for output-by-output comparison')
    a = ap.parse_args()
    if a.steps < 1:
        ap.error('--steps must be >= 1')
    if a.layers is None:
        a.layers = '19,38' if (a.pp or a.gpus) >= 4 else '10,20'
    return a


DUMP_SAMPLES_PER_TENSOR = 4096        # x ~1000 parameter tensors of the full model: < 16 MB of float32 per stage
DUMP_MAX_BYTES = 60 << 20             # every file of one --dump-outputs run together


def dump_outputs(out_dir, loss, params, stage, stages):
    """loss of the last timed step (float64) and, for this stage, the same seeded positions of every parameter tensor after
    that step's optimizer update (float32), concatenated in parameter order.  Called on data-parallel rank 0 only (the
    replicas of a stage hold the same parameters); the stages share DUMP_MAX_BYTES equally."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)
    g = torch.Generator().manual_seed(0)
    parts, left = [], DUMP_MAX_BYTES // 4 // stages
    for p_ in params:
        flat = p_.detach().reshape(-1)
        n = min(flat.numel(), DUMP_SAMPLES_PER_TENSOR, left)
        if n <= 0:
            break
        idx = torch.randint(flat.numel(), (n,), generator=g)
        parts.append(flat[idx.to(flat.device)].float().cpu())
        left -= n
    sample = torch.cat(parts).numpy() if parts else np.zeros(0, np.float32)
    np.save(os.path.join(out_dir, f'params_sample_stage{stage}.npy'), sample.astype(np.float32))
    if loss is not None:
        np.save(os.path.join(out_dir, 'loss.npy'), np.array([loss], dtype=np.float64))


# ---------------------------------------------------------------------------------------------------------------------
# clocks
# ---------------------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = ('index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,'
         'clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,'
         'clocks_event_reasons.sw_power_cap')

    def __init__(self, index):
        self.index = index
        self.rows = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(['nvidia-smi', f'--query-gpu={self.Q}', '--format=csv,noheader,nounits', '-lms', '200',
                                          '-i', str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(',')])

    def stop(self):
        if self.proc is None:
            return {'sm_mhz': None, 'sm_max_mhz': None, 'reasons': ['nvidia-smi unavailable']}
        self.proc.terminate()
        sm = sorted(int(r[1]) for r in self.rows if len(r) > 2 and r[1].isdigit())
        mx = [int(r[2]) for r in self.rows if len(r) > 2 and r[2].isdigit()]
        reasons = set()
        names = ['hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown', 'sw_power_cap']
        for r in self.rows:
            for i, n in enumerate(names):
                if len(r) > 5 + i and r[5 + i].lower().startswith('active'):
                    reasons.add(n)
        return {'sm_mhz': sm[len(sm) // 2] if sm else None, 'sm_max_mhz': max(mx) if mx else None,
                'reasons': sorted(reasons), 'samples': len(sm)}


# ---------------------------------------------------------------------------------------------------------------------
# CPU baseline: the oracle restatement of the reference blocks on host cores
# ---------------------------------------------------------------------------------------------------------------------
def cpu_reference_sample(res, text_len, n_double, n_single, reps=1):
    """One double + one single block forward+backward at full shapes in fp32 on all host cores; returns
    (samples_per_sec extrapolated to the whole model, description, cores)."""
    import torch
    from oracle import flux_ref as R
    cores = os.cpu_count() or 1
    torch.set_num_threads(cores)
    D, H = 3072, 24
    Li, Lt = (res // 16) ** 2, text_len
    torch.manual_seed(0)
    ids = torch.zeros(Lt + Li, 3)
    ids[Lt:, 1] = torch.arange(Li) // (res // 16)
    ids[Lt:, 2] = torch.arange(Li) % (res // 16)
    cos, sin = R.flux_rope_tables(ids)
    times = {}
    for kind, cls in (('double', R.RefFluxTransformerBlock), ('single', R.RefFluxSingleTransformerBlock)):
        blk = cls(D, H)
        hid = torch.randn(1, Li, D, requires_grad=True)
        enc = torch.randn(1, Lt, D, requires_grad=True)
        temb = torch.randn(1, D, requires_grad=True)
        best = None
        for _ in range(reps):
            t0 = time.perf_counter()
            e, h = blk(hid, enc, temb, (cos, sin))
            (h.sum() + e.sum()).backward()
            dt = time.perf_counter() - t0
            best = dt if best is None else min(best, dt)
        times[kind] = best
        del blk
    per_sample = n_double * times['double'] + n_single * times['single']
    desc = (f'oracle/flux_ref.py blocks, fp32, torch CPU, {cores} threads: 1 double ({times["double"]:.2f}s) + 1 single '
            f'({times["single"]:.2f}s) block fwd+bwd at L={Li + Lt}, D=3072, extrapolated x{n_double}/x{n_single}')
    return 1.0 / per_sample, desc, cores


def gpu_library_sample(res, text_len, n_double, n_single, device, iters=3):
    """SURVEY.md 8(d): what the reference's blocks would dispatch on this GPU — the restated blocks (oracle/flux_ref.py) under
    torch.autocast(bf16), i.e. cuBLAS GEMMs, ATen elementwise kernels and torch SDPA (flash) — one double + one single
    block forward+backward at the full shape, CUDA events, extrapolated to the whole model.  No activation checkpointing
    (the reference adds a forward recompute on top when `activation_checkpointing = true`).  Context for the bench line, not
    part of it; any failure here is reported as a string and never takes the bench line down."""
    import torch
    import torch.nn.functional as F
    from oracle import flux_ref as R
    D, H = 3072, 24
    Li, Lt = (res // 16) ** 2, text_len
    ids = torch.zeros(Lt + Li, 3, device=device)
    ids[Lt:, 1] = torch.arange(Li, device=device) // (res // 16)
    ids[Lt:, 2] = torch.arange(Li, device=device) % (res // 16)
    cos, sin = R.flux_rope_tables(ids)

    def library_sdpa(q, k, v, emulate):
        o = F.scaled_dot_product_attention(q.permute(0, 2, 1, 3).to(torch.bfloat16), k.permute(0, 2, 1, 3).to(torch.bfloat16),
                                           v.permute(0, 2, 1, 3).to(torch.bfloat16))
        return o.permute(0, 2, 1, 3)
    saved = R.sdpa
    R.sdpa = library_sdpa
    times = {}
    try:
        for kind, cls in (('double', R.RefFluxTransformerBlock), ('single', R.RefFluxSingleTransformerBlock)):
            blk = cls(D, H).to(device)
            hid = torch.randn(1, Li, D, device=device, requires_grad=True)
            enc = torch.randn(1, Lt, D, device=device, requires_grad=True)
            temb = torch.randn(1, D, device=device, requires_grad=True)

            def once():
                with torch.autocast('cuda', dtype=torch.bfloat16):
                    e, h = blk(hid, enc, temb, (cos, sin))
                (h.float().sum() + e.float().sum()).backward()
            once()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                once()
            e1.record()
            torch.cuda.synchronize()
            times[kind] = e0.elapsed_time(e1) / iters / 1000.0
            del blk, hid, enc, temb
    finally:
        R.sdpa = saved
    per_sample = n_double * times['double'] + n_single * times['single']
    return {'value': 1.0 / per_sample, 'unit': 'samples/s (blocks only, extrapolated)',
            'kind': 'restated reference blocks on the GPU: cuBLAS + ATen + torch SDPA under autocast(bf16), no recompute',
            'sample': f'1 double ({times["double"] * 1e3:.1f} ms) + 1 single ({times["single"] * 1e3:.1f} ms) block fwd+bwd at L={Li + Lt}, '
                      f'extrapolated x{n_double}/x{n_single}'}


def run_reference_arm(a):
    """--impl reference: the CPU restatement of the reference path (its DeepSpeed+diffusers stack cannot be installed in
    this image: deepspeed / diffusers / peft are absent from /opt/wheelhouse, see DESIGN.md) on the host cores."""
    rank = int(os.environ.get('RANK', 0))
    if rank != 0:
        return
    n_double, n_single = (int(x) for x in a.layers.split(','))
    # one sample = 1 double + 1 single block forward+backward at the full shape (~40 s on 128 threads): the arm is bounded
    # to one untimed and at most two timed samples whatever --warmup / --steps say, so that it ends within ~2 minutes
    vals = []
    n_warm, n_timed = min(a.warmup, 1), max(1, min(a.steps, 3))
    for i in range(n_warm + n_timed):
        t0 = time.perf_counter()
        v, desc, cores = cpu_reference_sample(a.res, a.text_len, n_double, n_single)
        if i >= n_warm:
            vals.append((v, time.perf_counter() - t0))
    value = sorted(v for v, _ in vals)[len(vals) // 2]           # median of the timed samples
    spread = [min(v for v, _ in vals), max(v for v, _ in vals)]
    out = {
        'impl': 'reference', 'metric': METRIC, 'value': value,
        'unit': 'samples/s', 'n_gpus': a.gpus, 'steps': a.steps, 'warmup': a.warmup,
        'ms_per_step': 1000.0 * a.micro_batches * a.micro_batch_size / value, 'higher_is_better': True, 'scaling': 'strong',
        'vs_baseline': None, 'dtype': 'f32', 'data': 'synthetic',
        'config': {'workload': f'Flux-dev full fine-tune bf16 {a.res}x{a.res} (configs[1]/[2] model), {n_double}+{n_single} blocks',
                   'global_batch': a.micro_batches * a.micro_batch_size, 'micro_batch': a.micro_batch_size,
                   'micro_batches': a.micro_batches, 'seq_len': (a.res // 16) ** 2 + a.text_len, 'parallelism': 'host cores',
                   'arithmetic': 'fp32 restatement of the reference path (oracle/flux_ref.py); the reference itself cannot be installed here'},
        'cpu_baseline': {'value': value, 'unit': 'samples/s', 'cores': cores, 'kind': 'port',
                         'sample': desc + f'; median of {len(vals)} timed sample(s) after {n_warm} untimed', 'min_max': spread},
        'e2e': {'value': value, 'unit': 'samples/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0},
        'gpu_launches': 0,
    }
    print(json.dumps(out), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# the GPU arm
# ---------------------------------------------------------------------------------------------------------------------
def gemm_traffic_from_profile():
    """(dram bytes read + written per launch of the dominant GEMM shape, which capture it comes from).  DRAM counters
    exist only under ncu, and a number measured under a profiler is never a bench value: the figure is read from the newest
    committed `ncu --set full` capture of this same command (profiles/rNN_gemm_traffic.json), named next to it."""
    import glob
    for fn in sorted(glob.glob(os.path.join(ROOT, 'profiles', 'r*_gemm_traffic.json')), reverse=True):
        try:
            with open(fn) as f:
                return json.load(f)['dram_bytes_total'], 'profiles/' + os.path.basename(fn)
        except Exception:
            continue
    return None, None


def flop_balanced_split(n_double, n_single, stages):
    """Stage boundaries over [embed, double..., single..., out]: every block costs the same FLOPs (SURVEY 7), the
    embedding rides with the first block and the output layer with the last.  When the block count does not divide, the
    EARLIEST stages take the extra block: a heavier first stage starts at t = 0 and fills its waits with deferred
    weight-gradient work, a heavier last stage delays every backward pass (simulated speed-up at 8 stages, 16
    micro-batches: 7.1x vs 6.3x, csrc/sched.cpp).  Returns (split, blocks_per_stage)."""
    nblk = n_double + n_single
    base, extra = divmod(nblk, stages)
    per_stage = [base + (1 if s < extra else 0) for s in range(stages)]
    bounds, acc = [], 1          # layer 0 is the embedding
    for s in range(stages - 1):
        acc += per_stage[s]
        bounds.append(acc)
    return bounds, per_stage


def synth_micro_batches(a, n, seed, device, pinned):
    import torch
    g = torch.Generator().manual_seed(seed)
    bs = a.micro_batch_size
    h = a.res // 8
    Li = (h // 2) ** 2
    out = []
    for _ in range(n):
        latents = torch.randn(bs, 16, h, h, generator=g)
        noise = torch.randn(bs, 16, h, h, generator=g)
        t = torch.sigmoid(torch.randn(bs, generator=g))
        te = t.view(-1, 1, 1, 1)
        x_t = ((1 - te) * latents + te * noise).view(bs, 16, h // 2, 2, h // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(bs, Li, 64)
        target = (noise - latents).view(bs, 16, h // 2, 2, h // 2, 2).permute(0, 2, 4, 1, 3, 5).reshape(bs, Li, 64)
        t5 = torch.randn(bs, a.text_len, 4096, generator=g).bfloat16()
        clip = torch.randn(bs, 768, generator=g).bfloat16()
        ids = torch.zeros(h // 2, h // 2, 3)
        ids[..., 1] += torch.arange(h // 2)[:, None]
        ids[..., 2] += torch.arange(h // 2)[None, :]
        img_ids = ids.reshape(1, Li, 3).repeat(bs, 1, 1)
        txt_ids = torch.zeros(bs, a.text_len, 3)
        guidance = torch.full((bs,), 1.0)
        img_seq_len = torch.tensor(Li).repeat(bs)
        feats = (x_t.contiguous(), t5, clip, t, img_ids, txt_ids, guidance, img_seq_len)
        label = (target.contiguous(), torch.tensor([]))
        if pinned:
            feats = tuple(x.pin_memory() for x in feats)
            label = (label[0].pin_memory(), label[1])
        else:
            feats = tuple(x.to(device) for x in feats)
            label = (label[0].to(device), label[1])
        out.append((feats, label))
    return out


# fallback calibration of the stage split, used when the probe below fails on every rank or gives an implausible ratio (it
# runs while the other ranks initialise, so a disturbed probe can read far too high): a double block costs 1.30x a single
# block; forward : input-gradient pass : weight-gradient pass = 30 : 47 : 23.  These values were taken on earlier hardware
# and are not measured on H100; the probe replaces them whenever it succeeds.
CALIBRATED_DOUBLE_OVER_SINGLE = 1.30
PLAUSIBLE_DOUBLE_OVER_SINGLE = (1.15, 1.45)
CALIBRATED_FBW = (30, 47, 23)


# bf16 activations a block keeps per sample until its weight-gradient pass (no recompute), GB: Flux-dev 1024^2 and
# Qwen-Image 1024^2 (4352-4608 tokens x 3072) ~0.54, Wan2.1-14B 33 frames 512^2 ~1.8 (from the saved tensors listed in
# DESIGN.md section 3).  HBM_BUDGET_GB leaves 12 GB of an 80 GB H100 for mailboxes, workspaces and the allocator.
ACT_GB_PER_BLOCK = {'flux': 0.54, 'qwen': 0.54, 'wan': 1.8}
HBM_BUDGET_GB = 68.0
# parameters per block: Flux double 36 D^2 (per stream qkv 3, proj 1, MLP 8, modulation 6) and single 15 D^2 at D = 3072;
# Wan2.1-14B 14 B / 40 blocks; Qwen-Image 20.4 B / 60 blocks
PARAMS_PER_BLOCK = {'flux': (36 * 3072 ** 2, 15 * 3072 ** 2), 'wan': (0.35e9, 0.35e9), 'qwen': (0.34e9, 0.34e9)}


def inflight_bound(family, n_double, n_single, stages):
    """micro-batches a stage may hold in the split-backward order so that weights + gradients + AdamW state (8 B per
    parameter) + held activations stay within HBM_BUDGET_GB; at least 1, at most the planner's default 2 x stages.
    Taken from the block counts alone (an even share of the parameters, and one block more than an even share for the
    time-balanced Flux split), so the same bound is known before the split is chosen and used both to choose and to run it.
    Wan / Qwen-Image pass all their blocks as n_double."""
    pd, ps = PARAMS_PER_BLOCK[family]
    params_per_stage = (n_double * pd + n_single * ps) / stages
    blocks = -(-(n_double + n_single) // stages) + (1 if family == 'flux' else 0)
    free = HBM_BUDGET_GB - 8.0 * params_per_stage / 1e9
    per_mb = ACT_GB_PER_BLOCK[family] * max(1, blocks)
    return max(1, min(2 * stages, int(free // per_mb)))


def probe_block_times(device, res, text_len, iters=5):
    """Measured cost of one Flux double and one single block at the bench shape, before the model is built: forward,
    input-gradient pass (weight gradients queued, as the split-backward order runs them) and the queued weight-gradient pass,
    CUDA events, MINIMUM over `iters` after two untimed passes (disturbances only ever add time).
    Returns {'double': (tf, tb, tw), 'single': (tf, tb, tw)} in ms."""
    import torch
    from diffusion_pipe_b200 import flux_blocks as FB
    from diffusion_pipe_b200 import ops
    D, H = 3072, 24
    Li, Lt = (res // 16) ** 2, text_len
    cos = torch.ones(Li + Lt, 128, device=device)
    sin = torch.zeros(Li + Lt, 128, device=device)
    out = {}
    for kind, cls in (('double', FB.FluxTransformerBlock), ('single', FB.FluxSingleTransformerBlock)):
        torch.manual_seed(1)
        blk = cls(D, H, device=device)
        hid = torch.randn(1, Li, D, device=device).bfloat16().requires_grad_(True)
        enc = torch.randn(1, Lt, D, device=device).bfloat16().requires_grad_(True)
        temb = torch.randn(1, D, device=device).bfloat16().requires_grad_(True)
        gh, ge = torch.randn_like(hid), torch.randn_like(enc)
        samples = []
        for it in range(iters + 2):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            eo, ho = blk(hid, enc, temb, (cos, sin))
            ev[1].record()
            q = []
            ops.WGRAD_DEFER = q
            try:
                torch.autograd.backward([ho, eo], [gh, ge])
            finally:
                ops.WGRAD_DEFER = None
            ev[2].record()
            with torch.no_grad():
                for fn in q:
                    fn()
            ev[3].record()
            torch.cuda.synchronize()
            if it >= 2:
                samples.append(tuple(ev[i].elapsed_time(ev[i + 1]) for i in range(3)))
            hid.grad = enc.grad = temb.grad = None
        out[kind] = tuple(min(x[i] for x in samples) for i in range(3))
        del blk, hid, enc, temb, gh, ge, q
    torch.cuda.empty_cache()
    return out


def time_balanced_split(n_double, n_single, stages, t_double, t_single, micro_batches=16, costs=(30, 40, 30), max_inflight=0):
    """Contiguous split of [embed, double x n, single x n, out] by MEASURED block time (a double block costs more time than
    a single block at equal FLOPs: two streams, twice the launches).  Start: the C++ min-max partitioner behind
    partition_method='parameters' fed with times instead of parameter counts; then a local search moves one stage boundary at
    a time while the SIMULATED makespan of the split-backward schedule (csrc/sched.cpp, per-stage costs = the stage's summed
    block time) keeps falling — the pipeline's fill/drain makes the best split slightly uneven.  The embedding and the output
    head are charged 2 % of a single block.  Returns (split, per-stage time in ms, per-stage blocks)."""
    import ctypes
    from diffusion_pipe_b200 import _lib
    from diffusion_pipe_b200.pipe.module import partition_balanced
    unit = 1000.0 / t_single
    w = [20] + [int(round(t_double * unit))] * n_double + [1000] * n_single + [20]
    parts = list(partition_balanced(w, stages))

    def stage_w(pt):
        return [max(1, sum(w[pt[i]:pt[i + 1]]) // 10) for i in range(stages)]

    def makespan(pt):
        sw = (ctypes.c_int * stages)(*stage_w(pt))
        m = _lib.lib().dpipe_sched_zb_makespan_ex(micro_batches, stages, *costs, max_inflight or 2 * stages, sw)
        return (m, sum(x * x for x in sw)) if m > 0 else (0, 0)      # ties: the more even split
    best = makespan(parts)
    improved = True
    while improved and best[0] > 0:
        improved = False
        for b in range(1, stages):
            for d in (-1, 1):
                cand = list(parts)
                cand[b] += d
                if not (cand[b - 1] < cand[b] < cand[b + 1]):
                    continue
                m = makespan(cand)
                if m[0] > 0 and m < best:
                    parts, best, improved = cand, m, True
    per_time = [sum(w[parts[i]:parts[i + 1]]) * t_single / 1000.0 for i in range(stages)]
    per_blocks = [parts[i + 1] - parts[i] - (1 if i == 0 else 0) - (1 if i == stages - 1 else 0) for i in range(stages)]
    return list(parts[1:-1]), per_time, per_blocks


def split_from_probe(t, n_double, n_single, stages, micro_batches, max_inflight):
    """t = [double total, single total, double F, B, W, single F, B, W] in ms, the element-wise minimum of every rank's probe
    (inf where no rank measured).  Returns (split, blocks per stage, planner stage weights, planner F:B:W costs, description);
    a ratio outside the plausible band, or no measurement at all, falls back to the calibrated constants."""
    import math
    t = list(t)
    finite = all(math.isfinite(x) and x > 0 for x in t)
    ratio = t[0] / t[1] if finite else float('nan')
    probe_ok = finite and PLAUSIBLE_DOUBLE_OVER_SINGLE[0] <= ratio <= PLAUSIBLE_DOUBLE_OVER_SINGLE[1]
    if not finite:                 # no rank measured anything: nominal times (only their ratio matters below)
        f_, b_, w_ = (x / 100.0 for x in CALIBRATED_FBW)
        t = [0.0, 4.0] + [4.0 * CALIBRATED_DOUBLE_OVER_SINGLE * x for x in (f_, b_, w_)] + [4.0 * x for x in (f_, b_, w_)]
    if not probe_ok:
        t[0] = CALIBRATED_DOUBLE_OVER_SINGLE * t[1]
    tf, tb, tw = (n_double * t[2 + i] + n_single * t[5 + i] for i in range(3))
    zb_costs = tuple(max(1, int(round(100.0 * x / (tf + tb + tw)))) for x in (tf, tb, tw))     # measured F : B : W shares
    if not probe_ok or any(abs(c - ref) > 0.35 * ref for c, ref in zip(zb_costs, CALIBRATED_FBW)):
        zb_costs = CALIBRATED_FBW
    split, stage_ms, blocks_per_stage = time_balanced_split(n_double, n_single, stages, t[0], t[1], micro_batches, zb_costs, max_inflight)
    stage_weights = [max(1, int(round(100 * x))) for x in stage_ms]
    desc = {'method': 'measured block times, contiguous min-max' if probe_ok else
            f'calibrated block-time ratio {CALIBRATED_DOUBLE_OVER_SINGLE} (the probe measured {ratio:.2f}: implausible or failed)',
            'double_ms': round(t[0], 3), 'single_ms': round(t[1], 3), 'double_over_single': round(t[0] / t[1], 3),
            'blocks_per_stage': blocks_per_stage, 'stage_ms_per_micro_batch': [round(x, 2) for x in stage_ms]}
    return split, blocks_per_stage, stage_weights, zb_costs, desc


def build_family(a, device):
    """(model, layers, example-batch maker or None, workload string, n_blocks)"""
    import torch
    if a.family == 'flux':
        from diffusion_pipe_b200.flux import FluxPipeline
        n_double, n_single = (int(x) for x in a.layers.split(','))
        model = FluxPipeline({'model': {'dtype': 'bfloat16', 'guidance': 1.0, 'lazy_layers': True,
                                        'transformer_config': {'num_layers': n_double, 'num_single_layers': n_single}}},
                             device=device)
        return model, None, f'Flux-dev full fine-tune bf16 {a.res}x{a.res} (configs[1]/[2] model), {n_double}+{n_single} blocks', n_double + n_single
    if a.family == 'wan':
        from diffusion_pipe_b200.wan import WAN_T2V_14B_CONFIG, WanPipeline
        n_blocks = a.blocks or WAN_T2V_14B_CONFIG['num_layers']
        res = a.res if a.res != 1024 else 512
        model = WanPipeline({'model': {'dtype': 'bfloat16', 'lazy_layers': True, 'transformer_config': {'num_layers': n_blocks}}}, device=device)
        lat_f = (a.frames - 1) // 4 + 1

        def example(g):
            return {'latents': torch.randn(16, lat_f, res // 8, res // 8, generator=g),
                    'text_embeddings': torch.randn(512, 4096, generator=g).bfloat16(), 'seq_lens': torch.tensor(512), 'mask': None}
        return model, example, f'Wan2.1-14B t2v full fine-tune bf16, {a.frames} frames {res}x{res} (configs[3] model), {n_blocks} blocks', n_blocks
    from diffusion_pipe_b200.qwen_image import QWEN_IMAGE_CONFIG, QwenImagePipeline
    n_blocks = a.blocks or QWEN_IMAGE_CONFIG['num_layers']
    text_len = a.text_len if a.text_len != 512 else 256
    model = QwenImagePipeline({'model': {'dtype': 'bfloat16', 'lazy_layers': True, 'transformer_config': {'num_layers': n_blocks}}}, device=device)

    def example(g):
        return {'latents': torch.randn(16, 1, a.res // 8, a.res // 8, generator=g),
                'prompt_embeds': torch.randn(text_len, 3584, generator=g).bfloat16(), 'mask': None}
    return model, example, f'Qwen-Image full fine-tune bf16, {a.res}x{a.res}, {text_len} text tokens (configs[4] model), {n_blocks} blocks', n_blocks


def seed_layers(layers):
    """every lazily built layer draws its initial weights from WEIGHT_SEED + its index in the model: the same model whatever
    the partition and whichever rank builds the layer, so the loss of the bench line must agree across --gpus 1/2/4/8"""
    import torch
    from diffusion_pipe_b200.pipe.module import LayerSpec
    for idx, spec in enumerate(layers):
        if isinstance(spec, LayerSpec):
            def build(orig=spec.build, idx=idx):
                torch.manual_seed(WEIGHT_SEED + idx)
                return orig()
            spec.build = build
    return layers


def main():
    a = parse()
    if a.impl == 'reference':
        return run_reference_arm(a)

    import torch
    import torch.distributed as tdist
    from diffusion_pipe_b200 import data_feed, ops
    from diffusion_pipe_b200.pipe import ManualPipelineModule, initialize
    from diffusion_pipe_b200.pipe import dist

    world = int(os.environ.get('WORLD_SIZE', 1))
    rank = int(os.environ.get('RANK', 0))
    local_rank = int(os.environ.get('LOCAL_RANK', 0))
    if world != a.gpus:
        if world == 1 and a.gpus > 1:
            raise SystemExit(f'--gpus {a.gpus} needs `python -m torch.distributed.run --nproc-per-node {a.gpus} bench.py ...`')
    torch.cuda.set_device(local_rank)
    device = torch.device('cuda', local_rank)
    if world > 1:
        dist.init_distributed('nccl')
    stages = a.pp or world
    if world % stages:
        raise SystemExit(f'--pp {stages} does not divide the world size {world}')
    dp = world // stages
    M, mbs = a.micro_batches, a.micro_batch_size
    fam = FAMILIES[a.family]
    # auto: the split-backward order from 2 stages up; the planner's replay gives 1.97x / 3.72x / 6.83x for 2 / 4 / 8 stages
    # against the 1F1B bounds 1.88x / 3.37x / 5.57x at 16 micro-batches (simulated, not measured on H100).
    # (2 stages x data parallel keeps the reference's 1F1B order: only that order lets the gradient all-reduce of a layer
    # start under the last backward pass)
    schedule = ('zb' if stages > 2 or (stages == 2 and dp == 1) else '1f1b') if a.schedule == 'auto' else a.schedule
    max_inflight = a.max_inflight
    if not max_inflight and stages > 1 and schedule == 'zb':
        if a.family == 'flux':
            nd_, ns_ = (int(x) for x in a.layers.split(','))
        else:
            from diffusion_pipe_b200.qwen_image import QWEN_IMAGE_CONFIG
            from diffusion_pipe_b200.wan import WAN_T2V_14B_CONFIG
            nd_, ns_ = a.blocks or (WAN_T2V_14B_CONFIG if a.family == 'wan' else QWEN_IMAGE_CONFIG)['num_layers'], 0
        max_inflight = inflight_bound(a.family, nd_, ns_, stages)

    # ---- stage partition: measured block times (Flux: double vs single), block count otherwise ----
    probe = None
    zb_costs = None
    if a.family == 'flux':
        n_double, n_single = (int(x) for x in a.layers.split(','))
        if stages > 1 and a.partition == 'time' and n_double and n_single:
            try:
                probe = probe_block_times(device, a.res, a.text_len)
                vals = [sum(probe['double']), sum(probe['single'])] + list(probe['double']) + list(probe['single'])
            except Exception as exc:       # a failed probe on one rank must not take the run down: the other ranks' numbers decide
                print(f'[rank {rank}] block-time probe failed: {exc!r}', file=sys.stderr, flush=True)
                probe, vals = None, [float('inf')] * 8
                torch.cuda.empty_cache()
            t = torch.tensor(vals, device=device, dtype=torch.float64)
            tdist.all_reduce(t, op=tdist.ReduceOp.MIN)   # every rank must derive the same split: the least disturbed measurement
            t = t.tolist()
            split, blocks_per_stage, stage_weights, zb_costs, partition_desc = split_from_probe(
                t, n_double, n_single, stages, M, max_inflight)
        else:
            split, blocks_per_stage = flop_balanced_split(n_double, n_single, stages)
            stage_weights = [max(1, b) for b in blocks_per_stage]
            partition_desc = {'method': 'equal block count (extra blocks on the earliest stages)', 'blocks_per_stage': blocks_per_stage}
    model, example, workload, n_blocks = build_family(a, device)
    if a.family != 'flux':
        split, blocks_per_stage = flop_balanced_split(n_blocks, 0, stages)
        stage_weights = [max(1, b) for b in blocks_per_stage]
        partition_desc = {'method': 'equal block count (identical blocks)', 'blocks_per_stage': blocks_per_stage}
    layers = seed_layers(model.to_layers())
    pm = ManualPipelineModule(layers=layers, num_stages=stages, partition_method='manual' if stages > 1 else 'uniform',
                              manual_partition_split=split if stages > 1 else None, loss_fn=model.get_loss_fn(),
                              dynamic_shape=True)
    cfg = {'train_micro_batch_size_per_gpu': mbs, 'gradient_accumulation_steps': M, 'gradient_clipping': 1.0, 'steps_per_print': 0,
           'pipeline_schedule': schedule, 'zb_stage_weights': stage_weights}
    if zb_costs is not None:
        cfg['zb_costs'] = zb_costs
    if max_inflight:
        cfg['zb_max_inflight'] = max_inflight
    engine, _, _, _ = initialize(model=pm, config=cfg)
    params = [p for p in pm.parameters() if p.requires_grad]
    if not a.no_optimizer:
        engine._configure_optimizer(lambda ps: torch.optim.AdamW(ps, lr=1e-5, betas=(0.9, 0.99), weight_decay=0.01,
                                                                 fused=True) if ps else None, params)
    seen, n_local = set(), 0
    for p_ in params:
        if p_.data_ptr() not in seen:
            seen.add(p_.data_ptr())
            n_local += p_.numel()
    np_t = torch.tensor([float(n_local)], device=device, dtype=torch.float64)
    if world > 1:
        tdist.all_reduce(np_t)
    n_params = np_t.item() / dp                     # one replica of the model (every stage once)

    need_data = engine.is_first_stage() or engine.is_last_stage()
    dp_rank = engine.grid.get_data_parallel_rank()

    def family_micro_batches(pinned):
        if not need_data:
            return None
        if a.family == 'flux':
            return synth_micro_batches(a, M, 1234 + dp_rank, device, pinned=pinned)
        g = torch.Generator().manual_seed(1234 + dp_rank)
        torch.manual_seed(99 + dp_rank)
        batch = data_feed.BatchedDataset.collate([example(g) for _ in range(M * mbs)])
        feats, label = model.prepare_inputs(batch)
        out = []
        for f, l in data_feed.split_batch((feats, label), M):
            mv = (lambda t: t.pin_memory()) if pinned else (lambda t: t.to(device))
            out.append((tuple(mv(t) for t in f), tuple(mv(t) for t in l)))
        return out
    dev_batches, host_batches = family_micro_batches(False), family_micro_batches(True)

    h2d_local = 0
    if need_data:
        for feats, label in host_batches:
            if engine.is_first_stage():
                h2d_local += sum(x.numel() * x.element_size() for x in feats)
            if engine.is_last_stage():
                h2d_local += sum(x.numel() * x.element_size() for x in label)
    h2d_t = torch.tensor([h2d_local], device=device, dtype=torch.float64)
    if world > 1:
        tdist.all_reduce(h2d_t)

    def step(batches, read_loss):
        engine.reset_activation_shape()
        loss = engine.train_batch(iter(batches) if batches is not None else None)
        return loss.item() if read_loss else loss

    def barrier():
        if world > 1:
            tdist.barrier()
        torch.cuda.synchronize()

    reduce_ms = []

    def timed(batches, read_loss, nsteps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        last = None
        waits = []
        for _ in range(nsteps):
            last = step(batches, read_loss)
            if engine.dp_reduce_events is not None:
                waits.append(engine.dp_reduce_events)
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=device)
        if world > 1:
            tdist.all_reduce(ms, op=tdist.ReduceOp.MAX)
        reduce_ms[:] = [x.elapsed_time(y) for x, y in waits]
        return ms.item(), float(last)

    first_loss = None
    for i in range(a.warmup):
        l0 = step(dev_batches, False)
        if i == 0:
            first_loss = l0            # loss of the untouched initial model: must be the same number for every --gpus N
    clocks = ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    launches0 = ops.LAUNCHES
    ms_dev, loss_dev = timed(dev_batches, False, a.steps)           # `value`: no per-kernel events inside
    launches = ops.LAUNCHES - launches0
    if a.dump_outputs and engine.grid.get_data_parallel_rank() == 0:
        dump_outputs(a.dump_outputs, loss_dev if engine.is_last_stage() else None, params, engine.stage_id, stages)
    exposed_reduce = sum(reduce_ms) / max(1, len(reduce_ms)) if reduce_ms else 0.0
    ms_e2e, loss_e2e = timed(host_batches, True, a.steps)
    # the same step again with a CUDA event pair around EVERY kernel launch: per-kernel time, roofline, shares (costs ~3 %)
    prof, ms_prof = None, None
    if a.profile_kernels and a.instrumented_steps > 0:
        ops.PROFILE = []
        ms_prof, _ = timed(dev_batches, False, a.instrumented_steps)
        prof, ops.PROFILE = ops.PROFILE, None
    clk = clocks.stop() if rank == 0 else None

    # data parallel: what the same gradient all-reduce costs when nothing else runs (the serial cost the overlap is hiding)
    standalone_reduce_ms = None
    if dp > 1:
        nbytes = int(2 * n_params / stages)
        chunk = torch.empty(min(nbytes // 2, 256 << 20), dtype=torch.bfloat16, device=device).zero_()
        group = engine.grid.get_data_parallel_group()
        reps = max(1, nbytes // (2 * chunk.numel()))
        tdist.all_reduce(chunk, group=group)
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            tdist.all_reduce(chunk, op=tdist.ReduceOp.AVG, group=group)
        e1.record()
        torch.cuda.synchronize()
        t = torch.tensor([e0.elapsed_time(e1)], device=device)
        tdist.all_reduce(t, op=tdist.ReduceOp.MAX)
        standalone_reduce_ms = float(t.item())
        del chunk

    samples_per_step = mbs * M * dp
    value = samples_per_step * a.steps / (ms_dev / 1000.0)
    e2e_value = samples_per_step * a.steps / (ms_e2e / 1000.0)
    lt = torch.tensor([launches], device=device, dtype=torch.float64)
    mem_t = torch.tensor([torch.cuda.max_memory_allocated(device) / 2**30], device=device, dtype=torch.float64)
    red_t = torch.tensor([exposed_reduce], device=device, dtype=torch.float64)
    if world > 1:
        tdist.all_reduce(lt)
        tdist.all_reduce(mem_t, op=tdist.ReduceOp.MAX)
        tdist.all_reduce(red_t, op=tdist.ReduceOp.MAX)
    train_tflop = fam['train_tflop'] * n_blocks / fam['blocks']

    # ---- roofline of the dominant kernel (the wgmma GEMM): algorithmic 2MNK per launch / CUDA-event duration ----
    roof = None
    busy_local = 0.0
    if prof:
        torch.cuda.synchronize()
        tot_ms = sum(s.elapsed_time(e) for s, e, _, _, _ in prof)
        busy_local = tot_ms / ms_prof if ms_prof else 0.0
        gemm_ms = sum(s.elapsed_time(e) for s, e, _, k, _ in prof if k == 'gemm')
        gemm_fl = sum(f for _, _, f, k, _ in prof if k == 'gemm')
        attn = {}
        for s_, e_, f_, k_, _t in prof:
            if k_.startswith('attn'):
                d = attn.setdefault(k_, [0.0, 0.0])
                d[0] += s_.elapsed_time(e_)
                d[1] += f_
        attn_ms = sum(v[0] for v in attn.values())
        attn_fl = sum(v[1] for v in attn.values())
        n_gemm = sum(1 for p in prof if p[3] == 'gemm')
        kind_ms = {}
        for s_, e_, f_, k_, _t in prof:
            kind_ms[k_] = kind_ms.get(k_, 0.0) + s_.elapsed_time(e_)
        kind_share = {k: round(v / (ms_prof if ms_prof else 1), 4) for k, v in sorted(kind_ms.items(), key=lambda kv: -kv[1])}
        by_shape = {}
        for s_, e_, f_, k_, tag in prof:
            if k_ == 'gemm':
                d = by_shape.setdefault(tag, [0, 0.0, 0.0])
                d[0] += 1
                d[1] += s_.elapsed_time(e_)
                d[2] += f_
        breakdown = [{'MNK_aMN_bMN_epi_acc': list(t), 'n': v[0], 'ms': round(v[1], 2), 'tflops': round(v[2] / v[1] / 1e9, 1)}
                     for t, v in sorted(by_shape.items(), key=lambda kv: -kv[1][1])[:16]]
        try:
            with open(os.path.join(tempfile.gettempdir(), f'bench_gemm_breakdown_{a.family}_rank{rank}.json'), 'w') as f:
                json.dump(breakdown, f, indent=1)
        except OSError:
            pass
        peaks = {}
        try:
            with open(os.path.join(ROOT, 'MEASURED_PEAKS.json')) as f:
                peaks = json.load(f)
        except Exception:
            pass
        peak = peaks.get('bf16_tflops_sustained', 989.0)
        achieved = gemm_fl / gemm_ms / 1e9 if gemm_ms > 0 else 0.0
        traffic = gemm_traffic_from_profile()
        roof = {'bound': 'tensor', 'kernel': 'gemm_bf16_kernel (wgmma, all epilogues/layouts)', 'achieved': achieved,
                'peak': peak, 'peak_source': 'MEASURED_PEAKS.json bf16_tflops_sustained' if peaks else 'H100 SXM data sheet, dense bf16 at 700 W',
                'peak_measured_at_sm_mhz': (peaks.get('clocks_under_load') or {}).get('sm_mhz_median'),
                'unit': 'TFLOP/s', 'frac': achieved / peak, 'traffic': traffic[0], 'traffic_source': traffic[1],
                'launches_timed': n_gemm, 'avg_launch_ms': gemm_ms / max(1, n_gemm),
                'measured_over': f'{a.instrumented_steps} instrumented step(s) after the timed region ({ms_prof / a.instrumented_steps:.1f} ms/step; '
                                 f'the timed region itself carries no per-kernel events: {ms_dev / a.steps:.1f} ms/step)',
                'share_of_step': gemm_ms / (ms_prof if ms_prof else 1),
                'attention': {'achieved': attn_fl / attn_ms / 1e9 if attn_ms > 0 else None, 'unit': 'TFLOP/s (algorithmic: 4LqLkD fwd, 2.5x bwd)',
                              'share_of_step': attn_ms / (ms_prof if ms_prof else 1),
                              'by_kernel': {k: round(v[1] / v[0] / 1e9, 1) for k, v in attn.items() if v[0] > 0}},
                'kernels_share_of_step': tot_ms / (ms_prof if ms_prof else 1), 'share_by_kernel': kind_share,
                'step_tflops_per_gpu': train_tflop * value / max(1, world)}

    # kernel-busy fraction of every rank (instrumented kernels / step time): separates pipeline bubbles from imbalance
    busy_t = torch.zeros(world, device=device, dtype=torch.float64)
    busy_t[rank] = busy_local
    if world > 1:
        tdist.all_reduce(busy_t)
    stage_busy = [round(float(x), 4) for x in busy_t.tolist()]

    cpu = None
    if rank == 0 and world == 1 and not a.no_cpu_baseline and a.family == 'flux':
        del dev_batches, host_batches
        n_double, n_single = (int(x) for x in a.layers.split(','))
        vals = []
        try:
            for _ in range(3):
                vals.append(cpu_reference_sample(a.res, a.text_len, n_double, n_single))
        except Exception as exc:          # a baseline sample that fails must not take the measured line down with it
            print(f'cpu baseline sample failed: {exc!r}', file=sys.stderr, flush=True)
        if vals:
            vs = sorted(v for v, _, _ in vals)
            cpu = {'value': vs[len(vs) // 2], 'unit': 'samples/s', 'cores': vals[0][2], 'kind': 'port',
                   'sample': vals[-1][1] + f'; median of {len(vs)} sample(s)', 'min_max': [vs[0], vs[-1]]}

    link_name, schedule_name = type(engine.link).__name__, engine.pipeline_schedule

    if rank == 0:
        h2d = int(h2d_t.item())
        out = {
            'metric': fam['metric'], 'value': value,
            'unit': 'samples/s', 'n_gpus': world, 'steps': a.steps, 'warmup': a.warmup, 'ms_per_step': ms_dev / a.steps,
            'higher_is_better': True, 'scaling': 'strong' if dp == 1 else 'strong in pp, weak in dp', 'vs_baseline': None,
            'dtype': 'bf16', 'data': 'synthetic',
            'config': {'workload': workload + f', {n_params / 1e9:.2f}B parameters',
                       'global_batch': samples_per_step, 'micro_batch': mbs, 'micro_batches': M,
                       'seq_len': (4096 + a.text_len) if a.family == 'flux' else None,
                       'parallelism': f'pp{stages}' + (f' x dp{dp}' if dp > 1 else ''), 'partition': partition_desc,
                       'activation_recompute': False, 'train_tflop_per_sample': train_tflop,
                       'optimizer': 'none (diagnostic)' if a.no_optimizer else 'torch.optim.AdamW(fused) bf16, clip 1.0 (fused squared-norm kernel)',
                       'l2_flush': 'working set (>=24 GB of weights+grads per step) is far larger than the 50 MB L2',
                       'weights': f'random init, layer i seeded {WEIGHT_SEED}+i (identical model for every partition / GPU count)',
                       'stage_link': link_name, 'pipeline_schedule': schedule_name},
            'e2e': {'value': e2e_value, 'unit': 'samples/s', 'h2d_bytes_per_step': h2d, 'd2h_bytes_per_step': 4,
                    'ms_per_step': ms_e2e / a.steps, 'loss': loss_e2e},
            'gpu_launches': int(lt.item()),
            'loss': loss_dev,
            'first_step_loss': float(first_loss) if first_loss is not None else None,
            'peak_mem_gib_max_rank': round(float(mem_t.item()), 1),
            'stage_kernel_busy_frac': stage_busy,
            'clocks': clk,
        }
        if dp > 1:
            out['dp_allreduce'] = {'exposed_ms_per_step_max_rank': round(float(red_t.item()), 3),
                                   'standalone_ms_same_bytes': round(standalone_reduce_ms, 3) if standalone_reduce_ms else None,
                                   'standalone_busbw_gbs': round(2 * (dp - 1) / dp * int(2 * n_params / stages) / (standalone_reduce_ms / 1e3) / 1e9, 1) if standalone_reduce_ms else None,
                                   'overlapped_with_backward': bool(engine.dp_overlap and schedule_name != 'zb'),
                                   'layers_started_in_backward_rank0': engine.dp_early_layers,
                                   'bytes_per_rank': int(2 * n_params / stages)}
        if probe:
            out['config']['partition']['probe_ms_fwd_bwdin_bwdw'] = {k: [round(x, 3) for x in v] for k, v in probe.items()}
        if roof:
            out['roofline'] = roof
        if cpu:
            out['cpu_baseline'] = cpu
        # every value of `out` is a plain Python number by now: whatever the context measurement below does, the line prints
        library = None
        if world == 1 and not a.no_library_baseline and a.family == 'flux':
            try:
                del engine, pm, model, layers, params
                import gc
                gc.collect()
                torch.cuda.empty_cache()
                n_double, n_single = (int(x) for x in a.layers.split(','))
                library = gpu_library_sample(a.res, a.text_len, n_double, n_single, device)
            except Exception as exc:      # context only: never lose the bench line over it
                library = {'error': repr(exc)[:300]}
        if library:
            # part of the baseline leg: the same restated reference blocks as `cpu_baseline`, dispatched to the library kernels
            # of this GPU (SURVEY.md 8d) instead of the host cores
            (out['cpu_baseline'] if 'cpu_baseline' in out else out)['gpu_library'] = library
        print(json.dumps(out), flush=True)
    if world > 1:
        tdist.barrier()
        tdist.destroy_process_group()


if __name__ == '__main__':
    main()
