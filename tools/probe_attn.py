"""GPU bring-up probe for the attention kernels: accuracy against fp32 PyTorch and timing, one JSON record per case."""
import argparse
import json
import math
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from probe_gemm import _err  # noqa: E402

def ref_attn(q, k, v, scale):
    import torch
    s = torch.einsum('bhqd,bhkd->bhqk', q.float(), k.float()) * scale
    lse = torch.logsumexp(s, dim=-1)
    p = torch.softmax(s, dim=-1)
    o = torch.einsum('bhqk,bhkd->bhqd', p, v.float())
    return o, lse, p


def run_case(name):
    import torch
    from diffusion_pipe_b200 import ops
    torch.manual_seed(0)
    dev = 'cuda'
    res = {'case': name}
    parts = name.split(':')
    kind = parts[0]
    B, H, Lq, Lk = [int(x) for x in parts[1].split('x')]
    scale = 128 ** -0.5
    if kind == 'fwd':
        q = torch.randn(B, H, Lq, 128, device=dev).bfloat16()
        k = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        v = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        if len(parts) > 2 and parts[2] == 'peaky':   # large logits: exercises the lazy-rescale path
            q = q * 6
        o, lse = ops.attn_fwd(q, k, v)
        torch.cuda.synchronize()
        oref, lseref, _ = ref_attn(q, k, v, scale)
        res['lse'] = _err(lse * math.log(2.0), lseref)
        res.update(_err(o.view(B, Lq, H, 128).permute(0, 2, 1, 3).reshape(-1, 128), oref.reshape(-1, 128)))
    elif kind in ('bwd', 'perfbwd'):
        q = torch.randn(B, H, Lq, 128, device=dev).bfloat16()
        k = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        v = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        ld = H * 128 + (64 if kind == 'bwd' else 0)      # exercise a padded leading dimension
        o = torch.zeros(B * Lq, ld, device=dev, dtype=torch.bfloat16)
        d_o = (torch.randn(B * Lq, ld, device=dev) * 0.5).bfloat16()
        _, lse = ops.attn_fwd(q, k, v, out=o)
        dq, dk, dv = ops.attn_bwd(q, k, v, o, d_o, lse)
        torch.cuda.synchronize()
        if kind == 'bwd':
            qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
            oref, _, _ = ref_attn(qf, kf, vf, scale)
            g = d_o[:, :H * 128].float().view(B, Lq, H, 128).permute(0, 2, 1, 3)
            oref.backward(g)
            res['dq'] = _err(dq.reshape(-1, 128), qf.grad.reshape(-1, 128))
            res['dk'] = _err(dk.reshape(-1, 128), kf.grad.reshape(-1, 128))
            res.update(_err(dv.reshape(-1, 128), vf.grad.reshape(-1, 128)))
            res['ok_all'] = all(res[x]['rel'] < 2e-2 and res[x]['bad_frac'] == 0 for x in ('dq', 'dk'))
        else:
            flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
            delta = torch.empty(B, H, Lq, device=dev)

            def ours():
                ops.attn_bwd(q, k, v, o, d_o, lse, dq=dq, dk=dk, dv=dv, delta=delta)
            ts = []
            for it in range(8):
                flush.zero_()
                s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
                s.record(); ours(); e.record(); torch.cuda.synchronize()
                if it >= 3:
                    ts.append(s.elapsed_time(e))
            ts.sort()
            t = ts[len(ts) // 2]
            fl = 2.5 * 4.0 * B * H * Lq * Lk * 128    # algorithmic backward = 2.5x forward (5 tile GEMMs)
            res['ours_ms'] = t; res['ours_tflops_algorithmic'] = fl / t / 1e9
            try:
                from flash_attn import flash_attn_func
                qf, kf, vf = (x.transpose(1, 2).contiguous().requires_grad_(True) for x in (q, k, v))
                of = flash_attn_func(qf, kf, vf)
                gof = torch.randn_like(of)
                ts = []
                for it in range(8):
                    flush.zero_()
                    s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
                    s.record(); of.backward(gof, retain_graph=True); e.record(); torch.cuda.synchronize()
                    if it >= 3:
                        ts.append(s.elapsed_time(e))
                ts.sort()
                res['fa2_bwd_ms'] = ts[len(ts) // 2]; res['fa2_bwd_tflops'] = fl / ts[len(ts) // 2] / 1e9
            except Exception as ex:  # noqa
                res['fa2_err'] = repr(ex)[:200]
            # torch SDPA backward: the library path diffusers' Flux / Qwen attention processors dispatch to (cuDNN or flash)
            for name, backend in (('cudnn', 'CUDNN_ATTENTION'), ('flash', 'FLASH_ATTENTION')):
                try:
                    from torch.nn.attention import SDPBackend, sdpa_kernel
                    qs, ks, vs = (x.clone().requires_grad_(True) for x in (q, k, v))
                    with sdpa_kernel(getattr(SDPBackend, backend)):
                        osd = torch.nn.functional.scaled_dot_product_attention(qs, ks, vs)
                        gos = torch.randn_like(osd)
                        ts = []
                        for it in range(8):
                            flush.zero_()
                            s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
                            s.record(); osd.backward(gos, retain_graph=True); e.record(); torch.cuda.synchronize()
                            if it >= 3:
                                ts.append(s.elapsed_time(e))
                    ts.sort()
                    res[f'sdpa_{name}_bwd_ms'] = ts[len(ts) // 2]; res[f'sdpa_{name}_bwd_tflops'] = fl / ts[len(ts) // 2] / 1e9
                except Exception as ex:  # noqa
                    res[f'sdpa_{name}_err'] = repr(ex)[:200]
            res['rel'] = 0.0; res['bad_frac'] = 0.0
    elif kind == 'perf':
        q = torch.randn(B, H, Lq, 128, device=dev).bfloat16()
        k = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        v = torch.randn(B, H, Lk, 128, device=dev).bfloat16()
        o = torch.empty(B * Lq, H * 128, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(B, H, Lq, device=dev)
        flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

        def ours():
            ops.attn_fwd(q, k, v, out=o, lse=lse)

        def sdpa():
            torch.nn.functional.scaled_dot_product_attention(q, k, v)

        def timeit(fn, iters=10):
            for _ in range(3):
                fn()
            ts = []
            for _ in range(iters):
                flush.zero_()
                s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
                s.record(); fn(); e.record(); torch.cuda.synchronize()
                ts.append(s.elapsed_time(e))
            ts.sort()
            return ts[len(ts) // 2]
        fl = 4.0 * B * H * Lq * Lk * 128
        t = timeit(ours)
        res['ours_ms'] = t; res['ours_tflops'] = fl / t / 1e9
        t = timeit(sdpa)
        res['sdpa_ms'] = t; res['sdpa_tflops'] = fl / t / 1e9
        try:
            from flash_attn import flash_attn_func
            qf, kf, vf = (x.transpose(1, 2).contiguous() for x in (q, k, v))
            t = timeit(lambda: flash_attn_func(qf, kf, vf))
            res['fa2_ms'] = t; res['fa2_tflops'] = fl / t / 1e9
        except Exception as ex:  # noqa
            res['fa2_err'] = repr(ex)[:200]
        ours(); torch.cuda.synchronize()
        oref = torch.nn.functional.scaled_dot_product_attention(q, k, v)
        res.update(_err(o.view(B, Lq, H, 128).permute(0, 2, 1, 3).reshape(-1, 128), oref.reshape(-1, 128)))
    torch.cuda.synchronize()
    res['ok'] = bool(res.get('rel', 1) < 2e-2 and not res.get('nan', False) and res.get('bad_frac', 1) == 0)
    return res


CASES = ['fwd:1x2x256x256', 'fwd:2x3x512x384', 'fwd:1x2x300x200', 'fwd:1x2x1024x1024:peaky', 'fwd:1x1x128x640',
         'bwd:1x2x256x256', 'bwd:2x3x512x384', 'bwd:1x2x300x200', 'bwd:1x1x128x640',
         'perf:1x24x4608x4608', 'perf:1x40x9216x9216']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--case')
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'probe_attn.json'), help='JSON file the records are written to')
    a = ap.parse_args()
    if a.case:
        try:
            r = run_case(a.case)
        except Exception as ex:  # noqa
            r = {'case': a.case, 'ok': False, 'exception': repr(ex)[:500]}
        print('RESULT ' + json.dumps(r))
        return
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    results = []
    for c in CASES:
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, __file__, '--case', c], capture_output=True, text=True, timeout=240)
            line = [l for l in p.stdout.splitlines() if l.startswith('RESULT ')]
            r = json.loads(line[-1][7:]) if line else {'case': c, 'ok': False, 'rc': p.returncode,
                                                        'stderr': p.stderr[-800:], 'stdout': p.stdout[-600:]}
        except subprocess.TimeoutExpired:
            r = {'case': c, 'ok': False, 'timeout': True}
        r['secs'] = round(time.time() - t0, 1)
        results.append(r)
        print(json.dumps(r), flush=True)
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)
    print(f'probe_attn: {sum(1 for r in results if not r.get("ok"))} failing of {len(results)}')


if __name__ == '__main__':
    main()
