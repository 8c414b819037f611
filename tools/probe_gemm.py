"""GPU bring-up probe for the wgmma GEMM:

    python tools/probe_gemm.py            # runs every case, each in its own subprocess
    python tools/probe_gemm.py --case NAME

Writes probe_gemm.json in the temp directory (--out).  Each case compares against torch (fp32 math on the same bf16 inputs).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _err(out, ref):
    import torch
    out = out.float()
    ref = ref.float()
    d = (out - ref).abs()
    scale = ref.abs().max().item() + 1e-12
    bad = (d > 0.02 * scale + 0.02 * ref.abs())
    info = {
        'max_abs': d.max().item(), 'ref_max': scale, 'rel': d.max().item() / scale,
        'bad_frac': bad.float().mean().item(), 'nan': bool(torch.isnan(out).any().item()),
    }
    if bad.any() and out.dim() == 2:
        idx = bad.nonzero()[:6].tolist()
        info['first_bad'] = idx
        info['bad_rows_mod128'] = sorted(set((bad.nonzero()[:, 0] % 128).tolist()))[:16]
        info['bad_cols_mod256'] = sorted(set((bad.nonzero()[:, 1] % 256).tolist()))[:16]
    return info


def run_case(name):
    import torch
    from diffusion_pipe_b200 import ops, _lib
    torch.manual_seed(0)
    dev = 'cuda'
    res = {'case': name}
    parts = name.split(':')
    kind = parts[0]
    cg = int(parts[1])
    if kind in ('nt', 'nn', 'tt'):
        M, N, K = [int(x) for x in parts[2].split('x')]
        A = torch.randn(M, K, device=dev).bfloat16()
        B = torch.randn(N, K, device=dev).bfloat16()
        ref = A.float() @ B.float().t()
        if kind == 'nt':
            out = ops.gemm(A, B, cta_group=cg)
        elif kind == 'nn':   # dgrad layout: B stored [K,N]
            out = ops.gemm(A, B.t().contiguous(), b_mn=True, cta_group=cg)
        else:                # wgrad layout: both stored [K, *]
            out = ops.gemm(A.t().contiguous(), B.t().contiguous(), a_mn=True, b_mn=True, cta_group=cg)
        torch.cuda.synchronize()
        res.update(_err(out, ref))
    elif kind == 'acc':
        M, N, K = 384, 512, 256
        A = torch.randn(M, K, device=dev).bfloat16()
        B = torch.randn(N, K, device=dev).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16()
        old = torch.randn(M, N, device=dev).bfloat16()
        out = old.clone()
        ops.gemm(A, B, out=out, bias=bias, accumulate=True, cta_group=cg)
        ref = A.float() @ B.float().t() + bias.float() + old.float()
        res.update(_err(out, ref))
    elif kind == 'gelu':
        M, N, K = 384, 512, 256
        A = torch.randn(M, K, device=dev).bfloat16()
        B = (torch.randn(N, K, device=dev) * 0.1).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16()
        u = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        h = ops.gemm(A, B, bias=bias, epilogue=_lib.EPI_BIAS_GELU, out2=u, cta_group=cg)
        uref = (A.float() @ B.float().t() + bias.float()).bfloat16()
        href = torch.nn.functional.gelu(uref.float(), approximate='tanh')
        res['u'] = _err(u, uref)
        res.update(_err(h, href))
    elif kind == 'gate':
        Bsz, L, N, K = 2, 192, 512, 256
        M = Bsz * L
        A = torch.randn(M, K, device=dev).bfloat16()
        B = (torch.randn(N, K, device=dev) * 0.1).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16()
        resid = torch.randn(M, N, device=dev).bfloat16()
        gate = torch.randn(Bsz, N, device=dev).bfloat16()
        y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        o = ops.gemm(A, B, bias=bias, epilogue=_lib.EPI_GATE_RES, aux=resid, gate=gate, out2=y,
                     rows_per_batch=L, cta_group=cg)
        yref = (A.float() @ B.float().t() + bias.float()).bfloat16()
        oref = resid.float() + (gate.float().repeat_interleave(L, 0) * yref.float()).bfloat16().float()
        res['y'] = _err(y, yref)
        res.update(_err(o, oref))
    elif kind == 'gelugrad':
        M, N, K = 384, 512, 256
        A = torch.randn(M, K, device=dev).bfloat16()
        Bt = (torch.randn(K, N, device=dev) * 0.1).bfloat16()   # stored [K,N]
        u = torch.randn(M, N, device=dev).bfloat16()
        o = ops.gemm(A, Bt, b_mn=True, epilogue=_lib.EPI_MUL_GELU_GRAD, aux=u, cta_group=cg)
        uf = u.float().requires_grad_(True)
        torch.nn.functional.gelu(uf, approximate='tanh').sum().backward()
        ref = (A.float() @ Bt.float()) * uf.grad
        res.update(_err(o, ref))
    elif kind == 'qkv':
        Bsz, L, H, K = 2, 160, 2, 256   # heads*128 = 256 -> N = 768 (+256 mlp columns)
        Lt_total, off = 224, 64
        mlp = 256
        N = 3 * H * 128 + mlp
        M = Bsz * L
        A = torch.randn(M, K, device=dev).bfloat16()
        W = (torch.randn(N, K, device=dev) * 0.1).bfloat16()
        bias = torch.randn(N, device=dev).bfloat16()
        wq = (1 + 0.1 * torch.randn(128, device=dev)).bfloat16()
        wk = (1 + 0.1 * torch.randn(128, device=dev)).bfloat16()
        ang = torch.rand(Lt_total, 64, device=dev) * 6.28
        cos = torch.cos(ang).repeat_interleave(2, dim=1).contiguous()
        sin = torch.sin(ang).repeat_interleave(2, dim=1).contiguous()
        shp = (Bsz, H, Lt_total, 128)
        q = torch.zeros(shp, device=dev, dtype=torch.bfloat16)
        k = torch.zeros_like(q); v = torch.zeros_like(q); qh = torch.zeros_like(q); kh = torch.zeros_like(q)
        qr = torch.zeros(Bsz, H, Lt_total, device=dev); kr = torch.zeros_like(qr)
        e = ops.make_qkv_epilogue(q, k, v, wq, wk, cos, sin, H, Lt_total, off, qh, kh, qr, kr)
        hmlp = torch.empty(M, mlp, device=dev, dtype=torch.bfloat16)
        umlp = torch.empty(M, mlp, device=dev, dtype=torch.bfloat16)
        ops.gemm(A, W, bias=bias, epilogue=_lib.EPI_QKV_ROPE, out=hmlp, out2=umlp, rows_per_batch=L,
                 cta_group=cg, qkv=e)
        torch.cuda.synchronize()
        full = (A.float() @ W.float().t() + bias.float()).bfloat16()
        qkv = full[:, :3 * H * 128].view(Bsz, L, 3, H, 128).permute(2, 0, 3, 1, 4)   # K B H L D
        def norm_rope(x, w):
            xf = x.float()
            rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6)
            xh = (xf * rstd).bfloat16()
            y = (xh * w).float()
            c = cos[off:off + L][None, None]; s = sin[off:off + L][None, None]
            yr = torch.stack([-y[..., 1::2], y[..., 0::2]], -1).flatten(-2)
            return (y * c + yr * s).bfloat16(), xh, rstd.squeeze(-1)
        qref, qhref, qrref = norm_rope(qkv[0], wq)
        kref, khref, krref = norm_rope(qkv[1], wk)
        sl = slice(off, off + L)
        res['q'] = _err(q[:, :, sl].reshape(-1, 128), qref.reshape(-1, 128))
        res['k'] = _err(k[:, :, sl].reshape(-1, 128), kref.reshape(-1, 128))
        res['v'] = _err(v[:, :, sl].reshape(-1, 128), qkv[2].reshape(-1, 128))
        res['qhat'] = _err(qh[:, :, sl].reshape(-1, 128), qhref.reshape(-1, 128))
        res['q_rstd'] = _err(qr[:, :, sl].reshape(-1, L), qrref.reshape(-1, L))
        res['untouched'] = float(q[:, :, :off].abs().max().item())
        uref = full[:, 3 * H * 128:]
        res['umlp'] = _err(umlp, uref)
        res.update(_err(hmlp, torch.nn.functional.gelu(uref.float(), approximate='tanh')))
    elif kind == 'perf':
        M, N, K = [int(x) for x in parts[2].split('x')]
        layout = parts[3] if len(parts) > 3 else 'nt'
        A = torch.randn(M, K, device=dev).bfloat16()
        B = torch.randn(N, K, device=dev).bfloat16()
        At, Bt = A.t().contiguous(), B.t().contiguous()
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

        def ours():
            if layout == 'nt':
                ops.gemm(A, B, out=out, cta_group=cg)
            elif layout == 'nn':
                ops.gemm(A, Bt, b_mn=True, out=out, cta_group=cg)
            else:
                ops.gemm(At, Bt, a_mn=True, b_mn=True, out=out, cta_group=cg)

        def cublas():
            torch.matmul(A, Bt, out=out)

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
            return ts[len(ts) // 2], ts[0]
        fl = 2.0 * M * N * K
        med, best = timeit(ours)
        res['ours_ms'] = med; res['ours_tflops'] = fl / med / 1e9; res['ours_best_tflops'] = fl / best / 1e9
        med, best = timeit(cublas)
        res['cublas_ms'] = med; res['cublas_tflops'] = fl / med / 1e9
        ours(); torch.cuda.synchronize()
        ref = A.float() @ B.float().t()
        res.update(_err(out, ref))
    else:
        raise SystemExit('unknown case ' + name)
    torch.cuda.synchronize()
    res['ok'] = bool(res.get('rel', 1) < 2e-2 and not res.get('nan', False) and res.get('bad_frac', 1) == 0)
    return res


CASES = []
for cg in (1, 2):
    CASES += [f'nt:{cg}:512x768x512', f'nt:{cg}:300x264x200', f'nn:{cg}:512x768x512', f'nn:{cg}:300x264x200',
              f'tt:{cg}:512x768x512', f'tt:{cg}:304x264x200',
              f'acc:{cg}', f'gelu:{cg}', f'gate:{cg}', f'gelugrad:{cg}', f'qkv:{cg}']
for cg in (1, 2):
    CASES += [f'perf:{cg}:4608x12288x3072:nt', f'perf:{cg}:4608x3072x12288:nn', f'perf:{cg}:12288x3072x4608:tt',
              f'perf:{cg}:4096x9216x3072:nt', f'perf:{cg}:512x9216x3072:nt']



def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--case')
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'probe_gemm.json'), help='JSON file the records are written to')
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

    def spawn(case, env=None):
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, __file__, '--case', case], capture_output=True, text=True,
                               timeout=240, env=env)
            line = [l for l in p.stdout.splitlines() if l.startswith('RESULT ')]
            r = json.loads(line[-1][7:]) if line else {'case': case, 'ok': False, 'rc': p.returncode,
                                                        'stderr': p.stderr[-800:], 'stdout': p.stdout[-400:]}
        except subprocess.TimeoutExpired:
            r = {'case': case, 'ok': False, 'timeout': True}
        r['secs'] = round(time.time() - t0, 1)
        return r

    for c in CASES:
        r = spawn(c)
        results.append(r)
        print(json.dumps(r), flush=True)
        with open(a.out, 'w') as f:
            json.dump(results, f, indent=1)
    nfail = sum(1 for r in results if not r.get('ok'))
    print(f'probe_gemm: {len(results)} results, {nfail} failing')


if __name__ == '__main__':
    main()
