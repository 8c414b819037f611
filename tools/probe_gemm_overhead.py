"""Fixed per-tile cost of the wgmma GEMM: time each (layout, epilogue, accumulate) the Flux blocks launch at M = 4096,
N = 3072 and K in {64, 256, 1024, 3072}, and fit t(K) = a + b * K per wave of tiles.  The intercept a is what a tile
pays besides its mainloop (prologue, pipeline fill, epilogue); the slope b is the mainloop rate.

    python tools/probe_gemm_overhead.py [--breakdown bench_gemm_breakdown_flux_rank0.json] [--out probe.json]
                                        [--dump DIR]
    python tools/probe_gemm_overhead.py --compare DIR_A DIR_B

--breakdown also times every shape of the bench's per-shape GEMM breakdown.  --dump writes every output of the K = 1024
cases to DIR, and --compare checks two such dumps (for example of two builds) for identical bits.  Times are CUDA
events over --iters launches after warm-up; the card's name, power limit and clocks are recorded next to them.
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

M, N = 4096, 3072
KS = (64, 256, 1024, 3072)
HEADS = 8                      # QKV_ROPE at N = 3072: 3 x 8 heads of 128
# (name, a_mn, b_mn, epilogue, accumulate): the GEMMs of the Flux double and single blocks
CASES = [('fwd store', 0, 0, 0, 0), ('qkv_rope', 0, 0, 3, 0), ('bias_gelu', 0, 0, 1, 0), ('gate_res', 0, 0, 2, 0),
         ('dgrad store', 0, 1, 0, 0), ('mul_gelu_grad', 0, 1, 4, 0), ('wgrad store', 1, 1, 0, 0),
         ('wgrad accumulate', 1, 1, 0, 1)]


def card():
    import torch
    info = {'name': torch.cuda.get_device_name(0), 'sms': torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info['power_limit'], info['sm_clock'], info['max_sm_clock'] = [x.strip() for x in q.split(',')]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        info['nvidia_smi'] = f'unavailable: {e}'
    return info


class Problem:
    """operands and outputs of one GEMM launch, from a fixed seed"""

    def __init__(self, m, n, k, a_mn, b_mn, epi, acc, heads=None):
        import torch
        from diffusion_pipe_b200 import ops
        g = torch.Generator(device='cuda').manual_seed(m * 7 + n * 131 + k * 1009 + epi * 17 + acc)
        r = lambda *s, sc=1.0: (torch.randn(*s, generator=g, device='cuda') * sc).bfloat16()  # noqa: E731
        A, B = r(m, k), r(n, k, sc=k ** -0.5)
        self.a = A.t().contiguous() if a_mn else A
        self.b = B.t().contiguous() if b_mn else B
        self.old = r(m, n) if acc else None
        self.kw = dict(a_mn=bool(a_mn), b_mn=bool(b_mn), epilogue=epi, bias=None if (a_mn and b_mn) else r(n),
                       out=self.old.clone() if acc else torch.empty(m, n, device='cuda', dtype=torch.bfloat16),
                       accumulate=bool(acc))
        self.outs = {'out': self.kw['out']}
        if epi in (1, 2):
            self.kw['out2'] = self.outs['out2'] = torch.empty(m, n, device='cuda', dtype=torch.bfloat16)
        if epi == 2:
            self.kw['aux'], self.kw['gate'] = r(m, n), r(1, n)
        if epi == 4:
            self.kw['aux'] = r(m, n, sc=2.0)
        if epi == 3:
            heads = heads or HEADS
            n_qkv = 3 * heads * 128
            mlp = n - n_qkv
            ang = torch.rand(m, 64, generator=g, device='cuda') * 6.28
            self.rope = (torch.cos(ang).repeat_interleave(2, 1).contiguous(),
                         torch.sin(ang).repeat_interleave(2, 1).contiguous())
            self.w = (r(128), r(128))
            for t in ('q', 'k', 'v', 'qhat', 'khat'):
                self.outs[t] = torch.empty(1, heads, m, 128, device='cuda', dtype=torch.bfloat16)
            for t in ('q_rstd', 'k_rstd'):
                self.outs[t] = torch.empty(1, heads, m, device='cuda', dtype=torch.float32)
            o = self.outs
            self.kw['qkv'] = ops.make_qkv_epilogue(o['q'], o['k'], o['v'], self.w[0], self.w[1], *self.rope, heads, m, 0,
                                                   qhat=o['qhat'], khat=o['khat'], q_rstd=o['q_rstd'],
                                                   k_rstd=o['k_rstd'])
            self.kw['rows_per_batch'] = m
            if mlp:
                self.kw['out'] = self.outs['out'] = torch.empty(m, mlp, device='cuda', dtype=torch.bfloat16)
                self.kw['out2'] = self.outs['out2'] = torch.empty(m, mlp, device='cuda', dtype=torch.bfloat16)
            else:
                del self.outs['out']
            self.kw['N'] = n

    def launch(self):
        from diffusion_pipe_b200 import ops
        ops.gemm(self.a, self.b, **self.kw)

    def time_ms(self, iters):
        import torch
        for _ in range(5):
            self.launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            self.launch()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters


def fit(ks, ts):
    n = len(ks)
    mk, mt = sum(ks) / n, sum(ts) / n
    b = sum((k - mk) * (t - mt) for k, t in zip(ks, ts)) / sum((k - mk) ** 2 for k in ks)
    return mt - b * mk, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--breakdown', default=None, help="the bench's bench_gemm_breakdown_<family>_rank0.json")
    ap.add_argument('--out', default=None)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--dump', default=None, metavar='DIR', help='save every output of the K = 1024 cases')
    ap.add_argument('--compare', nargs=2, default=None, metavar=('DIR_A', 'DIR_B'))
    a = ap.parse_args()
    import torch
    if a.compare:
        names = sorted(f for f in os.listdir(a.compare[0]) if f.endswith('.pt'))
        bad = [f for f in names if not torch.equal(torch.load(os.path.join(a.compare[0], f)).view(torch.int16),
                                                   torch.load(os.path.join(a.compare[1], f)).view(torch.int16))]
        print(json.dumps({'compared': len(names), 'differ': bad}))
        sys.exit(1 if bad or not names else 0)
    assert torch.cuda.is_available(), 'the probe times the GPU kernel: it needs a GPU'
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = math.ceil(M / 128) * math.ceil(N / 256)
    waves = math.ceil(tiles / sms)
    res = {'card': card(), 'M': M, 'N': N, 'tiles': tiles, 'waves': waves, 'iters': a.iters, 'fits': [], 'shapes': []}
    for name, a_mn, b_mn, epi, acc in CASES:
        ts = []
        for k in KS:
            p = Problem(M, N, k, a_mn, b_mn, epi, acc)
            ts.append(p.time_ms(a.iters))
            if a.dump and k == 1024:
                os.makedirs(a.dump, exist_ok=True)
                if acc:
                    p.kw['out'].copy_(p.old)
                p.launch()
                torch.cuda.synchronize()
                for t, v in p.outs.items():
                    torch.save(v.view(torch.int16).cpu(), os.path.join(a.dump, f'{name.replace(" ", "_")}_{t}.pt'))
            del p
        icpt, slope = fit(KS, ts)
        row = {'case': name, 'ms': dict(zip(KS, [round(t, 4) for t in ts])),
               'intercept_us_per_tile': round(icpt * 1e3 / waves, 2),
               'mainloop_us_per_tile_at_k3072': round(slope * 3072 * 1e3 / waves, 2),
               'tflops_k3072': round(2.0 * M * N * 3072 / ts[-1] / 1e9, 1)}
        res['fits'].append(row)
        print(json.dumps(row), flush=True)
    if a.breakdown and os.path.exists(a.breakdown):
        for ent in json.load(open(a.breakdown)):
            m, n, k, a_mn, b_mn, epi, acc = ent['MNK_aMN_bMN_epi_acc']
            heads = 24 if n >= 9216 else n // 384
            p = Problem(m, n, k, a_mn, b_mn, epi, acc, heads=heads)
            t = p.time_ms(a.iters)
            row = {'MNK_aMN_bMN_epi_acc': ent['MNK_aMN_bMN_epi_acc'], 'ms': round(t, 4),
                   'tflops': round(2.0 * m * n * k / t / 1e9, 1)}
            res['shapes'].append(row)
            print(json.dumps(row), flush=True)
            del p
    res['card_after'] = card()
    print(json.dumps(res['card']))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
