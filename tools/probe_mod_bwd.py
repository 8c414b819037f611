"""Compares dpipe_mod_bwd (the modulation-linear backward, csrc/modulation.cu) of this build with another build of the
library, for example the previous commit's: same inputs, bit-for-bit equal outputs, and the time per call of each,
measured alternately in the same process.

    python tools/probe_mod_bwd.py --baseline-lib /path/to/other/libdpipe_b200.so [--iters 50] [--rounds 7] [--out f.json]

Shapes: the Flux / Qwen-Image AdaLN linear (N = 18432, K = 3072) at 1, 2, 5 and 8 samples and the Wan2.1-14B time
projection (N = 30720, K = 5120) at 1 and 2 samples, dW accumulated (the engine's gradient-accumulation path).
Prints one JSON line with the card's name and power limit next to the times."""
import argparse
import ctypes
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(1, 18432, 3072), (2, 18432, 3072), (5, 18432, 3072), (8, 18432, 3072), (1, 30720, 5120), (2, 30720, 5120)]


def _load(path, tmp):
    """a private copy, so that two builds of the same file name load side by side"""
    dst = os.path.join(tmp, f'lib{len(os.listdir(tmp))}.so')
    shutil.copy(path, dst)
    lib = ctypes.CDLL(dst)
    lib.dpipe_last_error.restype = ctypes.c_char_p
    lib.dpipe_mod_bwd.argtypes = [ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 3 + [ctypes.c_int] + \
        [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p]
    return lib


def main():
    import torch
    from diffusion_pipe_b200 import _lib
    ap = argparse.ArgumentParser()
    ap.add_argument('--baseline-lib', required=True)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--out')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'probe_mod_bwd needs a GPU'
    tmp = tempfile.mkdtemp()
    libs = {'baseline': _load(a.baseline_lib, tmp), 'this': _load(_lib.LIB_PATH, tmp)}
    stream = torch.cuda.current_stream()
    P = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip().splitlines()
    rows = []
    for B, N, K in SHAPES:
        g = torch.Generator(device='cuda').manual_seed(B * 131 + N + K)
        W = (torch.randn(N, K, generator=g, device='cuda') * 0.02).bfloat16()
        temb = torch.randn(B, K, generator=g, device='cuda').bfloat16()
        dmod = torch.randn(B, N, generator=g, device='cuda')
        dW0 = (torch.randn(N, K, generator=g, device='cuda') * 0.1).bfloat16()
        dtemb0 = torch.randn(B, K, generator=g, device='cuda')
        nchunk = (N + 63) // 64
        bufs = {}
        for name, lib in libs.items():
            dW, dtemb = dW0.clone(), dtemb0.clone()
            dbias, partials = torch.empty(N, device='cuda'), torch.empty(nchunk * B * K, device='cuda')
            rc = lib.dpipe_mod_bwd(P(dmod), dmod.stride(0), P(temb), P(W), P(dW), 1, P(dbias), P(partials), P(dtemb), B, N, K,
                                   ctypes.c_void_p(stream.cuda_stream))
            torch.cuda.synchronize()
            if rc != 0:
                bufs[name] = lib.dpipe_last_error().decode()
                continue
            bufs[name] = (dW, dbias, dtemb, partials)
        row = {'B': B, 'N': N, 'K': K}
        if all(isinstance(v, tuple) for v in bufs.values()):
            row['bit_identical'] = all(torch.equal(x, y) for x, y in zip(bufs['baseline'], bufs['this']))
        else:
            row['errors'] = {k: v for k, v in bufs.items() if isinstance(v, str)}
        times = {name: [] for name in libs if isinstance(bufs[name], tuple)}
        for _ in range(a.rounds):
            for name in times:
                dW, dbias, dtemb, partials = bufs[name]
                lib = libs[name]
                args = (P(dmod), dmod.stride(0), P(temb), P(W), P(dW), 1, P(dbias), P(partials), P(dtemb), B, N, K,
                        ctypes.c_void_p(stream.cuda_stream))
                for _ in range(3):
                    lib.dpipe_mod_bwd(*args)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    lib.dpipe_mod_bwd(*args)
                e1.record()
                e1.synchronize()
                times[name].append(e0.elapsed_time(e1) * 1000.0 / a.iters)
        for name, ts in times.items():
            row[f'{name}_us_median'] = round(statistics.median(ts), 2)
            row[f'{name}_us_range'] = [round(min(ts), 2), round(max(ts), 2)]
        # W and dW read, dW written: the bytes the call must move
        row['this_GBps'] = round(3 * N * K * 2 / (row.get('this_us_median', float('nan')) * 1e3), 1) if 'this' in times else None
        rows.append(row)
        del bufs, W, dW0
        torch.cuda.empty_cache()
    res = {'card': card, 'iters': a.iters, 'rounds': a.rounds, 'shapes': rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
