"""Builds libdpipe_b200.so (all sm_90a kernels + the C ABI) in-tree with nvcc.

    python tools/build_native.py [--force] [--verbose]

Objects go to build/ (git-ignored); the shared library lands in diffusion-pipe_b200/ next to the
Python package that loads it.  Called by __graft_entry__.build().
"""
import argparse
import concurrent.futures as cf
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'diffusion-pipe_b200', 'csrc')
OUT = os.path.join(ROOT, 'diffusion-pipe_b200', 'libdpipe_b200.so')
BUILD = os.path.join(ROOT, 'build')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-lineinfo', '-O3', '-std=c++17',
         '--expt-relaxed-constexpr', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include')]


def _newer(src, dst, deps):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(d) > t for d in [src] + deps)


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(('.cu', '.cpp')))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hdrs += [os.path.join(ROOT, 'include', f) for f in os.listdir(os.path.join(ROOT, 'include'))]
    jobs = []
    objs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(BUILD, os.path.splitext(s)[0] + '.o')
        objs.append(obj)
        if force or _newer(src, obj, hdrs):
            cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-x', 'cu', '-c', src, '-o', obj]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    with cf.ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for cmd, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(' '.join(cmd) + '\n' + r.stdout + r.stderr + '\n')
            if r.returncode != 0:
                raise RuntimeError('nvcc failed for ' + cmd[-3])
    if jobs or force or not os.path.exists(OUT):
        cmd = [NVCC, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', OUT] + objs      # (the arch also names the link stub)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError('link failed')
    return OUT


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--force', action='store_true')
    ap.add_argument('--verbose', action='store_true')
    a = ap.parse_args()
    print(build(a.force, a.verbose))
