"""Per-kernel SASS evidence for the sm_90a kernels: counts of the warpgroup tensor-core (HGMMA, from wgmma), TMA
(UTMALDG / UTMASTG / UBLKCP), mbarrier (SYNCS) and legacy mma.sync (HMMA)
mnemonics in every kernel of the built library, plus registers / shared memory from the ELF.  No GPU needed.

    python tools/sass_evidence.py r01        ->  profiles/r01_sass_evidence.md
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'diffusion-pipe_b200', 'libdpipe_b200.so')
R = sys.argv[1] if len(sys.argv) > 1 else 'r01'
PATTERNS = [('HGMMA (wgmma)', r'\bHGMMA'), ('WARPGROUP (wgmma fence / wait)', r'\bWARPGROUP'),
            ('UTMALDG (TMA load)', r'\bUTMALDG'), ('UTMASTG (TMA store)', r'\bUTMASTG'), ('UBLKCP', r'\bUBLKCP'),
            ('SYNCS (mbarrier)', r'\bSYNCS'), ('MUFU.EX2', r'\bMUFU\.EX2'), ('HMMA (legacy)', r'\bHMMA\b'),
            ('LDG / STG', r'\bLDG|\bSTG'), ('LDS / STS', r'\bLDS|\bSTS')]


def main():
    sass = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True, check=True).stdout
    res = subprocess.run(['cuobjdump', '-res-usage', LIB], capture_output=True, text=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.search(r'Function (\S+):', line)
        if m:
            cur = m.group(1)
        m = re.search(r'REG:(\d+).*?SHARED:(\d+)', line)
        if m and cur:
            usage[cur] = (int(m.group(1)), int(m.group(2)))
    kernels = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            kernels[cur] = collections.Counter()
            continue
        if cur is None:
            continue
        for label, pat in PATTERNS:
            if re.search(pat, line):
                kernels[cur][label] += 1
        if re.search(r'^\s+/\*[0-9a-f]{4}\*/', line):
            kernels[cur]['instructions'] += 1

    def demangle(n):
        out = subprocess.run(['c++filt', n], capture_output=True, text=True).stdout.strip() or n
        return re.sub(r'\(.*', '', out).replace('void ', '')
    os.makedirs(os.path.join(ROOT, 'profiles'), exist_ok=True)
    out = os.path.join(ROOT, 'profiles', f'{R}_sass_evidence.md')
    arch = subprocess.run(['cuobjdump', '-lelf', LIB], capture_output=True, text=True).stdout
    with open(out, 'w') as f:
        f.write(f'# {R}: SASS evidence per kernel (`cuobjdump -sass diffusion-pipe_b200/libdpipe_b200.so`, built with '
                '`-gencode arch=compute_90a,code=sm_90a`)\n\n')
        f.write('ELF images: ' + ', '.join(sorted(set(re.findall(r'sm_\d+a?', arch)))) + '\n\n')
        f.write('Counts of static instructions.  `HGMMA` = `wgmma.mma_async`, '
                '`UTMALDG`/`UTMASTG` = TMA tensor copies; `HMMA` would be the legacy `mma.sync` path (none).\n\n')
        cols = [p[0] for p in PATTERNS]
        f.write('| kernel | instr | regs | smem (static) | ' + ' | '.join(cols) + ' |\n')
        f.write('|---|---:|---:|---:|' + '---:|' * len(cols) + '\n')
        for k, c in kernels.items():
            reg, sh = usage.get(k, ('', ''))
            f.write(f'| `{demangle(k)}` | {c["instructions"]} | {reg} | {sh} | ' + ' | '.join(str(c[x]) if c[x] else '·' for x in cols) + ' |\n')
        tc = [demangle(k) for k, c in kernels.items() if c['HGMMA (wgmma)']]
        f.write(f'\nKernels issuing `wgmma`: {len(tc)} — ' + ', '.join(f'`{t}`' for t in sorted(set(tc))) + '.\n')
        f.write(f'Kernels with `HMMA`: {sum(1 for c in kernels.values() if c["HMMA (legacy)"])}.\n')
    print('wrote', out, len(kernels), 'kernels')


if __name__ == '__main__':
    main()
