"""SASS census of the shipped library: which tensor-core / matrix-load / warp-collective / atomic instructions each kernel
contains.  python profiles/sass_census.py > census.md   (needs cuobjdump and c++filt; no GPU)

python profiles/sass_census.py --bodies: one line per kernel -- a hash of its instruction text (addresses and encodings
stripped), its instruction count and its demangled name -- to diff two builds and show which kernels a change recompiled."""
import collections
import hashlib
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'log_b200', '_lib', 'liblog_b200_raster.so')
PATS = collections.OrderedDict([
    ('HMMA (mma.sync tf32)', r'\bHMMA\.'), ('LDSM (ldmatrix)', r'\bLDSM'), ('HGMMA (wgmma)', r'\bHGMMA'),
    ('UBLKCP / UTMA (bulk / tensor copies)', r'UBLKCP|UTMA'), ('REDUX', r'\bREDUX'), ('VOTE', r'\bVOTE'), ('MATCH', r'\bMATCH'),
    ('SHFL', r'\bSHFL'), ('ATOMS / REDS (shared)', r'\bATOMS|\bREDS'), ('ATOMG (returning)', r'\bATOMG'), ('RED (global)', r'\bRED\.'),
    ('MUFU.EX2', r'MUFU\.EX2'), ('BAR', r'\bBAR\.'), ('LDG.128', r'LDG\.E\.(\w+\.)*128'), ('STG.128', r'STG\.E\.(\w+\.)*128'),
    ('CCTL (L2 prefetch)', r'\bCCTL')])


def bodies(sass):
    body, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            body[cur] = []
        elif cur:
            m = re.search(r'/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;', line)
            if m:
                body[cur].append(m.group(1))
    # enum template arguments demangle as (lgr::Colour)0: keep the whole name
    names = subprocess.run(['c++filt'], input='\n'.join(body), capture_output=True, text=True, check=True).stdout.split('\n')
    for name, ins in zip(names, body.values()):
        print(hashlib.sha256('\n'.join(ins).encode()).hexdigest()[:16], f'{len(ins):6d}', name)


def main():
    sass = subprocess.run(['cuobjdump', '-sass', LIB], capture_output=True, text=True, check=True).stdout
    if '--bodies' in sys.argv[1:]:
        return bodies(sass)
    stats, cur = collections.OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            cur = m.group(1)
            stats[cur] = collections.Counter()
        elif cur and re.search(r'/\*[0-9a-f]{4}\*/', line):
            stats[cur]['instructions'] += 1
            for k, p in PATS.items():
                if re.search(p, line):
                    stats[cur][k] += 1
    print('# SASS census of `liblog_b200_raster.so` (sm_90a), static instruction counts per kernel\n')
    print('`cuobjdump -sass` of the shipped library, grouped by `profiles/sass_census.py`. The tensor-core path is the legacy')
    print('`mma.sync.m16n8k8.tf32` (`HMMA.1688.F32.TF32`) fed by `ldmatrix` (`LDSM`) in `blend_bwd_kernel`.\n')
    print('| kernel | instructions | ' + ' | '.join(PATS) + ' |')
    print('|---|---|' + '---|' * len(PATS))
    for k, c in stats.items():
        name = subprocess.run(['c++filt', k], capture_output=True, text=True).stdout.strip().split('(')[0].replace('void ', '').replace('lgr::', '')
        print(f'| `{name}` | {c["instructions"]} | ' + ' | '.join(str(c[p]) if c[p] else '' for p in PATS) + ' |')


if __name__ == '__main__':
    main()
