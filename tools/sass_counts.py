"""SASS mnemonic counts per kernel of the shipped library (profiles/rN_sass_counts.txt):
    python tools/sass_counts.py [phiflow_b200/lib/libphicuda.so] > profiles/r2_sass_counts.txt
UBLKCP = TMA-engine bulk copies (cp.async.bulk), SYNCS = mbarrier operations, LDS.128 / LDG.E.128 / STG.E.128 = 16-byte accesses,
SHFL = warp shuffles, MEMBAR/FENCE = system- or gpu-scope fences, ATOM/RED = atomics, FP32 = single-precision ALU instructions
(FFMA, FADD, FMUL, FSETP, FMNMX, FCHK, MUFU; static count over the whole function)."""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'phiflow_b200', 'lib', 'libphicuda.so')
sass = subprocess.run(['cuobjdump', '-sass', lib], capture_output=True, text=True, check=True).stdout
COLS = [('lines', None), ('UBLKCP', r'\bUBLKCP'), ('SYNCS', r'\bSYNCS'), ('LDS.128', r'\bLDS\S*\.128'), ('LDG', r'\bLDG'), ('LDG.128', r'\bLDG\S*\.128'),
        ('STG.128', r'\bSTG\S*\.128'), ('SHFL', r'\bSHFL'), ('FENCE', r'\b(MEMBAR|FENCE)'), ('ATOM', r'\b(ATOM|RED)\b|\b(ATOMG|ATOMS|REDG)'), ('BAR', r'\bBAR\.'),
        ('FP32', r'\b(FFMA|FADD|FMUL|FSETP|FMNMX|FCHK|MUFU)\b')]
counts, name = collections.OrderedDict(), None
for line in sass.splitlines():
    m = re.match(r'\s*Function : (\S+)', line)
    if m:
        name = m.group(1)
        counts[name] = collections.Counter()
        continue
    if name is None or not re.match(r'\s*/\*[0-9a-f]{4,}\*/\s+\S', line):
        continue
    counts[name]['lines'] += 1
    for col, pat in COLS[1:]:
        if re.search(pat, line):
            counts[name][col] += 1
demangled = subprocess.run(['cu++filt'] + list(counts), capture_output=True, text=True).stdout.splitlines()
print('# ' + ' '.join(f'{c:>8s}' for c, _ in COLS) + '  kernel   (' + os.path.relpath(lib, ROOT) + ', sm_90a)')
for (mangled, c), nice in zip(counts.items(), demangled):
    print('  ' + ' '.join(f'{c[col]:8d}' for col, _ in COLS) + '  ' + (nice[:nice.index('>(') + 1] if '>(' in nice else nice.split('(')[0]).replace('(int)', '').replace('(bool)', ''))
