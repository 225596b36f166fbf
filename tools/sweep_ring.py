#!/usr/bin/env python
"""Ring-geometry sweep for the CG / laplace kernels (diagnostic knobs PHICUDA_RING_TY / PHICUDA_RING_NZC / PHICUDA_RING_R):
   python tools/sweep_ring.py 256 512x512x64 ... [--ty=2,4] [--nzc=1,2] [--r=4,5]
prints us per CG iteration for every (TY, NZC, ring depth) combination.  Defaults: TY auto,2,4,8,16, NZC auto,1,2,4, depth auto
('auto' = ring_config's choice; a TY whose stage does not fit falls back to a smaller one, a depth outside the fit is ignored)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
shapes = [a for a in sys.argv[1:] if a[0].isdigit()] or ['256', '512x512x64']
knobs = {'ty': ('', '2', '4', '8', '16'), 'nzc': ('', '1', '2', '4'), 'r': ('',)}
for a in sys.argv[1:]:
    for k in knobs:
        if a.startswith(f'--{k}='):
            knobs[k] = tuple('' if v == 'auto' else v for v in a.split('=', 1)[1].split(','))
passthrough = [a for a in sys.argv[1:] if a.startswith('--') and a.split('=', 1)[0][2:] not in knobs]
for shape in shapes:
    for ty in knobs['ty']:
        for nzc in knobs['nzc']:
            for r in knobs['r']:
                env = dict(os.environ)
                for name, v in (('PHICUDA_RING_TY', ty), ('PHICUDA_RING_NZC', nzc), ('PHICUDA_RING_R', r)):
                    if v:
                        env[name] = v
                out = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'microbench.py'), shape, '--ring-only'] + passthrough,
                                     env=env, capture_output=True, text=True)
                line = [l for l in out.stdout.splitlines() if l.startswith('n=')]
                print(f"TY={ty or 'auto':4s} NZC={nzc or 'auto':4s} R={r or 'auto':4s} {line[-1] if line else out.stderr[-300:]}", flush=True)
