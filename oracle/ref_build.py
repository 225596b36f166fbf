"""
Installs an unmodified copy of the reference's tensor library (PhiML 1.7.2) into oracle/_ref (git-ignored) for the tests of the
phiml plugin `phiflow_b200/phi_cuda` on real phiml objects (tests/_phiml.py).  The source is the PhiML tree that the reference
checkout vendors (PhiFlow 3.4.0, `PhiML/`), at DEFAULT_SOURCE unless the environment variable PHIML_SOURCE names another one; where
neither exists nothing is installed and those tests skip.  The installed copy is self-contained, so the tests also run on machines
without the reference.  No network: pip installs the local tree only.
"""
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEST = os.path.join(ROOT, 'oracle', '_ref')
DEFAULT_SOURCE = '/root/reference/PhiML'


def install_reference_phiml() -> None:
    src = os.environ.get('PHIML_SOURCE') or DEFAULT_SOURCE
    if os.path.isdir(os.path.join(DEST, 'phiml')) or not os.path.isdir(os.path.join(src, 'phiml')):
        return
    with tempfile.TemporaryDirectory() as tmp:                 # the source may be read-only and the build writes into it
        copy = os.path.join(tmp, 'PhiML')
        shutil.copytree(src, copy)
        rc = subprocess.call([sys.executable, '-m', 'pip', 'install', '--no-index', '--no-build-isolation', '--no-deps', '--quiet',
                              '--no-cache-dir', '--target', DEST, copy])
    if rc != 0:  # pragma: no cover
        print('note: could not install PhiML into oracle/_ref; the phi_cuda plugin tests will be skipped', file=sys.stderr)
