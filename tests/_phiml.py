"""
Where the tests find the reference's tensor library (PhiML 1.7.2) for the plugin tests on real phiml objects: an installed `phiml`, or
the unmodified copy that `__graft_entry__.build()` installs into oracle/_ref from the reference's PhiML tree
(oracle/ref_build.py).  Without either, those tests skip.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INSTALLED = os.path.join(ROOT, 'oracle', '_ref')


def ensure_phiml() -> bool:
    try:
        import phiml  # noqa: F401
        return True
    except ImportError:
        pass
    if not os.path.isdir(os.path.join(INSTALLED, 'phiml')):
        return False
    if INSTALLED not in sys.path:
        sys.path.insert(0, INSTALLED)
    return True
