"""Copy the unmodified reference package (cmusatyalab/mega-nerf: `mega_nerf/` and `scripts/`) to the git-ignored oracle/_ref/.

The reference is a plain source tree without setup.py / pyproject.toml, so the copy is what an install would produce.  Source
directory: $MEGA_NERF_REFERENCE, a checkout of the reference repository (default /root/reference).  Where it does not exist, an existing oracle/_ref/ is kept and
nothing else happens: bench.py's reference legs then fall back to the oracle port, and the tests that drive the reference's own
Runner / loader skip.  Nothing under mega_nerf_b200/ imports the copy."""
from __future__ import annotations

import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get('MEGA_NERF_REFERENCE', '/root/reference')
DST = os.path.join(HERE, '_ref')


def make(force: bool = False) -> str | None:
    src = os.path.join(SRC, 'mega_nerf')
    if not os.path.isdir(src):
        return DST if os.path.isdir(os.path.join(DST, 'mega_nerf')) else None
    dst = os.path.join(DST, 'mega_nerf')
    if os.path.isdir(dst) and not force:
        return DST
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    os.makedirs(DST)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    # the two scripts of the hot path's callers that tests drive (cluster masks, container merge) live outside the package
    sdir = os.path.join(SRC, 'scripts')
    if os.path.isdir(sdir):
        shutil.copytree(sdir, os.path.join(DST, 'scripts'), ignore=shutil.ignore_patterns('__pycache__', '*.pyc'))
    return DST


if __name__ == '__main__':
    print(make(force='--force' in sys.argv))
