"""Build recipe for libmn_b200.so (sm_90a only; the library is written next to this file)."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libmn_b200.so')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '-fmad=false',                      # parity: no implicit FMA contraction (see csrc/mn_common.cuh)
    '-Xcompiler', '-fPIC', '-shared',
    '-Xptxas', '-v',
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + [os.path.join(HERE, '..', 'include', 'mn_b200.h')]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    objs = []
    build_dir = os.path.join(HERE, 'build')
    os.makedirs(build_dir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(build_dir, os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [nvcc] + [f for f in NVCC_FLAGS if f != '-shared'] + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f'== {os.path.basename(src)}\n{out}')
        if p.returncode != 0:
            sys.stderr.write('\n'.join(log))
            raise RuntimeError(f'nvcc failed on {src}')
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError('link failed')
    with open(os.path.join(build_dir, 'ptxas.log'), 'w') as f:
        f.write('\n'.join(log))
    if verbose:
        print('\n'.join(log))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
