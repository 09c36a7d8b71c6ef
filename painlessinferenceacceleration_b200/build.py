# -*- coding: utf-8 -*-
"""In-tree build of libpia_b200.so (explicit nvcc, sm_90a only)."""
import glob
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, 'csrc')
SO = os.environ.get('PIA_B200_LIB') or os.path.join(PKG, 'libpia_b200.so')   # override: diagnostic builds
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr'] + os.environ.get('PIA_NVCC_EXTRA', '').split()


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def _stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + [os.path.join(PKG, '..', 'include', 'pia_b200.h')]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force=False, verbose=False):
    """Compile every .cu under csrc/ into one shared library. Objects are built in parallel."""
    if not force and not _stale():
        return SO
    objdir = os.path.join(PKG, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + '.o')
        cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs = []
    for src, obj, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{out}')
        if verbose and out:
            print(out)
        objs.append(obj)
    cmd = [NVCC, '-shared', '-o', SO] + objs + ['-lcudart_static', '-ldl', '-lrt', '-lpthread']
    subprocess.check_call(cmd)
    return SO


if __name__ == '__main__':
    print(build_library(force='--force' in sys.argv, verbose='-v' in sys.argv))
