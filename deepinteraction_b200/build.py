"""Build libdi_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m deepinteraction_b200.build [--force]

The library is compiled for sm_90a ONLY (-gencode arch=compute_90a,code=sm_90a): there is no
other backend and no CPU fallback.  nvcc cross-compiles without a GPU.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libdi_b200.so')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr']


def sources():
    return sorted(glob.glob(os.path.join(CSRC, '*.cu')))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, '*.cuh')) + glob.glob(os.path.join(HERE, '..', 'include', '*.h'))
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=True):
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get('NVCC', 'nvcc')
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, 'build', os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ['-I', os.path.join(HERE, '..', 'include'), '-c', src, '-o', obj]
        if verbose:
            print(' '.join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd)))
    for src, p in procs:
        if p.wait() != 0:
            raise RuntimeError(f'nvcc failed on {src}')
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-cudart', 'static']
    if verbose:
        print(' '.join(cmd), flush=True)
    subprocess.check_call(cmd)
    return LIB


if __name__ == '__main__':
    build(force='--force' in sys.argv)
    print(LIB)
