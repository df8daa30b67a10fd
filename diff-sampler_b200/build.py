"""Build libdiffsampler_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libdiffsampler_b200.so')
SOURCES = ['gemm_tc.cu', 'attention.cu', 'elementwise.cu', 'solver.cu', 'optimal.cu', 'inception.cu', 'clip.cu', 'prdc.cu', 'engine.cu']
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17',
                     '-Xcompiler', '-fPIC', '--use_fast_math' if False else '-DDSB_NO_FAST_MATH']


def _newest_src_mtime():
    m = 0.0
    for root, _, files in os.walk(CSRC):
        for f in files:
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    m = max(m, os.path.getmtime(os.path.join(HERE, '..', 'include', 'diffsampler_b200.h')))
    return m


def build(force=False, verbose=False):
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= _newest_src_mtime():
        return OUT
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    objs, procs = [], []
    for src in SOURCES:                  # independent translation units: compile them concurrently
        obj = os.path.join(CSRC, src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + ['-c', os.path.join(CSRC, src), '-o', obj]
        if verbose:
            print(' '.join(cmd))
        procs.append((subprocess.Popen(cmd), cmd))
        objs.append(obj)
    for proc, cmd in procs:
        if proc.wait() != 0:
            raise subprocess.CalledProcessError(proc.returncode, cmd)
    cmd = [nvcc, '-shared', '-o', OUT] + objs + ARCH + ['-ldl']
    if verbose:
        print(' '.join(cmd))
    subprocess.check_call(cmd)
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose=True))
