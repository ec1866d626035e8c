"""Build cpp_functions.so (the CUDA engine behind the reference's ctypes boundary) in-tree with nvcc.

    python -m porechop_b200.build            # builds porechop_b200/cpp_functions.so for sm_90a (H100)

The file name and location mirror the reference (porechop/cpp_functions.so next to
cpp_function_wrappers.py, Makefile:24 / cpp_function_wrappers.py:21-25 of the reference).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
TARGET = os.path.join(HERE, 'cpp_functions.so')
SOURCES = [os.path.join(CSRC, 'engine.cu')]
HOSTPACK = os.path.join(CSRC, 'hostpack.cpp')       # host half of the packed upload path: plain C++ (g++, AVX-512 / AVX2, own thread team)
DEPS = SOURCES + [HOSTPACK, os.path.join(CSRC, 'kernels.cuh'), os.path.join(CSRC, 'dp_core.cuh'),
                  os.path.join(os.path.dirname(HERE), 'include', 'porechop_b200.h')]


def nvcc_path():
    for cand in (os.environ.get('NVCC'), shutil.which('nvcc'), '/usr/local/cuda/bin/nvcc'):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError('nvcc not found')


def needs_build():
    if not os.path.exists(TARGET):
        return True
    t = os.path.getmtime(TARGET)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return TARGET
    obj = os.path.join(CSRC, 'hostpack.o')
    r = subprocess.run([shutil.which('g++') or 'g++', '-O3', '-std=c++17', '-fPIC', '-pthread', '-Wall', '-Wextra', '-c', '-o', obj,
                        HOSTPACK], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('g++ failed on hostpack.cpp:\n' + r.stdout + r.stderr)
    cmd = [nvcc_path(), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
           '-Xcompiler', '-fPIC', '-shared', '-o', TARGET] + os.environ.get('PB200_NVCC_FLAGS', '').split() + SOURCES + \
          [obj, '-lpthread', '-ldl']
    if verbose:
        cmd.insert(1, '-Xptxas')
        cmd.insert(2, '-v')
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed:\n' + ' '.join(cmd) + '\n' + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return TARGET


HOSTIO_TARGET = os.path.join(HERE, 'libhostio.so')
HOSTIO_DEPS = [os.path.join(CSRC, 'hostio.c'), os.path.join(os.path.dirname(HERE), 'include', 'porechop_b200_io.h')]


def build_hostio(force=False):
    """libhostio.so: the host-side FASTQ ingest / emit helpers (plain C + OpenMP, gcc; no CUDA)."""
    if not force and os.path.exists(HOSTIO_TARGET) and \
            all(os.path.getmtime(d) <= os.path.getmtime(HOSTIO_TARGET) for d in HOSTIO_DEPS):
        return HOSTIO_TARGET
    base = [shutil.which('gcc') or 'gcc', '-O3', '-fPIC', '-shared', '-std=c11', '-Wall', '-Wextra', '-Wno-unknown-pragmas',
            '-o', HOSTIO_TARGET, HOSTIO_DEPS[0]]
    omp, zl = ['-fopenmp'], ['-DPBIO_HAVE_ZLIB', '-lz']
    # preferred: OpenMP + zlib; a gcc without libgomp / zlib headers still builds it (single-threaded / Python gzip)
    for extra_front, extra_back in ((omp, zl), (omp, []), ([], zl), ([], [])):
        cmd = base[:2] + extra_front + [x for x in extra_back if x.startswith('-D')] + base[2:] + [x for x in extra_back if x.startswith('-l')]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode == 0:
            return HOSTIO_TARGET
    raise RuntimeError('gcc failed:\n' + ' '.join(cmd) + '\n' + r.stdout + r.stderr)


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
    print(build_hostio(force='--force' in sys.argv))
