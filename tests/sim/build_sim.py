"""Build tests/sim/_build/libengine_sim.so: the PRODUCT'S engine.cu + kernels.cuh + dp_core.cuh + hostpack.cpp compiled
for the host against tests/sim/pbsim_cuda.h (a stand-in for the CUDA runtime and execution model).  TESTS ONLY.

The sources are taken as they are; three textual substitutions make them host C++:
    #include <cuda_runtime.h>                ->  #include "pbsim_cuda.h"
    kernel<<<grid, block, smem, stream>>>(   ->  pbsim::launch(site, kernel, grid, block, smem, stream,
    extern __shared__ uint32_t smem[];       ->  uint32_t *smem = pbsim::dynamic_smem();
    __shared__ T name[N];                    ->  static T name[N]; pbsim::poison_shared(name, sizeof(name));
(`site`: the kernel's name, argument expressions and line, for the race reports of the stream-ordering check; the
pointer fields of the kernels' argument structs are classified in pbsim_fields.h, included after kernels.cuh) and the one inline-PTX statement outside dp_core.cuh's #if __CUDA_ARCH__ branches (discard.global.L2, a cache hint) is
dropped.  Nothing else changes: the kernels' control flow, shared-memory staging, shuffles and the host engine's launch
sequences are the product's own.
"""
import hashlib
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, 'porechop_b200', 'csrc')
BUILD = os.path.join(HERE, '_build')
TARGET = os.path.join(BUILD, 'libengine_sim.so')


def _site(kernel, src, start):
    """pbsim::Site{kernel, argument expressions, function, line} of the launch whose argument list starts at src[start]:
    the stream-ordering check names the two operations of a race with it"""
    depth, args, cur = 0, [], ''
    for ch in src[start:]:
        if ch == ')' and depth == 0:
            break
        depth += ch in '([{'
        depth -= ch in ')]}'
        if ch == ',' and depth == 0:
            args.append(cur.strip()); cur = ''
        else:
            cur += ch
    args.append(cur.strip())
    text = '\\037'.join(' '.join(a.split()).replace('\\', '\\\\').replace('"', '\\"') for a in args)
    return 'pbsim::Site{"%s", "%s", __func__, __LINE__}' % (kernel, text)


def transform(src):
    src = src.replace('#include <cuda_runtime.h>', '#include "pbsim_cuda.h"')
    src, n = re.subn(r'(\b[A-Za-z_]\w*)<<<(.*?)>>>\(', lambda m: 'pbsim::launch(%s, %s, %s, ' % (
        _site(m.group(1), src, m.end()), m.group(1), m.group(2)), src, flags=re.S)
    src = src.replace('#include "kernels.cuh"', '#include "kernels.cuh"\n#include "pbsim_fields.h"')
    src = src.replace('extern __shared__ uint32_t smem[];', 'uint32_t *smem = pbsim::dynamic_smem();')
    # static shared arrays: poisoned at the start of every block (the device gives no initial value either)
    src = re.sub(r'^(\s*)__shared__\s+([^;\n]+?)\s+(\w+)((?:\[[^\n;]*\])+);',
                 lambda m: '%sstatic %s %s%s; pbsim::poison_shared(%s, sizeof(%s));' % (m.group(1), m.group(2), m.group(3), m.group(4),
                                                                                  m.group(3), m.group(3)), src, flags=re.M)
    src = re.sub(r'asm volatile\("discard\.global\.L2.*?"memory"\);', '(void)0;', src)
    return src, n


def build(force=False, flags=None):
    """the simulated engine with the product's default compile options -- or with `flags` (default: $PB200_SIM_FLAGS), extra
    -D switches of the product sources; each set of switches has its own library, so tests can load both side by side"""
    srcs = [os.path.join(CSRC, f) for f in ('engine.cu', 'kernels.cuh', 'dp_core.cuh', 'hostpack.cpp')] + \
           [os.path.join(HERE, f) for f in ('pbsim_cuda.h', 'pbsim_fields.h', 'pbsim.cpp', 'build_sim.py')] + \
           [os.path.join(ROOT, 'include', 'porechop_b200.h')]
    # PB200_SIM_FLAGS: extra -D switches of the product sources (the compile-time A/B options, e.g. -DPB_SCORE_PREFETCH); the
    # library is rebuilt whenever they differ from the ones it was built with
    flags = os.environ.get('PB200_SIM_FLAGS', '').split() if flags is None else list(flags)
    tag = ('_' + hashlib.sha1(' '.join(flags).encode()).hexdigest()[:10]) if flags else ''
    target = TARGET[:-3] + tag + '.so'
    stamp = os.path.join(BUILD, 'flags%s.txt' % tag)
    same_flags = os.path.exists(stamp) and open(stamp).read().split() == flags
    if not force and same_flags and os.path.exists(target) and all(os.path.getmtime(s) <= os.path.getmtime(target) for s in srcs):
        return target
    os.makedirs(os.path.join(BUILD, 'porechop_b200', 'csrc'), exist_ok=True)
    os.makedirs(os.path.join(BUILD, 'include'), exist_ok=True)
    launches = 0
    for f, out in (('engine.cu', 'engine_sim.cpp'), ('kernels.cuh', 'kernels.cuh'), ('dp_core.cuh', 'dp_core.cuh')):
        text, n = transform(open(os.path.join(CSRC, f)).read())
        launches += n
        with open(os.path.join(BUILD, 'porechop_b200', 'csrc', out), 'w') as o:
            o.write(text)
    assert launches >= 14, 'kernel launch sites not found'
    with open(os.path.join(BUILD, 'include', 'porechop_b200.h'), 'w') as o:
        o.write(open(os.path.join(ROOT, 'include', 'porechop_b200.h')).read())
    cmd = ['g++', '-O2', '-g', '-std=c++17', '-fPIC', '-shared', '-fopenmp', '-Wno-unknown-pragmas', '-Wno-unused-value'] + flags + \
          ['-I', HERE, '-o', target + '.tmp%d' % os.getpid(),
           os.path.join(BUILD, 'porechop_b200', 'csrc', 'engine_sim.cpp'), os.path.join(HERE, 'pbsim.cpp'),
           os.path.join(CSRC, 'hostpack.cpp')]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('g++ failed on the simulated engine:\n' + r.stdout + r.stderr[-6000:])
    os.replace(target + '.tmp%d' % os.getpid(), target)      # atomic: a concurrent loader never sees a half-written library
    with open(stamp, 'w') as o:
        o.write(' '.join(flags))
    return target


def build_asan():
    """the same sources with -fsanitize=address (portable ucontext switch: ASan cannot follow the hand-written one)"""
    build()
    target = os.path.join(BUILD, 'libengine_sim_asan.so')
    cmd = ['g++', '-O1', '-g', '-std=c++17', '-fPIC', '-shared', '-fopenmp', '-fsanitize=address', '-fno-omit-frame-pointer',
           '-DPBSIM_NO_FAST_SWITCH', '-Wno-unknown-pragmas', '-Wno-unused-value', '-I', HERE, '-o', target,
           os.path.join(BUILD, 'porechop_b200', 'csrc', 'engine_sim.cpp'), os.path.join(HERE, 'pbsim.cpp'),
           os.path.join(CSRC, 'hostpack.cpp')]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('g++ -fsanitize=address failed:\n' + r.stderr[-4000:])
    return target


if __name__ == '__main__':
    print(build(force=True))
