#!/usr/bin/env python3
"""Stand-in for the reference's porechop-runner.py while ITS OWN unittest suite runs (tests/refsuite/run_reference_suite.py
copies this file next to a copy of the reference's test/).  TEST INFRASTRUCTURE ONLY.

PB200_SUITE_MODE   reference  the unmodified CLI on the reference's own C++ (oracle/_ref/cpp_functions.so) -- the baseline
                   patch      the unmodified CLI with porechop_b200.patch installed (phases prefetched as batches)
                   flat       porechop_b200.flat_cli (flat-buffer data path, Porechop's own parser / policy)
PB200_SUITE_ENGINE oracle     (CPU container) the C restatement stands in for the CUDA engine -- checker only
                   sim        (CPU container) the product's own engine.cu + kernels.cuh in the host simulation (tests/sim)
                   cuda       the real engine (GPU box with a reference checkout)
"""
import ctypes
import os
import sys
import types
import warnings

warnings.simplefilter('ignore')
REPO = os.environ['PB200_SUITE_REPO']
REF = os.environ['PB200_SUITE_REF']
mode = os.environ.get('PB200_SUITE_MODE', 'reference')
engine = os.environ.get('PB200_SUITE_ENGINE', 'oracle')
sys.path[:0] = [REPO, os.path.join(REPO, 'tests')]


def ref_adapter_alignment():
    lib = ctypes.CDLL(os.path.join(REPO, 'oracle', '_ref', 'cpp_functions.so'))
    lib.adapterAlignment.argtypes = [ctypes.c_char_p, ctypes.c_char_p] + [ctypes.c_int] * 4
    lib.adapterAlignment.restype = ctypes.c_void_p
    lib.freeCString.argtypes = [ctypes.c_void_p]

    def adapter_alignment(read_sequence, adapter_sequence, scoring_scheme_vals):
        p = lib.adapterAlignment(read_sequence.encode(), adapter_sequence.encode(), *scoring_scheme_vals)
        s = ctypes.cast(p, ctypes.c_char_p).value.decode()
        lib.freeCString(p)
        return s
    return adapter_alignment


stub = types.ModuleType('porechop.cpp_function_wrappers')
if mode == 'reference':
    stub.adapter_alignment = ref_adapter_alignment()
else:
    if engine == 'sim':
        sys.path.insert(0, os.path.join(REPO, 'tests', 'sim'))
        import sim_engine
        import porechop_b200
        W = sim_engine.load()
        sys.modules['porechop_b200.cpp_function_wrappers'] = W        # patch.py / fastq.py / flat_cli.py bind this module
        porechop_b200.cpp_function_wrappers = W
    else:
        from porechop_b200 import cpp_function_wrappers as W
    if engine == 'oracle':
        import numpy as np
        from helpers import oracle_batch, oracle_string
        W.adapter_alignment_batch = lambda sb, so, ab, ao, sc, ps=None, pa=None, out=None: oracle_batch(
            np.asarray(sb), np.asarray(so), np.asarray(ab), np.asarray(ao), list(sc), ps, pa)
        W.adapter_alignment = lambda r, a, sc: oracle_string(r, a, list(sc))
    stub.adapter_alignment = lambda r, a, sc: W.adapter_alignment(r, a, sc)
sys.path.insert(0, REF)
import porechop                                           # noqa: E402
sys.modules['porechop.cpp_function_wrappers'] = stub
from porechop import porechop as cli                      # noqa: E402

if __name__ == '__main__':
    if mode == 'flat':
        from porechop_b200 import flat_cli
        flat_cli.main()
    elif mode == 'patch':
        from porechop_b200 import patch
        memo = patch.install(porechop)
        try:
            cli.main()
        finally:
            patch.uninstall(memo)
    else:
        cli.main()
