"""GPU tier: the REFERENCE'S OWN unittest suite (test/*.py, 85 CLI-level tests, SURVEY.md section 4) against the drop-ins
running on the real CUDA engine (`--engine cuda`), with the unmodified reference CLI on its own C++ as the baseline --
VERDICT r1 item 7 / north star "bit-identical trim/split coordinates on test/*.fastq" through the real CLI.

The suite runs from baseline/_ref, the unmodified reference tree staged by `make -C oracle stage` from a Porechop
checkout (PORECHOP_REFERENCE; git-ignored, see oracle/Makefile); without it the test is skipped.

  patch  (python -m porechop_b200)            every one of the 85 tests has the baseline's outcome -- including the three
                                              tests that fail against the reference itself at this commit (SURVEY 0.10)
  flat   (python -m porechop_b200.flat_cli)   identical except for tests that assert on the progress report text
"""
import os
import sys

import pytest

from helpers import ROOT

pytestmark = pytest.mark.gpu
REF = os.path.join(ROOT, 'baseline', '_ref')
KNOWN_FAILING = ['test_albacore_directory.TestAlbacoreDirectory.test_albacore_directory_3',
                 'test_albacore_directory.TestAlbacoreDirectory.test_albacore_directory_all',
                 'test_albacore_directory.TestAlbacoreDirectory.test_albacore_directory_unclassified']


def test_reference_unittest_suite_on_the_cuda_engine_matches_the_baseline():
    if not (os.path.isdir(os.path.join(REF, 'test')) and os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'cpp_functions.so'))):
        pytest.skip('baseline/_ref not staged (make -C oracle stage with PORECHOP_REFERENCE set)')
    sys.path.insert(0, os.path.join(ROOT, 'tests', 'refsuite'))
    try:
        import run_reference_suite as R
    finally:
        sys.path.pop(0)
    from test_reference_suite import REPORT_TESTS
    jobs = max(2, min(16, (os.cpu_count() or 2) // 2))
    base = R.run_mode('reference', 'oracle', REF, '', jobs)
    assert len(base) == 85
    assert sorted(k for k, v in base.items() if v != 'ok') == KNOWN_FAILING
    # the two drop-ins run side by side (85 CLI-level tests each; most of the time is process start + CUDA context creation)
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(2) as ex:
        f_patch = ex.submit(R.run_mode, 'patch', 'cuda', REF, '', max(1, jobs // 2))
        f_flat = ex.submit(R.run_mode, 'flat', 'cuda', REF, '', max(1, jobs // 2))
        patch, flat = f_patch.result(), f_flat.result()
    assert patch == base, sorted(k for k in base if patch.get(k) != base[k])
    assert sorted(flat) == sorted(base)
    differs = {k for k in base if flat[k] != base[k]}
    assert differs <= REPORT_TESTS, sorted(differs - REPORT_TESTS)
