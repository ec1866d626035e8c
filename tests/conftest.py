import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100); run with -m gpu on a machine that has one')


def _have_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _have_gpu():
        return
    skip = pytest.mark.skip(reason='no CUDA device in this container')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session', autouse=True)
def built():
    """Build the checker (oracle, emulation) and the product library once per session."""
    subprocess.check_call(['make', '-s', '-C', os.path.join(ROOT, 'oracle'), 'liboracle.so', 'harness', 'ref'])
    emu_src = os.path.join(ROOT, 'tests', 'emu', 'emu_group.cpp')
    emu_so = os.path.join(ROOT, 'tests', 'emu', 'libemu.so')
    core = os.path.join(ROOT, 'porechop_b200', 'csrc', 'dp_core.cuh')
    if (not os.path.exists(emu_so) or os.path.getmtime(emu_so) < max(os.path.getmtime(emu_src), os.path.getmtime(core))):
        subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-Wno-unknown-pragmas', '-o', emu_so, emu_src])
    from porechop_b200 import build
    build.build()
    build.build_hostio()
    return True
