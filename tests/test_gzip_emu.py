"""The deflate pieces of dp_core.cuh (code lengths, canonical codes, dynamic header, CRC-32) compiled for the host
(tests/emu/emu_gzip.cpp) and checked against zlib.  CPU tier; the kernels that run them are tested in test_gzip_device.py."""
import ctypes
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

from helpers import ROOT
from gzip_inputs import edge_inputs, ont_fastq


@pytest.fixture(scope='module')
def emu():
    d = tempfile.mkdtemp(prefix='pb200_emu_gzip_')
    so = os.path.join(d, 'libemu_gzip.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', so, os.path.join(ROOT, 'tests', 'emu', 'emu_gzip.cpp')])
    lib = ctypes.CDLL(so)
    lib.emu_code_lengths.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.emu_crc32.argtypes = [ctypes.c_uint32, ctypes.c_char_p, ctypes.c_int64]
    lib.emu_crc32.restype = ctypes.c_uint32
    lib.emu_crc32_combine.argtypes = [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int64]
    lib.emu_crc32_combine.restype = ctypes.c_uint32
    lib.emu_deflate_block.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
    lib.emu_deflate_block.restype = ctypes.c_int64
    return lib


def _lengths(emu, freq, limit):
    f = np.ascontiguousarray(freq, dtype=np.uint32)
    out = np.zeros(len(f), dtype=np.uint8)
    emu.emu_code_lengths(f.ctypes.data, len(f), limit, out.ctypes.data)
    return out


def _fib(n):
    a, b, out = 1, 1, []
    for _ in range(n):
        out.append(a)
        a, b = b, a + b
    return out


def _histograms():
    rng = np.random.default_rng(0)
    hs = {'single': [0] * 100 + [7] + [0] * 185, 'two': [3] + [0] * 284 + [9], 'all_286': [1] * 286,
          'fibonacci_286': (_fib(25) + [1] * 261)[:286], 'fibonacci_30': _fib(30), 'one_distance': [0] * 7 + [5] + [0] * 22,
          'no_distance': [0] * 30, 'fibonacci_19': _fib(19)}
    for k in range(40):
        n = [286, 30, 19][k % 3]
        hs['random_%d' % k] = (rng.integers(0, 1 << rng.integers(1, 17), n) * (rng.random(n) < rng.random())).tolist()
    return hs


@pytest.mark.parametrize('name', list(_histograms()))
@pytest.mark.parametrize('limit', [15, 7])
def test_emu_code_lengths_limited_and_complete(emu, name, limit):
    """every used symbol gets a code, no code exceeds the limit, and the code is complete (inflate refuses incomplete ones,
    except a single distance code) -- at least two symbols always have a code"""
    freq = np.array(_histograms()[name], dtype=np.uint64)
    if limit == 7 and len(freq) > 128:
        freq = freq[:19]
    lens = _lengths(emu, freq, limit)
    assert lens.max() <= limit
    assert ((freq > 0) <= (lens > 0)).all()
    assert (lens > 0).sum() >= 2
    assert sum(2.0 ** -int(x) for x in lens if x) == 1.0


def test_emu_code_lengths_are_huffman_when_the_limit_does_not_bind(emu):
    """the cost equals an unlimited Huffman code's when no length reaches the limit"""
    import heapq
    rng = np.random.default_rng(1)
    for _ in range(50):
        freq = rng.integers(1, 1000, 60)
        lens = _lengths(emu, freq, 15)
        h = list(freq.tolist())
        heapq.heapify(h)
        cost = 0
        while len(h) > 1:
            a, b = heapq.heappop(h), heapq.heappop(h)
            cost += a + b
            heapq.heappush(h, a + b)
        assert int((freq * lens).sum()) == cost


def test_emu_crc32_and_combine(emu):
    rng = np.random.default_rng(2)
    for _ in range(200):
        n = int(rng.integers(0, 5000))
        data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        k = int(rng.integers(0, n + 1))
        a, b = emu.emu_crc32(0, data[:k], k), emu.emu_crc32(0, data[k:], n - k)
        assert a == zlib.crc32(data[:k]) and b == zlib.crc32(data[k:])
        assert emu.emu_crc32_combine(a, b, n - k) == zlib.crc32(data)
        assert emu.emu_crc32(a, data[k:], n - k) == zlib.crc32(data)


@pytest.mark.parametrize('name', ['one', 'two', 'three', 'block', 'zeros', 'every_byte', 'period_32768', 'random', 'fastq'])
def test_emu_dynamic_block_inflates(emu, name):
    data = ont_fastq(100_000, 8) if name == 'fastq' else edge_inputs()[name]
    cap = 2 * len(data) + 1024
    out = np.zeros(cap, dtype=np.uint8)
    n = emu.emu_deflate_block(data, len(data), out.ctypes.data, cap)
    assert n > 0
    assert zlib.decompress(out[:n].tobytes(), wbits=-15) == data
