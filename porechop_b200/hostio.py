"""ctypes binding of porechop_b200/libhostio.so (include/porechop_b200_io.h): flat-buffer FASTQ ingest / emit in C.

`LIB` is None when the library has not been built (python -m porechop_b200.build); porechop_b200/fastq.py then uses its
numpy implementations of the same functions (identical results, much slower on long reads).  This is host I/O only --
the alignment engine itself has no fallback of any kind."""
import os
from ctypes import CDLL, c_double, c_int, c_int64, c_uint64, c_void_p

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libhostio.so')
EXPORTED_SYMBOLS = ['pbioSetThreads', 'pbioCountLines', 'pbioLineEnds', 'pbioLineSpans', 'pbioFastqIndex', 'pbioGather', 'pbioNormalise', 'pbioEmit', 'pbioScores', 'pbioEndTrim',
                    'pbioFullScores', 'pbioGzipBound', 'pbioGzip', 'pbioRandomBases']


def usable_cpus():
    """CPUs this process can really run on at once: the affinity mask capped by the cgroup CPU quota (a host may show many
    more hardware threads than its quota lets run; a larger team only gets the whole process throttled)."""
    try:
        n = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        n = os.cpu_count() or 1
    try:
        with open('/sys/fs/cgroup/cpu.max') as f:
            q, p = f.read().split()[:2]
        if q != 'max' and int(p) > 0:
            n = min(n, max(1, -(-int(q) // int(p))))
    except (OSError, ValueError):
        pass
    return max(1, n)


def _load():
    if not os.path.exists(_PATH) or os.environ.get('PB200_NO_HOSTIO'):
        return None
    # idle OpenMP threads sleep instead of spinning (must be set before libgomp is loaded): spinning burns the CPU quota
    os.environ.setdefault('OMP_WAIT_POLICY', 'passive')
    try:
        lib = CDLL(_PATH)
    except OSError:                 # e.g. built against a libgomp / libz this machine lacks: numpy + gzip module instead
        return None
    lib.pbioSetThreads.argtypes = [c_int]
    lib.pbioSetThreads.restype = c_int
    lib.pbioCountLines.argtypes = [c_void_p, c_int64]
    lib.pbioCountLines.restype = c_int64
    lib.pbioLineEnds.argtypes = [c_void_p, c_int64, c_void_p, c_int64]
    lib.pbioLineEnds.restype = c_int
    lib.pbioLineSpans.argtypes = [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]
    lib.pbioLineSpans.restype = None
    lib.pbioFastqIndex.argtypes = [c_void_p, c_int64, c_void_p, c_int64] + [c_void_p] * 6
    lib.pbioFastqIndex.restype = c_int
    lib.pbioGather.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64]
    lib.pbioGather.restype = None
    lib.pbioNormalise.argtypes = [c_void_p, c_void_p, c_int64, c_void_p]
    lib.pbioNormalise.restype = None
    lib.pbioEmit.argtypes = [c_void_p, c_void_p, c_int64, c_int] + [c_void_p] * 10
    lib.pbioEmit.restype = None
    lib.pbioScores.argtypes = [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.pbioScores.restype = None
    lib.pbioEndTrim.argtypes = [c_void_p, c_int64, c_int64, c_int, c_int64, c_int64, c_double, c_int64, c_void_p]
    lib.pbioEndTrim.restype = None
    lib.pbioFullScores.argtypes = [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p]
    lib.pbioFullScores.restype = None
    lib.pbioGzipBound.argtypes = [c_int64, c_int64]
    lib.pbioGzipBound.restype = c_int64
    lib.pbioGzip.argtypes = [c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64]
    lib.pbioGzip.restype = c_int64
    lib.pbioRandomBases.argtypes = [c_void_p, c_int64, c_uint64]
    lib.pbioRandomBases.restype = None
    if not os.environ.get('OMP_NUM_THREADS'):
        lib.pbioSetThreads(usable_cpus())
    return lib


LIB = _load()


def _p(a):
    return a.ctypes.data_as(c_void_p) if a is not None else None


def _i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def fastq_index(buf):
    """buf: contiguous uint8.  Returns (name_a, name_len, seq_a, seq_len, qual_a, qual_len) int64 arrays, or raises
    ValueError exactly where the numpy parser does."""
    n = len(buf)
    n_lines = int(LIB.pbioCountLines(_p(buf), n))
    if n_lines % 4 != 0:
        raise ValueError('FASTQ chunk is not a whole number of 4-line records')
    line_end = np.empty(n_lines, dtype=np.int64)
    if LIB.pbioLineEnds(_p(buf), n, _p(line_end), n_lines) != 0:
        raise ValueError('FASTQ chunk is not a whole number of 4-line records')
    out = [np.empty(n_lines // 4, dtype=np.int64) for _ in range(6)]
    rc = LIB.pbioFastqIndex(_p(buf), n, _p(line_end), n_lines, *[_p(x) for x in out])
    if rc == 2:
        raise ValueError('FASTQ record does not start with @')
    if rc != 0:
        raise ValueError('FASTQ chunk is not a whole number of 4-line records')
    return out


def line_spans(buf):
    """stripped extent (start, length) of every line of buf, as two int64 arrays."""
    n = len(buf)
    n_lines = int(LIB.pbioCountLines(_p(buf), n))
    line_end = np.empty(n_lines, dtype=np.int64)
    if LIB.pbioLineEnds(_p(buf), n, _p(line_end), n_lines) != 0:
        raise ValueError('could not index the lines')
    a, ln = np.empty(n_lines, dtype=np.int64), np.empty(n_lines, dtype=np.int64)
    LIB.pbioLineSpans(_p(buf), _p(line_end), n_lines, _p(a), _p(ln))
    return a, ln


def gather(src, src_a, lens, src_len=None, fill=0, alloc=None):
    """concatenate src[src_a[i] : src_a[i]+lens[i]] (short sources padded with `fill`) -> (flat uint8, int64 offsets).
    alloc(nbytes) -> uint8 array or None: where the result goes (e.g. the engine's pinned staging buffer)."""
    lens = _i64(lens)
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    dst = alloc(int(off[-1])) if alloc is not None else None
    if dst is None:
        dst = np.empty(int(off[-1]), dtype=np.uint8)
    src_a = _i64(src_a)
    sl = _i64(src_len) if src_len is not None else None
    LIB.pbioGather(_p(dst), _p(off), _p(src), _p(src_a), _p(sl), int(fill), len(lens))
    return dst, off


def normalise(seq, off):
    rna = np.zeros(len(off) - 1, dtype=np.uint8)
    LIB.pbioNormalise(_p(seq), _p(off), len(off) - 1, _p(rna))
    return rna.astype(bool)


def emit(out_off, fmt, names, name_a, name_len, seq, seq_a, seq_len, qual, qual_a, qual_len, rna):
    out = np.empty(int(out_off[-1]), dtype=np.uint8)
    arrs = [_i64(x) for x in (out_off, name_a, name_len, seq_a, seq_len, qual_a, qual_len)]
    rna8 = np.ascontiguousarray(rna, dtype=np.uint8)
    LIB.pbioEmit(_p(out), _p(arrs[0]), len(arrs[1]), 0 if fmt == 'fastq' else 1, _p(names), _p(arrs[1]), _p(arrs[2]),
                 _p(seq), _p(arrs[3]), _p(arrs[4]), _p(qual), _p(arrs[5]), _p(arrs[6]), _p(rna8))
    return out


def scores(records):
    """int32[n, 9] records -> (full, part, read_start, read_end) as align_adapter() would parse them."""
    r = np.ascontiguousarray(records, dtype=np.int32).reshape(-1, 9)
    n = len(r)
    full, part = np.empty(n, dtype=np.float64), np.empty(n, dtype=np.float64)
    rs, re_ = np.empty(n, dtype=np.int64), np.empty(n, dtype=np.int64)
    LIB.pbioScores(_p(r), n, _p(full), _p(part), _p(rs), _p(re_))
    return full, part, rs, re_


def end_trim(records, is_start, end_size, extra_trim_size, end_threshold, min_trim_size):
    """records int32[n, a, 9] -> int64[n] trim amounts (the start or the end rule of nanopore_read.py:166-208)."""
    r = np.ascontiguousarray(records, dtype=np.int32)
    n, a = r.shape[0], r.shape[1]
    out = np.zeros(n, dtype=np.int64)
    if n and a:
        LIB.pbioEndTrim(_p(r), n, a, 1 if is_start else 0, int(end_size), int(extra_trim_size), float(end_threshold),
                        int(min_trim_size), _p(out))
    return out


def full_scores(records, cols):
    """records int32[n, a, 9], cols: adapter indices -> float64[n, len(cols)] full-adapter identities."""
    r = np.ascontiguousarray(records, dtype=np.int32)
    n, a = r.shape[0], r.shape[1]
    cols = _i64(cols)
    out = np.zeros((n, len(cols)), dtype=np.float64)
    if n and len(cols):
        LIB.pbioFullScores(_p(r), n, a, _p(cols), len(cols), _p(out))
    return out


def gzip_members(payload, level=6, block=4 << 20):
    """payload (bytes-like / uint8 array) -> memoryview of a multi-member .gz of it, compressed block-parallel in C;
    None when the library has no zlib (the caller then uses Python's gzip)."""
    if LIB is None:
        return None
    src = np.frombuffer(payload, dtype=np.uint8) if not isinstance(payload, np.ndarray) else np.ascontiguousarray(payload)
    cap = int(LIB.pbioGzipBound(len(src), block))
    if cap < 0:
        return None
    dst = np.empty(cap, dtype=np.uint8)
    size = int(LIB.pbioGzip(_p(src), len(src), int(level), int(block), _p(dst), cap))
    if size < 0:
        return None
    return memoryview(dst)[:size]


def set_threads(n=0):
    """set (n > 0) / query the number of worker threads of the C helpers; 1 when the library is absent."""
    return int(LIB.pbioSetThreads(int(n))) if LIB is not None else 1


def random_bases(n, seed, out=None):
    """n iid uniform ACGT bytes, a pure function of (seed, n) (pbioRandomBases: one generator per 1 MiB block, so the
    bytes do not depend on the thread count); written into `out` (uint8, length >= n) when given.  Workload generator of
    bench.py / workloads.py, not part of the alignment path."""
    if out is None:
        out = np.empty(n, dtype=np.uint8)
    assert out.dtype == np.uint8 and out.flags.c_contiguous and len(out) >= n
    if LIB is not None:
        LIB.pbioRandomBases(_p(out), int(n), int(seed) & 0xFFFFFFFFFFFFFFFF)
        return out[:n]
    # numpy restatement of the same generator (splitmix64 per 1 MiB block, 32 bases per draw)
    acgt = np.frombuffer(b'ACGT', dtype=np.uint8)
    M = (1 << 64) - 1
    blk = 1 << 20
    for b in range((n + blk - 1) // blk):
        lo, hi = b * blk, min(n, (b + 1) * blk)
        draws = (hi - lo + 31) // 32
        st = (int(seed) * 0xD1342543DE82EF95 + b * 0x2545F4914F6CDD1D + 1) & M
        x = (np.uint64(st) + np.arange(1, draws + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        codes = ((z[:, None] >> (np.arange(32, dtype=np.uint64) * np.uint64(2))) & np.uint64(3)).astype(np.uint8).reshape(-1)
        out[lo:hi] = acgt[codes[:hi - lo]]
    return out[:n]
