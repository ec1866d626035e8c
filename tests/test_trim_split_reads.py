"""Porechop's output reads cut on the device (include/porechop_b200.h adapterTrimSplitReadsDevice, device_reads.trim_reads,
fastq.emit_parts).  CPU tier: the product's engine code on the host simulator (tests/sim) against the reference CLI's bytes
and against fastq.emit over the record path's decisions; the split rule through tests/emu against fastq._split_parts.  The
GPU tier is tests/test_gpu_trim_split_reads.py."""
import ctypes
import os
import random
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from helpers import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

DEFAULT = (3, -6, -5, -2)
LINEAR = (3, -6, -5, -5)
OPTS = dict(end_size=150, extra_end_trim=2, end_threshold=75.0, min_trim_size=4, no_split=False, middle_threshold=85.0,
            extra_middle_trim_good_side=10, extra_middle_trim_bad_side=100, min_split_read_size=1000, discard_middle=False,
            untrimmed=False)


@pytest.fixture(autouse=True)
def _stream_order_checked():
    """every test here also passes the simulated runtime's stream-ordering check (pbsim_cuda.h): no race between streams"""
    import sim_engine
    sim_engine.clear_races()
    yield
    sim_engine.assert_no_races()


@pytest.fixture(scope='module')
def SW():
    import sim_engine
    return sim_engine.load()


# ---- simulated device buffers in the shape device_reads expects of its allocator ----
class SimBuf:
    def __init__(self, ptr, n, dtype):
        self.ptr, self.n, self.dtype = ptr, int(n), np.dtype(dtype)


class SimDevice:
    """device_reads' allocator on the simulated engine: exact-size heap blocks (so that AddressSanitizer sees every byte past
    the end), the library's own stream"""

    def __init__(self, W):
        self.W, self.bufs = W, []

    def empty(self, n, dtype):
        b = SimBuf(self.W.device_alloc(max(int(n) * np.dtype(dtype).itemsize, 1)), n, dtype)
        self.bufs.append(b)
        return b

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        b = self.empty(len(arr), arr.dtype)
        if arr.nbytes:
            self.W.upload(b.ptr, arr.ctypes.data, arr.nbytes, None)
        return b

    def ptr(self, b):
        return b.ptr if b is not None else 0

    def numel(self, b):
        return b.n

    def head(self, b, n):
        return SimBuf(b.ptr, n, b.dtype)

    def stream(self):
        return 0

    def host(self, b):
        if b is None:
            return None
        nb = b.n * b.dtype.itemsize
        return np.frombuffer((ctypes.c_uint8 * nb).from_address(b.ptr), dtype=b.dtype).copy() if nb else np.zeros(0, b.dtype)

    def free(self):
        for b in self.bufs:
            self.W.device_free(b.ptr)
        self.bufs = []


def _batch(reads, rna_read=None):
    from porechop_b200 import fastq
    text = ''.join('@r%d extra words\n%s\n+\n%s\n' % (k, r, ''.join(chr(33 + (k * 7 + j) % 40) for j in range(len(r))))
                   for k, r in enumerate(reads))
    return fastq.parse_fastq(text.encode())


def _sets(which='both'):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    top, bottom = ('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb)
    return {'both': [(top, bottom)], 'start': [(top, None)], 'end': [(None, bottom)], 'none': []}[which]


def _expected(W, monkeypatch, batch, sets, scheme, o, fmt='fastq'):
    """fastq.emit over the record path's decisions (trim_end_adapters without device decisions + find_middle_hits with the
    host rounds) -- what the device output stage must reproduce"""
    from porechop_b200 import fastq
    monkeypatch.setattr(fastq, 'W', W)
    sets = fastq._norm_sets(sets)
    starts, ends = [s[1] for _, s, _ in sets if s], [e[1] for _, _, e in sets if e]
    adapters = [] if o['no_split'] else fastq._middle_adapters(sets)
    st, et, _, _ = fastq.trim_end_adapters(batch, starts, ends, scheme, o['end_size'], o['extra_end_trim'], o['end_threshold'],
                                           o['min_trim_size'], device_decisions=False)
    hits = fastq.find_middle_hits(batch, st, et, adapters, o['middle_threshold'], scheme, device=False) if adapters else {}
    middle = fastq.middle_trim_ranges(hits, adapters, {s[0] for _, s, _ in sets if s}, {e[0] for _, _, e in sets if e},
                                      o['extra_middle_trim_good_side'], o['extra_middle_trim_bad_side'])
    out = fastq.emit(batch, st, et, middle, fmt, o['min_split_read_size'], o['discard_middle'], o['untrimmed'])
    return st, et, hits, out


def _device_run(W, monkeypatch, batch, sets, scheme, o, fmt='fastq', barcodes=None):
    """device_reads.trim_reads on the simulated engine; returns (result with host copies of the records, emitted bytes)"""
    from porechop_b200 import device_reads, fastq
    D = SimDevice(W)
    monkeypatch.setattr(device_reads, 'W', W)
    monkeypatch.setattr(device_reads, '_device', D)
    try:
        seq, off = D.upload(batch.seq), D.upload(batch.seq_off)
        qual = D.upload(batch.qual) if fmt == 'fastq' else None
        r = device_reads.trim_reads(seq, off, sets, scheme, qual, barcodes=barcodes, **o)
        parts = tuple(D.host(x) for x in r[:5])
        # the caller's reads, qualities and offsets are as they were
        assert np.array_equal(D.host(seq), batch.seq) and np.array_equal(D.host(off), batch.seq_off)
        if qual is not None:
            assert np.array_equal(D.host(qual), batch.qual)
    finally:
        D.free()
    r = r._replace(seq=parts[0], qual=parts[1], off=parts[2], read=parts[3], part=parts[4])
    return r, fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, parts, fmt)


# ---- the reference CLI's bytes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case_name', ['default', 'small_parts', 'discard_middle', 'no_split_fasta', 'fasta_split'])
def test_sim_golden_trim_cases(SW, monkeypatch, case_name):
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    c = g['cases'][case_name]
    o = dict(c['options'])
    fmt = o.pop('fmt')
    batch = fastq.parse_fastq(g['input_fastq'].encode())
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    r, out = _device_run(SW, monkeypatch, batch, sets, c['scoring'], o, fmt)
    assert out.decode() == c['output']
    if case_name == 'default':
        assert (r.part > 0).any() and len(r.hits) >= 4


@pytest.mark.parametrize('case_name', ['bins_default', 'bins_two_barcodes', 'bins_loose_discard', 'bins_fasta_untrimmed'])
def test_sim_golden_barcode_cases(SW, monkeypatch, case_name):
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases'][case_name]
    o = dict(c['options'])
    fmt, discard_unassigned = o.pop('fmt'), o.pop('discard_unassigned')
    barcodes = {k: o.pop(k) for k in ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes')}
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    r, _ = _device_run(SW, monkeypatch, batch, c['matching_sets'], c['scoring'], o, fmt, barcodes=barcodes)
    calls = np.array(r.calls, dtype=object)
    bins = {}
    for name in dict.fromkeys(r.calls):
        if discard_unassigned and name == 'none':
            continue
        out = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, r[:5], fmt, select=(calls == name))
        if len(out):
            bins[name] = out
    assert sorted(k + '.' + fmt for k in bins) == sorted(c['bins'])
    for k, v in bins.items():
        assert v.decode() == c['bins'][k + '.' + fmt], k


# ---- against the host path -----------------------------------------------------------------------------------------------
def _compare(W, monkeypatch, which='both', scheme=DEFAULT, fmt='fastq', reads=None, **kw):
    from test_trim_reads import trim_reads_set
    o = dict(OPTS, **kw)
    batch = _batch(reads or trim_reads_set())
    st, et, hits, exp = _expected(W, monkeypatch, batch, _sets(which), scheme, o, fmt)
    r, got = _device_run(W, monkeypatch, batch, _sets(which), scheme, o, fmt)
    assert np.array_equal(r.start_trim, st) and np.array_equal(r.end_trim, et)
    assert r.hits == hits
    assert got == exp
    return r


@pytest.mark.parametrize('min_split', [0, 1, 50, 1000])
def test_sim_split_equals_host_path_min_split(SW, monkeypatch, min_split):
    r = _compare(SW, monkeypatch, min_split_read_size=min_split, middle_threshold=70.0)
    if min_split <= 50:
        assert (r.part >= 2).any()                              # reads really split into several parts


def test_sim_split_equals_host_path_options(SW, monkeypatch):
    _compare(SW, monkeypatch, discard_middle=True, min_split_read_size=50)
    _compare(SW, monkeypatch, untrimmed=True, min_split_read_size=50)
    _compare(SW, monkeypatch, untrimmed=True, discard_middle=True)
    _compare(SW, monkeypatch, fmt='fasta', min_split_read_size=50)


def test_sim_split_equals_host_path_adapter_sets(SW, monkeypatch):
    _compare(SW, monkeypatch, 'start', min_split_read_size=50)
    _compare(SW, monkeypatch, 'end', min_split_read_size=50)
    _compare(SW, monkeypatch, no_split=True)
    r = _compare(SW, monkeypatch, 'none')                       # "No adapters found": every non-empty read unchanged
    assert (r.part == 0).all() and len(r.read) == int((_batch(__import__('test_trim_reads').trim_reads_set()).lengths() > 0).sum())


def test_sim_split_equals_host_path_schemes_and_windows(SW, monkeypatch):
    _compare(SW, monkeypatch, scheme=LINEAR, min_split_read_size=50)
    _compare(SW, monkeypatch, end_size=400, min_split_read_size=50)


def test_sim_split_extra_trims_past_both_ends_and_hits_without_parts(SW, monkeypatch):
    # ranges that stick out of both ends of the trimmed read; hits whose parts are all too short
    _compare(SW, monkeypatch, extra_middle_trim_good_side=300, extra_middle_trim_bad_side=700, min_split_read_size=1)
    r = _compare(SW, monkeypatch, min_split_read_size=400, middle_threshold=70.0)
    assert len(r.hits) > len(set(r.read[r.part > 0].tolist()))


def test_sim_emit_parts_names_numbers_rna_and_fasta_columns():
    """emit_parts on hand-made records: '_k' before the first space, U for RNA reads, 70-column FASTA"""
    from porechop_b200 import fastq
    batch = fastq.parse_fastq(b'@a x y\nACGT\n+\n!!!!\n@b\nACGUACGU\n+\n########\n')
    assert batch.rna.tolist() == [False, True]
    seq = np.frombuffer(b'CGTACGTACGT' + b'A' * 150, dtype=np.uint8)
    qual = np.frombuffer(b'12345678901' + b'I' * 150, dtype=np.uint8)
    parts = (seq, qual, np.array([0, 3, 5, 11, 161]), np.array([0, 1, 1, 0]), np.array([0, 1, 2, 3]))
    got = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, parts, 'fastq')
    assert got == b'@a x y\nCGT\n+\n123\n@b_1\nAC\n+\n45\n@b_2\nGUACGU\n+\n678901\n@a_3 x y\n' + b'A' * 150 + b'\n+\n' + \
        b'I' * 150 + b'\n'
    got = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, (seq, None) + parts[2:], 'fasta', select=[True, False])
    assert got == b'>a x y\nCGT\n>a_3 x y\n' + b'A' * 70 + b'\n' + b'A' * 70 + b'\n' + b'A' * 10 + b'\n'


# ---- segments, capacity, preconditions -------------------------------------------------------------------------------------
class _Raw:
    """adapterTrimSplitReadsDevice with every argument struct built here, for the error paths"""

    def __init__(self, W, batch, qual=True, parts_cap=10000, hits_cap=10000):
        from porechop_b200 import workloads as wl
        yt, yb = wl.nsk007()
        self.W, self.D, n = W, SimDevice(W), len(batch)
        self.n, self.nbytes = n, len(batch.seq)
        self.d_seq, self.d_off = self.D.upload(batch.seq), self.D.upload(batch.seq_off)
        self.d_qual = self.D.upload(batch.qual) if qual else None
        self.keep = [wl.pack_adapters([yt]), wl.pack_adapters([yb]), wl.pack_adapters([yt, yb])]
        self.trims = [np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)]
        self.n_hits, self.hits, self.total = np.zeros(n, dtype=np.int32), np.zeros((max(hits_cap, 1), 10), dtype=np.int32), \
            ctypes.c_int64(0)
        self.extra = (np.array([100, 10], dtype=np.int32), np.array([10, 100], dtype=np.int32))
        self.n_parts, self.n_bases = ctypes.c_int64(-1), ctypes.c_int64(-1)
        self.out = dict(seq=self.D.empty(self.nbytes, np.uint8), qual=self.D.empty(self.nbytes, np.uint8) if qual else None,
                        off=self.D.empty(parts_cap + 1, np.int64), read=self.D.empty(parts_cap, np.int32),
                        part=self.D.empty(parts_cap, np.int32))
        sides = [W.TrimSideDesc(a.ctypes.data, o.ctypes.data, 1, None, 0, t.ctypes.data, None, None)
                 for (a, o), t in zip(self.keep[:2], self.trims)]
        ma, mo = self.keep[2]
        self.args = W.TrimArgsDesc(150, 2, 4, 75.0, sides[0], sides[1], ma.ctypes.data, mo.ctypes.data, 2, 70.0,
                                   self.n_hits.ctypes.data, self.hits.ctypes.data, hits_cap, ctypes.addressof(self.total))
        P = lambda b: b.ptr if b is not None else None      # noqa: E731
        self.split = W.SplitArgsDesc(P(self.d_qual), self.extra[0].ctypes.data, self.extra[1].ctypes.data, 50, 0, 0,
                                     P(self.out['seq']), P(self.out['qual']), P(self.out['off']), P(self.out['read']),
                                     P(self.out['part']), parts_cap, ctypes.addressof(self.n_parts), ctypes.addressof(self.n_bases))

    def call(self, split=True, **fields):
        for k, v in fields.items():
            setattr(self.split, k, v)
        return self.W.C_LIB.adapterTrimSplitReadsDevice(self.d_seq.ptr, self.d_off.ptr, self.n, self.nbytes, -1,
                                                        ctypes.byref(self.args), ctypes.byref(self.split) if split else None,
                                                        *DEFAULT, None)

    def records(self):
        k = self.n_parts.value
        o = self.out
        return (self.D.host(self.D.head(o['seq'], self.n_bases.value)),
                self.D.host(self.D.head(o['qual'], self.n_bases.value)) if o['qual'] is not None else None,
                self.D.host(self.D.head(o['off'], k + 1)), self.D.host(self.D.head(o['read'], k)), self.D.host(self.D.head(o['part'], k)))


def _same_records(a, b):
    return all((x is None and y is None) or np.array_equal(x, y) for x, y in zip(a, b))


def test_sim_several_segments_give_the_same_records():
    """PB_TEST_SEGMENT_READS=7: the 33 reads run as 5 segments -- record offsets continue across them"""
    import sim_engine
    from test_trim_reads import trim_reads_set
    batch = _batch(trim_reads_set())
    W1, W7 = sim_engine.load(), sim_engine.load(['-DPB_TEST_SEGMENT_READS=7'])
    got = []
    for W in (W1, W7):
        R = _Raw(W, batch)
        try:
            assert R.call() == 0
            got.append((R.records(), R.trims[0].copy(), R.trims[1].copy(), R.n_hits.copy(), R.n_parts.value, R.n_bases.value))
        finally:
            R.D.free()
    assert _same_records(got[0][0], got[1][0]) and all(np.array_equal(x, y) for x, y in zip(got[0][1:4], got[1][1:4]))
    assert got[0][4:] == got[1][4:] and got[0][4] > len(batch) // 2 and (got[0][0][4] > 0).any()
    n, text = W7.races()
    assert n == 0, text[:4000]


def test_sim_parts_cap_and_hits_cap_too_small(SW):
    from test_trim_reads import trim_reads_set
    batch = _batch(trim_reads_set())
    R = _Raw(SW, batch)
    try:
        assert R.call() == 0
        full, n_parts, n_bases = R.records(), R.n_parts.value, R.n_bases.value
        trims, n_hits, total = [t.copy() for t in R.trims], R.n_hits.copy(), R.total.value
    finally:
        R.D.free()
    for kw in (dict(parts_cap=3), dict(hits_cap=2), dict(parts_cap=0, hits_cap=0)):
        R = _Raw(SW, batch, **kw)
        try:
            assert R.call() == SW.ERR_SPACE, kw
            assert (R.n_parts.value, R.n_bases.value) == (n_parts, n_bases) and R.total.value == total
            assert np.array_equal(R.trims[0], trims[0]) and np.array_equal(R.trims[1], trims[1]) and np.array_equal(R.n_hits, n_hits)
        finally:
            R.D.free()
    R = _Raw(SW, batch, parts_cap=n_parts, hits_cap=total)       # the retry with the exact counts
    try:
        assert R.call() == 0 and _same_records(R.records(), full)
    finally:
        R.D.free()


def test_sim_preconditions_fail_before_any_launch(SW):
    from test_trim_reads import trim_reads_set
    batch = _batch(trim_reads_set()[:8])
    R = _Raw(SW, batch)
    fake = R.out['seq'].ptr
    try:
        bad = [dict(parts_cap=-1), dict(mid_extra_left=None), dict(mid_extra_right=None), dict(d_out_qual=None),
               dict(d_quals=None), dict(d_out_off=None), dict(d_out_read=None), dict(d_out_part=None), dict(d_out_seq=None),
               dict(n_parts=None), dict(n_out_bases=None)]
        for kw in bad:
            saved = {k: getattr(R.split, k) for k in kw}
            n0 = SW.kernel_launches()
            R.n_parts.value = R.n_bases.value = -1
            assert R.call(**kw) == SW.ERR_ARG, kw
            assert SW.kernel_launches() == n0, kw
            assert kw.get('n_parts', 1) is None or R.n_parts.value == 0, kw
            for k, v in saved.items():
                setattr(R.split, k, v)
        n0 = SW.kernel_launches()
        assert R.call(split=False) == SW.ERR_ARG and SW.kernel_launches() == n0
        R.args.end_size = 0                                       # a precondition of adapterTrimReadsDevice
        assert R.call() == SW.ERR_ARG and SW.kernel_launches() == n0 and R.n_parts.value == 0
        R.args.end_size = 150
        # a FASTA call: no qualities in, none out
        assert R.call(d_quals=None, d_out_qual=None) == 0 and R.n_parts.value > 0
        assert R.call(d_quals=R.d_qual.ptr, d_out_qual=fake) == 0
    finally:
        R.D.free()


# ---- the torch-level module's logic -----------------------------------------------------------------------------------------
def test_sim_device_reads_retries_with_the_exact_count_and_calls_barcodes(SW, monkeypatch):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases']['bins_default']
    o = dict(c['options'])
    fmt = o.pop('fmt')
    o.pop('discard_unassigned')
    barcodes = {k: o.pop(k) for k in ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes')}
    o['discard_middle'] = False
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    exp, exp_bytes = _device_run(SW, monkeypatch, batch, c['matching_sets'], c['scoring'], o, fmt, barcodes=barcodes)
    calls = []
    orig = SW.adapter_trim_split_reads_device

    def spy(*a, **k):
        calls.append(k['parts_cap'])
        return orig(*a, **k)
    monkeypatch.setattr(SW, 'adapter_trim_split_reads_device', spy)
    monkeypatch.setattr(device_reads, 'initial_parts_cap', lambda n: 2)
    got, got_bytes = _device_run(SW, monkeypatch, batch, c['matching_sets'], c['scoring'], o, fmt, barcodes=barcodes)
    assert calls == [2, len(exp.read)] and got_bytes == exp_bytes and got.calls == exp.calls
    # the calls are demux_fastq's
    monkeypatch.setattr(fastq, 'W', SW)
    _, info = fastq.demux_fastq(g['barcoded_fastq'].encode(), c['matching_sets'], c['scoring'], fmt=fmt, **barcodes, **o)
    assert got.calls == info['calls']


# ---- the split rule through tests/emu ------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu_split():
    d = tempfile.mkdtemp(prefix='pb200_emu_split_')
    so = os.path.join(d, 'libemu_split.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', so, os.path.join(ROOT, 'tests', 'emu', 'emu_split.cpp')])
    lib = ctypes.CDLL(so)
    lib.emu_split_parts.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p]
    lib.emu_split_parts.restype = ctypes.c_int64
    return lib


def test_emu_split_rule_equals_host_rule(emu_split):
    from porechop_b200 import fastq
    rng = random.Random(5)
    for trial in range(3000):
        length = rng.choice([0, 1, 2, 5, 40, 300, 2000])
        hits = [(rng.randint(0, 1), rng.randint(-50, length + 50), 0, 90.0) for _ in range(rng.randint(0, 6))]
        hits = [(p, x, x + rng.randint(0, 60), s) for p, x, _, s in hits]
        adapters = [('s', 'A'), ('e', 'C')]
        good, bad = rng.choice([0, 3, 10]), rng.choice([0, 40, 100, 5000])
        ranges = fastq.middle_trim_ranges({0: hits}, adapters, {'s'}, {'e'}, good, bad).get(0, [])
        min_size = rng.choice([0, 1, 5, 50, 1000])
        exp = fastq._split_parts(length, ranges, min_size)
        r = np.array(sorted(ranges), dtype=np.int32).reshape(-1)
        out = np.zeros(2 * (len(ranges) + 1), dtype=np.int64)
        k = emu_split.emu_split_parts(length, r.ctypes.data if len(r) else None, len(ranges), min_size, out.ctypes.data)
        assert [tuple(x) for x in out[:2 * k].reshape(-1, 2).tolist()] == exp, (length, ranges, min_size)


# ---- AddressSanitizer -------------------------------------------------------------------------------------------------------
def _asan_body():
    """the output stage on exact-size "device" heap blocks: golden cases, the host-path comparison, capacity and argument
    errors (run by test_sim_trim_split_under_address_sanitizer in a process with the ASan build of the simulated engine)"""
    import sim_engine

    class MP:                                              # the part of pytest's monkeypatch the helpers use
        def __init__(self):
            self.undo = []

        def setattr(self, obj, name, value):
            self.undo.append((obj, name, getattr(obj, name)))
            setattr(obj, name, value)

        def close(self):
            for obj, name, value in reversed(self.undo):
                setattr(obj, name, value)
    W = sim_engine.load()
    for case in ('default', 'small_parts', 'fasta_split', 'no_split_fasta'):
        mp = MP()
        test_sim_golden_trim_cases(W, mp, case)
        mp.close()
    mp = MP()
    test_sim_golden_barcode_cases(W, mp, 'bins_fasta_untrimmed')
    mp.close()
    for kw in (dict(min_split_read_size=1, middle_threshold=70.0), dict(untrimmed=True), dict(which='none')):
        mp = MP()
        _compare(W, mp, **kw)
        mp.close()
    test_sim_parts_cap_and_hits_cap_too_small(W)
    test_sim_preconditions_fail_before_any_launch(W)
    print('ASAN RUN COMPLETE')


@pytest.mark.skipif(os.environ.get('PB200_SIM_ASAN', '0') != '1', reason='minutes: set PB200_SIM_ASAN=1')
def test_sim_trim_split_under_address_sanitizer():
    import build_sim
    lib = build_sim.build_asan()
    asan = subprocess.check_output(['gcc', '-print-file-name=libasan.so']).decode().strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS='detect_leaks=0:detect_stack_use_after_return=0', PB200_SIM_ASAN_LIB=lib)
    code = ('import os, sys; sys.path[:0] = [%r, %r, %r]; import build_sim; '
            'build_sim.build = lambda force=False, flags=None: os.environ["PB200_SIM_ASAN_LIB"]; '
            'import test_trim_split_reads as T; T._asan_body()') % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and 'ASAN RUN COMPLETE' in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    assert 'ERROR: AddressSanitizer' not in r.stderr
