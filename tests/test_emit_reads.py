"""Porechop's output files formatted on the device (include/porechop_b200.h pb200EmitReadsDevice, device_reads.emit_reads).  CPU
tier: the product's engine code on the host simulator (tests/sim) against the reference CLI's files and against
fastq.emit_parts over host copies of the same records.  The GPU tier is tests/test_gpu_emit_reads.py."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

from test_demux_reads import _golden  # noqa: E402
from test_trim_split_reads import DEFAULT, LINEAR, OPTS, SimDevice, _batch, _sets  # noqa: E402

SENTINEL = 0xA5


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


def _names(D, batch, rna=None):
    """the reads' names and RNA flags as device buffers"""
    rna = batch.rna if rna is None else rna
    return D.upload(batch.name_buf), D.upload(batch.name_off), D.upload(np.asarray(rna, dtype=np.uint8))


def _host_records(D, r):
    return tuple(D.host(x) for x in r[:5])


def _run(W, monkeypatch, batch, sets, scheme, o, fmts=('fastq',), rna=None, bc=None):
    """upload -> trim_reads (demux_reads with bc) -> emit_reads in each format, on the simulated engine.  Returns (host copies
    of the records, {fmt: (bytes, byte offsets, bins)})"""
    from porechop_b200 import device_reads
    D = SimDevice(W)
    monkeypatch.setattr(device_reads, 'W', W)
    monkeypatch.setattr(device_reads, '_device', D)
    try:
        seq, off = D.upload(batch.seq), D.upload(batch.seq_off)
        qual = D.upload(batch.qual) if 'fastq' in fmts else None
        r = device_reads.trim_reads(seq, off, sets, scheme, qual, **o) if bc is None else \
            device_reads.demux_reads(seq, off, sets, scheme, qual, **bc, **o)
        names, name_off, d_rna = _names(D, batch, rna)
        out = {}
        for fmt in fmts:
            em = device_reads.emit_reads(r, names, name_off, d_rna, fmt)
            out[fmt] = (D.host(em.data).tobytes(), D.host(em.off), em.bins)
        parts = _host_records(D, r)
    finally:
        D.free()
    return r, parts, out


# ---- the reference CLI's bytes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case_name', ['default', 'small_parts', 'discard_middle', 'no_split_fasta', 'fasta_split'])
def test_sim_emit_golden_trim_cases(SW, monkeypatch, case_name):
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    c = g['cases'][case_name]
    o = dict(c['options'])
    fmt = o.pop('fmt')
    batch = fastq.parse_fastq(g['input_fastq'].encode())
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    _, parts, out = _run(SW, monkeypatch, batch, sets, c['scoring'], o, (fmt,))
    data, off, bins = out[fmt]
    assert data.decode() == c['output'] and bins is None
    assert off[0] == 0 and off[-1] == len(data) and len(off) == len(parts[3]) + 1
    if case_name == 'default':
        assert (parts[4] > 0).any() and batch.rna.any()


@pytest.mark.parametrize('case_name', ['bins_default', 'bins_two_barcodes', 'bins_loose_discard', 'bins_fasta_untrimmed'])
def test_sim_emit_golden_barcode_cases(SW, monkeypatch, case_name):
    batch, sets, scheme, o, bc, fmt, exp = _golden(case_name)
    r, _, out = _run(SW, monkeypatch, batch, sets, scheme, o, (fmt,), bc=bc)
    data, off, bins = out[fmt]
    assert sorted(k + '.' + fmt for k in bins) == sorted(exp)
    assert [b for b, _ in bins.values()] == sorted(b for b, _ in bins.values())
    for k, (b0, b1) in bins.items():
        assert data[b0:b1].decode() == exp[k + '.' + fmt], k
        r0, r1 = r.bins[k]
        assert (off[r0], off[r1]) == (b0, b1)


# ---- against fastq.emit_parts ----------------------------------------------------------------------------------------------
VARIANTS = [dict(min_split_read_size=0, middle_threshold=70.0), dict(min_split_read_size=1, middle_threshold=70.0),
            dict(min_split_read_size=50, middle_threshold=70.0), dict(min_split_read_size=1000, middle_threshold=70.0),
            dict(discard_middle=True, min_split_read_size=50), dict(untrimmed=True, min_split_read_size=50),
            dict(untrimmed=True, discard_middle=True), dict(which='start', min_split_read_size=50),
            dict(which='end', min_split_read_size=50), dict(no_split=True), dict(which='none'),
            dict(scheme=LINEAR, min_split_read_size=50), dict(end_size=400, min_split_read_size=50),
            dict(extra_middle_trim_good_side=300, extra_middle_trim_bad_side=700, min_split_read_size=1)]


@pytest.mark.parametrize('variant', range(len(VARIANTS)))
def test_sim_emit_equals_emit_parts(SW, monkeypatch, variant):
    """the bytes of both formats equal emit_parts over host copies of the same records; every third read is an RNA read"""
    from porechop_b200 import fastq
    from test_trim_reads import trim_reads_set
    kw = dict(VARIANTS[variant])
    which, scheme = kw.pop('which', 'both'), kw.pop('scheme', DEFAULT)
    batch = _batch(trim_reads_set())
    rna = np.arange(len(batch)) % 3 == 1
    _, parts, out = _run(SW, monkeypatch, batch, _sets(which), scheme, dict(OPTS, **kw), ('fastq', 'fasta'), rna=rna)
    for fmt in ('fastq', 'fasta'):
        exp = fastq.emit_parts(batch.name_buf, batch.name_off, rna, parts if fmt == 'fastq' else (parts[0], None) + parts[2:], fmt)
        assert out[fmt][0] == exp, fmt
    if variant < 3:
        assert (parts[4] >= 2).any()                            # reads really split into several parts


# ---- hand-made records through the raw binding ---------------------------------------------------------------------------
class _Raw:
    """pb200EmitReadsDevice over host arrays uploaded to simulated device memory"""

    def __init__(self, W, seq, qual, off, read, part, names, rna=None, cap=None):
        from porechop_b200 import cpp_function_wrappers as real
        self.W, self.D = W, SimDevice(W)
        self.seq, self.qual = np.frombuffer(bytes(seq), dtype=np.uint8), np.frombuffer(bytes(qual), dtype=np.uint8)
        self.off, self.read, self.part = (np.asarray(off, dtype=np.int64), np.asarray(read, dtype=np.int32),
                                          np.asarray(part, dtype=np.int32))
        self.name_buf, self.name_off = real.pack_sequences([n.encode() if isinstance(n, str) else n for n in names])
        self.rna = np.zeros(len(names), dtype=bool) if rna is None else np.asarray(rna, dtype=bool)
        D = self.D
        self.d = dict(seq=D.upload(self.seq), qual=D.upload(self.qual), off=D.upload(self.off), read=D.upload(self.read),
                      part=D.upload(self.part), names=D.upload(self.name_buf), name_off=D.upload(self.name_off),
                      rna=D.upload(self.rna.astype(np.uint8)))
        self.n_rec = len(self.read)
        self.cap = (2 * len(self.seq) + self.n_rec * (int(np.diff(self.name_off).max(initial=0)) + 20)) if cap is None else cap

    def expected(self, fmt, r0=0, r1=None):
        from porechop_b200 import fastq
        r1 = self.n_rec if r1 is None else r1
        parts = (self.seq, self.qual if fmt == 'fastq' else None, self.off[r0:r1 + 1], self.read[r0:r1], self.part[r0:r1])
        return fastq.emit_parts(self.name_buf, self.name_off, self.rna, parts, fmt)

    def call(self, fmt='fastq', r0=0, r1=None, cap=None, stream=0, **over):
        """(bytes, offsets) of records [r0, r1) -- sliced device arrays; `over` replaces keyword arguments of the binding"""
        r1 = self.n_rec if r1 is None else r1
        cap = self.cap if cap is None else cap
        self.out, self.out_off = self.D.empty(max(cap, 1), np.uint8), self.D.empty(r1 - r0 + 1, np.int64)
        ctypes.memset(self.out.ptr, SENTINEL, max(cap, 1))
        d = self.d
        kw = dict(d_seq_ptr=d['seq'].ptr, d_qual_ptr=d['qual'].ptr, seq_bytes=len(self.seq), d_off_ptr=d['off'].ptr + 8 * r0,
                  d_read_ptr=d['read'].ptr + 4 * r0, d_part_ptr=d['part'].ptr + 4 * r0, d_names_ptr=d['names'].ptr,
                  d_name_off_ptr=d['name_off'].ptr, n_reads=len(self.name_off) - 1, name_bytes=len(self.name_buf),
                  d_rna_ptr=d['rna'].ptr, fmt=fmt, d_out_ptr=self.out.ptr, out_cap=cap, d_out_off_ptr=self.out_off.ptr,
                  stream_ptr=stream)
        kw.update(over)
        n = self.W.pb200_emit_reads_device(r1 - r0, **kw)
        return self.D.host(self.D.head(self.out, n)).tobytes(), self.D.host(self.out_off)

    def untouched(self):
        return bool((self.D.host(self.out) == SENTINEL).all())

    def free(self):
        self.D.free()


def _hand_made():
    """names with one and several spaces, only a tab, empty; parts 0, 1, 9, 10, 99, 100 and 2^31 - 1; RNA reads with T, t and U;
    empty records; FASTA lengths around the 70-column line; qualities that differ from the bases"""
    rng = np.random.default_rng(7)
    names = ['a b', 'x  y z w', 'tab\there', '', 'plain', 'r5 runid=1 ch=3']
    rna = [True, True, False, False, False, True]
    lengths = [12, 0, 69, 70, 71, 140, 141, 0, 1, 5]
    parts = [0, 1, 9, 10, 99, 100, 2 ** 31 - 1]
    n_rec = len(lengths) * len(names)
    lens = [lengths[k % len(lengths)] for k in range(n_rec)]
    seq = bytearray(rng.choice(np.frombuffer(b'ACGTUacgtuN', dtype=np.uint8), sum(lens)).tobytes())
    seq[:12] = b'TTtUTgTUAtTT'
    qual = rng.integers(33, 75, len(seq), dtype=np.uint8).tobytes()
    off = np.concatenate([[0], np.cumsum(lens)])
    read = [k % len(names) for k in range(n_rec)]
    part = [parts[k % len(parts)] for k in range(n_rec)]
    return seq, qual, off, read, part, names, rna


def _rec_len(n, name_len, fmt):
    return 6 + name_len + 2 * n if fmt == 'fastq' else 2 + name_len + n + (n + 69) // 70


def _alignment_sweep(lengths):
    """records of every length in `lengths` at every source alignment mod 16 and every FASTQ output alignment mod 16 of their
    bases: a filler record before each one sets both (its length the source alignment, its read's name length 0 .. 15 the
    output's).  Reads 0 .. 15 have names of those lengths; the records under test alternate between read 16 (DNA) and read 17
    (RNA), names of 3 bytes."""
    rng = np.random.default_rng(11)
    names = ['n' * k for k in range(16)] + ['dna', 'rna']
    rna = [False] * 16 + [False, True]
    lens, read = [], []
    src = out = 0
    for n in lengths:
        for sa in range(16):
            for oa in range(16):
                a = (sa - src) % 16
                lf = (oa - 5 - out - _rec_len(a, 0, 'fastq')) % 16
                lens += [a, n]
                read += [lf, 16 + (sa + oa) % 2]
                src += a + n
                out += _rec_len(a, lf, 'fastq') + _rec_len(n, 3, 'fastq')
    seq = rng.choice(np.frombuffer(b'ACGTUacgtuN', dtype=np.uint8), src).tobytes()
    qual = rng.integers(33, 75, src, dtype=np.uint8).tobytes()
    return seq, qual, np.concatenate([[0], np.cumsum(lens)]), read, [0] * len(read), names, rna


def test_sim_emit_hand_made_records(SW):
    R = _Raw(SW, *_hand_made())
    try:
        for fmt in ('fastq', 'fasta'):
            got, off = R.call(fmt)
            assert got == R.expected(fmt), fmt
            assert off[-1] == len(got) and off[0] == 0
        assert b'@a_2147483647 b\n' in got.replace(b'>', b'@') and b'@tab\there_9\n' in got.replace(b'>', b'@')
        assert b'UUtUUgUUAtUU' in R.call('fastq')[0]                # read 0 is RNA: T -> U only
    finally:
        R.free()


def test_sim_emit_alignment_sweep(SW):
    """lengths 0 .. 40 and about 100 at every source and output alignment mod 16 (warp_copy's head, body and tail)"""
    R = _Raw(SW, *_alignment_sweep(list(range(41)) + [100, 103]))
    try:
        got, off = R.call('fastq')
        assert got == R.expected('fastq')
        base = off[1::2] + 2 + 3                                 # where the bases of the records under test start
        assert set((base % 16).tolist()) == set(range(16)) and set((R.off[1:-1:2] % 16).tolist()) == set(range(16))
        assert R.call('fasta')[0] == R.expected('fasta')
    finally:
        R.free()


def test_sim_emit_one_bin_alone_is_its_slice(SW):
    """records [r0, r1) formatted alone -- sliced device arrays, d_off[0] > 0 -- give that slice of the whole call's bytes"""
    R = _Raw(SW, *_hand_made())
    try:
        for fmt in ('fastq', 'fasta'):
            whole, off = R.call(fmt)
            for r0, r1 in ((0, 7), (7, 31), (31, R.n_rec), (12, 13), (20, 20)):
                got, o = R.call(fmt, r0, r1)
                assert got == whole[off[r0]:off[r1]] and np.array_equal(o, off[r0:r1 + 1] - off[r0])
    finally:
        R.free()


def test_sim_emit_zero_records(SW):
    R = _Raw(SW, *_hand_made())
    try:
        for fmt in ('fastq', 'fasta'):
            got, off = R.call(fmt, 0, 0)
            assert got == b'' and off.tolist() == [0]
        got, off = R.call('fastq', 0, 0, cap=0, d_out_ptr=0)
        assert got == b'' and off.tolist() == [0]
    finally:
        R.free()


def test_sim_emit_out_cap_one_byte_short(SW):
    R = _Raw(SW, *_hand_made())
    try:
        for fmt in ('fastq', 'fasta'):
            whole, off = R.call(fmt)
            with pytest.raises(SW.EngineError) as e:
                R.call(fmt, cap=len(whole) - 1)
            assert e.value.code == SW.ERR_SPACE and e.value.n_out_bytes == len(whole)
            assert R.untouched() and np.array_equal(R.D.host(R.out_off), off)
            assert R.call(fmt, cap=len(whole))[0] == whole
    finally:
        R.free()


def test_sim_emit_reads_retries_from_a_tiny_bound(SW, monkeypatch):
    from porechop_b200 import device_reads
    batch, sets, scheme, o, bc, fmt, _ = _golden('bins_default')
    _, _, exp = _run(SW, monkeypatch, batch, sets, scheme, o, ('fastq', 'fasta'), bc=bc)
    caps = []
    orig = SW.pb200_emit_reads_device
    monkeypatch.setattr(SW, 'pb200_emit_reads_device', lambda *a, **k: caps.append(k['out_cap']) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_out_cap', lambda *a: 5)
    _, _, got = _run(SW, monkeypatch, batch, sets, scheme, o, ('fastq', 'fasta'), bc=bc)
    assert caps == [5, len(exp['fastq'][0]), 5, len(exp['fasta'][0])]
    for fmt in ('fastq', 'fasta'):
        assert got[fmt][0] == exp[fmt][0] and got[fmt][2] == exp[fmt][2] and np.array_equal(got[fmt][1], exp[fmt][1])


# ---- errors ------------------------------------------------------------------------------------------------------------------
def test_sim_emit_host_preconditions_fail_before_any_launch(SW):
    R = _Raw(SW, *_hand_made())
    try:
        R.call('fastq')
        d = R.d
        bad = [dict(fmt='fastq', d_qual_ptr=0), dict(seq_bytes=-1), dict(n_reads=-1), dict(name_bytes=-1), dict(out_cap=-1),
               dict(d_out_off_ptr=0), dict(d_seq_ptr=0), dict(d_names_ptr=0), dict(d_name_off_ptr=0), dict(d_out_ptr=0),
               dict(d_off_ptr=0), dict(d_read_ptr=0), dict(d_part_ptr=0)]
        for kw in bad:
            n0 = SW.kernel_launches()
            with pytest.raises(SW.EngineError) as e:
                R.call(**kw)
            assert e.value.code == SW.ERR_ARG and SW.kernel_launches() == n0 and R.untouched(), kw
        n_out = ctypes.c_int64(-1)
        args = SW.EmitArgsDesc(d['seq'].ptr, d['qual'].ptr, len(R.seq), d['off'].ptr, d['read'].ptr, d['part'].ptr, d['names'].ptr,
                               d['name_off'].ptr, len(R.name_off) - 1, len(R.name_buf), None, 0, R.out.ptr, R.cap,
                               R.out_off.ptr, ctypes.addressof(n_out))
        n0 = SW.kernel_launches()
        assert SW.C_LIB.pb200EmitReadsDevice(None, R.n_rec, None) == SW.ERR_ARG
        assert SW.C_LIB.pb200EmitReadsDevice(ctypes.byref(args), -1, None) == SW.ERR_ARG and n_out.value == 0
        for f in (2, -1):
            args.fmt = f
            assert SW.C_LIB.pb200EmitReadsDevice(ctypes.byref(args), R.n_rec, None) == SW.ERR_ARG
        args.fmt, args.n_out_bytes = 0, None
        assert SW.C_LIB.pb200EmitReadsDevice(ctypes.byref(args), R.n_rec, None) == SW.ERR_ARG
        assert SW.kernel_launches() == n0
        # FASTA needs no qualities; the RNA flags may be absent
        assert R.call('fasta', d_qual_ptr=0)[0] == R.expected('fasta')
        R.rna[:] = False
        assert R.call('fastq', d_rna_ptr=0)[0] == R.expected('fastq')
    finally:
        R.free()


def test_sim_emit_device_checks_leave_the_output_untouched(SW):
    seq, qual, off, read, part, names, rna = _hand_made()
    n_reads, n_bytes = len(names), len(seq)
    name_bytes = sum(len(n) for n in names)
    cases = []
    for k, v in ((5, n_reads), (9, -1)):
        r = list(read)
        r[k] = v
        cases.append(dict(read=r))
    p = list(part)
    p[3] = -2
    cases.append(dict(part=p))
    o = off.copy()
    o[4] = o[3] - 1                                          # decreasing offsets
    cases.append(dict(off=o))
    o = off.copy()
    o[-1] = n_bytes + 1                                      # past seq_bytes
    cases.append(dict(off=o))
    o = off.copy()
    o[0] = -1
    cases.append(dict(off=o))
    for case in cases:
        a = dict(seq=seq, qual=qual, off=off, read=read, part=part, names=names, rna=rna)
        a.update(case)
        R = _Raw(SW, a['seq'], a['qual'], a['off'], a['read'], a['part'], a['names'], a['rna'])
        try:
            for fmt in ('fastq', 'fasta'):
                with pytest.raises(SW.EngineError) as e:
                    R.call(fmt)
                assert e.value.code == SW.ERR_ARG and R.untouched(), (case, fmt)
        finally:
            R.free()
    R = _Raw(SW, seq, qual, off, read, part, names, rna)      # a name range past name_bytes
    try:
        with pytest.raises(SW.EngineError) as e:
            R.call('fastq', name_bytes=name_bytes - 1)
        assert e.value.code == SW.ERR_ARG and R.untouched()
        assert R.call('fastq', name_bytes=name_bytes)[0] == R.expected('fastq')
    finally:
        R.free()


# ---- streams ---------------------------------------------------------------------------------------------------------------
def test_sim_emit_after_a_split_call_on_another_stream(SW):
    """records cut by adapterTrimSplitReadsDevice on stream A are formatted on stream B with no synchronisation in between;
    then inputs uploaded on the legacy default stream are formatted on the library's own stream (NULL)"""
    from porechop_b200 import fastq
    from test_trim_reads import trim_reads_set
    from test_trim_split_reads import _Raw as SplitRaw
    batch = _batch(trim_reads_set()[:12])
    A, B = SW.stream_create(), SW.stream_create()
    S = SplitRaw(SW, batch)
    try:
        assert SW.C_LIB.adapterTrimSplitReadsDevice(S.d_seq.ptr, S.d_off.ptr, S.n, S.nbytes, -1, ctypes.byref(S.args),
                                                    ctypes.byref(S.split), *DEFAULT, ctypes.c_void_p(A)) == 0
        k, nb = S.n_parts.value, S.n_bases.value
        names, name_off, rna = _names(S.D, batch)
        cap = 4 * nb + 64 * k + 64
        out, out_off = S.D.empty(cap, np.uint8), S.D.empty(k + 1, np.int64)
        o = S.out
        n = SW.pb200_emit_reads_device(k, d_seq_ptr=o['seq'].ptr, d_qual_ptr=o['qual'].ptr, seq_bytes=nb, d_off_ptr=o['off'].ptr,
                                       d_read_ptr=o['read'].ptr, d_part_ptr=o['part'].ptr, d_names_ptr=names.ptr,
                                       d_name_off_ptr=name_off.ptr, n_reads=len(batch), name_bytes=len(batch.name_buf),
                                       d_rna_ptr=rna.ptr, fmt='fastq', d_out_ptr=out.ptr, out_cap=cap, d_out_off_ptr=out_off.ptr,
                                       stream_ptr=B)
        got = S.D.host(S.D.head(out, n)).tobytes()
        assert got == fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, S.records(), 'fastq') and k > 0
        names2 = S.D.empty(len(batch.name_buf), np.uint8)
        SW.upload(names2.ptr, batch.name_buf.ctypes.data, len(batch.name_buf), 1)      # the legacy default stream
        n2 = SW.pb200_emit_reads_device(k, d_seq_ptr=o['seq'].ptr, d_qual_ptr=o['qual'].ptr, seq_bytes=nb, d_off_ptr=o['off'].ptr,
                                        d_read_ptr=o['read'].ptr, d_part_ptr=o['part'].ptr, d_names_ptr=names2.ptr,
                                        d_name_off_ptr=name_off.ptr, n_reads=len(batch), name_bytes=len(batch.name_buf),
                                        d_rna_ptr=rna.ptr, fmt='fastq', d_out_ptr=out.ptr, out_cap=cap, d_out_off_ptr=out_off.ptr)
        assert n2 == n and S.D.host(S.D.head(out, n)).tobytes() == got
    finally:
        S.D.free()


# ---- AddressSanitizer -------------------------------------------------------------------------------------------------------
def _asan_body():
    """the golden and hand-made cases on exact-size "device" heap blocks (run by test_sim_emit_under_address_sanitizer in a
    process with the ASan build of the simulated engine)"""
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
    for case in ('default', 'fasta_split', 'no_split_fasta'):
        mp = MP()
        test_sim_emit_golden_trim_cases(W, mp, case)
        mp.close()
    mp = MP()
    test_sim_emit_golden_barcode_cases(W, mp, 'bins_default')
    mp.close()
    test_sim_emit_hand_made_records(W)
    test_sim_emit_alignment_sweep(W)
    test_sim_emit_one_bin_alone_is_its_slice(W)
    test_sim_emit_zero_records(W)
    test_sim_emit_out_cap_one_byte_short(W)
    test_sim_emit_host_preconditions_fail_before_any_launch(W)
    test_sim_emit_device_checks_leave_the_output_untouched(W)
    print('ASAN RUN COMPLETE')


@pytest.mark.skipif(os.environ.get('PB200_SIM_ASAN', '0') != '1', reason='minutes: set PB200_SIM_ASAN=1')
def test_sim_emit_under_address_sanitizer():
    import build_sim
    lib = build_sim.build_asan()
    asan = subprocess.check_output(['gcc', '-print-file-name=libasan.so']).decode().strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS='detect_leaks=0:detect_stack_use_after_return=0', PB200_SIM_ASAN_LIB=lib)
    code = ('import os, sys; sys.path[:0] = [%r, %r, %r]; import build_sim; '
            'build_sim.build = lambda force=False, flags=None: os.environ["PB200_SIM_ASAN_LIB"]; '
            'import test_emit_reads as T; T._asan_body()') % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and 'ASAN RUN COMPLETE' in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    assert 'ERROR: AddressSanitizer' not in r.stderr
