"""FASTQ / FASTA parsed on the device (include/porechop_b200.h pb200ParseReadsDevice, device_reads.parse_reads) and whole chunks
from input bytes to output bytes (device_reads.trim_fastq / demux_fastq).  CPU tier: the product's engine code on the host
simulator (tests/sim) against the host parser (fastq.parse_fastq / parse_fasta) field for field, and against the reference
CLI's files.  The GPU tier is tests/test_gpu_parse_reads.py."""
import os
import random
import sys

import numpy as np
import pytest

from helpers import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

from test_trim_split_reads import SimDevice  # noqa: E402

WS = [9, 11, 12, 13, 28, 29, 30, 31, 32]          # stripped inside a line (10 ends it)
TILE = 8192                                        # PB_PARSE_TILE


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


@pytest.fixture
def sim(SW, monkeypatch):
    """device_reads, and the host path it falls back to, on the simulated engine"""
    from porechop_b200 import device_reads, fastq
    D = SimDevice(SW)
    monkeypatch.setattr(device_reads, 'W', SW)
    monkeypatch.setattr(fastq, 'W', SW)
    monkeypatch.setattr(device_reads, '_device', D)
    yield D
    D.free()


def _device_parse(D, data, kind=None, qual=True):
    """parse_reads on the simulator; host copies of every field"""
    from porechop_b200 import device_reads
    p = device_reads.parse_reads(D.upload(np.frombuffer(data, dtype=np.uint8)), kind, qual)
    return tuple(D.host(x) if x is not None else None for x in p[:6]) + (p.kind,)


def _host_parse(data, kind):
    from porechop_b200 import fastq
    return fastq.parse_fastq(data) if kind == 'fastq' else fastq.parse_fasta(data)


def _check(D, data, kind, qual=True):
    """the device parse equals the host parser on every field"""
    b = _host_parse(data, kind)
    names, name_off, seq, seq_off, q, rna, k = _device_parse(D, data, kind, qual)
    assert k == kind
    assert names.tobytes() == b.name_buf.tobytes() and np.array_equal(name_off, b.name_off)
    assert seq.tobytes() == b.seq.tobytes() and np.array_equal(seq_off, b.seq_off)
    assert np.array_equal(rna.astype(bool), b.rna)
    if qual:
        assert np.array_equal(b.qual_off, b.seq_off) and q.tobytes() == b.qual.tobytes()
    else:
        assert q is None
    return b


def _error(fn):
    try:
        fn()
    except ValueError as e:
        return type(e), str(e)
    return None


def to_fasta(batch, width=7, blank=True):
    """a FastqBatch as multi-line FASTA text: `width` bases a line, with blank and whitespace-only lines between records"""
    out = []
    nb = batch.name_buf.tobytes()
    for i in range(len(batch)):
        out.append(b'>' + nb[batch.name_off[i]:batch.name_off[i + 1]] + b'\n')
        s = batch.seq[batch.seq_off[i]:batch.seq_off[i + 1]].tobytes()
        out += [s[j:j + width] + b'\n' for j in range(0, len(s), width)]
        if blank and i % 2:
            out.append(b'\n \t\n')
    return b''.join(out)


# ---- golden inputs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('key', ['input_fastq', 'barcoded_fastq'])
def test_sim_parse_golden_inputs(sim, key):
    data = load_golden('golden_emit.json')[key].encode()
    b = _check(sim, data, 'fastq')
    assert len(b) > 10 and b.rna.any() == (key == 'input_fastq')
    _check(sim, data, 'fastq', qual=False)
    for width in (7, 70, 1000):
        _check(sim, to_fasta(b, width), 'fasta')
    _check(sim, to_fasta(b, 70).replace(b'\n', b'\r\n'), 'fasta', qual=False)


def test_sim_parse_kind_from_first_byte(sim):
    from porechop_b200 import device_reads
    assert _device_parse(sim, b'@a\nAC\n+\nII\n')[6] == 'fastq'
    assert _device_parse(sim, b'>a\nAC\n')[6] == 'fasta'
    assert _device_parse(sim, b'')[6] == 'fastq'
    with pytest.raises(ValueError, match='File is neither FASTA or FASTQ'):
        _device_parse(sim, b'#a\n')
    with pytest.raises(ValueError, match="kind must be"):
        device_reads.parse_reads(sim.upload(np.zeros(1, np.uint8)), 'sam')


# ---- line endings, whitespace, case, RNA -----------------------------------------------------------------------------------
FASTQ_CASES = [
    b'@r1 a b\r\nACGT\r\n+\r\nIIII\r\n@r2\r\nacgu\r\n+\r\n!!!!\r\n',                       # CRLF
    b'@r1\nACGT\n+\nIIII\n@r2\nAC\n+\nII',                                                 # no final newline
    b'@r1\n\n+\n\n@r2\nA\n+\n\n',                                                           # empty bases and qualities
    b'@low\nacgtnx\n+\nIIIIII\n@rna\nUUUaG\n+\nIIIII\n@tie\nUUTT\n+\nIIII\n@dna\nUTT\n+\nIII\n',   # case, RNA, U = T tie
    b'@short\nACGTACGT\n+\nII\n@none\nACG\n+\n\n',                                          # qualities shorter than the bases
    b'@name with\tspaces and\ttabs \t\nAC\n+\nII\n@\t lead\nA\n+\nI\n',                      # spaces and tabs in names
]


@pytest.mark.parametrize('case', range(len(FASTQ_CASES)))
def test_sim_parse_fastq_cases(sim, case):
    _check(sim, FASTQ_CASES[case], 'fastq')
    _check(sim, FASTQ_CASES[case], 'fastq', qual=False)


def test_sim_parse_rna_rules(sim):
    b = _check(sim, FASTQ_CASES[3], 'fastq')
    assert b.rna.tolist() == [False, True, False, False]
    assert b.seq.tobytes() == b'ACGTNX' + b'TTTAG' + b'UUTT' + b'UTT'


@pytest.mark.parametrize('c', WS)
def test_sim_parse_every_whitespace_class_on_every_line(sim, c):
    w = bytes([c])
    fq = b''.join([w + b'@r' + w + b'x' + w + b'\n', w + b'ACGT' + w + b'\n', w + b'+' + w + b'\n', w + b'IIII' + w + b'\n'] * 3)
    _check(sim, fq, 'fastq')
    fa = w + b'>r' + w + b'x' + w + b'\n' + w + b'ACG' + w + b'\n' + w + b'\n' + w + b'TT' + w + b'\n>s\n' + w + b'\n'
    _check(sim, fa, 'fasta')
    # bytes that are not stripped: non-ASCII whitespace and '\r' inside a line (no line break)
    _check(sim, b'@a\x85\nAC\xa0\n+\nI\rI\n', 'fastq')
    _check(sim, b'>a\rb\n\xa0ACGT\r\rAC\n', 'fasta')


def test_sim_parse_fasta_cases(sim):
    _check(sim, b'>empty\n>two lines\nAC\nGT\n\n>last\nacgu', 'fasta')          # a record without body lines; no final newline
    _check(sim, b'\n\n  \n>a\nAC\n', 'fasta')                                     # leading blank lines are dropped
    _check(sim, b'>a\n>b\n>c\n', 'fasta')


def test_sim_parse_empty_and_one_read(sim):
    for kind in ('fastq', 'fasta'):
        names, name_off, seq, seq_off, q, rna, _ = _device_parse(sim, b'', kind)
        assert len(names) == len(seq) == len(q) == len(rna) == 0 and name_off.tolist() == seq_off.tolist() == [0]
    _check(sim, b'\n\n\n', 'fasta')
    _check(sim, b'@one\nACGT\n+\nIIII\n', 'fastq')
    _check(sim, b'>one\nACGT\n', 'fasta')


def _record_ending_at(t):
    """a FASTQ record whose last '\\n' is at byte t (the record starts at byte 0): a name of 1 or 2 bytes sets the parity"""
    nm = b'x' * (1 + (t - 4) % 2)
    L = (t - 4 - len(nm)) // 2
    rec = b'@' + nm + b'\n' + b'ACGT' * (L // 4) + b'A' * (L % 4) + b'\n+\n' + b'I' * L + b'\n'
    assert rec.rindex(b'\n') == t, (t, len(rec))
    return rec


@pytest.mark.parametrize('t', [TILE - 33, TILE - 32, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE + 31])
def test_sim_parse_newline_on_tile_boundaries(sim, t):
    data = _record_ending_at(t) + b'@next\nAC\n+\nII\n'
    assert data[t] == 10
    _check(sim, data, 'fastq')
    fa = b'>' + b'n' * (t - 1) + b'\nACGT\n'                                       # the header's newline at t
    assert fa[t] == 10
    _check(sim, fa, 'fasta')


def test_sim_parse_read_longer_than_a_tile(sim):
    rng = np.random.default_rng(5)
    s = bytes(rng.choice(list(b'ACGTacgt'), 3 * TILE + 77))
    _check(sim, b'@long\n' + s + b'\n+\n' + b'#' * (len(s) - 9) + b'\n@x\nA\n+\nI\n', 'fastq')
    _check(sim, b'>long\n' + s + b'\n>x\nA\n', 'fasta')
    _check(sim, b'>wrapped\n' + b'\n'.join(s[j:j + 70] for j in range(0, len(s), 70)) + b'\n', 'fasta')


# ---- random inputs ---------------------------------------------------------------------------------------------------------
def _pad(r, kept=True):
    """0-2 bytes of stripped whitespace -- or, with kept, now and then 0xa0, which is not stripped"""
    return bytes(r.choice(WS + [0xa0] if kept else WS) for _ in range(r.choice([0, 0, 0, 1, 2])))


def random_fastq(r):
    eol = r.choice([b'\n', b'\r\n'])
    out = []
    for i in range(r.randint(0, 12)):
        name = bytes(r.choice(b'abcXYZ019_ \t:=') for _ in range(r.randint(0, 12)))
        bases = bytes(r.choice(b'ACGTUNacgtun' if r.random() < 0.5 else b'UUUTac') for _ in range(r.randint(0, 90)))
        q = bytes(r.randint(33, 73) for _ in range(max(0, len(bases) - r.choice([0, 0, 0, 1, 5]))))
        out += [_pad(r, False) + b'@' + name + _pad(r), _pad(r) + bases + _pad(r), b'+' + _pad(r), _pad(r) + q + _pad(r)]
    text = eol.join(out)
    return text + (eol if out and r.random() < 0.8 else b'')


def random_fasta(r):
    eol = r.choice([b'\n', b'\r\n'])
    out = [_pad(r, False) for _ in range(r.randint(0, 2))]
    for i in range(r.randint(0, 10)):
        out.append(_pad(r, False) + b'>' + bytes(r.choice(b'abcXYZ019_ \t') for _ in range(r.randint(1, 10))).strip(b' \t') + b'n')
        for _ in range(r.choice([0, 1, 2, 5])):
            out.append(_pad(r) + bytes(r.choice(b'ACGTUNacgtu') for _ in range(r.randint(0, 80))) + _pad(r))
            if r.random() < 0.2:
                out.append(_pad(r, False))
    text = eol.join(out)
    return text + (eol if out and r.random() < 0.8 else b'')


def test_sim_parse_random_inputs(sim):
    """(0xa0 padding is not stripped, so some quality lines come out longer than their bases: those chunks are refused with
    qualities and parsed without them)"""
    from porechop_b200 import device_reads
    r = random.Random(2024)
    refused = 0
    for i in range(200):
        kind = 'fastq' if i % 2 == 0 else 'fasta'
        data = random_fastq(r) if kind == 'fastq' else random_fasta(r)
        b = _host_parse(data, kind)
        qual = r.random() < 0.8
        if qual and not np.array_equal(b.qual_off, b.seq_off):
            with pytest.raises(device_reads.QualityTooLong) as ei:
                _device_parse(sim, data, kind)
            assert ei.value.index == np.flatnonzero(np.diff(b.qual_off) > np.diff(b.seq_off))[0]
            refused += 1
            qual = False
        _check(sim, data, kind, qual=qual)
    assert 0 < refused < 80


# ---- malformed input -------------------------------------------------------------------------------------------------------
MALFORMED = [('fastq', b'@only\n'), ('fastq', b'@a\nAC\n+\nII\n@b\nAC\n+\n'), ('fastq', b'@a\nAC\n+\nII\nb\nAC\n+\nII\n'),
             ('fastq', b'@a\nAC\n+\nII\n  \t\nAC\n+\nII\n'), ('fastq', b' x@a\nAC\n+\nII\n'), ('fastq', b'    '),
             ('fasta', b'ACGT\n>a\nAC\n'), ('fasta', b'\n  \nAC\n'), ('fasta', b'>a\nAC\n>\nAC\n'), ('fasta', b'>a\n> \t\nAC\n'),
             ('fasta', b'AC\n>\n')]


@pytest.mark.parametrize('case', range(len(MALFORMED)))
def test_sim_parse_malformed_raises_host_error(sim, case):
    kind, data = MALFORMED[case]
    exp = _error(lambda: _host_parse(data, kind))
    assert exp is not None
    assert _error(lambda: _device_parse(sim, data, kind)) == exp
    assert _error(lambda: _device_parse(sim, data, kind, qual=False)) == exp


def test_sim_parse_error_reason_and_index(SW, sim):
    """the raw binding reports the reason and the first bad record / line; nothing is written"""
    def call(data, fmt):
        d = sim.upload(np.frombuffer(data, dtype=np.uint8))
        outs = [sim.upload(np.full(64, 0x5A, np.uint8)) for _ in range(3)]
        offs = [sim.upload(np.full(8, 7, np.int64)) for _ in range(2)]
        with pytest.raises(SW.EngineError) as ei:
            SW.pb200_parse_reads_device(sim.ptr(d), len(data), fmt, d_names_ptr=sim.ptr(outs[0]), names_cap=64,
                                        d_name_off_ptr=sim.ptr(offs[0]), d_seq_ptr=sim.ptr(outs[1]), seq_cap=64,
                                        d_seq_off_ptr=sim.ptr(offs[1]), d_qual_ptr=sim.ptr(outs[2]),
                                        d_rna_ptr=sim.ptr(sim.upload(np.zeros(7, np.uint8))), reads_cap=7)
        assert all((sim.host(x) == 0x5A).all() for x in outs) and all((sim.host(x) == 7).all() for x in offs)
        return ei.value.code, ei.value.reason, ei.value.index
    assert call(b'@a\nAC\n+\nII\n@b\nAC\n+\nII\n@c\n', 'fastq') == (SW.ERR_ARG, SW.PARSE_LINES, 2)
    assert call(b'@a\nAC\n+\nII\n@b\nAC\n+\nII\nc\nAC\n+\nI\n@d\nA\n+\nII\n', 'fastq') == (SW.ERR_ARG, SW.PARSE_HEADER, 2)
    assert call(b'@a\nAC\n+\nII\n@b\nAC\n+\nIII\n', 'fastq') == (SW.ERR_ARG, SW.PARSE_LONG_QUAL, 1)
    assert call(b'\n\nAC\n>\n', 'fasta') == (SW.ERR_ARG, SW.PARSE_FASTA_START, 2)
    assert call(b'>a\nAC\n\n>\nAC\n>\n', 'fasta') == (SW.ERR_ARG, SW.PARSE_FASTA_NAME, 3)


def test_sim_parse_preconditions(SW, sim):
    d = sim.upload(np.frombuffer(b'@a\nA\n+\nI\n', dtype=np.uint8))
    off = sim.upload(np.zeros(4, np.int64))
    ok = dict(d_name_off_ptr=sim.ptr(off), d_seq_off_ptr=sim.ptr(off))
    for kw in (dict(ok, names_cap=-1), dict(ok, reads_cap=4), dict(ok, seq_cap=4), dict(d_name_off_ptr=sim.ptr(off))):
        with pytest.raises(SW.EngineError) as ei:
            SW.pb200_parse_reads_device(sim.ptr(d), 10, 'fastq', **kw)
        assert ei.value.code == SW.ERR_ARG and ei.value.reason == 0
    with pytest.raises(SW.EngineError):
        SW.pb200_parse_reads_device(0, 10, 'fastq', **ok)


# ---- a quality line longer than its bases ----------------------------------------------------------------------------------
def _long_qual_input():
    text = load_golden('golden_emit.json')['input_fastq']
    lines = text.split('\n')
    lines[7] += 'IIII'                                     # the second read's qualities
    return '\n'.join(lines).encode()


def test_sim_parse_long_quality_is_refused(sim):
    from porechop_b200 import device_reads
    data = _long_qual_input()
    with pytest.raises(device_reads.QualityTooLong) as ei:
        _device_parse(sim, data, 'fastq')
    assert ei.value.index == 1
    _check(sim, data, 'fastq', qual=False)                 # without qualities the read fits


def test_sim_trim_fastq_long_quality_falls_back_to_host(sim, monkeypatch):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['cases']['default']
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    data = _long_qual_input()
    calls = []
    host = fastq.trim_fastq
    monkeypatch.setattr(fastq, 'trim_fastq', lambda *a, **k: calls.append(1) or host(*a, **k))
    got, info = device_reads.trim_fastq(data, sets, c['scoring'], **o)
    exp, _ = host(data, sets, c['scoring'], **o)
    assert got == exp and calls == [1] and info['n_reads'] == len(fastq.parse_fastq(data))


# ---- ERR_SPACE ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('caps', [(1, 1, 1), (0, 0, 0), (1000, 1, 1000), (1000, 1000, 3)])
def test_sim_parse_space_retry(SW, sim, monkeypatch, caps):
    from porechop_b200 import device_reads
    monkeypatch.setattr(device_reads, 'initial_parse_caps', lambda n, kind: caps)
    n_calls = []
    raw = SW.pb200_parse_reads_device
    monkeypatch.setattr(SW, 'pb200_parse_reads_device', lambda *a, **k: n_calls.append(1) or raw(*a, **k))
    data = load_golden('golden_emit.json')['input_fastq'].encode()
    b = _check(sim, data, 'fastq')
    _check(sim, to_fasta(b), 'fasta')
    assert len(n_calls) == 4


def test_sim_parse_space_reports_exact_counts(SW, sim):
    data = b'@ab\nACGT\n+\nIIII\n@c\nA\n+\nI\n'
    d = sim.upload(np.frombuffer(data, dtype=np.uint8))
    off = [sim.upload(np.full(2, 9, np.int64)) for _ in range(2)]
    with pytest.raises(SW.EngineError) as ei:
        SW.pb200_parse_reads_device(sim.ptr(d), len(data), 'fastq', d_name_off_ptr=sim.ptr(off[0]), d_seq_off_ptr=sim.ptr(off[1]),
                                    d_rna_ptr=sim.ptr(sim.upload(np.zeros(1, np.uint8))), reads_cap=1,
                                    d_names_ptr=sim.ptr(sim.upload(np.zeros(3, np.uint8))), names_cap=3,
                                    d_seq_ptr=sim.ptr(sim.upload(np.zeros(5, np.uint8))), seq_cap=5)
    e = ei.value
    assert (e.code, e.n_reads, e.n_name_bytes, e.n_seq_bytes) == (SW.ERR_SPACE, 2, 3, 5)
    assert all((sim.host(x) == 9).all() for x in off)


# ---- whole chunks: input bytes -> output bytes ------------------------------------------------------------------------------
@pytest.mark.parametrize('case_name', ['default', 'small_parts', 'discard_middle', 'no_split_fasta', 'fasta_split'])
def test_sim_trim_fastq_golden(sim, monkeypatch, case_name):
    from porechop_b200 import device_reads, fastq
    monkeypatch.setattr(fastq, 'trim_fastq', None)         # the device path only
    g = load_golden('golden_emit.json')
    c = g['cases'][case_name]
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    got, info = device_reads.trim_fastq(g['input_fastq'].encode(), sets, c['scoring'], **o)
    assert got.decode() == c['output']
    assert info['n_reads'] == len(info['start_trim']) == len(info['end_trim']) > 0
    arr, _ = device_reads.trim_fastq(g['input_fastq'].encode(), sets, c['scoring'], as_array=True, kind='fastq', **o)
    assert arr.tobytes() == got


@pytest.mark.parametrize('case_name', ['bins_default', 'bins_two_barcodes', 'bins_loose_discard', 'bins_fasta_untrimmed'])
def test_sim_demux_fastq_golden(sim, monkeypatch, case_name):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases'][case_name]
    o = dict(c['options'])
    fmt = o['fmt']
    data = g['barcoded_fastq'].encode()
    exp_bins, exp_info = fastq.demux_fastq(data, c['matching_sets'], c['scoring'], **o)
    monkeypatch.setattr(fastq, 'demux_fastq', None)        # the device path only
    bins, info = device_reads.demux_fastq(data, c['matching_sets'], c['scoring'], **o)
    assert sorted(k + '.' + fmt for k in bins) == sorted(c['bins'])
    for k, v in bins.items():
        assert v.decode() == c['bins'][k + '.' + fmt], k
    assert info['calls'] == exp_info['calls'] and bins == exp_bins


def test_sim_demux_fastq_albacore_calls(sim):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases']['bins_default']
    o = dict(c['options'])
    data = g['barcoded_fastq'].encode()
    n = len(fastq.parse_fastq(data))
    exp, exp_info = fastq.demux_fastq(data, c['matching_sets'], c['scoring'], albacore_calls=['BC01'] * n, **o)
    got, info = device_reads.demux_fastq(data, c['matching_sets'], c['scoring'], albacore_calls='BC01', **o)
    assert got == exp and info['calls'] == exp_info['calls'] and set(info['calls']) <= {'BC01', 'none'}


def test_sim_trim_fastq_fasta_input(sim, monkeypatch):
    """FASTA input, FASTA and FASTQ output: the bytes fastq.trim_fastq writes for the host parse of the same bytes"""
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['cases']['small_parts']
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    data = to_fasta(fastq.parse_fastq(g['input_fastq'].encode()), 70)
    for fmt in ('fasta', 'fastq'):
        o['fmt'] = fmt
        exp, _ = fastq.trim_fastq(fastq.parse_fasta(data), sets, c['scoring'], **o)
        got, _ = device_reads.trim_fastq(data, sets, c['scoring'], **o)
        assert got == exp and got


def test_sim_trim_fastq_inputs_the_device_does_not_take(sim, monkeypatch):
    """no adapters, no reads, or a call that returns PB200_ERR_ARG: fastq.trim_fastq's bytes"""
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['cases']['default']
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    data = g['input_fastq'].encode()
    for s, d in (([], data), (sets, b''), ([(('bad', 'ACGTNNRY' * 2), None)], data)):
        exp, _ = fastq.trim_fastq(data if d else b'', s, c['scoring'], **o)
        got, _ = device_reads.trim_fastq(d, s, c['scoring'], **o)
        assert got == exp
    with pytest.raises(ValueError, match='FASTQ record does not start with @'):
        device_reads.trim_fastq(b'x\nA\n+\nI\n', sets, c['scoring'], kind='fastq', **o)
    with pytest.raises(ValueError, match='File is neither FASTA or FASTQ'):
        device_reads.trim_fastq(b'x\nA\n+\nI\n', sets, c['scoring'], **o)
