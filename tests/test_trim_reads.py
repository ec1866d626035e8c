"""Whole-read trimming in one engine call (include/porechop_b200.h adapterTrimReads / adapterTrimReadsDevice): Phase B over
end windows cut on the device, then Phase C over the trimmed reads the device made from the trims.  CPU tier: the product's
engine code on the host simulator (tests/sim) against the record path (trim_end_adapters without device decisions +
find_middle_hits with the host rounds), the two-call device path and the reference CLI's bytes.  The GPU tier is
tests/test_gpu_trim_reads.py."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest

from helpers import ROOT

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

DEFAULT = (3, -6, -5, -2)
LINEAR = (3, -6, -5, -5)


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


def _batch(reads):
    from porechop_b200 import fastq
    text = ''.join('@r%d\n%s\n+\n%s\n' % (k, r, '5' * len(r)) for k, r in enumerate(reads))
    return fastq.parse_fastq(text.encode())


def trim_reads_set(seed=11):
    """reads for the trim rules and the middle scan: adapters at either end of reads shorter and longer than end_size,
    start trims past the end of the read, end trims that wrap (Python's negative slice), trimmed reads that are empty,
    chimeras with repeated hits of both adapters, non-ACGT bytes, empty reads"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    rng = random.Random(seed)

    def rnd(k):
        return ''.join(rng.choice('ACGT') for _ in range(k))
    reads = ['', 'A', rnd(10) + yt, rnd(3) + yt + rnd(2), rnd(30) + yb + rnd(40), rnd(50) + yb + rnd(20), yt + rnd(30) + yb,
             yt + rnd(120) + yb, yt + rnd(200) + yt + rnd(60) + yb + yb + rnd(300) + yb, rnd(60) + yt + yt + rnd(500) + yb + yb,
             yt[:12] + yt[12:].lower() + 'NNNN' + rnd(90) + yb.replace('A', 'U'), 'X' + yt + '-' * 5 + rnd(80) + yt + 'n' * 7,
             rnd(400) + yt + rnd(160) + yb + rnd(210) + yb, yb + yb + yb, yt * 3, 'N' * 170, rnd(155) + yb]
    for _ in range(16):
        parts = [rng.choice(('', yt, yt[4:]))]
        for _ in range(rng.randint(0, 3)):
            parts += [rnd(rng.randint(0, 260)), rng.choice((yt, yb, yb[:-3]))]
        parts += [rnd(rng.randint(0, 80)), rng.choice(('', yb, yb[:-5]))]
        reads.append(''.join(parts))
    return reads


def _record_path(W, batch, starts, ends, mids, scheme, end_size, thr_mid, cols, names, monkeypatch):
    """what the fused call must return, from the record path: trims, full-adapter identities of the score columns (or
    their ranking) and the middle hits"""
    from porechop_b200 import fastq
    from porechop_b200.align import scores_from_records
    monkeypatch.setattr(fastq, 'W', W)
    st, et, srec, erec = fastq.trim_end_adapters(batch, starts, ends, scheme, end_size, 2, 75.0, 4, device_decisions=False)
    hits = fastq.find_middle_hits(batch, st, et, mids, thr_mid, scheme, device=False) if mids else {}
    scores = []
    for rec, c in zip((srec, erec), cols):
        n = len(batch)
        full = scores_from_records(rec[:, c, :].reshape(-1, 9))[0].reshape(n, len(c)) if len(c) else np.zeros((n, 0))
        scores.append(fastq.top2_from_scores(full) if names else full)
    return st, et, scores, hits


def _fused(W, batch, starts, ends, mids, scheme, end_size, thr_mid, cols, names):
    from porechop_b200 import fastq
    pk = lambda x: W.pack_sequences(x, offset_dtype=np.int32)    # noqa: E731
    middle = pk([m[1] for m in mids]) if mids else None
    st, et, ss, es, n_hits, h = W.adapter_trim_reads(batch.seq, batch.seq_off, pk(starts) + (cols[0],), pk(ends) + (cols[1],),
                                                     middle, scheme, end_size, 2, 75.0, 4, thr_mid, want_top2=bool(names))
    scores = []
    for s, c, nm in zip((ss, es), cols, names or (None, None)):
        scores.append(fastq.Top2Scores(nm, s).ranked() if names else fastq.PairScores(c, s).full(c))
    return st, et, scores, fastq._hits_dict(n_hits, h), (st, et, ss, es, n_hits, h)


def _same(a, b):
    if isinstance(a, tuple):
        return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))
    return np.array_equal(a, b)


def _compare(W, monkeypatch, scheme=DEFAULT, end_size=150, sides='both', middle=True, barcodes=0, top2=False, thr_mid=85.0,
             reads=None):
    """the fused host call against the record path; returns the fused call's raw outputs"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    batch = _batch(reads or trim_reads_set())
    starts = [yt] if sides in ('both', 'start') else []
    ends = [yb] if sides in ('both', 'end') else []
    cols, names = ([], []), None
    if barcodes:
        bs, be = wl.demux_adapters()
        starts, ends = starts + bs[:barcodes], ends + be[:barcodes]
        cols = (list(range(1, 1 + barcodes)), list(range(1, 1 + barcodes)))
        names = (['s%d' % k for k in cols[0]], ['e%d' % k for k in cols[1]]) if top2 else None
    mids = [('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb)] if middle else []
    exp = _record_path(W, batch, starts, ends, mids, scheme, end_size, thr_mid, cols, names, monkeypatch)
    got = _fused(W, batch, starts, ends, mids, scheme, end_size, thr_mid, cols, names)
    assert np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1])
    assert all(_same(g, e) for g, e in zip(got[2], exp[2]))
    assert got[3] == exp[3]
    return batch, got[4]


def test_sim_fused_call_equals_record_path(SW, monkeypatch):
    from porechop_b200 import fastq
    batch, (st, et, _, _, n_hits, _) = _compare(SW, monkeypatch)
    lens = batch.lengths()
    a, b = fastq.trimmed_ranges(lens, st, et)
    assert (st > lens).any()                                  # start trims past the end of the read
    assert ((et > lens) & (et < 2 * lens) & (b > 0)).any()    # end trims that wrap around
    assert ((b == a) & (lens > 0)).any()                      # trimmed reads that are empty
    assert n_hits.max() >= 3 and (st > 0).sum() >= 5 and (et > 0).sum() >= 5
    _compare(SW, monkeypatch, scheme=LINEAR)
    _compare(SW, monkeypatch, thr_mid=60.0)


@pytest.mark.parametrize('end_size', [200, 400])
def test_sim_fused_call_two_pass_windows(SW, monkeypatch, end_size):
    """windows longer than direct_max: encoded first, then the score pass + bounded windows"""
    _compare(SW, monkeypatch, end_size=end_size)


def test_sim_fused_call_argument_sets(SW, monkeypatch):
    _compare(SW, monkeypatch, sides='start')
    _compare(SW, monkeypatch, sides='end')
    _compare(SW, monkeypatch, middle=False)
    _compare(SW, monkeypatch, sides='end', middle=False)


def test_sim_fused_call_barcode_columns(SW, monkeypatch):
    reads = trim_reads_set()[:20]
    _compare(SW, monkeypatch, barcodes=4, reads=reads)
    _compare(SW, monkeypatch, barcodes=4, top2=True, reads=reads)


def test_sim_fused_call_equals_the_two_device_calls(SW):
    """the same bytes as adapterEndDecisions + adapterMiddleScan on seq[st : len - et]"""
    from porechop_b200 import fastq, workloads as wl
    yt, yb = wl.nsk007()
    batch = _batch(trim_reads_set())
    sa, so = wl.pack_adapters([yt])
    ea, eo = wl.pack_adapters([yb])
    ma, mo = wl.pack_adapters([yt, yb])
    (sw, swo), (ew, ewo) = fastq.end_windows(batch.seq, batch.seq_off, 150)
    (st, sp, _), (et, ep, _) = SW.adapter_end_decisions([(sw, swo, sa, so, True, [0]), (ew, ewo, ea, eo, False, [0])], DEFAULT, 150,
                                                        2, 75.0, 4)
    a, b = fastq.trimmed_ranges(batch.lengths(), st, et)
    tb, to = fastq._gather_ranges(batch.seq, batch.seq_off[:-1] + a, batch.seq_off[:-1] + b)
    n_hits, h = SW.adapter_middle_scan(tb, to, ma, mo, DEFAULT, 85.0)
    got = SW.adapter_trim_reads(batch.seq, batch.seq_off, (sa, so, [0]), (ea, eo, [0]), (ma, mo), DEFAULT, 150, 2, 75.0, 4, 85.0)
    for g, e in zip(got, (st, et, sp, ep, n_hits, h)):
        assert g.dtype == e.dtype and np.array_equal(g, e)


def _device_copy(W, buf, off):
    d_seq, d_off = W.device_alloc(len(buf) + 16), W.device_alloc(off.nbytes)
    W.upload(d_seq, buf.ctypes.data, len(buf), None)
    W.upload(d_off, off.ctypes.data, off.nbytes, None)
    return d_seq, d_off


def _read_back(addr, n, dtype):
    return np.frombuffer((ctypes.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(addr), dtype=dtype).copy()


def test_sim_device_variant_equals_host_variant_and_leaves_the_reads(SW):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    batch = _batch(trim_reads_set())
    buf, off = np.ascontiguousarray(batch.seq), np.ascontiguousarray(batch.seq_off)
    sides = (wl.pack_adapters([yt]) + ([0],), wl.pack_adapters([yb]) + ([0],))
    mid = wl.pack_adapters([yt, yb])
    exp = SW.adapter_trim_reads(buf, off, sides[0], sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0)
    d_seq, d_off = _device_copy(SW, buf, off)
    try:
        for max_len, stream in ((int(np.diff(off).max()), SW.stream_create()), (-1, 0)):
            got = SW.adapter_trim_reads_device(d_seq, d_off, len(off) - 1, len(buf), max_len, sides[0], sides[1], mid, DEFAULT, 150,
                                               2, 75.0, 4, 85.0, stream_ptr=stream or 0)
            assert all(np.array_equal(g, e) for g, e in zip(got, exp))
        assert np.array_equal(_read_back(d_seq, len(buf), np.uint8), buf)
        assert np.array_equal(_read_back(d_off, len(off), np.int64), off)
    finally:
        SW.device_free(d_seq)
        SW.device_free(d_off)


def test_sim_several_segments_give_the_same_results(SW):
    """PB_TEST_SEGMENT_READS=7: the 33 reads run as 5 segments -- hits, trims and scores as in one segment"""
    import sim_engine
    from porechop_b200 import workloads as wl
    W7 = sim_engine.load(['-DPB_TEST_SEGMENT_READS=7'])
    yt, yb = wl.nsk007()
    batch = _batch(trim_reads_set())
    buf, off = np.ascontiguousarray(batch.seq), np.ascontiguousarray(batch.seq_off)
    assert len(off) - 1 > 28
    sides = (wl.pack_adapters([yt]) + ([0],), wl.pack_adapters([yb]) + ([0],))
    mid = wl.pack_adapters([yt, yb])
    for end_size in (150, 200):
        exp = SW.adapter_trim_reads(buf, off, sides[0], sides[1], mid, DEFAULT, end_size, 2, 75.0, 4, 70.0)
        got = W7.adapter_trim_reads(buf, off, sides[0], sides[1], mid, DEFAULT, end_size, 2, 75.0, 4, 70.0)
        assert all(np.array_equal(g, e) for g, e in zip(got, exp))
        assert exp[4].sum() > 10
    d_seq, d_off = _device_copy(W7, buf, off)
    try:
        got = W7.adapter_trim_reads_device(d_seq, d_off, len(off) - 1, len(buf), -1, sides[0], sides[1], mid, DEFAULT, 200, 2, 75.0,
                                           4, 70.0)
        assert all(np.array_equal(g, e) for g, e in zip(got, exp))
    finally:
        W7.device_free(d_seq)
        W7.device_free(d_off)
    n, text = W7.races()
    assert n == 0, text[:4000]


def test_sim_hits_cap_too_small_reports_the_total_after_the_trims(SW):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    batch = _batch(trim_reads_set())
    buf, off = np.ascontiguousarray(batch.seq), np.ascontiguousarray(batch.seq_off)
    sa, so = wl.pack_adapters([yt])
    ea, eo = wl.pack_adapters([yb])
    ma, mo = wl.pack_adapters([yt, yb])
    st, et, _, _, n_hits, hits = SW.adapter_trim_reads(buf, off, (sa, so, []), (ea, eo, []), (ma, mo), DEFAULT, 150, 2, 75.0, 4, 85.0)
    n = len(off) - 1
    trims = [np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)]
    nh, small, total = np.zeros(n, dtype=np.int32), np.zeros((2, 10), dtype=np.int32), ctypes.c_int64(0)
    sides = [SW.TrimSideDesc(a.ctypes.data, o.ctypes.data, 1, None, 0, t.ctypes.data, None, None)
             for (a, o), t in zip(((sa, so), (ea, eo)), trims)]
    args = SW.TrimArgsDesc(150, 2, 4, 75.0, sides[0], sides[1], ma.ctypes.data, mo.ctypes.data, 2, 85.0, nh.ctypes.data,
                           small.ctypes.data, 2, ctypes.addressof(total))
    rc = SW.C_LIB.adapterTrimReads(buf.ctypes.data, off.ctypes.data, n, ctypes.byref(args), *DEFAULT)
    assert rc == SW.ERR_SPACE and total.value == len(hits) > 2
    assert np.array_equal(nh, n_hits) and np.array_equal(trims[0], st) and np.array_equal(trims[1], et)


def test_sim_preconditions_fail_before_any_launch(SW):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    batch = _batch(trim_reads_set()[:6])
    buf, off = np.ascontiguousarray(batch.seq), np.ascontiguousarray(batch.seq_off)
    s = wl.pack_adapters([yt]) + ([0],)
    e = wl.pack_adapters([yb]) + ([0],)
    m = wl.pack_adapters([yt, yb])
    ok = dict(start=s, end=e, middle=m, scoring_scheme_vals=DEFAULT, end_size=150, extra_trim_size=2, end_threshold=75.0,
              min_trim_size=4, middle_threshold=85.0)
    bad = [dict(end_size=0), dict(end_size=-3), dict(end_threshold=-1.0), dict(end_threshold=float('nan')),
           dict(middle_threshold=0.0), dict(middle_threshold=float('nan')),
           dict(middle=wl.pack_adapters([yt, yb[:8] + 'N' + yb[9:]])),         # middle adapter outside A/C/G/T/U
           dict(scoring_scheme_vals=(3, -6, 0, -2)),                           # no window bound
           dict(scoring_scheme_vals=(3, -6, 1, -2)),                           # generic int32 scheme
           dict(start=wl.pack_adapters([yt]) + ([1],)),                        # score column out of range
           dict(end=wl.pack_adapters(['A' * 300]) + ([],)),                    # adapter outside the int16 classes
           dict(end_size=65530)]                                               # windows too long for the decision tables
    for kw in bad:
        n0 = SW.kernel_launches()
        with pytest.raises(SW.EngineError) as err:
            SW.adapter_trim_reads(buf, off, **dict(ok, **kw))
        assert err.value.code == SW.ERR_ARG, kw
        assert SW.kernel_launches() == n0, kw
    n0 = SW.kernel_launches()
    with pytest.raises(SW.EngineError) as err:
        SW.adapter_trim_reads(buf, off, want_top2=True, **dict(ok, end_size=4090))      # top2 keys need windows < 4096
    assert err.value.code == SW.ERR_ARG and SW.kernel_launches() == n0


def test_sim_flat_pipeline_falls_back_to_the_two_calls_on_err_arg(SW, monkeypatch):
    from porechop_b200 import fastq, workloads as wl
    monkeypatch.setattr(fastq, 'W', SW)
    monkeypatch.setattr(fastq, 'DEVICE_DECISIONS', True)
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
    yt, yb = wl.nsk007()
    reads = trim_reads_set()[:20]
    text = ''.join('@r%d\n%s\n+\n%s\n' % (k, r, '5' * len(r)) for k, r in enumerate(reads)).encode()
    calls = []
    orig = SW.adapter_trim_reads

    def spy(*a, **k):
        try:
            r = orig(*a, **k)
        except SW.EngineError as e:
            calls.append(e.code)
            raise
        calls.append(0)
        return r
    monkeypatch.setattr(SW, 'adapter_trim_reads', spy)
    for scheme, sets in ((DEFAULT, [(('t', yt), ('b', yb[:8] + 'N' + yb[9:]))]),      # middle adapter the device scan refuses
                         ((3, -6, 0, -2), [(('t', yt), ('b', yb))])):                # no window bound
        calls.clear()
        fused, _ = fastq.trim_fastq(text, sets, scheme)
        assert calls == [SW.ERR_ARG]
        monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', False)
        two, _ = fastq.trim_fastq(text, sets, scheme)
        monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
        assert fused == two and len(calls) == 1


def test_sim_trim_and_demux_reproduce_the_reference_cli_in_one_call_per_chunk(SW, monkeypatch):
    """the flat pipeline with both device switches on: the reference CLI's files byte for byte, one adapterTrimReads call per
    chunk and no adapterEndDecisions / adapterMiddleScan call"""
    from porechop_b200 import fastq
    import test_fastq_emit as T
    monkeypatch.setattr(fastq, 'W', SW)
    monkeypatch.setattr(fastq, 'DEVICE_DECISIONS', True)
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
    calls = {'trim': 0, 'other': 0}
    orig = SW.adapter_trim_reads
    monkeypatch.setattr(SW, 'adapter_trim_reads', lambda *a, **k: calls.__setitem__('trim', calls['trim'] + 1) or orig(*a, **k))
    for name in ('adapter_end_decisions', 'adapter_middle_scan', 'adapter_middle_scan_device'):
        f = getattr(SW, name)
        monkeypatch.setattr(SW, name, lambda *a, _f=f, **k: calls.__setitem__('other', calls['other'] + 1) or _f(*a, **k))
    runs = 0
    for case in T.CASES:
        T._run(case)
        runs += 1
    for case in T.BARCODE_CASES:
        T._run_demux(case)
        runs += 1
    assert calls == {'trim': runs, 'other': 0}
