"""Demultiplexed output reads on the device (include/porechop_b200.h adapterDemuxReadsDevice, device_reads.demux_reads).  CPU
tier: the product's engine code on the host simulator (tests/sim) against the reference CLI's bin files and against
fastq.demux_fastq; the call rule through tests/emu against fastq.call_barcodes_top2.  The GPU tier is
tests/test_gpu_demux_reads.py."""
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

from test_trim_split_reads import SimDevice  # noqa: E402

DEFAULT = (3, -6, -5, -2)
BARCODE_KEYS = ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes', 'discard_unassigned')


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


def _golden(case_name):
    """(batch, sets, scheme, trim options, barcode options, fmt, expected bins) of a golden barcode case"""
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases'][case_name]
    o = dict(c['options'])
    fmt = o.pop('fmt')
    bc = {k: o.pop(k) for k in BARCODE_KEYS}
    return fastq.parse_fastq(g['barcoded_fastq'].encode()), c['matching_sets'], c['scoring'], o, bc, fmt, c['bins']


def _demux(W, monkeypatch, batch, sets, scheme, o, bc, fmt='fastq', albacore_calls=None):
    """device_reads.demux_reads on the simulated engine; returns (result with host copies of the records, {bin: bytes})"""
    from porechop_b200 import device_reads, fastq
    D = SimDevice(W)
    monkeypatch.setattr(device_reads, 'W', W)
    monkeypatch.setattr(device_reads, '_device', D)
    try:
        seq, off = D.upload(batch.seq), D.upload(batch.seq_off)
        qual = D.upload(batch.qual) if fmt == 'fastq' else None
        r = device_reads.demux_reads(seq, off, sets, scheme, qual, albacore_calls=albacore_calls, **bc, **o)
        parts = tuple(D.host(x) for x in r[:5])
        # the caller's reads, qualities and offsets are as they were
        assert np.array_equal(D.host(seq), batch.seq) and np.array_equal(D.host(off), batch.seq_off)
        if qual is not None:
            assert np.array_equal(D.host(qual), batch.qual)
    finally:
        D.free()
    r = r._replace(seq=parts[0], qual=parts[1], off=parts[2], read=parts[3], part=parts[4])
    return r, _bin_bytes(batch, r, fmt)


def _bin_bytes(batch, r, fmt):
    """each bin's file: emit_parts over the bin's slice of records (no select); checks the grouping on the way"""
    from porechop_b200 import fastq
    out, ends = {}, []
    names = list(r.bins)
    for name, (r0, r1) in r.bins.items():
        assert r1 > r0
        rd, pt = r.read[r0:r1], r.part[r0:r1]
        # inside a bin: read order, and the parts of a read in position order
        assert np.all((np.diff(rd) > 0) | ((np.diff(rd) == 0) & (np.diff(pt) > 0)))
        assert all(r.calls[k] == name for k in rd.tolist())
        out[name] = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna,
                                     (r.seq, r.qual, r.off[r0:r1 + 1], rd, pt), fmt)
        ends.append((r0, r1))
    # the bins tile the records in bin order, 'none' last
    assert [e[0] for e in ends] == sorted(e[0] for e in ends)
    assert sum(r1 - r0 for r0, r1 in ends) == len(r.read) and (not ends or ends[0][0] == 0)
    assert 'none' not in names or names[-1] == 'none'
    assert len(r.off) == len(r.read) + 1 and np.all(np.diff(r.off) > 0)
    return out


def _expected(W, monkeypatch, batch, sets, scheme, o, bc, fmt='fastq', albacore_calls=None):
    from porechop_b200 import fastq
    monkeypatch.setattr(fastq, 'W', W)
    return fastq.demux_fastq(batch, sets, scheme, fmt=fmt, albacore_calls=albacore_calls, **bc, **o)


def _compare(W, monkeypatch, batch, sets, o, bc, fmt='fastq', albacore_calls=None, scheme=DEFAULT):
    bins, info = _expected(W, monkeypatch, batch, sets, scheme, o, bc, fmt, albacore_calls)
    r, got = _demux(W, monkeypatch, batch, sets, scheme, o, bc, fmt, albacore_calls)
    assert r.calls == info['calls']
    assert np.array_equal(r.start_trim, info['start_trim']) and np.array_equal(r.end_trim, info['end_trim'])
    assert sorted(got) == sorted(bins)
    for k in bins:
        assert got[k] == bins[k], k
    return r


# ---- the reference CLI's bytes -------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case_name', ['bins_default', 'bins_two_barcodes', 'bins_loose_discard', 'bins_fasta_untrimmed'])
def test_sim_demux_golden_barcode_cases(SW, monkeypatch, case_name):
    batch, sets, scheme, o, bc, fmt, exp = _golden(case_name)
    r, got = _demux(SW, monkeypatch, batch, sets, scheme, o, bc, fmt)
    assert sorted(k + '.' + fmt for k in got) == sorted(exp)
    for k, v in got.items():
        assert v.decode() == exp[k + '.' + fmt], k


# ---- against fastq.demux_fastq -------------------------------------------------------------------------------------------
def _golden_variant(**kw):
    batch, sets, scheme, o, bc, fmt, _ = _golden('bins_default')
    for k, v in kw.items():
        (bc if k in BARCODE_KEYS else o)[k] = v
    return batch, sets, o, bc


@pytest.mark.parametrize('direction', ['forward', 'reverse'])
@pytest.mark.parametrize('two', [False, True])
def test_sim_demux_equals_demux_fastq_directions(SW, monkeypatch, direction, two):
    batch, sets, o, bc = _golden_variant(forward_or_reverse=direction, require_two_barcodes=two, discard_middle=False,
                                         min_split_read_size=100)
    r = _compare(SW, monkeypatch, batch, sets, o, bc)
    assert len(set(r.calls)) >= (1 if direction == 'forward' else 2)


def test_sim_demux_equals_demux_fastq_options(SW, monkeypatch):
    for kw, fmt in ((dict(discard_unassigned=True, barcode_threshold=60.0, barcode_diff=1.0), 'fastq'),
                    (dict(untrimmed=True), 'fastq'), (dict(discard_middle=False, min_split_read_size=50), 'fastq'),
                    (dict(no_split=True), 'fastq'), (dict(discard_middle=False, min_split_read_size=50), 'fasta'),
                    (dict(discard_unassigned=True, require_two_barcodes=True), 'fasta')):
        batch, sets, o, bc = _golden_variant(**kw)
        r = _compare(SW, monkeypatch, batch, sets, o, bc, fmt)
        if kw.get('discard_unassigned'):
            assert 'none' not in r.bins and 'none' in r.calls


def _observed_scores(W, monkeypatch, batch, sets, bc):
    """the best / second scores of every read per side (the device ranking as demux_fastq reads it)"""
    from porechop_b200 import fastq
    nsets = fastq._norm_sets(sets)
    s_cols, e_cols, su, eu = fastq.barcode_columns(nsets, bc['forward_or_reverse'])
    pk = lambda x: W.pack_sequences(x, offset_dtype=np.int32)     # noqa: E731
    st, et, ss, es, _, _ = W.adapter_trim_reads(batch.seq, batch.seq_off, pk([s[1] for _, s, _ in nsets if s]) + (s_cols,),
                                                pk([e[1] for _, _, e in nsets if e]) + (e_cols,), None, DEFAULT, 150, 2, 75.0, 4,
                                                want_top2=True)
    return fastq.Top2Scores(su, ss).ranked(), fastq.Top2Scores(eu, es).ranked()


def test_sim_demux_thresholds_and_diffs_on_achievable_scores(SW, monkeypatch):
    """threshold exactly a best score that occurs (>= passes, one ulp more fails) and diff exactly best - second"""
    batch, sets, o, bc = _golden_variant()
    (sp1, ss1, sp2, ss2), (ep1, es1, ep2, es2) = _observed_scores(SW, monkeypatch, batch, sets, bc)
    best = sorted(set(np.concatenate([ss1[sp1 >= 0], es1[ep1 >= 0]]).tolist()))
    assert len(best) >= 3
    gaps = sorted(set((ss1 - ss2)[sp2 >= 0].tolist()) | set((es1 - es2)[ep2 >= 0].tolist()))
    for thr in best[-3:] + [np.nextafter(best[-2], np.inf)]:
        for diff in [0.0] + gaps[-2:]:
            for two in (False, True):
                batch, sets, o, bc = _golden_variant(barcode_threshold=float(thr), barcode_diff=float(diff),
                                                     require_two_barcodes=two)
                _compare(SW, monkeypatch, batch, sets, o, bc)


def _barcoded_reads(pairs, seed=0):
    """reads with barcode j at the start and k at the end (-1 = none) around the Y adapters"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    bs, be = wl.demux_adapters()
    rng = random.Random(seed)
    reads = []
    for j, k in pairs:
        mid = ''.join(rng.choice('ACGT') for _ in range(700))
        reads.append((bs[j] if j >= 0 else '') + yt + mid + yb + (be[k] if k >= 0 else ''))
    names, name_off = W.pack_sequences(['r%d x' % i for i in range(len(reads))])
    seq, off = W.pack_sequences(reads)
    qual = np.frombuffer(bytes(33 + (i * 7) % 40 for i in range(len(seq))), dtype=np.uint8)
    return fastq.FastqBatch(names, name_off, seq, off.astype(np.int64), qual, off.astype(np.int64).copy(),
                            np.zeros(len(reads), dtype=bool))


def _bc_sets(ids, dup=None):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    bs, be = wl.demux_adapters()
    sets = [('SQK-NSK007', ('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))] + \
           [('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[j]), ('BC%02d_end' % (j + 1), be[j])) for j in ids]
    if dup is not None:     # a second set of the same barcode name with other sequences (the reference's dicts: last value)
        j, other = dup
        sets.append(('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[other]), ('BC%02d_end' % (j + 1), be[other])))
    return sets


BC = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
          discard_unassigned=False)
O = dict(min_split_read_size=100)


def test_sim_demux_start_end_ties_and_repeated_names(SW, monkeypatch):
    # start barcode 0 / end barcode 1 both perfect: a tie the start side wins (and second + diff fails); one-sided reads
    batch = _barcoded_reads([(0, 1), (1, 0), (0, 0), (2, -1), (-1, 2), (-1, -1), (1, 2)])
    for two in (False, True):
        for diff in (0.0, 5.0):
            r = _compare(SW, monkeypatch, batch, _bc_sets([0, 1, 2]), O, dict(BC, require_two_barcodes=two, barcode_diff=diff))
            if not two and diff == 0.0:
                # 100.0 on both sides and on two columns of a side: the start side's first column wins every tie
                assert r.calls[:2] == ['BC01', 'BC01']
    r = _compare(SW, monkeypatch, batch, _bc_sets([0, 1, 2], dup=(1, 3)), O, BC)


def test_sim_demux_without_barcodes_or_adapters(SW, monkeypatch):
    batch = _barcoded_reads([(0, 0), (1, 1), (-1, -1)])
    r = _compare(SW, monkeypatch, batch, _bc_sets([]), O, BC)               # no barcode set: everything 'none'
    assert set(r.calls) == {'none'} and list(r.bins) == ['none']
    r = _compare(SW, monkeypatch, batch, [], O, BC)                        # no adapters at all
    assert set(r.calls) == {'none'} and (r.part == 0).all() and len(r.read) == 3
    r = _compare(SW, monkeypatch, batch, [], O, dict(BC, discard_unassigned=True))
    assert r.bins == {} and len(r.read) == 0


def test_sim_demux_albacore_calls(SW, monkeypatch):
    batch = _barcoded_reads([(0, 0), (1, 1), (2, 2), (0, 0), (1, 1), (-1, -1)])
    sets, bc = _bc_sets([0, 1, 2]), dict(BC, barcode_diff=0.0)
    base = _compare(SW, monkeypatch, batch, sets, O, bc, albacore_calls=[None] * 6).calls
    assert 'none' not in base[:5]
    other = ['BC02' if c == 'BC01' else 'BC01' for c in base]
    for alb, exp in ((base, base), (other, ['none'] * 6),
                     ([base[0], None, 'zzz', 'none', other[4], None], [base[0], base[1], 'none', 'none', 'none', base[5]])):
        assert _compare(SW, monkeypatch, batch, sets, O, bc, albacore_calls=alb).calls == exp


# ---- segments, capacity, preconditions -------------------------------------------------------------------------------------
def test_sim_demux_several_segments_give_the_same_records(monkeypatch):
    """PB_TEST_SEGMENT_READS=7: the 18 reads run as 3 segments -- the grouping by bin is over the whole call"""
    import sim_engine
    batch, sets, o, bc = _golden_variant(discard_middle=False, min_split_read_size=100)
    got = []
    for W in (sim_engine.load(), sim_engine.load(['-DPB_TEST_SEGMENT_READS=7'])):
        r, b = _demux(W, monkeypatch, batch, sets, DEFAULT, o, bc)
        got.append((r, b))
    (r1, b1), (r7, b7) = got
    assert all(np.array_equal(x, y) for x, y in zip(r1[:5], r7[:5]))
    assert r1.bins == r7.bins and r1.calls == r7.calls and b1 == b7 and len(r1.bins) >= 3
    assert not np.all(np.diff(r1.read) >= 0)                      # grouped by bin, not in read order overall
    n, text = sim_engine.load(['-DPB_TEST_SEGMENT_READS=7']).races()
    assert n == 0, text[:4000]


def _raw_demux(W, batch, sets, o, bc, parts_cap, fmt='fastq'):
    """adapter_demux_reads_device straight, with buffers for parts_cap records; returns its outputs or the EngineError"""
    from porechop_b200 import device_reads, fastq
    D = SimDevice(W)
    nsets, starts, ends, adapters, left, right = device_reads._options(sets, o.get('no_split', False), 10, 100)
    s_cols, e_cols, su, eu = fastq.barcode_columns(nsets, bc['forward_or_reverse'])
    names = list(dict.fromkeys(su + eu))
    pk = lambda x: W.pack_sequences(x, offset_dtype=np.int32)     # noqa: E731
    try:
        seq, off, qual = D.upload(batch.seq), D.upload(batch.seq_off), D.upload(batch.qual)
        out = [D.empty(len(batch.seq), np.uint8), D.empty(len(batch.seq), np.uint8), D.empty(parts_cap + 1, np.int64),
               D.empty(max(parts_cap, 1), np.int32), D.empty(max(parts_cap, 1), np.int32)]
        try:
            res = W.adapter_demux_reads_device(
                seq.ptr, off.ptr, len(batch), len(batch.seq), -1, pk(starts) + (s_cols,), pk(ends) + (e_cols,),
                pk([a[1] for a in adapters]), DEFAULT, 150, 2, 75.0, 4, o.get('middle_threshold', 85.0),
                start_bin=[names.index(x) for x in su], end_bin=[names.index(x) for x in eu], n_bins=len(names),
                barcode_threshold=bc['barcode_threshold'], barcode_diff=bc['barcode_diff'],
                require_two_barcodes=bc['require_two_barcodes'], discard_unassigned=bc['discard_unassigned'],
                d_quals_ptr=qual.ptr, mid_extra=(left, right), min_split_read_size=o['min_split_read_size'],
                discard_middle=o['discard_middle'], d_out_seq_ptr=out[0].ptr, d_out_qual_ptr=out[1].ptr, d_out_off_ptr=out[2].ptr,
                d_out_read_ptr=out[3].ptr, d_out_part_ptr=out[4].ptr, parts_cap=parts_cap)
            k = res[4]
            return res, [D.host(D.head(out[2], k + 1)), D.host(D.head(out[3], k)), D.host(D.head(out[4], k)),
                         D.host(D.head(out[0], res[5]))]
        except W.EngineError as e:
            return e, None
    finally:
        D.free()


def test_sim_demux_parts_cap_too_small_and_the_retry(SW, monkeypatch):
    from porechop_b200 import device_reads
    for discard in (False, True):
        batch, sets, o, bc = _golden_variant(discard_middle=False, min_split_read_size=100, discard_unassigned=discard,
                                             barcode_threshold=60.0)
        full, recs = _raw_demux(SW, batch, sets, o, bc, 1000)
        st, et, n_hits, hits, n_parts, n_bases, read_bin, bin_parts = full
        assert bin_parts[-1] == n_parts and (not discard or (read_bin == len(bin_parts) - 2).any())
        for cap in (0, 2, n_parts - 1):
            e, _ = _raw_demux(SW, batch, sets, o, bc, cap)
            assert isinstance(e, SW.EngineError) and e.code == SW.ERR_SPACE
            assert (e.n_parts, e.n_out_bases) == (n_parts, n_bases)
            assert np.array_equal(e.read_bin, read_bin) and np.array_equal(e.bin_parts, bin_parts)
        again, recs2 = _raw_demux(SW, batch, sets, o, bc, n_parts)      # exactly the kept records fit
        assert again[4] == n_parts and all(np.array_equal(x, y) for x, y in zip(recs, recs2))
    # the module's single retry with the exact count
    batch, sets, o, bc = _golden_variant(discard_middle=False, min_split_read_size=100)
    exp, exp_bytes = _demux(SW, monkeypatch, batch, sets, DEFAULT, o, bc)
    caps = []
    orig = SW.adapter_demux_reads_device
    monkeypatch.setattr(SW, 'adapter_demux_reads_device', lambda *a, **k: caps.append(k['parts_cap']) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_parts_cap', lambda n: 2)
    got, got_bytes = _demux(SW, monkeypatch, batch, sets, DEFAULT, o, bc)
    assert caps == [2, len(exp.read)] and got_bytes == exp_bytes and got.calls == exp.calls and got.bins == exp.bins


def test_sim_demux_preconditions_fail_before_any_launch(SW):
    from test_trim_split_reads import _Raw, _batch
    from test_trim_reads import trim_reads_set
    R = _Raw(SW, _batch(trim_reads_set()[:8]))
    cols = np.array([0, 0], dtype=np.int32)
    R.args.start.score_cols, R.args.start.n_score_cols = cols.ctypes.data, 1
    read_bin, bin_parts = np.zeros(8, dtype=np.int32), np.zeros(4, dtype=np.int64)
    good_map, bad_maps = np.array([0], dtype=np.int32), {k: np.array(v, dtype=np.int32) for k, v in
                                                          (('hi', [2]), ('neg', [-1]), ('dup', [1, 1]))}

    def demux(**kw):
        d = SW.DemuxArgsDesc(good_map.ctypes.data, None, 2, 75.0, 5.0, 0, 0, None, read_bin.ctypes.data, bin_parts.ctypes.data)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def call(d, **split):
        for k, v in split.items():
            setattr(R.split, k, v)
        return SW.C_LIB.adapterDemuxReadsDevice(R.d_seq.ptr, R.d_off.ptr, R.n, R.nbytes, -1, ctypes.byref(R.args),
                                                ctypes.byref(R.split), ctypes.byref(d) if d is not None else None, *DEFAULT, None)
    try:
        assert call(demux()) == 0 and R.n_parts.value > 0
        bad = [dict(read_bin=None), dict(bin_parts=None), dict(n_bins=-1), dict(n_bins=4096), dict(start_bin=None),
               dict(barcode_threshold=float('nan')), dict(barcode_diff=float('nan')), dict(start_bin=bad_maps['hi'].ctypes.data),
               dict(start_bin=bad_maps['neg'].ctypes.data), dict(n_bins=0)]
        for kw in bad + [None, 'dup', 'parts_cap', 'end_size']:
            n0 = SW.kernel_launches()
            R.n_parts.value = R.n_bases.value = -1
            if kw is None:
                rc = call(None)
            elif kw == 'dup':                     # a bin twice on one side
                R.args.start.n_score_cols = 2
                rc = call(demux(start_bin=bad_maps['dup'].ctypes.data))
                R.args.start.n_score_cols = 1
            elif kw == 'parts_cap':               # a precondition of adapterTrimSplitReadsDevice
                rc = call(demux(), parts_cap=-1)
                R.split.parts_cap = 10000
            elif kw == 'end_size':                # windows outside the device ranking's domain
                R.args.end_size = 4090
                rc = call(demux())
                R.args.end_size = 150
            else:
                rc = call(demux(**kw))
            assert rc == SW.ERR_ARG, kw
            assert SW.kernel_launches() == n0, kw
            assert R.n_parts.value == 0 and R.n_bases.value == 0, kw
        assert call(demux()) == 0 and bin_parts[-1] == R.n_parts.value
    finally:
        R.D.free()


# ---- the call rule through tests/emu -------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu_demux():
    d = tempfile.mkdtemp(prefix='pb200_emu_demux_')
    so = os.path.join(d, 'libemu_demux.so')
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-fPIC', '-shared', '-o', so, os.path.join(ROOT, 'tests', 'emu', 'emu_demux.cpp')])
    lib = ctypes.CDLL(so)
    lib.emu_barcode_calls.argtypes = [ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                      ctypes.c_int32, ctypes.c_double, ctypes.c_double, ctypes.c_int32, ctypes.c_void_p,
                                      ctypes.c_void_p]
    lib.emu_barcode_calls.restype = None
    return lib


def _random_side(rng, n, k, scores):
    """a top-2 ranking of k columns per read: positions (-1 = none) and scores, second <= best"""
    p1, p2, s1, s2 = np.full(n, -1), np.full(n, -1), np.zeros(n), np.zeros(n)
    for i in range(n):
        if k == 0 or rng.random() < 0.1:
            continue
        a = rng.sample(range(k), min(k, 2))
        v = sorted([rng.choice(scores), rng.choice(scores)], reverse=True)
        p1[i], s1[i] = a[0], v[0]
        if len(a) > 1 and rng.random() < 0.9:
            p2[i], s2[i] = a[1], v[1]
    return p1, s1, p2, s2


@pytest.mark.parametrize('two', [False, True])
def test_emu_barcode_call_equals_call_barcodes_top2(emu_demux, two):
    from porechop_b200 import fastq
    rng = random.Random(11 + two)
    pool = ['BC%02d' % j for j in range(1, 9)]
    adversarial = [0.0, 50.0, 74.999999, 75.0, 75.000001, 80.0, 80.000001, 85.0, 100.0]
    for trial in range(300):
        ks, ke = rng.randint(0, 5), rng.randint(0, 5)
        s_names, e_names = rng.sample(pool, ks), rng.sample(pool, ke)
        n = 64
        scores = adversarial if trial % 2 else [round(rng.uniform(40, 100), rng.choice([0, 1, 6])) for _ in range(6)]
        S, E = _random_side(rng, n, ks, scores), _random_side(rng, n, ke, scores)
        thr = rng.choice([75.0, 80.0, 0.0, rng.choice(scores)])
        diff = rng.choice([0.0, 5.0, 0.000001, abs(rng.choice(scores) - rng.choice(scores))])
        alb = None if trial % 3 == 0 else [rng.choice(pool + [None, 'zzz', 'none']) for _ in range(n)]
        exp = fastq.call_barcodes_top2((s_names, S), (e_names, E), thr, diff, two, alb)
        names = list(dict.fromkeys(s_names + e_names))
        nb = len(names)
        sid = np.array([names.index(x) for x in s_names] + [-1], dtype=np.int32)
        eid = np.array([names.index(x) for x in e_names] + [-1], dtype=np.int32)
        sb = np.ascontiguousarray(np.stack([sid[S[0]], sid[S[2]]], axis=1), dtype=np.int32)
        eb = np.ascontiguousarray(np.stack([eid[E[0]], eid[E[2]]], axis=1), dtype=np.int32)
        ss = np.ascontiguousarray(np.stack([S[1], S[3]], axis=1), dtype=np.float64)
        es = np.ascontiguousarray(np.stack([E[1], E[3]], axis=1), dtype=np.float64)
        a = None if alb is None else np.array([-1 if x is None else (names.index(x) if x in names else nb + 1) for x in alb],
                                              dtype=np.int32)
        out = np.zeros(n, dtype=np.int32)
        emu_demux.emu_barcode_calls(n, sb.ctypes.data, ss.ctypes.data, eb.ctypes.data, es.ctypes.data, nb, thr, diff, int(two),
                                    a.ctypes.data if a is not None else None, out.ctypes.data)
        got = [(names + ['none'])[b] for b in out.tolist()]
        assert got == exp, (trial, s_names, e_names, thr, diff)


# ---- AddressSanitizer -------------------------------------------------------------------------------------------------------
def _asan_body():
    """the demux stage on exact-size "device" heap blocks: golden cases, options, capacity and argument errors (run by
    test_sim_demux_under_address_sanitizer in a process with the ASan build of the simulated engine)"""
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
    for case in ('bins_default', 'bins_loose_discard', 'bins_fasta_untrimmed'):
        mp = MP()
        test_sim_demux_golden_barcode_cases(W, mp, case)
        mp.close()
    mp = MP()
    test_sim_demux_without_barcodes_or_adapters(W, mp)
    mp.close()
    mp = MP()
    test_sim_demux_parts_cap_too_small_and_the_retry(W, mp)
    mp.close()
    test_sim_demux_preconditions_fail_before_any_launch(W)
    print('ASAN RUN COMPLETE')


@pytest.mark.skipif(os.environ.get('PB200_SIM_ASAN', '0') != '1', reason='minutes: set PB200_SIM_ASAN=1')
def test_sim_demux_under_address_sanitizer():
    import build_sim
    lib = build_sim.build_asan()
    asan = subprocess.check_output(['gcc', '-print-file-name=libasan.so']).decode().strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS='detect_leaks=0:detect_stack_use_after_return=0', PB200_SIM_ASAN_LIB=lib)
    code = ('import os, sys; sys.path[:0] = [%r, %r, %r]; import build_sim; '
            'build_sim.build = lambda force=False, flags=None: os.environ["PB200_SIM_ASAN_LIB"]; '
            'import test_demux_reads as T; T._asan_body()') % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0 and 'ASAN RUN COMPLETE' in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
    assert 'ERROR: AddressSanitizer' not in r.stderr
