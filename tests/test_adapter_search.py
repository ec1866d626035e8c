"""The adapter-set search on the device (include/porechop_b200.h adapterSetSearch): Porechop's Phase A reduced to one best
full-adapter identity per adapter sequence before anything is copied back.  CPU tier: the product's engine code on the host
simulator (tests/sim) against the reference's set scores, against the host reduction of the simulated engine's own records,
across chunks, stages, interleavings and streams, and the flat CLI's files with Phase A over every read.  GPU tier (marked):
the same comparisons through the real engine, and 10^6 reads x the 236 table sequences."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

SC = (3, -6, -5, -2)
LINEAR = (3, -6, -5, -5)
GENERIC = (3, -6, 1, -2)          # a positive gap score: the generic int32 kernel


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


def _table_sets():
    ad = load_golden('adapters.json')
    return [(d['name'], d['start'] or None, d['end'] or None) for d in ad['sets']]


def _host_best(W, buf, off, abuf, aoff, scheme):
    """the host reduction of the engine's own records: max(0, max over windows of float("%f" % fullAdapter%ID))"""
    from porechop_b200.align import scores_from_records
    n, m = len(off) - 1, len(aoff) - 1
    if n == 0:
        return np.zeros(m), np.zeros((0, 9), dtype=np.int32)
    rec = W.adapter_alignment_batch(buf, off, abuf, aoff, scheme)
    full, _, _, _ = scores_from_records(rec)
    return np.maximum(full.reshape(n, m).max(axis=0), 0.0), rec


# ---- reference goldens ------------------------------------------------------------------------------------------------
def _check_reference_case(W, monkeypatch, case):
    from porechop_b200 import fastq
    from test_fastq_bulk import fixture, fastq_text
    monkeypatch.setattr(fastq, 'W', W)
    sets = _table_sets()
    b = fastq.parse_fastq(fastq_text(fixture(case['file'])))
    calls = []
    orig = W.adapter_set_search
    monkeypatch.setattr(W, 'adapter_set_search', lambda *a, **k: calls.append(1) or orig(*a, **k))
    bs, be = fastq.search_adapter_sets(b, sets, SC, device=True)
    monkeypatch.setattr(W, 'adapter_set_search', orig)
    assert calls == [1]                                       # both batches in one submit
    want = {nm: (s, e) for nm, s, e in case['set_scores']}
    assert len(want) == len(sets) == 119
    for (nm, _, _), s, e in zip(sets, bs, be):
        assert (s, e) == want[nm], nm


def _check_reference_phases(W, monkeypatch, case):
    from porechop_b200 import phases
    from test_gpu_phases import AdapterSet, Read
    monkeypatch.setattr(phases, 'W', W)
    ad = load_golden('adapters.json')
    reads = [Read(r['name'], r['seq']) for r in load_golden('fixture_reads.json') if r['file'] == case['file']]
    table = [AdapterSet(d) for d in ad['sets']]
    phases.align_adapter_sets(reads, table, 150, list(SC), device=True)
    assert [[s.name, s.best_start_score, s.best_end_score] for s in table] == case['set_scores']


@pytest.mark.parametrize('case_index', [0, 1, 2, 3])
def test_sim_search_reproduces_the_reference_set_scores(SW, monkeypatch, case_index):
    case = load_golden('golden_phases.json')[case_index]
    _check_reference_case(SW, monkeypatch, case)
    _check_reference_phases(SW, monkeypatch, case)


# ---- device reduction == host reduction of the records -----------------------------------------------------------------
def _random_windows(seed, n, size, seqs):
    """n windows of at most `size` bytes: empty windows, all-N, lowercase, U for T, bytes outside ACGTUN, and windows that
    carry a mutated copy of one of `seqs` (so that scores spread over the whole range)"""
    rng = random.Random(seed)
    out = []
    for i in range(n):
        kind = i % 7
        if kind == 0:
            w = ''
        elif kind == 1:
            w = 'N' * rng.randint(1, size)
        else:
            w = ''.join(rng.choice('ACGT') for _ in range(rng.randint(1, size)))
            if kind >= 3:
                ad = rng.choice(seqs)
                ad = ''.join(c if rng.random() > 0.08 else rng.choice('ACGT') for c in ad)
                p = rng.randint(0, max(0, len(w) - 1))
                w = (w[:p] + ad + w[p:])[:size]
            if kind == 4:
                w = w.lower()
            elif kind == 5:
                w = w.replace('T', 'U')
            elif kind == 6:
                w = ''.join(c if rng.random() > 0.1 else rng.choice('XR-#*.n\x7f') for c in w)
        out.append(w)
    return out


def _search_inputs(seed, n, size, n_start, n_end):
    """(start windows, end windows, start sequences, end sequences) with subsets of the 236 table sequences"""
    from porechop_b200 import workloads as wl
    starts, ends = wl.all_table_sequences()
    rng = random.Random(seed)
    ss, es = rng.sample(starts, n_start), rng.sample(ends, n_end)
    return _random_windows(seed, n, size, ss), _random_windows(seed + 1, n, size, es), ss, es


def _check_against_records(W, wins_s, wins_e, ss, es, scheme, with_out):
    pack = W.pack_sequences
    batches, expect = [], []
    for wins, seqs in ((wins_s, ss), (wins_e, es)):
        buf, off = pack(wins)
        abuf, aoff = pack(seqs, offset_dtype=np.int32)
        best, rec = _host_best(W, buf, off, abuf, aoff, scheme)
        out = np.full((len(wins) * len(seqs), 9), -7, dtype=np.int32) if with_out else None
        batches.append((buf, off, abuf, aoff, out))
        expect.append((best, rec, out))
    got = W.adapter_set_search(batches, scheme)
    for g, (best, rec, out) in zip(got, expect):
        assert np.array_equal(g, best)
        assert g.dtype == np.float64 and (g >= 0).all()
        if with_out:
            assert np.array_equal(out, rec)
    return got


@pytest.mark.parametrize('scheme,size,n,n_start,n_end', [(SC, 150, 70, 40, 25), (LINEAR, 150, 50, 30, 30),
                                                         (SC, 500, 24, 14, 10), (GENERIC, 150, 14, 5, 4)],
                         ids=['default', 'linear', 'two_pass', 'generic'])
def test_sim_search_equals_host_reduction_of_records(SW, scheme, size, n, n_start, n_end):
    wins_s, wins_e, ss, es = _search_inputs(size + n, n, size, n_start, n_end)
    for with_out in (False, True):
        got = _check_against_records(SW, wins_s, wins_e, ss, es, scheme, with_out)
    assert any((g > 50).any() for g in got)                  # real hits, not only empty / failed alignments


def test_sim_search_over_many_chunks_and_a_lower_second_call(SW):
    """a small chunk_tasks: one submit spans many chunks on all three stages; then a call whose inputs score lower than the
    previous call's must return its own values (the accumulators are reset per submit)"""
    wins_s, wins_e, ss, es = _search_inputs(5, 60, 150, 12, 9)
    SW.set_option('chunk_tasks', 40)
    try:
        hi = _check_against_records(SW, wins_s, wins_e, ss, es, SC, False)
        rng = random.Random(9)
        plain = [''.join(rng.choice('ACGT') for _ in range(60)) for _ in range(30)]
        lo = _check_against_records(SW, plain, plain[:7], ss, es, SC, True)
    finally:
        SW.set_option('chunk_tasks', 131072)
    assert all((h >= l).all() for h, l in zip(hi, lo)) and any((h > l).any() for h, l in zip(hi, lo))


_ORDER_SCRIPT = r'''
import json, sys
sys.path[:0] = [%r, %r, %r]
import sim_engine, test_adapter_search as T
W = sim_engine.load()
ws, we, ss, es = T._search_inputs(3, 40, 150, 10, 8)
W.set_option('chunk_tasks', 64)
bs, bo = W.pack_sequences(ws)
eb, eo = W.pack_sequences(we)
a1, o1 = W.pack_sequences(ss, offset_dtype=__import__('numpy').int32)
a2, o2 = W.pack_sequences(es, offset_dtype=__import__('numpy').int32)
got = W.adapter_set_search([(bs, bo, a1, o1), (eb, eo, a2, o2)], T.SC)
print(json.dumps([g.tolist() for g in got]))
'''


def test_sim_result_does_not_depend_on_the_interleaving(SW):
    """the order of the threads' atomics differs between interleavings (PBSIM_ORDER); the maxima must not"""
    script = _ORDER_SCRIPT % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    outs = []
    for order in ('', 'reverse', 'random:3', 'random:11'):
        env = dict(os.environ)
        env.pop('PBSIM_ORDER', None)
        if order:
            env['PBSIM_ORDER'] = order
        r = subprocess.run([sys.executable, '-c', script], env=env, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(json.loads(r.stdout.strip().splitlines()[-1]))
    assert all(o == outs[0] for o in outs[1:])
    assert max(max(v) for v in outs[0]) > 50


# ---- edges -----------------------------------------------------------------------------------------------------------
def _check_edges(W):
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    abuf, aoff = W.pack_sequences([yt, yb, 'ACGT'], offset_dtype=np.int32)
    z8, z64, z32 = np.zeros(0, np.uint8), np.zeros(1, np.int64), np.zeros(1, np.int32)
    wb, wo = W.pack_sequences(['ACGTTT' + yt, 'GGG'])
    # n_seqs == 0 -> zeros; only empty windows -> 0.0; a batch without adapters is skipped
    got = W.adapter_set_search([(z8, z64, abuf, aoff), (z8, np.zeros(4, np.int64), abuf, aoff), (wb, wo, z8, z32)], SC)
    assert [g.tolist() for g in got] == [[0.0] * 3, [0.0] * 3, []]
    # ... and its `best` is not touched, while a real batch in the same call is computed
    keep = np.full(2, 7.5)
    real = np.zeros(3)
    B = W.BatchDesc
    descs = (W.SearchBatchDesc * 2)(
        W.SearchBatchDesc(B(wb.ctypes.data, wo.ctypes.data, 2, None, z32.ctypes.data, 0, None), keep.ctypes.data),
        W.SearchBatchDesc(B(wb.ctypes.data, wo.ctypes.data, 2, abuf.ctypes.data, aoff.ctypes.data, 3, None), real.ctypes.data))
    assert W.C_LIB.adapterSetSearch(descs, 2, *SC) == 0
    assert keep.tolist() == [7.5, 7.5] and real[0] == 100.0 and real[1] < 100.0
    # NULL best, negative counts, bad offsets: PB200_ERR_ARG
    bad_ad = np.array([0, 5, 3, 8], dtype=np.int32)
    bad_off, neg_off = np.array([0, 9, 4], np.int64), np.array([-2, 9, 12], np.int64)
    cases = [(B(wb.ctypes.data, wo.ctypes.data, 2, abuf.ctypes.data, aoff.ctypes.data, 3, None), None),
             (B(wb.ctypes.data, wo.ctypes.data, -1, abuf.ctypes.data, aoff.ctypes.data, 3, None), real.ctypes.data),
             (B(wb.ctypes.data, wo.ctypes.data, 2, abuf.ctypes.data, aoff.ctypes.data, -3, None), real.ctypes.data),
             (B(wb.ctypes.data, wo.ctypes.data, 2, abuf.ctypes.data, bad_ad.ctypes.data, 3, None), real.ctypes.data),
             (B(wb.ctypes.data, bad_off.ctypes.data, 2, abuf.ctypes.data, aoff.ctypes.data, 3, None),
              real.ctypes.data),
             (B(wb.ctypes.data, neg_off.ctypes.data, 2, abuf.ctypes.data, aoff.ctypes.data, 3, None),
              real.ctypes.data)]
    for desc, best in cases:
        d = (W.SearchBatchDesc * 1)(W.SearchBatchDesc(desc, best))
        assert W.C_LIB.adapterSetSearch(d, 1, *SC) == W.ERR_ARG
    assert W.C_LIB.adapterSetSearch(None, 1, *SC) == W.ERR_ARG
    assert W.C_LIB.adapterSetSearch(descs, -1, *SC) == W.ERR_ARG
    assert W.C_LIB.adapterSetSearch(None, 0, *SC) == 0


def test_sim_edges(SW):
    _check_edges(SW)


# ---- stream order ----------------------------------------------------------------------------------------------------
def test_sim_search_after_a_device_call_on_another_stream(SW):
    """adapterAlignmentBatchDevice returns with its work queued on another stream; adapterSetSearch, issued without any
    synchronisation, must wait for it (the stream-ordering check reports any race) and still return the right values"""
    from test_stream_order import DeviceCall
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, _ = wl.synth_end_windows(300, yt, yb, seed=21)
    buf, off = wl.windows_to_batch(sw)
    wins_s, wins_e, ss, es = _search_inputs(17, 40, 150, 10, 8)
    expect = []
    for wins, seqs in ((wins_s, ss), (wins_e, es)):
        b, o = SW.pack_sequences(wins)
        a, ao = SW.pack_sequences(seqs, offset_dtype=np.int32)
        expect.append(((b, o, a, ao), _host_best(SW, b, o, a, ao, SC)[0]))
    SW.synchronize()
    SW.clear_races()
    for sc in (SC, GENERIC):
        A = SW.stream_create()
        c = DeviceCall(SW, buf[:150 * 40], off[:41], [yt, yb], sc, A)()
        got = SW.adapter_set_search([e[0] for e in expect], SC)
        for g, (_, best) in zip(got, expect):
            assert np.array_equal(g, best)
        SW.synchronize()
        c.check()


# ---- Phase A, then the flat pipeline ------------------------------------------------------------------------------
def _check_emit_with_device_search(W, monkeypatch):
    """the golden_emit inputs with Phase A through adapterSetSearch: for the trim cases the sets it finds (best start or end
    score >= 90, porechop.py:327) are the ones the reference CLI chose, and trim_fastq with them writes the golden bytes; for
    the barcoded input the device search equals the record path and finds the barcode sets, and demux_fastq writes the
    golden bins"""
    from porechop_b200 import fastq
    import test_fastq_emit as T
    monkeypatch.setattr(fastq, 'W', W)
    g = load_golden('golden_emit.json')
    sets = _table_sets()
    table = [[list(st) if st else None, list(en) if en else None] for _, st, en in sets]
    batch = fastq.parse_fastq(g['input_fastq'].encode())
    for name in T.CASES:
        c = g['cases'][name]
        bs, be = fastq.search_adapter_sets(batch, sets, c['scoring'], end_size=c['options']['end_size'], device=True)
        chosen = [t for t, x, y in zip(table, bs, be) if max(x, y) >= 90.0]
        assert chosen == c['matching_sets'], name
        T._run(name)
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    dev = fastq.search_adapter_sets(batch, sets, list(SC), device=True)
    host = fastq.search_adapter_sets(batch, sets, list(SC), device=False)
    assert all(np.array_equal(d, h) for d, h in zip(dev, host))
    assert sum(max(x, y) >= 90.0 and nm.startswith('Barcode ') for (nm, _, _), x, y in zip(sets, *dev)) >= 2
    for name in T.BARCODE_CASES:
        T._run_demux(name)


def test_sim_trim_and_demux_reproduce_the_reference_cli_with_the_device_search(SW, monkeypatch):
    _check_emit_with_device_search(SW, monkeypatch)


# ---- flat CLI --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('chunk', [3000, 1 << 20])
@pytest.mark.parametrize('input_name,argv', [('test_barcodes.fastq', ['-b', '{out}/bins']),
                                             ('test_two_adapter_sets.fastq', ['-o', '{out}/o.fastq']),
                                             ('GOLDEN:input_fastq', ['-o', '{out}/o.fastq', '--min_split_read_size', '50'])])
def test_sim_flat_cli_phase_a_over_all_reads_with_the_device_search(SW, chunk, input_name, argv, monkeypatch, tmp_path):
    """PB200_CHECK_ALL_READS=1 with Phase A through adapterSetSearch on the simulated engine: the reference CLI's files, byte
    for byte.  Needs the Porechop checkout (skipped without it, as tests/test_flat_cli.py is)."""
    import test_flat_cli as T
    import test_patch_cli
    if T.pytestmark.args[0]:
        pytest.skip(T.pytestmark.kwargs['reason'])
    from porechop_b200 import cpp_function_wrappers as W, fastq
    calls = []
    monkeypatch.setattr(W, 'adapter_set_search', lambda *a, **k: calls.append(1) or SW.adapter_set_search(*a, **k))
    monkeypatch.setattr(fastq, 'DEVICE_SEARCH', True)
    T.test_flat_cli_phase_a_over_all_reads(chunk, input_name, argv, test_patch_cli.load_reference(), monkeypatch, tmp_path)
    assert calls


# ---- GPU tier --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case_index', [0, 1, 2, 3])
def test_gpu_search_reproduces_the_reference_set_scores(monkeypatch, case_index):
    from porechop_b200 import cpp_function_wrappers as W
    case = load_golden('golden_phases.json')[case_index]
    _check_reference_case(W, monkeypatch, case)
    _check_reference_phases(W, monkeypatch, case)


@pytest.mark.gpu
@pytest.mark.parametrize('scheme,size,n,n_start,n_end', [(SC, 150, 3000, 119, 117), (LINEAR, 150, 2000, 60, 60),
                                                         (SC, 500, 800, 119, 117), (GENERIC, 150, 200, 20, 12)],
                         ids=['default', 'linear', 'two_pass', 'generic'])
def test_gpu_search_equals_host_reduction_of_records(scheme, size, n, n_start, n_end):
    from porechop_b200 import cpp_function_wrappers as W
    wins_s, wins_e, ss, es = _search_inputs(size + n, n, size, n_start, n_end)
    for with_out in (False, True):
        got = _check_against_records(W, wins_s, wins_e, ss, es, scheme, with_out)
    assert any((g > 50).any() for g in got)


@pytest.mark.gpu
def test_gpu_edges():
    from porechop_b200 import cpp_function_wrappers as W
    _check_edges(W)


@pytest.mark.gpu
def test_gpu_million_reads_times_the_table_sequences():
    """10^6 synthetic reads x the 236 table sequences (Phase A with every read checked): the device reduction equals the
    host reduction of the record API's output for the same windows"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    n = 1000000
    buf, off = wl.synth_reads_fast(n, yt, yb, chimera_p=0.05)
    (sbuf, soff), (ebuf, eoff) = fastq.end_windows(buf, off, 150)
    starts, ends = wl.all_table_sequences()
    assert len(starts) + len(ends) == 236
    batches = [(sbuf, soff) + W.pack_sequences(starts, offset_dtype=np.int32),
               (ebuf, eoff) + W.pack_sequences(ends, offset_dtype=np.int32)]
    got = W.adapter_set_search(batches, wl.DEFAULT_SCORING)
    step = 100000                                             # the record path in slices of reads (bounded host memory)
    for (b, o, a, ao), g in zip(batches, got):
        best = np.zeros(len(ao) - 1)
        for s in range(0, n, step):
            best = np.maximum(best, _host_best(W, b, o[s:s + step + 1], a, ao, wl.DEFAULT_SCORING)[0])
        assert np.array_equal(g, best)
    assert got[0].max() > 90 and got[1].max() > 90          # the implanted Y adapters are found


@pytest.mark.gpu
def test_gpu_trim_and_demux_reproduce_the_reference_cli_with_the_device_search(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W
    _check_emit_with_device_search(W, monkeypatch)
