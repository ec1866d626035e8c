"""The middle-adapter scan on the device (include/porechop_b200.h adapterMiddleScan): Porechop's Phase C with its masking
rounds in one engine call.  CPU tier: the threshold table against Python's own float('%f') chain, and the product's engine
code on the host simulator (tests/sim) against the host rounds of fastq.find_middle_hits and the reference CLI's bytes.
GPU tier (marked): the same comparisons through the real engine, the device-resident entry point, and the config-4 shape."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from helpers import ROOT

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

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


def _brute_table(thr, length):
    out = [2147483647]
    for l in range(1, length):
        c = next((c for c in range(l + 1) if float('%f' % (100.0 * c / l)) >= thr), l + 1)
        out.append(c)
    return np.array(out[:length], dtype=np.int32)


def test_middle_threshold_table_equals_python_float_chain():
    from porechop_b200 import cpp_function_wrappers as W
    for thr in (0.5, 70, 85, 90, 96.43, 99.999, 100, 101):
        assert np.array_equal(W.middle_threshold_table(thr, 701), _brute_table(thr, 701)), thr
    for bad in (0.0, -1.0, float('nan')):
        with pytest.raises(W.EngineError):
            W.middle_threshold_table(bad, 10)


def _batch(reads):
    from porechop_b200 import fastq
    text = ''.join('@r%d\n%s\n+\n%s\n' % (k, r, '5' * len(r)) for k, r in enumerate(reads))
    return fastq.parse_fastq(text.encode())


def _stress_reads(seed=7):
    """reads built to stress the rounds: adjacent and overlapping copies of one adapter, copies of different adapters,
    reads shorter than an adapter, empty trimmed reads, all-N reads, lengths on both sides of direct_max (160)"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    rng = random.Random(seed)

    def rnd(k):
        return ''.join(rng.choice('ACGT') for _ in range(k))
    reads = [yt * 3, rnd(20) + yt + yt + rnd(20), rnd(5) + yt + yt[6:] + rnd(30), yt + rnd(40) + yb + rnd(10) + yt,
             yb + yb + yb + yb, 'ACG', yt[:10], 'N' * 200, 'N' * 40, rnd(120) + yt + rnd(10), rnd(150), yt + yb,
             rnd(400) + yb + rnd(300) + yt + yt + rnd(200), rnd(900) + yt + rnd(500) + yb + yb + rnd(100), rnd(1400),
             yt[:12] + yt[12:].lower() + 'N' * 30 + yt, 'X' + yt + '-' * 5 + yt, '']
    for _ in range(24):
        parts = [rnd(rng.randint(0, 300))]
        for _ in range(rng.randint(0, 4)):
            parts += [rng.choice((yt, yb, yt[3:], yb[:-4])), rnd(rng.randint(0, 120))]
        reads.append(''.join(parts))
    st = np.zeros(len(reads), dtype=np.int64)
    et = np.zeros(len(reads), dtype=np.int64)
    st[5] = 10                              # 'ACG' trimmed to nothing
    st[11] = len(reads[11])                 # an empty trimmed read
    et[12] = 50
    st[13], et[13] = 30, 30
    return reads, st, et


def _adapters():
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    return [('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb)]


def _compare_paths(W, monkeypatch, scheme, threshold=85.0, adapters=None, expect_device=True):
    from porechop_b200 import fastq
    monkeypatch.setattr(fastq, 'W', W)
    reads, st, et = _stress_reads()
    batch = _batch(reads)
    ads = adapters or _adapters()
    host = fastq.find_middle_hits(batch, st, et, ads, threshold, scheme, device=False)
    calls = []
    orig = W.adapter_middle_scan

    def spy(*a, **k):
        try:
            r = orig(*a, **k)
        except W.EngineError as e:
            calls.append(e.code)
            raise
        calls.append(0)
        return r
    monkeypatch.setattr(W, 'adapter_middle_scan', spy)
    dev = fastq.find_middle_hits(batch, st, et, ads, threshold, scheme, device=True)
    monkeypatch.setattr(W, 'adapter_middle_scan', orig)
    assert dev == host
    assert calls == [0 if expect_device else W.ERR_ARG]
    return host


def test_sim_find_middle_hits_device_equals_host_rounds(SW, monkeypatch):
    for scheme in ((3, -6, -5, -2), LINEAR):
        hits = _compare_paths(SW, monkeypatch, scheme)
        assert max(len(v) for v in hits.values()) >= 3       # several rounds ran (masking exercised)
    hits = _compare_paths(SW, monkeypatch, (3, -6, -5, -2), threshold=60.0)
    assert sum(len(v) for v in hits.values()) > 40
    from porechop_b200 import workloads as wl
    bc = [s for s in wl.load_adapter_sets()['sets'] if s['name'].endswith('(forward)')][0]
    _compare_paths(SW, monkeypatch, (3, -6, -5, -2), adapters=_adapters() + [tuple(bc['start']), tuple(bc['end'])])
    # direct_max below / above every read: the two-pass class and the one-pass class on the same inputs
    for dm in (40, 5000):
        SW.set_option('direct_max', dm)
        try:
            _compare_paths(SW, monkeypatch, (3, -6, -5, -2))
        finally:
            SW.set_option('direct_max', 160)


def test_sim_inputs_outside_the_device_scan_fall_back_to_host_rounds(SW, monkeypatch):
    yt = _adapters()[0][1]
    _compare_paths(SW, monkeypatch, (3, -6, -5, -2), threshold=float('nan'), expect_device=False)
    _compare_paths(SW, monkeypatch, (3, -6, -5, -2), adapters=[('a', yt), ('n', yt[:8] + 'N' + yt[9:])], expect_device=False)
    _compare_paths(SW, monkeypatch, (3, -6, 1, -2), expect_device=False)       # positive gap open: generic int32 kernel
    _compare_paths(SW, monkeypatch, (3, -6, 0, -2), expect_device=False)       # zero gap score: no window bound
    reads, _, _ = _stress_reads()
    sb, so = SW.pack_sequences(reads)
    ab, ao = SW.pack_sequences([a[1] for a in _adapters()], offset_dtype=np.int32)
    for thr in (0.0, -5.0):                 # (no host comparison: with a threshold <= 0 the reference's loop need not end)
        with pytest.raises(SW.EngineError) as e:
            SW.adapter_middle_scan(sb, so, ab, ao, (3, -6, -5, -2), thr)
        assert e.value.code == SW.ERR_ARG


def test_sim_hits_cap_too_small_reports_the_total_and_the_wrapper_retries(SW):
    from ctypes import byref, c_int64
    reads, _, _ = _stress_reads()
    sb, so = SW.pack_sequences(reads)
    ab, ao = SW.pack_sequences([a[1] for a in _adapters()], offset_dtype=np.int32)
    n_hits, hits = SW.adapter_middle_scan(sb, so, ab, ao, (3, -6, -5, -2), 85.0)
    assert len(hits) == n_hits.sum() > 20
    nh = np.zeros(len(reads), dtype=np.int32)
    small = np.zeros((3, 10), dtype=np.int32)
    total = c_int64(0)
    rc = SW.C_LIB.adapterMiddleScan(sb.ctypes.data, so.ctypes.data, len(reads), ab.ctypes.data, ao.ctypes.data, len(ao) - 1,
                                    3, -6, -5, -2, 85.0, nh.ctypes.data, small.ctypes.data, 3, byref(total))
    assert rc == SW.ERR_SPACE and total.value == len(hits) and np.array_equal(nh, n_hits)
    # each hit is {adapter, the alignment's ordinary record}: the record formats like any other
    from porechop_b200.align import scores_from_records
    full, _, _, _ = scores_from_records(np.ascontiguousarray(hits[:, 1:]))
    assert (full >= 85.0).all() and set(hits[:, 0]) <= {0, 1}
    assert SW.format_record(hits[0, 1:]).count(',') == 6


_ORDER_SCRIPT = r'''
import json, sys
sys.path[:0] = [%r, %r, %r]
import sim_engine, test_middle_scan as T
W = sim_engine.load()
reads, st, et = T._stress_reads()
sb, so = W.pack_sequences(reads)
ab, ao = W.pack_sequences([a[1] for a in T._adapters()], offset_dtype=__import__('numpy').int32)
W.set_option('chunk_tasks', 16)
n, h = W.adapter_middle_scan(sb, so, ab, ao, (3, -6, -5, -2), 70.0)
print(json.dumps([n.tolist(), h.tolist()]))
'''


def test_sim_result_does_not_depend_on_the_append_order(SW):
    """the order of the warps' atomic appends differs between interleavings (PBSIM_ORDER); the hits must not"""
    script = _ORDER_SCRIPT % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    outs = []
    for order in ('', 'reverse', 'random:3', 'random:11'):
        env = dict(os.environ, PBSIM_ORDER=order) if order else dict(os.environ)
        env.pop('PBSIM_ORDER', None) if not order else None
        r = subprocess.run([sys.executable, '-c', script], env=env, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(json.loads(r.stdout.strip().splitlines()[-1]))
    assert all(o == outs[0] for o in outs[1:])
    assert sum(outs[0][0]) > 20


def test_sim_trim_and_demux_reproduce_the_reference_cli_with_the_device_scan(SW, monkeypatch):
    """the flat pipeline with PB200_DEVICE_MIDDLE on the simulated engine: the reference CLI's files, byte for byte (the
    golden cases include chimeras with one and two middle adapters)"""
    from porechop_b200 import fastq
    import test_fastq_emit as T
    monkeypatch.setattr(fastq, 'W', SW)
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
    calls = []
    orig = SW.adapter_middle_scan
    monkeypatch.setattr(SW, 'adapter_middle_scan', lambda *a, **k: calls.append(1) or orig(*a, **k))
    for case in T.CASES:
        T._run(case)
    for case in T.BARCODE_CASES:
        T._run_demux(case)
    assert len(calls) >= 4


# ---- GPU tier ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_trim_and_demux_reproduce_the_reference_cli_with_the_device_scan(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, fastq
    import test_fastq_emit as T
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
    n0 = W.kernel_launches()
    for case in T.CASES:
        T._run(case)
    for case in T.BARCODE_CASES:
        T._run_demux(case)
    assert W.kernel_launches() > n0


@pytest.mark.gpu
def test_gpu_find_middle_hits_device_equals_host_rounds(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W
    for scheme in ((3, -6, -5, -2), LINEAR):
        hits = _compare_paths(W, monkeypatch, scheme)
        assert max(len(v) for v in hits.values()) >= 3
    _compare_paths(W, monkeypatch, (3, -6, -5, -2), threshold=60.0)
    _compare_paths(W, monkeypatch, (3, -6, -5, -2), threshold=float('nan'), expect_device=False)
    _compare_paths(W, monkeypatch, (3, -6, 1, -2), expect_device=False)


@pytest.mark.gpu
def test_gpu_device_resident_entry_point_equals_host_buffers():
    import torch
    from porechop_b200 import cpp_function_wrappers as W, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads(400, yt, yb, seed=5, chimera_p=0.5, max_len=6000)
    reads, _, _ = _stress_reads()
    sb, so = W.pack_sequences(reads)
    buf = np.concatenate([buf, sb])
    off = np.concatenate([off, so[1:] + off[-1]])
    ab, ao = wl.pack_adapters([yt, yb])
    exp_n, exp_h = W.adapter_middle_scan(buf, off, ab, ao, wl.DEFAULT_SCORING, 75.0)
    assert exp_n.max() >= 2
    d_buf = torch.from_numpy(buf).cuda()
    d_off = torch.from_numpy(off).cuda()
    keep = d_buf.clone()
    for max_len in (int(np.diff(off).max()), -1):
        n_hits, hits = W.adapter_middle_scan_device(d_buf.data_ptr(), d_off.data_ptr(), len(off) - 1, len(buf), max_len, ab, ao,
                                                    wl.DEFAULT_SCORING, 75.0, torch.cuda.current_stream().cuda_stream)
        assert np.array_equal(n_hits, exp_n) and np.array_equal(hits, exp_h)
    assert torch.equal(d_buf, keep)                       # the caller's reads are not masked


@pytest.mark.gpu
def test_gpu_config4_shape_device_equals_host_rounds():
    """BASELINE config 4 per GPU: 1.25 M synthetic reads, 5 % chimeras, {Y_Top, Y_Bottom}"""
    from porechop_b200 import fastq, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(1250000, yt, yb, chimera_p=0.05)
    n = len(off) - 1
    z8 = np.zeros(0, dtype=np.uint8)
    batch = fastq.FastqBatch(z8, np.zeros(n + 1, dtype=np.int64), buf, off, buf, off, np.zeros(n, dtype=bool))
    zero = np.zeros(n, dtype=np.int64)
    ads = _adapters()
    dev = fastq.find_middle_hits(batch, zero, zero, ads, 85.0, wl.DEFAULT_SCORING, device=True)
    host = fastq.find_middle_hits(batch, zero, zero, ads, 85.0, wl.DEFAULT_SCORING, device=False)
    assert dev == host
    assert len(dev) > 0.03 * n
    assert max(len(v) for v in dev.values()) >= 2        # a hit in round >= 1: masking and re-alignment ran
