"""CPU tier, on the host-simulated engine (tests/sim): ordering between engine calls that use different CUDA streams.

The simulator runs every stream synchronously, so records come out right whatever the order; what it also does is track
the order CUDA guarantees (vector clocks over streams, events and host synchronisation, pbsim_cuda.h) and report every pair
of accesses to one device buffer that no such order separates.  adapterAlignmentBatchDevice returns with its work still
queued, and every entry point shares the engine's stage buffers (trace scratch, task records, codes, status word), so each
sequence below -- a device-resident call followed, without any synchronisation, by another call on another stream -- must
report no race, and every call's records must equal the oracle's."""
import ctypes
import os
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_batch

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

LEGACY = 1            # cudaStreamLegacy
DEFAULT = (3, -6, -5, -2)
GENERIC = (3, -6, 1, -2)      # a positive gap score: the generic int32 kernel


@pytest.fixture(scope='module')
def W():
    import sim_engine
    return sim_engine.load()


@pytest.fixture(autouse=True)
def _no_races(W):
    W.synchronize()
    W.clear_races()
    yield
    W.synchronize()


def _assert_no_races(W):
    n, text = W.races()
    assert n == 0, '%d racing accesses:\n%s' % (n, text[:6000])


class DeviceCall:
    """one adapterAlignmentBatchDevice call on reads uploaded to tracked device memory on `upload_stream`"""

    def __init__(self, W, buf, off, ads, sc, stream, upload_stream=None):
        from porechop_b200 import workloads as wl
        self.W, self.sc = W, sc
        self.buf, self.off = np.ascontiguousarray(buf, dtype=np.uint8), np.ascontiguousarray(off, dtype=np.int64)
        self.abuf, self.aoff = wl.pack_adapters(ads)
        self.n, self.n_ad = len(self.off) - 1, len(ads)
        self.exp = oracle_batch(self.buf, self.off, self.abuf, self.aoff, sc)
        self.out_bytes = self.n * self.n_ad * 36
        self.d_seq = W.device_alloc(len(self.buf) + 16)
        self.d_off = W.device_alloc(self.off.nbytes)
        self.d_out = W.device_alloc(self.out_bytes)
        up = stream if upload_stream is None else upload_stream
        W.upload(self.d_seq, self.buf.ctypes.data, len(self.buf), up)
        W.upload(self.d_off, self.off.ctypes.data, self.off.nbytes, up)
        self.stream = stream

    def __call__(self):
        self.W.adapter_alignment_batch_device(self.d_seq, self.d_off, self.n, len(self.buf), -1, self.abuf, self.aoff, self.sc,
                                              self.d_out, self.stream or 0)
        return self

    def check(self):
        got = np.ctypeslib.as_array((ctypes.c_int32 * (self.n * self.n_ad * 9)).from_address(self.d_out)).reshape(-1, 9)
        assert np.array_equal(got, self.exp)
        for p in (self.d_seq, self.d_off, self.d_out):
            self.W.device_free(p)


def _inputs():
    """(reads, offsets, adapters, scheme) of the three paths: 150-base end windows (single pass), long reads (score pass,
    windows from tasks2 / ends, codes in seq_codes), and a scheme outside the int16 kernels (generic class)"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    _, sw, ew = wl.synth_end_windows(300, yt, yb, seed=21)
    _, sw2, _ = wl.synth_end_windows(200, yt, yb, seed=22)
    w1, w2 = wl.windows_to_batch(sw), wl.windows_to_batch(ew)
    w3 = wl.windows_to_batch(sw2)
    l1 = wl.synth_reads(6, yt, yb, seed=23, chimera_p=0.5, max_len=2500)
    l2 = wl.synth_reads(5, yt, yb, seed=24, chimera_p=0.5, max_len=2500)
    g1, g2 = wl.windows_to_batch(sw[:20]), wl.windows_to_batch(ew[:25])
    return {'windows': (w1, w2, [yt, yb], DEFAULT), 'windows_cached': (w1, w3, [yt], DEFAULT),
            'long': (l1, l2, [yt, yb], DEFAULT), 'generic': (g1, g2, [yt], GENERIC)}


@pytest.fixture(scope='module')
def inputs():
    return _inputs()


@pytest.mark.parametrize('kind', ['windows', 'windows_cached', 'long', 'generic'])
def test_a_device_calls_on_two_streams(W, inputs, kind):
    (b1, o1), (b2, o2), ads, sc = inputs[kind]
    A, B = W.stream_create(), W.stream_create()
    c1 = DeviceCall(W, b1, o1, ads, sc, A)
    c2 = DeviceCall(W, b2, o2, ads, sc, B)
    c1()                # the first call may plan the adapters (a device synchronise); the second finds them cached
    c2()
    c3 = DeviceCall(W, b1, o1, ads, sc, A)()       # and back to the first stream
    W.synchronize()
    _assert_no_races(W)
    for c in (c1, c2, c3):
        c.check()


@pytest.mark.parametrize('kind', ['windows', 'long'])
def test_b_device_call_then_null_stream(W, inputs, kind):
    """NULL is the library's own stream; it waits for the work queued so far on the legacy default stream, here the
    upload of the second call's reads"""
    (b1, o1), (b2, o2), ads, sc = inputs[kind]
    A = W.stream_create()
    c1 = DeviceCall(W, b1, o1, ads, sc, A)()
    c2 = DeviceCall(W, b2, o2, ads, sc, None, upload_stream=LEGACY)()
    c3 = DeviceCall(W, b1, o1, ads, sc, A)()
    W.synchronize()
    _assert_no_races(W)
    for c in (c1, c2, c3):
        c.check()


@pytest.mark.parametrize('kind', ['windows', 'long', 'generic'])
def test_c_device_call_then_host_buffer_calls(W, inputs, kind):
    (b1, o1), (b2, o2), ads, sc = inputs[kind]
    from porechop_b200 import workloads as wl
    abuf, aoff = wl.pack_adapters(ads)
    A = W.stream_create()
    exp2 = oracle_batch(b2, o2, abuf, aoff, sc)
    calls = []
    calls.append(DeviceCall(W, b1, o1, ads, sc, A)())
    assert np.array_equal(W.adapter_alignment_batch(b2, o2, abuf, aoff, sc), exp2)
    calls.append(DeviceCall(W, b1, o1, ads, sc, A)())
    got = W.adapter_alignment_batch_multi([(b2, o2, abuf, aoff), (b1, o1, abuf, aoff)], sc)
    assert np.array_equal(got[0], exp2) and np.array_equal(got[1], calls[0].exp)
    calls.append(DeviceCall(W, b1, o1, ads, sc, A)())
    n2 = len(o2) - 1
    ps = np.repeat(np.arange(n2, dtype=np.int32), len(ads))[::-1].copy()
    pa = np.tile(np.arange(len(ads), dtype=np.int32), n2)[::-1].copy()
    got = W.adapter_alignment_batch(b2, o2, abuf, aoff, sc, ps, pa)
    assert np.array_equal(got, oracle_batch(b2, o2, abuf, aoff, sc, ps, pa))
    W.synchronize()
    _assert_no_races(W)
    for c in calls:
        c.check()


def _middle_reads():
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads(8, yt, yb, seed=31, chimera_p=0.8, max_len=1200)
    return np.ascontiguousarray(buf), np.ascontiguousarray(off, dtype=np.int64), [yt, yb]


def test_d_device_call_then_middle_scans(W, inputs):
    from porechop_b200 import workloads as wl
    (b1, o1), _, ads, sc = inputs['long']
    mbuf, moff, mads = _middle_reads()
    mabuf, maoff = wl.pack_adapters(mads)
    exp_nh, exp_hits = W.adapter_middle_scan(mbuf, moff, mabuf, maoff, sc, 90.0)
    W.synchronize()
    W.clear_races()
    A, B = W.stream_create(), W.stream_create()
    d_seq, d_off = W.device_alloc(len(mbuf) + 16), W.device_alloc(moff.nbytes)
    W.upload(d_seq, mbuf.ctypes.data, len(mbuf), B)
    W.upload(d_off, moff.ctypes.data, moff.nbytes, B)
    c1 = DeviceCall(W, b1, o1, ads, sc, A)()
    nh, hits = W.adapter_middle_scan_device(d_seq, d_off, len(moff) - 1, len(mbuf), -1, mabuf, maoff, sc, 90.0, B)
    assert np.array_equal(nh, exp_nh) and np.array_equal(hits, exp_hits)
    c2 = DeviceCall(W, b1, o1, ads, sc, A)()
    nh, hits = W.adapter_middle_scan(mbuf, moff, mabuf, maoff, sc, 90.0)
    assert np.array_equal(nh, exp_nh) and np.array_equal(hits, exp_hits)
    W.synchronize()
    _assert_no_races(W)
    for c in (c1, c2):
        c.check()
    W.device_free(d_seq)
    W.device_free(d_off)


def test_e_device_call_then_end_decisions(W, inputs):
    from porechop_b200 import hostio, workloads as wl
    (b1, o1), (b2, o2), ads, sc = inputs['windows']
    abuf, aoff = wl.pack_adapters(ads)
    A = W.stream_create()
    c1 = DeviceCall(W, b1, o1, ads, sc, A)()
    (trim, _, rec), = W.adapter_end_decisions([(b2, o2, abuf, aoff, True, [])], sc, 150, 2, 75.0, 4, want_records=True)
    full = oracle_batch(b2, o2, abuf, aoff, sc)
    assert np.array_equal(rec.reshape(-1, 9), full)
    assert np.array_equal(trim.astype(np.int64), hostio.end_trim(full.reshape(-1, len(ads), 9), True, 150, 2, 75.0, 4))
    W.synchronize()
    _assert_no_races(W)
    c1.check()


def test_f_deferred_status_error_survives_host_calls():
    """A device-resident call leaves an error in the sticky status word (here set by a test-only switch of the engine, as a
    trace kernel sets it when a traceback leaves its window); the host-buffer calls queued behind it must not clear it:
    they report it, and pb200Synchronize still reports it, and clears it."""
    import sim_engine
    from porechop_b200 import workloads as wl
    W2 = sim_engine.load(['-DPB_TEST_DEFERRED_STATUS'])
    W2.synchronize()
    W2.clear_races()
    yt, yb = wl.nsk007()
    lbuf, loff = wl.synth_reads(6, yt, yb, seed=41, chimera_p=0.8, max_len=2500)
    _, sw, _ = wl.synth_end_windows(50, yt, yb, seed=42)
    wbuf, woff = wl.windows_to_batch(sw)
    abuf, aoff = wl.pack_adapters([yt, yb])
    A = W2.stream_create()
    n = len(wl.windows_to_batch(sw)[1]) - 1
    ps = np.repeat(np.arange(n, dtype=np.int32), 2)
    pa = np.tile(np.arange(2, dtype=np.int32), n)
    for host_call in (lambda: W2.adapter_alignment_batch(wbuf, woff, abuf, aoff, DEFAULT),
                      lambda: W2.adapter_alignment_batch(wbuf, woff, abuf, aoff, DEFAULT, ps, pa)):
        c = DeviceCall(W2, lbuf, loff, [yt, yb], DEFAULT, A)()
        # the host call finds the device call's error in the status word it shares with it, and leaves it there
        with pytest.raises(W2.EngineError) as e:
            host_call()
        assert e.value.code == 103 and 'window bound' in str(e.value)
        with pytest.raises(W2.EngineError) as e:
            W2.synchronize()
        assert e.value.code == 103 and 'window bound' in str(e.value)
        W2.synchronize()                         # reported once, then cleared
        for p in (c.d_seq, c.d_off, c.d_out):
            W2.device_free(p)
    # with the word clear, the host calls succeed
    assert np.array_equal(W2.adapter_alignment_batch(wbuf, woff, abuf, aoff, DEFAULT), oracle_batch(wbuf, woff, abuf, aoff, DEFAULT))
    n_races, text = W2.races()
    assert n_races == 0, text[:6000]
