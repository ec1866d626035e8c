"""GPU tier (pytest -m gpu): engine calls on different CUDA streams, with no synchronisation between them.

adapterAlignmentBatchDevice returns with its work queued, and every entry point uses the engine's shared stage buffers;
the engine orders each call after the work an earlier call left queued (include/porechop_b200.h).  Here the first call is
large enough to be still running when the next one is issued -- asserted with a CUDA event, so that a pass proves real
overlap -- and every call's records must equal the oracle's, computed before any call.  tests/test_stream_order.py checks
the same sequences for races on the host-simulated engine."""
import threading

import numpy as np
import pytest

from helpers import oracle_batch

pytestmark = pytest.mark.gpu

SC = (3, -6, -5, -2)


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope='module')
def W():
    from porechop_b200 import cpp_function_wrappers as w
    assert w.device_count() > 0
    return w


@pytest.fixture(scope='module')
def data():
    """a long first batch (300 000 end windows and 200 reads of up to 15 kb: the two-pass path) and smaller second batches
    (windows, long reads), all against the two NSK007 adapters, with their oracle records"""
    from porechop_b200 import workloads as wl
    yt, yb = wl.nsk007()
    abuf, aoff = wl.pack_adapters([yt, yb])
    _, sw, _ = wl.synth_end_windows(300000, yt, yb, seed=51)
    wb, wo = wl.windows_to_batch(sw)
    lb, lo = wl.synth_reads(200, yt, yb, seed=52, chimera_p=0.3, max_len=15000)
    big = (np.concatenate([wb, lb]), np.concatenate([wo, lo[1:] + wo[-1]]))
    _, ew, _ = wl.synth_end_windows(20000, yt, yb, seed=53)
    small_w = wl.windows_to_batch(ew)
    small_l = wl.synth_reads(40, yt, yb, seed=54, chimera_p=0.3, max_len=8000)
    out = {}
    for name, (b, o) in (('big', big), ('windows', small_w), ('long', small_l)):
        b, o = np.ascontiguousarray(b, dtype=np.uint8), np.ascontiguousarray(o, dtype=np.int64)
        out[name] = (b, o, oracle_batch(b, o, abuf, aoff, SC))
    return out, abuf, aoff


def _warm(torch, W, d, abuf, aoff):
    """one synchronised call per batch first: the engine's buffers reach the sizes these batches need, so no later call
    grows one -- a cudaFree, which would wait for the device and end the overlap the tests assert"""
    for batch in d.values():
        Call(torch, W, batch, abuf, aoff, torch.cuda.Stream())().check()


class Call:
    """one adapter_alignment_batch_device call: reads uploaded on `stream` (a torch stream, or None = torch's default stream
    and the library's NULL stream), records compared with the oracle's"""

    def __init__(self, torch, W, batch, abuf, aoff, stream):
        self.torch, self.W, self.abuf, self.aoff, self.stream = torch, W, abuf, aoff, stream
        b, o, self.exp = batch
        self.n, self.total, self.max_len = len(o) - 1, len(b), int(np.diff(o).max())
        s = stream if stream is not None else torch.cuda.default_stream()
        with torch.cuda.stream(s):
            self.db = torch.from_numpy(b).pin_memory().to('cuda', non_blocking=True)
            self.do = torch.from_numpy(o).pin_memory().to('cuda', non_blocking=True)
            self.dout = torch.empty((self.n * 2, 9), dtype=torch.int32, device='cuda')
            self.dout.fill_(-7)

    def __call__(self):
        self.W.adapter_alignment_batch_device(self.db.data_ptr(), self.do.data_ptr(), self.n, self.total, self.max_len, self.abuf,
                                              self.aoff, SC, self.dout.data_ptr(),
                                              self.stream.cuda_stream if self.stream is not None else 0)
        self.done = self.torch.cuda.Event()
        self.done.record(self.stream if self.stream is not None else self.torch.cuda.default_stream())
        return self

    def check(self):
        self.torch.cuda.synchronize()
        assert np.array_equal(self.dout.cpu().numpy(), self.exp)


def test_device_calls_on_two_streams(torch, W, data):
    d, abuf, aoff = data
    _warm(torch, W, d, abuf, aoff)
    for second in ('windows', 'long'):
        A, B = torch.cuda.Stream(), torch.cuda.Stream()
        c1 = Call(torch, W, d['big'], abuf, aoff, A)
        c2 = Call(torch, W, d[second], abuf, aoff, B)
        torch.cuda.synchronize()
        c1()
        c2()
        assert not c1.done.query(), 'the first call finished before the second was queued: nothing overlapped'
        c3 = Call(torch, W, d['windows'], abuf, aoff, A)()
        W.synchronize()
        for c in (c1, c2, c3):
            c.check()


def test_device_call_then_null_stream(torch, W, data):
    """NULL = the library's own stream, which waits for the work queued on the legacy default stream (torch's default
    stream): the second call's reads are uploaded there, asynchronously, right before the call"""
    d, abuf, aoff = data
    _warm(torch, W, d, abuf, aoff)
    A = torch.cuda.Stream()
    c1 = Call(torch, W, d['big'], abuf, aoff, A)
    torch.cuda.synchronize()
    c1()
    c2 = Call(torch, W, d['long'], abuf, aoff, None)()
    assert not c1.done.query(), 'the first call finished before the second was queued: nothing overlapped'
    W.synchronize()
    c1.check()
    c2.check()


def test_device_call_then_host_buffer_calls(torch, W, data):
    d, abuf, aoff = data
    _warm(torch, W, d, abuf, aoff)
    b, o, exp = d['windows']
    lb, lo, lexp = d['long']
    n = len(o) - 1
    ps = np.repeat(np.arange(n, dtype=np.int32), 2)[::-1].copy()
    pa = np.tile(np.arange(2, dtype=np.int32), n)[::-1].copy()
    for host in (lambda: np.array_equal(W.adapter_alignment_batch(b, o, abuf, aoff, SC), exp),
                 lambda: all(np.array_equal(g, e) for g, e in zip(
                     W.adapter_alignment_batch_multi([(lb, lo, abuf, aoff), (b, o, abuf, aoff)], SC), (lexp, exp))),
                 lambda: np.array_equal(W.adapter_alignment_batch(b, o, abuf, aoff, SC, ps, pa), exp[::-1])):
        A = torch.cuda.Stream()
        c1 = Call(torch, W, d['big'], abuf, aoff, A)
        torch.cuda.synchronize()
        c1()
        assert not c1.done.query(), 'the device call finished before the host call started: nothing overlapped'
        assert host()
        c1.check()


def test_device_call_then_middle_scans_and_end_decisions(torch, W, data):
    from porechop_b200 import hostio
    d, abuf, aoff = data
    lb, lo, _ = d['long']
    b, o, exp = d['windows']
    exp_nh, exp_hits = W.adapter_middle_scan(lb, lo, abuf, aoff, SC, 90.0)
    dlb, dlo = torch.from_numpy(lb).cuda(), torch.from_numpy(lo).cuda()
    exp_trim = hostio.end_trim(exp.reshape(-1, 2, 9), True, 150, 2, 75.0, 4)
    _warm(torch, W, d, abuf, aoff)
    calls = [
        lambda B: W.adapter_middle_scan_device(dlb.data_ptr(), dlo.data_ptr(), len(lo) - 1, len(lb), -1, abuf, aoff, SC, 90.0,
                                               B.cuda_stream),
        lambda B: W.adapter_middle_scan(lb, lo, abuf, aoff, SC, 90.0),
        lambda B: W.adapter_end_decisions([(b, o, abuf, aoff, True, [])], SC, 150, 2, 75.0, 4, want_records=True)]
    for k, call in enumerate(calls):
        A, B = torch.cuda.Stream(), torch.cuda.Stream()
        c1 = Call(torch, W, d['big'], abuf, aoff, A)
        torch.cuda.synchronize()
        c1()
        assert not c1.done.query(), 'the device call finished before the next call started: nothing overlapped'
        got = call(B)
        if k < 2:
            assert np.array_equal(got[0], exp_nh) and np.array_equal(got[1], exp_hits)
        else:
            (trim, _, rec), = got
            assert np.array_equal(rec.reshape(-1, 9), exp)
            assert np.array_equal(trim.astype(np.int64), exp_trim)
        c1.check()


def test_four_host_threads_each_with_its_own_stream(torch, W, data):
    from porechop_b200 import workloads as wl
    d, abuf, aoff = data
    yt, yb = wl.nsk007()
    batches = []
    for t in range(4):
        per = []
        for k in range(3):
            if k == 1:
                bb, oo = wl.synth_reads(30, yt, yb, seed=600 + 10 * t + k, chimera_p=0.3, max_len=6000)
            else:
                _, sw, _ = wl.synth_end_windows(30000, yt, yb, seed=600 + 10 * t + k)
                bb, oo = wl.windows_to_batch(sw)
            bb, oo = np.ascontiguousarray(bb), np.ascontiguousarray(oo, dtype=np.int64)
            per.append((bb, oo, oracle_batch(bb, oo, abuf, aoff, SC)))
        batches.append(per)
    calls = [[None] * 3 for _ in range(4)]
    errors = []

    def run(t):
        try:
            s = torch.cuda.Stream()
            for k in range(3):
                calls[t][k] = Call(torch, W, batches[t][k], abuf, aoff, s)()
        except Exception as e:           # reported after the join
            errors.append(e)
    threads = [threading.Thread(target=run, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    W.synchronize()
    for per in calls:
        for c in per:
            c.check()
