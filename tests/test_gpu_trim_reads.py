"""Whole-read trimming in one engine call (adapterTrimReads / adapterTrimReadsDevice) through the real engine on the GPU: the
comparisons of tests/test_trim_reads.py, the config-4 read model and a demux shape against the two separate device calls,
the device-resident entry point on torch tensors on a non-default stream, and the reference CLI's bytes."""
import numpy as np
import pytest

import test_trim_reads as T

pytestmark = pytest.mark.gpu

DEFAULT = T.DEFAULT


def test_gpu_fused_call_equals_record_path(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W
    T._compare(W, monkeypatch)
    T._compare(W, monkeypatch, scheme=T.LINEAR)
    T._compare(W, monkeypatch, thr_mid=60.0)
    for end_size in (200, 400):
        T._compare(W, monkeypatch, end_size=end_size)
    T._compare(W, monkeypatch, sides='start')
    T._compare(W, monkeypatch, sides='end')
    T._compare(W, monkeypatch, middle=False)
    T._compare(W, monkeypatch, barcodes=12)
    T._compare(W, monkeypatch, barcodes=12, top2=True)


def _separate(W, buf, off, sides, mid, scheme, end_size, thr, want_top2=False):
    """adapterEndDecisions over the host-cut windows + adapterMiddleScan over the host-gathered trimmed reads"""
    from porechop_b200 import fastq
    (sw, swo), (ew, ewo) = fastq.end_windows(buf, off, end_size)
    (st, sp, _), (et, ep, _) = W.adapter_end_decisions([(sw, swo) + sides[0][:2] + (True, sides[0][2]),
                                                        (ew, ewo) + sides[1][:2] + (False, sides[1][2])], scheme, end_size, 2,
                                                       75.0, 4, want_top2=want_top2)
    a, b = fastq.trimmed_ranges(np.diff(off), st, et)
    tb, to = fastq._gather_ranges(buf, off[:-1] + a, off[:-1] + b)
    n_hits, h = W.adapter_middle_scan(tb, to, mid[0], mid[1], scheme, thr)
    return st, et, sp, ep, n_hits, h


def _same(got, exp):
    return all(g.dtype == e.dtype and np.array_equal(g, e) for g, e in zip(got, exp))


def test_gpu_config4_shape_and_demux_shape_equal_the_separate_calls():
    """config 4's read model (8-kb log-normal lengths, 5 % chimeras, {Y_Top, Y_Bottom}) over 60 000 reads, and a demux shape:
    barcode start / end columns ranked on the device (top2)"""
    from porechop_b200 import cpp_function_wrappers as W, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(60000, yt, yb, chimera_p=0.05)
    sides = (wl.pack_adapters([yt]) + ([0],), wl.pack_adapters([yb]) + ([0],))
    mid = wl.pack_adapters([yt, yb])
    got = W.adapter_trim_reads(buf, off, sides[0], sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0)
    exp = _separate(W, buf, off, sides, mid, DEFAULT, 150, 85.0)
    assert _same(got, exp)
    assert (got[0] > 0).mean() > 0.5 and (got[1] > 0).mean() > 0.5 and (got[4] > 0).mean() > 0.03 and got[4].max() >= 2
    bs, be = wl.demux_adapters()
    k = 48
    sides = (wl.pack_adapters([yt] + bs[:k]) + (list(range(1, k + 1)),), wl.pack_adapters([yb] + be[:k]) + (list(range(1, k + 1)),))
    n = 20000
    got = W.adapter_trim_reads(buf[:off[n]], off[:n + 1], sides[0], sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0, want_top2=True)
    exp = _separate(W, buf[:off[n]], off[:n + 1], sides, mid, DEFAULT, 150, 85.0, want_top2=True)
    assert _same(got, exp)


def test_gpu_device_variant_on_torch_tensors_on_a_side_stream():
    """the reads are written by a torch op on a non-default stream right before the call on that stream"""
    import torch
    from porechop_b200 import cpp_function_wrappers as W, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(20000, yt, yb, chimera_p=0.05)
    batch = T._batch(T.trim_reads_set())
    buf = np.concatenate([buf, batch.seq])
    off = np.concatenate([off, batch.seq_off[1:] + off[-1]])
    sides = (wl.pack_adapters([yt]) + ([0],), wl.pack_adapters([yb]) + ([0],))
    mid = wl.pack_adapters([yt, yb])
    exp = W.adapter_trim_reads(buf, off, sides[0], sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0)
    src = torch.from_numpy(buf).cuda()
    d_off = torch.from_numpy(off).cuda()
    s = torch.cuda.Stream()
    for max_len in (int(np.diff(off).max()), -1):
        d_buf = torch.zeros(len(buf), dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            d_buf.copy_(src)                                  # queued on s, still running when the call is issued
            got = W.adapter_trim_reads_device(d_buf.data_ptr(), d_off.data_ptr(), len(off) - 1, len(buf), max_len, sides[0],
                                              sides[1], mid, DEFAULT, 150, 2, 75.0, 4, 85.0, stream_ptr=s.cuda_stream)
        assert _same(got, exp)
        s.synchronize()
        assert torch.equal(d_buf, src)                        # the caller's reads are not masked
    assert exp[4].max() >= 2


def test_gpu_trim_and_demux_reproduce_the_reference_cli_in_one_call_per_chunk(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, fastq
    import test_fastq_emit as F
    monkeypatch.setattr(fastq, 'DEVICE_DECISIONS', True)
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', True)
    calls = {'trim': 0, 'other': 0}
    orig = W.adapter_trim_reads
    monkeypatch.setattr(W, 'adapter_trim_reads', lambda *a, **k: calls.__setitem__('trim', calls['trim'] + 1) or orig(*a, **k))
    for name in ('adapter_end_decisions', 'adapter_middle_scan'):
        f = getattr(W, name)
        monkeypatch.setattr(W, name, lambda *a, _f=f, **k: calls.__setitem__('other', calls['other'] + 1) or _f(*a, **k))
    for case in F.CASES:
        F._run(case)
    for case in F.BARCODE_CASES:
        F._run_demux(case)
    assert calls == {'trim': len(F.CASES) + len(F.BARCODE_CASES), 'other': 0}
