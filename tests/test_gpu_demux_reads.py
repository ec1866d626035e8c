"""Demultiplexed output reads on the device (adapterDemuxReadsDevice through device_reads.demux_reads on torch tensors) on the
GPU: the reference CLI's bin files, 48- and 96-barcode shapes of the config-4 read model against fastq.demux_fastq, inputs
written on a side stream right before the call, the ERR_SPACE retry, and each bin as one contiguous slice."""
import numpy as np
import pytest

from helpers import load_golden

pytestmark = pytest.mark.gpu

DEFAULT = (3, -6, -5, -2)
BARCODE_KEYS = ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes', 'discard_unassigned')


def _bins(batch, r, fmt):
    """each bin's file: emit_parts over the bin's slice (host copies); checks that every bin is one contiguous slice"""
    from porechop_b200 import fastq
    seq, qual = r.seq.cpu().numpy(), r.qual.cpu().numpy() if r.qual is not None else None
    off, read, part = r.off.cpu().numpy(), r.read.cpu().numpy(), r.part.cpu().numpy()
    starts = [r0 for r0, _ in r.bins.values()]
    assert starts == sorted(starts) and (not starts or starts[0] == 0)
    assert sum(r1 - r0 for r0, r1 in r.bins.values()) == len(read) and np.all(np.diff(off) > 0) and off[0] == 0
    out = {}
    for name, (r0, r1) in r.bins.items():
        rd = read[r0:r1]
        assert np.all(np.diff(rd) >= 0) and all(r.calls[k] == name for k in np.unique(rd).tolist())
        out[name] = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, (seq, qual, off[r0:r1 + 1], rd, part[r0:r1]), fmt)
    return out


def _run(batch, sets, scheme, o, bc, fmt='fastq'):
    import torch
    from porechop_b200 import device_reads
    seq = torch.from_numpy(np.ascontiguousarray(batch.seq)).cuda()
    off = torch.from_numpy(np.ascontiguousarray(batch.seq_off)).cuda()
    qual = torch.from_numpy(np.ascontiguousarray(batch.qual)).cuda() if fmt == 'fastq' else None
    r = device_reads.demux_reads(seq, off, sets, scheme, qual, **bc, **o)
    assert torch.equal(seq.cpu(), torch.from_numpy(np.ascontiguousarray(batch.seq)))
    return r, _bins(batch, r, fmt)


def test_gpu_demux_golden_barcode_cases():
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    for name, c in g['barcode_cases'].items():
        o = dict(c['options'])
        fmt = o.pop('fmt')
        bc = {k: o.pop(k) for k in BARCODE_KEYS}
        _, bins = _run(batch, c['matching_sets'], c['scoring'], o, bc, fmt)
        assert sorted(k + '.' + fmt for k in bins) == sorted(c['bins']), name
        for k, v in bins.items():
            assert v.decode() == c['bins'][k + '.' + fmt], (name, k)


def _shape(k, n=60000):
    """config-4 reads with a barcode before the Y adapters (6 blocks, barcodes spread over the k bins), and the adapter sets"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    from test_gpu_trim_split_reads import _synth_batch
    yt, yb = wl.nsk007()
    bs, be = wl.demux_adapters()
    sets = [('SQK-NSK007', ('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))] + \
           [('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[j]), ('BC%02d_end' % (j + 1), be[j])) for j in range(k)]
    blocks = [_synth_batch(n // 6, bs[j] + yt, yb + be[j], seed=j) for j in range(0, k, k // 6)[:6]]
    seq, qual = np.concatenate([b.seq for b in blocks]), np.concatenate([b.qual for b in blocks])
    off, base = [np.zeros(1, dtype=np.int64)], 0
    for b in blocks:
        off.append(b.seq_off[1:] + base)
        base += len(b.seq)
    off = np.concatenate(off)
    names, name_off = W.pack_sequences(['r%d' % j for j in range(len(off) - 1)])
    return fastq.FastqBatch(names, name_off, seq, off, qual, off.copy(), np.zeros(len(off) - 1, dtype=bool)), sets


@pytest.mark.parametrize('k', [48, 96])
def test_gpu_demux_shapes_equal_demux_fastq(k):
    from porechop_b200 import fastq
    batch, sets = _shape(k)
    o = dict(min_split_read_size=200)
    for bc in (dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
                    discard_unassigned=False),
               dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=True,
                    discard_unassigned=True)):
        r, got = _run(batch, sets, DEFAULT, o, bc)
        bins, info = fastq.demux_fastq(batch, sets, DEFAULT, **o, **bc)
        assert r.calls == info['calls'] and len(set(r.calls)) >= 4
        assert sorted(got) == sorted(bins) and all(got[b] == bins[b] for b in bins)
        assert ('none' in got) == (not bc['discard_unassigned'])


def test_gpu_demux_inputs_written_on_a_side_stream_right_before_the_call():
    import torch
    from porechop_b200 import device_reads
    batch, sets = _shape(48, 24000)
    bc = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
              discard_unassigned=False)
    exp, exp_bins = _run(batch, sets, DEFAULT, {}, bc)
    src_seq, src_qual = torch.from_numpy(batch.seq).cuda(), torch.from_numpy(batch.qual).cuda()
    off = torch.from_numpy(batch.seq_off).cuda()
    seq, qual = torch.zeros_like(src_seq), torch.zeros_like(src_qual)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        seq.copy_(src_seq)                                     # queued on s, still running when the call is issued
        qual.copy_(src_qual)
        r = device_reads.demux_reads(seq, off, sets, DEFAULT, qual, **bc)
        got = _bins(batch, r, 'fastq')
    s.synchronize()
    assert r.calls == exp.calls and r.bins == exp.bins and got == exp_bins
    assert torch.equal(seq, src_seq) and torch.equal(qual, src_qual)


def test_gpu_demux_err_space_retry_from_a_tiny_capacity(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, device_reads
    batch, sets = _shape(48, 6000)
    bc = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
              discard_unassigned=True)
    o = dict(min_split_read_size=100)
    exp, exp_bins = _run(batch, sets, DEFAULT, o, bc)
    caps = []
    orig = W.adapter_demux_reads_device
    monkeypatch.setattr(W, 'adapter_demux_reads_device', lambda *a, **k: caps.append(k['parts_cap']) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_parts_cap', lambda n: 3)
    got, got_bins = _run(batch, sets, DEFAULT, o, bc)
    assert caps == [3, len(exp.read)] and got_bins == exp_bins and got.bins == exp.bins
    assert all(np.array_equal(g.cpu().numpy(), e.cpu().numpy()) for g, e in zip(got[:5], exp[:5]))
