"""Porechop's output reads cut on the device (adapterTrimSplitReadsDevice through device_reads.trim_reads on torch tensors) on
the GPU: the reference CLI's bytes, the config-4 read model and a 48-barcode demux shape against fastq.emit over the host
path's decisions, inputs written on a side stream right before the call, and the ERR_SPACE retry."""
import numpy as np
import pytest

from helpers import load_golden

pytestmark = pytest.mark.gpu

DEFAULT = (3, -6, -5, -2)


def _run(batch, sets, scheme, o, fmt='fastq', barcodes=None, stream=None):
    """device_reads.trim_reads on torch copies of the batch; returns (result with host copies of the records, output bytes)"""
    import torch
    from porechop_b200 import device_reads, fastq
    seq = torch.from_numpy(np.ascontiguousarray(batch.seq)).cuda()
    off = torch.from_numpy(np.ascontiguousarray(batch.seq_off)).cuda()
    qual = torch.from_numpy(np.ascontiguousarray(batch.qual)).cuda() if fmt == 'fastq' else None
    r = device_reads.trim_reads(seq, off, sets, scheme, qual, barcodes=barcodes, **o)
    parts = tuple(x.cpu().numpy() if x is not None else None for x in r[:5])
    assert torch.equal(seq.cpu(), torch.from_numpy(np.ascontiguousarray(batch.seq)))
    r = r._replace(seq=parts[0], qual=parts[1], off=parts[2], read=parts[3], part=parts[4])
    return r, fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, parts, fmt)


def _bins(batch, r, fmt, discard_unassigned=False):
    from porechop_b200 import fastq
    calls, bins = np.array(r.calls, dtype=object), {}
    for name in dict.fromkeys(r.calls):
        if discard_unassigned and name == 'none':
            continue
        out = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, r[:5], fmt, select=(calls == name))
        if len(out):
            bins[name] = out
    return bins


def test_gpu_golden_cases_give_the_reference_cli_bytes():
    from porechop_b200 import fastq
    g = load_golden('golden_emit.json')
    batch = fastq.parse_fastq(g['input_fastq'].encode())
    for name, c in g['cases'].items():
        o = dict(c['options'])
        fmt = o.pop('fmt')
        sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
        _, out = _run(batch, sets, c['scoring'], o, fmt)
        assert out.decode() == c['output'], name
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    for name, c in g['barcode_cases'].items():
        o = dict(c['options'])
        fmt, discard_unassigned = o.pop('fmt'), o.pop('discard_unassigned')
        barcodes = {k: o.pop(k) for k in ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes')}
        r, _ = _run(batch, c['matching_sets'], c['scoring'], o, fmt, barcodes=barcodes)
        bins = _bins(batch, r, fmt, discard_unassigned)
        assert sorted(k + '.' + fmt for k in bins) == sorted(c['bins']), name
        for k, v in bins.items():
            assert v.decode() == c['bins'][k + '.' + fmt], (name, k)


def _synth_batch(n, start, end, seed=0, chimera_p=0.05):
    """the config-4 read model with names r<k> and synthetic qualities"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    buf, off = wl.synth_reads_fast(n, start, end, chimera_p=chimera_p)
    rng = np.random.default_rng(seed)
    qual = rng.integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences(['r%d' % k for k in range(n)])
    return fastq.FastqBatch(names, name_off, buf, off, qual, off.copy(), np.zeros(n, dtype=bool))


def test_gpu_config4_shape_equals_emit_over_the_host_decisions():
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    batch = _synth_batch(60000, yt, yb)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    adapters = fastq._middle_adapters(fastq._norm_sets(sets))
    for min_split in (1000, 100):
        o = dict(min_split_read_size=min_split)
        r, got = _run(batch, sets, DEFAULT, o)
        st, et, _, _, n_hits, h = W.adapter_trim_reads(batch.seq, batch.seq_off, wl.pack_adapters([yt]) + ([],),
                                                       wl.pack_adapters([yb]) + ([],), wl.pack_adapters([a[1] for a in adapters]),
                                                       DEFAULT, 150, 2, 75.0, 4, 85.0)
        hits = fastq._hits_dict(n_hits, h)
        assert np.array_equal(r.start_trim, st) and np.array_equal(r.end_trim, et) and r.hits == hits
        middle = fastq.middle_trim_ranges(hits, adapters, {'SQK-NSK007_Y_Top'}, {'SQK-NSK007_Y_Bottom'}, 10, 100)
        assert got == fastq.emit(batch, st, et, middle, 'fastq', min_split)
        assert len(hits) > 1000 and (r.part > 0).sum() > 1000


def test_gpu_demux_shape_48_barcodes_equals_demux_fastq():
    from porechop_b200 import fastq, workloads as wl
    yt, yb = wl.nsk007()
    bs, be = wl.demux_adapters()
    k = 48
    sets = [('SQK-NSK007', ('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))] + \
           [('Barcode %d (forward)' % (j + 1), ('BC%02d' % (j + 1), bs[j]), ('BC%02d_end' % (j + 1), be[j])) for j in range(k)]
    halves = [_synth_batch(6000, bs[j] + yt, yb + be[j], seed=j) for j in (3, 17)]
    parts = [np.concatenate(x) for x in zip(*[(b.seq, b.qual) for b in halves])]
    off = np.concatenate([halves[0].seq_off, halves[1].seq_off[1:] + halves[0].seq_off[-1]])
    n = len(off) - 1
    from porechop_b200 import cpp_function_wrappers as W
    names, name_off = W.pack_sequences(['r%d' % j for j in range(n)])
    batch = fastq.FastqBatch(names, name_off, parts[0], off, parts[1], off.copy(), np.zeros(n, dtype=bool))
    o = dict(min_split_read_size=200)
    barcodes = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False)
    r, _ = _run(batch, sets, DEFAULT, o, barcodes=barcodes)
    bins, info = fastq.demux_fastq(batch, sets, DEFAULT, **o, **barcodes)
    assert r.calls == info['calls'] and len(set(r.calls)) >= 3
    got = _bins(batch, r, 'fastq')
    assert sorted(got) == sorted(bins) and all(got[b] == bins[b] for b in bins)


def test_gpu_inputs_written_on_a_side_stream_right_before_the_call():
    import torch
    from porechop_b200 import device_reads, fastq, workloads as wl
    yt, yb = wl.nsk007()
    batch = _synth_batch(20000, yt, yb)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    exp, exp_bytes = _run(batch, sets, DEFAULT, {})
    src_seq, src_qual = torch.from_numpy(batch.seq).cuda(), torch.from_numpy(batch.qual).cuda()
    off = torch.from_numpy(batch.seq_off).cuda()
    seq, qual = torch.zeros_like(src_seq), torch.zeros_like(src_qual)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        seq.copy_(src_seq)                                     # queued on s, still running when the call is issued
        qual.copy_(src_qual)
        r = device_reads.trim_reads(seq, off, sets, DEFAULT, qual)
        parts = tuple(x.cpu().numpy() for x in r[:5])
    s.synchronize()
    assert fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, parts, 'fastq') == exp_bytes
    assert torch.equal(seq, src_seq) and torch.equal(qual, src_qual)


def test_gpu_err_space_retry_from_a_tiny_capacity(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, device_reads, workloads as wl
    yt, yb = wl.nsk007()
    batch = _synth_batch(5000, yt, yb)
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    exp, exp_bytes = _run(batch, sets, DEFAULT, dict(min_split_read_size=100))
    caps = []
    orig = W.adapter_trim_split_reads_device
    monkeypatch.setattr(W, 'adapter_trim_split_reads_device', lambda *a, **k: caps.append(k['parts_cap']) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_parts_cap', lambda n: 3)
    got, got_bytes = _run(batch, sets, DEFAULT, dict(min_split_read_size=100))
    assert caps == [3, len(exp.read)] and got_bytes == exp_bytes
    assert all(np.array_equal(g, e) for g, e in zip(got[:5], exp[:5]))
