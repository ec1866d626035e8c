"""Porechop's output files formatted on the device (pb200EmitReadsDevice through device_reads.emit_reads on torch tensors) on the
GPU: the reference CLI's files, the config-4 read model against fastq.emit_parts in FASTQ and FASTA with names with spaces and
RNA reads, a 48-barcode demux shape bin by bin, the alignment sweep of hand-made records, inputs written on a side stream right
before the call, and the ERR_SPACE retry."""
import numpy as np
import pytest

from helpers import load_golden

pytestmark = pytest.mark.gpu

DEFAULT = (3, -6, -5, -2)
BARCODE_KEYS = ('forward_or_reverse', 'barcode_threshold', 'barcode_diff', 'require_two_barcodes', 'discard_unassigned')


def _cuda(*arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _names(batch, rna=None):
    return _cuda(batch.name_buf, batch.name_off, np.asarray(batch.rna if rna is None else rna, dtype=np.uint8))


def _host(r):
    return tuple(x.cpu().numpy() if x is not None else None for x in r[:5])


def test_gpu_emit_golden_trim_and_barcode_cases():
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    batch = fastq.parse_fastq(g['input_fastq'].encode())
    for name, c in g['cases'].items():
        o = dict(c['options'])
        fmt = o.pop('fmt')
        sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
        seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
        r = device_reads.trim_reads(seq, off, sets, c['scoring'], qual if fmt == 'fastq' else None, **o)
        em = device_reads.emit_reads(r, *_names(batch), fmt)
        assert em.data.cpu().numpy().tobytes().decode() == c['output'], name
    batch = fastq.parse_fastq(g['barcoded_fastq'].encode())
    for name, c in g['barcode_cases'].items():
        o = dict(c['options'])
        fmt = o.pop('fmt')
        bc = {k: o.pop(k) for k in BARCODE_KEYS}
        seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
        r = device_reads.demux_reads(seq, off, c['matching_sets'], c['scoring'], qual if fmt == 'fastq' else None, **bc, **o)
        em = device_reads.emit_reads(r, *_names(batch), fmt)
        data = em.data.cpu().numpy().tobytes()
        assert sorted(k + '.' + fmt for k in em.bins) == sorted(c['bins']), name
        for k, (b0, b1) in em.bins.items():
            assert data[b0:b1].decode() == c['bins'][k + '.' + fmt], (name, k)


def _config4(n, seed=0):
    """the config-4 read model with random qualities, names with spaces (every fifth with a tab) and 20 % RNA reads"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(n, yt, yb, chimera_p=0.05)
    rng = np.random.default_rng(seed)
    qual = rng.integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences([('r%d\tch=%d' if k % 5 == 0 else 'r%d runid=ab%d ch=7') % (k, k) for k in range(n)])
    rna = rng.random(n) < 0.2
    sets = [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]
    return fastq.FastqBatch(names, name_off, buf, off, qual, off.copy(), rna), sets


def test_gpu_emit_config4_equals_emit_parts():
    from porechop_b200 import device_reads, fastq
    batch, sets = _config4(60000)
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    r = device_reads.trim_reads(seq, off, sets, DEFAULT, qual, min_split_read_size=100)
    parts = _host(r)
    assert (parts[4] > 0).sum() > 1000
    for fmt in ('fastq', 'fasta'):
        em = device_reads.emit_reads(r, *_names(batch), fmt)
        exp = fastq.emit_parts(batch.name_buf, batch.name_off, batch.rna, parts if fmt == 'fastq' else (parts[0], None) + parts[2:],
                               fmt)
        assert em.data.cpu().numpy().tobytes() == exp, fmt
        assert em.bins is None and em.off[-1].item() == len(exp)


def test_gpu_emit_demux_48_bins_slice_by_slice():
    from porechop_b200 import device_reads, fastq
    from test_gpu_demux_reads import _shape
    batch, sets = _shape(48)
    rna = np.arange(len(batch)) % 5 == 2
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    r = device_reads.demux_reads(seq, off, sets, DEFAULT, qual, forward_or_reverse='forward', barcode_threshold=75.0,
                                 barcode_diff=5.0, require_two_barcodes=False, discard_unassigned=False, min_split_read_size=200)
    em = device_reads.emit_reads(r, *_names(batch, rna), 'fastq')
    data, parts = em.data.cpu().numpy().tobytes(), _host(r)
    assert len(em.bins) >= 4 and list(em.bins) == list(r.bins)
    for name, (r0, r1) in r.bins.items():
        b0, b1 = em.bins[name]
        exp = fastq.emit_parts(batch.name_buf, batch.name_off, rna, parts[:2] + (parts[2][r0:r1 + 1], parts[3][r0:r1],
                                                                                  parts[4][r0:r1]), 'fastq')
        assert data[b0:b1] == exp, name


def _raw(W, seq, qual, off, read, part, names, rna, fmt, stream_ptr=0):
    import torch
    from porechop_b200 import cpp_function_wrappers as real, fastq
    name_buf, name_off = real.pack_sequences([n.encode() for n in names])
    d = _cuda(np.frombuffer(bytes(seq), dtype=np.uint8), np.frombuffer(bytes(qual), dtype=np.uint8), np.asarray(off, dtype=np.int64),
              np.asarray(read, dtype=np.int32), np.asarray(part, dtype=np.int32), name_buf, name_off, np.asarray(rna, dtype=np.uint8))
    cap = 2 * len(seq) + len(read) * 40
    out, out_off = torch.empty(cap, dtype=torch.uint8, device='cuda'), torch.empty(len(read) + 1, dtype=torch.int64, device='cuda')
    n = W.pb200_emit_reads_device(len(read), d_seq_ptr=d[0].data_ptr(), d_qual_ptr=d[1].data_ptr(), seq_bytes=len(seq),
                                  d_off_ptr=d[2].data_ptr(), d_read_ptr=d[3].data_ptr(), d_part_ptr=d[4].data_ptr(),
                                  d_names_ptr=d[5].data_ptr(), d_name_off_ptr=d[6].data_ptr(), n_reads=len(names),
                                  name_bytes=len(name_buf), d_rna_ptr=d[7].data_ptr(), fmt=fmt, d_out_ptr=out.data_ptr(),
                                  out_cap=cap, d_out_off_ptr=out_off.data_ptr(), stream_ptr=stream_ptr)
    got = out[:n].cpu().numpy().tobytes()
    exp = fastq.emit_parts(name_buf, name_off, np.asarray(rna, dtype=bool),
                           (np.frombuffer(bytes(seq), dtype=np.uint8), np.frombuffer(bytes(qual), dtype=np.uint8) if fmt == 'fastq' else None,
                            np.asarray(off), np.asarray(read), np.asarray(part)), fmt)
    return got, exp


def test_gpu_emit_hand_made_records_and_alignment_sweep():
    from porechop_b200 import cpp_function_wrappers as W
    from test_emit_reads import _alignment_sweep, _hand_made
    for make in (_hand_made, lambda: _alignment_sweep(list(range(41)) + [100, 103])):
        args = make()
        for fmt in ('fastq', 'fasta'):
            got, exp = _raw(W, *args, fmt)
            assert got == exp, fmt


def test_gpu_emit_inputs_written_on_a_side_stream_right_before_the_call():
    import torch
    from porechop_b200 import device_reads
    batch, sets = _config4(12000, seed=3)
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    r = device_reads.trim_reads(seq, off, sets, DEFAULT, qual, min_split_read_size=100)
    src = _names(batch)
    exp = device_reads.emit_reads(r, *src, 'fastq').data.cpu()
    dst = [torch.zeros_like(x) for x in src]
    rec = [torch.zeros_like(x) for x in (r.seq, r.qual)]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for d, x in zip(dst + rec, src + [r.seq, r.qual]):
            d.copy_(x)                                       # queued on s, still running when the call is issued
        em = device_reads.emit_reads(r._replace(seq=rec[0], qual=rec[1]), *dst, 'fastq')
    s.synchronize()
    assert torch.equal(em.data.cpu(), exp)


def test_gpu_emit_err_space_retry_from_a_tiny_bound(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, device_reads
    batch, sets = _config4(6000, seed=4)
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    r = device_reads.trim_reads(seq, off, sets, DEFAULT, qual, min_split_read_size=100)
    exp = device_reads.emit_reads(r, *_names(batch), 'fastq')
    caps = []
    orig = W.pb200_emit_reads_device
    monkeypatch.setattr(W, 'pb200_emit_reads_device', lambda *a, **k: caps.append(k['out_cap']) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_out_cap', lambda *a: 7)
    got = device_reads.emit_reads(r, *_names(batch), 'fastq')
    assert caps == [7, exp.data.numel()]
    assert np.array_equal(got.data.cpu().numpy(), exp.data.cpu().numpy()) and np.array_equal(got.off.cpu().numpy(), exp.off.cpu().numpy())
