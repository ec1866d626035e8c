"""gzip members written on the H100 (pb200GzipDevice, device_reads.gzip_bytes, trim_fastq / demux_fastq with gz=True).  The
device must write exactly the simulated engine's bytes (golden_gzip.json, tests/golden/make_golden_gzip.py), and every file
must decompress to its input.  The CPU tier is tests/test_gzip_device.py."""
import gzip
import hashlib

import numpy as np
import pytest

from gzip_inputs import BLOCK, check_file, edge_inputs, golden_cases
from helpers import load_golden

pytestmark = pytest.mark.gpu


def _run(data, seg=None, block=BLOCK, stream_ptr=0, d=None):
    import torch
    from porechop_b200 import cpp_function_wrappers as W
    if d is None:
        d = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()
    cap = W.gzip_bound(len(data), 1 if seg is None else len(seg) - 1, block)
    out = torch.empty(max(cap, 1), dtype=torch.uint8, device='cuda')
    total, off = W.pb200_gzip_device(d.data_ptr(), len(data), seg, block=block, d_out_ptr=out.data_ptr(), out_cap=cap,
                                     stream_ptr=stream_ptr)
    return out[:total].cpu().numpy().tobytes(), off


def test_gpu_gzip_equals_simulator_golden():
    """the device's bytes are the simulated engine's, case by case"""
    g = load_golden('golden_gzip.json')
    cases = golden_cases()
    assert sorted(cases) == sorted(g)
    for name, (data, seg, block) in cases.items():
        gz, off = _run(data, seg, block)
        assert len(gz) == g[name]['size'] and [int(x) for x in off] == g[name]['seg_out'], name
        assert hashlib.sha256(gz).hexdigest() == g[name]['sha256'], name
        assert gzip.decompress(gz) == data, name


def test_gpu_gzip_edges():
    for name, data in edge_inputs().items():
        gz, _ = _run(data)
        check_file(gz, data, BLOCK)


def test_gpu_gzip_config4_file_and_48_bins():
    """a config-4-sized emit output as one file and as 48 barcode bins, round-tripped bin by bin"""
    import torch
    from porechop_b200 import device_reads
    from test_gpu_demux_reads import _shape
    from test_gpu_emit_reads import _config4, _cuda, _names
    batch, sets = _config4(30000)
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    em = device_reads.emit_reads(device_reads.trim_reads(seq, off, sets, (3, -6, -5, -2), qual), *_names(batch), 'fastq')
    plain = em.data.cpu().numpy().tobytes()
    g = device_reads.gzip_bytes(em.data)
    assert g.ranges is None
    check_file(g.data.cpu().numpy().tobytes(), plain, 65536)

    batch, sets = _shape(48, 30000)
    seq, off, qual = _cuda(batch.seq, batch.seq_off, batch.qual)
    r = device_reads.demux_reads(seq, off, sets, (3, -6, -5, -2), qual, forward_or_reverse='forward', barcode_threshold=75.0,
                                 barcode_diff=5.0, require_two_barcodes=False, discard_unassigned=False)
    em = device_reads.emit_reads(r, *_names(batch), 'fastq')
    plain = em.data.cpu().numpy().tobytes()
    g = device_reads.gzip_bytes(em.data, em.bins)
    host = torch.empty(g.data.numel(), dtype=torch.uint8, pin_memory=True).copy_(g.data).numpy().tobytes()
    assert len(em.bins) >= 30 and set(g.ranges) == set(em.bins)
    for name, (b0, b1) in g.ranges.items():
        p0, p1 = em.bins[name]
        check_file(host[b0:b1], plain[p0:p1], 65536)


def test_gpu_gzip_input_written_on_a_side_stream_right_before_the_call():
    import torch
    data = edge_inputs()['several_blocks'] * 20
    src = torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).pin_memory()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d = torch.empty(len(data), dtype=torch.uint8, device='cuda')
        d.fill_(0)
        d.copy_(src, non_blocking=True)
        gz, _ = _run(data, block=BLOCK, stream_ptr=side.cuda_stream, d=d)
    assert gzip.decompress(gz) == data


def test_gpu_trim_and_demux_fastq_gz():
    """trim_fastq / demux_fastq with gz=True decompress to the host functions' bytes"""
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['cases']['default']
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    data = g['input_fastq'].encode()
    got, _ = device_reads.trim_fastq(data, sets, c['scoring'], gz=True, **o)
    assert gzip.decompress(got).decode() == c['output']
    c = g['barcode_cases']['bins_default']
    o = dict(c['options'])
    data = g['barcoded_fastq'].encode()
    exp, _ = fastq.demux_fastq(data, c['matching_sets'], c['scoring'], **o)
    bins, _ = device_reads.demux_fastq(data, c['matching_sets'], c['scoring'], gz=True, **o)
    assert {k: gzip.decompress(v) for k, v in bins.items()} == exp
