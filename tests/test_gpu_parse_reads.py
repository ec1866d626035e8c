"""FASTQ / FASTA parsed on the GPU (pb200ParseReadsDevice through device_reads.parse_reads on torch tensors) and whole chunks from
input bytes to output bytes (device_reads.trim_fastq / demux_fastq): the host parser's fields on the golden inputs and on 10^5
config-4 reads as FASTQ, CRLF FASTQ and 70-column FASTA; the reference CLI's files; fastq.trim_fastq / demux_fastq byte for byte
on the config-4 model (trim, and 48 barcodes); input written on a side stream right before the call; the ERR_SPACE retry."""
import numpy as np
import pytest

from helpers import load_golden

pytestmark = pytest.mark.gpu

DEFAULT = (3, -6, -5, -2)


def _cuda_bytes(data):
    import torch
    return torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda()


def _check(data, kind, qual=True):
    """parse_reads equals the host parser on every field"""
    from porechop_b200 import device_reads, fastq
    b = fastq.parse_fastq(data) if kind == 'fastq' else fastq.parse_fasta(data)
    p = device_reads.parse_reads(_cuda_bytes(data), kind, qual)
    assert p.kind == kind
    assert p.names.cpu().numpy().tobytes() == b.name_buf.tobytes() and np.array_equal(p.name_off.cpu().numpy(), b.name_off)
    assert p.seq.cpu().numpy().tobytes() == b.seq.tobytes() and np.array_equal(p.seq_off.cpu().numpy(), b.seq_off)
    assert np.array_equal(p.rna.cpu().numpy().astype(bool), b.rna)
    if qual:
        assert np.array_equal(b.qual_off, b.seq_off) and p.qual.cpu().numpy().tobytes() == b.qual.tobytes()
    return b


def _config4_bytes(n, seed=0):
    """the config-4 read model as FASTQ bytes: random qualities (every 9th read's shorter than its bases), names with spaces and
    tabs, 20 % RNA reads (written with U), every 7th read in lower case"""
    from porechop_b200 import cpp_function_wrappers as W, fastq, workloads as wl
    yt, yb = wl.nsk007()
    buf, off = wl.synth_reads_fast(n, yt, yb, chimera_p=0.05)
    rng = np.random.default_rng(seed)
    qual = rng.integers(33, 75, len(buf), dtype=np.uint8)
    names, name_off = W.pack_sequences([('r%d\tch=%d' if k % 5 == 0 else 'r%d runid=ab%d ch=7') % (k, k) for k in range(n)])
    rna = rng.random(n) < 0.2
    batch = fastq.FastqBatch(names, name_off, buf, off, qual, off.copy(), rna)
    lines = fastq.emit(batch, fmt='fastq').split(b'\n')
    for k in range(0, n, 7):
        lines[4 * k + 1] = lines[4 * k + 1].lower()
    for k in range(3, n, 9):
        lines[4 * k + 3] = lines[4 * k + 3][:-5]
    return b'\n'.join(lines), [(('SQK-NSK007_Y_Top', yt), ('SQK-NSK007_Y_Bottom', yb))]


def test_gpu_parse_golden_inputs():
    from test_parse_reads import to_fasta
    for key in ('input_fastq', 'barcoded_fastq'):
        data = load_golden('golden_emit.json')[key].encode()
        b = _check(data, 'fastq')
        _check(data.replace(b'\n', b'\r\n'), 'fastq')
        for width in (7, 70):
            _check(to_fasta(b, width), 'fasta')


def test_gpu_parse_config4_fastq_crlf_fasta():
    from porechop_b200 import fastq
    data, _ = _config4_bytes(100000)
    b = _check(data, 'fastq')
    assert len(b) == 100000 and b.rna.sum() > 15000 and len(b.seq) > 5e8
    _check(data.replace(b'\n', b'\r\n'), 'fastq')
    fa = fastq.emit(b, fmt='fasta')                      # 70-column FASTA of the parsed reads
    _check(fa, 'fasta')
    _check(fa, 'fasta', qual=False)


def test_gpu_trim_and_demux_fastq_golden():
    from porechop_b200 import device_reads
    g = load_golden('golden_emit.json')
    for name, c in g['cases'].items():
        sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
        got, _ = device_reads.trim_fastq(g['input_fastq'].encode(), sets, c['scoring'], **c['options'])
        assert got.decode() == c['output'], name
    for name, c in g['barcode_cases'].items():
        fmt = c['options']['fmt']
        bins, _ = device_reads.demux_fastq(g['barcoded_fastq'].encode(), c['matching_sets'], c['scoring'], **c['options'])
        assert sorted(k + '.' + fmt for k in bins) == sorted(c['bins']), name
        for k, v in bins.items():
            assert v.decode() == c['bins'][k + '.' + fmt], (name, k)


def test_gpu_trim_fastq_config4_equals_host(monkeypatch):
    from porechop_b200 import device_reads, fastq
    data, sets = _config4_bytes(20000, seed=1)
    exp, exp_info = fastq.trim_fastq(data, sets, DEFAULT, min_split_read_size=100)
    monkeypatch.setattr(fastq, 'trim_fastq', None)       # the device path only
    for fmt in ('fastq', 'fasta'):
        got, info = device_reads.trim_fastq(data, sets, DEFAULT, min_split_read_size=100, fmt=fmt, as_array=True)
        if fmt == 'fastq':
            assert got.tobytes() == exp
            assert np.array_equal(info['start_trim'], exp_info['start_trim']) and info['n_reads'] == 20000
        else:
            assert got.tobytes() == fastq.emit(fastq.parse_fastq(data), exp_info['start_trim'], exp_info['end_trim'],
                                               exp_info['middle'], 'fasta', 100)


def test_gpu_demux_fastq_48_barcodes_equals_host():
    from porechop_b200 import device_reads, fastq
    from test_gpu_demux_reads import _shape
    batch, sets = _shape(48, n=24000)
    data = fastq.emit(batch, fmt='fastq')
    kw = dict(forward_or_reverse='forward', barcode_threshold=75.0, barcode_diff=5.0, require_two_barcodes=False,
              discard_unassigned=False, min_split_read_size=200)
    exp, exp_info = fastq.demux_fastq(data, sets, DEFAULT, **kw)
    got, info = device_reads.demux_fastq(data, sets, DEFAULT, **kw)
    assert len(got) >= 4 and got == exp and info['calls'] == exp_info['calls']


def test_gpu_parse_input_written_on_a_side_stream_right_before_the_call():
    import torch
    from porechop_b200 import device_reads
    data, _ = _config4_bytes(12000, seed=3)
    src = _cuda_bytes(data)
    exp = device_reads.parse_reads(src, 'fastq')
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dst.copy_(src)                                    # queued on s, still running when the call is issued
        got = device_reads.parse_reads(dst, 'fastq')
    s.synchronize()
    for a, b in zip(got[:6], exp[:6]):
        assert torch.equal(a.cpu(), b.cpu())


def test_gpu_parse_err_space_retry(monkeypatch):
    from porechop_b200 import cpp_function_wrappers as W, device_reads
    data, _ = _config4_bytes(6000, seed=4)
    caps = []
    orig = W.pb200_parse_reads_device
    monkeypatch.setattr(W, 'pb200_parse_reads_device',
                        lambda *a, **k: caps.append((k['reads_cap'], k['names_cap'], k['seq_cap'])) or orig(*a, **k))
    monkeypatch.setattr(device_reads, 'initial_parse_caps', lambda n, kind: (5, 7, 11))
    b = _check(data, 'fastq')
    assert caps == [(5, 7, 11), (len(b), len(b.name_buf), len(b.seq))]
