"""gzip members written on the device (include/porechop_b200.h pb200GzipDevice, device_reads.gzip_bytes and the gz=True
chunks of device_reads.trim_fastq / demux_fastq).  CPU tier: the product's engine code on the host simulator (tests/sim),
through the product's own ctypes wrapper, checked with Python's gzip / zlib.  The GPU tier is tests/test_gpu_gzip.py."""
import gzip
import os
import sys

import numpy as np
import pytest

from gzip_inputs import BLOCK, HEADER, check_file, edge_inputs, members, ont_fastq, segments_of, zlib_level_bytes
from helpers import ROOT, load_golden

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

from test_trim_split_reads import SimDevice  # noqa: E402

SENTINEL = 0xA5


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


@pytest.fixture
def sim(SW, monkeypatch):
    """device_reads, and the host path it falls back to, on the simulated engine"""
    from porechop_b200 import device_reads, fastq
    D = SimDevice(SW)
    monkeypatch.setattr(device_reads, 'W', SW)
    monkeypatch.setattr(fastq, 'W', SW)
    monkeypatch.setattr(device_reads, '_device', D)
    yield D
    D.free()


def _gzip(W, D, data, seg_off=None, block=BLOCK, cap=None, stream=0):
    """pb200GzipDevice through the wrapper: (compressed bytes, segment offsets)"""
    d = D.upload(np.frombuffer(data, dtype=np.uint8))
    n_segs = 1 if seg_off is None else len(seg_off) - 1
    cap = W.gzip_bound(len(data), n_segs, block) if cap is None else cap
    out = D.empty(max(cap, 1), np.uint8)
    total, off = W.pb200_gzip_device(D.ptr(d), len(data), seg_off, block=block, d_out_ptr=D.ptr(out), out_cap=cap,
                                     stream_ptr=stream)
    return D.host(D.head(out, total)).tobytes(), off


def _emit_outputs():
    """the golden emit outputs: every trim case's file and every barcode case's bins, as {name: bytes}"""
    g = load_golden('golden_emit.json')
    out = {'trim_' + k: c['output'].encode() for k, c in g['cases'].items()}
    for k, c in g['barcode_cases'].items():
        out.update({'bins_%s_%s' % (k, b): v.encode() for b, v in sorted(c['bins'].items())})
    return out


# ---- round trips --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(edge_inputs()))
def test_sim_gzip_edges(SW, sim, name):
    data = edge_inputs()[name]
    gz, off = _gzip(SW, sim, data)
    assert list(off) == [0, len(gz)] and gzip.decompress(gz) == data
    check_file(gz, data, BLOCK)


def test_sim_gzip_default_block_and_stored_bound(SW, sim):
    """block 0 is 65536; random bytes are stored, and then the output is exactly the bound"""
    rng = np.random.default_rng(11)
    data = rng.integers(0, 256, 2 * 65536, dtype=np.uint8).tobytes()
    gz, _ = _gzip(SW, sim, data, block=0)
    check_file(gz, data, 65536)
    assert len(gz) == SW.gzip_bound(len(data), 1, 0) == SW.gzip_bound(len(data), 1, 65536)
    gz, _ = _gzip(SW, sim, data[:4 * BLOCK])
    assert len(gz) == SW.gzip_bound(4 * BLOCK, 1, BLOCK)
    for m, _ in members(gz):                               # two stored blocks are needed from 65536 bytes on, not here
        assert m[10] == 1                                  # one final stored block per member


@pytest.mark.parametrize('block', [BLOCK, 3 * BLOCK + 5, 65536, 131072])
def test_sim_gzip_block_sizes(SW, sim, block):
    data = ont_fastq(3 * block // 2, 1)
    gz, _ = _gzip(SW, sim, data, block=block)
    check_file(gz, data, block)


def test_sim_gzip_golden_emit_outputs(SW, sim):
    """the golden emit outputs as one file, and as segments (one per output, as the bins of a demux)"""
    outs = _emit_outputs()
    data = b''.join(outs.values())
    gz, _ = _gzip(SW, sim, data)
    check_file(gz, data, BLOCK)
    seg = segments_of([len(v) for v in outs.values()])
    gz, off = _gzip(SW, sim, data, seg)
    for k, v in enumerate(outs.values()):
        check_file(gz[off[k]:off[k + 1]], v, BLOCK)


def test_sim_gzip_many_segments(SW, sim):
    """empty segments, segments shorter than a block, exactly one block and longer; each slice is a file of its own"""
    rng = np.random.default_rng(3)
    lengths = [0, 0, 1, 5, 0, BLOCK, BLOCK - 1, BLOCK + 1, 3, 0, 2 * BLOCK + 7, 100, 0]
    lengths += rng.integers(0, 3 * BLOCK, 20).tolist()
    data = ont_fastq(sum(lengths), 9)[:sum(lengths)]
    seg = segments_of(lengths)
    gz, off = _gzip(SW, sim, data, seg)
    assert off[0] == 0 and off[-1] == len(gz) and all(np.diff(off) >= 0)
    for k in range(len(lengths)):
        piece, plain = gz[off[k]:off[k + 1]], data[seg[k]:seg[k + 1]]
        if not plain:
            assert piece == b''
            continue
        assert piece[:10] == HEADER
        check_file(piece, plain, BLOCK)
    assert gzip.decompress(gz) == data                     # the members of all segments make one valid file too


# ---- size ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('which', ['golden_emit', 'ont_model'])
def test_sim_gzip_size_target(SW, sim, which):
    """at most 1.10 x the bytes of zlib level 1 on the same 64 KiB members (deterministic: the device writes the same bytes).
    Ratios on the ONT model (uncompressed / compressed): this encoder 2.37, zlib level 1 2.52, level 6 2.83."""
    data = b''.join(_emit_outputs().values()) if which == 'golden_emit' else ont_fastq(3_000_000, 5)
    gz, _ = _gzip(SW, sim, data, block=65536)
    assert gzip.decompress(gz) == data
    level1 = zlib_level_bytes(data, 65536, 1)
    assert len(gz) <= 1.10 * level1, (len(gz), level1, zlib_level_bytes(data, 65536, 6))


# ---- determinism and stream order -----------------------------------------------------------------------------------------
_ORDER_SCRIPT = r"""
import hashlib, sys
import numpy as np
sys.path[:0] = [%r, %r, %r]
import sim_engine
from gzip_inputs import BLOCK, ont_fastq
from test_trim_split_reads import SimDevice
W = sim_engine.load()
D = SimDevice(W)
data = ont_fastq(6 * BLOCK, 2)[:6 * BLOCK + 99]
seg = [0, 1000, 1000, 5 * BLOCK, len(data)]
outs = []
for _ in range(2):
    d = D.upload(np.frombuffer(data, dtype=np.uint8))
    cap = W.gzip_bound(len(data), len(seg) - 1, BLOCK)
    out = D.empty(cap, np.uint8)
    total, off = W.pb200_gzip_device(D.ptr(d), len(data), seg, block=BLOCK, d_out_ptr=D.ptr(out), out_cap=cap)
    outs.append(hashlib.sha256(D.host(D.head(out, total)).tobytes() + off.tobytes()).hexdigest())
print(outs[0] if outs[0] == outs[1] else 'differs')
"""


def test_sim_gzip_deterministic():
    """the same bytes on every call, whatever order the simulator resumes the threads in (separate processes: the order is
    read once)"""
    import subprocess
    script = _ORDER_SCRIPT % (ROOT, os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'tests', 'sim'))
    outs = []
    for order in ('', 'reverse', 'random:3', 'random:11'):
        env = dict(os.environ)
        env.pop('PBSIM_ORDER', None)
        if order:
            env['PBSIM_ORDER'] = order
        r = subprocess.run([sys.executable, '-c', script], env=env, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(r.stdout.strip().splitlines()[-1])
    assert outs[0] != 'differs' and len(set(outs)) == 1, outs


def test_sim_gzip_input_written_on_another_stream(SW, sim):
    """input written on a caller's stream right before a call on that stream: ordered, no race"""
    data = ont_fastq(3 * BLOCK, 4)
    s = SW.stream_create()
    d = sim.empty(len(data), np.uint8)
    host = np.frombuffer(data, dtype=np.uint8).copy()
    SW.upload(d.ptr, host.ctypes.data, len(data), s)
    cap = SW.gzip_bound(len(data), 1, BLOCK)
    out = sim.empty(cap, np.uint8)
    total, _ = SW.pb200_gzip_device(d.ptr, len(data), None, block=BLOCK, d_out_ptr=out.ptr, out_cap=cap, stream_ptr=s)
    assert gzip.decompress(sim.host(sim.head(out, total)).tobytes()) == data


# ---- errors ------------------------------------------------------------------------------------------------------------
def test_sim_gzip_preconditions(SW, sim):
    """each precondition fails with PB200_ERR_ARG before anything is launched"""
    data = b'ACGT' * 100
    d = sim.upload(np.frombuffer(data, dtype=np.uint8))
    out = sim.empty(10000, np.uint8)
    ok = dict(block=BLOCK, d_out_ptr=out.ptr, out_cap=10000)
    bad = [((d.ptr, 400, [0, 500]), ok), ((d.ptr, 400, [1, 400]), ok), ((d.ptr, 400, [0, 300, 200, 400]), ok),
           ((d.ptr, 400, [0]), ok), ((d.ptr, -1, [0, -1]), ok), ((0, 400, None), ok),
           ((d.ptr, 400, None), dict(ok, block=4095)), ((d.ptr, 400, None), dict(ok, block=131073)),
           ((d.ptr, 400, None), dict(ok, block=-1)), ((d.ptr, 400, None), dict(ok, out_cap=-1)),
           ((d.ptr, 400, None), dict(ok, d_out_ptr=0))]
    for args, kw in bad:
        before = SW.kernel_launches()
        with pytest.raises(SW.EngineError) as e:
            SW.pb200_gzip_device(*args, **kw)
        assert e.value.code == SW.ERR_ARG, (args, kw)
        assert SW.kernel_launches() == before
    for n, segs, block in ((-1, 1, 0), (5, 0, 0), (5, 1, 100), (5, 1, 200000)):
        with pytest.raises(ValueError):
            SW.gzip_bound(n, segs, block)


def test_sim_gzip_space(SW, sim):
    """out_cap one byte short: PB200_ERR_SPACE with the exact total and offsets, and d_out untouched"""
    data = ont_fastq(3 * BLOCK, 6)
    seg = [0, BLOCK, len(data)]
    gz, off = _gzip(SW, sim, data, seg)
    d = sim.upload(np.frombuffer(data, dtype=np.uint8))
    out = sim.upload(np.full(len(gz), SENTINEL, dtype=np.uint8))
    with pytest.raises(SW.EngineError) as e:
        SW.pb200_gzip_device(d.ptr, len(data), seg, block=BLOCK, d_out_ptr=out.ptr, out_cap=len(gz) - 1)
    assert e.value.code == SW.ERR_SPACE and e.value.n_out_bytes == len(gz) and list(e.value.out_seg_off) == list(off)
    assert (sim.host(out) == SENTINEL).all()
    total, _ = SW.pb200_gzip_device(d.ptr, len(data), seg, block=BLOCK, d_out_ptr=out.ptr, out_cap=len(gz))
    assert total == len(gz) and sim.host(out).tobytes() == gz


# ---- device_reads ------------------------------------------------------------------------------------------------------
def test_sim_gzip_bytes_ranges(sim):
    from porechop_b200 import device_reads
    outs = _emit_outputs()
    data = b''.join(outs.values())
    d = sim.upload(np.frombuffer(data, dtype=np.uint8))
    g = device_reads.gzip_bytes(d)
    assert g.ranges is None and gzip.decompress(sim.host(g.data).tobytes()) == data
    at, ranges = 0, {}
    for k, v in outs.items():
        ranges[k] = (at, at + len(v))
        at += len(v)
    ranges.pop(next(iter(ranges)))                          # bytes outside every range are compressed but named by nothing
    g = device_reads.gzip_bytes(d, ranges, block=BLOCK)
    host = sim.host(g.data).tobytes()
    assert set(g.ranges) == set(ranges)
    for k, (b0, b1) in g.ranges.items():
        check_file(host[b0:b1], outs[k], BLOCK)
    with pytest.raises(ValueError):
        device_reads.gzip_bytes(d, {'a': (0, 10), 'b': (5, 20)})


@pytest.mark.parametrize('case_name', ['default', 'small_parts', 'no_split_fasta'])
def test_sim_trim_fastq_gz(sim, monkeypatch, case_name):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['cases'][case_name]
    o = dict(c['options'])
    sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
    data = g['input_fastq'].encode()
    calls = []
    raw = device_reads.W.pb200_gzip_device
    monkeypatch.setattr(device_reads.W, 'pb200_gzip_device', lambda *a, **k: calls.append(1) or raw(*a, **k))
    got, info = device_reads.trim_fastq(data, sets, c['scoring'], gz=True, **o)
    assert gzip.decompress(got).decode() == c['output'] and calls == [1]
    arr, _ = device_reads.trim_fastq(data, sets, c['scoring'], gz=True, as_array=True, **o)
    assert arr.tobytes() == got
    # a chunk the host path takes (no adapter sets) comes back compressed the same way
    exp, _ = fastq.trim_fastq(data, [], c['scoring'], **o)
    got, _ = device_reads.trim_fastq(data, [], c['scoring'], gz=True, **o)
    assert gzip.decompress(got) == exp and got[:10] == HEADER and len(calls) == 3


@pytest.mark.parametrize('case_name', ['bins_default', 'bins_loose_discard', 'bins_fasta_untrimmed'])
def test_sim_demux_fastq_gz(sim, monkeypatch, case_name):
    from porechop_b200 import device_reads, fastq
    g = load_golden('golden_emit.json')
    c = g['barcode_cases'][case_name]
    o = dict(c['options'])
    data = g['barcoded_fastq'].encode()
    exp, exp_info = fastq.demux_fastq(data, c['matching_sets'], c['scoring'], **o)
    bins, info = device_reads.demux_fastq(data, c['matching_sets'], c['scoring'], gz=True, **o)
    assert sorted(bins) == sorted(exp) and info['calls'] == exp_info['calls']
    for k, v in bins.items():
        assert gzip.decompress(v) == exp[k], k
        assert v[:10] == HEADER
    # the host path (no adapter sets) too
    exp, _ = fastq.demux_fastq(data, [], c['scoring'], **o)
    bins, _ = device_reads.demux_fastq(data, [], c['scoring'], gz=True, **o)
    assert {k: gzip.decompress(v) for k, v in bins.items()} == exp
