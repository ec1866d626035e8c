"""CPU tier (needs the Porechop checkout, helpers.REFERENCE): `python -m porechop_b200.flat_cli` with PB200_DEVICE_READS=1 and
PB200_DEVICE_GZIP=1 -- a chunk with matching adapter sets comes home as gzip members written by pb200GzipDevice and is written
as it is -- against the UNMODIFIED reference CLI (the files decompress to its bytes).  The device calls run on the simulated
engine (tests/sim), as in tests/test_flat_cli_device_reads.py, whose fixture pattern this reuses."""
import os
import sys

import pytest

from helpers import ROOT
import test_flat_cli as flat
from test_patch_cli import porechop_modules, pytestmark  # noqa: F401

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

from test_trim_split_reads import SimDevice  # noqa: E402

GZ_CASES = [c for c in flat.CASES if any('.gz' in a for a in c[2]) or (c[1].endswith('.gz') and '-b' in c[2])]


@pytest.fixture
def device_gzip(monkeypatch):
    """both switches on, device_reads on the simulated engine; counts the device path's chunks, the pb200GzipDevice calls, the
    host emits of chunks with nothing to align, and the host's gzip_members calls"""
    import sim_engine
    from porechop_b200 import device_reads, fastq, hostio
    SW = sim_engine.load()
    sim_engine.clear_races()
    D = SimDevice(SW)
    monkeypatch.setattr(device_reads, 'W', SW)
    monkeypatch.setattr(device_reads, '_device', D)
    monkeypatch.setenv('PB200_DEVICE_READS', '1')
    monkeypatch.setenv('PB200_DEVICE_GZIP', '1')
    n = dict(device=0, gzip_device=0, emit=0, host=0, gzip_members=0)

    def counted(fn, key):
        def call(*a, **k):
            n[key] += 1
            return fn(*a, **k)
        return call
    for mod, name, key in ((device_reads, 'trim_fastq', 'device'), (device_reads, 'demux_fastq', 'device'),
                           (SW, 'pb200_gzip_device', 'gzip_device'), (fastq, 'emit', 'emit'),
                           (fastq, 'trim_fastq', 'host'), (fastq, 'demux_fastq', 'host'), (hostio, 'gzip_members', 'gzip_members')):
        monkeypatch.setattr(mod, name, counted(getattr(mod, name), key))
    yield n
    D.free()
    sim_engine.assert_no_races()


def _check_counts(n):
    assert n['host'] == 0                                         # no chunk fell back to the host trim / demux
    assert n['gzip_device'] == n['device']                        # every device chunk was compressed by pb200GzipDevice
    assert n['gzip_members'] <= n['emit']                         # the host compressed only chunks with nothing to align


@pytest.mark.parametrize('name,input_name,argv', GZ_CASES, ids=[c[0] for c in GZ_CASES])
def test_flat_cli_device_gzip_writes_the_reference_cli_files(name, input_name, argv, porechop_modules, monkeypatch, tmp_path,  # noqa: F811
                                                             device_gzip):
    flat.test_flat_cli_writes_the_reference_cli_files(name, input_name, argv, porechop_modules, monkeypatch, tmp_path)
    _check_counts(device_gzip)


@pytest.mark.parametrize('input_name,argv', [('GOLDEN:input_fastq', ['-o', '{out}/o.fastq.gz', '--check_reads', '4',
                                                                     '--min_split_read_size', '50']),
                                             ('test_format_barcodes.fastq.gz', ['-b', '{out}/bins'])])
def test_flat_cli_device_gzip_tiny_chunks(input_name, argv, porechop_modules, monkeypatch, tmp_path, device_gzip):  # noqa: F811
    """tiny chunks: many device-compressed pieces appended to each file"""
    monkeypatch.setenv('PB200_FLAT_CHUNK_BYTES', '3000')
    flat.test_flat_cli_writes_the_reference_cli_files('chunked', input_name, argv, porechop_modules, monkeypatch, tmp_path)
    _check_counts(device_gzip)
    assert device_gzip['gzip_device'] > 1
