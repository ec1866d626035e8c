"""CPU tier (needs the Porechop checkout, helpers.REFERENCE): `python -m porechop_b200.flat_cli` with PB200_DEVICE_READS=1 --
every chunk with matching adapter sets goes from input bytes to output bytes through device_reads.trim_fastq / demux_fastq
(parse, trim / demux and emit on the device) -- against the UNMODIFIED reference CLI.  The device calls run on the simulated
engine (tests/sim), Phase A on the oracle, as in tests/test_flat_cli.py, whose cases and helpers this reuses."""
import os
import sys

import pytest

from helpers import ROOT
import test_flat_cli as flat
from test_patch_cli import porechop_modules, pytestmark  # noqa: F401

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

from test_trim_split_reads import SimDevice  # noqa: E402

SINGLE_FILE = [c for c in flat.CASES if not c[1].startswith('test_albacore')]
ALBACORE = [c for c in flat.CASES if c[1].startswith('test_albacore')]


@pytest.fixture
def device_path(monkeypatch):
    """PB200_DEVICE_READS=1 with device_reads on the simulated engine; counts the chunks the main pass processes, the device
    calls, the host emits of chunks with nothing to align, and host trims / demuxes (fallbacks)"""
    import sim_engine
    from porechop_b200 import device_reads, fastq, flat_cli
    SW = sim_engine.load()
    sim_engine.clear_races()
    D = SimDevice(SW)
    monkeypatch.setattr(device_reads, 'W', SW)
    monkeypatch.setattr(device_reads, '_device', D)
    monkeypatch.setenv('PB200_DEVICE_READS', '1')
    n = dict(chunks=0, device=0, emit=0, host=0)

    def counted(fn, key):
        def call(*a, **k):
            n[key] += 1
            return fn(*a, **k)
        return call
    for mod, name, key in ((device_reads, 'trim_fastq', 'device'), (device_reads, 'demux_fastq', 'device'),
                           (fastq, 'emit', 'emit'), (fastq, 'trim_fastq', 'host'), (fastq, 'demux_fastq', 'host')):
        monkeypatch.setattr(mod, name, counted(getattr(mod, name), key))
    prefetch = flat_cli._prefetch

    def counting_prefetch(it, depth=2):
        for item in prefetch(it, depth):
            n['chunks'] += 1
            yield item
    monkeypatch.setattr(flat_cli, '_prefetch', counting_prefetch)
    yield n
    D.free()
    sim_engine.assert_no_races()


def _check_counts(n):
    assert n['chunks'] >= 1 and n['host'] == 0                    # no chunk fell back to the host trim / demux
    assert n['device'] + n['emit'] == n['chunks']                 # every chunk with adapter sets went through the device path


@pytest.mark.parametrize('name,input_name,argv', SINGLE_FILE + ALBACORE, ids=[c[0] for c in SINGLE_FILE + ALBACORE])
def test_flat_cli_device_reads_writes_the_reference_cli_files(name, input_name, argv, porechop_modules, monkeypatch, tmp_path,  # noqa: F811
                                                              device_path):
    flat.test_flat_cli_writes_the_reference_cli_files(name, input_name, argv, porechop_modules, monkeypatch, tmp_path)
    _check_counts(device_path)


@pytest.mark.parametrize('chunk', [3000, 20000])
@pytest.mark.parametrize('input_name,argv', [('test_barcodes.fastq', ['-b', '{out}/bins', '--check_reads', '5']),
                                             ('test_format.fasta', ['-o', '{out}/o.fasta', '--check_reads', '7']),
                                             ('GOLDEN:input_fastq', ['-o', '{out}/o.fastq.gz', '--check_reads', '4',
                                                                     '--min_split_read_size', '50'])])
def test_flat_cli_device_reads_streams_in_chunks(chunk, input_name, argv, porechop_modules, monkeypatch, tmp_path,  # noqa: F811
                                                 device_path):
    """tiny chunks (many whole-record pieces, bins appended piece by piece): same files as the reference CLI"""
    monkeypatch.setenv('PB200_FLAT_CHUNK_BYTES', str(chunk))
    flat.test_flat_cli_writes_the_reference_cli_files('chunked', input_name, argv, porechop_modules, monkeypatch, tmp_path)
    _check_counts(device_path)
    assert device_path['device'] > 1
