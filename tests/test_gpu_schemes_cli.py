"""GPU tier (pytest -m gpu): `--scoring_scheme` end to end on the real engine -- the reference CLI's output recorded in
tests/golden/golden_schemes.json (five non-default schemes x noisy trim FASTQ, the same reads as FASTA, barcoded FASTQ into
bins) from
  - fastq.trim_fastq / demux_fastq with the engine's window and read batches, and again with the end-trim decisions and the
    middle scan in one adapterTrimReads call per chunk;
  - device_reads.trim_fastq / demux_fastq: parse -> trim / demux -> emit in GPU memory, with no host fallback."""
import pytest

from test_flat_cli_schemes import G, run_golden_case

pytestmark = pytest.mark.gpu
KEYS = sorted(G['cases'])


@pytest.mark.parametrize('fused', [False, True], ids=['batch_calls', 'trim_reads_call'])
@pytest.mark.parametrize('key', KEYS)
def test_flat_pipeline_real_engine(key, fused, monkeypatch):
    from porechop_b200 import fastq
    monkeypatch.setattr(fastq, 'DEVICE_DECISIONS', fused)
    monkeypatch.setattr(fastq, 'DEVICE_MIDDLE', fused)
    calls = []
    orig = fastq.W.adapter_trim_reads
    monkeypatch.setattr(fastq.W, 'adapter_trim_reads', lambda *a, **k: calls.append(1) or orig(*a, **k))
    run_golden_case(key, fastq.trim_fastq, fastq.demux_fastq, host_batch=True)
    assert (len(calls) > 0) == fused, key


@pytest.mark.parametrize('key', KEYS)
def test_device_reads_real_engine(key, monkeypatch):
    from porechop_b200 import device_reads, fastq
    monkeypatch.setattr(fastq, 'trim_fastq', None)       # the device path only: a fallback to the host would fail
    monkeypatch.setattr(fastq, 'demux_fastq', None)
    run_golden_case(key, device_reads.trim_fastq, device_reads.demux_fastq, host_batch=False)
