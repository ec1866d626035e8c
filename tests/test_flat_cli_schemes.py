"""CPU tier: `--scoring_scheme` end to end.  Five non-default schemes x three inputs (scheme_edges.cli_inputs: noisy end
adapters and chimeras as FASTQ and as FASTA, barcoded reads into bins), recorded in tests/golden/golden_schemes.json by
tests/golden/make_golden_schemes.py:
  - the flat CLI against the UNMODIFIED reference CLI, with the oracle as the engine and with PB200_DEVICE_READS=1 on the
    simulated engine (needs the Porechop checkout, as tests/test_flat_cli.py);
  - the flat pipeline (fastq.trim_fastq / demux_fastq) on the oracle engine against the recorded reference output, which
    tests/test_gpu_schemes_cli.py runs on the real engine."""
import hashlib

import pytest

import test_flat_cli as flat
from helpers import load_golden
from scheme_edges import cli_inputs
from test_fastq_emit import _oracle_engine as _oracle_batch_engine
from test_flat_cli_device_reads import _check_counts, device_path  # noqa: F401
from test_patch_cli import REF, _oracle_engine, _run_cli, porechop_modules  # noqa: F401
from test_patch_cli import pytestmark as needs_reference

G = load_golden('golden_schemes.json')
INPUTS = cli_inputs()
ARGV = {'trim_fastq': ['-o', '{out}/o.fastq', '--min_split_read_size', '50'], 'barcoded_fastq': ['-b', '{out}/bins'],
        'trim_fasta': ['-o', '{out}/o.fasta', '--min_split_read_size', '100']}
CLI_CASES = [(name, scheme) for name in ARGV for scheme in G['schemes']]


def digests(files):
    """{file name as the reference writes it: SHA-256} -- the form golden_schemes.json records"""
    return {k.split('/')[-1]: hashlib.sha256(v).hexdigest() for k, v in files.items()}


def _cli_case(name, scheme, porechop_modules, monkeypatch, tmp_path):  # noqa: F811
    porechop, P, A = porechop_modules
    inp = str(tmp_path / ('in.' + name.split('_')[1]))
    with open(inp, 'w', newline='') as f:
        f.write(INPUTS[name])

    def args_for(out):
        return ['-i', inp, '-v', '0', '-t', '1', '--scoring_scheme', scheme] + [a.replace('{out}', out) for a in ARGV[name]]
    _, base = _run_cli(P, A, args_for(str(tmp_path / 'a')), str(tmp_path / 'a'))
    _oracle_engine(monkeypatch)
    monkeypatch.syspath_prepend(REF)
    got = flat._flat_cli(A, args_for(str(tmp_path / 'b')), str(tmp_path / 'b'))
    assert sorted(got) == sorted(base) and len(base) >= 1, (sorted(got), sorted(base))
    for k in base:
        assert got[k] == base[k], k
    want = G['cases']['%s %s' % (name, scheme)]['sha256']
    assert digests(base) == (want if isinstance(want, dict) else {'o.' + name.split('_')[1]: want}), \
        'golden_schemes.json is stale: rerun tests/golden/make_golden_schemes.py'


@needs_reference
@pytest.mark.parametrize('name,scheme', CLI_CASES, ids=['%s-%s' % c for c in CLI_CASES])
def test_flat_cli_scoring_scheme_writes_the_reference_cli_files(name, scheme, porechop_modules, monkeypatch, tmp_path):  # noqa: F811
    _cli_case(name, scheme, porechop_modules, monkeypatch, tmp_path)


@needs_reference
@pytest.mark.parametrize('name,scheme', CLI_CASES, ids=['%s-%s' % c for c in CLI_CASES])
def test_flat_cli_device_reads_scoring_scheme_writes_the_reference_cli_files(name, scheme, porechop_modules, monkeypatch,  # noqa: F811
                                                                             tmp_path, device_path):  # noqa: F811
    _cli_case(name, scheme, porechop_modules, monkeypatch, tmp_path)
    _check_counts(device_path)
    assert device_path['device'] >= 1


def run_golden_case(key, trim_fastq, demux_fastq, host_batch):
    """one case of golden_schemes.json through the given trim / demux functions (fastq.* with host_batch: the parsed reads,
    or device_reads.*: the input bytes); the output must have the recorded digests"""
    from porechop_b200 import fastq
    c = G['cases'][key]
    data = INPUTS[c['input']].encode()
    if host_batch:
        data = fastq.parse_reads(data)[0]
    if c['mode'] == 'trim':
        sets = [(tuple(s) if s else None, tuple(e) if e else None) for s, e in c['matching_sets']]
        out, _ = trim_fastq(data, sets, c['scoring'], **c['options'])
        assert hashlib.sha256(out).hexdigest() == c['sha256'], key
    else:
        bins, _ = demux_fastq(data, c['matching_sets'], c['scoring'], **c['options'])
        assert digests({k + '.' + c['options']['fmt']: v for k, v in bins.items()}) == c['sha256'], key


@pytest.mark.parametrize('key', sorted(G['cases']))
def test_golden_schemes_flat_pipeline_oracle_engine(key, monkeypatch):
    from porechop_b200 import fastq
    _oracle_batch_engine(monkeypatch)
    run_golden_case(key, fastq.trim_fastq, fastq.demux_fastq, host_batch=True)


def test_golden_schemes_differ_by_scheme():
    """every scheme changes what the reference writes for every input: the cases tell the schemes apart"""
    for name in ARGV:
        outs = [str(G['cases']['%s %s' % (name, s)]['sha256']) for s in G['schemes']]
        assert len(set(outs)) == len(outs), name
