#!/usr/bin/env python3
"""Golden vectors for the flat FASTQ pipeline (porechop_b200/fastq.py::trim_fastq): whole-CLI outputs of the
UNMODIFIED reference (porechop.main() imported from tests/helpers.py REFERENCE, running on oracle/_ref/cpp_functions.so) on a
small synthetic FASTQ of this repo's own making.  Authoring container only; writes tests/golden/golden_emit.json.

The input is built to hit the corners of the reference's load / trim / split / write code: lower-case bases, an RNA
read (U > T), names with and without spaces, trailing blanks and CRLF line ends, an empty read, reads shorter than
end_size (incl. one whose end trim exceeds its length: Python's negative-slice behaviour, nanopore_read.py:57-63),
qualities shorter than the bases, chimeras with one and two middle adapters, reads with no adapter at all.
"""
import contextlib
import ctypes
import io
import json
import os
import random
import sys
import tempfile
import types
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import REFERENCE as REF  # noqa: E402  (a Porechop v0.2.4 checkout)
warnings.simplefilter('ignore')

lib = ctypes.CDLL(os.path.join(ROOT, 'oracle', '_ref', 'cpp_functions.so'))
lib.adapterAlignment.argtypes = [ctypes.c_char_p, ctypes.c_char_p] + [ctypes.c_int] * 4
lib.adapterAlignment.restype = ctypes.c_void_p
lib.freeCString.argtypes = [ctypes.c_void_p]


def adapter_alignment(read_sequence, adapter_sequence, scoring_scheme_vals):
    p = lib.adapterAlignment(read_sequence.encode(), adapter_sequence.encode(), *scoring_scheme_vals)
    s = ctypes.cast(p, ctypes.c_char_p).value.decode()
    lib.freeCString(p)
    return s


sys.path.insert(0, REF)
stub = types.ModuleType('porechop.cpp_function_wrappers')
stub.adapter_alignment = adapter_alignment
import porechop  # noqa: E402,F401
sys.modules['porechop.cpp_function_wrappers'] = stub
from porechop import adapters as A  # noqa: E402
from porechop import porechop as P  # noqa: E402

Y_TOP = 'AATGTACTTCGTTCAGTTACGTATTGCT'       # SQK-NSK007 start / end sequences (public kit sequences)
Y_BOTTOM = 'GCAATACGTAACTGAACGAAGT'


def mutate(rng, s, p=0.08):
    out = []
    for c in s:
        r = rng.random()
        if r < p * 0.3:
            continue
        if r < p * 0.7:
            out.append(rng.choice('ACGT'))
            continue
        out.append(c)
        if r > 1 - p * 0.3:
            out.append(rng.choice('ACGT'))
    return ''.join(out)


def make_fastq(seed=20260923):
    rng = random.Random(seed)
    recs = []

    def rand(n):
        return ''.join(rng.choice('ACGT') for _ in range(n))

    def add(name, seq, nl='\n', qual=None, pad=''):
        q = qual if qual is not None else ''.join(chr(rng.randint(35, 73)) for _ in range(len(seq)))
        recs.append('@' + name + pad + nl + seq + pad + nl + '+' + nl + q + nl)

    for k in range(6):                                            # plain reads with (mutated) end adapters
        body = rand(rng.randint(300, 1400))
        s = (Y_TOP if k < 2 else mutate(rng, Y_TOP)) + body + (Y_BOTTOM if k < 2 else mutate(rng, Y_BOTTOM))
        add('plain_%d runid=abc ch=%d' % (k, k), s)
    add('lower_case_bases', (mutate(rng, Y_TOP) + rand(500)).lower())
    add('no_adapters_at_all', rand(800))
    rna = (Y_TOP + rand(400)).replace('T', 'U')
    add('rna read', rna)
    add('mostly_t_some_u', rand(300).replace('G', 'U', 3))
    add('crlf_read extra', mutate(rng, Y_TOP) + rand(350), nl='\r\n')
    add('trailing_blanks', rand(200) + mutate(rng, Y_BOTTOM), pad='  ')
    add('empty_read', '')
    add('short_40', rand(12) + Y_BOTTOM + rand(6))
    add('short_just_adapter', Y_TOP[5:])
    add('short_end_trim_exceeds_length', rand(8) + Y_BOTTOM + rand(70))
    add('short_quals', Y_TOP + rand(260), qual='#' * 100)
    add('chimera_one small', rand(700) + mutate(rng, Y_BOTTOM, 0.04) + mutate(rng, Y_TOP, 0.04) + rand(900))
    add('chimera_two', Y_TOP + rand(1300) + Y_BOTTOM + Y_TOP + rand(1100) + Y_TOP + rand(1250) + Y_BOTTOM)
    add('chimera_near_start', rand(60) + Y_TOP + rand(1500))
    add('chimera_same_adapter_twice', rand(1200) + Y_TOP + rand(1100) + Y_TOP + rand(1300))
    add('chimera_long_parts', mutate(rng, Y_TOP) + rand(2100) + Y_BOTTOM + mutate(rng, Y_TOP, 0.03) + rand(1900))
    for k in range(4):
        add('tail_%d' % k, rand(rng.randint(150, 600)) + (mutate(rng, Y_BOTTOM) if k % 2 else ''))
    return ''.join(recs)


def make_barcoded_fastq(seed=20260924):
    """native-barcoding style reads (NBxx_start ... NBxx_end, sequences from tests/golden/adapters.json): clean and
    noisy pairs, start-only / end-only, mismatched start/end barcodes, a near-tie between two barcodes, a chimera."""
    rng = random.Random(seed)
    full = {d['name']: d for d in json.load(open(os.path.join(HERE, 'adapters.json')))['full_barcode_sets']}
    nb = {k: full['Native barcoding %d (full sequence)' % k] for k in (1, 2, 3, 4, 5)}
    recs = []

    def rand(n):
        return ''.join(rng.choice('ACGT') for _ in range(n))

    def add(name, seq):
        q = ''.join(chr(rng.randint(35, 73)) for _ in range(len(seq)))
        recs.append('@' + name + '\n' + seq + '\n+\n' + q + '\n')

    for k in (1, 2, 3):
        for j in range(3):
            p = 0.0 if j == 0 else 0.06 * j
            add('bc%d_pair_%d' % (k, j), mutate(rng, nb[k]['start'][1], p) + rand(rng.randint(400, 1500)) +
                mutate(rng, nb[k]['end'][1], p))
    add('bc4_start_only', nb[4]['start'][1] + rand(700))
    add('bc4_end_only lonely', rand(650) + nb[4]['end'][1])
    add('mismatch_1_start_2_end', nb[1]['start'][1] + rand(900) + nb[2]['end'][1])
    add('mismatch_noisy', mutate(rng, nb[3]['start'][1], 0.1) + rand(500) + mutate(rng, nb[1]['end'][1], 0.1))
    half = nb[2]['start'][1][:44] + nb[3]['start'][1][44:]
    add('near_tie', half + rand(800))
    add('no_barcode', rand(1000))
    add('very_noisy', mutate(rng, nb[2]['start'][1], 0.25) + rand(600) + mutate(rng, nb[2]['end'][1], 0.25))
    add('chimera_bc', nb[1]['start'][1] + rand(1200) + nb[1]['end'][1] + nb[1]['start'][1] + rand(1300) + nb[1]['end'][1])
    add('short_bc', nb[5]['start'][1][10:] + rand(30))
    return ''.join(recs)


BARCODE_CASES = [
    ('bins_default', 'fastq', []),
    ('bins_two_barcodes', 'fastq', ['--require_two_barcodes', '--min_split_read_size', '100']),
    ('bins_loose_discard', 'fastq', ['--discard_unassigned', '--barcode_diff', '1', '--barcode_threshold', '60',
                                      '--discard_middle']),
    ('bins_fasta_untrimmed', 'fasta', ['--untrimmed', '--format', 'fasta']),
]


def run_barcode_case(fastq_path, fmt, extra):
    for a in A.ADAPTERS:
        a.best_start_score, a.best_end_score = 0.0, 0.0
    captured = {}
    orig = P.find_adapters_at_read_ends

    def spy(reads, matching_sets, *args, **kwargs):
        captured['sets'] = [[s.name, list(s.start_sequence) if s.start_sequence else None,
                             list(s.end_sequence) if s.end_sequence else None] for s in matching_sets]
        captured['direction'] = args[-1]
        return orig(reads, matching_sets, *args, **kwargs)
    P.find_adapters_at_read_ends = spy
    with tempfile.TemporaryDirectory() as d:
        old = sys.argv
        sys.argv = ['porechop', '-i', fastq_path, '-b', os.path.join(d, 'bins'), '-v', '0', '-t', '1'] + extra
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                P.main()
            args = P.get_arguments()
        finally:
            sys.argv = old
            P.find_adapters_at_read_ends = orig
        bins = {f: open(os.path.join(d, 'bins', f)).read() for f in sorted(os.listdir(os.path.join(d, 'bins')))}
    opts = {k: getattr(args, k) for k in ('end_size', 'extra_end_trim', 'end_threshold', 'min_trim_size', 'no_split',
                                          'middle_threshold', 'extra_middle_trim_good_side', 'extra_middle_trim_bad_side',
                                          'min_split_read_size', 'discard_middle', 'barcode_threshold', 'barcode_diff',
                                          'require_two_barcodes', 'discard_unassigned', 'untrimmed')}
    opts['fmt'] = fmt
    opts['forward_or_reverse'] = captured['direction']
    return {'matching_sets': captured['sets'], 'options': opts, 'scoring': list(args.scoring_scheme_vals), 'bins': bins}


CASES = [
    ('default', 'o.fastq', []),
    ('small_parts', 'o.fastq', ['--min_split_read_size', '50', '--extra_end_trim', '5', '--middle_threshold', '80']),
    ('discard_middle', 'o.fastq', ['--discard_middle', '--end_threshold', '70', '--min_trim_size', '6']),
    ('no_split_fasta', 'o.fasta', ['--no_split', '--end_size', '100']),
    ('fasta_split', 'o.fasta', ['--min_split_read_size', '200', '--extra_middle_trim_good_side', '3',
                                '--extra_middle_trim_bad_side', '40']),
]


def run_case(fastq_path, out_name, extra):
    for a in A.ADAPTERS:
        a.best_start_score, a.best_end_score = 0.0, 0.0
    captured = {}
    orig = P.find_adapters_at_read_ends

    def spy(reads, matching_sets, *args, **kwargs):
        captured['sets'] = [[list(s.start_sequence) if s.start_sequence else None,
                             list(s.end_sequence) if s.end_sequence else None] for s in matching_sets]
        return orig(reads, matching_sets, *args, **kwargs)
    P.find_adapters_at_read_ends = spy
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, out_name)
        old = sys.argv
        sys.argv = ['porechop', '-i', fastq_path, '-o', out, '-v', '0', '-t', '1'] + extra
        try:
            with contextlib.redirect_stdout(io.StringIO()):
                P.main()
            args = P.get_arguments()
        finally:
            sys.argv = old
            P.find_adapters_at_read_ends = orig
        text = open(out).read()
    opts = {k: getattr(args, k) for k in ('end_size', 'extra_end_trim', 'end_threshold', 'min_trim_size', 'no_split',
                                          'middle_threshold', 'extra_middle_trim_good_side', 'extra_middle_trim_bad_side',
                                          'min_split_read_size', 'discard_middle')}
    opts['fmt'] = 'fasta' if out_name.endswith('.fasta') else 'fastq'
    return {'matching_sets': captured['sets'], 'options': opts, 'scoring': list(args.scoring_scheme_vals), 'output': text}


def main():
    fq = make_fastq()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, 'in.fastq')
        with open(p, 'w', newline='') as f:
            f.write(fq)
        cases = {name: run_case(p, out_name, extra) for name, out_name, extra in CASES}
    bq = make_barcoded_fastq()
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, 'in.fastq')
        with open(p, 'w', newline='') as f:
            f.write(bq)
        bcases = {name: run_barcode_case(p, fmt, extra) for name, fmt, extra in BARCODE_CASES}
    json.dump({'input_fastq': fq, 'cases': cases, 'barcoded_fastq': bq, 'barcode_cases': bcases},
              open(os.path.join(HERE, 'golden_emit.json'), 'w'), indent=0)
    for k, c in bcases.items():
        print(k, c['options']['forward_or_reverse'], len(c['matching_sets']), {f: len(t) for f, t in c['bins'].items()})
    for k, c in cases.items():
        print(k, len(c['output']), [s[0][0] if s[0] else s[1][0] for s in c['matching_sets']])


if __name__ == '__main__':
    main()
