#!/usr/bin/env python3
"""Golden vectors for the batched phase drivers (porechop_b200/phases.py), produced by the UNMODIFIED reference
Python (porechop/porechop.py + nanopore_read.py + adapters.py imported from tests/helpers.py REFERENCE) running on the
UNMODIFIED reference C++ (oracle/_ref/cpp_functions.so).  Authoring container only; writes
tests/golden/golden_phases.json.

The reference's cpp_function_wrappers.py insists on porechop/cpp_functions.so inside the (read-only) reference tree,
so a stub module with the same `adapter_alignment` signature that loads oracle/_ref/cpp_functions.so is registered
under that module name before the reference modules are imported -- nothing of the reference is modified.
"""
import ctypes
import json
import os
import sys
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
import porechop  # noqa: E402
sys.modules['porechop.cpp_function_wrappers'] = stub
from porechop import adapters as A  # noqa: E402
from porechop import porechop as P  # noqa: E402
from porechop.nanopore_read import NanoporeRead  # noqa: E402

SC = [3, -6, -5, -2]


def run(file_name, reads_json, barcodes, middle_threshold):
    for a in A.ADAPTERS:
        a.best_start_score, a.best_end_score = 0.0, 0.0
    reads = [NanoporeRead(r['name'], r['seq'], 'I' * len(r['seq'])) for r in reads_json if r['file'] == file_name]
    null = open(os.devnull, 'w')
    matching = P.find_matching_adapter_sets(reads, 0, 150, SC, null, 90.0, 1)
    set_scores = [[a.name, a.best_start_score, a.best_end_score] for a in A.ADAPTERS if '(full sequence)' not in a.name]
    matching = P.fix_up_1d2_sets(matching)
    fwd_rev = P.choose_barcoding_kit(matching, 0, null) if barcodes else None
    matching = P.add_full_barcode_adapter_sets(matching)
    P.find_adapters_at_read_ends(reads, matching, 0, 150, 2, 75.0, SC, null, 4, 1, barcodes, 75.0, 5.0, False, fwd_rev)
    P.find_adapters_in_read_middles(reads, matching, 0, middle_threshold, 10, 100, SC, null, 1, False)
    out_reads = []
    for r in reads:
        out_reads.append({
            'name': r.name,
            'start_trim_amount': r.start_trim_amount, 'end_trim_amount': r.end_trim_amount,
            'start_adapter_alignments': [[x[0].name, x[1], x[2], x[3], x[4]] for x in r.start_adapter_alignments],
            'end_adapter_alignments': [[x[0].name, x[1], x[2], x[3], x[4]] for x in r.end_adapter_alignments],
            'start_barcode_scores': list(r.start_barcode_scores.items()),
            'end_barcode_scores': list(r.end_barcode_scores.items()),
            'middle_adapter_positions': sorted(r.middle_adapter_positions),
            'middle_trim_positions': sorted(r.middle_trim_positions),
            'middle_hit_str': r.middle_hit_str,
            'barcode_call': r.barcode_call,
        })
    return {'file': file_name, 'barcodes': barcodes, 'forward_or_reverse': fwd_rev, 'middle_threshold': middle_threshold,
            'set_scores': set_scores, 'matching_sets': [m.name for m in matching], 'reads': out_reads}


def main():
    reads_json = json.load(open(os.path.join(HERE, 'fixture_reads.json')))
    cases = [run('test_one_adapter_set.fastq', reads_json, False, 90.0),
             run('test_one_adapter_set.fastq', reads_json, False, 85.0),
             run('test_two_adapter_sets.fastq', reads_json, False, 85.0),
             run('test_barcodes.fastq', reads_json, True, 90.0)]
    json.dump(cases, open(os.path.join(HERE, 'golden_phases.json'), 'w'))
    for c in cases:
        print(c['file'], c['matching_sets'][:4], len(c['matching_sets']), [len(r['middle_adapter_positions']) for r in c['reads']],
              [(r['start_trim_amount'], r['end_trim_amount']) for r in c['reads']])


if __name__ == '__main__':
    main()
