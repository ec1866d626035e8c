#!/usr/bin/env python3
"""Golden vectors for `--scoring_scheme`: whole-CLI outputs of the UNMODIFIED reference (porechop.main() of tests/helpers.py
REFERENCE on oracle/_ref/cpp_functions.so) under five non-default scoring schemes, for the three inputs of
tests/scheme_edges.py cli_inputs().  Authoring container only; writes tests/golden/golden_schemes.json.

Each case keeps what the flat pipeline needs to reproduce the run without the reference -- the adapter sets Phase A chose
under the scheme, the options and the scheme -- and the SHA-256 of the output file (of every bin file)."""
import hashlib
import json
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden_emit as E  # noqa: E402  (loads the reference package on oracle/_ref)
from scheme_edges import cli_inputs  # noqa: E402

SCHEMES = ['1,-1,-1,-1', '3,-6,-5,-5', '5,-4,-8,-1', '10,-20,-15,-7', '3,-6,-2,-2']
OUT = {'trim_fastq': ('o.fastq', ['--min_split_read_size', '50']), 'trim_fasta': ('o.fasta', ['--min_split_read_size', '100']),
       'barcoded_fastq': ('', [])}      # '' = into bins


def sha(text):
    return hashlib.sha256(text.encode()).hexdigest()


def main():
    cases = {}
    with tempfile.TemporaryDirectory() as d:
        for name, text in sorted(cli_inputs().items()):
            out_name, extra = OUT[name]
            path = os.path.join(d, 'in.' + name.split('_')[1])
            with open(path, 'w', newline='') as f:
                f.write(text)
            for scheme in SCHEMES:
                args = extra + ['--scoring_scheme', scheme]
                c = E.run_case(path, out_name, args) if out_name else E.run_barcode_case(path, 'fastq', args)
                assert c['scoring'] == [int(x) for x in scheme.split(',')]
                if out_name:
                    c['sha256'] = sha(c.pop('output'))
                else:
                    c['sha256'] = {f: sha(t) for f, t in c.pop('bins').items()}
                c.update(input=name, mode='trim' if out_name else 'bins')
                cases['%s %s' % (name, scheme)] = c
    lines = ['%s: %s' % (json.dumps(k), json.dumps(cases[k], sort_keys=True)) for k in sorted(cases)]
    with open(os.path.join(HERE, 'golden_schemes.json'), 'w') as f:
        f.write('{"schemes": %s, "cases": {\n%s\n}}\n' % (json.dumps(SCHEMES), ',\n'.join(lines)))


if __name__ == '__main__':
    main()
