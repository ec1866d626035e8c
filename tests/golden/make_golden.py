#!/usr/bin/env python3
"""Generate the committed golden fixtures from the UNMODIFIED reference (tests/helpers.py REFERENCE).

Runs the reference C++ (oracle/_ref/cpp_functions.so, built by oracle/Makefile from
<REFERENCE>/porechop/src/*.cpp + vendored SeqAn) through its own C-ABI
(porechop/include/adapter_align.h:12-16) and imports the reference's adapter table
(porechop/adapters.py:77-498) to write:

  tests/golden/adapters.json         the 119 adapter sets + the synthesised full-barcode sets (data only)
  tests/golden/fixture_reads.json    reads of test/test_one_adapter_set.fastq, test_two_adapter_sets.fastq,
                                     test_barcodes.fastq (the reference's own parity corpus, SURVEY 8c)
  tests/golden/golden_windows.json   reference strings for 150-nt end windows x a panel of adapters
  tests/golden/golden_fullread.json  reference strings for full reads (incl. '-'-masked re-alignments)
  tests/golden/golden_random.json    reference strings for seeded random / edge-case inputs
  tests/golden/golden_live.json      reference strings for the seeded cases of tests/helpers.py live_cases()

Nothing at test time reads the reference checkout; only these files.
"""
import ctypes, json, os, random, sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(HERE))
from helpers import REFERENCE as REF, live_cases  # noqa: E402

sys.path.insert(0, REF)

lib = ctypes.CDLL(os.path.join(ROOT, 'oracle', '_ref', 'cpp_functions.so'))
lib.adapterAlignment.argtypes = [ctypes.c_char_p, ctypes.c_char_p] + [ctypes.c_int] * 4
lib.adapterAlignment.restype = ctypes.c_void_p
lib.freeCString.argtypes = [ctypes.c_void_p]


def ref_align(read, adapter, sc):
    p = lib.adapterAlignment(read.encode(), adapter.encode(), *sc)
    s = ctypes.cast(p, ctypes.c_char_p).value.decode()
    lib.freeCString(p)
    return s


def load_fastq(path):
    out = []
    with open(path) as f:
        lines = [l.rstrip('\n') for l in f]
    for i in range(0, len(lines) - 3, 4):
        out.append((lines[i][1:], lines[i + 1]))
    return out


def main():
    import warnings
    warnings.simplefilter('ignore')
    from porechop import adapters as A
    sets = []
    for a in A.ADAPTERS:
        sets.append({'name': a.name, 'start': list(a.start_sequence), 'end': list(a.end_sequence)})
    full = []
    for i in range(1, 13):
        a = A.make_full_native_barcode_adapter(i)
        full.append({'name': a.name, 'start': list(a.start_sequence), 'end': list(a.end_sequence)})
    for i in range(1, 13):
        a = A.make_old_full_rapid_barcode_adapter(i)
        full.append({'name': a.name, 'start': list(a.start_sequence), 'end': list(a.end_sequence)})
    for i in range(1, 97):
        a = A.make_new_full_rapid_barcode_adapter(i)
        full.append({'name': a.name, 'start': list(a.start_sequence), 'end': list(a.end_sequence)})
    json.dump({'sets': sets, 'full_barcode_sets': full}, open(os.path.join(HERE, 'adapters.json'), 'w'), indent=0)

    reads = []
    for fn in ('test_one_adapter_set.fastq', 'test_two_adapter_sets.fastq', 'test_barcodes.fastq'):
        for name, seq in load_fastq(os.path.join(REF, 'test', fn)):
            reads.append({'file': fn, 'name': name, 'seq': seq.upper()})
    json.dump(reads, open(os.path.join(HERE, 'fixture_reads.json'), 'w'), indent=0)

    default = [3, -6, -5, -2]
    byname = {s['name']: s for s in sets}
    panel = []
    for nm in ('SQK-NSK007', 'SQK-MAP006', 'SQK-MAP006 short', 'Rapid', 'PCR adapters 1', 'cDNA SSP',
               'Barcode 1 (reverse)', 'Barcode 2 (reverse)', 'Barcode 3 (reverse)', 'Barcode 1 (forward)',
               'Barcode 96 (forward)'):
        s = byname[nm]
        for seq in (s['start'], s['end']):
            if seq and seq[1] not in [p[1] for p in panel]:
                panel.append([seq[0], seq[1]])
    for s in (full[0], full[12], full[24]):
        for seq in (s['start'], s['end']):
            if seq:
                panel.append([seq[0], seq[1]])

    win = []
    for ri, r in enumerate(reads):
        for kind, w in (('start', r['seq'][:150]), ('end', r['seq'][-150:])):
            for ai, (an, aseq) in enumerate(panel):
                win.append([ri, kind, ai, ref_align(w, aseq, default)])
    json.dump({'scoring': default, 'end_size': 150, 'panel': panel, 'results': win},
              open(os.path.join(HERE, 'golden_windows.json'), 'w'))

    # full-read (Phase C style) alignments incl. masked re-alignments (nanopore_read.py:210-243)
    fr = []
    ytop, ybot = byname['SQK-NSK007']['start'][1], byname['SQK-NSK007']['end'][1]
    for ri, r in enumerate(reads):
        for an, aseq in (('Y_Top', ytop), ('Y_Bottom', ybot), (panel[-1][0], panel[-1][1])):
            seq = r['seq']
            for rnd in range(3):
                s = ref_align(seq, aseq, default)
                fr.append([ri, rnd, an, aseq, seq.count('-'), s])
                parts = s.split(',')
                rs, re_ = int(parts[0]), int(parts[1]) + 1
                if float(parts[6]) < 70.0 or rs < 0:
                    break
                seq = seq[:rs] + '-' * (re_ - rs) + seq[re_:]
    # store masks as the list of masked intervals to rebuild the sequence in tests
    json.dump({'scoring': default, 'results': fr}, open(os.path.join(HERE, 'golden_fullread.json'), 'w'))

    # randomized + edge cases
    random.seed(20260923)
    schemes = [[3, -6, -5, -2], [3, -6, -2, -2], [1, -1, -1, -1], [2, -3, -2, -5], [5, -4, -8, -1],
               [3, -6, -5, -5], [1, 0, -1, -1], [3, -6, -4, -2], [10, -20, -15, -7]]

    def mut(s, al):
        o = []
        for c in s:
            x = random.random()
            if x < 0.04:
                continue
            if x < 0.09:
                o.append(random.choice(al)); continue
            if x < 0.13:
                o.append(c); o.append(random.choice(al)); continue
            o.append(c)
        return ''.join(o)

    rnd = []
    edge = [('', 'ACGT'), ('ACGT', ''), ('', ''), ('N' * 20, ytop), ('-' * 20, ytop), ('A', 'C'), ('A', 'A'),
            ('ACGTTTTTTTTTTACGT', 'ACGT'), ('TTTTACG', 'ACGT'), ('acgu', 'ACGT'), ('--A-', 'A'),
            (ytop, ytop), (ytop[5:], ytop), (ytop[:-5], ytop), ('GG' + ytop + 'GG', ytop), (ytop, 'GG' + ytop + 'GG'),
            ('ACGT' * 40, 'ACGT' * 10), ('A' * 150, 'A' * 28), ('A' * 150, 'C' * 28), ('NNNN', 'NNNN'),
            ('ACGTNACGT', 'ACGTNACGT'), ('XYZ', 'XYZ')]
    for rd, ad in edge:
        for sc in schemes[:4]:
            rnd.append([rd, ad, sc, ref_align(rd, ad, sc)])
    for it in range(2000):
        al = random.choice(['A', 'AC', 'ACGT', 'ACGTN', 'ACGT', 'ACGT'])
        m = random.choice([random.randint(1, 40), random.randint(20, 34), random.randint(60, 130)])
        n = random.choice([random.randint(1, 200), 150, random.randint(100, 400)])
        ad = ''.join(random.choice(al) for _ in range(m))
        rd = ''.join(random.choice(al) for _ in range(n))
        if random.random() < 0.7:
            p = random.randint(0, n)
            ins = mut(ad, al)
            if random.random() < 0.3:
                ins = ins[random.randint(0, len(ins)):]
            if random.random() < 0.3:
                ins = ins[:random.randint(0, len(ins))]
            rd = rd[:p] + ins + rd[p:]
            if random.random() < 0.5:
                rd = rd[:n] if random.random() < 0.5 else rd[-n:]
        if not rd:
            rd = 'A'
        sc = random.choice(schemes)
        rnd.append([rd, ad, sc, ref_align(rd, ad, sc)])
    json.dump(rnd, open(os.path.join(HERE, 'golden_random.json'), 'w'))
    live = [ref_align(rd, ad, sc) for rd, ad, sc in live_cases()]
    json.dump(live, open(os.path.join(HERE, 'golden_live.json'), 'w'), indent=0)
    print('adapters', len(sets), 'full', len(full), 'reads', len(reads), 'windows', len(win), 'fullread', len(fr),
          'random', len(rnd), 'live', len(live))


if __name__ == '__main__':
    main()
