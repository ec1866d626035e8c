"""Scoring schemes at the edge of the int16 kernels' domain and the inputs the scheme tests align under them (TESTS ONLY).

route() and two_pass() restate the engine's routing (engine.cu scheme_info / int16_ok / class_of, run_class_tasks): an
adapter of length m goes to row-capacity class k (capacity G*R >= m) when A*(m+3) <= 4000 (A = max |score|), ma >= mi,
ma - mi <= 4096, both gap scores <= 0 and m <= 256, else to the int32 generic kernel; a class takes the score pass plus the
windowed trace when both gap scores are negative and its longest sequence is longer than direct_max (160) and W(m) + 1."""
import random

LIMIT = 4000
DIRECT_MAX = 160
CAPS = [(4 << (k // 4)) * (5 + k % 4) for k in range(16)]
GENERIC = 'generic'


def class_lengths(k):
    """the largest length of class k, one less, and the smallest (the previous capacity + 1)"""
    return sorted({CAPS[k], CAPS[k] - 1, CAPS[k - 1] + 1 if k else 1}, reverse=True)


def edge_schemes(A):
    """(shape name, [ma, mi, go, ge]) with max |score| == A (A >= 2)"""
    h, t = max(1, A // 2), max(1, A // 3)
    return [('all_A', [A, -A, -A, -A]), ('cheap_gaps', [A, -A, -1, -1]), ('unit_match', [1, -A, -A, -A]),
            ('affine_open_A', [A, -1, -A, -1]), ('zero_mismatch', [A, 0, -A, -A]), ('linear', [t, -A, -h, -h]),
            ('ma_eq_mi', [A, A, -h, -t]), ('mi_positive', [A, t, -h, -A]), ('ma_nonpositive', [0, -A, -h, -t]),
            ('free_open', [A, -h, 0, -t]), ('free_extend', [A, -A, -h, 0])]


def route(sc, m):
    """row-capacity class index of an adapter of length m, or GENERIC"""
    ma, mi, go, ge = sc
    A = max(abs(x) for x in sc)
    if not (ma >= mi and ma - mi <= 4096 and go <= 0 and ge <= 0 and A * (m + 3) <= LIMIT and m <= 256):
        return GENERIC
    return next(k for k in range(16) if m <= CAPS[k])


def window(sc, m):
    """W(m) of a scheme with a window bound, else None"""
    ma, mi, go, ge = sc
    return m + m * max(ma, mi, 0) // min(-go, -ge) if go < 0 and ge < 0 else None


def two_pass(sc, m_max, max_n, direct_max=DIRECT_MAX):
    W = window(sc, m_max)
    return W is not None and max_n > direct_max and W + 1 < max_n


def rand_seq(rng, n):
    return ''.join(rng.choice('ACGT') for _ in range(n))


def gappy(rng, s, p_ins=0.3, p_del=0.05, p_sub=0.05):
    """a copy of s with insertions after most bases, a few deletions and substitutions"""
    out = []
    for c in s:
        x = rng.random()
        if x < p_del:
            continue
        out.append(rng.choice('ACGT') if x < p_del + p_sub else c)
        while rng.random() < p_ins:
            out.append(rng.choice('ACGT'))
    return ''.join(out)


def implant(rng, body, ad):
    p = rng.randint(0, len(body))
    return body[:p] + ad + body[p:]


def edge_reads(rng, adapters, sc, n_random=6, long_reads=2):
    """(reads of at most DIRECT_MAX bases, longer reads): the adapter, repeats, a gappy copy, all-N, empty, one base, random
    reads with implants on both sides of DIRECT_MAX, and reads longer than the window of the longest adapter"""
    ad = adapters[0]
    reads = [ad, ad * 2, ad * 3, gappy(rng, ad), 'N' * rng.randint(1, 200), '', rand_seq(rng, 1), ad[:max(1, len(ad) // 2)]]
    for _ in range(n_random):
        r = rand_seq(rng, rng.choice([rng.randint(1, DIRECT_MAX), rng.randint(DIRECT_MAX + 1, 400)]))
        if rng.random() < 0.7:
            a = rng.choice(adapters)
            r = implant(rng, r, gappy(rng, a, 0.1) if rng.random() < 0.5 else a[rng.randint(0, len(a) // 2):])
        reads.append(r)
    m_max = max(len(a) for a in adapters)
    lo = max(DIRECT_MAX + 1, (window(sc, m_max) or 0) + 2, 3 * m_max)
    for _ in range(long_reads):
        r = rand_seq(rng, lo + rng.randint(0, 300))
        for _ in range(rng.randint(1, 2)):
            r = implant(rng, r, gappy(rng, rng.choice(adapters), 0.2))
        reads.append(r)
    return [r for r in reads if len(r) <= DIRECT_MAX], [r for r in reads if len(r) > DIRECT_MAX]


def edge_cases(seed=2026, n_random=6, long_reads=2):
    """16 classes x 3 lengths x 11 shapes with A = 4000 // (m+3): dicts with class, m, shape, scoring, adapters (one of
    length m first, then shorter ones of the class; 2 or 3 of them, so that the query-profile score pass sees an even and
    an odd number), short and long reads"""
    rng = random.Random(seed)
    cases = []
    for k in range(16):
        lo = CAPS[k - 1] + 1 if k else 1
        for m in class_lengths(k):
            for j, (shape, sc) in enumerate(edge_schemes(LIMIT // (m + 3))):
                ads = [rand_seq(rng, m)] + [rand_seq(rng, rng.randint(lo, m)) for _ in range(1 + (j + m) % 2)]
                short, long_ = edge_reads(rng, ads, sc, n_random, long_reads)
                cases.append(dict(cls=k, m=m, shape=shape, scoring=sc, adapters=ads, short=short, long=long_))
    return cases


def noisy_fastq(seed=20261019):
    """30 reads whose end and middle (chimera) adapters carry 4-30 % errors, some truncated: identities near the end (75)
    and middle (85) thresholds, where the scoring scheme decides the trims"""
    top, bottom = 'AATGTACTTCGTTCAGTTACGTATTGCT', 'GCAATACGTAACTGAACGAAGT'     # SQK-NSK007 (public kit sequences)
    rng = random.Random(seed)
    recs = []
    for k in range(30):
        p = (0.04, 0.1, 0.16, 0.22, 0.3)[k % 5]
        noisy = lambda s, q=p: gappy(rng, s, q / 3, q / 3, q / 3)              # noqa: E731
        end = noisy(bottom)
        s = rand_seq(rng, rng.randint(0, 12)) + noisy(top)[rng.randint(0, 8) if k % 4 == 1 else 0:] + \
            rand_seq(rng, rng.randint(200, 700))
        if k % 3 == 0:
            s += noisy(bottom, p / 2) + noisy(top, p / 2) + rand_seq(rng, rng.randint(200, 700))
        s += (end[:len(end) - rng.randint(1, 8)] if k % 4 == 2 else end) + rand_seq(rng, rng.randint(0, 12))
        recs.append('@noisy_%d p=%.2f\n%s\n+\n%s\n' % (k, p, s, ''.join(chr(rng.randint(35, 73)) for _ in s)))
    return ''.join(recs)


def cli_inputs():
    """the inputs of the --scoring_scheme cases (tests/golden/golden_schemes.json): noisy trim reads as FASTQ and as 70-column
    FASTA, and the barcoded reads of golden_emit.json (into bins)"""
    from helpers import load_golden
    from porechop_b200 import fastq
    fq = noisy_fastq()
    return {'trim_fastq': fq, 'trim_fasta': fastq.emit(fastq.parse_fastq(fq.encode()), fmt='fasta').decode(),
            'barcoded_fastq': load_golden('golden_emit.json')['barcoded_fastq']}
