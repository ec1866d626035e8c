"""CPU tier, on the host-simulated engine (tests/sim): the traceback of trace_kernel -- its incremental trace cursor
(TraceCursor) and the match count taken from the score (traceback_stats_cur<true>) -- against the oracle.  Paths cross chunk
and lane boundaries at every step residue mod 4 (every window length 1..170, every lane-group class G = 4 / 8 / 16 / 32),
long vertical and horizontal gap runs end at row 1 and column 1, N bases match N, the given-end windows of the two-pass path
start at col0 > 0, and the scoring schemes include linear ones and ones with match == mismatch (matches compared base by
base)."""
import os
import random
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_batch

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

SCHEMES = [[3, -6, -5, -2], [3, -6, -2, -2], [1, -1, -1, -1], [2, -3, -2, -5], [5, -4, -8, -1], [3, -6, -5, -5], [1, 0, -1, -1],
           [10, -20, -15, -7], [2, 2, -3, -1], [1, 1, -2, -2]]


@pytest.fixture(scope='module')
def W():
    import sim_engine
    return sim_engine.load()


@pytest.fixture(autouse=True)
def _stream_order_checked():
    import sim_engine
    sim_engine.clear_races()
    yield
    sim_engine.assert_no_races()


def _seq(rng, n, alphabet='ACGT'):
    return ''.join(rng.choice(alphabet) for _ in range(n))


def _check(W, reads, ads, scoring, direct_max=None):
    rbuf, roff = W.pack_sequences(reads)
    abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
    exp = oracle_batch(rbuf, roff, abuf, aoff, scoring)
    try:
        if direct_max is not None:
            W.set_option('direct_max', direct_max)
        got = W.adapter_alignment_batch(rbuf, roff, abuf, aoff, scoring)
    finally:
        W.set_option('direct_max', 160)
    assert np.array_equal(got, exp), scoring


def _mutate(rng, s, p, alphabet='ACGT'):
    """substitutions, insertions and deletions at rate p each: gap runs of several lengths in the path"""
    out = []
    for c in s:
        x = rng.random()
        if x < p:
            out.append(rng.choice(alphabet))
        elif x < 2 * p:
            out.append(c + _seq(rng, rng.randint(1, 4), alphabet))
        elif x >= 3 * p:
            out.append(c)
    return ''.join(out)


def _windows(rng, lengths, ad, p=0.08, alphabet='ACGT'):
    out = []
    for k, n in enumerate(lengths):
        s = _seq(rng, n, alphabet)
        copy = _mutate(rng, ad, p, alphabet)
        cut = rng.randint(len(copy) // 2, len(copy)) if copy else 0
        part = (copy[:cut] if k % 2 else copy[len(copy) - cut:])[:n]
        out.append(s[:n - len(part)] + part if k % 2 else part + s[len(part):])
    return out


@pytest.mark.parametrize('m', [20, 28, 40, 100, 200])      # G = 4 (R = 5 / 7), 8, 16, 32
def test_every_window_length_every_group_class(W, m):
    rng = random.Random(11 + m)
    ad = _seq(rng, m)
    lengths = list(range(1, 171))
    rng.shuffle(lengths)
    for scoring in ([3, -6, -5, -2], [1, -1, -1, -1]):
        _check(W, _windows(rng, lengths, ad), [ad], scoring, direct_max=170)


def test_every_scheme_with_gaps_and_n_bases(W):
    rng = random.Random(3)
    ad = _seq(rng, 28, 'ACGTN')
    ad2 = _seq(rng, 22)
    reads = _windows(rng, [rng.randint(1, 170) for _ in range(48)], ad, p=0.12, alphabet='ACGTN') + \
        ['N' * 40, 'N' * 3 + ad + 'N' * 5, ad, '', 'A']
    for scoring in SCHEMES:
        _check(W, reads, [ad, ad2], scoring)


def test_gap_runs_ending_at_row_1_and_column_1(W):
    """paths whose last (backwards) run is a long vertical run down to row 1 or a long horizontal run down to column 1"""
    rng = random.Random(9)
    ad = _seq(rng, 28)
    reads = []
    for k in range(1, 20):
        reads.append(ad[k:] + _seq(rng, 30))                  # adapter rows 1..k before the read: vertical run to row 1
        reads.append(ad[:8] + _seq(rng, k) + ad[8:])          # horizontal run inside the path
        reads.append(_seq(rng, k) + ad[:20] + _seq(rng, 5))   # read columns before the adapter: horizontal / free start
        reads.append(ad[0] + _seq(rng, k + 3) + ad[1:])       # horizontal run that ends at column 1
    for scoring in ([3, -6, -5, -2], [3, -6, -2, -2], [5, -4, -8, -1], [1, 0, -1, -1], [2, 2, -3, -1]):
        _check(W, reads, [ad], scoring, direct_max=170)


def test_given_end_windows(W):
    """reads longer than direct_max: score pass, then windows with col0 > 0 and a given end cell"""
    rng = random.Random(13)
    ad = _seq(rng, 24)
    reads = _windows(rng, [rng.randint(150, 400) for _ in range(40)], ad, p=0.1)
    for scoring in ([3, -6, -5, -2], [1, -1, -1, -1], [2, -3, -2, -5], [2, 2, -3, -1]):
        _check(W, reads, [ad, _seq(rng, 30)], scoring, direct_max=100)
