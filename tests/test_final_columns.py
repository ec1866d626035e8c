"""CPU tier, on the host-simulated engine (tests/sim): the final columns of a trace slot -- the careful chunks whose step also
scans the final column (lane_step<.., FCOL>) -- against the oracle over every window length 1..170 (every residue mod 4),
every adapter length of the end-trim row classes (20..32 rows), ragged and uniform slots, empty halves, the wider lane groups
(G = 8 / 16 / 32) and the given-end windows of the two-pass path."""
import os
import random
import sys

import numpy as np
import pytest

from helpers import ROOT, oracle_batch

sys.path.insert(0, os.path.join(ROOT, 'tests', 'sim'))

SCORING = [3, -6, -5, -2]


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


def _seq(rng, n):
    return ''.join(rng.choice('ACGT') for _ in range(n))


def _check(W, reads, ads, direct_max=None):
    rbuf, roff = W.pack_sequences(reads)
    abuf, aoff = W.pack_sequences(ads, offset_dtype=np.int32)
    exp = oracle_batch(rbuf, roff, abuf, aoff, SCORING)
    try:
        if direct_max is not None:
            W.set_option('direct_max', direct_max)
        got = W.adapter_alignment_batch(rbuf, roff, abuf, aoff, SCORING)
    finally:
        W.set_option('direct_max', 160)
    assert np.array_equal(got, exp)


def _windows(rng, lengths, ad):
    """reads of the given lengths that end with a mutated prefix of `ad` (odd positions: the adapter runs past the read's end,
    so the best cell is in the read's final column, above the last row) or start with a mutated suffix of it"""
    out = []
    for k, n in enumerate(lengths):
        s = _seq(rng, n)
        copy = ''.join(c if rng.random() > 0.1 else rng.choice('ACGT') for c in ad)
        cut = rng.randint(len(ad) // 2, len(ad))
        part = (copy[:cut] if k % 2 else copy[len(ad) - cut:])[:n]
        out.append(s[:n - len(part)] + part if k % 2 else part + s[len(part):])
    return out


def test_every_window_length_and_end_trim_adapter_length(W):
    rng = random.Random(5)
    lengths = list(range(1, 171))
    ragged = lengths[:]
    rng.shuffle(ragged)                                  # the two halves of a slot differ in length
    uniform = [n for n in lengths for _ in (0, 1)]       # both halves of every slot equally long
    for m in range(20, 33):           # direct_max 170: every window in the single trace pass (longer ones take two passes)
        ad = _seq(rng, m)
        _check(W, _windows(rng, ragged, ad) + [''], [ad], direct_max=170)
        _check(W, _windows(rng, uniform, ad), [ad], direct_max=170)


def test_ragged_pairs_wide_groups_and_given_end_windows(W):
    rng = random.Random(7)
    reads = _windows(rng, [rng.randint(1, 170) for _ in range(60)], _seq(rng, 28)) + ['', 'A', 'ACG', 'N' * 7]
    for ads in ([_seq(rng, 28), _seq(rng, 22)], [_seq(rng, 40)], [_seq(rng, 100), ''], [_seq(rng, 200)]):
        _check(W, reads, ads)
    longer = _windows(rng, [rng.randint(150, 400) for _ in range(24)], _seq(rng, 24))
    _check(W, longer, [_seq(rng, 24), _seq(rng, 30)], direct_max=100)     # score pass -> given-end windows -> trace pass
