"""
Batched drivers for Porechop's three alignment phases (SURVEY.md 8(f) row 1, INTEGRATION.md section 3).

Each function replaces one per-read loop of the reference's `porechop.py` by: gather every (window, adapter) pair ->
ONE submit to the engine -> scatter the results back onto the read / adapter-set objects, filling exactly the fields
the reference's `NanoporeRead` methods fill.  They are duck-typed on Porechop's own objects:

  reads         objects with the `NanoporeRead` attributes (`seq`, `start_trim_amount`, `end_trim_amount`,
                `start_adapter_alignments`, `end_adapter_alignments`, `start_barcode_scores`, `end_barcode_scores`,
                `middle_adapter_positions`, `middle_trim_positions`, `middle_hit_str`; nanopore_read.py:21-55)
  adapter sets  objects with the `Adapter` attributes/methods (`name`, `start_sequence`, `end_sequence`,
                `best_start_score`, `best_end_score`, `is_barcode()`, `barcode_direction()`, `get_barcode_name()`;
                adapters.py:18-52)

Reference behaviour reproduced (file:line in the reference):
  align_adapter_sets            porechop.py:300-322  + nanopore_read.py:149-164
  find_adapters_at_read_ends    porechop.py:463-509  + nanopore_read.py:166-208
  find_adapters_in_read_middles porechop.py:563-591  + nanopore_read.py:210-243 (sequential '-' masking, reproduced with
                                speculative rounds: a read is re-submitted only after one of its alignments was a hit)
Result order per read = adapter order of the input lists (SURVEY 7.4: the insertion order of the barcode-score dicts
breaks ties in determine_barcode).
"""
import numpy as np

from . import cpp_function_wrappers as W
from .align import scores_from_records


def _pack(strings, offset_dtype):
    return W.pack_sequences(strings, offset_dtype=offset_dtype)


def _cross(windows, adapter_seqs, scoring):
    """every window x every adapter -> (full, partial, read_start, read_end) arrays of shape [n_windows, n_adapters]."""
    n, m = len(windows), len(adapter_seqs)
    if n == 0 or m == 0:
        z = np.zeros((n, m))
        return z, z.copy(), np.zeros((n, m), dtype=np.int64), np.zeros((n, m), dtype=np.int64)
    sbuf, soff = _pack(windows, np.int64)
    abuf, aoff = _pack(adapter_seqs, np.int32)
    rec = W.adapter_alignment_batch(sbuf, soff, abuf, aoff, scoring)
    full, part, rs, re_ = scores_from_records(rec)
    return full.reshape(n, m), part.reshape(n, m), rs.reshape(n, m), re_.reshape(n, m)


# ----------------------------------------------------------------------------------------------------------------
def align_adapter_sets(check_reads, adapter_sets, end_size, scoring_scheme_vals, device=None):
    """Phase A: keep, per adapter set, the best full-adapter identity of its start / end sequence over the check
    reads' end windows (reference: best_start_score / best_end_score updated read by read with max()).
    device (default: fastq.DEVICE_SEARCH, PB200_DEVICE_SEARCH=1): one adapterSetSearch call reduces both batches on the
    device and fills the same fields."""
    starts = [(k, s.start_sequence[1]) for k, s in enumerate(adapter_sets) if s.start_sequence]
    ends = [(k, s.end_sequence[1]) for k, s in enumerate(adapter_sets) if s.end_sequence]
    if not check_reads:
        return
    if device is None:
        from .fastq import DEVICE_SEARCH as device
    if device:
        batches, fields = [], []
        for lst, windows, field in ((starts, [r.seq[:end_size] for r in check_reads], 'best_start_score'),
                                    (ends, [r.seq[-end_size:] for r in check_reads], 'best_end_score')):
            if lst:
                batches.append(_pack(windows, np.int64) + _pack([x[1] for x in lst], np.int32))
                fields.append((lst, field))
        for (lst, field), best in zip(fields, W.adapter_set_search(batches, scoring_scheme_vals)):
            for (k, _), b in zip(lst, best):
                setattr(adapter_sets[k], field, max(getattr(adapter_sets[k], field), float(b)))
        return
    if starts:
        full, _, _, _ = _cross([r.seq[:end_size] for r in check_reads], [x[1] for x in starts], scoring_scheme_vals)
        best = full.max(axis=0)
        for (k, _), b in zip(starts, best):
            adapter_sets[k].best_start_score = max(adapter_sets[k].best_start_score, float(b))
    if ends:
        full, _, _, _ = _cross([r.seq[-end_size:] for r in check_reads], [x[1] for x in ends], scoring_scheme_vals)
        best = full.max(axis=0)
        for (k, _), b in zip(ends, best):
            adapter_sets[k].best_end_score = max(adapter_sets[k].best_end_score, float(b))


# ----------------------------------------------------------------------------------------------------------------
def find_adapters_at_read_ends(reads, matching_sets, end_size, extra_trim_size, end_threshold, scoring_scheme_vals,
                               min_trim_size, check_barcodes=False, forward_or_reverse='forward'):
    """Phase B: start/end trim amounts, recorded alignments and barcode scores for every read."""
    if not reads:
        return
    start_sets = [s for s in matching_sets if s.start_sequence]
    end_sets = [s for s in matching_sets if s.end_sequence]
    if start_sets:
        full, part, rs, re_ = _cross([r.seq[:end_size] for r in reads], [s.start_sequence[1] for s in start_sets],
                                     scoring_scheme_vals)
        # partial_score > end_threshold (NaN -> False), read_end != end_size, read_end - read_start >= min_trim_size
        with np.errstate(invalid='ignore'):
            ok = (part > end_threshold) & (re_ != end_size) & ((re_ - rs) >= min_trim_size)
        # only hits (and barcode scores) touch Python objects; np.nonzero is row-major = (read, adapter) order
        for i, a in zip(*np.nonzero(ok)):
            read, aset = reads[i], start_sets[a]
            read.start_trim_amount = max(read.start_trim_amount, int(re_[i, a]) + extra_trim_size)
            read.start_adapter_alignments.append((aset, float(full[i, a]), float(part[i, a]), int(rs[i, a]), int(re_[i, a])))
        if check_barcodes:
            cols = [a for a, s in enumerate(start_sets) if s.is_barcode() and s.barcode_direction() == forward_or_reverse]
            names = [start_sets[a].get_barcode_name() for a in cols]
            for i, read in enumerate(reads):
                for a, nm in zip(cols, names):
                    read.start_barcode_scores[nm] = float(full[i, a])
    if end_sets:
        full, part, rs, re_ = _cross([r.seq[-end_size:] for r in reads], [s.end_sequence[1] for s in end_sets],
                                     scoring_scheme_vals)
        with np.errstate(invalid='ignore'):
            ok = (part > end_threshold) & (rs != 0) & ((re_ - rs) >= min_trim_size)
        for i, a in zip(*np.nonzero(ok)):
            read, aset = reads[i], end_sets[a]
            read.end_trim_amount = max(read.end_trim_amount, (end_size - int(rs[i, a])) + extra_trim_size)
            read.end_adapter_alignments.append((aset, float(full[i, a]), float(part[i, a]), int(rs[i, a]), int(re_[i, a])))
        if check_barcodes:
            cols = [a for a, s in enumerate(end_sets) if s.is_barcode() and s.barcode_direction() == forward_or_reverse]
            names = [end_sets[a].get_barcode_name() for a in cols]
            for i, read in enumerate(reads):
                for a, nm in zip(cols, names):
                    read.end_barcode_scores[nm] = float(full[i, a])


# ----------------------------------------------------------------------------------------------------------------
def _trimmed(read):
    if not read.start_trim_amount and not read.end_trim_amount:
        return read.seq
    return read.seq[read.start_trim_amount:len(read.seq) - read.end_trim_amount]


def find_adapters_in_read_middles(reads, adapters, middle_threshold, extra_middle_trim_good_side,
                                  extra_middle_trim_bad_side, scoring_scheme_vals, start_sequence_names,
                                  end_sequence_names):
    """Phase C: `adapters` is the list of (name, sequence) the reference builds at porechop.py:541-548.
    The reference aligns adapter after adapter against a per-read `masked_seq` and re-aligns the same adapter after
    every hit.  Here round r submits, for every still-active read, its current masked sequence against the adapters
    from its current index on; results are consumed in adapter order and stay valid until the first hit, which masks
    the read and schedules it for the next round starting at the same adapter."""
    n_ad = len(adapters)
    if not reads or n_ad == 0:
        return
    masked = [_trimmed(r) for r in reads]
    next_adapter = [0] * len(reads)
    active = list(range(len(reads)))
    ad_seqs = [a[1] for a in adapters]
    abuf, aoff = _pack(ad_seqs, np.int32)
    first = True
    while active:
        seqs = [masked[i] for i in active]
        sbuf, soff = _pack(seqs, np.int64)
        if first:
            rec = W.adapter_alignment_batch(sbuf, soff, abuf, aoff, scoring_scheme_vals)   # cross product
            pair_index, stride = None, n_ad
        else:
            # pair list without per-pair Python objects: read k's block holds adapters next_adapter .. n_ad-1 and starts
            # at base[k]; pair (k, a) sits at base[k] + a - next_adapter (same construction as fastq.find_middle_hits)
            first_ad = np.array([next_adapter[i] for i in active], dtype=np.int64)
            counts = n_ad - first_ad
            base = np.zeros(len(active) + 1, dtype=np.int64)
            np.cumsum(counts, out=base[1:])
            ps = np.repeat(np.arange(len(active), dtype=np.int32), counts)
            pa = (np.arange(base[-1], dtype=np.int64) - np.repeat(base[:-1] - first_ad, counts)).astype(np.int32)
            rec = W.adapter_alignment_batch(sbuf, soff, abuf, aoff, scoring_scheme_vals, ps, pa)
            pair_index, stride = (base, first_ad), None
        full, _, rs, re_ = scores_from_records(rec)
        still = []
        for k, i in enumerate(active):
            read = reads[i]
            a = next_adapter[i]
            hit = False
            while a < n_ad:
                p = (k * stride + a) if stride is not None else int(pair_index[0][k] + a - pair_index[1][k])
                full_score, read_start, read_end = float(full[p]), int(rs[p]), int(re_[p])
                if full_score >= middle_threshold:
                    name = adapters[a][0]
                    masked[i] = masked[i][:read_start] + '-' * (read_end - read_start) + masked[i][read_end:]
                    read.middle_adapter_positions.update(range(read_start, read_end))
                    read.middle_hit_str += '  ' + name + ' (read coords: ' + str(read_start) + '-' + str(read_end) + \
                                           ', ' + 'identity: ' + '%.1f' % full_score + '%)\n'
                    trim_start = read_start - extra_middle_trim_good_side
                    if name in start_sequence_names:
                        trim_start = read_start - extra_middle_trim_bad_side
                    trim_end = read_end + extra_middle_trim_good_side
                    if name in end_sequence_names:
                        trim_end = read_end + extra_middle_trim_bad_side
                    read.middle_trim_positions.update(range(trim_start, trim_end))
                    next_adapter[i] = a          # the reference re-aligns the SAME adapter after a hit
                    hit = True
                    break
                a += 1
            if hit:
                still.append(i)
        active = still
        first = False
