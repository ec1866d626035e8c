"""
ctypes wrapper around cpp_functions.so -- the H100 adapter-alignment engine.

Mirror of the reference's porechop/cpp_function_wrappers.py (same module name, same library file name next
to the module, same `adapter_alignment(read_sequence, adapter_sequence, scoring_scheme_vals) -> str`
signature and result string, reference lines 21-63), plus the batched call the Python host uses to submit
every (read window, adapter) / (full read, adapter) pair at once (SURVEY.md 8(b)).

There is no CPU fallback: if cpp_functions.so is missing the import exits like the reference does
(cpp_function_wrappers.py:23-24), and every call raises if no sm_90 (H100) CUDA device is usable.
"""

import os
import sys
from ctypes import CDLL, POINTER, Structure, addressof, byref, c_char_p, c_double, c_int, c_int32, c_int64, c_longlong, c_void_p, cast, \
    create_string_buffer

import numpy as np

SO_FILE = 'cpp_functions.so'
SO_FILE_FULL = os.path.join(os.path.dirname(os.path.realpath(__file__)), SO_FILE)
if not os.path.isfile(SO_FILE_FULL):
    sys.exit('could not find ' + SO_FILE + ' - please reinstall (python -m porechop_b200.build)')
C_LIB = CDLL(SO_FILE_FULL)

# ---- reference ABI (porechop/include/adapter_align.h:13-15) ----
C_LIB.adapterAlignment.argtypes = [c_char_p,  # Read sequence
                                   c_char_p,  # Adapter sequence
                                   c_int,     # Match score
                                   c_int,     # Mismatch score
                                   c_int,     # Gap open score
                                   c_int]     # Gap extension score
C_LIB.adapterAlignment.restype = c_void_p     # String describing alignment
C_LIB.freeCString.argtypes = [c_void_p]
C_LIB.freeCString.restype = None

# ---- batched ABI (include/porechop_b200.h) ----
C_LIB.adapterAlignmentBatch.argtypes = [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                                        c_int64, c_int, c_int, c_int, c_int, c_void_p]
C_LIB.adapterAlignmentBatch.restype = c_int


class BatchDesc(Structure):
    """pb200_batch_t (include/porechop_b200.h)"""
    _fields_ = [('seqs', c_void_p), ('seq_off', c_void_p), ('n_seqs', c_int64),
                ('adapters', c_void_p), ('ad_off', c_void_p), ('n_adapters', c_int32), ('out', c_void_p)]


class EndBatchDesc(Structure):
    """pb200_end_batch_t (include/porechop_b200.h)"""
    _fields_ = [('batch', BatchDesc), ('is_start', c_int32), ('end_size', c_int32), ('extra_trim_size', c_int32),
                ('min_trim_size', c_int32), ('end_threshold', c_double), ('score_cols', c_void_p), ('n_score_cols', c_int32),
                ('trim', c_void_p), ('score_pairs', c_void_p), ('top2', c_void_p)]


C_LIB.adapterEndDecisions.argtypes = [POINTER(EndBatchDesc), c_int, c_int, c_int, c_int, c_int]
C_LIB.adapterEndDecisions.restype = c_int


class SearchBatchDesc(Structure):
    """pb200_search_batch_t (include/porechop_b200.h)"""
    _fields_ = [('batch', BatchDesc), ('best', c_void_p)]


C_LIB.adapterSetSearch.argtypes = [POINTER(SearchBatchDesc), c_int, c_int, c_int, c_int, c_int]
C_LIB.adapterSetSearch.restype = c_int
C_LIB.pb200TrimThresholdTable.argtypes = [c_double, c_int32, c_void_p]
C_LIB.pb200TrimThresholdTable.restype = c_int
C_LIB.adapterAlignmentBatchMulti.argtypes = [POINTER(BatchDesc), c_int, c_int, c_int, c_int, c_int]
C_LIB.adapterAlignmentBatchMulti.restype = c_int
C_LIB.adapterAlignmentBatchDevice.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p,
                                              c_int32, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
C_LIB.adapterAlignmentBatchDevice.restype = c_int
C_LIB.adapterMiddleScan.argtypes = [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int32, c_int, c_int, c_int, c_int,
                                    c_double, c_void_p, c_void_p, c_int64, c_void_p]
C_LIB.adapterMiddleScan.restype = c_int
C_LIB.adapterMiddleScanDevice.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_int32, c_int,
                                          c_int, c_int, c_int, c_double, c_void_p, c_void_p, c_int64, c_void_p, c_void_p]
C_LIB.adapterMiddleScanDevice.restype = c_int


class TrimSideDesc(Structure):
    """pb200_trim_side_t (include/porechop_b200.h)"""
    _fields_ = [('adapters', c_void_p), ('ad_off', c_void_p), ('n_adapters', c_int32), ('score_cols', c_void_p),
                ('n_score_cols', c_int32), ('trim', c_void_p), ('score_pairs', c_void_p), ('top2', c_void_p)]


class TrimArgsDesc(Structure):
    """pb200_trim_args_t (include/porechop_b200.h)"""
    _fields_ = [('end_size', c_int32), ('extra_trim_size', c_int32), ('min_trim_size', c_int32), ('end_threshold', c_double),
                ('start', TrimSideDesc), ('end', TrimSideDesc), ('mid_adapters', c_void_p), ('mid_ad_off', c_void_p),
                ('n_mid_adapters', c_int32), ('middle_threshold', c_double), ('n_hits', c_void_p), ('hits', c_void_p),
                ('hits_cap', c_int64), ('n_total', c_void_p)]


C_LIB.adapterTrimReads.argtypes = [c_void_p, c_void_p, c_int64, POINTER(TrimArgsDesc), c_int, c_int, c_int, c_int]
C_LIB.adapterTrimReads.restype = c_int
C_LIB.adapterTrimReadsDevice.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int64, POINTER(TrimArgsDesc), c_int, c_int,
                                         c_int, c_int, c_void_p]
C_LIB.adapterTrimReadsDevice.restype = c_int


class SplitArgsDesc(Structure):
    """pb200_split_args_t (include/porechop_b200.h)"""
    _fields_ = [('d_quals', c_void_p), ('mid_extra_left', c_void_p), ('mid_extra_right', c_void_p),
                ('min_split_read_size', c_int32), ('discard_middle', c_int32), ('untrimmed', c_int32),
                ('d_out_seq', c_void_p), ('d_out_qual', c_void_p), ('d_out_off', c_void_p), ('d_out_read', c_void_p),
                ('d_out_part', c_void_p), ('parts_cap', c_int64), ('n_parts', c_void_p), ('n_out_bases', c_void_p)]


C_LIB.adapterTrimSplitReadsDevice.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int64, POINTER(TrimArgsDesc),
                                              POINTER(SplitArgsDesc), c_int, c_int, c_int, c_int, c_void_p]
C_LIB.adapterTrimSplitReadsDevice.restype = c_int


class DemuxArgsDesc(Structure):
    """pb200_demux_args_t (include/porechop_b200.h)"""
    _fields_ = [('start_bin', c_void_p), ('end_bin', c_void_p), ('n_bins', c_int32), ('barcode_threshold', c_double),
                ('barcode_diff', c_double), ('require_two_barcodes', c_int32), ('discard_unassigned', c_int32),
                ('d_albacore', c_void_p), ('read_bin', c_void_p), ('bin_parts', c_void_p)]


C_LIB.adapterDemuxReadsDevice.argtypes = [c_void_p, c_void_p, c_int64, c_int64, c_int64, POINTER(TrimArgsDesc),
                                          POINTER(SplitArgsDesc), POINTER(DemuxArgsDesc), c_int, c_int, c_int, c_int, c_void_p]
C_LIB.adapterDemuxReadsDevice.restype = c_int


class EmitArgsDesc(Structure):
    """pb200_emit_args_t (include/porechop_b200.h)"""
    _fields_ = [('d_seq', c_void_p), ('d_qual', c_void_p), ('seq_bytes', c_int64), ('d_off', c_void_p), ('d_read', c_void_p),
                ('d_part', c_void_p), ('d_names', c_void_p), ('d_name_off', c_void_p), ('n_reads', c_int64),
                ('name_bytes', c_int64), ('d_rna', c_void_p), ('fmt', c_int32), ('d_out', c_void_p), ('out_cap', c_int64),
                ('d_out_off', c_void_p), ('n_out_bytes', c_void_p)]


C_LIB.pb200EmitReadsDevice.argtypes = [POINTER(EmitArgsDesc), c_int64, c_void_p]
C_LIB.pb200EmitReadsDevice.restype = c_int


class ParseArgsDesc(Structure):
    """pb200_parse_args_t (include/porechop_b200.h)"""
    _fields_ = [('d_in', c_void_p), ('n_in', c_int64), ('fmt', c_int32), ('d_names', c_void_p), ('names_cap', c_int64),
                ('d_name_off', c_void_p), ('d_seq', c_void_p), ('seq_cap', c_int64), ('d_seq_off', c_void_p), ('d_qual', c_void_p),
                ('d_rna', c_void_p), ('reads_cap', c_int64), ('n_reads', c_void_p), ('n_name_bytes', c_void_p),
                ('n_seq_bytes', c_void_p), ('error', c_void_p), ('error_index', c_void_p)]


C_LIB.pb200ParseReadsDevice.argtypes = [POINTER(ParseArgsDesc), c_void_p]
C_LIB.pb200ParseReadsDevice.restype = c_int


class GzipArgsDesc(Structure):
    """pb200_gzip_args_t (include/porechop_b200.h)"""
    _fields_ = [('d_src', c_void_p), ('n', c_int64), ('seg_off', c_void_p), ('n_segs', c_int64), ('block', c_int32),
                ('d_out', c_void_p), ('out_cap', c_int64), ('out_seg_off', c_void_p), ('n_out_bytes', c_void_p)]


C_LIB.pb200GzipDevice.argtypes = [POINTER(GzipArgsDesc), c_void_p]
C_LIB.pb200GzipDevice.restype = c_int
C_LIB.pb200GzipBound.argtypes = [c_int64, c_int64, c_int32]
C_LIB.pb200GzipBound.restype = c_int64
C_LIB.pb200MiddleThresholdTable.argtypes = [c_double, c_int32, c_void_p]
C_LIB.pb200MiddleThresholdTable.restype = c_int
C_LIB.pb200FormatRecord.argtypes = [c_void_p, c_char_p, c_int]
C_LIB.pb200FormatRecord.restype = c_int
C_LIB.pb200DeviceCount.restype = c_int
C_LIB.pb200SetDevice.argtypes = [c_int]
C_LIB.pb200SetDevice.restype = c_int
C_LIB.pb200Synchronize.restype = c_int
C_LIB.pb200LastError.restype = c_char_p
C_LIB.pb200KernelLaunches.restype = c_longlong
C_LIB.pb200TimingEnable.argtypes = [c_int]
C_LIB.pb200TimingEnable.restype = None
C_LIB.pb200TimingRead.argtypes = [POINTER(c_double), POINTER(c_longlong), POINTER(c_double), c_int]
C_LIB.pb200TimingRead.restype = c_int
C_LIB.pb200TimingReadKinds.argtypes = [POINTER(c_double), POINTER(c_longlong), POINTER(c_double), c_int]
C_LIB.pb200TimingReadKinds.restype = c_int
C_LIB.pb200SetOption.argtypes = [c_char_p, c_char_p]
C_LIB.pb200SetOption.restype = c_int
C_LIB.pb200PackNibbles.argtypes = [c_void_p, c_int64, c_void_p, c_int]
C_LIB.pb200PackNibbles.restype = c_int

EXPORTED_SYMBOLS = ['adapterAlignment', 'freeCString', 'adapterAlignmentBatch', 'adapterAlignmentBatchMulti',
                    'adapterAlignmentBatchDevice', 'adapterEndDecisions', 'pb200TrimThresholdTable', 'adapterSetSearch',
                    'adapterMiddleScan',
                    'adapterMiddleScanDevice', 'pb200MiddleThresholdTable', 'adapterTrimReads', 'adapterTrimReadsDevice',
                    'adapterTrimSplitReadsDevice', 'adapterDemuxReadsDevice', 'pb200EmitReadsDevice', 'pb200ParseReadsDevice', 'pb200GzipDevice', 'pb200GzipBound', 'pb200FormatRecord', 'pb200DeviceCount', 'pb200SetDevice', 'pb200Synchronize', 'pb200LastError',
                    'pb200KernelLaunches', 'pb200TimingEnable', 'pb200TimingRead', 'pb200TimingReadKinds', 'pb200SetOption',
                    'pb200GetOption', 'pb200HostBuffer', 'pb200PackNibbles']

RECORD_INTS = 9
HIT_INTS = 10                 # adapterMiddleScan: {adapter index, 9-int record}
SCORE_EMPTY = -2147483648
ERR_ARG, ERR_SPACE = 102, 104


class EngineError(RuntimeError):
    code = None               # the PB200_ERR_* code of a failed engine call


def _check(rc):
    if rc != 0:
        e = EngineError('porechop_b200 engine error %d: %s' % (rc, C_LIB.pb200LastError().decode()))
        e.code = rc
        raise e


def adapter_alignment(read_sequence, adapter_sequence, scoring_scheme_vals):
    """
    Python wrapper for the adapterAlignment C function (same contract as the reference,
    cpp_function_wrappers.py:42-53): returns 'rs,re,as,ae,score,aligned%ID,full%ID'.
    """
    match_score = scoring_scheme_vals[0]
    mismatch_score = scoring_scheme_vals[1]
    gap_open_score = scoring_scheme_vals[2]
    gap_extend_score = scoring_scheme_vals[3]
    ptr = C_LIB.adapterAlignment(read_sequence.encode('utf-8'), adapter_sequence.encode('utf-8'),
                                 match_score, mismatch_score, gap_open_score, gap_extend_score)
    if not ptr:
        raise EngineError('porechop_b200: adapterAlignment failed: ' + C_LIB.pb200LastError().decode())
    return c_string_to_python_string(ptr)


def c_string_to_python_string(c_string):
    """
    Casts a C string to a Python string and then frees the C string (reference lines 56-63).
    """
    python_string = cast(c_string, c_char_p).value.decode()
    C_LIB.freeCString(c_string)
    return python_string


# ---------------------------------------------------------------------------------------------------------
def pack_sequences(seqs, offset_dtype=np.int64):
    """list of str/bytes -> (uint8 buffer, offsets[n+1]).  No per-base Python work (one join + frombuffer)."""
    bs = [s.encode('ascii', 'replace') if isinstance(s, str) else bytes(s) for s in seqs]
    off = np.zeros(len(bs) + 1, dtype=offset_dtype)
    if bs:
        np.cumsum([len(b) for b in bs], out=off[1:])
    buf = np.frombuffer(b''.join(bs), dtype=np.uint8) if bs and off[-1] else np.zeros(0, dtype=np.uint8)
    return np.ascontiguousarray(buf), off


def _ptr(a):
    return a.ctypes.data_as(c_void_p) if a is not None else None


def adapter_alignment_batch(seq_buf, seq_off, ad_buf, ad_off, scoring_scheme_vals, pair_seq=None, pair_adapter=None,
                            out=None):
    """
    Batched alignment through the C-ABI with HOST buffers (numpy arrays; pinned memory works too if the
    arrays wrap it).  seq_buf/ad_buf: uint8, seq_off: int64[n_seqs+1], ad_off: int32[n_adapters+1].
    pair_seq/pair_adapter: int32[n_pairs] or both None for the full cross product (sequence-major).
    Returns int32[n_pairs, 9] records (see include/porechop_b200.h).
    """
    seq_buf = np.ascontiguousarray(seq_buf, dtype=np.uint8)
    ad_buf = np.ascontiguousarray(ad_buf, dtype=np.uint8)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.int64)
    ad_off = np.ascontiguousarray(ad_off, dtype=np.int32)
    n_seqs, n_ad = len(seq_off) - 1, len(ad_off) - 1
    if pair_seq is None:
        n_pairs = n_seqs * n_ad
    else:
        pair_seq = np.ascontiguousarray(pair_seq, dtype=np.int32)
        pair_adapter = np.ascontiguousarray(pair_adapter, dtype=np.int32)
        n_pairs = len(pair_seq)
    if out is None:
        out = np.empty((n_pairs, RECORD_INTS), dtype=np.int32)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    _check(C_LIB.adapterAlignmentBatch(_ptr(seq_buf), _ptr(seq_off), n_seqs, _ptr(ad_buf), _ptr(ad_off), n_ad,
                                       _ptr(pair_seq), _ptr(pair_adapter), n_pairs, ma, mi, go, ge, _ptr(out)))
    return out


def adapter_alignment_batch_multi(batches, scoring_scheme_vals):
    """
    Several cross-product batches in one submit (adapterAlignmentBatchMulti): `batches` is a list of
    (seq_buf, seq_off, ad_buf, ad_off) or (seq_buf, seq_off, ad_buf, ad_off, out) tuples with the array conventions of
    adapter_alignment_batch.  Returns the list of int32[n_seqs * n_adapters, 9] record arrays, one per batch.
    """
    descs = (BatchDesc * max(len(batches), 1))()
    keep, outs = [], []
    for k, b in enumerate(batches):
        seq_buf = np.ascontiguousarray(b[0], dtype=np.uint8)
        seq_off = np.ascontiguousarray(b[1], dtype=np.int64)
        ad_buf = np.ascontiguousarray(b[2], dtype=np.uint8)
        ad_off = np.ascontiguousarray(b[3], dtype=np.int32)
        n_seqs, n_ad = len(seq_off) - 1, len(ad_off) - 1
        out = b[4] if len(b) > 4 and b[4] is not None else np.empty((n_seqs * n_ad, RECORD_INTS), dtype=np.int32)
        keep.append((seq_buf, seq_off, ad_buf, ad_off, out))
        outs.append(out)
        descs[k] = BatchDesc(seq_buf.ctypes.data, seq_off.ctypes.data, n_seqs, ad_buf.ctypes.data, ad_off.ctypes.data, n_ad,
                             out.ctypes.data)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    _check(C_LIB.adapterAlignmentBatchMulti(descs, len(batches), ma, mi, go, ge))
    return outs


def adapter_end_decisions(batches, scoring_scheme_vals, end_size, extra_trim_size, end_threshold, min_trim_size,
                          want_records=False, out_arrays=None, want_top2=False):
    """
    End-trim decisions on the device (adapterEndDecisions): `batches` is a list of
    (seq_buf, seq_off, ad_buf, ad_off, is_start, score_cols) -- windows x adapters, which trim rule, and the adapter
    indices whose full-adapter identity the host still needs (barcode columns; may be empty).
    Returns one (trim int32[n], pairs uint16[n, n_cols, 2], records or None) per batch.
    out_arrays: optional preallocated [(trim, pairs, records-or-None), ...] (e.g. views of pinned memory) to write into.
    want_top2: the barcode ranking stays on the device too -- the second element of every result is then int32[n, 6] =
    (position in score_cols, match_ad, len_ad) of the best and the second-best score column (determine_barcode's sorted order:
    identity descending, ties in score_cols order; position -1 = no such column) instead of the pairs of all columns.
    """
    descs = (EndBatchDesc * max(len(batches), 1))()
    keep, outs = [], []
    for k, b in enumerate(batches):
        seq_buf = np.ascontiguousarray(b[0], dtype=np.uint8)
        seq_off = np.ascontiguousarray(b[1], dtype=np.int64)
        ad_buf = np.ascontiguousarray(b[2], dtype=np.uint8)
        ad_off = np.ascontiguousarray(b[3], dtype=np.int32)
        cols = np.ascontiguousarray(b[5] if b[5] is not None else [], dtype=np.int32)
        n_seqs, n_ad = len(seq_off) - 1, len(ad_off) - 1
        if out_arrays is not None:
            trim, pairs, rec = out_arrays[k]
            assert trim.dtype == np.int32 and len(trim) == n_seqs and trim.flags.c_contiguous and pairs.flags.c_contiguous
            if want_top2:
                assert pairs.dtype == np.int32 and pairs.shape == (n_seqs, 6)
            else:
                assert pairs.dtype == np.uint16 and pairs.shape == (n_seqs, len(cols), 2)
        else:
            trim = np.zeros(n_seqs, dtype=np.int32)
            if want_top2:
                pairs = np.tile(np.array([-1, 0, 1], dtype=np.int32), (n_seqs, 2))
            else:
                pairs = np.zeros((n_seqs, len(cols), 2), dtype=np.uint16)
            rec = np.empty((n_seqs * n_ad, RECORD_INTS), dtype=np.int32) if want_records else None
        keep.append((seq_buf, seq_off, ad_buf, ad_off, cols))
        outs.append((trim, pairs, rec))
        descs[k] = EndBatchDesc(BatchDesc(seq_buf.ctypes.data, seq_off.ctypes.data, n_seqs, ad_buf.ctypes.data,
                                          ad_off.ctypes.data, n_ad, rec.ctypes.data if rec is not None else None),
                                1 if b[4] else 0, int(end_size), int(extra_trim_size), int(min_trim_size), float(end_threshold),
                                cols.ctypes.data if len(cols) else None, len(cols), trim.ctypes.data,
                                pairs.ctypes.data if (len(cols) and not want_top2) else None,
                                pairs.ctypes.data if (len(cols) and want_top2) else None)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    _check(C_LIB.adapterEndDecisions(descs, len(batches), ma, mi, go, ge))
    return outs


def adapter_set_search(batches, scoring_scheme_vals):
    """
    Phase A on the device (adapterSetSearch): `batches` is a list of (seq_buf, seq_off, ad_buf, ad_off) or
    (seq_buf, seq_off, ad_buf, ad_off, out) tuples with the array conventions of adapter_alignment_batch (`out`: an
    int32[n_seqs * n_adapters, 9] array that receives the records too).  Returns one float64[n_adapters] per batch: the
    best full-adapter identity of each adapter over the batch's windows, starting from 0.0, exactly as the reference's
    best_start_score / best_end_score.
    """
    descs = (SearchBatchDesc * max(len(batches), 1))()
    keep, bests = [], []
    for k, b in enumerate(batches):
        seq_buf = np.ascontiguousarray(b[0], dtype=np.uint8)
        seq_off = np.ascontiguousarray(b[1], dtype=np.int64)
        ad_buf = np.ascontiguousarray(b[2], dtype=np.uint8)
        ad_off = np.ascontiguousarray(b[3], dtype=np.int32)
        n_seqs, n_ad = len(seq_off) - 1, len(ad_off) - 1
        out = b[4] if len(b) > 4 else None
        if out is not None:
            assert out.dtype == np.int32 and out.size == n_seqs * n_ad * RECORD_INTS and out.flags.c_contiguous
        best = np.zeros(n_ad)
        keep.append((seq_buf, seq_off, ad_buf, ad_off, out))
        bests.append(best)
        descs[k] = SearchBatchDesc(BatchDesc(seq_buf.ctypes.data, seq_off.ctypes.data, n_seqs, ad_buf.ctypes.data,
                                             ad_off.ctypes.data, n_ad, out.ctypes.data if out is not None else None),
                                   best.ctypes.data)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    _check(C_LIB.adapterSetSearch(descs, len(batches), ma, mi, go, ge))
    return bests


def trim_threshold_table(end_threshold, length):
    """cmin[l] of pb200TrimThresholdTable: smallest match count whose float("%f") identity exceeds end_threshold."""
    t = np.zeros(length, dtype=np.int32)
    rc = C_LIB.pb200TrimThresholdTable(float(end_threshold), int(length), _ptr(t))
    if rc != 0:
        raise EngineError('pb200TrimThresholdTable: error %d' % rc)
    return t


def adapter_alignment_batch_device(d_seqs_ptr, d_seq_off_ptr, n_seqs, total_seq_bytes, max_seq_len, ad_buf, ad_off,
                                   scoring_scheme_vals, d_out_ptr, stream_ptr=0):
    """Cross-product batch with the bulk data already in device memory (raw device pointers as ints)."""
    ad_buf = np.ascontiguousarray(ad_buf, dtype=np.uint8)
    ad_off = np.ascontiguousarray(ad_off, dtype=np.int32)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    _check(C_LIB.adapterAlignmentBatchDevice(c_void_p(d_seqs_ptr), c_void_p(d_seq_off_ptr), n_seqs, total_seq_bytes,
                                             max_seq_len, _ptr(ad_buf), _ptr(ad_off), len(ad_off) - 1, ma, mi, go, ge,
                                             c_void_p(d_out_ptr), c_void_p(stream_ptr)))


def _middle_scan(call, n_seqs):
    """adapterMiddleScan(Device) with caller-owned outputs: starts with room for 2n + 1024 hits and retries once with exactly
    *n_total when the engine answers PB200_ERR_SPACE."""
    n_hits = np.zeros(n_seqs, dtype=np.int32)
    total = c_int64(0)
    cap = 2 * n_seqs + 1024
    for _ in range(2):
        hits = np.empty((cap, HIT_INTS), dtype=np.int32)
        rc = call(_ptr(n_hits), _ptr(hits), cap, byref(total))
        if rc == ERR_SPACE and total.value > cap:
            cap = total.value
            continue
        _check(rc)
        return n_hits, hits[:total.value]
    _check(rc)


def adapter_middle_scan(seq_buf, seq_off, ad_buf, ad_off, scoring_scheme_vals, middle_threshold):
    """
    Porechop's Phase C on the device (adapterMiddleScan): every hit of every sequence, masking rounds included.
    seq_buf / seq_off: the end-trimmed reads (uint8, int64[n+1]); ad_buf / ad_off: the adapters in the reference's order.
    Returns (n_hits int32[n], hits int32[total, 10]): hits are sequence-major, each sequence's in the order found, each
    {adapter index, 9-int record} -- hits[:, 1:] goes to scores_from_records / format_record as it is.
    """
    seq_buf = np.ascontiguousarray(seq_buf, dtype=np.uint8)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.int64)
    ad_buf = np.ascontiguousarray(ad_buf, dtype=np.uint8)
    ad_off = np.ascontiguousarray(ad_off, dtype=np.int32)
    n_seqs, n_ad = len(seq_off) - 1, len(ad_off) - 1
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    return _middle_scan(lambda nh, h, cap, total: C_LIB.adapterMiddleScan(
        _ptr(seq_buf), _ptr(seq_off), n_seqs, _ptr(ad_buf), _ptr(ad_off), n_ad, ma, mi, go, ge, float(middle_threshold), nh, h,
        cap, total), n_seqs)


def adapter_middle_scan_device(d_seqs_ptr, d_seq_off_ptr, n_seqs, total_seq_bytes, max_seq_len, ad_buf, ad_off,
                               scoring_scheme_vals, middle_threshold, stream_ptr=0):
    """adapter_middle_scan with the reads already in device memory (raw device pointers as ints, the conventions of
    adapter_alignment_batch_device).  The caller's device buffers are not modified."""
    ad_buf = np.ascontiguousarray(ad_buf, dtype=np.uint8)
    ad_off = np.ascontiguousarray(ad_off, dtype=np.int32)
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    return _middle_scan(lambda nh, h, cap, total: C_LIB.adapterMiddleScanDevice(
        c_void_p(d_seqs_ptr), c_void_p(d_seq_off_ptr), n_seqs, total_seq_bytes, max_seq_len, _ptr(ad_buf), _ptr(ad_off),
        len(ad_off) - 1, ma, mi, go, ge, float(middle_threshold), nh, h, cap, total, c_void_p(stream_ptr)), int(n_seqs))


def _trim_reads(call, n_seqs, start, end, middle, end_size, extra_trim_size, end_threshold, min_trim_size, middle_threshold,
                want_top2, want_scores=True):
    """adapterTrimReads(Device) with caller-owned outputs: builds pb200_trim_args_t, starts with room for 2n + 1024 hits and
    retries once with exactly *n_total when the engine answers PB200_ERR_SPACE (as _middle_scan).  want_scores=False: no
    score output at all (the demux stage ranks the columns on the device); the scores are then returned as None."""
    keep, sides, outs = [], [], []
    for ad_buf, ad_off, cols in (start, end):
        ad_buf = np.ascontiguousarray(ad_buf, dtype=np.uint8)
        ad_off = np.ascontiguousarray(ad_off, dtype=np.int32)
        cols = np.ascontiguousarray(cols if cols is not None else [], dtype=np.int32)
        trim = np.zeros(n_seqs, dtype=np.int32)
        if want_top2:
            scores = np.tile(np.array([-1, 0, 1], dtype=np.int32), (n_seqs, 2))
        else:
            scores = np.zeros((n_seqs, len(cols), 2), dtype=np.uint16)
        keep.append((ad_buf, ad_off, cols))
        outs.append((trim, scores))
        give = len(cols) and want_scores
        sides.append(TrimSideDesc(ad_buf.ctypes.data, ad_off.ctypes.data, len(ad_off) - 1, cols.ctypes.data if len(cols) else None,
                                  len(cols), trim.ctypes.data, scores.ctypes.data if (give and not want_top2) else None,
                                  scores.ctypes.data if (give and want_top2) else None))
    if middle is not None:
        mid_buf = np.ascontiguousarray(middle[0], dtype=np.uint8)
        mid_off = np.ascontiguousarray(middle[1], dtype=np.int32)
    else:
        mid_buf, mid_off = np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int32)
    n_hits = np.zeros(n_seqs, dtype=np.int32)
    total = c_int64(0)
    cap = 2 * n_seqs + 1024
    for _ in range(2):
        hits = np.empty((cap, HIT_INTS), dtype=np.int32)
        args = TrimArgsDesc(int(end_size), int(extra_trim_size), int(min_trim_size), float(end_threshold), sides[0], sides[1],
                            mid_buf.ctypes.data, mid_off.ctypes.data, len(mid_off) - 1, float(middle_threshold),
                            n_hits.ctypes.data, hits.ctypes.data, cap, addressof(total))
        rc = call(byref(args))
        if rc == ERR_SPACE and total.value > cap:
            cap = total.value
            continue
        break
    _check(rc)
    (st, ss), (et, es) = outs
    if not want_scores:
        ss = es = None
    return st, et, ss, es, n_hits, hits[:total.value]


def adapter_trim_reads(seq_buf, seq_off, start, end, middle, scoring_scheme_vals, end_size, extra_trim_size, end_threshold,
                       min_trim_size, middle_threshold=85.0, want_top2=False):
    """
    Porechop's Phase B and Phase C on whole reads in one engine call (adapterTrimReads): the end windows are cut, the trims
    decided, and the trimmed reads scanned for middle adapters on the device; the reads are uploaded once.
    seq_buf / seq_off: the reads (uint8, int64[n+1]).  start / end: (ad_buf, ad_off, score_cols) of find_start_trim /
    find_end_trim (ad_off int32; no adapters = the side is not searched); middle: (ad_buf, ad_off) of the middle adapters in
    the reference's order, or None (--no_split).
    Returns (start_trim int32[n], end_trim int32[n], start scores, end scores, n_hits int32[n], hits int32[total, 10]): the
    scores are the score pairs uint16[n, n_cols, 2] of adapter_end_decisions, or with want_top2 its int32[n, 6] ranking; the
    hits are those of adapter_middle_scan on seq[start_trim : len - end_trim].
    """
    seq_buf = np.ascontiguousarray(seq_buf, dtype=np.uint8)
    seq_off = np.ascontiguousarray(seq_off, dtype=np.int64)
    n_seqs = len(seq_off) - 1
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    return _trim_reads(lambda args: C_LIB.adapterTrimReads(_ptr(seq_buf), _ptr(seq_off), n_seqs, args, ma, mi, go, ge), n_seqs,
                       start, end, middle, end_size, extra_trim_size, end_threshold, min_trim_size, middle_threshold, want_top2)


def adapter_trim_reads_device(d_seqs_ptr, d_seq_off_ptr, n_seqs, total_seq_bytes, max_seq_len, start, end, middle,
                              scoring_scheme_vals, end_size, extra_trim_size, end_threshold, min_trim_size, middle_threshold=85.0,
                              want_top2=False, stream_ptr=0):
    """adapter_trim_reads with the reads already in device memory (raw device pointers as ints, the conventions of
    adapter_middle_scan_device).  The caller's device buffers are not modified."""
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    return _trim_reads(lambda args: C_LIB.adapterTrimReadsDevice(
        c_void_p(d_seqs_ptr), c_void_p(d_seq_off_ptr), n_seqs, total_seq_bytes, max_seq_len, args, ma, mi, go, ge,
        c_void_p(stream_ptr)), int(n_seqs), start, end, middle, end_size, extra_trim_size, end_threshold, min_trim_size,
        middle_threshold, want_top2)


def adapter_trim_split_reads_device(d_seqs_ptr, d_seq_off_ptr, n_seqs, total_seq_bytes, max_seq_len, start, end, middle,
                                    scoring_scheme_vals, end_size, extra_trim_size, end_threshold, min_trim_size,
                                    middle_threshold=85.0, want_top2=False, stream_ptr=0, *, d_quals_ptr=0, mid_extra=None,
                                    min_split_read_size=1000, discard_middle=False, untrimmed=False, d_out_seq_ptr=0,
                                    d_out_qual_ptr=0, d_out_off_ptr=0, d_out_read_ptr=0, d_out_part_ptr=0, parts_cap=0):
    """adapter_trim_reads_device, then Porechop's output records cut into caller-owned device buffers
    (adapterTrimSplitReadsDevice): bases (d_out_seq), qualities (d_out_qual, when d_quals is given), offsets int64[parts_cap + 1],
    source read and part number int32[parts_cap] (0 = not split, k >= 1 = the k-th part).  mid_extra: (left, right) per middle
    adapter -- the bases cut before and after a hit (None when there are no middle adapters).
    Returns the outputs of adapter_trim_reads_device plus (n_parts, n_out_bases).  When the records do not fit parts_cap it
    raises EngineError with code ERR_SPACE and the totals as .n_parts / .n_out_bases: the buffers are the caller's, so the
    caller allocates them again and repeats the call."""
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    n_mid = len(middle[1]) - 1 if middle is not None else 0
    left, right = mid_extra if mid_extra is not None else ([], [])
    left = np.ascontiguousarray(left, dtype=np.int32)
    right = np.ascontiguousarray(right, dtype=np.int32)
    if len(left) != n_mid or len(right) != n_mid:
        raise ValueError('mid_extra needs one (left, right) value per middle adapter')
    n_parts, n_bases = c_int64(0), c_int64(0)
    split = SplitArgsDesc(d_quals_ptr or None, left.ctypes.data if n_mid else None, right.ctypes.data if n_mid else None,
                          int(min_split_read_size), int(bool(discard_middle)), int(bool(untrimmed)), d_out_seq_ptr or None,
                          d_out_qual_ptr or None, d_out_off_ptr or None, d_out_read_ptr or None, d_out_part_ptr or None,
                          int(parts_cap), addressof(n_parts), addressof(n_bases))
    try:
        out = _trim_reads(lambda args: C_LIB.adapterTrimSplitReadsDevice(
            c_void_p(d_seqs_ptr), c_void_p(d_seq_off_ptr), n_seqs, total_seq_bytes, max_seq_len, args, byref(split), ma, mi, go,
            ge, c_void_p(stream_ptr)), int(n_seqs), start, end, middle, end_size, extra_trim_size, end_threshold, min_trim_size,
            middle_threshold, want_top2)
    except EngineError as e:
        e.n_parts, e.n_out_bases = n_parts.value, n_bases.value
        raise
    return out + (n_parts.value, n_bases.value)


def adapter_demux_reads_device(d_seqs_ptr, d_seq_off_ptr, n_seqs, total_seq_bytes, max_seq_len, start, end, middle,
                               scoring_scheme_vals, end_size, extra_trim_size, end_threshold, min_trim_size, middle_threshold=85.0,
                               stream_ptr=0, *, start_bin, end_bin, n_bins, barcode_threshold=75.0, barcode_diff=5.0,
                               require_two_barcodes=False, discard_unassigned=False, d_albacore_ptr=0, d_quals_ptr=0,
                               mid_extra=None, min_split_read_size=1000, discard_middle=False, untrimmed=False, d_out_seq_ptr=0,
                               d_out_qual_ptr=0, d_out_off_ptr=0, d_out_read_ptr=0, d_out_part_ptr=0, parts_cap=0):
    """adapter_trim_split_reads_device plus the barcode call of every read, with the records grouped by bin
    (adapterDemuxReadsDevice).  start_bin / end_bin: the bin id of each start / end score column (start[2] / end[2]), bins
    0 .. n_bins - 1 named, n_bins = 'none'; d_albacore_ptr: int32 per read on the device (-1 = no Albacore call), or 0.
    Returns (start_trim, end_trim, n_hits, hits, n_parts, n_out_bases, read_bin int32[n], bin_parts int64[n_bins + 2]): the
    records of bin b are bin_parts[b] .. bin_parts[b + 1].  When the kept records do not fit parts_cap it raises EngineError
    with code ERR_SPACE and the totals as .n_parts / .n_out_bases (read_bin / bin_parts as .read_bin / .bin_parts)."""
    ma, mi, go, ge = [int(x) for x in scoring_scheme_vals]
    n_mid = len(middle[1]) - 1 if middle is not None else 0
    left, right = mid_extra if mid_extra is not None else ([], [])
    left = np.ascontiguousarray(left, dtype=np.int32)
    right = np.ascontiguousarray(right, dtype=np.int32)
    if len(left) != n_mid or len(right) != n_mid:
        raise ValueError('mid_extra needs one (left, right) value per middle adapter')
    start_bin = np.ascontiguousarray(start_bin, dtype=np.int32)
    end_bin = np.ascontiguousarray(end_bin, dtype=np.int32)
    read_bin = np.zeros(int(n_seqs), dtype=np.int32)
    bin_parts = np.zeros(int(n_bins) + 2, dtype=np.int64)
    n_parts, n_bases = c_int64(0), c_int64(0)
    split = SplitArgsDesc(d_quals_ptr or None, left.ctypes.data if n_mid else None, right.ctypes.data if n_mid else None,
                          int(min_split_read_size), int(bool(discard_middle)), int(bool(untrimmed)), d_out_seq_ptr or None,
                          d_out_qual_ptr or None, d_out_off_ptr or None, d_out_read_ptr or None, d_out_part_ptr or None,
                          int(parts_cap), addressof(n_parts), addressof(n_bases))
    demux = DemuxArgsDesc(start_bin.ctypes.data if len(start_bin) else None, end_bin.ctypes.data if len(end_bin) else None,
                          int(n_bins), float(barcode_threshold), float(barcode_diff), int(bool(require_two_barcodes)),
                          int(bool(discard_unassigned)), d_albacore_ptr or None, read_bin.ctypes.data, bin_parts.ctypes.data)
    try:
        st, et, _, _, n_hits, hits = _trim_reads(lambda args: C_LIB.adapterDemuxReadsDevice(
            c_void_p(d_seqs_ptr), c_void_p(d_seq_off_ptr), n_seqs, total_seq_bytes, max_seq_len, args, byref(split), byref(demux),
            ma, mi, go, ge, c_void_p(stream_ptr)), int(n_seqs), start, end, middle, end_size, extra_trim_size, end_threshold,
            min_trim_size, middle_threshold, False, want_scores=False)
    except EngineError as e:
        e.n_parts, e.n_out_bases, e.read_bin, e.bin_parts = n_parts.value, n_bases.value, read_bin, bin_parts
        raise
    return st, et, n_hits, hits, n_parts.value, n_bases.value, read_bin, bin_parts


def pb200_emit_reads_device(n_rec, *, d_seq_ptr, d_qual_ptr, seq_bytes, d_off_ptr, d_read_ptr, d_part_ptr, d_names_ptr,
                            d_name_off_ptr, n_reads, name_bytes, d_rna_ptr=0, fmt='fastq', d_out_ptr=0, out_cap=0,
                            d_out_off_ptr=0, stream_ptr=0):
    """The bytes Porechop writes for n_rec records in device memory (pb200EmitReadsDevice): record r is
    seq[off[r] .. off[r + 1]) with its qualities, source read read[r] and part number part[r]; the output goes to d_out
    (out_cap bytes) and the record byte offsets to d_out_off (int64[n_rec + 1]).  fmt: 'fastq' or 'fasta'.
    Returns the number of bytes written.  When they do not fit out_cap it raises EngineError with code ERR_SPACE and the
    total as .n_out_bytes (d_out_off is then valid)."""
    if fmt not in ('fastq', 'fasta'):
        raise ValueError("fmt must be 'fastq' or 'fasta'")
    n_out = c_int64(0)
    args = EmitArgsDesc(d_seq_ptr or None, d_qual_ptr or None, int(seq_bytes), d_off_ptr or None, d_read_ptr or None,
                        d_part_ptr or None, d_names_ptr or None, d_name_off_ptr or None, int(n_reads), int(name_bytes),
                        d_rna_ptr or None, 0 if fmt == 'fastq' else 1, d_out_ptr or None, int(out_cap), d_out_off_ptr or None,
                        addressof(n_out))
    try:
        _check(C_LIB.pb200EmitReadsDevice(byref(args), int(n_rec), c_void_p(stream_ptr)))
    except EngineError as e:
        e.n_out_bytes = n_out.value
        raise
    return n_out.value


# reason codes of pb200ParseReadsDevice (PB200_PARSE_*)
PARSE_LINES, PARSE_HEADER, PARSE_FASTA_START, PARSE_FASTA_NAME, PARSE_LONG_QUAL = 1, 2, 3, 4, 5


def pb200_parse_reads_device(d_in_ptr, n_in, fmt='fastq', *, d_names_ptr=0, names_cap=0, d_name_off_ptr=0, d_seq_ptr=0, seq_cap=0,
                             d_seq_off_ptr=0, d_qual_ptr=0, d_rna_ptr=0, reads_cap=0, stream_ptr=0):
    """The reads of n_in FASTQ / FASTA bytes in device memory (pb200ParseReadsDevice) into caller-owned device buffers: names
    (names_cap bytes) at name_off (int64[reads_cap + 1]), bases (seq_cap bytes) and, with d_qual_ptr, qualities at seq_off
    (int64[reads_cap + 1]), and one RNA flag (uint8) per read.  fmt: 'fastq' or 'fasta'.
    Returns (n_reads, name bytes, bases).  When they do not fit it raises EngineError with code ERR_SPACE and the exact counts as
    .n_reads / .n_name_bytes / .n_seq_bytes; malformed input raises EngineError with code ERR_ARG, .reason (PARSE_*) and .index
    (the first bad record or line)."""
    if fmt not in ('fastq', 'fasta'):
        raise ValueError("fmt must be 'fastq' or 'fasta'")
    outs = [c_int64(0) for _ in range(3)]
    err, err_index = c_int32(0), c_int64(-1)
    args = ParseArgsDesc(d_in_ptr or None, int(n_in), 0 if fmt == 'fastq' else 1, d_names_ptr or None, int(names_cap),
                         d_name_off_ptr or None, d_seq_ptr or None, int(seq_cap), d_seq_off_ptr or None, d_qual_ptr or None,
                         d_rna_ptr or None, int(reads_cap), *(addressof(x) for x in outs), addressof(err), addressof(err_index))
    try:
        _check(C_LIB.pb200ParseReadsDevice(byref(args), c_void_p(stream_ptr)))
    except EngineError as e:
        e.n_reads, e.n_name_bytes, e.n_seq_bytes = (x.value for x in outs)
        e.reason, e.index = err.value, err_index.value
        raise
    return tuple(x.value for x in outs)


def gzip_bound(n, n_segs=1, block=0):
    """the most bytes pb200_gzip_device writes for n bytes in n_segs segments with this block size (pb200GzipBound)"""
    b = C_LIB.pb200GzipBound(int(n), int(n_segs), int(block))
    if b < 0:
        raise ValueError('n must be >= 0, n_segs >= 1 and block 0 or 4096 .. 131072')
    return b


def pb200_gzip_device(d_src_ptr, n, seg_off=None, *, block=0, d_out_ptr=0, out_cap=0, stream_ptr=0):
    """gzip members of n bytes in device memory (pb200GzipDevice) into d_out (out_cap bytes): seg_off (int64[n_segs + 1],
    ascending from 0 to n; None = one segment) partitions the input into files, each cut into members of `block` bytes
    (0 = the default).  Returns (total bytes, int64 array of the segments' byte offsets in d_out).  When they do not fit
    out_cap it raises EngineError with code ERR_SPACE, the total as .n_out_bytes and the offsets as .out_seg_off."""
    seg = np.ascontiguousarray(np.array([0, n] if seg_off is None else seg_off, dtype=np.int64))
    out_off = np.zeros(max(len(seg), 1), dtype=np.int64)
    n_out = c_int64(0)
    args = GzipArgsDesc(d_src_ptr or None, int(n), _ptr(seg), len(seg) - 1, int(block), d_out_ptr or None, int(out_cap),
                        _ptr(out_off), addressof(n_out))
    try:
        _check(C_LIB.pb200GzipDevice(byref(args), c_void_p(stream_ptr)))
    except EngineError as e:
        e.n_out_bytes, e.out_seg_off = n_out.value, out_off
        raise
    return n_out.value, out_off


def middle_threshold_table(middle_threshold, length):
    """cmin[l] of pb200MiddleThresholdTable: smallest match count whose float("%f") identity reaches middle_threshold."""
    t = np.zeros(length, dtype=np.int32)
    rc = C_LIB.pb200MiddleThresholdTable(float(middle_threshold), int(length), _ptr(t))
    if rc != 0:
        raise EngineError('pb200MiddleThresholdTable: error %d' % rc)
    return t


def synchronize():
    _check(C_LIB.pb200Synchronize())


def format_record(rec):
    """One 9-int record -> the reference result string."""
    rec = np.ascontiguousarray(rec, dtype=np.int32)
    buf = create_string_buffer(96)
    n = C_LIB.pb200FormatRecord(_ptr(rec), buf, 96)
    if n < 0:
        raise EngineError('format failed')
    return buf.value.decode()


def device_count():
    return int(C_LIB.pb200DeviceCount())


def kernel_launches():
    return int(C_LIB.pb200KernelLaunches())


def timing_enable(on=True):
    C_LIB.pb200TimingEnable(1 if on else 0)


def timing_read(reset=True):
    ms, n, cells = c_double(0), c_longlong(0), c_double(0)
    _check(C_LIB.pb200TimingRead(ms, n, cells, 1 if reset else 0))
    return ms.value, n.value


TIMING_KINDS = ('trace_kernel', 'trace_kernel<score-only>', 'trace_kernel<window pass>', 'score_kernel')


def timing_read_kinds(reset=True):
    """{kind: {'ms': total CUDA-event ms, 'n': launches[, 'cells': DP cells of the window pass]}} of the timed DP launches"""
    ms, n, wc = (c_double * 4)(), (c_longlong * 4)(), c_double(0)
    _check(C_LIB.pb200TimingReadKinds(ms, n, wc, 1 if reset else 0))
    out = {}
    for k, name in enumerate(TIMING_KINDS):
        if n[k]:
            out[name] = {'ms': ms[k], 'n': int(n[k])}
            if k == 2:
                out[name]['cells'] = wc.value
    return out


def pack_nibbles(ascii_buf, threads=0):
    """uint8 ASCII bases -> uint8[(n+1)//2], two 4-bit Dna5 codes per byte (the host half of option h2d_pack)."""
    a = np.ascontiguousarray(ascii_buf, dtype=np.uint8)
    out = np.zeros((len(a) + 1) // 2, dtype=np.uint8)
    _check(C_LIB.pb200PackNibbles(_ptr(a), len(a), _ptr(out), int(threads)))
    return out


def set_option(name, value):
    _check(C_LIB.pb200SetOption(name.encode(), str(value).encode()))


def pinned_buffer(slot, nbytes):
    """uint8[nbytes] view of the library's pinned staging buffer `slot` (pb200HostBuffer), or None without a device.  The
    view is valid until the next call for the same slot."""
    import ctypes
    C_LIB.pb200HostBuffer.argtypes = [c_int, ctypes.c_size_t]
    C_LIB.pb200HostBuffer.restype = c_void_p
    p = C_LIB.pb200HostBuffer(int(slot), int(max(nbytes, 1)))
    if not p:
        return None
    return np.ctypeslib.as_array(cast(p, POINTER(ctypes.c_uint8)), shape=(int(max(nbytes, 1)),))[:int(nbytes)]


def get_option(name):
    """current integer value of a tunable (pb200GetOption); 'h2d_pack_large_submit' = what h2d_pack=auto resolves to here"""
    C_LIB.pb200GetOption.argtypes = [c_char_p]
    C_LIB.pb200GetOption.restype = c_int
    return int(C_LIB.pb200GetOption(name.encode()))
