/*
 * include/porechop_b200.h -- C-ABI of the H100 adapter-alignment engine (cpp_functions.so).
 *
 * Drop-in boundary (SURVEY.md 8(b)): the library is loaded by ctypes exactly like the reference's
 * porechop/cpp_functions.so (porechop/cpp_function_wrappers.py:21-39) and exports the reference's two
 * symbols with the same signatures, ownership and string format, plus a batched entry point so that the
 * host can submit every (read window, adapter) / (full read, adapter) pair in one call.
 *
 * Plain C types only (no torch / CUDA types): pointers, sizes, ints.  Every call runs on the CUDA
 * device that is current for the calling thread (cudaSetDevice / torch.cuda.set_device /
 * pb200SetDevice); there is NO CPU fallback -- without a usable sm_90 (H100) device the batch calls return
 * PB200_ERR_NO_DEVICE and adapterAlignment() returns NULL after printing the reason to stderr.
 */
#ifndef PORECHOP_B200_H
#define PORECHOP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- reference ABI, unchanged -------------------------------------------------------------------
 * replaces porechop/include/adapter_align.h:13-14 (implemented in porechop/src/adapter_align.cpp:11-31).
 * readSeq / adapterSeq: NUL-terminated ASCII, borrowed for the call.  Returns a malloc'd NUL-terminated
 * string "readStart,readEnd,adapterStart,adapterEnd,rawScore,alignedRegion%ID,fullAdapter%ID"
 * (ints "%d", doubles "%f"; ends are inclusive 0-based; "-1,0,-1,0,-2147483648,0.000000,0.000000" for an
 * empty read or adapter).  Ownership passes to the caller, who releases it with freeCString().
 * Thread-safe (calls are serialised on the device). */
char *adapterAlignment(char *readSeq, char *adapterSeq, int matchScore, int mismatchScore, int gapOpenScore,
                       int gapExtensionScore);

/* replaces porechop/include/adapter_align.h:15 (porechop/src/adapter_align.cpp:34-36): free(p). */
void freeCString(char *p);

/* ---- batched entry points (new; SURVEY.md 8(b) "new batch export") --------------------------------
 * One record of 9 int32 per alignment:
 *   {readStart, readEnd, adapterStart, adapterEnd, rawScore, matchAligned, lenAligned, matchAdapter, lenAdapter}
 * alignedRegion%ID = 100.0*matchAligned/lenAligned and fullAdapter%ID = 100.0*matchAdapter/lenAdapter in
 * double, exactly the two divisions of porechop/src/alignment.cpp:82,90; an empty read or adapter gives
 * {-1,0,-1,0,INT32_MIN,0,0,0,0}.  pb200FormatRecord() turns a record into the reference string.
 *
 * seqs/seq_off   : concatenated ASCII reads (or read windows); sequence s is seqs[seq_off[s] .. seq_off[s+1])
 * adapters/ad_off: concatenated ASCII adapters, same convention (int32 offsets)
 * pair_seq/pair_adapter (n_pairs each): the alignments to compute; both NULL = the full cross product in
 *                  sequence-major order (n_pairs must equal n_seqs*n_adapters, record p = s*n_adapters + a)
 * out            : n_pairs * 9 int32, caller-owned
 * Returns 0 on success or a PB200_ERR_* code (pb200LastError() has the text).  Host pointers; pinned host
 * memory lets the internal host<->device copies overlap with the kernels. */
int adapterAlignmentBatch(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
                          const int32_t *ad_off, int32_t n_adapters, const int32_t *pair_seq,
                          const int32_t *pair_adapter, int64_t n_pairs, int matchScore, int mismatchScore,
                          int gapOpenScore, int gapExtensionScore, int32_t *out);

/* Several independent cross-product batches in ONE submit -- e.g. the two batches of Porechop's end-trim phase
 * (find_start_trim: start windows x start adapters, find_end_trim: end windows x end adapters,
 * porechop/nanopore_read.py:166-208) -- pipelined through the same ring of streams, so the upload of the second batch
 * overlaps the kernels of the first and the copy pipeline fills and drains once per submit instead of once per batch.
 * Each batch has the cross-product semantics of adapterAlignmentBatch (records in sequence-major order in its own
 * `out`); batches with no sequences or no adapters are skipped.  Same scoring scheme for all batches. */
typedef struct {
    const uint8_t *seqs; const int64_t *seq_off; int64_t n_seqs;        /* as in adapterAlignmentBatch */
    const uint8_t *adapters; const int32_t *ad_off; int32_t n_adapters;
    int32_t *out;                                                       /* n_seqs * n_adapters * 9 int32 */
} pb200_batch_t;
int adapterAlignmentBatchMulti(const pb200_batch_t *batches, int n_batches, int matchScore, int mismatchScore,
                               int gapOpenScore, int gapExtensionScore);

/* End-trim DECISIONS on the device (SURVEY.md 8(f) row 3).  Each batch is one cross product of read-end windows x
 * adapters (as in adapterAlignmentBatchMulti); the 9-int records stay on the device and a second kernel reduces them per
 * read to what Porechop's host logic consumes:
 *   trim[s]         find_start_trim / find_end_trim (porechop/nanopore_read.py:166-208): the largest trim amount over the
 *                   adapters whose alignment passes `aligned-region identity > end_threshold`, the end_size / 0 edge test
 *                   and `read_end - read_start >= min_trim_size`; 0 when none passes
 *   score_pairs     for every adapter index listed in score_cols (the barcode adapters, nanopore_read.py:181-183,
 *                   203-205): (matchAdapter, lenAdapter) as two uint16 -- full-adapter identity =
 *                   float("%f" % (100.0 * matchAdapter / lenAdapter)) on the host; a failed alignment gives (0, 1) = 0.0
 * so 4 + 4*n_score_cols bytes per read come back instead of 36 per alignment.  The identity test is exact: the host
 * builds, with the reference's own snprintf("%f") / strtod chain, the smallest passing match count per aligned length
 * (pb200TrimThresholdTable) and the kernel compares integers.  end_threshold must be >= 0.  batch.out may be NULL (records
 * not copied back) or a buffer for the full records. */
typedef struct {
    pb200_batch_t batch;
    int32_t is_start;                 /* 1 = find_start_trim rule (start windows), 0 = find_end_trim rule (end windows) */
    int32_t end_size;                 /* --end_size (porechop.py:130), the window length the edge tests refer to */
    int32_t extra_trim_size;          /* --extra_end_trim */
    int32_t min_trim_size;            /* --min_trim_size */
    double end_threshold;             /* --end_threshold */
    const int32_t *score_cols;        /* adapter indices whose full-adapter identity is wanted (may be NULL if none) */
    int32_t n_score_cols;
    int32_t *trim;                    /* out: n_seqs */
    uint16_t *score_pairs;            /* out: n_seqs * n_score_cols * 2; may be NULL when only top2 is wanted */
    int32_t *top2;                    /* out, optional (NULL = not wanted): n_seqs * 6 = {position, matchAdapter, lenAdapter}
                                       * of the best and of the second-best score column -- the first two entries of
                                       * determine_barcode's `sorted(scores.items(), reverse=True, key=score)`
                                       * (porechop/nanopore_read.py:404-415): highest full-adapter identity first, equal
                                       * identities in score_cols order; `position` indexes score_cols (-1, 0, 1 when
                                       * there are fewer columns).  The caller lists each barcode NAME once in score_cols
                                       * (the reference's dict keeps a repeated name's last value).  24 bytes per read
                                       * instead of 4*n_score_cols. */
} pb200_end_batch_t;
int adapterEndDecisions(const pb200_end_batch_t *batches, int n_batches, int matchScore, int mismatchScore,
                        int gapOpenScore, int gapExtensionScore);
/* cmin[l], l = 0 .. len-1: the smallest match count c for which float("%f" % (100.0*c/l)) > end_threshold, or l+1 if
 * none does (cmin[0] = INT32_MAX: 0/0 is NaN and never passes).  Pure host code. */
int pb200TrimThresholdTable(double end_threshold, int32_t len, int32_t *cmin);

/* Phase A of Porechop on the device: the adapter-set search (find_matching_adapter_sets, porechop.py:286-327, and
 * NanoporeRead.align_adapter_set, nanopore_read.py:149-164).  Each batch is one cross product of read-end windows x adapter
 * sequences (as in adapterAlignmentBatchMulti); the records stay on the device and a second kernel reduces them per adapter,
 * so 8 bytes per adapter come back per submit instead of 36 per alignment:
 *   best[a]  the value the reference leaves in best_start_score / best_end_score: 0.0, max'd (Python's max) with
 *            float("%f" % fullAdapter%ID) of every alignment of adapter a in the batch.  A failed alignment (an empty
 *            window included) contributes 0.0; a record with lenAdapter == 0 would be NaN, which never raises the maximum.
 * The reduction is exact: the record with the largest 100.0*matchAdapter/lenAdapter in double gives the largest float, and
 * the host formats that one with the reference's own snprintf("%f") / strtod chain.  Start windows x start sequences and end
 * windows x end sequences go in one call as two batches.  A batch with n_seqs == 0 gives all 0.0; a batch with
 * n_adapters == 0 is skipped (best is not touched).  batch.out may be NULL (records not copied back) or a buffer for the full
 * records.  No preconditions beyond those of adapterAlignmentBatch: long windows (two-pass path) and scoring schemes of the
 * generic int32 kernel are taken too. */
typedef struct {
    pb200_batch_t batch;   /* one cross product, as in adapterAlignmentBatchMulti; batch.out may be NULL */
    double *best;          /* out: batch.n_adapters values */
} pb200_search_batch_t;
int adapterSetSearch(const pb200_search_batch_t *batches, int n_batches, int matchScore, int mismatchScore,
                     int gapOpenScore, int gapExtensionScore);

/* Same, with the bulk data already resident in device memory (d_seqs, d_seq_off, d_out are device pointers on
 * the current device; adapters/ad_off stay host pointers -- a few KB).  Cross-product mode only.
 * max_seq_len: length of the longest sequence, or -1 to let the library compute it on the device.
 * The work is enqueued on `stream` (a cudaStream_t passed as void*) and the call returns after enqueueing everything
 * unless the score pass needs a host decision; call cudaStreamSynchronize / torch.cuda.synchronize before reading d_out.
 * The reads must be in place when `stream` reaches the call: work the caller queued on `stream` before the call is
 * ordered before it.  NULL = the library's own stream, which first waits for the work queued so far on the legacy default
 * stream (where torch and plain CUDA calls go when no stream is chosen); it does not wait for other streams of the caller.
 * Engine calls are ordered among themselves whatever their streams: every later call of this library, on any stream or
 * thread, waits for this one's queued work before it touches the engine's buffers.  Deferred errors (a traceback that left
 * its window) stay in a status word until pb200Synchronize reports and clears them; later calls that check the word
 * (adapterMiddleScanDevice and the host-buffer calls, adapterSetSearch included) report them too. */
int adapterAlignmentBatchDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs,
                                int64_t total_seq_bytes, int64_t max_seq_len, const uint8_t *adapters,
                                const int32_t *ad_off, int32_t n_adapters, int matchScore, int mismatchScore,
                                int gapOpenScore, int gapExtensionScore, int32_t *d_out, void *stream);

/* Phase C of Porechop on the device: find_middle_adapters (porechop/nanopore_read.py:216-243) for every sequence.
 * Sequences are the end-trimmed reads; adapters are in the reference's order (porechop.py:541-548).  For each sequence,
 * for each adapter in order: align; if float("%f" % fullAdapter%ID) >= middle_threshold, record the hit, overwrite read
 * positions [readStart, readEnd] with the N code (the reference's '-') and align the same adapter again; otherwise move on
 * to the next adapter.  The masked reads and the records of reads without a hit never leave the device.
 * Output (caller-owned host buffers): n_hits[s] = number of hits of sequence s; hits = hits_cap records of 10 int32
 * {adapter index, the 9-int record of the alignment that hit}, sequence-major, each sequence's hits in the order found.
 * *n_total is always written.  If *n_total > hits_cap, only n_hits and *n_total are valid and the call returns
 * PB200_ERR_SPACE.
 * Preconditions, checked before the device is touched (PB200_ERR_ARG otherwise): middle_threshold > 0 (not NaN), every
 * adapter byte in ACGTUacgtu, and every adapter served by the int16 kernels with a finite window bound (both gap scores
 * negative).  Under them every hit masks at least one base that was not masked before, so the loop ends; more rounds
 * than the longest sequence has bases give PB200_ERR_INTERNAL. */
int adapterMiddleScan(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
                      const int32_t *ad_off, int32_t n_adapters, int matchScore, int mismatchScore, int gapOpenScore,
                      int gapExtensionScore, double middle_threshold, int32_t *n_hits, int32_t *hits, int64_t hits_cap,
                      int64_t *n_total);
/* Same, with seqs / seq_off in device memory (conventions of adapterAlignmentBatchDevice; the caller's sequences are not
 * modified: the masking works on the library's encoded copy).  The work is enqueued on `stream` (NULL: as above) after the
 * work earlier calls of this library left queued on any stream; the outputs are host buffers, so the call returns only
 * after they are written. */
int adapterMiddleScanDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                            int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters,
                            int matchScore, int mismatchScore, int gapOpenScore, int gapExtensionScore,
                            double middle_threshold, int32_t *n_hits, int32_t *hits, int64_t hits_cap, int64_t *n_total,
                            void *stream);
/* Phase B and Phase C of Porechop on whole reads in one call: the semantics of adapterEndDecisions over the windows
 * seq[:end_size] / seq[-end_size:] of every read, followed by adapterMiddleScan over seq[start_trim : len - end_trim] (Python's
 * slice: an end position below 0 counts from the end of the read again; an untrimmed read is the whole read).  The windows
 * are cut, the trims decided and turned into the trimmed reads, and the trimmed reads encoded and masked on the device, so
 * the read bytes cross PCIe once (host variant) or not at all (device variant), and 4 bytes per read per side, the score
 * outputs and the hits come back.
 *   start / end    one side of Phase B (find_start_trim / find_end_trim): adapters, score columns and outputs with the
 *                  meaning of the pb200_end_batch_t fields of the same names; n_adapters = 0: the side is not searched, its
 *                  trims are 0 (and top2, if given, the "no column" entries)
 *   mid_*          the middle adapters in the reference's order; n_mid_adapters = 0: no Phase C (--no_split), and n_hits /
 *                  hits / n_total may then be NULL (written as zero / empty when given)
 *   n_hits, hits   as adapterMiddleScan, in trimmed-read coordinates; on PB200_ERR_SPACE the trims, the score outputs,
 *                  n_hits and *n_total are valid
 * Preconditions, checked before the device is touched (PB200_ERR_ARG otherwise): those of adapterEndDecisions for each side
 * and of adapterMiddleScan for the middle adapters, end_size >= 1, and every adapter of every side served by the int16
 * kernels with a finite window bound (both gap scores negative; no generic-class scheme). */
typedef struct {
    const uint8_t *adapters; const int32_t *ad_off; int32_t n_adapters;   /* 0 = side not searched, trims = 0 */
    const int32_t *score_cols; int32_t n_score_cols;                      /* as pb200_end_batch_t */
    int32_t *trim;                                                        /* out: n_seqs */
    uint16_t *score_pairs;                                                /* out: as pb200_end_batch_t (may be NULL) */
    int32_t *top2;                                                        /* out: as pb200_end_batch_t (may be NULL) */
} pb200_trim_side_t;
typedef struct {
    int32_t end_size, extra_trim_size, min_trim_size;   /* --end_size (>= 1), --extra_end_trim, --min_trim_size */
    double end_threshold;                               /* --end_threshold (>= 0) */
    pb200_trim_side_t start, end;
    const uint8_t *mid_adapters; const int32_t *mid_ad_off; int32_t n_mid_adapters;   /* 0 = no Phase C */
    double middle_threshold;                            /* --middle_threshold (> 0 when there are middle adapters) */
    int32_t *n_hits; int32_t *hits; int64_t hits_cap; int64_t *n_total;   /* outputs, as adapterMiddleScan */
} pb200_trim_args_t;
int adapterTrimReads(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const pb200_trim_args_t *args,
                     int matchScore, int mismatchScore, int gapOpenScore, int gapExtensionScore);
/* Same, with seqs / seq_off in device memory (conventions of adapterMiddleScanDevice: max_seq_len = longest read or -1; the
 * caller's buffers are only read; the work runs on `stream` -- NULL: the library's own stream after the legacy default
 * stream -- after the work earlier calls of this library left queued on any stream; the outputs are host buffers, so the
 * call returns only after they are written, and reports a deferred error an earlier device-resident call left in the status
 * word). */
int adapterTrimReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                           int64_t max_seq_len, const pb200_trim_args_t *args, int matchScore, int mismatchScore,
                           int gapOpenScore, int gapExtensionScore, void *stream);
/* Porechop's output reads on the device: adapterTrimReadsDevice (same semantics, preconditions, stream and ordering rules, and
 * host outputs), then the records get_fastq / get_fasta would write (porechop/nanopore_read.py:57-147) cut into caller-owned
 * device buffers -- the records fastq.emit writes for these decisions, in the same order:
 *   - a read without a middle hit: seq[start_trim : len - end_trim] (the whole read with `untrimmed`), if not empty;
 *   - a read with hits: nothing with `discard_middle`, else the runs of its trimmed range outside the union of
 *     [readStart - mid_extra_left[a], readEnd + 1 + mid_extra_right[a]) over its hits (clipped to the trimmed range), each
 *     at least min_split_read_size long (get_split_read_parts), numbered 1, 2, ... in position order.
 * Per record: bases (and qualities, from d_quals at the same offsets) copied as given -- no case or U/T change -- at
 * d_out_off[r] .. d_out_off[r + 1]; d_out_read[r] = source read; d_out_part[r] = 0 (not split) or k >= 1 (the k-th part: the
 * number add_number_to_read_name appends).  Records are in read order, the parts of a read in position order; names stay on
 * the host.  Every record is a disjoint piece of its read, so total_seq_bytes bytes always suffice for d_out_seq / d_out_qual;
 * the number of records is at most n_seqs + the number of hits.
 * *n_parts and *n_out_bases are always written (0 on an argument error).  If *n_parts > parts_cap, or the hits do not fit
 * hits_cap, the call returns PB200_ERR_SPACE: the host outputs and both totals are valid, the device outputs are not.  The
 * call returns once the device outputs are written.
 * Preconditions, checked before the device is touched (PB200_ERR_ARG otherwise): those of adapterTrimReadsDevice, split not
 * NULL, parts_cap >= 0, both mid_extra_* arrays when n_mid_adapters > 0, d_out_qual NULL exactly when d_quals is NULL, and
 * (n_seqs > 0) d_out_off, plus -- when parts_cap > 0 -- d_out_read / d_out_part and (total_seq_bytes > 0) d_out_seq.
 * With no adapter on any side and no middle adapter every non-empty read comes out unchanged ("No adapters found"). */
typedef struct {
    const uint8_t *d_quals;            /* device, at the reads' offsets (quality length == read length), or NULL (FASTA) */
    const int32_t *mid_extra_left;     /* host, per middle adapter: bases cut before a hit  (bad side if a start sequence) */
    const int32_t *mid_extra_right;    /* host, per middle adapter: bases cut after a hit   (bad side if an end sequence)  */
    int32_t min_split_read_size, discard_middle, untrimmed;
    uint8_t *d_out_seq, *d_out_qual;   /* device, total_seq_bytes each (always enough); d_out_qual NULL iff d_quals NULL */
    int64_t *d_out_off;                /* device, parts_cap + 1 */
    int32_t *d_out_read, *d_out_part;  /* device, parts_cap */
    int64_t parts_cap;
    int64_t *n_parts, *n_out_bases;    /* host, always written */
} pb200_split_args_t;
int adapterTrimSplitReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                                int64_t max_seq_len, const pb200_trim_args_t *args, const pb200_split_args_t *split,
                                int matchScore, int mismatchScore, int gapOpenScore, int gapExtensionScore, void *stream);
/* Porechop's demultiplexed output reads on the device (porechop -b DIR): adapterTrimSplitReadsDevice (same semantics, stream
 * and ordering rules, status word, trims, hits and PB200_ERR_SPACE behaviour), plus the barcode call of every read, with the
 * records grouped by bin.
 *   - The call of a read is determine_barcode (porechop/nanopore_read.py:399-470) on the top-2 ranking of each side's score
 *     columns (adapterEndDecisions' `top2`): the column's bin is start_bin[pos] / end_bin[pos], its score the exact double the
 *     reference parses, float("%f" % (100.0 * match / len)), 0.0 when the side has no column.  Without require_two_barcodes
 *     the best of both sides wins (the start side on ties) if it reaches barcode_threshold and beats by barcode_diff the best
 *     entry of either side with another bin; with it both sides' best must agree, reach the threshold and beat their own
 *     side's second by barcode_diff.  d_albacore[s] >= 0: the call stands only if it equals d_albacore[s] (Porechop and
 *     Albacore must agree), else the read goes to 'none'.  read_bin[s] = the call (n_bins = 'none').
 *   - Records are grouped by bin in bin-id order, 'none' last; inside a bin in read order, the parts of a read in position
 *     order (the sequence fastq.demux_fastq writes into each bin's file).  bin_parts[b] .. bin_parts[b + 1] are the records
 *     of bin b (b = n_bins: 'none'), their bases d_out_off[bin_parts[b]] .. d_out_off[bin_parts[b + 1]].
 *   - discard_unassigned: the 'none' records are not written and do not count in *n_parts, *n_out_bases or parts_cap.
 * On PB200_ERR_SPACE read_bin, bin_parts, the trims and the hits are valid; the device outputs are not.  The top2 outputs of
 * args->start / args->end may be NULL (the ranking stays on the device).
 * Preconditions, checked before the device is touched (PB200_ERR_ARG otherwise): those of adapterTrimSplitReadsDevice, demux /
 * read_bin / bin_parts not NULL, start_bin / end_bin present when the side has score columns, bin ids in [0, n_bins) and no
 * bin twice on one side, 0 <= n_bins < 4096, barcode_threshold / barcode_diff not NaN, and the side windows within the
 * device ranking's domain (end_size + longest adapter + 2 <= 4095).  With no barcode columns every read is 'none'. */
typedef struct {
    const int32_t *start_bin;          /* host, args->start.n_score_cols: bin id of each start score column            */
    const int32_t *end_bin;            /* host, args->end.n_score_cols: bin id of each end score column                */
    int32_t n_bins;                    /* named bins 0 .. n_bins - 1; bin n_bins is 'none'                              */
    double barcode_threshold, barcode_diff;
    int32_t require_two_barcodes, discard_unassigned;
    const int32_t *d_albacore;         /* device, per read, or NULL: -1 = no Albacore call, else the bin the call must
                                          equal (n_bins + 1 = a name that is no bin: the read always goes to 'none')    */
    int32_t *read_bin;                 /* host out, n_seqs: the call of every read (n_bins = 'none')                    */
    int64_t *bin_parts;                /* host out, n_bins + 2: record offsets of the bins in output order              */
} pb200_demux_args_t;
int adapterDemuxReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                            int64_t max_seq_len, const pb200_trim_args_t *args, const pb200_split_args_t *split,
                            const pb200_demux_args_t *demux, int matchScore, int mismatchScore, int gapOpenScore,
                            int gapExtensionScore, void *stream);
/* The bytes Porechop writes for output records already in device memory -- e.g. those of adapterTrimSplitReadsDevice or
 * adapterDemuxReadsDevice, or any slice of them (one bin) -- into a caller-owned device buffer: the bytes fastq.emit_parts
 * writes for the same records, in record order (get_fastq / get_fasta, porechop/nanopore_read.py:97-147).
 *   - FASTQ: '@' name' '\n' bases' '\n' '+' '\n' quals '\n'.  FASTA: '>' name' '\n', then bases' in lines of 70, each ending in
 *     '\n' (no base line for a record without bases).
 *   - name' is the source read's name; for part k >= 1 the decimal tag "_k" goes before its first 0x20 byte, or at its end when
 *     it has none (add_number_to_read_name, nanopore_read.py:494-498).
 *   - bases' are the stored bytes, except that records of a read with d_rna[read] != 0 have every 'T' written as 'U' (and only
 *     'T').  Qualities are written as stored.
 * d_out_off gets every record's byte offset (0 for the first; the scanned lengths) and *n_out_bytes the total.  If the total
 * exceeds out_cap the call returns PB200_ERR_SPACE: *n_out_bytes and d_out_off are valid, d_out is not written.  The call
 * returns once the device outputs are written; stream and ordering rules as adapterTrimReadsDevice (NULL: the library's own
 * stream after the legacy default stream; after the work earlier calls of this library left queued; a deferred error in the
 * status word is reported).
 * Preconditions, checked before the device is touched (PB200_ERR_ARG otherwise): args not NULL, fmt 0 or 1, d_qual for FASTQ,
 * no negative count, and the pointers the sizes need (n_out_bytes and d_out_off always).  The record arrays are checked on the
 * device before anything is written to d_out (PB200_ERR_ARG, d_out untouched): 0 <= d_off[r] <= d_off[r + 1] <= seq_bytes,
 * 0 <= d_read[r] < n_reads, d_part[r] >= 0 and 0 <= d_name_off[read] <= d_name_off[read + 1] <= name_bytes. */
typedef struct {
    const uint8_t *d_seq, *d_qual;     /* device: record bases / qualities at the same offsets; d_qual NULL: FASTA only       */
    int64_t seq_bytes;                 /* length of d_seq (and d_qual)                                                        */
    const int64_t *d_off;              /* device, n_rec + 1: record r = d_seq[d_off[r] .. d_off[r + 1]) (absolute offsets)    */
    const int32_t *d_read, *d_part;    /* device, n_rec: source read; 0 = not split, k >= 1 = the k-th part                   */
    const uint8_t *d_names;            /* device: the source reads' names, read s at d_names[d_name_off[s] .. d_name_off[s+1]) */
    const int64_t *d_name_off;         /* device, n_reads + 1                                                                 */
    int64_t n_reads, name_bytes;
    const uint8_t *d_rna;              /* device, n_reads, or NULL: nonzero = RNA read (T written as U)                       */
    int32_t fmt;                       /* 0 = FASTQ, 1 = FASTA                                                                */
    uint8_t *d_out;                    /* device, out_cap bytes                                                               */
    int64_t out_cap;
    int64_t *d_out_off;                /* device out, n_rec + 1: byte offset of every record, then the total                 */
    int64_t *n_out_bytes;              /* host out, always written                                                            */
} pb200_emit_args_t;
int pb200EmitReadsDevice(const pb200_emit_args_t *args, int64_t n_rec, void *stream);
/* The reads of FASTQ / FASTA bytes in device memory, parsed into caller-owned device buffers: the fields fastq.parse_fastq /
 * fastq.parse_fasta return (the reference's loader, misc.py:123-166, and NanoporeRead.__init__, nanopore_read.py:23-36).
 *   - Lines end at '\n'; an unterminated last line ends at n_in.  Every line is stripped of the ASCII bytes str.strip()
 *     removes (9-13, 28-31, 32); other bytes ('\r' alone, non-ASCII) are kept.
 *   - FASTQ (fmt 0): record r is lines 4r .. 4r+3.  The stripped header must be non-empty and start with '@'; the name is the
 *     stripped header minus that byte, the bases are line 4r+1, the qualities line 4r+3 (line 4r+2 is not looked at).
 *   - FASTA (fmt 1): blank lines are dropped; the first kept line must start with '>'; every '>' line starts a record whose
 *     name is the line minus '>' (never empty), and the record's bases are its body lines concatenated.
 *   - Bases are upper-cased (a-z only); d_rna[r] = 1 when the read has more 'U' than 'T' bytes, and such a read stores every
 *     'U' as 'T'.
 *   - d_qual (optional) gets one quality per base at the bases' offsets: FASTQ qualities padded with '+' to the bases' length,
 *     FASTA '+' for every base.
 * d_name_off / d_seq_off get n_reads + 1 offsets (0 first).  n_reads, n_name_bytes and n_seq_bytes are always written.  When
 * a count exceeds its capacity the call returns PB200_ERR_SPACE with the exact counts and writes no device output.
 * Malformed input returns PB200_ERR_ARG with *error set (PB200_PARSE_*) and *error_index = the first bad FASTQ record or FASTA
 * line (0-based); no device output is written.  A FASTQ quality line longer than its bases cannot be held at the bases'
 * offsets: with d_qual set that is PB200_PARSE_LONG_QUAL (callers parse such a chunk on the host).  Empty input gives 0 reads
 * without a kernel launch.  The call returns once the device outputs are written; stream and ordering rules as
 * pb200EmitReadsDevice.
 * Preconditions, checked before the device is touched (PB200_ERR_ARG, *error 0): args not NULL, fmt 0 or 1, no negative
 * size, every host output, d_name_off and d_seq_off, and the device pointers whose capacity is nonzero. */
enum {
    PB200_PARSE_OK = 0,
    PB200_PARSE_LINES = 1,       /* FASTQ: the number of lines is not a multiple of 4 (index: the incomplete record)       */
    PB200_PARSE_HEADER = 2,      /* FASTQ: a stripped header is empty or does not start with '@'                          */
    PB200_PARSE_FASTA_START = 3, /* FASTA: a body line comes before the first '>' line                                     */
    PB200_PARSE_FASTA_NAME = 4,  /* FASTA: a '>' line with an empty name                                                   */
    PB200_PARSE_LONG_QUAL = 5    /* FASTQ with d_qual: a quality line longer than its bases                               */
};
typedef struct {
    const uint8_t *d_in;               /* device, n_in bytes of whole records                                                 */
    int64_t n_in;
    int32_t fmt;                       /* 0 = FASTQ, 1 = FASTA                                                                */
    uint8_t *d_names;                  /* device out, names_cap bytes: read r's name at d_name_off[r] .. d_name_off[r + 1]    */
    int64_t names_cap;
    int64_t *d_name_off;               /* device out, reads_cap + 1                                                           */
    uint8_t *d_seq;                    /* device out, seq_cap bytes: read r's bases at d_seq_off[r] .. d_seq_off[r + 1]       */
    int64_t seq_cap;
    int64_t *d_seq_off;                /* device out, reads_cap + 1                                                           */
    uint8_t *d_qual;                   /* device out, seq_cap bytes at the bases' offsets, or NULL: no qualities              */
    uint8_t *d_rna;                    /* device out, reads_cap: 1 = RNA read                                                 */
    int64_t reads_cap;
    int64_t *n_reads, *n_name_bytes, *n_seq_bytes;   /* host out, always written                                             */
    int32_t *error;                    /* host out: PB200_PARSE_* (0 unless malformed input)                                  */
    int64_t *error_index;              /* host out: first bad record (FASTQ) or line (FASTA), -1 when none                    */
} pb200_parse_args_t;
int pb200ParseReadsDevice(const pb200_parse_args_t *args, void *stream);
/* cmin[l], l = 0 .. len-1: the smallest c with float("%f" % (100.0*c/l)) >= middle_threshold, or l+1 if none does
 * (cmin[0] = INT32_MAX).  The ">=" sibling of pb200TrimThresholdTable.  Pure host code; middle_threshold must be > 0. */
int pb200MiddleThresholdTable(double middle_threshold, int32_t len, int32_t *cmin);

/* Format one 9-int record as the reference string (alignment.cpp:113-121). Returns strlen, or -1 if buflen is
 * too small (64 bytes always suffice). */
int pb200FormatRecord(const int32_t *record, char *buf, int buflen);

/* Host-side Dna5 conversion of the packed upload path (option "h2d_pack"): n ASCII bases -> (n+1)/2 bytes, the code
 * of base 2k (A/a=0 C/c=1 G/g=2 T/t/U/u=3, anything else 4: seqan/basic/alphabet_residue_tabs.h:113-140) in the low
 * nibble of byte k and base 2k+1 in the high nibble.  Pure host code (AVX-512BW / AVX2 when the CPU has it, its own thread
 * team; threads <= 0 = the hardware threads the cgroup CPU quota allows); exported so that tests and hosts that already hold
 * packed reads can use the same packer. */
int pb200PackNibbles(const uint8_t *ascii, int64_t n, uint8_t *packed, int threads);

/* ---- device / diagnostics ------------------------------------------------------------------------------ */
int pb200DeviceCount(void);               /* number of CUDA devices visible (0 if none / no driver) */
int pb200SetDevice(int device);           /* cudaSetDevice for the calling thread */
int pb200Synchronize(void);               /* wait for everything this library enqueued on the current device and
                                             report deferred errors of adapterAlignmentBatchDevice calls */
const char *pb200LastError(void);         /* text of the last error on this thread ("" if none) */
long long pb200KernelLaunches(void);      /* kernels launched by this library since load (all threads) */
/* Kernel timing with CUDA events on the launching stream: enable, run, then read back the accumulated
 * duration and launch count of the DP kernels (trace_kernel + score_kernel) since the last reset. */
void pb200TimingEnable(int on);
int pb200TimingRead(double *dp_kernel_ms, long long *dp_kernel_launches, double *cells, int reset);
/* The same per kind of DP launch, arrays of PB200_TIMING_KINDS entries: 0 trace_kernel (windows, single pass),
 * 1 unused, 2 trace_kernel on the bounded windows of a two-pass class, 3 score_kernel (long reads).
 * window_cells = DP cells computed by the launches of kind 2 (the other kinds sweep every cell of their batch). */
#define PB200_TIMING_KINDS 4
int pb200TimingReadKinds(double *ms, long long *launches, double *window_cells, int reset);
/* Tunables (also read from the environment at first use, PB200_<NAME>); none of them changes a result:
 *   "direct_max"  longest sequence aligned in one pass (default 160; longer ones take score pass + bounded window)
 *   "chunk_tasks" alignments per pipeline chunk of the host-buffer API (default 131072)
 *   "scratch_mb"  cap on the resident trace scratch in MB (default 128; 72 keeps it L2-resident, DESIGN.md)
 *   "hbuf"        staging of a slot's packed bases: "auto" | "smem" | "global"
 *   "h2d_pack"    1 = the host-buffer calls convert the sequences to 4-bit codes on the host cores (a packer thread that
 *                 runs ahead of the submit loop) and upload half the bytes; 0 (default) = never; -1 = auto: submits of at
 *                 least 32 MB when the packer team has 12 or more threads; "pack_threads" = host threads of the packer
 *                 (default = the hardware threads the cgroup CPU quota allows / LOCAL_WORLD_SIZE, minus two for the submit
 *                 and driver threads, at most 32)
 *   "profile"     1 (default) = the long-read score pass fetches its substitution operands from a query profile in shared
 *                 memory when every slot is one read x two adapters (cross-product mode); 0 = always computed
 *   "tight_window" 1 (default) = second-pass windows sized per alignment from the end cell's row and score; 0 = the
 *                 per-adapter worst case
 * ("short2p", "rowoff" and trace-kernel query profiles were measured and removed: none was faster) */
int pb200SetOption(const char *name, const char *value);
/* Current value of an integer tunable ("h2d_pack", "pack_threads", "tight_window", "profile", "scratch_mb", "direct_max",
 * "chunk_tasks", "hbuf" as 0/1/2), or "h2d_pack_large_submit": what h2d_pack = auto resolves to for a large submit on this
 * host (1 = packed).  -1 for an unknown name. */
int pb200GetOption(const char *name);
/* Pinned (page-locked) staging memory for host callers that assemble a batch before submitting it: slot 0..3, at least `bytes`
 * long, owned by the library and valid until the next call for the same slot; NULL when there is no device.  Uploads from it
 * are asynchronous DMA; the buffer is reused call after call. */
void *pb200HostBuffer(int slot, size_t bytes);

enum {
    PB200_OK = 0,
    PB200_ERR_NO_DEVICE = 100,   /* no CUDA device / driver, or device is not sm_90 */
    PB200_ERR_CUDA = 101,        /* a CUDA call failed (see pb200LastError) */
    PB200_ERR_ARG = 102,         /* invalid argument */
    PB200_ERR_INTERNAL = 103,    /* internal invariant violated (e.g. window bound) */
    PB200_ERR_SPACE = 104        /* an output buffer is too small (adapterMiddleScan: *n_total > hits_cap) */
};

#ifdef __cplusplus
}
#endif
#endif /* PORECHOP_B200_H */
