// tests/emu/emu_demux.cpp -- the barcode call of the demux stage (dp_core.cuh barcode_call, which barcode_call_kernel runs per
// read) compiled for the host, so that the no-GPU tier can compare it with the host statement of determine_barcode
// (fastq.call_barcodes_top2).  TEST ONLY: the product never builds or loads this file.
#include <cstdint>
#include "../../porechop_b200/csrc/dp_core.cuh"

// n reads: per side the bins of the best / second-best column (b[2s], b[2s + 1]; -1 = none) and their scores; albacore
// NULL or one bin per read (-1 = no call).  The calls (n_bins = 'none') go to out.
extern "C" void emu_barcode_calls(int64_t n, const int32_t *sb, const double *ss, const int32_t *eb, const double *es,
                                  int32_t n_bins, double threshold, double diff, int32_t require_two, const int32_t *albacore,
                                  int32_t *out) {
    for (int64_t s = 0; s < n; ++s) {
        const pb::BarcodeSide bs = {sb[2 * s], sb[2 * s + 1], ss[2 * s], ss[2 * s + 1]};
        const pb::BarcodeSide be = {eb[2 * s], eb[2 * s + 1], es[2 * s], es[2 * s + 1]};
        out[s] = pb::barcode_call(bs, be, n_bins, threshold, diff, require_two, albacore ? albacore[s] : -1);
    }
}
