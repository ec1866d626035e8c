// tests/emu/emu_split.cpp -- the split rule of the output stage (dp_core.cuh split_runs, which split_count_kernel and
// split_write_kernel run per read) compiled for the host, so that the no-GPU tier can compare it with the host statement of
// get_split_read_parts (fastq._split_parts).  TEST ONLY: the product never builds or loads this file.
#include <cstdint>
#include "../../porechop_b200/csrc/dp_core.cuh"

// parts of one trimmed read of `len` bases: their number is returned, (start, end) pairs go to out (room for n_rng + 1)
extern "C" int64_t emu_split_parts(int64_t len, const int32_t *rng, int32_t n_rng, int64_t min_size, int64_t *out) {
    return pb::split_runs(len, rng, n_rng, min_size, [&](int64_t k, int64_t x, int64_t y) {
        out[2 * k] = x;
        out[2 * k + 1] = y;
    });
}
