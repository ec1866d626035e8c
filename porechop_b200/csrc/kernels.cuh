// porechop_b200/csrc/kernels.cuh -- sm_90a kernels of the adapter-alignment engine.
//
//   encode_kernel        ASCII -> Dna5 code (seqan/basic/alphabet_residue_tabs.h:113-140), HBM-bound
//   unpack_kernel        host-packed 4-bit codes -> the same code bytes (option h2d_pack)
//   build_tasks_*        (read, adapter) pairs -> Task records in slot order
//   trace_kernel<G,R,S>  overlap DP *with* 4-bit trace + in-kernel traceback + statistics (windows)
//   score_kernel<G,R,P>  streaming score-only overlap DP with exact scout (long reads), dynamic slot refill
//   window_tasks_kernel  end cells of the score pass -> bounded-window tasks for trace_kernel
//   decide_kernel        records -> per-read end-trim amounts + barcode score pairs (decisions stay on the device)
//   search_best_kernel   records -> per-adapter best full-adapter identity of the adapter-set search (Phase A)
//   middle_decide_kernel one round of the middle-adapter scan: first hit per active read, masking, next active list
//   window_len / cut_windows / trimmed_range / gather_encode + scan_*: whole-read trimming (adapterTrimReads) -- end windows
//                        cut from resident reads, trims turned into the trimmed reads the middle scan masks
//   split_mark / split_count / split_write / split_gather: output stage of adapterTrimSplitReadsDevice -- Porechop's output
//                        records counted, placed and gathered (bases + qualities) into the caller's buffers
//   barcode_call / demux_count / demux_bin_parts / demux_scatter: demux stage of adapterDemuxReadsDevice -- the barcode call
//                        of every read, and the records partitioned stably by bin before split_gather copies them
//   generic_kernel       int32 thread-serial fallback for scoring schemes / adapters outside the int16 domain
//
// The arithmetic is in dp_core.cuh (shared with the CPU emulation used by the tests).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "dp_core.cuh"

namespace pb {

constexpr int PB_WARPS_PER_BLOCK = 4;
// trace_kernel blocks per SM.  Groups of G <= 8 lanes: 6 (80 registers), which the default trace scratch and the shared
// memory hold for end windows (the scratch of a warp grows with G: 128 MB holds 6 blocks per SM of G = 4 / 8 at 150 columns,
// 5 of G = 16 / 32).  Since the final-column scout runs inside the careful step (lane_step<.., FCOL>) the end-trim classes
// spill at most 4 bytes (DESIGN.md section 4).  On an H100 80GB HBM3 at a 700 W power limit the end-trim launches ran 2.9 %
// faster than at 5 blocks.  Wider groups keep 5 blocks (96 registers): a sixth block would not fit their scratch.
#ifndef PB_TRACE_MIN_BLOCKS
#define PB_TRACE_MIN_BLOCKS 6
#endif
#ifndef PB_TRACE_MIN_BLOCKS_WIDE
#define PB_TRACE_MIN_BLOCKS_WIDE 5
#endif
constexpr int PB_TB_WORDS = 16 * 12;           // TbTask per half of the (at most 8) slots of a warp
constexpr int PB_SCRATCH_WORDS = 32 * 2 * 6 + PB_TB_WORDS;   // ScoutCand per lane per half, then the TbTasks
constexpr int PB_TCHUNK = 4;                   // trace steps per 128-bit store (must stay 4: uint4)

// ---------------------------------------------------------------------------------------------------
// encode: one byte in, one byte out (code << 4).  16 bytes per thread, fully coalesced.
__device__ __forceinline__ uint32_t encode_word(uint32_t w) {
    return encode_byte(w & 0xFFu) | (encode_byte((w >> 8) & 0xFFu) << 8) | (encode_byte((w >> 16) & 0xFFu) << 16) |
           (encode_byte(w >> 24) << 24);
}
__global__ void encode_kernel(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int64_t n) {
    int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * 16;
    for (; i < n; i += stride) {
        if (i + 16 <= n && ((((uintptr_t)in) | ((uintptr_t)out)) & 15) == 0) {
            uint4 v = *reinterpret_cast<const uint4 *>(in + i);
            v.x = encode_word(v.x); v.y = encode_word(v.y); v.z = encode_word(v.z); v.w = encode_word(v.w);
            *reinterpret_cast<uint4 *>(out + i) = v;
        } else {
            for (int64_t k = i; k < n && k < i + 16; ++k) out[k] = (uint8_t)encode_byte(in[k]);
        }
    }
}

// unpack (option h2d_pack): 4-bit codes packed by the host (hostpack.cpp) -> the code bytes encode_kernel produces.
// 8 packed bytes in, 16 bytes out per thread; `n` = number of bases.  HBM-bound, 1.5 B/base of traffic.
__global__ void unpack_kernel(const uint8_t *__restrict__ in, uint8_t *__restrict__ out, int64_t n) {
    int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 16;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x * 16;
    for (; i < n; i += stride) {
        if (i + 16 <= n && ((((uintptr_t)in) & 7) | (((uintptr_t)out) & 15)) == 0) {
            const uint2 p = *reinterpret_cast<const uint2 *>(in + (i >> 1));
            uint4 v;
            unpack_nibbles8(p.x, v.x, v.y);
            unpack_nibbles8(p.y, v.z, v.w);
            *reinterpret_cast<uint4 *>(out + i) = v;
        } else {
            for (int64_t k = i; k < n && k < i + 16; ++k) out[k] = (uint8_t)unpack_nibble1(in[k >> 1], (int)(k & 1));
        }
    }
}

// max sequence length (for planning) -- one int64 atomicMax
__global__ void max_len_kernel(const int64_t *__restrict__ off, int64_t n, unsigned long long *out) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long v = 0;
    for (; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        unsigned long long l = (unsigned long long)(off[i + 1] - off[i]);
        v = l > v ? l : v;
    }
    for (int o = 16; o > 0; o >>= 1) { unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
    if ((threadIdx.x & 31) == 0 && v) atomicMax(out, v);
}

// ---------------------------------------------------------------------------------------------------
// Sequence order by decreasing length (bucket sort, PB_ORDER_BINS log-spaced-ish linear bins): used by the two-pass
// path so that the dynamically scheduled score pass starts with the longest reads (no long tail) and neighbouring
// slots have similar lengths.  Order inside a bin is arbitrary (atomics) -- results do not depend on it.
constexpr int PB_ORDER_BINS = 2048;
__device__ __forceinline__ int order_bin(int64_t len, int64_t max_len) {
    int64_t b = (len * (PB_ORDER_BINS - 1)) / (max_len > 0 ? max_len : 1);
    if (b > PB_ORDER_BINS - 1) b = PB_ORDER_BINS - 1;
    return (PB_ORDER_BINS - 1) - (int)b;          // bin 0 = longest
}
__global__ void order_hist_kernel(const int64_t *__restrict__ off, int64_t n, int64_t max_len, unsigned *__restrict__ bins) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicAdd(&bins[order_bin(off[i + 1] - off[i], max_len)], 1u);
}
__global__ void order_scan_kernel(unsigned *bins) {   // one block of PB_ORDER_BINS/2 threads: exclusive scan in place
    __shared__ unsigned sh[PB_ORDER_BINS];
    for (int i = threadIdx.x; i < PB_ORDER_BINS; i += blockDim.x) sh[i] = bins[i];
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned run = 0;
        for (int i = 0; i < PB_ORDER_BINS; ++i) { unsigned v = sh[i]; sh[i] = run; run += v; }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < PB_ORDER_BINS; i += blockDim.x) bins[i] = sh[i];
}
__global__ void order_scatter_kernel(const int64_t *__restrict__ off, int64_t n, int64_t max_len, unsigned *__restrict__ bins,
                                     int32_t *__restrict__ order) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        unsigned pos = atomicAdd(&bins[order_bin(off[i + 1] - off[i], max_len)], 1u);
        order[pos] = (int32_t)i;
    }
}

// ---------------------------------------------------------------------------------------------------
// Task sources.
// Cross mode: every sequence x every adapter of one class; the Task records are never materialised -- the kernels
// synthesise them from the offset arrays (saves 64 B written + 128 B read per alignment).  `cls_ad` lists the class's
// adapter ids; adapters 2q and 2q+1 share a slot (same read, two adapters); an odd last adapter pairs two consecutive
// reads instead.  Task index layout: pair q occupies [q*2*n_seqs, (q+1)*2*n_seqs) as (s0,a),(s0,a'),(s1,a),(s1,a')...;
// the odd adapter occupies the tail [n_full*2*n_seqs, +n_seqs).
struct TaskSrc {
    const Task *tasks;        // explicit task records (pair-list mode, windowed second pass) or nullptr = cross mode
    int64_t n_tasks;
    const int32_t *cls_ad;    // cross mode: adapter ids of the class
    int32_t n_cls_ad;
    int32_t n_adapters;       // adapters per sequence in the caller's record layout (out index = s*n_adapters + a)
    int64_t n_seqs;
    const int64_t *seq_off;
    const int32_t *ad_off;
    const int32_t *seq_order; // cross mode, optional: sequence permutation (longest first) -- slot i of a pair region is
                              // sequence seq_order[i]: balances the tail of the score pass and pairs similar lengths
};

__device__ __forceinline__ Task cross_task(const TaskSrc &ts, int64_t k) {
    const int n_full = ts.n_cls_ad / 2;
    const int64_t paired = (int64_t)n_full * 2 * ts.n_seqs;
    int64_t s; int a;
    if (k < paired) {
        int64_t q, rem;
        if (paired <= 0xFFFFFFFFll) {      // launch-uniform: a 32-bit division is a fifth of the 64-bit one (this runs 3-4 times per slot)
            const uint32_t d = (uint32_t)(2 * ts.n_seqs), q32 = (uint32_t)k / d;
            q = q32; rem = (uint32_t)k - q32 * d;
        } else {
            q = k / (2 * ts.n_seqs); rem = k - q * (2 * ts.n_seqs);
        }
        s = rem >> 1; a = __ldg(ts.cls_ad + 2 * q + (rem & 1));
    } else {
        s = k - paired; a = __ldg(ts.cls_ad + ts.n_cls_ad - 1);
    }
    if (ts.seq_order) s = __ldg(ts.seq_order + s);
    Task t;
    const int64_t o0 = __ldg(ts.seq_off + s), o1 = __ldg(ts.seq_off + s + 1);
    const int32_t a0 = __ldg(ts.ad_off + a), a1 = __ldg(ts.ad_off + a + 1);
    t.seq_off = o0;
    t.n = (int32_t)(o1 - o0);
    t.m = a1 - a0;
    t.ad_off = a0;
    t.out_idx = (int32_t)(s * ts.n_adapters + a);
    t.flags = 0; t.end_j = 0; t.end_i = 0; t.end_corr = 0; t.end_score = 0;
    t.col0 = 0; t.n_total = t.n; t.pad0 = t.pad1 = t.pad2 = 0;
    return t;
}
// Pair-list mode: `order` is the host-computed slot order of pair indices for one class.
__global__ void build_tasks_pairs_kernel(Task *__restrict__ tasks, int64_t n_tasks, const int32_t *__restrict__ order,
                                         const int32_t *__restrict__ pair_seq, const int32_t *__restrict__ pair_ad,
                                         const int64_t *__restrict__ seq_off, const int32_t *__restrict__ ad_off) {
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_tasks) return;
    int32_t p = order[k];
    int64_t s = pair_seq[p]; int a = pair_ad[p];
    Task t;
    t.seq_off = seq_off[s];
    t.n = (int32_t)(seq_off[s + 1] - seq_off[s]);
    t.m = ad_off[a + 1] - ad_off[a];
    t.ad_off = ad_off[a];
    t.out_idx = p;
    t.flags = 0; t.end_j = 0; t.end_i = 0; t.end_corr = 0; t.end_score = 0;
    t.col0 = 0; t.n_total = t.n; t.pad0 = t.pad1 = t.pad2 = 0;
    tasks[k] = t;
}

// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ Task get_task(const TaskSrc &ts, int64_t idx) {
    Task t;
    if (idx < ts.n_tasks) {
        if (ts.tasks == nullptr) return cross_task(ts, idx);
        const int4 *p = reinterpret_cast<const int4 *>(ts.tasks + idx);
        int4 *q = reinterpret_cast<int4 *>(&t);
        q[0] = __ldcs(p); q[1] = __ldcs(p + 1); q[2] = __ldcs(p + 2); q[3] = __ldcs(p + 3);   // read once: evict-first in L2
    } else {
        t.seq_off = 0; t.n = 0; t.m = 0; t.ad_off = 0; t.out_idx = -1; t.flags = 0; t.end_j = 0; t.end_i = 0;
        t.end_corr = 0; t.end_score = 0; t.col0 = 0; t.n_total = 0; t.pad0 = t.pad1 = t.pad2 = 0;
    }
    return t;
}

// Score pass results -> windowed tasks.  The traced path has score >= 0, hence at most m diagonals and
// floor(m*max(ma,mi,0)/min(|go|,|ge|)) read-only gap columns: it starts no further than `wbound(m)` columns
// left of its end (DESIGN.md "window bound").  wnum/wden: W = m + (m*wnum)/wden; `tight` = the per-alignment bound
// of dp_core.cuh window_cols() that also uses the end cell's row and score.
__global__ void window_tasks_kernel(const TaskSrc ts, const EndCell *__restrict__ ends, Task *__restrict__ out,
                                    int wnum, int wden, int tight, unsigned long long *__restrict__ window_cells) {
    const int64_t n_tasks = ts.n_tasks;
    int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long cells = 0;      // DP cells the second pass will compute (measurement only: pb200TimingReadKinds)
    if (k < n_tasks) {
        Task t = get_task(ts, k);
        EndCell e = ends[k];
        if (t.n > 0 && t.m > 0) {
            const int64_t W = window_cols(t.m, e.i, e.score, wnum, wden, tight != 0);
            int64_t c0 = (int64_t)e.j - W;
            if (c0 < 0) c0 = 0;
            t.col0 = (int32_t)c0;
            t.seq_off += c0;
            t.n = e.j - (int32_t)c0;
            t.flags = TASK_END_GIVEN | (c0 > 0 ? TASK_LEFT_INF : 0);
            t.end_j = t.n; t.end_i = e.i; t.end_corr = e.corr; t.end_score = e.score;
            cells = (unsigned long long)t.n * (unsigned long long)t.m;
        } else {
            // empty read or adapter: no columns to compute, the trace pass only emits the -1 record
            t.n = 0; t.flags = TASK_END_GIVEN; t.end_j = 0; t.end_i = 0; t.end_corr = 0; t.end_score = PB_SCORE_EMPTY;
        }
        out[k] = t;
    }
    for (int o = 16; o > 0; o >>= 1) cells += __shfl_xor_sync(0xffffffffu, cells, o);
    if ((threadIdx.x & 31) == 0 && cells && window_cells) atomicAdd(window_cells, cells);
}


__device__ __forceinline__ uint32_t pack_bases(uint32_t bA, uint32_t bB) {
    // byte1 <- bA, byte3 <- bB (code<<4 in a byte becomes code<<12 in each half)
    return __byte_perm(bA, bB, 0x4101);
}

// Stage the packed read bases of a slot's columns: hbuf[c] = pack_bases(A[c], B[c]) for c < nmax, PB_PAD_H past the end
// of a half.  Each lane of the group builds every G-th column from single-byte streaming loads, PB_STAGE_COLS columns at a
// time with all their loads issued before any of them is used.  `ascii` (launch-uniform): the sequence buffer holds the
// caller's bytes, and each one is encoded by a lookup in `code_tab` (shared memory, encode_byte of every byte value), so a
// single-pass launch needs no encode pass over the whole batch.  (Calling encode_byte here instead, a chain of compares and
// selects per byte, made the end-trim launches 0.27 ms per step slower: more than the encode pass they replace.)
// (Walking the window in 16-column blocks with one aligned 128-bit load per half and block, funnel-shifted into place, was
// slower: the shift / extract / bounds work per column outweighs the saved LSU instructions, so the byte loads stay.)
constexpr int PB_STAGE_COLS = 4;
constexpr int PB_CODE_TAB_WORDS = 256 / 4;
template <int G>
__device__ __forceinline__ void stage_columns(uint32_t *hbuf, int g, const uint8_t *seqA, int nA, const uint8_t *seqB, int nB,
                                              int nmax, bool ascii, const uint8_t *code_tab) {
    for (int c0 = g; c0 < nmax; c0 += PB_STAGE_COLS * G) {
        uint32_t bA[PB_STAGE_COLS], bB[PB_STAGE_COLS];
#pragma unroll
        for (int k = 0; k < PB_STAGE_COLS; ++k) {
            const int c = c0 + k * G;
            bA[k] = (c < nA) ? (uint32_t)__ldcs(seqA + c) : (uint32_t)PB_PAD_H;
            bB[k] = (c < nB) ? (uint32_t)__ldcs(seqB + c) : (uint32_t)PB_PAD_H;
        }
        if (ascii) {
#pragma unroll
            for (int k = 0; k < PB_STAGE_COLS; ++k) {
                const int c = c0 + k * G;
                if (c < nA) bA[k] = code_tab[bA[k]];
                if (c < nB) bB[k] = code_tab[bB[k]];
            }
        }
#pragma unroll
        for (int k = 0; k < PB_STAGE_COLS; ++k) {
            const int c = c0 + k * G;
            if (c < nmax) hbuf[c] = pack_bases(bA[k], bB[k]);
        }
    }
}

// What the traceback of one half needs from its Task: written to shared memory at slot set-up by the lane that later traces
// the half, so the traceback does not synthesise the Task a second time.  (Keeping n and m here rather than taking them from
// the forward pass's registers also keeps the end-trim classes free of spills.)
struct TbTask {
    int32_t out_idx, flags, col0, n_total, ad_off, end_j, end_i, end_score, n, m, pad0, pad1;   // flags: TASK_* | end_corr << 8
};
static_assert(sizeof(TbTask) * 16 == PB_TB_WORDS * 4, "PB_TB_WORDS holds 16 TbTasks");

// Cursor of trace_kernel's traceback over the trace of one half (see traceback_stats_cur).  The current cell (column j,
// group row q = i + pad - 1) is lane gg = q / R, row r = q % R, step t = j - 1 + gg; its flags are the nibble of row r in
// the trace word of step t, which is word t & 3 of the 128-bit chunk (lane gg, steps t & ~3).  Everything moves
// incrementally: `k` indexes the chunk, `u` = t & 3, and `s` shifts row r's nibble to the top of the word (a move up one
// row adds 4; from row 0 it wraps to row R-1 of lane gg - 1, which is also one step earlier).  A move loads nothing: the
// chunk is fetched by the next flags(), which the caller only asks for inside the matrix.
template <int R, int WPS>
struct TraceCursor {
    const uint4 *base;         // chunk 0 of lane 0 of the group (this half's words)
    const uint32_t *hp;        // staged column word of the current column
    const uint8_t *ap;         // adapter code of the current row
    uint4 cv;                  // base[k] once loaded
    int k;                     // chunk of the current cell: (t >> 2) * WPS * 32 + gg
    int u, s, h;
    int fresh;                 // k has moved since cv was loaded (an int: a bool costs byte moves in the loop)
#ifdef PB_EXPERIMENT_PATH_STEPS
    int steps;
#endif
    __device__ __forceinline__ void init(const uint32_t *tr_half, int end_j, int end_i, int pad, int hh, const uint32_t *hbuf,
                                         const uint8_t *ad) {
        const int q = max(end_i + pad - 1, 0), gg = q / R, r = q % R, t = end_j - 1 + gg;
        h = hh;
        base = reinterpret_cast<const uint4 *>(tr_half);
        k = (t >> 2) * (WPS * 32) + gg;
        u = t & 3; s = 28 - trace_shift<R>(h, r); fresh = 1;
        hp = hbuf + end_j - 1; ap = ad + end_i - 1;
        cv = make_uint4(0u, 0u, 0u, 0u);
#ifdef PB_EXPERIMENT_PATH_STEPS
        steps = 0;
#endif
    }
    __device__ __forceinline__ uint32_t flags() {
        if (fresh) { cv = base[k]; fresh = 0; }
        const uint32_t lo = (u & 1) ? cv.y : cv.x, hi = (u & 1) ? cv.w : cv.z;
        return (((u & 2) ? hi : lo) << s) >> 28;
    }
    __device__ __forceinline__ bool eq() { return ((*hp >> (8 + 16 * h)) & 0xFFu) == (uint32_t)__ldg(ap); }
    __device__ __forceinline__ void move(bool consR, bool consA) {
        const int s0 = 28 - trace_shift<R>(h, 0);
        const bool wrap = consA && s == s0;
        s = wrap ? s0 - 4 * (R - 1) : (consA ? s + 4 : s);
        const int dt = (consR ? 1 : 0) + (wrap ? 1 : 0);
        const bool back = u < dt;
        u = (u - dt) & 3;
        k -= (back ? WPS * 32 : 0) + (wrap ? 1 : 0);
        fresh |= (back || wrap) ? 1 : 0;
        if (consA) --ap;
        if (consR) --hp;
#ifdef PB_EXPERIMENT_PATH_STEPS
        ++steps;
#endif
    }
};

#ifdef PB_EXPERIMENT_PATH_STEPS   // (measurement only: path steps of the traceback; tools/trace_path_steps.py)
// [0] path steps, [1] traced alignments, [2] sum over warp slots of the longest path of the warp, [3] warp slots
extern "C" { __device__ unsigned long long pb_path_stats[4]; }
#endif

// ---------------------------------------------------------------------------------------------------
// trace_kernel: one group of G lanes per slot (two alignments in the s16x2 halves), 32/G slots per warp, R adapter
// rows per lane (G*R >= adapter length; R = 5..8 so common adapter lengths 22/24/28 waste no rows).
// Forward wavefront with a 4-bit trace per cell (two 32-bit words per lane per step), then traceback + statistics
// by two lanes of the group, 9-int record per alignment.  Grid-stride over "warp slots" so the trace scratch is
// bounded by the resident grid and stays in L2.
// (Measured and removed: a score-only first pass + bounded trace window for 150-column windows, and shared-memory query
// profiles for the substitution operands -- neither beat this single pass.  Running the final columns as unrolled 4-step
// chunks too (the general scout behind a warp vote, lanes past the end on the last staged column) made the end-trim launches
// 27 % slower: 6.31-6.36 instead of 4.96-5.01 ms per step.)
template <int G, int R, bool HBUF_SMEM>
__global__ void __launch_bounds__(PB_WARPS_PER_BLOCK * 32, G <= 8 ? PB_TRACE_MIN_BLOCKS : PB_TRACE_MIN_BLOCKS_WIDE)
trace_kernel(const TaskSrc ts, const uint8_t *__restrict__ seq,
             const uint8_t *__restrict__ ads, Scoring sc, int32_t *__restrict__ out, uint32_t *__restrict__ gtrace,
             int max_steps, int max_n, int seq_ascii, int *__restrict__ status) {
    constexpr int SPW = 32 / G;
    constexpr int WPS = TraceWords<R>::value;
    extern __shared__ uint32_t smem[];
    // Shared memory: [ASCII input only: code table, byte value v -> encode_byte(v), PB_CODE_TAB_WORDS] then the per-warp
    // regions (below).  The table is written once per block, before the slot loop.
    const uint8_t *code_tab = reinterpret_cast<const uint8_t *>(smem);
    if (seq_ascii) {
        for (int w = threadIdx.x; w < PB_CODE_TAB_WORDS; w += blockDim.x)
            smem[w] = encode_byte(4u * w) | (encode_byte(4u * w + 1) << 8) | (encode_byte(4u * w + 2) << 16) |
                      (encode_byte(4u * w + 3) << 24);
        __syncthreads();
    }
    uint32_t *const warp_smem = smem + (seq_ascii ? PB_CODE_TAB_WORDS : 0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = lane / G, g = lane % G;
    const int warps_per_block = blockDim.x >> 5;
    const int64_t total_warps = (int64_t)gridDim.x * warps_per_block;
    const int64_t wglobal = (int64_t)blockIdx.x * warps_per_block + warp;
    const int64_t n_tasks = ts.n_tasks;
    const int64_t n_slots = (n_tasks + 1) / 2;
    const int64_t n_wslots = (n_slots + SPW - 1) / SPW;

    // The 4-bit trace goes to a warp-private region of a global scratch buffer that is sized by the RESIDENT grid
    // (grid-stride loop): it is rewritten for every slot and lives in L2.  Layout of the per-warp scratch:
    // [trace max_steps*WPS*32 words] [HBUF_SMEM ? nothing : packed bases SPW*max_n words].
    // Shared memory per warp: [HBUF_SMEM ? packed bases SPW*max_n words : nothing] [scout scratch].
    const size_t trace_words = (size_t)((max_steps + PB_TCHUNK - 1) / PB_TCHUNK) * PB_TCHUNK * WPS * 32;
    // (the staging area is rounded up to 32 words so that every warp's region starts on a 128-byte line: the
    // discard.global.L2 below needs 128-byte aligned addresses and must never touch a neighbour's staged bases)
    const size_t gwarp_words = trace_words + (HBUF_SMEM ? 0 : (((size_t)SPW * max_n + 31) & ~(size_t)31));
    uint32_t *gw = gtrace + (size_t)wglobal * gwarp_words;
    uint32_t *tr = gw;
    const int hb_words = HBUF_SMEM ? SPW * max_n : 0;
    const int per_warp_words = hb_words + PB_SCRATCH_WORDS;
    uint32_t *wsm = warp_smem + (size_t)warp * per_warp_words;
    uint32_t *hbuf = HBUF_SMEM ? (wsm + grp * max_n) : (gw + trace_words + (size_t)grp * max_n);
    ScoutCand *cand = reinterpret_cast<ScoutCand *>(wsm + hb_words);  // [half][lane]
    TbTask *tbt = reinterpret_cast<TbTask *>(cand + 64) + grp * 2;    // [slot][half], this group's slot
    for (int64_t ws = wglobal; ws < n_wslots; ws += total_warps) {
        const int64_t slot = ws * SPW + grp;
        int nA, nB, mA, mB, nmax, nmin;
        bool need_track;
        Lane<R> L;
        {
            // everything that is only needed to set the slot up lives in this scope (keeps the loop's register set small)
            const Task tA = get_task(ts, slot * 2);
            const Task tB = get_task(ts, slot * 2 + 1);
            nA = tA.n; nB = tB.n; mA = tA.m; mB = tB.m;
            if (g < 2) {             // lane g traces half g
                const Task &tk = g ? tB : tA;
                TbTask b;
                b.out_idx = tk.out_idx; b.flags = tk.flags | (tk.end_corr << 8); b.col0 = tk.col0; b.n_total = tk.n_total;
                b.ad_off = tk.ad_off; b.end_j = tk.end_j; b.end_i = tk.end_i; b.end_score = tk.end_score;
                b.n = tk.n; b.m = tk.m; b.pad0 = b.pad1 = 0;
                tbt[g] = b;
            }
            nmax = max(nA, nB);
            stage_columns<G>(hbuf, g, seq + tA.seq_off, nA, seq + tB.seq_off, nB, nmax, seq_ascii != 0, code_tab);
            lane_init<R>(L, g, G, sc, ads + tA.ad_off, mA, (tA.flags & TASK_LEFT_INF) != 0, ads + tB.ad_off, mB,
                         (tB.flags & TASK_LEFT_INF) != 0);
            // scout: fast path while both halves are in inner columns; an empty half never limits it
            const bool emptyA = nA <= 0 || mA <= 0, emptyB = nB <= 0 || mB <= 0;
            nmin = emptyA ? nB : (emptyB ? nA : min(nA, nB));
            need_track = !((tA.flags & TASK_END_GIVEN) && (tB.flags & TASK_END_GIVEN));
        }
        int T = nmax > 0 ? nmax + G - 1 : 0;
        T = __reduce_max_sync(0xffffffffu, T);
        __syncwarp();

        // PB_TCHUNK steps of trace words are collected in registers and written as one 128-bit store per lane:
        // a warp store covers 512 contiguous bytes, and the traceback later gets 4 consecutive steps of a lane
        // with a single (L2-latency) load.
        // Hot chunks (straight-line, 4 steps unrolled): every lane of the warp is inside its matrix (t >= G-1) and in an
        // inner column (fast scout only) -- no per-step activity checks.  Careful chunks (not unrolled): the first
        // G-1 ramp-up steps and the tail with the final columns (general scout, per-lane activity checks).
        const int T4 = (T + PB_TCHUNK - 1) & ~(PB_TCHUNK - 1);
        constexpr int TWARM = (G - 1 + PB_TCHUNK - 1) & ~(PB_TCHUNK - 1);
        int tfast = need_track ? (nmin - 1) : nmax;
        tfast = __reduce_min_sync(0xffffffffu, max(tfast, 0)) & ~(PB_TCHUNK - 1);
#ifdef PB_EXPERIMENT_ALL_HOT   // (timing experiment only, wrong records: every chunk takes the hot path; tools/trace_phase_cost.py)
#define PB_HOT_COL(j) max(min((j) - 1, nmax - 1), 0)       // stay inside the staged bases
#else
#define PB_HOT_COL(j) ((j) - 1)
#endif
        for (int t0 = 0; t0 < T4; t0 += PB_TCHUNK) {
            uint4 acc[WPS];
#ifdef PB_EXPERIMENT_ALL_HOT
            if (true) {
#else
            if (t0 >= TWARM && t0 < tfast) {
#endif
                uint32_t buf[PB_TCHUNK][WPS];
#pragma unroll
                for (int u = 0; u < PB_TCHUNK; ++u) {
                    uint32_t recvS = __shfl_up_sync(0xffffffffu, L.botX, 1, G);
                    uint32_t recvV = __shfl_up_sync(0xffffffffu, L.botV, 1, G);
                    if (g == 0) { recvS = sc.borderX2; recvV = sc.negb2; }
                    const int j = t0 + u - g + 1;
                    lane_step<R, true, false>(L, recvS, recvV, hbuf[PB_HOT_COL(j)], sc, buf[u]);
                    if (need_track) lane_track_lastrow<R>(L, j, sc);
                }
#pragma unroll
                for (int w = 0; w < WPS; ++w) acc[w] = make_uint4(buf[0][w], buf[1][w], buf[2][w], buf[3][w]);
            } else {
#pragma unroll
                for (int w = 0; w < WPS; ++w) acc[w] = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll 1
                for (int u = 0; u < PB_TCHUNK; ++u) {
                    const int t = t0 + u;
                    uint32_t recvS = __shfl_up_sync(0xffffffffu, L.botX, 1, G);
                    uint32_t recvV = __shfl_up_sync(0xffffffffu, L.botV, 1, G);
                    if (g == 0) { recvS = sc.borderX2; recvV = sc.negb2; }
                    const int j = t - g + 1;
                    uint32_t tw[WPS];
#pragma unroll
                    for (int w = 0; w < WPS; ++w) tw[w] = 0u;
                    // the final-column scout runs inside the step, row by row, and only in the steps in which some lane of the
                    // warp is past the inner columns of a half (G steps per slot for uniform windows): no Vs registers kept
                    const bool in = j >= 1 && j <= nmax;
                    const bool fin = in && need_track && j >= nmin;
                    const bool any_fin = !__all_sync(0xffffffffu, !fin);
                    if (in) {
                        if (any_fin) {
                            FinalCol fc;
                            fc.mask = fin ? ((j == nA ? 1 : 0) | (j == nB ? 2 : 0)) : 0;
                            fc.i0[0] = g * R + 1 - (G * R - mA); fc.i0[1] = g * R + 1 - (G * R - mB);
                            lane_step<R, true, false, false, true>(L, recvS, recvV, hbuf[j - 1], sc, tw, nullptr, nullptr, &fc);
                            if (need_track) lane_track_general<R, false>(L, g, j, make_geom(nA, mA, G, R), make_geom(nB, mB, G, R), nullptr, sc);
                        } else {
                            lane_step<R, true, false>(L, recvS, recvV, hbuf[j - 1], sc, tw);
                            if (need_track) lane_track_lastrow<R>(L, j, sc);
                        }
                    }
#pragma unroll
                    for (int w = 0; w < WPS; ++w) {
                        if (u == 0) acc[w].x = tw[w]; else if (u == 1) acc[w].y = tw[w]; else if (u == 2) acc[w].z = tw[w]; else acc[w].w = tw[w];
                    }
                }
            }
#pragma unroll
            for (int w = 0; w < WPS; ++w)
                *reinterpret_cast<uint4 *>(tr + (((size_t)(t0 / PB_TCHUNK) * WPS + w) * 32 + lane) * PB_TCHUNK) = acc[w];
        }
        // scout candidates -> shared scratch, then lanes g==0 / g==1 finish halves A / B
        cand[lane] = make_cand<R>(L, 0, sc);
        cand[32 + lane] = make_cand<R>(L, 1, sc);
        __syncwarp();
#ifndef PB_EXPERIMENT_SKIP_TRACEBACK   // (profiling experiments only: measure the forward pass alone)
#ifdef PB_EXPERIMENT_PATH_STEPS
        int path_steps = 0;
#endif
        if (g < 2) {
            const int h = g;
            const TbTask tk = tbt[h];
            const HalfGeom gh = make_geom(tk.n, tk.m, G, R);
            if (tk.out_idx >= 0) {
                EndCell end;
                if (tk.flags & TASK_END_GIVEN) {
                    end.j = tk.end_j; end.i = tk.end_i; end.score = tk.end_score; end.corr = tk.flags >> 8;
                    if (tk.n_total <= 0 || gh.m <= 0) end.score = PB_SCORE_EMPTY;
                } else {
                    end = scout_combine(cand + h * 32 + grp * G, G, gh);
                }
#ifdef PB_EXPERIMENT_ALL_HOT   // the scout saw columns past the end: keep the traceback inside the matrix
                end.j = min(end.j, gh.n); end.i = min(end.i, gh.m);
#endif
                TraceCursor<R, WPS> cur;
                cur.init(tr + ((size_t)trace_word<R>(h, 0) * 32 + grp * G) * PB_TCHUNK, end.j, end.i, gh.pad, h, hbuf,
                         ads + tk.ad_off);
                int32_t rec[PB_REC];
                // matches from the score unless the scheme cannot tell a match from a mismatch by score
                const int st = sc.ma != sc.mi ? traceback_stats_cur<true>(cur, end, sc.linear != 0, tk.col0, tk.n_total, gh.m, rec, &sc)
                                              : traceback_stats_cur(cur, end, sc.linear != 0, tk.col0, tk.n_total, gh.m, rec);
                if (st) atomicOr(status, 1);
                int32_t *o = out + (size_t)tk.out_idx * PB_REC;
#pragma unroll
                for (int k = 0; k < PB_REC; ++k) __stcs(o + k, rec[k]);
#ifdef PB_EXPERIMENT_PATH_STEPS
                path_steps = cur.steps;
                atomicAdd(&pb_path_stats[0], (unsigned long long)cur.steps);
                atomicAdd(&pb_path_stats[1], 1ull);
#endif
            }
        }
#ifdef PB_EXPERIMENT_PATH_STEPS
        path_steps = __reduce_max_sync(0xffffffffu, path_steps);
        if (lane == 0) { atomicAdd(&pb_path_stats[2], (unsigned long long)path_steps); atomicAdd(&pb_path_stats[3], 1ull); }
#endif
#endif
        __syncwarp();
        // The slot's trace is dead now: drop its (dirty) L2 lines instead of letting them be written back to HBM
        // when the next slots push them out -- the scratch of all resident warps is about as large as L2.
        for (int l = lane; l < T4 * WPS; l += 32)
            asm volatile("discard.global.L2 [%0], 128;" ::"l"(tr + (size_t)l * 32) : "memory");
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------
// score_kernel: streaming score-only pass for long reads.  Same wavefront, no trace (7 instructions per row:
// 3x VIADDMNMX, LOP3, VIADDMNMX-fused diagonal, VIMNMX, X update), exact scout.  Groups pull slots from a global
// counter and refill independently, so a warp's groups never wait for each other's read lengths.
// Read bases are streamed through a per-group shared-memory ring of packed columns (64 entries = two blocks of 32
// columns).  A block is fetched with aligned 64/32-bit loads (funnel-shifted to the unaligned start) one block
// ahead of its store, which is itself one block ahead of its use: the L2/HBM latency of the stream is never on the
// critical path.  The step loop runs in 32-step segments aligned for the whole warp; refill and staging happen
// only between segments.
constexpr int PB_RING = 64;
constexpr int PB_BLK = 32;
// Ring entries: the packed bases of a column (byte 0 = half A, byte 1 = half B, expanded with one PRMT) or the column's
// profile-table offset, 16 bits each: with 4 KB of ring per block the profile variant (36 KB) fits 6 blocks per SM.
// (-DPB_RING32: the round-1 layout, 32-bit entries in pack_bases form.)
#ifndef PB_RING32
typedef uint16_t ring_t;
__device__ __forceinline__ ring_t ring_pack(uint32_t bA, uint32_t bB) { return (ring_t)(bA | (bB << 8)); }
__device__ __forceinline__ uint32_t ring_bases(uint32_t x) { return __byte_perm(x, 0u, 0x1404); }   // byte1 <- A, byte3 <- B
#else
typedef uint32_t ring_t;
__device__ __forceinline__ ring_t ring_pack(uint32_t bA, uint32_t bB) { return pack_bases(bA, bB); }
__device__ __forceinline__ uint32_t ring_bases(uint32_t x) { return x; }
#endif

// CPL consecutive encoded bytes starting at an arbitrary address, in the low bytes of the result
template <int CPL>
__device__ __forceinline__ uint64_t load_cols(const uint8_t *p) {
    if (CPL == 8) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(p);
        const unsigned long long *q = reinterpret_cast<const unsigned long long *>(a & ~(uintptr_t)7);
        const unsigned sh = (unsigned)(a & 7) * 8;
        const unsigned long long lo = __ldcs(q), hi = __ldcs(q + 1);
        return sh ? ((lo >> sh) | (hi << (64 - sh))) : lo;
    } else if (CPL == 4) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(p);
        const unsigned *q = reinterpret_cast<const unsigned *>(a & ~(uintptr_t)3);
        const unsigned sh = (unsigned)(a & 3) * 8;
        const unsigned lo = __ldcs(q), hi = __ldcs(q + 1);
        return (uint64_t)__funnelshift_r(lo, hi, sh);
    } else {
        uint64_t v = 0;
#pragma unroll
        for (int c = 0; c < CPL; ++c) v |= (uint64_t)__ldcs(p + c) << (8 * c);
        return v;
    }
}

// 6 blocks per SM (<= 85 registers: the profile variant compiles to 79-84 without spills; 36 KB of shared memory per block
// with 16-bit ring entries): the score pass is latency-bound (dependent-chain and shared-memory scoreboard stalls), so more
// resident warps pay.  (Fetching the profile operands one step ahead did not.)
#ifndef PB_SCORE_MIN_BLOCKS
#define PB_SCORE_MIN_BLOCKS 6
#endif
// the computed-operand variant keeps the row operands (16 more registers): 5 blocks per SM (96 registers) without spilling
#ifndef PB_SCORE_MIN_BLOCKS_NOPROF
#define PB_SCORE_MIN_BLOCKS_NOPROF 5
#endif
// PROF = query profile (dp_core.cuh profile_word; option "profile"): every slot aligns ONE read against two adapters
// (cross mode, even number of adapters in the class), so the R substitution operands of a column are fetched from a
// per-group table in shared memory (6 base codes x G*R rows, two 128-bit loads per step) instead of being computed
// (LOP3 + VIADDMNMX per row): 5 instead of 7 instructions per row, 4 instead of 6 on the ALU pipe -- the pipe that bounds
// this kernel.  The ring then holds the table offset of a column's base instead of the packed bases.
// Shared-memory layout (free of bank conflicts -- conflicts, not bytes, bounded an earlier layout of the score pass):
//   profile table   per group and base code two PLANES of G x 4 words: plane 0 holds the operands of every lane's rows 0..3,
//                   plane 1 those of rows 4..7, lane g's four words at g*4.  A 128-bit load of 8 consecutive lanes then reads 32
//                   consecutive words (one wavefront); with G = 4 the two groups of a quarter-warp sit 16 banks apart
//                   (STRIDE = 16 mod 32).  (Keeping a lane's 8 words together would make the first load of 8 lanes
//                   touch only half the banks, twice.)
//   ring            every group's ring is padded to 64 + 2G entries = 32 + G words: all groups of a warp read the same ring index
//                   in the same instruction, and unpadded rings put that index in the same bank for every group (8-way).
template <int G, int R> struct ProfGeom {
    static constexpr int ROWS = G * R;
    static constexpr int PLANE = 4 * G;                 // words per plane
    static constexpr int STRIDE = 6 * ROWS + 16;        // words per group; = 16 mod 32
    static constexpr int RING = PB_RING + 2 * G;        // ring entries per group incl. padding (entries 64.. are never used)
};
template <int G, int R, bool PROF = false>
__global__ void __launch_bounds__(PB_WARPS_PER_BLOCK * 32, PROF ? PB_SCORE_MIN_BLOCKS : PB_SCORE_MIN_BLOCKS_NOPROF)
score_kernel(const TaskSrc ts, unsigned long long *__restrict__ counter,
             const uint8_t *__restrict__ seq, const uint8_t *__restrict__ ads, Scoring sc, EndCell *__restrict__ ends) {
    constexpr int SPW = 32 / G;
    constexpr int CPL = PB_BLK / G;          // columns of a block each lane fetches
    static_assert(!PROF || R == 8, "the profile variant fetches 8 operands per step");
    __shared__ ScoutCand scratch[PB_WARPS_PER_BLOCK][2 * 32];
    __shared__ __align__(16) ring_t rings[PB_WARPS_PER_BLOCK][SPW][ProfGeom<G, R>::RING];
    __shared__ __align__(16) uint32_t profs[PROF ? PB_WARPS_PER_BLOCK * SPW * ProfGeom<G, R>::STRIDE : 4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int grp = lane / G, g = lane % G;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    const int64_t n_tasks = ts.n_tasks;
    const int64_t n_slots = (n_tasks + 1) / 2;
    ScoutCand *cand = scratch[warp];
    ring_t *ring = rings[warp][grp];
    // this lane's rows of the group's profile table (PROF): word [b * ROWS + r] = operand of row g*R + r + 1 for base code b
    uint32_t *myprof = profs + (PROF ? ((size_t)(warp * SPW + grp) * ProfGeom<G, R>::STRIDE + g * 4) : 0);

    Lane<R> L;
    HalfGeom gA, gB;
    const uint8_t *seqA = seq, *seqB = seq;
    int64_t slot = -1;
    int nA = 0, nB = 0, nmax = 0, nmin = 0, T = 0, t = 0;
    bool exhausted = false;
    uint64_t pendA = 0, pendB = 0;           // raw bytes of the block that will be stored at the next block boundary
    gA = make_geom(0, 0, G, R); gB = gA;
    L.botX = sc.borderX2; L.botV = sc.negb2;
    uint32_t top_keep = g != 0 ? 1u : 0u;
    const uint32_t top_addS = g == 0 ? sc.borderX2 : 0u, top_addV = g == 0 ? sc.negb2 : 0u;
    asm volatile("" : "+r"(top_keep));      // opaque: keeps `x * top_keep + add` a multiply-add (the compiler would fold it back into a select)
    if (PROF) {      // a group that never gets a slot still runs the hot segments on dead state: its ring must hold valid offsets
        for (int c = g; c < PB_RING; c += G) ring[c] = (ring_t)0;
        __syncwarp();
    }

    // fetch this lane's CPL columns of block `blk` (raw bytes; columns past the end are fixed up when stored).  PROF: both
    // halves read sequence A, only its bytes are fetched.
    // (Fetch + store are a few % of the kernel's instructions, the loads alone less -- the most a TMA bulk copy into the
    // ring could remove, since the byte -> ring entry conversion and the shared-memory stores stay; not built.  Skipping half B and the per-column bounds tests of
    // interior blocks in the profile variant removes about a third of it.)
    auto fetch = [&](int blk) {
        const int c0 = blk * PB_BLK + g * CPL;
        pendA = (c0 < nA) ? load_cols<CPL>(seqA + c0) : 0ull;
        if (!PROF) pendB = (c0 < nB) ? load_cols<CPL>(seqB + c0) : 0ull;
    };
    // store the pending block into the ring as packed columns: this lane's CPL entries with ONE store (16 / 8 / 4 / 2 bytes;
    // the group rings and a lane's first entry are aligned to that size)
    auto store = [&](int blk) {
        const int c0 = blk * PB_BLK + g * CPL;
        uint32_t e[CPL];
        if (PROF && c0 + CPL <= nA) {        // interior block: every column is a real base of sequence A
#pragma unroll
            for (int c = 0; c < CPL; ++c) e[c] = (uint32_t)((pendA >> (8 * c + 4)) & 0xFu) * (uint32_t)ProfGeom<G, R>::ROWS;
        } else {
#pragma unroll
            for (int c = 0; c < CPL; ++c) {
                const int col = c0 + c;
                const uint32_t bA = (col < nA) ? (uint32_t)((pendA >> (8 * c)) & 0xFFu) : (uint32_t)PB_PAD_H;
                const uint32_t bB = PROF ? bA : ((col < nB) ? (uint32_t)((pendB >> (8 * c)) & 0xFFu) : (uint32_t)PB_PAD_H);
                e[c] = PROF ? (bA >> 4) * (uint32_t)ProfGeom<G, R>::ROWS : (uint32_t)ring_pack(bA, bB);
            }
        }
        ring_t *dst = ring + (c0 & (PB_RING - 1));
#ifndef PB_RING32
        if (CPL == 8) *reinterpret_cast<uint4 *>(dst) = make_uint4(e[0] | (e[1 % CPL] << 16), e[2 % CPL] | (e[3 % CPL] << 16),
                                                                    e[4 % CPL] | (e[5 % CPL] << 16), e[6 % CPL] | (e[7 % CPL] << 16));
        else if (CPL == 4) *reinterpret_cast<uint2 *>(dst) = make_uint2(e[0] | (e[1 % CPL] << 16), e[2 % CPL] | (e[3 % CPL] << 16));
        else if (CPL == 2) *reinterpret_cast<uint32_t *>(dst) = e[0] | (e[1 % CPL] << 16);
        else dst[0] = (ring_t)e[0];
#else
#pragma unroll
        for (int c = 0; c < CPL; ++c) dst[c] = (ring_t)e[c];
#endif
    };

    for (;;) {
        // every read of the previous segment is ordered before the ring stores below.  (The lanes cannot drift apart anyway --
        // each step's full-mask shuffle joins them, and a block is overwritten 25+ steps after its last read -- but a shuffle
        // is not a memory barrier: compute-sanitizer racecheck reports the write-after-read pair without it.)
        __syncwarp();
        if (!exhausted) {
            if (t >= T) {                      // group-uniform: this group's slot is finished (or none yet)
                if (slot >= 0) {
                    cand[lane] = make_cand<R>(L, 0, sc);
                    cand[32 + lane] = make_cand<R>(L, 1, sc);
                    __syncwarp(gmask);
                    if (g < 2) {
                        const int64_t ti = slot * 2 + g;
                        if (ti < n_tasks) ends[ti] = scout_combine(cand + g * 32 + grp * G, G, g ? gB : gA);
                    }
                    __syncwarp(gmask);
                }
                unsigned long long s = 0;
                if (g == 0) s = atomicAdd(counter, 1ull);
                s = __shfl_sync(gmask, s, 0, G);
                if ((int64_t)s >= n_slots) {
                    exhausted = true; slot = -1; T = 0; t = 0; nmax = 0; nmin = 0; nA = nB = 0;
                } else {
                    slot = (int64_t)s;
                    const Task tA = get_task(ts, slot * 2);
                    const Task tB = get_task(ts, slot * 2 + 1);
                    nA = tA.n; nB = tB.n;
                    gA = make_geom(tA.n, tA.m, G, R); gB = make_geom(tB.n, tB.m, G, R);
                    nmax = max(nA, nB);
                    seqA = seq + tA.seq_off; seqB = seq + tB.seq_off;
                    lane_init<R>(L, g, G, sc, ads + tA.ad_off, tA.m, false, ads + tB.ad_off, tB.m, false);
                    if (PROF) {
                        // both halves read sequence A (the launcher guarantees same-read slots); every lane fills, and later
                        // reads, only its own rows of the table -- no synchronisation needed
#pragma unroll
                        for (int b = 0; b < 6; ++b) {       // from the row operands lane_init has just set up: two 128-bit stores
                            uint32_t w[8];
#pragma unroll
                            for (int r = 0; r < 8; ++r) w[r] = PB_PROF_ENCODE(profile_from(L.v2[r], L.sf2[r], (uint32_t)b, sc));
                            uint32_t *dst = myprof + b * ProfGeom<G, R>::ROWS;
                            *reinterpret_cast<uint4 *>(dst) = make_uint4(w[0], w[1], w[2], w[3]);
                            *reinterpret_cast<uint4 *>(dst + ProfGeom<G, R>::PLANE) = make_uint4(w[4], w[5], w[6], w[7]);
                        }
                    }
                    const bool emptyA = tA.n <= 0 || tA.m <= 0, emptyB = tB.n <= 0 || tB.m <= 0;
                    nmin = emptyA ? nB : (emptyB ? nA : min(nA, nB));
                    T = nmax + G - 1; t = 0;
                    fetch(0); store(0);         // first block: its latency is exposed once per slot
                    fetch(1);
                }
            } else {                               // block boundary: publish block t/32, prefetch the next one
                store(t / PB_BLK);
                fetch(t / PB_BLK + 1);
            }
        }
        __syncwarp();
        if (__all_sync(0xffffffffu, exhausted)) break;
        // One segment = PB_BLK steps.  Every group of the warp starts its slots on a segment boundary (a group that
        // finishes inside a segment idles for the < 32 remaining steps, ~0.2 % of an 8-kb read), so all block boundaries
        // of the warp coincide and the step loop carries no refill / staging checks.
        // A segment is "hot" when every lane of every (live) group stays inside its matrix and in inner columns for
        // all 32 steps: straight-line code, fast scout only.  Exhausted groups just compute on dead state.
        const bool hot = __all_sync(0xffffffffu, exhausted || (t >= G - 1 && t + PB_BLK < nmin));
        if (hot) {
#pragma unroll 4
            for (int k = 0; k < PB_BLK; ++k) {
                uint32_t recvS = __shfl_up_sync(0xffffffffu, L.botX, 1, G);
                uint32_t recvV = __shfl_up_sync(0xffffffffu, L.botV, 1, G);
                // lane 0 of a group takes the border instead: as a multiply-add (x * 0 + border / x * 1 + 0) the two selects are
                // FMA-heavy work -- the ALU pipe is the busier one in this kernel
                recvS = recvS * top_keep + top_addS;
                recvV = recvV * top_keep + top_addV;
                const int j = t - g + 1;
                const uint32_t hx = ring[(j - 1) & (PB_RING - 1)];      // packed bases (ring form), or (PROF) the table offset of the base
                if (PROF) {
                    const uint4 p0 = *reinterpret_cast<const uint4 *>(myprof + hx);
                    const uint4 p1 = *reinterpret_cast<const uint4 *>(myprof + hx + ProfGeom<G, R>::PLANE);
                    const uint32_t subs[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
                    lane_step<R, false, false, true>(L, recvS, recvV, 0u, sc, nullptr, nullptr, subs);
                } else {
                    lane_step<R, false, false>(L, recvS, recvV, ring_bases(hx), sc, nullptr);
                }
                lane_track_lastrow<R>(L, j, sc);
                ++t;
            }
        } else {
#pragma unroll 1
            for (int k = 0; k < PB_BLK; ++k) {
                uint32_t recvS = __shfl_up_sync(0xffffffffu, L.botX, 1, G);
                uint32_t recvV = __shfl_up_sync(0xffffffffu, L.botV, 1, G);
                if (g == 0) { recvS = sc.borderX2; recvV = sc.negb2; }
                const int j = t - g + 1;
                if (j >= 1 && j <= nmax) {          // nmax == 0 for exhausted groups
                    const uint32_t h2 = ring[(j - 1) & (PB_RING - 1)];          // ring form: see ring_bases
                    uint32_t vr[R];
                    if (PROF) {
                        const uint4 p0 = *reinterpret_cast<const uint4 *>(myprof + h2);
                        const uint4 p1 = *reinterpret_cast<const uint4 *>(myprof + h2 + ProfGeom<G, R>::PLANE);
                        const uint32_t subs[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
                        lane_step<R, false, true, true>(L, recvS, recvV, 0u, sc, nullptr, vr, subs);
                    } else {
                        lane_step<R, false, true>(L, recvS, recvV, ring_bases(h2), sc, nullptr, vr);
                    }
                    if (j < nmin) lane_track_lastrow<R>(L, j, sc);
                    else lane_track_general<R>(L, g, j, gA, gB, vr, sc);
                }
                ++t;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// decide_kernel: records of one chunk (n reads x n_adapters, read-major, still in HBM/L2 from the DP kernels) -> per read
// the end-trim amount (max over the adapters that pass, 0 if none) and the (match_ad, len_ad) pairs of the barcode score
// columns.  One warp per read; 4 + 4*n_cols bytes per read leave the device instead of 36*n_adapters.
struct DecideArgs {
    const int32_t *records; int64_t n; int32_t n_adapters;
    int32_t is_start, end_size, extra_trim, min_trim;
    const int32_t *cmin; int32_t cmin_len;
    const int32_t *cols; int32_t n_cols;
    int32_t *trim; uint32_t *pairs;
    int32_t *top2;            // optional: 6 int32 per read (best / second-best score column), see barcode_key
};
// Ordering key of a barcode score column for determine_barcode's `sorted(..., reverse=True, key=score)`
// (porechop/nanopore_read.py:404-407): larger full-adapter identity first, equal identities keep their column order (Python's
// sort is stable).  The identity is float("%f" % (100.0 * c / l)); for l < 4096 two different fractions differ by more than
// 2^-24, far more than the 1e-6 of "%f", and equal fractions print identically, so ordering the fractions orders the floats:
// key = [valid | floor(c * 2^32 / l) | 0xFFFF - position], compared as one unsigned 64-bit number.
__device__ __forceinline__ unsigned long long barcode_key(uint32_t pair, int pos) {
    const unsigned long long c = pair & 0xFFFFu, l = pair >> 16;
    return (1ull << 62) | (((c << 32) / (l ? l : 1ull)) << 16) | (unsigned long long)(0xFFFF - pos);
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o); v = w > v ? w : v; }
    return v;
}
__global__ void decide_kernel(const DecideArgs a, int *__restrict__ status) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int ovf = 0;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n; i += warps) {
        const int32_t *rec = a.records + (size_t)i * a.n_adapters * PB_REC;
        int32_t best = 0;
        for (int32_t k = lane; k < a.n_adapters; k += 32) {
            int32_t r[PB_REC];
#pragma unroll
            for (int q = 0; q < PB_REC; ++q) r[q] = rec[(size_t)k * PB_REC + q];
            const int32_t t = end_trim_candidate(r, a.is_start, a.end_size, a.extra_trim, a.min_trim, a.cmin, a.cmin_len, &ovf);
            best = t > best ? t : best;
        }
        best = __reduce_max_sync(0xffffffffu, best);
        if (lane == 0) a.trim[i] = best;
        unsigned long long b1 = 0, b2 = 0;          // this lane's best and second-best column keys (0 = none)
        for (int32_t k = lane; k < a.n_cols; k += 32) {
            const int32_t *r = rec + (size_t)a.cols[k] * PB_REC;
            int32_t rr[PB_REC];
#pragma unroll
            for (int q = 0; q < PB_REC; ++q) rr[q] = r[q];
            const uint32_t pr = score_pair(rr, &ovf);
            if (a.pairs) a.pairs[(size_t)i * a.n_cols + k] = pr;
            if (a.top2) {
                if ((pr >> 16) >= 4096u || k >= 0xFFFF) ovf = 1;         // outside the key's exactness domain (never for end windows)
                const unsigned long long key = barcode_key(pr, k);
                if (key > b1) { b2 = b1; b1 = key; } else if (key > b2) b2 = key;
            }
        }
        if (a.top2) {
            // best of the warp, then the best of what is left (the winner's lane offers its own second)
            const unsigned long long w1 = warp_max_u64(b1);
            const unsigned long long w2 = warp_max_u64(b1 == w1 ? b2 : b1);
            if (lane == 0) {
                int32_t *o = a.top2 + (size_t)i * 6;
                const unsigned long long w[2] = {w1, w2};
#pragma unroll
                for (int t = 0; t < 2; ++t) {
                    if (w[t]) {
                        const int pos = 0xFFFF - (int)(w[t] & 0xFFFFull);
                        const int32_t *r = rec + (size_t)a.cols[pos] * PB_REC;
                        int32_t rr[PB_REC];
#pragma unroll
                        for (int q = 0; q < PB_REC; ++q) rr[q] = r[q];
                        const uint32_t pr = score_pair(rr, &ovf);
                        o[3 * t] = pos; o[3 * t + 1] = (int32_t)(pr & 0xFFFFu); o[3 * t + 2] = (int32_t)(pr >> 16);
                    } else {
                        o[3 * t] = -1; o[3 * t + 1] = 0; o[3 * t + 2] = 1;
                    }
                }
            }
        }
    }
    if (ovf) atomicOr(status, 2);
}

// ---------------------------------------------------------------------------------------------------
// search_best_kernel: records of one chunk (n reads x n_adapters, read-major, still in L2 from the DP kernels) -> per adapter
// the largest full-adapter identity, max-reduced into `best` (the stage's accumulator columns of the batch).  The key of a
// record is the bit pattern of d = 100.0 * c / l in IEEE double: 100 * c is exact and the division rounds to nearest, so d
// is non-decreasing in c / l, and so is float("%f" % d) -- the largest key is the record with the largest Python float, and
// a non-negative double's bits order like its value.  Records with l == 0 (failed alignments, empty windows) are skipped;
// 0 is the key of +0.0, the reference's starting score.  Keys are reduced in shared memory first (one u64 per adapter,
// use_smem = 1), then with one global atomic per adapter per block; use_smem = 0 (too many adapters for a block) goes
// straight to `best`.  Plain arguments, no argument struct: `records` is only read, `best` is only updated atomically.
__device__ __forceinline__ unsigned long long percent_key(int32_t c, int32_t l) {
    const double d = 100.0 * (double)c / (double)l;
#if defined(__CUDA_ARCH__)
    return (unsigned long long)__double_as_longlong(d);
#else
    unsigned long long k;
    memcpy(&k, &d, sizeof k);
    return k;
#endif
}
__global__ void search_best_kernel(const int32_t *__restrict__ records, int64_t n, int32_t n_adapters, unsigned long long *best,
                                   int use_smem) {
    extern __shared__ uint32_t smem[];
    unsigned long long *acc = use_smem ? reinterpret_cast<unsigned long long *>(smem) : best;
    if (use_smem) {
        for (int k = threadIdx.x; k < n_adapters; k += blockDim.x) acc[k] = 0ull;
        __syncthreads();
    }
    const int64_t total = n * n_adapters;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int32_t col = (int32_t)(i % n_adapters);
    const int32_t step = (int32_t)(stride % n_adapters);
    for (; i < total; i += stride) {
        const int32_t *r = records + (size_t)i * PB_REC;
        const int32_t l = r[8];
        if (l > 0) {
            const unsigned long long key = percent_key(r[7], l);
            if (key > acc[col]) atomicMax(&acc[col], key);       // the plain read only skips atomics that cannot raise it
        }
        col += step;
        if (col >= n_adapters) col -= n_adapters;
    }
    if (use_smem) {
        __syncthreads();
        for (int k = threadIdx.x; k < n_adapters; k += blockDim.x)
            if (acc[k]) atomicMax(&best[k], acc[k]);
    }
}

// ---------------------------------------------------------------------------------------------------
// middle_decide_kernel: one round of find_middle_adapters (porechop/nanopore_read.py:216-243) over the active reads of a
// resident segment.  One warp per read: the first adapter from the read's current one onward whose record hits
// (middle_hit) is the round's hit; the warp masks read positions [rs, re] with the N code in the resident code buffer
// (the byte encode_kernel writes for the reference's '-'), keeps the adapter as the read's next one and appends the read
// to the next round's active list.  A read without a hit leaves the active set.  Reads own disjoint byte ranges, so the
// masking needs no synchronisation between warps.  The append position varies from run to run; the hit is written at
// that position together with the read id (next_active), and the host orders the hits by (read, round), so the result
// does not depend on it.  Round 0: active == nullptr, the reads are first .. first+n-1 and every read starts at adapter 0.
struct MiddleArgs {
    const int32_t *records; int32_t n_adapters;   // segment-wide, read-major: read s's records start at s * n_adapters
    const int32_t *active; int64_t first, n;      // this round's reads (segment-relative ids), or nullptr (round 0)
    int32_t *next_ad;                             // per read: the adapter its next round starts from
    const int64_t *seq_off; uint8_t *codes;       // resident offsets (indexed by read id) and codes of the segment
    const int32_t *cmin; int32_t cmin_len;
    int32_t *hits;                                // out: PB200_HIT_INTS ints per hit {adapter, record}, at the append position
    int32_t *next_active;                         // out: the read id at the append position
    unsigned *count;                              // append counter (= hits of the round)
    unsigned long long *max_len;                  // longest appended read (sizes the next round's DP launch)
};
constexpr int PB_HIT_INTS = 1 + PB_REC;
constexpr uint8_t PB_CODE_N = 4u << 4;
__global__ void middle_decide_kernel(const MiddleArgs a, int *__restrict__ status) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    int ovf = 0;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < a.n; i += warps) {
        const int64_t s = a.active ? (int64_t)a.active[i] : a.first + i;
        const int32_t k0 = a.active ? a.next_ad[s] : 0;
        const int32_t *rec = a.records + (size_t)s * a.n_adapters * PB_REC;
        int hit = 0x7fffffff;
        for (int32_t kb = k0; kb < a.n_adapters && hit == 0x7fffffff; kb += 32) {
            const int32_t k = kb + lane;
            int mine = 0x7fffffff;
            if (k < a.n_adapters) {
                int32_t r[PB_REC];
#pragma unroll
                for (int q = 0; q < PB_REC; ++q) r[q] = rec[(size_t)k * PB_REC + q];
                if (middle_hit(r, a.cmin, a.cmin_len, &ovf)) mine = k;
            }
            hit = __reduce_min_sync(0xffffffffu, mine);
        }
        if (hit == 0x7fffffff) continue;              // warp-uniform: the read leaves the active set
        const int32_t *r = rec + (size_t)hit * PB_REC;
        const int64_t o0 = a.seq_off[s], len = a.seq_off[s + 1] - o0;
        const int32_t rs = r[0], re = r[1];
        if (rs < 0 || re < rs || re >= len) { ovf = 1; continue; }
        for (int64_t p = rs + lane; p <= re; p += 32) a.codes[o0 + p] = PB_CODE_N;
        unsigned pos = 0;
        if (lane == 0) {
            pos = atomicAdd(a.count, 1u);
            atomicMax(a.max_len, (unsigned long long)len);
            a.next_ad[s] = hit;
            a.next_active[pos] = (int32_t)s;
        }
        pos = __shfl_sync(0xffffffffu, pos, 0);
        if (lane < PB_HIT_INTS) a.hits[(size_t)pos * PB_HIT_INTS + lane] = lane == 0 ? hit : r[lane - 1];
    }
    if (ovf) atomicOr(status, 2);
}

// ---------------------------------------------------------------------------------------------------
// Whole-read trimming (adapterTrimReads): the glue between resident reads, the end-window DP of Phase B and the middle scan.
// Reads are ASCII at reads[off[s] .. off[s+1]); every kernel takes plain pointers (const = read, non-const = written).
//
// Lengths -> offsets: a length kernel writes len[s] into x[s+1] (and 0 into x[0]); the three scan kernels then turn
// x[1 .. n] into its inclusive prefix sums in place (reduce per tile, scan the tile sums in one block, scan each tile with its
// prefix), so that x becomes the exclusive offsets of the lengths.  A tile is PB_SCAN_THREADS x PB_SCAN_ITEMS values.
constexpr int PB_SCAN_THREADS = 256;
constexpr int PB_SCAN_ITEMS = 8;
constexpr int64_t PB_SCAN_TILE = (int64_t)PB_SCAN_THREADS * PB_SCAN_ITEMS;

// exclusive scan of one value per thread over the block (blockDim.x a multiple of 32); *total = the block's sum
__device__ __forceinline__ long long block_exclusive_scan(long long v, long long *total) {
    __shared__ long long warp_tot[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    long long inc = v;
    for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_tot[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        long long w = lane < n_warps ? warp_tot[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += t;
        }
        if (lane < n_warps) warp_tot[lane] = w;          // inclusive over the warps
    }
    __syncthreads();
    const long long excl = inc - v + (warp ? warp_tot[warp - 1] : 0);
    *total = warp_tot[n_warps - 1];
    __syncthreads();                                       // warp_tot may be reused by the caller's next scan
    return excl;
}
// tile sums of x[0 .. n): one block per tile
__global__ void scan_tiles_kernel(const int64_t *x, int64_t n, int64_t *tile_sums) {
    const int64_t base = (int64_t)blockIdx.x * PB_SCAN_TILE + (int64_t)threadIdx.x * PB_SCAN_ITEMS;
    long long s = 0;
    for (int k = 0; k < PB_SCAN_ITEMS; ++k) if (base + k < n) s += x[base + k];
    long long total = 0;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
// exclusive scan of the n tile sums in place: one block, each thread a contiguous run
__global__ void scan_tile_sums_kernel(int64_t *tile_sums, int64_t n) {
    const int64_t per = (n + blockDim.x - 1) / blockDim.x;
    const int64_t lo = (int64_t)threadIdx.x * per, hi = lo + per < n ? lo + per : n;
    long long s = 0;
    for (int64_t i = lo; i < hi; ++i) s += tile_sums[i];
    long long total = 0;
    long long run = block_exclusive_scan(s, &total);
    for (int64_t i = lo; i < hi; ++i) { const long long v = tile_sums[i]; tile_sums[i] = run; run += v; }
}
// inclusive scan of x[0 .. n) in place, tile by tile from the tile's exclusive prefix
__global__ void scan_apply_kernel(int64_t *x, int64_t n, const int64_t *tile_sums) {
    const int64_t base = (int64_t)blockIdx.x * PB_SCAN_TILE + (int64_t)threadIdx.x * PB_SCAN_ITEMS;
    long long v[PB_SCAN_ITEMS], s = 0;
#pragma unroll
    for (int k = 0; k < PB_SCAN_ITEMS; ++k) { v[k] = base + k < n ? x[base + k] : 0; s += v[k]; }
    long long total = 0;
    long long run = block_exclusive_scan(s, &total) + tile_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < PB_SCAN_ITEMS; ++k) {
        run += v[k];
        if (base + k < n) x[base + k] = run;
    }
}

// window lengths min(len, end_size) of every read -> wl[s + 1] (wl[0] = 0): scanned, the offsets of the start windows and of the
// end windows alike
__global__ void window_len_kernel(const int64_t *off, int64_t n, int64_t end_size, int64_t *wl) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s == 0) wl[0] = 0;
    if (s < n) {
        const int64_t len = off[s + 1] - off[s];
        wl[s + 1] = len < end_size ? len : end_size;
    }
}
// seq[:wl] and seq[len - wl:] of every read (ASCII, nanopore_read.py:172,194) -> the two window batches; one warp per read
__global__ void cut_windows_kernel(const uint8_t *reads, const int64_t *off, const int64_t *win_off, int64_t n, uint8_t *start,
                                   uint8_t *end) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < n; s += warps) {
        const int64_t w0 = win_off[s], wl = win_off[s + 1] - w0, tail = off[s + 1] - wl;
        for (int64_t k = lane; k < wl; k += 32) {
            start[w0 + k] = reads[off[s] + k];
            end[w0 + k] = reads[tail + k];
        }
    }
}
// [a, b) of seq[start_trim : len - end_trim] with Python's slice semantics (fastq.trimmed_ranges, nanopore_read.py:57-63): an
// end position below 0 counts from the end of the read again, an untouched read keeps [0, len).  first[s] = a,
// lens[s + 1] = b - a (lens[0] = 0) for the scan into the trimmed reads' offsets.
__global__ void trimmed_range_kernel(const int64_t *off, const int32_t *start_trim, const int32_t *end_trim, int64_t n,
                                     int64_t *first, int64_t *lens) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s == 0) lens[0] = 0;
    if (s >= n) return;
    const int64_t len = off[s + 1] - off[s], st = start_trim[s], et = end_trim[s];
    int64_t a = 0, b = len;
    if (st != 0 || et != 0) {
        int64_t e = len - et;
        if (e < 0) e = e + len > 0 ? e + len : 0;
        a = st < len ? st : len;
        b = e < len ? e : len;
        if (b < a) b = a;
    }
    first[s] = a;
    lens[s + 1] = b - a;
}
// the trimmed reads, encoded on the way (the bytes encode_kernel writes), into the middle scan's resident codes at dst_off;
// one warp per read
__global__ void gather_encode_kernel(const uint8_t *reads, const int64_t *off, const int64_t *first, const int64_t *dst_off,
                                     int64_t n, uint8_t *codes) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; s < n; s += warps) {
        const uint8_t *src = reads + off[s] + first[s];
        const int64_t d0 = dst_off[s], len = dst_off[s + 1] - d0;
        for (int64_t k = lane; k < len; k += 32) codes[d0 + k] = (uint8_t)encode_byte(src[k]);
    }
}

// ---------------------------------------------------------------------------------------------------
// Output stage of adapterTrimSplitReadsDevice, once per segment: the records Porechop writes (get_fastq / get_fasta) cut from
// the caller's reads.  Count records and bases per read, scan both, write each record's source, part number and output
// offset, then gather the bases (and qualities) into the caller's output buffers.
//
// What the segment's reads look like to the stage (all read only): reads at off[s] .. off[s+1]; the trimmed range starts at
// first[s] and is toff[s+1] - toff[s] long; hit_of[s] = -1 for a read without a middle hit, else its row of the CSR
// rng_off / rng of extended hit ranges (trimmed-read coordinates, sorted by start).  The kernels take these as plain pointer
// arguments (so that each is an access of its own, read because it is const) and assemble the view below themselves.
#define PB_SPLIT_READS_PARAMS const int64_t *off, const int64_t *first, const int64_t *toff, const int32_t *hit_of, \
                              const int32_t *rng_off, const int32_t *rng, int64_t n, int64_t min_split, int32_t discard_middle, \
                              int32_t untrimmed
#define PB_SPLIT_READS_VIEW {off, first, toff, hit_of, rng_off, rng, n, min_split, discard_middle, untrimmed}
struct SplitReads {
    const int64_t *off, *first, *toff;
    const int32_t *hit_of, *rng_off, *rng;
    int64_t n, min_split;
    int32_t discard_middle, untrimmed;
};
// the output records of read s: f(part, source offset, length) in position order; returns their number
template <class F>
__device__ __forceinline__ int64_t read_records(const SplitReads &r, int64_t s, F &&f) {
    const int64_t base = r.off[s], a = r.first[s], tl = r.toff[s + 1] - r.toff[s];
    const int32_t h = r.hit_of[s];
    if (h < 0) {                                  // not split: the trimmed read (the whole read with --untrimmed), if not empty
        const int64_t l = r.untrimmed ? r.off[s + 1] - base : tl;
        if (l <= 0) return 0;
        f(0, r.untrimmed ? base : base + a, l);
        return 1;
    }
    if (r.discard_middle) return 0;
    const int32_t k0 = r.rng_off[h];
    return split_runs(tl, r.rng + 2 * (int64_t)k0, r.rng_off[h + 1] - k0, r.min_split,
                      [&](int64_t k, int64_t x, int64_t y) { f(k + 1, base + a + x, y - x); });
}
// hit_of[hit_reads[i]] = i (hit_of was set to -1)
__global__ void split_mark_kernel(const int32_t *hit_reads, int64_t n_hit_reads, int32_t *hit_of) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_hit_reads) hit_of[hit_reads[i]] = (int32_t)i;
}
// records and bases of every read -> cnt[s + 1], bytes[s + 1] (cnt[0] = bytes[0] = 0), for scan_offsets
__global__ void split_count_kernel(PB_SPLIT_READS_PARAMS, int64_t *cnt, int64_t *bytes) {
    const SplitReads r = PB_SPLIT_READS_VIEW;
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s == 0) { cnt[0] = 0; bytes[0] = 0; }
    if (s >= r.n) return;
    int64_t b = 0;
    cnt[s + 1] = read_records(r, s, [&](int64_t, int64_t, int64_t l) { b += l; });
    bytes[s + 1] = b;
}
// the records of the segment from the scanned counts: record rec0 + rec_off[s] + j of read read0 + s gets its output offset
// byte0 + ..., read, part and (segment-relative record index) source offset; thread 0 also writes the offset after the
// segment's last record
__global__ void split_write_kernel(PB_SPLIT_READS_PARAMS, const int64_t *rec_off, const int64_t *byte_off, int64_t rec0,
                                   int64_t byte0, int64_t read0, int64_t *src, int64_t *out_off, int32_t *out_read,
                                   int32_t *out_part) {
    const SplitReads r = PB_SPLIT_READS_VIEW;
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s == 0) out_off[rec0 + rec_off[r.n]] = byte0 + byte_off[r.n];
    if (s >= r.n) return;
    int64_t i = rec_off[s], pos = byte0 + byte_off[s];
    read_records(r, s, [&](int64_t part, int64_t from, int64_t l) {
        out_off[rec0 + i] = pos;
        out_read[rec0 + i] = (int32_t)(read0 + s);
        out_part[rec0 + i] = (int32_t)part;
        src[i] = from;
        ++i;
        pos += l;
    });
}
// Byte maps of warp_copy, applied to 32-bit words of four bytes (a single byte is a word with three zero bytes).
struct CopyBytes {
    __device__ __forceinline__ unsigned operator()(unsigned w) const { return w; }
};
struct CopyTtoU {   // every 'T' byte becomes 'U' (0x54 -> 0x55), nothing else changes: RNA reads (get_fastq / get_fasta)
    __device__ __forceinline__ unsigned operator()(unsigned w) const {
        const unsigned t = w ^ 0x54545454u;                                          // zero bytes where w has a 'T'
        const unsigned nz = ((t & 0x7f7f7f7fu) + 0x7f7f7f7fu) | t;                   // high bit set in every nonzero byte
        return w + ((~nz & 0x80808080u) >> 7);                                       // +1 in the 'T' bytes (no carry out)
    }
};
// dst[0 .. n) = f(src[0 .. n)) by one warp: the bytes up to dst's next 16-byte boundary one per lane, then aligned 16-byte stores
// assembled from aligned 16-byte loads (each lane's chunk and the next lane's, shifted into place with __funnelshift_r), then
// the last bytes one per lane.  Loads never leave [src & ~15, src + n): the body stops where its next chunk would.
template <class F = CopyBytes>
__device__ __forceinline__ void warp_copy(const uint8_t *src, uint8_t *dst, int64_t n, int lane, F f = F()) {
    int64_t h = (int64_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (h > n) h = n;
    if (lane < h) dst[lane] = (uint8_t)f(src[lane]);
    const uintptr_t s1 = (uintptr_t)(src + h);
    const uint4 *A = reinterpret_cast<const uint4 *>(s1 & ~(uintptr_t)15);
    const int o = (int)(s1 & 15), q = o >> 2;
    const unsigned sh = (unsigned)(o & 3) * 8;
    const int64_t rem = n - h;
    int64_t nvec = o ? ((rem + o) >> 4) - 1 : rem >> 4;     // 16-byte stores; their chunks (+ the next one if o > 0) fit
    if (nvec < 0) nvec = 0;
    const int64_t nchunk = nvec + (o ? 1 : 0);
    uint4 *D = reinterpret_cast<uint4 *>(dst + h);
    for (int64_t v0 = 0; v0 < nvec; v0 += 32) {              // warp-uniform trip count
        const int64_t v = v0 + lane;
        const uint4 c = v < nchunk ? A[v] : make_uint4(0u, 0u, 0u, 0u);
        uint4 d;
        d.x = __shfl_sync(0xffffffffu, c.x, (lane + 1) & 31);
        d.y = __shfl_sync(0xffffffffu, c.y, (lane + 1) & 31);
        d.z = __shfl_sync(0xffffffffu, c.z, (lane + 1) & 31);
        d.w = __shfl_sync(0xffffffffu, c.w, (lane + 1) & 31);
        if (lane == 31 && v + 1 < nchunk) d = A[v + 1];
        // words o/4 .. o/4 + 4 of the 32 bytes c:d, then shifted right by (o & 3) bytes
        const bool q2 = q & 2, q1 = q & 1;
        const unsigned t0 = q2 ? c.z : c.x, t1 = q2 ? c.w : c.y, t2 = q2 ? d.x : c.z, t3 = q2 ? d.y : c.w, t4 = q2 ? d.z : d.x,
                       t5 = q2 ? d.w : d.y;
        const unsigned u0 = q1 ? t1 : t0, u1 = q1 ? t2 : t1, u2 = q1 ? t3 : t2, u3 = q1 ? t4 : t3, u4 = q1 ? t5 : t4;
        if (v < nvec)
            D[v] = make_uint4(f(__funnelshift_r(u0, u1, sh)), f(__funnelshift_r(u1, u2, sh)), f(__funnelshift_r(u2, u3, sh)),
                              f(__funnelshift_r(u3, u4, sh)));
    }
    const int64_t t = h + 16 * nvec;                         // at most 30 bytes are left
    if (lane < n - t) dst[t + lane] = (uint8_t)f(src[t + lane]);
}
// bases (and qualities) of records [0, n_rec) of the segment: source src[i], output out_off[i] .. out_off[i + 1] (out_off = the
// caller's offsets from the segment's first record on); one warp per record
__global__ void __launch_bounds__(256) split_gather_kernel(const uint8_t *__restrict__ seq, const uint8_t *__restrict__ qual,
                                                           const int64_t *__restrict__ src, const int64_t *__restrict__ out_off,
                                                           int64_t n_rec, uint8_t *__restrict__ out_seq,
                                                           uint8_t *__restrict__ out_qual) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_rec; i += warps) {
        const int64_t from = src[i], to = out_off[i], len = out_off[i + 1] - to;
        warp_copy(seq + from, out_seq + to, len, lane);
        if (qual) warp_copy(qual + from, out_qual + to, len, lane);
    }
}

// ---------------------------------------------------------------------------------------------------
// pb200EmitReadsDevice: the bytes Porechop writes for records in device memory (get_fastq / get_fasta, fastq.emit_parts).
// Record r: bases seq[off[r] .. off[r + 1]) (qualities at the same offsets), source read read[r], part part[r] (k >= 1: '_k'
// goes before the first space of the name, add_number_to_read_name); names[name_off[s] .. name_off[s + 1]) of read s.
// FASTQ: '@' name '\n' bases '\n' '+' '\n' quals '\n'; FASTA: '>' name '\n' and the bases in lines of 70, each ending in '\n'.

// decimal digits of k >= 1
__device__ __forceinline__ int emit_digits(int32_t k) {
    int d = 1;
    for (int64_t p = 10; p <= k; p *= 10) ++d;
    return d;
}
// byte length of record r, and whether its arrays are in range (checked here because they come from outside the library)
__device__ __forceinline__ int64_t emit_record_len(int64_t sl, int64_t nl, int32_t part, int32_t fmt) {
    const int64_t name = nl + (part > 0 ? 1 + emit_digits(part) : 0);
    return fmt == 0 ? 6 + name + 2 * sl : 2 + name + sl + (sl + 69) / 70;
}
// len[r + 1] = byte length of record r (len[0] = 0), for scan_offsets; a record that fails a check gets length 0 and sets
// *bad.  One thread per record.
__global__ void emit_count_kernel(const int64_t *off, const int32_t *read, const int32_t *part, const int64_t *name_off,
                                  int64_t n_rec, int64_t seq_bytes, int64_t n_reads, int64_t name_bytes, int32_t fmt, int64_t *len,
                                  int *bad) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) len[0] = 0;
    if (r >= n_rec) return;
    const int64_t a = off[r], b = off[r + 1];
    const int32_t s = read[r], k = part[r];
    bool ok = 0 <= a && a <= b && b <= seq_bytes && 0 <= s && s < n_reads && k >= 0;
    int64_t nl = 0;
    if (ok) {
        const int64_t n0 = name_off[s], n1 = name_off[s + 1];
        ok = 0 <= n0 && n0 <= n1 && n1 <= name_bytes;
        nl = n1 - n0;
    }
    if (!ok) atomicOr(bad, 1);
    len[r + 1] = ok ? emit_record_len(b - a, nl, k, fmt) : 0;
}
// the records at out + out_off[r] (scanned by emit_count_kernel + scan_offsets; every check passed); one warp per record.
// Names and the FASTA lines go one byte per lane; FASTQ bases and qualities through warp_copy.
__global__ void __launch_bounds__(256) emit_write_kernel(const uint8_t *seq, const uint8_t *qual, const int64_t *off,
                                                         const int32_t *read, const int32_t *part, const uint8_t *names,
                                                         const int64_t *name_off, const uint8_t *rna, int32_t fmt,
                                                         const int64_t *out_off, int64_t n_rec, uint8_t *out) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_rec; r += warps) {
        const int64_t s0 = off[r], sl = off[r + 1] - s0;
        const int32_t s = read[r], k = part[r];
        const int64_t n0 = name_off[s], nl = name_off[s + 1] - n0;
        const uint8_t *nm = names + n0;
        uint8_t *p = out + out_off[r];
        // ---- the name: the tag '_k' (td bytes) goes at sp, the first space (or the end) ----
        int td = 0;
        int64_t sp = nl;
        if (k > 0) {
            td = 1 + emit_digits(k);
            for (int64_t c = 0; c < nl; c += 32) {                // warp-uniform: 32 name bytes a step
                const int64_t j = c + lane;
                const int first = __reduce_min_sync(0xffffffffu, (j < nl && nm[j] == ' ') ? lane : 32);
                if (first < 32) { sp = c + first; break; }
            }
        }
        if (lane == 0) p[0] = fmt == 0 ? '@' : '>';
        const int64_t L = nl + td;
        for (int64_t j = lane; j < L; j += 32) {
            uint8_t v;
            if (j < sp) v = nm[j];
            else if (j >= sp + td) v = nm[j - td];
            else if (j == sp) v = '_';
            else {                                                 // digit q of k, most significant first
                int64_t div = 1;
                for (int64_t q = j - sp; q < td - 1; ++q) div *= 10;
                v = (uint8_t)('0' + (k / div) % 10);
            }
            p[1 + j] = v;
        }
        if (lane == 0) p[1 + L] = '\n';
        uint8_t *b = p + 2 + L;
        const bool u = rna && rna[s];
        if (fmt == 0) {
            if (u) warp_copy(seq + s0, b, sl, lane, CopyTtoU());
            else warp_copy(seq + s0, b, sl, lane);
            warp_copy(qual + s0, b + sl + 3, sl, lane);
            if (lane == 0) { b[sl] = '\n'; b[sl + 1] = '+'; b[sl + 2] = '\n'; b[2 * sl + 3] = '\n'; }
        } else {
            // output byte j of the base lines is column c of line l (71 bytes a line: 70 bases and '\n'); a lane moves 32 bytes
            // a step, so (l, c) follow without a division
            const int64_t nb = sl + (sl + 69) / 70;
            int64_t l = 0, c = lane;
            for (int64_t j = lane; j < nb; j += 32) {
                uint8_t v = '\n';
                if (c < 70 && j != nb - 1) {
                    v = seq[s0 + 70 * l + c];
                    if (u && v == 'T') v = 'U';
                }
                b[j] = v;
                c += 32;
                if (c >= 71) { c -= 71; ++l; }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// pb200ParseReadsDevice: FASTQ / FASTA bytes -> names, bases, qualities and RNA flags (fastq.parse_fastq / parse_fasta).
// The line index is one tile of PB_PARSE_TILE input bytes per block, 32 contiguous bytes per thread: parse_count_lines_kernel
// counts the '\n' bytes of every tile, scan_offsets turns the counts into each tile's first line, and parse_line_ends_kernel
// scatters every line's end (an unterminated last line ends at n).  Records (FASTQ) or lines (FASTA) are then stripped,
// checked and measured one per thread; scan_offsets places them; one warp per record or line copies the bytes.
constexpr int PB_PARSE_THREADS = 256;
constexpr int64_t PB_PARSE_TILE = (int64_t)PB_PARSE_THREADS * 32;

// what str.strip() removes from an ASCII line (is_ws of hostio.c)
__device__ __forceinline__ bool parse_ws(uint8_t c) { return c == ' ' || (c >= 9 && c <= 13) || (c >= 28 && c <= 31); }
__device__ __forceinline__ void parse_strip(const uint8_t *buf, int64_t &a, int64_t &b) {
    while (b > a && parse_ws(buf[b - 1])) --b;
    while (a < b && parse_ws(buf[a])) ++a;
}
// the 32 input bytes of this thread (zero past n): two 16-byte loads when they are whole and aligned
__device__ __forceinline__ void parse_load32(const uint8_t *buf, int64_t n, int64_t p, unsigned w[8]) {
    if (p + 32 <= n && (((uintptr_t)(buf + p)) & 15) == 0) {
        const uint4 *v = reinterpret_cast<const uint4 *>(buf + p);
        const uint4 x = v[0], y = v[1];
        w[0] = x.x; w[1] = x.y; w[2] = x.z; w[3] = x.w; w[4] = y.x; w[5] = y.y; w[6] = y.z; w[7] = y.w;
        return;
    }
    for (int k = 0; k < 8; ++k) {
        unsigned u = 0;
        for (int j = 0; j < 4; ++j)
            if (p + 4 * k + j < n) u |= (unsigned)buf[p + 4 * k + j] << (8 * j);
        w[k] = u;
    }
}
__device__ __forceinline__ int parse_count_nl(const unsigned w[8]) {
    int c = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) c += ((w[k] >> (8 * j)) & 0xff) == '\n';
    return c;
}
// cnt[t + 1] = the '\n' bytes of tile t (cnt[0] = 0), for scan_offsets
__global__ void __launch_bounds__(PB_PARSE_THREADS) parse_count_lines_kernel(const uint8_t *buf, int64_t n, int64_t *cnt) {
    const int64_t p = (int64_t)blockIdx.x * PB_PARSE_TILE + (int64_t)threadIdx.x * 32;
    unsigned w[8];
    parse_load32(buf, n, p, w);
    long long total = 0;
    block_exclusive_scan(parse_count_nl(w), &total);
    if (threadIdx.x == 0) {
        cnt[blockIdx.x + 1] = total;
        if (blockIdx.x == 0) cnt[0] = 0;
    }
}
// line_end[k] = the position of the k-th '\n' (first_line[t]: lines before tile t, scanned); the unterminated last line, if any,
// ends at n: its index is first_line[tiles], the number of '\n' bytes
__global__ void __launch_bounds__(PB_PARSE_THREADS) parse_line_ends_kernel(const uint8_t *buf, int64_t n, const int64_t *first_line,
                                                                           int64_t *line_end) {
    const int64_t p = (int64_t)blockIdx.x * PB_PARSE_TILE + (int64_t)threadIdx.x * 32;
    unsigned w[8];
    parse_load32(buf, n, p, w);
    long long total = 0;
    int64_t k = first_line[blockIdx.x] + block_exclusive_scan(parse_count_nl(w), &total);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (((w[i] >> (8 * j)) & 0xff) == '\n') line_end[k++] = p + 4 * i + j;
    if (p <= n - 1 && n - 1 < p + 32 && buf[n - 1] != '\n') line_end[first_line[gridDim.x]] = n;
}

// FASTQ, one thread per record: the stripped header (name = header minus '@'), bases and qualities; name_len / seq_len at [r + 1]
// ([0] = 0) for scan_offsets.  status[r]: 1 = the header is empty or lacks '@', 2 = qualities longer than the bases (checked when
// want_qual), else 0; *flags gets 1 << status.
__global__ void parse_fastq_index_kernel(const uint8_t *buf, const int64_t *line_end, int64_t n_rec, int want_qual,
                                         int64_t *name_a, int64_t *name_len, int64_t *seq_a, int64_t *seq_len, int64_t *qual_a,
                                         int64_t *qual_len, uint8_t *status, int *flags) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) { name_len[0] = 0; seq_len[0] = 0; }
    if (r >= n_rec) return;
    const int64_t k = 4 * r;
    int64_t a0 = k ? line_end[k - 1] + 1 : 0, b0 = line_end[k];
    int64_t a1 = line_end[k] + 1, b1 = line_end[k + 1];
    int64_t a3 = line_end[k + 2] + 1, b3 = line_end[k + 3];
    parse_strip(buf, a0, b0);
    parse_strip(buf, a1, b1);
    parse_strip(buf, a3, b3);
    const bool head_ok = b0 > a0 && buf[a0] == '@';
    const uint8_t st = !head_ok ? 1 : (want_qual && b3 - a3 > b1 - a1) ? 2 : 0;
    status[r] = st;
    if (st) atomicOr(flags, 1 << st);
    name_a[r] = a0 + 1;
    name_len[r + 1] = head_ok ? b0 - a0 - 1 : 0;
    seq_a[r] = a1;
    seq_len[r + 1] = b1 - a1;
    qual_a[r] = a3;
    qual_len[r] = b3 - a3;
}
// FASTA, one thread per line: the stripped span, and at [l + 1] ([0] = 0) for scan_offsets: 1 for a '>' line (hdr), the name
// length of a '>' line (nm) and the length of a kept body line (body)
__global__ void parse_fasta_lines_kernel(const uint8_t *buf, const int64_t *line_end, int64_t n_lines, int64_t *span_a,
                                         int64_t *span_len, int64_t *hdr, int64_t *nm, int64_t *body) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l == 0) { hdr[0] = 0; nm[0] = 0; body[0] = 0; }
    if (l >= n_lines) return;
    int64_t a = l ? line_end[l - 1] + 1 : 0, b = line_end[l];
    parse_strip(buf, a, b);
    const int64_t len = b - a;
    const bool head = len > 0 && buf[a] == '>';
    span_a[l] = a;
    span_len[l] = len;
    hdr[l + 1] = head;
    nm[l + 1] = head ? len - 1 : 0;
    body[l + 1] = head ? 0 : len;
}
// FASTA, one thread per line, after the scans (hdr[l] = records before line l): record hdr[l] of a '>' line starts at names
// nm[l] and bases body[l]; the end offsets go after the last record.  status[l]: 1 = a body line before the first '>' line,
// 2 = a '>' line with an empty name, else 0; *flags gets 1 << status.
__global__ void parse_fasta_records_kernel(const int64_t *span_len, const int64_t *hdr, const int64_t *nm, const int64_t *body,
                                           const uint8_t *buf, const int64_t *span_a, int64_t n_lines, int64_t *name_off,
                                           int64_t *seq_off, uint8_t *status, int *flags) {
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l == 0) {
        name_off[hdr[n_lines]] = nm[n_lines];
        seq_off[hdr[n_lines]] = body[n_lines];
    }
    if (l >= n_lines) return;
    const int64_t len = span_len[l];
    const bool head = len > 0 && buf[span_a[l]] == '>';
    uint8_t st = 0;
    if (head) {
        name_off[hdr[l]] = nm[l];
        seq_off[hdr[l]] = body[l];
        if (len < 2) st = 2;
    } else if (len > 0 && hdr[l] == 0) {
        st = 1;
    }
    status[l] = st;
    if (st) atomicOr(flags, 1 << st);
}

struct CopyUpper {  // a-z -> A-Z, nothing else changes (NanoporeRead.__init__: seq.upper() of ASCII bases)
    __device__ __forceinline__ unsigned operator()(unsigned w) const {
        const unsigned h = w & 0x7f7f7f7fu;
        const unsigned ge_a = h + 0x1f1f1f1fu, gt_z = h + 0x05050505u;     // high bit: byte >= 'a', byte > 'z'
        const unsigned m = ge_a & ~gt_z & ~w & 0x80808080u;                  // ASCII lower-case letters
        return w - (m >> 2);                                                  // -0x20 in those bytes (no borrow)
    }
};
// FASTQ, one warp per record: the name, the upper-cased bases and (qual not NULL) the qualities, padded with '+' to the bases'
// length (every check passed, so no quality line is longer than its bases)
__global__ void __launch_bounds__(256) parse_fastq_write_kernel(const uint8_t *buf, const int64_t *name_a, const int64_t *name_off,
                                                                const int64_t *seq_a, const int64_t *seq_off, const int64_t *qual_a,
                                                                const int64_t *qual_len, int64_t n_rec, uint8_t *names,
                                                                uint8_t *seq, uint8_t *qual) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_rec; r += warps) {
        const int64_t s0 = seq_off[r], sl = seq_off[r + 1] - s0;
        warp_copy(buf + name_a[r], names + name_off[r], name_off[r + 1] - name_off[r], lane);
        warp_copy(buf + seq_a[r], seq + s0, sl, lane, CopyUpper());
        if (qual) {
            const int64_t ql = qual_len[r] < sl ? qual_len[r] : sl;
            warp_copy(buf + qual_a[r], qual + s0, ql, lane);
            for (int64_t j = ql + lane; j < sl; j += 32) qual[s0 + j] = '+';
        }
    }
}
// FASTA, one warp per kept line: a '>' line's name to names + nm[l], a body line's upper-cased bases to seq + body[l]
__global__ void __launch_bounds__(256) parse_fasta_write_kernel(const uint8_t *buf, const int64_t *span_a, const int64_t *span_len,
                                                                const int64_t *nm, const int64_t *body, int64_t n_lines,
                                                                uint8_t *names, uint8_t *seq) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t l = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < n_lines; l += warps) {
        const int64_t len = span_len[l];
        if (len == 0) continue;
        const uint8_t *src = buf + span_a[l];
        if (*src == '>') warp_copy(src + 1, names + nm[l], len - 1, lane);
        else warp_copy(src, seq + body[l], len, lane, CopyUpper());
    }
}
// one warp per read of the written (upper-cased) bases: rna[r] = count('U') > count('T'), and an RNA read's 'U' become 'T'
__global__ void __launch_bounds__(256) parse_normalise_kernel(const int64_t *seq_off, int64_t n_rec, uint8_t *seq, uint8_t *rna) {
    const int lane = threadIdx.x & 31;
    const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < n_rec; r += warps) {
        const int64_t s0 = seq_off[r], sl = seq_off[r + 1] - s0;
        long long d = 0;                                           // count('U') - count('T') of this lane's bytes
        for (int64_t j = lane; j < sl; j += 32) {
            const uint8_t c = seq[s0 + j];
            d += (c == 'U') - (c == 'T');
        }
        for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (lane == 0) rna[r] = d > 0;
        if (d > 0)
            for (int64_t j = lane; j < sl; j += 32)
                if (seq[s0 + j] == 'U') seq[s0 + j] = 'T';
    }
}

// ---------------------------------------------------------------------------------------------------
// Demux stage of adapterDemuxReadsDevice.  Per segment, barcode_call_kernel turns the two sides' top-2 rankings (decide_kernel)
// into each read's bin.  Once per call, after the last segment, the records the output stage placed in read order (engine
// scratch: source offset, offsets, read, part) are partitioned stably by key = their read's bin ('none' = n_bins, or
// n_bins + 1 = dropped with discard_unassigned): a histogram per tile of PB_DEMUX_TILE records, the scan of the (key x tile)
// counts in key-major order, then a scatter that keeps the read order inside each tile.  split_gather_kernel then copies the
// bases from the permuted source offsets.
#define PB_DEMUX_TILE 256
#define PB_DEMUX_MAX_KEYS 4097                 // n_bins < 4096: the named bins, 'none', dropped

// read_bin[s] of the segment's reads: top2_* = decide_kernel's 6 ints per read of a side (NULL: the side has no barcode
// column), bin_* = bin of each score column, tab[c * tab_l + l] = float("%f" % (100.0 * c / max(l, 1))) for c < tab_c,
// l < tab_l; albacore = the reads' Albacore bins or NULL.  A pair outside the table sets status bit 2.
__device__ __forceinline__ BarcodeSide barcode_side(const int32_t *t, const int32_t *bin, const double *tab, int32_t tab_c,
                                                     int32_t tab_l, int *status) {
    BarcodeSide x = {-1, -1, 0.0, 0.0};
    if (!t) return x;
    for (int k = 0; k < 2; ++k) {
        const int32_t pos = t[3 * k], c = t[3 * k + 1], l = t[3 * k + 2];
        if (pos < 0) continue;
        double v = 0.0;
        if (c < 0 || c >= tab_c || l < 0 || l >= tab_l) atomicOr(status, 2);
        else v = tab[(int64_t)c * tab_l + l];
        if (k == 0) { x.b1 = bin[pos]; x.s1 = v; } else { x.b2 = bin[pos]; x.s2 = v; }
    }
    return x;
}
__global__ void barcode_call_kernel(const int32_t *top2_s, const int32_t *top2_e, const int32_t *bin_s, const int32_t *bin_e,
                                    const double *tab, int32_t tab_c, int32_t tab_l, int64_t n, int32_t n_bins, double threshold,
                                    double diff, int32_t require_two, const int32_t *albacore, int32_t *read_bin, int *status) {
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const BarcodeSide bs = barcode_side(top2_s ? top2_s + s * 6 : nullptr, bin_s, tab, tab_c, tab_l, status);
    const BarcodeSide be = barcode_side(top2_e ? top2_e + s * 6 : nullptr, bin_e, tab, tab_c, tab_l, status);
    read_bin[s] = barcode_call(bs, be, n_bins, threshold, diff, require_two, albacore ? albacore[s] : -1);
}
// the partition key of record r (-1 past the last record)
__device__ __forceinline__ int32_t demux_key(const int32_t *rec_read, const int32_t *read_bin, int64_t r, int64_t n_rec,
                                             int32_t n_bins, int32_t discard) {
    if (r >= n_rec) return -1;
    const int32_t b = read_bin[rec_read[r]];
    return (discard && b == n_bins) ? n_bins + 1 : b;
}
// counts of the keys in tile t -> cnt[1 + k * tiles + t] (cnt[0] = 0, for scan_offsets); the bases of the records that are
// kept (key <= n_bins) are added to *kept_bytes.  One block of PB_DEMUX_TILE threads per tile.
__global__ void __launch_bounds__(PB_DEMUX_TILE) demux_count_kernel(const int32_t *rec_read, const int64_t *rec_off, int64_t n_rec,
                                                                    const int32_t *read_bin, int32_t n_bins, int32_t discard,
                                                                    int64_t tiles, int64_t *cnt, unsigned long long *kept_bytes) {
    __shared__ unsigned hist[PB_DEMUX_MAX_KEYS];
    __shared__ unsigned long long bytes;
    const int32_t n_keys = n_bins + 2;
    for (int32_t k = threadIdx.x; k < n_keys; k += blockDim.x) hist[k] = 0u;
    if (threadIdx.x == 0) bytes = 0ull;
    if (blockIdx.x == 0 && threadIdx.x == 0) cnt[0] = 0;
    __syncthreads();
    const int64_t r = (int64_t)blockIdx.x * PB_DEMUX_TILE + threadIdx.x;
    const int32_t key = demux_key(rec_read, read_bin, r, n_rec, n_bins, discard);
    if (key >= 0) {
        atomicAdd(&hist[key], 1u);
        if (key <= n_bins) atomicAdd(&bytes, (unsigned long long)(rec_off[r + 1] - rec_off[r]));
    }
    __syncthreads();
    for (int32_t k = threadIdx.x; k < n_keys; k += blockDim.x) cnt[1 + (int64_t)k * tiles + blockIdx.x] = hist[k];
    if (threadIdx.x == 0 && bytes) atomicAdd(kept_bytes, bytes);
}
// parts[k] = base[k * tiles], k = 0 .. n_keys: the first record of every key in output order, then the total
__global__ void demux_bin_parts_kernel(const int64_t *base, int64_t tiles, int32_t n_keys, int64_t *parts) {
    const int32_t k = (int32_t)(blockIdx.x * blockDim.x + threadIdx.x);
    if (k <= n_keys) parts[k] = base[(int64_t)k * tiles];
}
// Stable scatter: record r of tile t with key k goes to base[k * tiles + t] + (the records of key k before it in the tile).
// Within a warp that rank comes from the keys of the lower lanes (shuffles); across the warps of the block a running count
// per key in shared memory, updated one warp after the other.  Kept records write their length to out_len (d_out_off + 1,
// scanned afterwards), read, part and source offset; dropped ones (key n_bins + 1) write nothing.
__global__ void __launch_bounds__(PB_DEMUX_TILE) demux_scatter_kernel(const int32_t *rec_read, const int32_t *rec_part,
                                                                      const int64_t *rec_off, const int64_t *rec_src,
                                                                      int64_t n_rec, const int32_t *read_bin, int32_t n_bins,
                                                                      int32_t discard, int64_t tiles, const int64_t *base,
                                                                      int64_t *out_len, int32_t *out_read, int32_t *out_part,
                                                                      int64_t *perm_src) {
    __shared__ unsigned run[PB_DEMUX_MAX_KEYS];
    const int32_t n_keys = n_bins + 2;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    for (int32_t k = threadIdx.x; k < n_keys; k += blockDim.x) run[k] = 0u;
    const int64_t r = (int64_t)blockIdx.x * PB_DEMUX_TILE + threadIdx.x;
    const int32_t key = demux_key(rec_read, read_bin, r, n_rec, n_bins, discard);
    unsigned before = 0;                        // lanes below with the same key
    bool last = true;                           // no lane above with the same key
    for (int j = 0; j < 32; ++j) {
        const int32_t kj = __shfl_sync(0xffffffffu, key, j);
        if (kj == key) {
            if (j < lane) ++before;
            if (j > lane) last = false;
        }
    }
    __syncthreads();
    unsigned rank = 0;
    for (int w = 0; w < n_warps; ++w) {
        if (warp == w && key >= 0) rank = run[key] + before;
        __syncthreads();
        if (warp == w && key >= 0 && last) run[key] = rank + 1;
        __syncthreads();
    }
    if (key < 0 || key > n_bins) return;
    const int64_t d = base[(int64_t)key * tiles + blockIdx.x] + rank;
    out_len[d] = rec_off[r + 1] - rec_off[r];
    out_read[d] = rec_read[r];
    out_part[d] = rec_part[r];
    perm_src[d] = rec_src[r];
}

// ---------------------------------------------------------------------------------------------------
// pb200GzipDevice: one gzip member per block of input (a block never crosses a segment), one CTA per block, written into a
// fixed slot of engine scratch.  The CTA stages the block in shared memory and
//   1. takes the CRC-32 of 256 slices (one per thread) and combines them in a tree;
//   2. finds matches in rounds of one position per thread: the most recent earlier position with the same 3-byte hash (a
//      shared table of positions from earlier rounds, updated with atomicMax after each round's lookups) and distances
//      1..PB_GZ_SHORT (runs inside a round), every candidate verified byte by byte, the longest kept (the nearest on ties);
//   3. walks the greedy parse through the round's matches on one thread, carrying the cursor into the next round, and
//      appends the tokens to the block's token buffer (global scratch);
//   4. counts the symbols with shared atomics and builds the code lengths on one thread (gz_code_lengths);
//   5. writes a dynamic block -- header by one thread, then each thread's contiguous run of tokens at its scanned bit offset
//      with atomicOr into zeroed shared words (disjoint bits) -- or stored blocks when those are not larger.
// Every choice depends on the input alone (the hash table keeps the largest position, atomics only add or OR disjoint
// bits), so the bytes are the same run to run.  sizes[1 + b] = the member's bytes (sizes[0] = 0), for scan_offsets.
constexpr int PB_GZ_THREADS = 256;
constexpr int PB_GZ_HASH_BITS = 12;
constexpr int PB_GZ_SHORT = 8;
constexpr int PB_GZ_WINDOW = 32768;
constexpr int PB_GZ_MIN_BLOCK = 4096, PB_GZ_MAX_BLOCK = 131072, PB_GZ_DEFAULT_BLOCK = 65536;

struct GzShared {                       // after the staged block and the hash table
    uint32_t crc_tab[256];
    uint32_t part[PB_GZ_THREADS];
    uint16_t mlen[PB_GZ_THREADS], mdist[PB_GZ_THREADS];
    uint32_t ll_freq[GZ_LITLEN], d_freq[GZ_DIST];
    uint32_t work[2 * GZ_LITLEN + 16];
    uint16_t ll_code[GZ_LITLEN], d_code[GZ_DIST];
    uint8_t ll_len[GZ_LITLEN], d_len[GZ_DIST], all_lens[GZ_LITLEN + GZ_DIST];
    GzDynHeader H;
    unsigned long long body_bits, head_bits;
    int32_t n_tok, stored;
};
__host__ __device__ __forceinline__ int64_t gz_stage_bytes(int32_t block) { return ((int64_t)block + 15) & ~(int64_t)15; }
__host__ __device__ __forceinline__ int64_t gz_smem_bytes(int32_t block) {
    return gz_stage_bytes(block) + 8 * (1 << PB_GZ_HASH_BITS) + (int64_t)sizeof(GzShared);
}
__device__ __forceinline__ uint32_t gz_hash(const uint8_t *p) {
    return (((uint32_t)p[0] << 16) | ((uint32_t)p[1] << 8) | p[2]) * 2654435761u >> (32 - PB_GZ_HASH_BITS);
}
__device__ __forceinline__ int gz_match(const uint8_t *in, int p, int d, int maxl) {
    int l = 0;
    while (l < maxl && in[p + l - d] == in[p + l]) ++l;
    return l;
}
// a token: bit 31 clear = literal byte; set = match, length - 3 in bits 16..23, distance - 1 in bits 0..14
__device__ __forceinline__ int gz_token_bits(uint32_t tk, const GzShared &S) {
    if (!(tk >> 31)) return S.ll_len[tk];
    int ls, le, lv, ds, de, dv;
    gz_len_sym((int)((tk >> 16) & 255u) + 3, ls, le, lv);
    gz_dist_sym((int)(tk & 32767u) + 1, ds, de, dv);
    return S.ll_len[ls] + le + S.d_len[ds] + de;
}
__device__ __forceinline__ void gz_or_bits(uint32_t *w, unsigned long long pos, uint32_t bits, int n) {
    if (!n) return;
    const int sh = (int)(pos & 31);
    atomicOr(reinterpret_cast<int *>(w + (pos >> 5)), (int)(bits << sh));
    if (sh + n > 32) atomicOr(reinterpret_cast<int *>(w + (pos >> 5) + 1), (int)(bits >> (32 - sh)));
}
__global__ void __launch_bounds__(PB_GZ_THREADS) gzip_block_kernel(const uint8_t *src, const int64_t *blk_start, const int64_t *blk_len,
                                                                   int32_t block, uint8_t *slots, int64_t slot_stride,
                                                                   uint32_t *tokens, int64_t *sizes) {
    extern __shared__ uint32_t smem[];
    const int t = threadIdx.x;
    const int64_t b = blockIdx.x;
    const int n = (int)blk_len[b];
    const uint8_t *g = src + blk_start[b];
    uint8_t *in = reinterpret_cast<uint8_t *>(smem);
    unsigned long long *head = reinterpret_cast<unsigned long long *>(in + gz_stage_bytes(block));
    GzShared &S = *reinterpret_cast<GzShared *>(in + gz_stage_bytes(block) + 8 * (1 << PB_GZ_HASH_BITS));
    uint32_t *tok = tokens + b * (int64_t)block;
    uint8_t *out = slots + b * slot_stride;

    for (int i = t; i < n; i += PB_GZ_THREADS) in[i] = g[i];
    for (int i = t; i < (1 << PB_GZ_HASH_BITS); i += PB_GZ_THREADS) head[i] = 0ull;
    S.crc_tab[t] = gz_crc_table_entry((uint32_t)t);
    for (int i = t; i < GZ_LITLEN + GZ_DIST; i += PB_GZ_THREADS) (i < GZ_LITLEN ? S.ll_freq[i] : S.d_freq[i - GZ_LITLEN]) = 0u;
    __syncthreads();

    // ---- 1. CRC-32 ----
    const int per = (n + PB_GZ_THREADS - 1) / PB_GZ_THREADS;
    {
        const int lo = min(n, t * per), hi = min(n, lo + per);
        S.part[t] = gz_crc_update(0u, S.crc_tab, in + lo, hi - lo);
        for (int s = 1; s < PB_GZ_THREADS; s <<= 1) {
            __syncthreads();
            if ((t & (2 * s - 1)) == 0) {
                const int r0 = min(n, (t + s) * per), r1 = min(n, (t + 2 * s) * per);
                S.part[t] = gz_crc_combine(S.part[t], S.part[t + s], r1 - r0);
            }
        }
    }
    // ---- 2./3. matches in rounds, greedy parse ----
    int cursor = 0, n_tok = 0;                            // thread 0's
    for (int base = 0; base < n; base += PB_GZ_THREADS) {
        const int p = base + t;
        int best_len = 0, best_dist = 0;
        if (p + 3 <= n) {
            const int maxl = min(258, n - p);
            for (int d = 1; d <= PB_GZ_SHORT && d <= p && best_len < maxl; ++d) {
                const int l = gz_match(in, p, d, maxl);
                if (l > best_len) { best_len = l; best_dist = d; }
            }
            const unsigned long long c = head[gz_hash(in + p)];
            if (best_len < maxl && c) {
                const int d = p - (int)(c - 1ull);
                if (d > PB_GZ_SHORT && d <= PB_GZ_WINDOW) {
                    const int l = gz_match(in, p, d, maxl);
                    if (l > best_len) { best_len = l; best_dist = d; }
                }
            }
        }
        S.mlen[t] = (uint16_t)(best_len >= 3 ? best_len : 0);
        S.mdist[t] = (uint16_t)best_dist;
        __syncthreads();
        if (p + 3 <= n) atomicMax(&head[gz_hash(in + p)], (unsigned long long)(p + 1));
        if (t == 0) {
            const int end = min(n, base + PB_GZ_THREADS);
            while (cursor < end) {
                const int l = S.mlen[cursor - base];
                if (l) {
                    tok[n_tok++] = 0x80000000u | ((uint32_t)(l - 3) << 16) | (uint32_t)(S.mdist[cursor - base] - 1);
                    cursor += l;
                } else {
                    tok[n_tok++] = in[cursor++];
                }
            }
            S.n_tok = n_tok;
        }
        __syncthreads();
    }
    const uint32_t crc = S.part[0];
    // ---- 4. symbol counts, code lengths, the cheaper encoding ----
    const int nt = S.n_tok;
    for (int i = t; i < nt; i += PB_GZ_THREADS) {
        const uint32_t tk = tok[i];
        if (tk >> 31) {
            int ls, le, lv, ds, de, dv;
            gz_len_sym((int)((tk >> 16) & 255u) + 3, ls, le, lv);
            gz_dist_sym((int)(tk & 32767u) + 1, ds, de, dv);
            atomicAdd(&S.ll_freq[ls], 1u);
            atomicAdd(&S.d_freq[ds], 1u);
        } else {
            atomicAdd(&S.ll_freq[tk], 1u);
        }
    }
    __syncthreads();
    if (t == 0) {
        S.ll_freq[256] = 1u;                              // end of block
        gz_code_lengths(S.ll_freq, GZ_LITLEN, GZ_MAX_BITS, S.ll_len, S.work);
        gz_code_lengths(S.d_freq, GZ_DIST, GZ_MAX_BITS, S.d_len, S.work);
        gz_canonical_codes(S.ll_len, GZ_LITLEN, S.ll_code);
        gz_canonical_codes(S.d_len, GZ_DIST, S.d_code);
        const unsigned long long head_bits = gz_dynamic_header(S.ll_len, S.d_len, S.H, S.all_lens, S.work);
        unsigned long long body = 0;
        for (int s = 0; s < GZ_LITLEN; ++s) body += (unsigned long long)S.ll_freq[s] * (S.ll_len[s] + gz_len_extra_bits(s));
        for (int s = 0; s < GZ_DIST; ++s) body += (unsigned long long)S.d_freq[s] * (S.d_len[s] + gz_dist_extra_bits(s));
        S.head_bits = head_bits;
        S.body_bits = body;
        S.stored = (int64_t)((head_bits + body + 7) / 8) >= gz_stored_bytes(n);
    }
    __syncthreads();
    // ---- 5. the member ----
    int64_t bytes;
    if (S.stored) {
        const int nst = (n + GZ_STORED_MAX - 1) / GZ_STORED_MAX;
        for (int i = t; i < n; i += PB_GZ_THREADS) out[GZ_HEADER + 5 * (i / GZ_STORED_MAX + 1) + i] = in[i];
        for (int k = t; k < nst; k += PB_GZ_THREADS) {
            uint8_t *h = out + GZ_HEADER + (int64_t)k * (GZ_STORED_MAX + 5);
            const int len = min(GZ_STORED_MAX, n - k * GZ_STORED_MAX);
            h[0] = (uint8_t)(k == nst - 1);
            h[1] = (uint8_t)len; h[2] = (uint8_t)(len >> 8);
            h[3] = (uint8_t)~len; h[4] = (uint8_t)(~len >> 8);
        }
        bytes = GZ_HEADER + gz_stored_bytes(n) + GZ_TRAILER;
    } else {
        // the deflate bits go to zeroed shared words over the staged block and the hash table, which are no longer needed
        const unsigned long long total = 8ull * GZ_HEADER + S.head_bits + S.body_bits;
        bytes = (int64_t)((total + 7) / 8) + GZ_TRAILER;
        uint32_t *w = smem;
        for (int i = t; i < (int)((bytes + 3) / 4); i += PB_GZ_THREADS) w[i] = 0u;
        __syncthreads();
        if (t == 0) {
            GzBitWriter bw{w, 0};
            const uint8_t hdr[GZ_HEADER] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};
            for (int i = 0; i < GZ_HEADER; ++i) bw.put(hdr[i], 8);
            gz_write_dynamic_header(bw, 1, S.H);
        }
        __syncthreads();
        const int tper = (nt + PB_GZ_THREADS - 1) / PB_GZ_THREADS;
        const int t0 = min(nt, t * tper), t1 = min(nt, t0 + tper);
        long long mine = 0, all = 0;
        for (int i = t0; i < t1; ++i) mine += gz_token_bits(tok[i], S);
        unsigned long long pos = 8ull * GZ_HEADER + S.head_bits + (unsigned long long)block_exclusive_scan(mine, &all);
        for (int i = t0; i < t1; ++i) {
            const uint32_t tk = tok[i];
            if (!(tk >> 31)) {
                gz_or_bits(w, pos, S.ll_code[tk], S.ll_len[tk]);
                pos += S.ll_len[tk];
                continue;
            }
            int ls, le, lv, ds, de, dv;
            gz_len_sym((int)((tk >> 16) & 255u) + 3, ls, le, lv);
            gz_dist_sym((int)(tk & 32767u) + 1, ds, de, dv);
            gz_or_bits(w, pos, S.ll_code[ls], S.ll_len[ls]);
            pos += S.ll_len[ls];
            gz_or_bits(w, pos, (uint32_t)lv, le);
            pos += le;
            gz_or_bits(w, pos, S.d_code[ds], S.d_len[ds]);
            pos += S.d_len[ds];
            gz_or_bits(w, pos, (uint32_t)dv, de);
            pos += de;
        }
        __syncthreads();
        if (t == 0) {                                     // end of block; the trailer starts at the next byte
            GzBitWriter bw{w, 8ull * GZ_HEADER + S.head_bits + (unsigned long long)all};
            bw.put(S.ll_code[256], S.ll_len[256]);
        }
        __syncthreads();
        const uint8_t *wb = reinterpret_cast<const uint8_t *>(w);
        for (int64_t i = t; i < bytes - GZ_TRAILER; i += PB_GZ_THREADS) out[i] = wb[i];
    }
    if (S.stored && t < GZ_HEADER) {
        const uint8_t hdr[GZ_HEADER] = {0x1f, 0x8b, 8, 0, 0, 0, 0, 0, 0, 3};
        out[t] = hdr[t];
    }
    if (t < GZ_TRAILER) out[bytes - GZ_TRAILER + t] = (uint8_t)((t < 4 ? crc : (uint32_t)n) >> (8 * (t & 3)));
    if (t == 0) {
        sizes[1 + b] = bytes;
        if (b == 0) sizes[0] = 0;
    }
}

// ---------------------------------------------------------------------------------------------------
// generic_kernel: int32, one thread per alignment, column sweep with S/Hs columns and a byte trace in
// global scratch.  Only used for inputs outside the int16 domain (huge scores, positive gap scores,
// adapters longer than 256) -- slow but exact for every scoring scheme the C-ABI accepts.
struct GenericJob {
    int64_t seq_off; int32_t n, m, ad_off, out_idx;
    int64_t scratch_off;   // byte offset of this job's scratch: (n+1)*(m+1) trace bytes, then 2*(m+1) int32
};
__global__ void generic_kernel(const GenericJob *__restrict__ jobs, int n_jobs, const uint8_t *__restrict__ seq,
                               const uint8_t *__restrict__ ads, int ma, int mi, int go, int ge,
                               uint8_t *__restrict__ scratch, int32_t *__restrict__ out) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const GenericJob jb = jobs[k];
    int32_t *o = out + (size_t)jb.out_idx * PB_REC;
    const int n = jb.n, m = jb.m;
    if (n <= 0 || m <= 0) {
        o[0] = -1; o[1] = 0; o[2] = -1; o[3] = 0; o[4] = PB_SCORE_EMPTY; o[5] = o[6] = o[7] = o[8] = 0;
        return;
    }
    const uint8_t *h = seq + jb.seq_off, *v = ads + jb.ad_off;
    uint8_t *tr = scratch + jb.scratch_off;                       // [(j)*(m+1) + i], flags as in dp_core
    size_t trbytes = ((size_t)(n + 1) * (size_t)(m + 1) + 3) & ~(size_t)3;
    int32_t *S = reinterpret_cast<int32_t *>(tr + trbytes);
    int32_t *Hs = S + (m + 1);
    const int NEG = -(1 << 30);
    const bool linear = (go == ge);
    for (int i = 0; i <= m; ++i) { S[i] = 0; Hs[i] = NEG; }
    int best = 0, bj = 0, bi = m, bcorr = 0;
    for (int j = 1; j <= n; ++j) {
        int diag = 0, up = 0, upV = NEG;
        const uint8_t hb = h[j - 1];
        uint8_t *tc = tr + (size_t)j * (m + 1);
        for (int i = 1; i <= m; ++i) {
            const int d = diag + ((hb == v[i - 1]) ? ma : mi);
            int hs, vs, s; uint32_t bits = 0;
            if (!linear) {
                const int h_ext = Hs[i] + ge, h_open = S[i] + go;
                if (h_ext >= h_open) { hs = h_ext; bits |= 8u; } else hs = h_open;
                const int v_ext = upV + ge, v_open = up + go;
                if (v_ext >= v_open) { vs = v_ext; bits |= 4u; } else vs = v_open;
            } else {
                hs = S[i] + ge; vs = up + ge;
            }
            int gm;
            if (vs >= hs) { gm = vs; bits |= 2u; } else gm = hs;
            if (d >= gm) { s = d; bits |= 1u; } else s = gm;
            diag = S[i]; S[i] = s; Hs[i] = hs; up = s; upV = vs;
            tc[i] = (uint8_t)bits;
            if ((j == n) || (i == m)) {
                if (s > best) { best = s; bj = j; bi = i; bcorr = (vs == s ? 1 : 0) | (hs == s ? 2 : 0); }
            }
        }
    }
    EndCell end; end.j = bj; end.i = bi; end.score = best; end.corr = bcorr;
    auto nib = [&](int jl, int i) -> uint32_t { return tr[(size_t)jl * (m + 1) + i]; };
    auto eq = [&](int jl, int i) -> bool { return h[jl - 1] == v[i - 1]; };
    int32_t rec[PB_REC];
    traceback_stats(nib, eq, end, linear, 0, n, m, rec);
    for (int q = 0; q < PB_REC; ++q) o[q] = rec[q];
}

}  // namespace pb
