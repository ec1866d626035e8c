// porechop_b200/csrc/kernels.cuh -- sm_90a kernels of the adapter-alignment engine.
//
//   encode_kernel        ASCII -> Dna5 code (seqan/basic/alphabet_residue_tabs.h:113-140), HBM-bound
//   unpack_kernel        host-packed 4-bit codes -> the same code bytes (option h2d_pack)
//   build_tasks_*        (read, adapter) pairs -> Task records in slot order
//   trace_kernel<G,R,S>  overlap DP *with* 4-bit trace + in-kernel traceback + statistics (windows)
//   score_kernel<G,R,P>  streaming score-only overlap DP with exact scout (long reads), dynamic slot refill
//   window_tasks_kernel  end cells of the score pass -> bounded-window tasks for trace_kernel
//   decide_kernel        records -> per-read end-trim amounts + barcode score pairs (decisions stay on the device)
//   middle_decide_kernel one round of the middle-adapter scan: first hit per active read, masking, next active list
//   generic_kernel       int32 thread-serial fallback for scoring schemes / adapters outside the int16 domain
//
// The arithmetic is in dp_core.cuh (shared with the CPU emulation used by the tests).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "dp_core.cuh"

namespace pb {

constexpr int PB_WARPS_PER_BLOCK = 4;
#ifndef PB_TRACE_MIN_BLOCKS
#define PB_TRACE_MIN_BLOCKS 5
#endif
constexpr int PB_SCRATCH_WORDS = 32 * 2 * 6;   // ScoutCand per lane per half
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
// of a half.  Each lane of the group builds every G-th column from single-byte streaming loads.
// (Walking the window in 16-column blocks with one aligned 128-bit load per half and block, funnel-shifted into place, was
// slower: the shift / extract / bounds work per column outweighs the saved LSU instructions, so the byte loads stay.)
template <int G>
__device__ __forceinline__ void stage_columns(uint32_t *hbuf, int g, const uint8_t *seqA, int nA, const uint8_t *seqB, int nB,
                                              int nmax) {
    for (int c = g; c < nmax; c += G) {
        const uint32_t bA = (c < nA) ? (uint32_t)__ldcs(seqA + c) : (uint32_t)PB_PAD_H;
        const uint32_t bB = (c < nB) ? (uint32_t)__ldcs(seqB + c) : (uint32_t)PB_PAD_H;
        hbuf[c] = pack_bases(bA, bB);
    }
}

// ---------------------------------------------------------------------------------------------------
// trace_kernel: one group of G lanes per slot (two alignments in the s16x2 halves), 32/G slots per warp, R adapter
// rows per lane (G*R >= adapter length; R = 5..8 so common adapter lengths 22/24/28 waste no rows).
// Forward wavefront with a 4-bit trace per cell (two 32-bit words per lane per step), then traceback + statistics
// by two lanes of the group, 9-int record per alignment.  Grid-stride over "warp slots" so the trace scratch is
// bounded by the resident grid and stays in L2.
// (Measured and removed: a score-only first pass + bounded trace window for 150-column windows, and shared-memory query
// profiles for the substitution operands -- neither beat this single pass.)
template <int G, int R, bool HBUF_SMEM>
__global__ void __launch_bounds__(PB_WARPS_PER_BLOCK * 32, PB_TRACE_MIN_BLOCKS)
trace_kernel(const TaskSrc ts, const uint8_t *__restrict__ seq,
             const uint8_t *__restrict__ ads, Scoring sc, int32_t *__restrict__ out, uint32_t *__restrict__ gtrace,
             int max_steps, int max_n, int *__restrict__ status) {
    constexpr int SPW = 32 / G;
    constexpr int WPS = TraceWords<R>::value;
    extern __shared__ uint32_t smem[];
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
    uint32_t *wsm = smem + (size_t)warp * per_warp_words;
    uint32_t *hbuf = HBUF_SMEM ? (wsm + grp * max_n) : (gw + trace_words + (size_t)grp * max_n);
    ScoutCand *cand = reinterpret_cast<ScoutCand *>(wsm + hb_words);  // [half][lane]
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
            nmax = max(nA, nB);
            stage_columns<G>(hbuf, g, seq + tA.seq_off, nA, seq + tB.seq_off, nB, nmax);
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
        for (int t0 = 0; t0 < T4; t0 += PB_TCHUNK) {
            uint4 acc[WPS];
            if (t0 >= TWARM && t0 < tfast) {
                uint32_t buf[PB_TCHUNK][WPS];
#pragma unroll
                for (int u = 0; u < PB_TCHUNK; ++u) {
                    uint32_t recvS = __shfl_up_sync(0xffffffffu, L.botX, 1, G);
                    uint32_t recvV = __shfl_up_sync(0xffffffffu, L.botV, 1, G);
                    if (g == 0) { recvS = sc.borderX2; recvV = sc.negb2; }
                    const int j = t0 + u - g + 1;
                    lane_step<R, true, false>(L, recvS, recvV, hbuf[j - 1], sc, buf[u]);
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
                    if (j >= 1 && j <= nmax) {
                        uint32_t vr[R];
                        lane_step<R, true, true>(L, recvS, recvV, hbuf[j - 1], sc, tw, vr);
                        if (need_track) {
                            if (j >= nmin) lane_track_general<R>(L, g, j, make_geom(nA, mA, G, R), make_geom(nB, mB, G, R), vr, sc);
                            else lane_track_lastrow<R>(L, j, sc);
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
        if (g < 2) {
            const int h = g;
            const Task tk = get_task(ts, slot * 2 + h);
            const HalfGeom gh = make_geom(tk.n, tk.m, G, R);
            if (tk.out_idx >= 0) {
                EndCell end;
                if (tk.flags & TASK_END_GIVEN) {
                    end.j = tk.end_j; end.i = tk.end_i; end.score = tk.end_score; end.corr = tk.end_corr;
                    if (tk.n_total <= 0 || tk.m <= 0) end.score = PB_SCORE_EMPTY;
                } else {
                    end = scout_combine(cand + h * 32 + grp * G, G, gh);
                }
                // cursor over the slot's trace: incremental addresses (lane of the row, row within the lane, step index) instead
                // of a division per path step; one 128-bit load serves up to PB_TCHUNK consecutive steps of a lane
                struct Cursor {
                    const uint32_t *base;      // trace words of this half, lane 0 of the group, chunk 0
                    const uint32_t *hp;        // staged column word of the current column
                    const uint8_t *ap;         // adapter code of the current row
                    int gg, r, t, key, h;
                    uint4 cv;
                    __device__ __forceinline__ uint32_t flags() {
                        const int k = (t >> 2) * (WPS * 32) + gg;
                        if (k != key) { cv = *reinterpret_cast<const uint4 *>(base + (size_t)k * PB_TCHUNK); key = k; }
                        const uint32_t lo = (t & 1) ? cv.y : cv.x, hi = (t & 1) ? cv.w : cv.z;
                        return (((t & 2) ? hi : lo) >> trace_shift<R>(h, r)) & 15u;
                    }
                    __device__ __forceinline__ bool eq() { return ((*hp >> (8 + 16 * h)) & 0xFFu) == (uint32_t)__ldg(ap); }
                    __device__ __forceinline__ void move(bool consR, bool consA) {
                        if (consA) { --ap; if (r == 0) { r = R - 1; --gg; --t; } else --r; }
                        if (consR) { --t; --hp; }
                    }
                } cur;
                {
                    const int q = max(end.i + gh.pad - 1, 0);
                    cur.gg = q / R; cur.r = q % R; cur.t = end.j - 1 + cur.gg; cur.key = -1; cur.h = h;
                    cur.base = tr + ((size_t)trace_word<R>(h, 0) * 32 + grp * G) * PB_TCHUNK;
                    cur.hp = hbuf + end.j - 1; cur.ap = ads + tk.ad_off + end.i - 1;
                    cur.cv = make_uint4(0u, 0u, 0u, 0u);
                }
                int32_t rec[PB_REC];
                int st = traceback_stats_cur(cur, end, sc.linear != 0, tk.col0, tk.n_total, tk.m, rec);
                if (st) atomicOr(status, 1);
                int32_t *o = out + (size_t)tk.out_idx * PB_REC;
#pragma unroll
                for (int k = 0; k < PB_REC; ++k) __stcs(o + k, rec[k]);
            }
        }
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
