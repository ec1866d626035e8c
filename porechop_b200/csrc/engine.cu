// porechop_b200/csrc/engine.cu -- host engine + C-ABI (include/porechop_b200.h) of cpp_functions.so.
//
// Replaces, behind the same ctypes boundary, the reference's C shim + SeqAn DP + ScoredAlignment
// (porechop/src/adapter_align.cpp:11-44, porechop/src/alignment.cpp:6-121, seqan/align/dp_*.h).
// The host side only plans and pipelines: chunking, class selection by adapter length, host<->device
// copies on a ring of streams, kernel launches.  All alignment arithmetic runs in the sm_90a kernels of
// kernels.cuh; there is no CPU alignment path in this library.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include "../../include/porechop_b200.h"
#include "kernels.cuh"

// NVTX ranges around submit / H2D / DP / D2H (SURVEY 5 "tracing"): header-only NVTX3, a no-op unless a profiler is attached.
// The host simulator (tests/sim) and -DPB_NO_NVTX build without it.
#if defined(__CUDACC__) && !defined(PB_NO_NVTX)
#include <nvtx3/nvToolsExt.h>
#define PB_NVTX 1
#endif

using namespace pb;

// hostpack.cpp (g++): ASCII -> two 4-bit Dna5 codes per byte on the host cores
extern "C" void pb_pack_nibbles(const uint8_t *in, int64_t n, uint8_t *out, int threads);

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};
std::atomic<int> g_timing{0};

int fail(int code, const std::string &msg) { g_err = msg; return code; }

struct NvtxRange {          // RAII range on the calling host thread
#ifdef PB_NVTX
    explicit NvtxRange(const char *name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
#else
    explicit NvtxRange(const char *) {}
#endif
    NvtxRange(const NvtxRange &) = delete;
    NvtxRange &operator=(const NvtxRange &) = delete;
};

#define CK(call)                                                                                     \
    do {                                                                                             \
        cudaError_t e_ = (call);                                                                     \
        if (e_ != cudaSuccess)                                                                       \
            return fail(PB200_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));         \
    } while (0)

struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; return fail(PB200_ERR_CUDA, std::string("cudaMalloc: ") + cudaGetErrorString(e)); }
        cap = want;
        return 0;
    }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// pinned host staging memory (packed upload path)
struct HostBuf {
    uint8_t *p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return 0;
        if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(&p), want, cudaHostAllocDefault);
        if (e != cudaSuccess) { p = nullptr; return fail(PB200_ERR_CUDA, std::string("cudaHostAlloc: ") + cudaGetErrorString(e)); }
        cap = want;
        return 0;
    }
};

struct Options {
    int64_t direct_max = 160;      // longest sequence aligned in a single (trace) pass: 150-column end windows are faster in one pass,
                                   // long reads in two (the one-pass trace of a long window is 10.5 instead of 3.7 instructions per
                                   // cell and its scratch, 129 KB per warp at 500 columns, leaves 2 blocks per SM)
    int64_t chunk_tasks = 1 << 17; // alignments per pipeline chunk (host-buffer API)
    int64_t device_chunk_tasks = 8 << 20; // alignments per launch group (device-resident API)
    int64_t chunk_bytes = 64ll << 20;   // sequence bytes per pipeline chunk (host-buffer API)
    int scratch_mb = 128;          // cap on the resident trace scratch (MB); see launch_trace_variant
    int profile = 1;               // 1: score pass fetches the substitution operands from a shared-memory query profile (same-read slots)
    int tight_window = 1;          // 1: second-pass windows sized per alignment from the end cell's row and score (window_cols)
    int h2d_pack = 0;              // 1: host-buffer API converts to 4-bit codes on the host cores and uploads half the bytes; 0 (default):
                                   // never; -1 = auto: for submits of >= 32 MB when the packer team has >= 12 threads (pack_wanted)
    int pack_threads = 0;          // host threads of the packer (default: hardware threads / ranks on the node, at most 32)
    int hbuf_mode = 0;             // 0 auto, 1 shared memory, 2 global scratch (staging of a slot's packed bases)
};
Options g_opt;
std::once_flag g_opt_once;
void load_env_options() {
    std::call_once(g_opt_once, [] {
        if (const char *v = getenv("PB200_DIRECT_MAX")) g_opt.direct_max = atoll(v);
        if (const char *v = getenv("PB200_CHUNK_TASKS")) g_opt.chunk_tasks = std::max(1ll, atoll(v));
        if (const char *v = getenv("PB200_SCRATCH_MB")) g_opt.scratch_mb = std::max(1, atoi(v));
        if (const char *v = getenv("PB200_TIGHT_WINDOW")) g_opt.tight_window = atoi(v);
        if (const char *v = getenv("PB200_H2D_PACK")) g_opt.h2d_pack = atoi(v);
        if (const char *v = getenv("PB200_PROFILE")) g_opt.profile = atoi(v);
        if (const char *v = getenv("PB200_PACK_THREADS")) g_opt.pack_threads = atoi(v);
        if (g_opt.pack_threads <= 0) {
            // packer threads: the host's hardware threads shared by the ranks of this node (torchrun exports
            // LOCAL_WORLD_SIZE, and OMP_NUM_THREADS=1 -- which would otherwise leave the packer single-threaded), at most 32
            // -- and no more than the cgroup CPU quota allows to run at once (a host may show many more hardware
            // threads than its quota lets run; a team larger than the quota is only throttled)
            unsigned hw = std::max(1u, std::thread::hardware_concurrency());
            if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
                char q[64]; long long period = 0;
                if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0) {
                    const long long quota = atoll(q);
                    if (quota > 0) hw = (unsigned)std::min<long long>(hw, std::max<long long>(1, (quota + period - 1) / period));
                }
                fclose(f);
            }
            const int lw = getenv("LOCAL_WORLD_SIZE") ? std::max(1, atoi(getenv("LOCAL_WORLD_SIZE"))) : 1;
            unsigned team = std::max<unsigned>(1u, hw / (unsigned)lw);
            if (team > 4) team -= 2;         // the submit thread and the driver's threads need CPUs of the same quota
            g_opt.pack_threads = (int)std::min<unsigned>(32u, team);
        }
        if (const char *v = getenv("PB200_HBUF")) g_opt.hbuf_mode = !strcmp(v, "smem") ? 1 : !strcmp(v, "global") ? 2 : 0;
    });
}

constexpr int NSTAGE = 3;
struct Stage {
    cudaStream_t stream = nullptr;
    DevBuf seq_raw, seq_codes, seq_off, tasks, tasks2, ends, out, order, bins, pair_seq, pair_ad, gtrace, misc;
    DevBuf dec_trim, dec_pairs, dec_top2;    // per-chunk outputs of decide_kernel
};

struct ClassPlan {
    int cls = 0;                      // row-capacity class (class_of); GENERIC_CLASS = int32 fallback
    std::vector<int32_t> ad_ids;      // adapters of the class, sorted by length
    int m_max = 0;
};

// timed DP launches by kind (pb200TimingReadKinds): which kernel dominates a step, and its per-launch duration
enum { TK_TRACE = 0, TK_TRACE_SCORE_ONLY = 1, TK_TRACE_WINDOW = 2, TK_SCORE = 3, TK_N = 4 };
struct TimedLaunch { cudaEvent_t a, b; int kind; };

struct Engine {
    int device = -1;
    int sm_count = 0;
    size_t smem_optin = 0;
    std::mutex mu;
    Stage st[NSTAGE];
    DevBuf gjobs, gscratch;
    static constexpr int MAX_DEC_JOBS = 8;
    DevBuf dec_cmin[MAX_DEC_JOBS], dec_cols[MAX_DEC_JOBS];   // threshold table + score columns of the decision jobs of a call
    // adapter plan cache (4 entries, LRU): repeated calls with the same adapters + scoring (the normal case: Porechop
    // alternates between its start-adapter and end-adapter lists) skip upload, encode and the host synchronisation
    struct PlanEntry {
        std::vector<uint8_t> ad;
        std::vector<int32_t> off;
        int sc[4] = {0, 0, 0, 0};
        bool valid = false;
        unsigned long long last_used = 0;
        DevBuf ad_raw, ad_codes, ad_off, cls_ad;
        std::shared_ptr<void> plan;
    };
    PlanEntry plans[4];
    unsigned long long plan_clock = 0;
    std::vector<TimedLaunch> timed;
    double timed_ms_acc[TK_N] = {0, 0, 0, 0};
    long long timed_n_acc[TK_N] = {0, 0, 0, 0};
    int next_trace_kind = TK_TRACE;      // set to TK_TRACE_WINDOW around the second-pass launch of a two-pass class
    DevBuf wcells;                       // device counter: DP cells of the windowed second passes (window_tasks_kernel)
    // middle-adapter scan (adapterMiddleScan*): the resident segment -- codes (masked in place), offsets, records, next adapter
    // per read, hit slots, two active lists, threshold table, append counter + longest appended read
    DevBuf mid_codes, mid_off, mid_rec, mid_next_ad, mid_hits, mid_active[2], mid_cmin, mid_ctr;
    // whole-read trimming (adapterTrimReads*): the segment's ASCII reads and offsets (host API), window offsets, start / end
    // windows, segment-wide start / end trims, the first base of every trimmed read, tile sums of the offset scans
    DevBuf trim_reads, trim_off, trim_win_off, trim_win[2], trim_d[2], trim_first, trim_scan;
    // output stage (adapterTrimSplitReadsDevice): the segment's hit reads, their CSR of extended hit ranges, hit row per read,
    // records and bases per read (scanned in place), source offset per record
    DevBuf split_hits, split_rng_off, split_rng, split_hit_of, split_cnt, split_bytes, split_src;
    // demux stage (adapterDemuxReadsDevice): the segment's top-2 rankings per side, bin of each score column per side, score
    // table, the call-wide bin per read; the call's records in read order (source offset, offsets, read, part), the (key x
    // tile) counts, bin offsets, kept bases, and the permuted source offsets
    DevBuf demux_top2[2], demux_map[2], demux_tab, demux_bin, demux_rsrc, demux_roff, demux_rread, demux_rpart, demux_cnt,
        demux_parts, demux_kept, demux_perm;
    // adapter-set search (adapterSetSearch): NSTAGE slices of search_cols u64 keys, one per stage, so that stages running at
    // once never share an accumulator; a batch owns the columns [search_col, search_col + n_adapters) of every slice
    DevBuf search_acc;
    int64_t search_cols = 0;
    // parse (pb200ParseReadsDevice): line counts per tile (scanned), line ends, the per-record (FASTQ) or per-line (FASTA) index
    // arrays, and one status byte per record or line
    DevBuf parse_tiles, parse_lines, parse_index, parse_status;
    // gzip (pb200GzipDevice): the block table (source offsets, lengths, slot offsets), one member slot and one token buffer per
    // block, the members' sizes (scanned into their offsets)
    DevBuf gz_table, gz_slots, gz_tokens, gz_sizes;
    std::shared_ptr<void> packer;       // Packer (below): the thread that plans and packs chunks ahead of the submit loop
    // Ordering between calls: every entry point uses the stage buffers above (st[0]'s trace scratch, tasks, codes, status word),
    // whatever stream it runs on.  A call that returns with work still queued (adapterAlignmentBatchDevice) records `last` on
    // its stream; every later call's streams wait for it before they touch a buffer (order_after_last).  `last_pending` is
    // cleared once a call has synchronised with that work.  `legacy` orders the library's own stream after the caller's work
    // on the legacy default stream (stream argument NULL, library_stream).
    cudaEvent_t last = nullptr, legacy = nullptr;
    cudaStream_t last_stream = nullptr;
    bool last_pending = false;
    // launch constants, queried once per (kernel, dynamic shared-memory size); all users hold `mu`.  The opt-in shared-memory
    // limit is a property of the KERNEL, not of a launch: it is only ever raised (a launch with less is always valid).
    std::map<std::pair<const void *, size_t>, int> bps_cache;
    std::map<const void *, size_t> smem_attr;
    int blocks_per_sm(const void *kern, int threads, size_t smem_bytes, int *bps) {
        const auto key = std::make_pair(kern, smem_bytes);
        auto it = bps_cache.find(key);
        if (it != bps_cache.end()) { *bps = it->second; return 0; }
        size_t &have = smem_attr[kern];
        if (smem_bytes > have) {
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
            have = smem_bytes;
        }
        int b = 0;
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, kern, threads, smem_bytes));
        if (b < 1) b = 1;
        bps_cache[key] = b;
        *bps = b;
        return 0;
    }
    bool init_done = false;
    int init() {
        if (init_done) return 0;
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        if (prop.major != 9 || prop.minor != 0)
            return fail(PB200_ERR_NO_DEVICE, "device is sm_" + std::to_string(prop.major * 10 + prop.minor) +
                                                 ", this library is built for sm_90a (H100) only");
        sm_count = prop.multiProcessorCount;
        smem_optin = prop.sharedMemPerBlockOptin;
        for (int i = 0; i < NSTAGE; ++i) CK(cudaStreamCreateWithFlags(&st[i].stream, cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&last, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&legacy, cudaEventDisableTiming));
        init_done = true;
        return 0;
    }
};

// cudaStreamWaitEvent: `s` waits on the device for the work `e` captured.  Every CUDA runtime has it; a host stand-in of the
// runtime that runs streams synchronously (an older tests/sim) may not, and then the overload below -- the stronger
// host-side wait for the event -- is chosen instead.  Likewise a runtime header without the legacy-stream handle gets
// stream 0, which is the legacy default stream in this library's builds (no per-thread default stream).
template <class S, class Ev>
auto stream_wait_event(S s, Ev e, int) -> decltype(cudaStreamWaitEvent(s, e, 0u)) { return cudaStreamWaitEvent(s, e, 0u); }
template <class S, class Ev>
cudaError_t stream_wait_event(S, Ev e, long) { return cudaEventSynchronize(e); }
#ifndef cudaStreamLegacy
#define cudaStreamLegacy ((cudaStream_t)0)
#endif

// `s` waits for the work an earlier call left queued on another stream (Engine::last).  Same stream: nothing to do, so a
// caller that keeps to one stream (bench.py) runs exactly as before.
int order_after_last(Engine &E, cudaStream_t s) {
    if (E.last_pending && E.last_stream != s) CK(stream_wait_event(s, E.last, 0));
    return 0;
}
int order_stages_after_last(Engine &E) {
    for (int i = 0; i < NSTAGE; ++i) if (int rc = order_after_last(E, E.st[i].stream)) return rc;
    return 0;
}
// the call's work on `s` is still queued when it returns: the next call waits for it
int record_last(Engine &E, cudaStream_t s) {
    CK(cudaEventRecord(E.last, s));
    E.last_stream = s;
    E.last_pending = true;
    return 0;
}
// The stream of a device-resident call: the caller's, or for NULL the library's own stream (st[0]), which first waits for the
// work queued so far on the legacy default stream -- where a caller that does not pick a stream has uploaded its reads.
int library_stream(Engine &E, void *user_stream, cudaStream_t *s) {
    if (user_stream) { *s = (cudaStream_t)user_stream; return 0; }
    CK(cudaEventRecord(E.legacy, cudaStreamLegacy));
    CK(stream_wait_event(E.st[0].stream, E.legacy, 0));
    *s = E.st[0].stream;
    return 0;
}

std::mutex g_engines_mu;
std::map<int, std::unique_ptr<Engine>> g_engines;

int get_engine(Engine **out) {
    load_env_options();
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0)
        return fail(PB200_ERR_NO_DEVICE, std::string("no CUDA device available: ") +
                                             (e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0"));
    int dev = 0;
    CK(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_engines_mu);
    auto &slot = g_engines[dev];
    if (!slot) { slot.reset(new Engine()); slot->device = dev; }
    *out = slot.get();
    return 0;
}

// Where an entry point runs: st[0]; the library stream of a device-resident call (library_stream); or st[0] with every
// stage's stream waiting for earlier queued work (the calls that run the chunk pipeline, run_cross_jobs, on all stages).
enum class CallOn { stage0, library, stages };

// The engine of the current device, locked and initialised, and the call's stream ordered after the work earlier calls left
// queued; then body(E, stream).
template <class Body>
int with_engine(CallOn on, void *user_stream, Body &&body) {
    Engine *Ep = nullptr;
    if (int rc = get_engine(&Ep)) return rc;
    Engine &E = *Ep;
    std::lock_guard<std::mutex> lk(E.mu);
    if (int rc = E.init()) return rc;
    cudaStream_t stream = E.st[0].stream;
    if (on == CallOn::library) { if (int rc = library_stream(E, user_stream, &stream)) return rc; }
    if (int rc = on == CallOn::stages ? order_stages_after_last(E) : order_after_last(E, stream)) return rc;
    return body(E, stream);
}

// with_engine for a call that returns with its work done: when the body fails, nothing may still be running (or reading and
// writing the caller's buffers) when the call returns, so the stream is drained, keeping the first error's message.  Either
// way the stream has waited for the earlier calls' queued work, and all of it is done.
template <class Body>
int sync_call(CallOn on, void *user_stream, Body &&body) {
    return with_engine(on, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        const int rc = body(E, stream);
        if (rc) {
            const std::string first_err = g_err;
            cudaStreamSynchronize(stream);
            g_err = first_err;
        }
        E.last_pending = false;
        return rc;
    });
}

// ---- int16 domain checks and the window bound ------------------------------------------------------------
struct SchemeInfo {
    bool int16_ok_base;   // sign conventions allow the packed kernels at all
    int A;                // max |score|
    bool bounded;         // window bound exists (both gap scores negative)
    int wnum, wden;       // W(m) = m + m*wnum/wden
};
SchemeInfo scheme_info(int ma, int mi, int go, int ge) {
    SchemeInfo s;
    auto ab = [](int x) { return x < 0 ? -(long long)x : (long long)x; };
    long long A = std::max(std::max(ab(ma), ab(mi)), std::max(ab(go), ab(ge)));
    s.A = (int)std::min<long long>(A, 1 << 30);
    s.int16_ok_base = (ma >= mi) && ((long long)ma - mi <= PB_MAX_SUBW) && go <= 0 && ge <= 0 && A <= PB_I16_LIMIT;
    s.bounded = (go < 0 && ge < 0);
    s.wnum = std::max(std::max(ma, mi), 0);
    s.wden = (int)std::min(ab(go), ab(ge));
    if (s.wden == 0) s.wden = 1;
    return s;
}
bool int16_ok(const SchemeInfo &s, int m) { return s.int16_ok_base && (long long)s.A * (m + 3) <= PB_I16_LIMIT; }
// Row capacity classes: G lanes x R rows per lane.  Class k: G = 4 << (k / 4), R = 5 + (k % 4)  -> capacities
// 20,24,28,32, 40,48,56,64, 80,96,112,128, 160,192,224,256.  Class 16 = generic int32 fallback.
constexpr int N_CLASSES = 17;
constexpr int GENERIC_CLASS = 16;
int class_G(int k) { return 4 << (k / 4); }
int class_R(int k) { return 5 + (k % 4); }
int class_of(const SchemeInfo &s, int m) {
    if (!int16_ok(s, m) || m > 256) return GENERIC_CLASS;
    for (int k = 0; k < GENERIC_CLASS; ++k)
        if (m <= class_G(k) * class_R(k)) return k;
    return GENERIC_CLASS;
}

// ---- kernel launch helpers -----------------------------------------------------------------------------
void timed_begin(Engine &E, cudaStream_t s, TimedLaunch &tl, bool &on, int kind) {
    on = g_timing.load() != 0;
    if (on) { tl.kind = kind; cudaEventCreate(&tl.a); cudaEventCreate(&tl.b); cudaEventRecord(tl.a, s); }
}
void timed_end(Engine &E, cudaStream_t s, TimedLaunch &tl, bool on) {
    if (on) { cudaEventRecord(tl.b, s); E.timed.push_back(tl); }
}

template <int G, int R, bool HS>
int launch_trace_variant(Engine &E, Stage &S, cudaStream_t stream, const TaskSrc &ts, int max_n, const uint8_t *seq_codes,
                         bool seq_ascii, const uint8_t *ad_codes, const Scoring &sc, int32_t *out, int *status) {
    constexpr int SPW = 32 / G;
    constexpr int WPS = TraceWords<R>::value;
    const int max_steps = max_n + G - 1;
    const int wpb = PB_WARPS_PER_BLOCK;
    const size_t hb_words = HS ? (size_t)SPW * max_n : 0;
    const size_t smem_bytes = ((size_t)wpb * (hb_words + PB_SCRATCH_WORDS) + (seq_ascii ? PB_CODE_TAB_WORDS : 0)) * 4;
    auto kern = trace_kernel<G, R, HS>;
    int bps = 0;
    if (int rc = E.blocks_per_sm(reinterpret_cast<const void *>(kern), wpb * 32, smem_bytes, &bps)) return rc;
    const size_t gwarp_bytes = ((size_t)((max_steps + PB_TCHUNK - 1) / PB_TCHUNK) * PB_TCHUNK * WPS * 32 +
                                (HS ? 0 : (((size_t)SPW * max_n + 31) & ~(size_t)31))) * 4;   // 128-byte lines per warp (kernels.cuh)
    // The trace scratch of the resident grid is rewritten slot after slot and partly lives in L2.  `scratch_mb` caps
    // it (whole blocks per SM, never below 2).  A smaller cap keeps more of the trace in L2 but leaves fewer warps
    // resident: on H100 (50 MB L2) 72 MB made the end-trim launches 23 % slower than the default 128 MB, the smallest cap
    // that reaches the kernel's occupancy limit; the dead trace lines written back to HBM are off the critical path.
    // See DESIGN.md, "trace scratch".
    int64_t max_blocks = std::max<int64_t>(2 * E.sm_count, (int64_t)(((size_t)g_opt.scratch_mb << 20) / std::max<size_t>(gwarp_bytes * wpb, 1)));
    max_blocks -= max_blocks % E.sm_count;     // whole blocks per SM: the grid-stride loop gives every block the same work
    const int64_t n_tasks = ts.n_tasks;
    const int64_t n_slots = (n_tasks + 1) / 2;
    const int64_t n_wslots = (n_slots + SPW - 1) / SPW;
    int64_t blocks = (n_wslots + wpb - 1) / wpb;
    blocks = std::min<int64_t>(blocks, std::min<int64_t>((int64_t)bps * E.sm_count, max_blocks));
    if ((size_t)blocks * wpb * gwarp_bytes > (24ull << 30)) blocks = std::max<int64_t>(1, (int64_t)((24ull << 30) / (gwarp_bytes * wpb)));
    if (blocks <= 0) return 0;
    if (int rc = S.gtrace.ensure((size_t)blocks * wpb * gwarp_bytes)) return rc;
    TimedLaunch tl; bool on;
    timed_begin(E, stream, tl, on, E.next_trace_kind);
    kern<<<(unsigned)blocks, wpb * 32, smem_bytes, stream>>>(ts, seq_codes, ad_codes, sc, out, S.gtrace.as<uint32_t>(), max_steps,
                                                              max_n, seq_ascii ? 1 : 0, status);
    timed_end(E, stream, tl, on);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}

template <int G, int R>
int launch_trace(Engine &E, Stage &S, cudaStream_t stream, const TaskSrc &ts, int max_n, const uint8_t *seq_codes,
                 bool seq_ascii, const uint8_t *ad_codes, const Scoring &sc, int32_t *out, int *status) {
    constexpr int SPW = 32 / G;
    if (max_n < 1) max_n = 1;
    // packed read bases of a slot are staged in shared memory when they fit (<= 12 KB per warp), else in global scratch
    const bool hs = g_opt.hbuf_mode == 1 ? true : g_opt.hbuf_mode == 2 ? false : ((size_t)SPW * max_n * 4 <= 12288);
    if (hs && ((size_t)PB_WARPS_PER_BLOCK * ((size_t)SPW * max_n + 4 + PB_SCRATCH_WORDS) + PB_CODE_TAB_WORDS) * 4 <= E.smem_optin)
        return launch_trace_variant<G, R, true>(E, S, stream, ts, max_n, seq_codes, seq_ascii, ad_codes, sc, out, status);
    return launch_trace_variant<G, R, false>(E, S, stream, ts, max_n, seq_codes, seq_ascii, ad_codes, sc, out, status);
}

// seq_ascii: `seq_codes` holds the caller's ASCII bytes, which the trace kernel encodes as it stages them (single pass only)
int launch_trace_class(Engine &E, Stage &S, cudaStream_t stream, int cls, const TaskSrc &ts, int max_n, const uint8_t *seq_codes,
                       bool seq_ascii, const uint8_t *ad_codes, const Scoring &sc, int32_t *out, int *status) {
#define PB_CASE(K, GG, RR) case K: return launch_trace<GG, RR>(E, S, stream, ts, max_n, seq_codes, seq_ascii, ad_codes, sc, out, status);
    switch (cls) {
        PB_CASE(0, 4, 5) PB_CASE(1, 4, 6) PB_CASE(2, 4, 7) PB_CASE(3, 4, 8)
        PB_CASE(4, 8, 5) PB_CASE(5, 8, 6) PB_CASE(6, 8, 7) PB_CASE(7, 8, 8)
        PB_CASE(8, 16, 5) PB_CASE(9, 16, 6) PB_CASE(10, 16, 7) PB_CASE(11, 16, 8)
        PB_CASE(12, 32, 5) PB_CASE(13, 32, 6) PB_CASE(14, 32, 7) PB_CASE(15, 32, 8)
    }
#undef PB_CASE
    return fail(PB200_ERR_INTERNAL, "bad class");
}

template <int G, int R, bool PROF>
int launch_score_variant(Engine &E, cudaStream_t stream, const TaskSrc &ts, unsigned long long *counter,
                         const uint8_t *seq_codes, const uint8_t *ad_codes, const Scoring &sc, EndCell *ends) {
    auto kern = score_kernel<G, R, PROF>;
    int bps = 0;
    if (int rc = E.blocks_per_sm(reinterpret_cast<const void *>(kern), PB_WARPS_PER_BLOCK * 32, 0, &bps)) return rc;
    constexpr int SPW = 32 / G;
    const int64_t n_tasks = ts.n_tasks;
    const int64_t n_slots = (n_tasks + 1) / 2;
    int64_t blocks = (n_slots + SPW * PB_WARPS_PER_BLOCK - 1) / (SPW * PB_WARPS_PER_BLOCK);
    blocks = std::min<int64_t>(blocks, (int64_t)bps * E.sm_count);
    if (blocks <= 0) return 0;
    CK(cudaMemsetAsync(counter, 0, sizeof(unsigned long long), stream));
    TimedLaunch tl; bool on;
    timed_begin(E, stream, tl, on, TK_SCORE);
    kern<<<(unsigned)blocks, PB_WARPS_PER_BLOCK * 32, 0, stream>>>(ts, counter, seq_codes, ad_codes, sc, ends);
    timed_end(E, stream, tl, on);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}
template <int G, int R>
int launch_score(Engine &E, cudaStream_t stream, const TaskSrc &ts, unsigned long long *counter, const uint8_t *seq_codes,
                 const uint8_t *ad_codes, const Scoring &sc, EndCell *ends) {
    // query profile: every slot is (one read, two adapters) -- cross mode with an even number of adapters in the class
    const bool prof = g_opt.profile != 0 && ts.tasks == nullptr && ts.n_cls_ad > 0 && (ts.n_cls_ad % 2) == 0;
    if (prof) return launch_score_variant<G, R, true>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
    return launch_score_variant<G, R, false>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
}
int launch_score_class(Engine &E, cudaStream_t stream, int cls, const TaskSrc &ts,
                       unsigned long long *counter, const uint8_t *seq_codes, const uint8_t *ad_codes, const Scoring &sc,
                       EndCell *ends) {
    switch (cls / 4) {
        case 0: return launch_score<4, 8>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
        case 1: return launch_score<8, 8>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
        case 2: return launch_score<16, 8>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
        case 3: return launch_score<32, 8>(E, stream, ts, counter, seq_codes, ad_codes, sc, ends);
    }
    return fail(PB200_ERR_INTERNAL, "bad class");
}

int launch_unpack(cudaStream_t stream, const uint8_t *in, uint8_t *out, int64_t n, int sm_count) {
    if (n <= 0) return 0;
    int64_t blocks = std::min<int64_t>((n + 256 * 16 - 1) / (256 * 16), (int64_t)sm_count * 16);
    unpack_kernel<<<(unsigned)blocks, 256, 0, stream>>>(in, out, n);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}

int launch_encode(cudaStream_t stream, const uint8_t *in, uint8_t *out, int64_t n, int sm_count) {
    if (n <= 0) return 0;
    int64_t blocks = std::min<int64_t>((n + 256 * 16 - 1) / (256 * 16), (int64_t)sm_count * 16);
    encode_kernel<<<(unsigned)blocks, 256, 0, stream>>>(in, out, n);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}


// Run every task of one class; `ts` describes the tasks in slot order (explicit records or the cross product).
// seq_ascii: the sequences are the caller's ASCII bytes (see single_pass_ascii); only the single-pass trace takes them.
int run_class_tasks(Engine &E, Stage &S, cudaStream_t stream, int cls, int m_max, const TaskSrc &ts, int64_t max_n,
                    const uint8_t *seq_codes, const uint8_t *ad_codes, const Scoring &sc, const SchemeInfo &si,
                    int32_t *out, int *status, unsigned long long *counter, bool seq_ascii = false) {
    const int64_t n_tasks = ts.n_tasks;
    if (n_tasks <= 0) return 0;
    if (seq_ascii && max_n > g_opt.direct_max) return fail(PB200_ERR_INTERNAL, "ASCII sequences reached the two-pass path");
    if (g_opt.profile != 0 && ts.tasks == nullptr && ts.cls_ad != nullptr && ts.n_cls_ad >= 3 && (ts.n_cls_ad & 1) &&
        si.bounded && max_n > g_opt.direct_max) {
        // the score pass's query profile needs same-read slots: the paired adapters (one read, two adapters per slot) and the
        // odd last adapter (two reads per slot) run as two launch sequences; cross_task() indexes both exactly as it does
        // inside the whole class
        TaskSrc paired = ts, tail = ts;
        paired.n_cls_ad = ts.n_cls_ad - 1;
        paired.n_tasks = ts.n_seqs * (int64_t)paired.n_cls_ad;
        tail.cls_ad = ts.cls_ad + (ts.n_cls_ad - 1);
        tail.n_cls_ad = 1;
        tail.n_tasks = ts.n_seqs;
        if (int rc = run_class_tasks(E, S, stream, cls, m_max, paired, max_n, seq_codes, ad_codes, sc, si, out, status, counter)) return rc;
        return run_class_tasks(E, S, stream, cls, m_max, tail, max_n, seq_codes, ad_codes, sc, si, out, status, counter);
    }
    int64_t W = si.bounded ? (int64_t)m_max + ((int64_t)m_max * si.wnum) / si.wden : (int64_t)1 << 40;
    const bool two_pass = si.bounded && max_n > g_opt.direct_max && W + 1 < max_n;
    if (!two_pass) return launch_trace_class(E, S, stream, cls, ts, (int)max_n, seq_codes, seq_ascii, ad_codes, sc, out, status);
    if (int rc = S.ends.ensure((size_t)n_tasks * sizeof(EndCell))) return rc;
    if (int rc = S.tasks2.ensure((size_t)n_tasks * sizeof(Task))) return rc;
    if (int rc = launch_score_class(E, stream, cls, ts, counter, seq_codes, ad_codes, sc, S.ends.as<EndCell>())) return rc;
    {
        int64_t blocks = (n_tasks + 255) / 256;
        if (!E.wcells.p) {
            if (int rc = E.wcells.ensure(8)) return rc;
            CK(cudaMemsetAsync(E.wcells.p, 0, 8, stream));
        }
        window_tasks_kernel<<<(unsigned)blocks, 256, 0, stream>>>(ts, S.ends.as<EndCell>(), S.tasks2.as<Task>(), si.wnum, si.wden, g_opt.tight_window,
                                                                   E.wcells.as<unsigned long long>());
        g_launches++;
        CK(cudaGetLastError());
    }
    TaskSrc t2 = ts;
    t2.tasks = S.tasks2.as<Task>();
    E.next_trace_kind = TK_TRACE_WINDOW;
    const int rc2 = launch_trace_class(E, S, stream, cls, t2, (int)W, seq_codes, false, ad_codes, sc, out, status);
    E.next_trace_kind = TK_TRACE;
    return rc2;
}

// Adapter-side planning shared by all entry points.
struct AdapterPlan {
    std::vector<ClassPlan> classes;   // non-empty classes only
    SchemeInfo si;
    Scoring sc;
    const uint8_t *d_ad_codes = nullptr;   // device copies owned by the engine's plan cache
    const int32_t *d_ad_off = nullptr;
    const int32_t *d_cls_ad = nullptr;
};
int plan_adapters(Engine &E, cudaStream_t stream, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters,
                  int ma, int mi, int go, int ge, AdapterPlan &P) {
    const size_t nb = (size_t)ad_off[n_adapters];
    Engine::PlanEntry *slot = nullptr;
    for (auto &e : E.plans) {
        if (e.valid && e.plan && e.sc[0] == ma && e.sc[1] == mi && e.sc[2] == go && e.sc[3] == ge &&
            e.off.size() == (size_t)n_adapters + 1 && e.ad.size() == nb &&
            memcmp(e.off.data(), ad_off, e.off.size() * 4) == 0 && (nb == 0 || memcmp(e.ad.data(), adapters, nb) == 0)) {
            e.last_used = ++E.plan_clock;
            P = *static_cast<AdapterPlan *>(e.plan.get());
            return 0;
        }
    }
    for (auto &e : E.plans) if (!slot || !e.valid || (slot->valid && e.last_used < slot->last_used)) { slot = &e; if (!e.valid) break; }
    slot->valid = false;
    // the entry's device copies are about to change: everything queued by earlier calls must be done with them
    CK(cudaDeviceSynchronize());
    Engine::PlanEntry &PE = *slot;
    P.si = scheme_info(ma, mi, go, ge);
    P.sc = make_scoring(ma, mi, go, ge);
    std::vector<ClassPlan> cl(N_CLASSES);
    for (int c = 0; c < N_CLASSES; ++c) cl[c].cls = c;
    // Slots pair two alignments.  In cross mode a slot is (one read, two adapters): sort the adapters by length and
    // pair neighbours; the pair runs in the row-capacity class of its longer member, provided the shorter one would
    // not waste more than ~1/3 of the rows (otherwise it stays single and pairs two consecutive reads instead).
    std::vector<int32_t> order16;
    for (int a = 0; a < n_adapters; ++a) {
        int m = ad_off[a + 1] - ad_off[a];
        if (m < 0) return fail(PB200_ERR_ARG, "adapter offsets not monotone");
        int c = class_of(P.si, m);
        if (c == GENERIC_CLASS) { cl[c].ad_ids.push_back(a); cl[c].m_max = std::max(cl[c].m_max, m); }
        else order16.push_back(a);
    }
    auto len = [&](int a) { return ad_off[a + 1] - ad_off[a]; };
    std::stable_sort(order16.begin(), order16.end(), [&](int x, int y) { return len(x) > len(y); });
    std::vector<int32_t> single_of(N_CLASSES, -1);
    for (size_t i = 0; i < order16.size();) {
        const int a = order16[i], ca = class_of(P.si, len(a));
        const int capa = class_G(ca) * class_R(ca);
        if (i + 1 < order16.size()) {
            const int b = order16[i + 1], cb = class_of(P.si, len(b));
            const int capb = class_G(cb) * class_R(cb);
            if (3 * capa <= 4 * capb) {            // cap ratio <= 1.33: share a slot
                cl[ca].ad_ids.push_back(a); cl[ca].ad_ids.push_back(b);
                cl[ca].m_max = std::max(cl[ca].m_max, len(a));
                i += 2;
                continue;
            }
        }
        single_of[ca] = a;                          // at most one per class (it sits at the class's lower boundary)
        cl[ca].m_max = std::max(cl[ca].m_max, len(a));
        i += 1;
    }
    for (int c = 0; c < GENERIC_CLASS; ++c) if (single_of[c] >= 0) cl[c].ad_ids.push_back(single_of[c]);
    for (auto &c : cl) if (!c.ad_ids.empty()) P.classes.push_back(c);
    const size_t ad_bytes = (size_t)ad_off[n_adapters];
    if (int rc = PE.ad_raw.ensure(ad_bytes + 16)) return rc;
    if (int rc = PE.ad_codes.ensure(ad_bytes + 16)) return rc;
    if (int rc = PE.ad_off.ensure((size_t)(n_adapters + 1) * 4)) return rc;
    if (ad_bytes) CK(cudaMemcpyAsync(PE.ad_raw.p, adapters, ad_bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaMemcpyAsync(PE.ad_off.p, ad_off, (size_t)(n_adapters + 1) * 4, cudaMemcpyHostToDevice, stream));
    if (int rc = launch_encode(stream, PE.ad_raw.as<uint8_t>(), PE.ad_codes.as<uint8_t>(), (int64_t)ad_bytes, E.sm_count)) return rc;
    // class adapter-id lists, concatenated
    std::vector<int32_t> flat;
    for (auto &c : P.classes) flat.insert(flat.end(), c.ad_ids.begin(), c.ad_ids.end());
    if (int rc = PE.cls_ad.ensure(flat.size() * 4 + 16)) return rc;
    if (!flat.empty()) CK(cudaMemcpyAsync(PE.cls_ad.p, flat.data(), flat.size() * 4, cudaMemcpyHostToDevice, stream));
    // the host vectors above are pageable: the async copies have been staged by the driver before returning
    CK(cudaStreamSynchronize(stream));
    P.d_ad_codes = PE.ad_codes.as<uint8_t>(); P.d_ad_off = PE.ad_off.as<int32_t>(); P.d_cls_ad = PE.cls_ad.as<int32_t>();
    PE.ad.assign(adapters, adapters + ad_bytes);
    PE.off.assign(ad_off, ad_off + n_adapters + 1);
    PE.sc[0] = ma; PE.sc[1] = mi; PE.sc[2] = go; PE.sc[3] = ge;
    PE.plan = std::make_shared<AdapterPlan>(P);
    PE.last_used = ++E.plan_clock;
    PE.valid = true;
    return 0;
}

// Alignments of the generic (int32) class, planned on the host (which needs the sequence lengths there) and batched so that
// a batch's trace matrices fit a 2 GiB scratch: one generic_kernel launch per batch, waited for before the scratch is reused.
// The last batch runs at flush().
struct GenericBatch {
    Engine &E;
    cudaStream_t stream;
    const uint8_t *seq_codes, *ad_codes;
    const Scoring &sc;
    int32_t *out;
    std::vector<GenericJob> jobs;
    size_t used = 0;
    int add(int64_t seq_off, int32_t n, int32_t m, int32_t ad_off, int32_t out_idx) {
        size_t tb = (((size_t)(n + 1) * (size_t)(m + 1) + 3) & ~(size_t)3) + (size_t)(m + 1) * 8;
        tb = (tb + 15) & ~(size_t)15;
        if (tb > (64ull << 30)) return fail(PB200_ERR_ARG, "alignment too large for the generic int32 path");
        if (used + tb > (2ull << 30) && !jobs.empty()) { if (int rc = flush()) return rc; }
        jobs.push_back(GenericJob{seq_off, n, m, ad_off, out_idx, (int64_t)used});
        used += tb;
        return 0;
    }
    int flush() {
        if (jobs.empty()) return 0;
        if (int rc = E.gjobs.ensure(jobs.size() * sizeof(GenericJob))) return rc;
        if (int rc = E.gscratch.ensure(used + 64)) return rc;
        CK(cudaMemcpyAsync(E.gjobs.p, jobs.data(), jobs.size() * sizeof(GenericJob), cudaMemcpyHostToDevice, stream));
        int nb = (int)((jobs.size() + 63) / 64);
        generic_kernel<<<nb, 64, 0, stream>>>(E.gjobs.as<GenericJob>(), (int)jobs.size(), seq_codes, ad_codes, sc.ma, sc.mi,
                                              sc.go, sc.ge, E.gscratch.as<uint8_t>(), out);
        g_launches++;
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(stream));
        jobs.clear(); used = 0;
        return 0;
    }
};

int run_generic_cross(Engine &E, cudaStream_t stream, const ClassPlan &C, const int64_t *h_seq_off, int64_t s0, int64_t cnt,
                      int64_t base_off, const int32_t *h_ad_off, int32_t n_adapters, const uint8_t *seq_codes,
                      const uint8_t *ad_codes, const Scoring &sc, int32_t *out) {
    GenericBatch G{E, stream, seq_codes, ad_codes, sc, out};
    for (int64_t s = s0; s < s0 + cnt; ++s)
        for (int32_t a : C.ad_ids)
            if (int rc = G.add(h_seq_off[s] - base_off, (int32_t)(h_seq_off[s + 1] - h_seq_off[s]), h_ad_off[a + 1] - h_ad_off[a],
                               h_ad_off[a], (int32_t)((s - s0) * n_adapters + a))) return rc;
    return G.flush();
}

// Cross product of sequences [s0, s0+cnt) (already encoded on the device, offsets on the device) with all adapters.
// d_seq_off points at the offset of sequence s0 (cnt+1 entries), base_off is subtracted from every offset.
// seq_order (optional): slot i is sequence seq_order[i] of d_seq_off (the active reads of a middle-scan round); without it
// the two-pass path orders the sequences longest first itself.
// seq_ascii: `seq_codes` holds the caller's ASCII bytes; only when single_pass_ascii(P, max_n) holds.
int run_cross_chunk(Engine &E, Stage &S, cudaStream_t stream, const AdapterPlan &P, const uint8_t *seq_codes,
                    const int64_t *d_seq_off, int64_t cnt, int64_t base_off, int64_t max_n, int32_t n_adapters,
                    int32_t *d_out, const int64_t *h_seq_off_abs, int64_t s0, const int32_t *h_ad_off,
                    const int32_t *seq_order = nullptr, bool seq_ascii = false) {
    if (int rc = S.misc.ensure(64)) return rc;
    int *status = S.misc.as<int>();
    unsigned long long *counter = reinterpret_cast<unsigned long long *>(S.misc.as<char>() + 16);
    // long reads (two-pass path): process sequences longest first
    const int32_t *d_order = seq_order;
    if (!seq_order && P.si.bounded && max_n > g_opt.direct_max && cnt > 1) {
        if (int rc = S.order.ensure((size_t)cnt * 4)) return rc;
        if (int rc = S.bins.ensure((size_t)PB_ORDER_BINS * 4)) return rc;
        CK(cudaMemsetAsync(S.bins.p, 0, (size_t)PB_ORDER_BINS * 4, stream));
        const unsigned nb = (unsigned)((cnt + 255) / 256);
        order_hist_kernel<<<nb, 256, 0, stream>>>(d_seq_off, cnt, max_n, S.bins.as<unsigned>());
        order_scan_kernel<<<1, 256, 0, stream>>>(S.bins.as<unsigned>());
        order_scatter_kernel<<<nb, 256, 0, stream>>>(d_seq_off, cnt, max_n, S.bins.as<unsigned>(), S.order.as<int32_t>());
        g_launches += 3;
        CK(cudaGetLastError());
        d_order = S.order.as<int32_t>();
    }
    size_t cls_pos = 0;
    for (const ClassPlan &C : P.classes) {
        const int32_t *d_cls = P.d_cls_ad + cls_pos;
        cls_pos += C.ad_ids.size();
        if (C.cls == GENERIC_CLASS) {
            if (!h_seq_off_abs) return fail(PB200_ERR_INTERNAL, "generic class needs host offsets");
            if (seq_ascii) return fail(PB200_ERR_INTERNAL, "ASCII sequences reached the generic class");
            if (int rc = run_generic_cross(E, stream, C, h_seq_off_abs, s0, cnt, base_off, h_ad_off, n_adapters, seq_codes,
                                           P.d_ad_codes, P.sc, d_out)) return rc;
            continue;
        }
        TaskSrc ts;
        ts.tasks = nullptr;                                  // cross product, synthesised in the kernels
        ts.n_tasks = cnt * (int64_t)C.ad_ids.size();
        ts.cls_ad = d_cls; ts.n_cls_ad = (int32_t)C.ad_ids.size(); ts.n_adapters = n_adapters;
        ts.n_seqs = cnt; ts.seq_off = d_seq_off; ts.ad_off = P.d_ad_off;
        ts.seq_order = d_order;
        if (ts.n_tasks == 0) continue;
        (void)base_off;
        if (int rc = run_class_tasks(E, S, stream, C.cls, C.m_max, ts, max_n, seq_codes, P.d_ad_codes, P.sc,
                                     P.si, d_out, status, counter, seq_ascii)) return rc;
    }
    return 0;
}

// True when every class of the plan runs through the single-pass trace kernel at reads of up to max_n bases (no generic
// class, no score pass): the trace kernel then encodes the caller's ASCII bytes as it stages them, and the encode pass over
// the batch (a read and a write of every byte) and its code buffer are not needed.
bool single_pass_ascii(const AdapterPlan &P, int64_t max_n) {
    if (max_n > g_opt.direct_max) return false;
    for (const ClassPlan &C : P.classes) if (C.cls == GENERIC_CLASS) return false;
    return true;
}

// the error a status word reports (0: none)
int status_error(int st) {
    if (st & 1) return fail(PB200_ERR_INTERNAL, "traceback left its window (window bound violated)");
    if (st & 2) return fail(PB200_ERR_INTERNAL, "decision kernel: value outside its table (len_aln >= table length or count > 65535)");
    return 0;
}
int check_status(Stage &S, cudaStream_t stream) {
    int st = 0;
    CK(cudaMemcpyAsync(&st, S.misc.p, 4, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    return status_error(st);
}

// S.misc: status word at offset 0, score-pass counter at 16, max-length scratch at 32, pb200EmitReadsDevice's record-check flag
// at 48, pb200ParseReadsDevice's check flags at 56.  The status word is sticky until
// pb200Synchronize, which reports and clears it: a deferred error of an earlier device-resident call must not be lost, so a
// call clears the word only when it allocates it, and everything behind it always.
int reset_misc(Stage &S, cudaStream_t stream) {
    const bool fresh = S.misc.p == nullptr;
    if (int rc = S.misc.ensure(64)) return rc;
    CK(cudaMemsetAsync(S.misc.as<char>() + (fresh ? 0 : 16), 0, fresh ? 64 : 48, stream));
    return 0;
}

// seq_off rebasing kernel: offsets of a chunk relative to its first byte
__global__ void rebase_kernel(int64_t *off, int64_t n, int64_t base) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) off[i] -= base;
}
// ... and for a chunk of equally long sequences the offsets are made on the device instead of crossing PCIe (8 bytes per
// 150-byte window are 5 % of the upload of an end-trim step)
__global__ void stride_offsets_kernel(int64_t *off, int64_t n, int64_t stride) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) off[i] = i * stride;
}

// ... and the offsets of a middle-scan chunk, shifted to the segment's resident code buffer (the last entry is also the next
// chunk's first: both chunks write the same value)
__global__ void shift_offsets_kernel(const int64_t *in, int64_t *out, int64_t n, int64_t delta) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] + delta;
}

// Resident state of one segment of a middle-adapter scan: the segment's codes (masked in place round after round), offsets of
// its reads into `codes` (segment-relative read ids), records (read-major), next adapter per read, hit slots, active lists.
struct MiddleSeg {
    uint8_t *codes = nullptr;
    int64_t *off = nullptr;               // off[s], s = 0 .. n (host API: written chunk by chunk in round 0)
    int64_t n = 0, max_len = 0;
    int32_t *rec = nullptr, *next_ad = nullptr, *hits = nullptr, *active[2] = {nullptr, nullptr};
    unsigned *count = nullptr;
    unsigned long long *max_len_d = nullptr;
    const int32_t *cmin = nullptr;
    int32_t cmin_len = 0;
};

int launch_middle_decide(Engine &E, cudaStream_t stream, const MiddleSeg &M, int32_t n_adapters, const int32_t *active,
                         int64_t first, int64_t n, int32_t *next_active, int *status) {
    if (n <= 0) return 0;
    MiddleArgs a;
    a.records = M.rec; a.n_adapters = n_adapters;
    a.active = active; a.first = first; a.n = n;
    a.next_ad = M.next_ad; a.seq_off = M.off; a.codes = M.codes;
    a.cmin = M.cmin; a.cmin_len = M.cmin_len;
    a.hits = M.hits; a.next_active = next_active; a.count = M.count; a.max_len = M.max_len_d;
    const int64_t blocks = std::min<int64_t>((n + 3) / 4, (int64_t)E.sm_count * 16);
    middle_decide_kernel<<<(unsigned)blocks, 128, 0, stream>>>(a, status);
    g_launches++;
    CK(cudaGetLastError());
    return 0;
}

// One pipeline chunk of the host-buffer API: sequences [s0, s1), longest sequence max_n.
struct HostChunk { int64_t s0, s1, max_n; bool uniform; };   // uniform: every sequence of the chunk has length max_n

// Pure host work done before the device is touched: argument validation (so a bad call fails the same way with or
// without a device).  Pair-list mode checks everything here; in cross mode the sequence offsets are checked chunk by chunk
// while the pipeline runs (next_chunk), so that the scan of chunk k+1 hides behind the device's work on chunk k.
int validate_args(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
                  const int32_t *ad_off, int32_t n_adapters, const int32_t *pair_seq, const int32_t *pair_adapter,
                  int64_t n_pairs, bool cross) {
    for (int32_t a = 0; a < n_adapters; ++a)
        if (ad_off[a + 1] < ad_off[a]) return fail(PB200_ERR_ARG, "adapter offsets not monotone");
    if (n_adapters > 0 && ad_off[0] < 0) return fail(PB200_ERR_ARG, "negative adapter offset");
    if (n_adapters > 0 && ad_off[n_adapters] > 0 && !adapters) return fail(PB200_ERR_ARG, "NULL adapter buffer");
    if (n_seqs > 0 && seq_off[n_seqs] > seq_off[0] && !seqs) return fail(PB200_ERR_ARG, "NULL sequence buffer");
    if (n_seqs > 0 && seq_off[0] < 0) return fail(PB200_ERR_ARG, "negative sequence offset");
    if (cross) return 0;
    if (n_pairs > 0x7fffffffll) return fail(PB200_ERR_ARG, "pair-list mode supports < 2^31 pairs per call");
    for (int64_t s = 0; s < n_seqs; ++s) {
        const int64_t len = seq_off[s + 1] - seq_off[s];
        if (len < 0) return fail(PB200_ERR_ARG, "sequence offsets not monotone");
        if (len > 0x7fff0000ll) return fail(PB200_ERR_ARG, "sequence longer than 2^31");
    }
    for (int64_t p = 0; p < n_pairs; ++p)
        if (pair_seq[p] < 0 || pair_seq[p] >= n_seqs || pair_adapter[p] < 0 || pair_adapter[p] >= n_adapters)
            return fail(PB200_ERR_ARG, "pair index out of range");
    return 0;
}

// The pipeline chunk that starts at sequence s0 of a cross-product job: chunk_tasks alignments (at most task_cap: the first
// chunks of a submit are smaller, see chunk_cap), at most chunk_bytes of sequence (but enough sequences to fill the GPU),
// its longest sequence, offsets checked.
int next_chunk(const int64_t *seq_off, int64_t n_seqs, int32_t n_adapters, int64_t s0, HostChunk &c, int64_t task_cap) {
    const int64_t max_cnt = std::max<int64_t>(1, std::min(g_opt.chunk_tasks, task_cap) / std::max<int32_t>(n_adapters, 1));
    int64_t s1 = std::min(n_seqs, s0 + max_cnt);
    while (s1 - s0 > 32768 && seq_off[s1] - seq_off[s0] > g_opt.chunk_bytes) s1 = s0 + std::max<int64_t>(32768, (s1 - s0) / 2);
    c = HostChunk{s0, s1, 0, false};
    int64_t mx = 0, mn = 0, shortest = INT64_MAX;
    for (int64_t s = s0; s < s1; ++s) {
        const int64_t len = seq_off[s + 1] - seq_off[s];
        mx = std::max(mx, len);
        mn = std::min(mn, len);
        shortest = std::min(shortest, len);
    }
    if (mn < 0) return fail(PB200_ERR_ARG, "sequence offsets not monotone");
    if (mx > 0x7fff0000ll) return fail(PB200_ERR_ARG, "sequence longer than 2^31");
    c.max_n = mx;
    c.uniform = s1 > s0 && shortest == mx;      // fixed-stride windows (the end windows of reads >= end_size): offsets are i * max_n
    return 0;
}

// One cross-product job of the host-buffer API (all sequences x all adapters of one call / one batch of a multi call).
struct CrossJob {
    const uint8_t *seqs; const int64_t *seq_off; int64_t n_seqs;
    const uint8_t *adapters; const int32_t *ad_off; int32_t n_adapters;
    int32_t *out;
    // decisions on the device (adapterEndDecisions): records are reduced per read before anything is copied back
    const pb200_end_batch_t *dec = nullptr;
    const int32_t *d_cmin = nullptr; int32_t cmin_len = 0;
    const int32_t *d_cols = nullptr;
    int64_t max_seq_len = 0;          // decision jobs: longest window the threshold table covers
    // middle scan (adapterMiddleScan): codes, offsets and records go to the segment's resident buffers instead of the stage's,
    // and middle_decide_kernel runs round 0 on each chunk; nothing is copied back
    const MiddleSeg *mid = nullptr;
    // adapter-set search (adapterSetSearch): search_best_kernel reduces each chunk's records into the batch's columns of the
    // stage's accumulator slice (Engine::search_acc); -1 = not a search batch
    int64_t search_col = -1;
};

// The first chunks of a submit ramp up (1/8, 1/4, 1/2 of chunk_tasks): the pipeline's fill -- pack + H2D of chunk 0 before
// any DP kernel can start -- costs an eighth of what a full chunk would; only when the submit is large enough to matter.
int64_t chunk_cap(size_t k, int64_t total_tasks) {
    if (total_tasks < 4 * g_opt.chunk_tasks || k >= 3) return g_opt.chunk_tasks;
    return std::max<int64_t>(4096, g_opt.chunk_tasks >> (3 - k));
}

// Packed upload or not for a submit of `total_bytes` of sequence.  The packed path is bound by the host conversion, so it
// only pays against the plain PCIe upload with a large packer team; with 8 threads or fewer it is slower.  So "auto" packs
// only large submits and only when the team is large enough (one rank per GPU on a box with few CPUs per rank uploads the
// ASCII bytes as they are).  The gain depends on how many host cycles the process really gets, and non-temporal stores in
// the packer make it slower (the DMA engine then reads the codes from DRAM instead of the last-level cache) -- so the
// default stays the plain upload and packing is an option.
bool pack_wanted(int64_t total_bytes) {
    if (total_bytes <= 0 || g_opt.h2d_pack == 0) return false;
    if (g_opt.h2d_pack > 0) return true;
    return g_opt.pack_threads >= 12 && total_bytes >= (32ll << 20);
}

// One planned (and, with h2d_pack, packed) chunk on its way from the planner to the submit loop.
struct PackItem {
    size_t job = 0;
    HostChunk c{0, 0, 0, false};
    int buf = -1;                 // index of the pinned pack buffer holding the chunk's 4-bit codes (-1: not packed)
    int rc = 0; std::string err;  // planning error (bad offsets): the submit loop stops here
    bool end = false;             // no more chunks
};

// Planning of a submit's chunk sequence (the order of run_cross_jobs' loop), shared by the inline path and the packer thread.
struct ChunkPlanner {
    const std::vector<CrossJob> *jobs;
    size_t j = 0, k = 0;
    int64_t s0 = 0, total_tasks = 0;
    explicit ChunkPlanner(const std::vector<CrossJob> &J) : jobs(&J) {
        for (const CrossJob &x : J) total_tasks += x.n_seqs * (int64_t)x.n_adapters;
    }
    // next chunk -> item (rc / end set accordingly); errors come back as text because the planner may run on another thread
    void next(PackItem &it) {
        it = PackItem();
        while (j < jobs->size() && ((*jobs)[j].n_seqs <= 0 || (*jobs)[j].n_adapters <= 0 || s0 >= (*jobs)[j].n_seqs)) { ++j; s0 = 0; }
        if (j >= jobs->size()) { it.end = true; return; }
        const CrossJob &J = (*jobs)[j];
        it.job = j;
        it.rc = next_chunk(J.seq_off, J.n_seqs, J.n_adapters, s0, it.c, chunk_cap(k, total_tasks));
        if (!it.rc && J.dec && it.c.max_n > J.max_seq_len)
            it.rc = fail(PB200_ERR_ARG, "decision batches take windows of at most end_size bases");
        if (it.rc) { it.err = g_err; return; }
        s0 = it.c.s1;
        ++k;
    }
};

// Packer: a persistent host thread per engine that plans the chunks of a submit and converts them to 4-bit codes (option
// h2d_pack; hostpack.cpp, OpenMP team of pack_threads) AHEAD of the submit loop, into a ring of NPACK pinned buffers -- the
// conversion of chunk k+1.. runs while the submit loop enqueues chunk k and the device works on chunk k-1 (with the
// packer inside the submit loop the e2e step would be bound by the host conversion).
constexpr int NPACK = NSTAGE + 2;
struct Packer {
    std::thread th;
    std::mutex mu;
    std::condition_variable cv;
    const std::vector<CrossJob> *jobs = nullptr;   // request: non-null while a run is wanted
    bool abort = false, stop = false, busy = false;
    std::deque<PackItem> q;
    HostBuf buf[NPACK];
    cudaEvent_t ev[NPACK];
    enum { FREE = 0, QUEUED = 1, INFLIGHT = 2 };
    int state[NPACK] = {0, 0, 0, 0, 0};
    int device = 0;
    bool ev_made = false;

    void loop() {
        cudaSetDevice(device);
        for (;;) {
            const std::vector<CrossJob> *J;
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return stop || (jobs && !busy && q.empty()); });
                if (stop) return;
                J = jobs; busy = true;
            }
            ChunkPlanner plan(*J);
            for (size_t k = 0;; ++k) {
                PackItem it;
                bool stop_now;
                { std::lock_guard<std::mutex> lk(mu); stop_now = abort; }
                if (stop_now) it.end = true; else plan.next(it);
                const int b = (int)(k % NPACK);
                if (!it.end && !it.rc) {
                    bool inflight = false;
                    {   // the buffer's previous chunk must have been taken by the submit loop and its upload must be complete
                        std::unique_lock<std::mutex> lk(mu);
                        cv.wait(lk, [&] { return abort || state[b] != QUEUED; });
                        if (abort) { it = PackItem(); it.end = true; }
                        inflight = state[b] == INFLIGHT;
                    }
                    if (!it.end) {
                        if (inflight) cudaEventSynchronize(ev[b]);
                        const CrossJob &X = (*J)[it.job];
                        const int64_t base = X.seq_off[it.c.s0], bytes = X.seq_off[it.c.s1] - base;
                        g_err.clear();
                        if (bytes > 0 && buf[b].ensure(((size_t)bytes + 1) / 2)) { it.rc = PB200_ERR_CUDA; it.err = g_err; }
                        else if (bytes > 0) { NvtxRange r("pb200:host_pack"); pb_pack_nibbles(X.seqs + base, bytes, buf[b].p, g_opt.pack_threads); }
                        it.buf = b;
                    }
                }
                const bool last = it.end || it.rc != 0;
                {
                    std::lock_guard<std::mutex> lk(mu);
                    if (it.buf >= 0) state[b] = QUEUED;
                    q.push_back(std::move(it));
                    if (last) { jobs = nullptr; busy = false; }
                }
                cv.notify_all();
                if (last) break;
            }
        }
    }
    ~Packer() {
        { std::lock_guard<std::mutex> lk(mu); stop = true; }
        cv.notify_all();
        if (th.joinable()) th.join();
        for (int i = 0; i < NPACK; ++i) if (buf[i].p) { cudaFreeHost(buf[i].p); buf[i].p = nullptr; }
    }
};

// decide_kernel over the records of `cnt` reads (the reads s0 .. s0+cnt-1 of decision batch D) on `stream`: the trims go to
// d_trim (the stage's chunk scratch, or a segment-wide array that later kernels read) and are copied home with the score
// pairs / top2 of the chunk into D's host outputs.  d_top2: the top2 ranking goes there instead (a device array that later
// kernels read), and home only when D.top2 is given.
int launch_decide(Engine &E, Stage &S, cudaStream_t stream, const pb200_end_batch_t &D, const int32_t *records, int64_t cnt,
                  int32_t n_adapters, const int32_t *d_cmin, int32_t cmin_len, const int32_t *d_cols, int32_t *d_trim, int64_t s0,
                  int32_t *d_top2 = nullptr) {
    if (int rc = S.dec_pairs.ensure((size_t)cnt * std::max<int32_t>(D.n_score_cols, 1) * 4)) return rc;
    DecideArgs a;
    a.records = records; a.n = cnt; a.n_adapters = n_adapters;
    a.is_start = D.is_start; a.end_size = D.end_size; a.extra_trim = D.extra_trim_size; a.min_trim = D.min_trim_size;
    a.cmin = d_cmin; a.cmin_len = cmin_len; a.cols = d_cols; a.n_cols = D.n_score_cols;
    a.trim = d_trim;
    a.pairs = (D.score_pairs && D.n_score_cols > 0) ? S.dec_pairs.as<uint32_t>() : nullptr;
    a.top2 = nullptr;
    if (d_top2) {
        a.top2 = d_top2;
    } else if (D.top2) {
        if (int rc = S.dec_top2.ensure((size_t)cnt * 6 * 4)) return rc;
        a.top2 = S.dec_top2.as<int32_t>();
    }
    const int64_t blocks = std::min<int64_t>((cnt + 3) / 4, (int64_t)E.sm_count * 16);
    decide_kernel<<<(unsigned)blocks, 128, 0, stream>>>(a, S.misc.as<int>());
    g_launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(D.trim + s0, d_trim, (size_t)cnt * 4, cudaMemcpyDeviceToHost, stream));
    if (a.pairs)
        CK(cudaMemcpyAsync(D.score_pairs + (size_t)s0 * D.n_score_cols * 2, S.dec_pairs.p,
                           (size_t)cnt * D.n_score_cols * 4, cudaMemcpyDeviceToHost, stream));
    if (a.top2 && D.top2)
        CK(cudaMemcpyAsync(D.top2 + (size_t)s0 * 6, a.top2, (size_t)cnt * 6 * 4, cudaMemcpyDeviceToHost, stream));
    return 0;
}

// Chunks of every job flow through ONE ring of NSTAGE streams (H2D / kernels / D2H of consecutive chunks overlap, also
// across job boundaries: no fill / drain bubble between the start-window and the end-window batch of an end-trim step).
// Caller holds E.mu and has run E.init().
int run_cross_jobs(Engine &E, std::vector<CrossJob> &jobs, int ma, int mi, int go, int ge) {
    NvtxRange submit_range("pb200:submit");
    for (int i = 0; i < NSTAGE; ++i) if (int rc = reset_misc(E.st[i], E.st[i].stream)) return rc;
    int64_t total_bytes = 0;
    for (const CrossJob &J : jobs) if (J.n_seqs > 0 && J.n_adapters > 0) total_bytes += J.seq_off[J.n_seqs] - J.seq_off[0];
    const bool packed = pack_wanted(total_bytes);
    Packer *PK = nullptr;
    if (packed) {
        if (!E.packer) {
            auto pk = std::make_shared<Packer>();
            pk->device = E.device;
            for (int i = 0; i < NPACK; ++i) CK(cudaEventCreateWithFlags(&pk->ev[i], cudaEventDisableTiming));
            pk->ev_made = true;
            pk->th = std::thread([p = pk.get()] { p->loop(); });
            E.packer = pk;
        }
        PK = static_cast<Packer *>(E.packer.get());
        {
            std::lock_guard<std::mutex> lk(PK->mu);
            PK->abort = false;
            PK->jobs = &jobs;
        }
        PK->cv.notify_all();
    }
    ChunkPlanner inline_plan(jobs);
    auto next_item = [&](PackItem &it) {
        if (!PK) { inline_plan.next(it); return; }
        std::unique_lock<std::mutex> lk(PK->mu);
        PK->cv.wait(lk, [&] { return !PK->q.empty(); });
        it = std::move(PK->q.front());
        PK->q.pop_front();
    };
    auto submit = [&](const CrossJob &J, const AdapterPlan &P, const PackItem &it, Stage &S) -> int {
        const HostChunk &c = it.c;
        const int64_t s0 = c.s0, cnt = c.s1 - c.s0;
        const int64_t base = J.seq_off[s0];
        const int64_t bytes = J.seq_off[c.s1] - base;
        cudaStream_t stream = S.stream;
        NvtxRange chunk_range("pb200:chunk");
        {
            NvtxRange r("pb200:stage_wait");
            CK(cudaStreamSynchronize(stream));   // previous use of this stage's buffers is complete
        }
        // a chunk uploaded as ASCII that only the single-pass trace reads is staged from the raw bytes (no encode pass)
        const bool ascii = !J.mid && it.buf < 0 && single_pass_ascii(P, c.max_n);
        if (int rc = S.seq_raw.ensure((size_t)bytes + 16)) return rc;
        if (!J.mid) {
            if (int rc = ascii ? 0 : S.seq_codes.ensure((size_t)bytes + 16)) return rc;
            if (int rc = S.out.ensure((size_t)cnt * J.n_adapters * PB_REC * 4)) return rc;
        }
        if (int rc = S.seq_off.ensure((size_t)(cnt + 1) * 8)) return rc;
        {
        NvtxRange r("pb200:h2d");
        if (it.buf >= 0) {
            // Dna5 conversion was done on the host cores by the packer thread, two codes per byte: half the bytes cross PCIe
            if (bytes) CK(cudaMemcpyAsync(S.seq_raw.p, PK->buf[it.buf].p, ((size_t)bytes + 1) / 2, cudaMemcpyHostToDevice, stream));
            CK(cudaEventRecord(PK->ev[it.buf], stream));
            { std::lock_guard<std::mutex> lk(PK->mu); PK->state[it.buf] = Packer::INFLIGHT; }
            PK->cv.notify_all();
        } else if (bytes) {
            CK(cudaMemcpyAsync(S.seq_raw.p, J.seqs + base, (size_t)bytes, cudaMemcpyHostToDevice, stream));
        }
        if (!c.uniform) CK(cudaMemcpyAsync(S.seq_off.p, J.seq_off + s0, (size_t)(cnt + 1) * 8, cudaMemcpyHostToDevice, stream));
        }
        NvtxRange dp_range("pb200:dp");
        const int64_t mid_rel = J.mid ? base - J.seq_off[0] : 0;     // the chunk's first byte in the segment's resident codes
        uint8_t *codes = J.mid ? J.mid->codes + mid_rel : ascii ? S.seq_raw.as<uint8_t>() : S.seq_codes.as<uint8_t>();
        int32_t *recs = J.mid ? J.mid->rec + (size_t)s0 * J.n_adapters * PB_REC : S.out.as<int32_t>();
        if (c.uniform) stride_offsets_kernel<<<(unsigned)((cnt + 1 + 255) / 256), 256, 0, stream>>>(S.seq_off.as<int64_t>(), cnt + 1, c.max_n);
        else rebase_kernel<<<(unsigned)((cnt + 1 + 255) / 256), 256, 0, stream>>>(S.seq_off.as<int64_t>(), cnt + 1, base);
        g_launches++;
        if (J.mid) {
            shift_offsets_kernel<<<(unsigned)((cnt + 1 + 255) / 256), 256, 0, stream>>>(S.seq_off.as<int64_t>(), J.mid->off + s0,
                                                                                     cnt + 1, mid_rel);
            g_launches++;
        }
        if (it.buf >= 0) {
            if (int rc = launch_unpack(stream, S.seq_raw.as<uint8_t>(), codes, bytes, E.sm_count)) return rc;
        } else if (!ascii) {
            if (int rc = launch_encode(stream, S.seq_raw.as<uint8_t>(), codes, bytes, E.sm_count)) return rc;
        }
        if (int rc = run_cross_chunk(E, S, stream, P, codes, S.seq_off.as<int64_t>(), cnt, base, c.max_n,
                                     J.n_adapters, recs, J.seq_off, s0, J.ad_off, nullptr, ascii)) return rc;
        if (J.mid) {
            if (int rc = launch_middle_decide(E, stream, *J.mid, J.n_adapters, nullptr, s0, cnt, J.mid->active[0],
                                              S.misc.as<int>())) return rc;
        }
        if (J.dec) {
            if (int rc = S.dec_trim.ensure((size_t)cnt * 4)) return rc;
            if (int rc = launch_decide(E, S, stream, *J.dec, S.out.as<int32_t>(), cnt, J.n_adapters, J.d_cmin, J.cmin_len, J.d_cols,
                                       S.dec_trim.as<int32_t>(), s0)) return rc;
        }
        if (J.search_col >= 0) {
            unsigned long long *best = E.search_acc.as<unsigned long long>() + (size_t)(&S - E.st) * E.search_cols + J.search_col;
            // one u64 per adapter in shared memory while that fits the default 48 KB of a block
            const size_t smem_bytes = (size_t)J.n_adapters * 8;
            const int use_smem = smem_bytes <= 48 * 1024 ? 1 : 0;
            const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((cnt * J.n_adapters + 4095) / 4096, (int64_t)E.sm_count * 2));
            search_best_kernel<<<(unsigned)blocks, 256, use_smem ? smem_bytes : 0, stream>>>(static_cast<const int32_t *>(S.out.as<int32_t>()),
                                                                                 cnt, J.n_adapters, best, use_smem);
            g_launches++;
            CK(cudaGetLastError());
        }
        if (J.out) {
            NvtxRange r("pb200:d2h");
            CK(cudaMemcpyAsync(J.out + (size_t)s0 * J.n_adapters * PB_REC, S.out.p, (size_t)cnt * J.n_adapters * PB_REC * 4,
                               cudaMemcpyDeviceToHost, stream));
        }
        return 0;
    };
    int rc_final = 0;
    std::string first_err;
    size_t k = 0, cur_job = (size_t)-1;
    AdapterPlan P;
    bool drained = false;
    while (!rc_final) {
        PackItem it;
        next_item(it);
        if (it.end) { drained = true; break; }
        if (it.rc) { rc_final = it.rc; first_err = it.err; drained = true; break; }     // planning error ends the planner's run too
        const CrossJob &J = jobs[it.job];
        if (it.job != cur_job) {
            // The adapter plan is made (or found in the 4-entry cache) right before the job's first chunk: a miss waits for the
            // device to go idle before it recycles an entry, so chunks of earlier jobs never lose their adapter copies.
            cur_job = it.job;
            P = AdapterPlan();
            rc_final = plan_adapters(E, E.st[k % NSTAGE].stream, J.adapters, J.ad_off, J.n_adapters, ma, mi, go, ge, P);
        }
        if (!rc_final) rc_final = submit(J, P, it, E.st[k % NSTAGE]);
        if (rc_final) first_err = g_err;
        ++k;
    }
    if (PK && !drained) {
        // an error on this side: stop the packer and take its remaining items so that it is idle (and its buffers free) again
        { std::lock_guard<std::mutex> lk(PK->mu); PK->abort = true; }
        PK->cv.notify_all();
        for (;;) {
            PackItem it;
            next_item(it);
            if (it.buf >= 0) { std::lock_guard<std::mutex> lk(PK->mu); PK->state[it.buf] = Packer::FREE; }
            PK->cv.notify_all();
            if (it.end || it.rc) break;
        }
    }
    // Whatever happened, nothing may still be writing into the caller's `out` (or reading `seqs`) when we return.
    for (int i = 0; i < NSTAGE; ++i) {
        if (!rc_final && E.st[i].misc.p) { rc_final = check_status(E.st[i], E.st[i].stream); if (rc_final) first_err = g_err; }
        cudaError_t e = cudaStreamSynchronize(E.st[i].stream);
        if (e != cudaSuccess && !rc_final) { rc_final = fail(PB200_ERR_CUDA, std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e)); first_err = g_err; }
    }
    E.last_pending = false;      // every stage waited for an earlier call's queued work and is now idle
    if (PK) {        // all uploads are complete: the pack buffers are free for the next submit
        std::lock_guard<std::mutex> lk(PK->mu);
        for (int i = 0; i < NPACK; ++i) PK->state[i] = Packer::FREE;
    }
    if (rc_final && !first_err.empty()) g_err = first_err;
    return rc_final;
}

int batch_host(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
               const int32_t *ad_off, int32_t n_adapters, const int32_t *pair_seq, const int32_t *pair_adapter,
               int64_t n_pairs, int ma, int mi, int go, int ge, int32_t *out) {
    if (n_seqs < 0 || n_adapters < 0 || n_pairs < 0) return fail(PB200_ERR_ARG, "negative count");
    if ((pair_seq == nullptr) != (pair_adapter == nullptr)) return fail(PB200_ERR_ARG, "pair_seq/pair_adapter must both be given or both NULL");
    const bool cross = pair_seq == nullptr;
    if (cross && n_pairs != n_seqs * (int64_t)n_adapters) return fail(PB200_ERR_ARG, "cross mode: n_pairs != n_seqs*n_adapters");
    if (n_pairs == 0) return 0;
    if (!seq_off || !ad_off || !out) return fail(PB200_ERR_ARG, "NULL pointer");
    load_env_options();
    std::vector<CrossJob> jobs(1);
    jobs[0] = CrossJob{seqs, seq_off, n_seqs, adapters, ad_off, n_adapters, out};
    if (int rc = validate_args(seqs, seq_off, n_seqs, adapters, ad_off, n_adapters, pair_seq, pair_adapter, n_pairs, cross)) return rc;
    if (cross)
        return with_engine(CallOn::stages, nullptr, [&](Engine &E, cudaStream_t) { return run_cross_jobs(E, jobs, ma, mi, go, ge); });

    // ---- pair-list mode: all sequences resident on st[0], pairs ordered per class on the host ----
    return sync_call(CallOn::stage0, nullptr, [&](Engine &E, cudaStream_t stream) -> int {
        AdapterPlan P;
        if (int rc = plan_adapters(E, stream, adapters, ad_off, n_adapters, ma, mi, go, ge, P)) return rc;
        NvtxRange submit_range("pb200:submit_pairs");
        Stage &S = E.st[0];
        const int64_t bytes = seq_off[n_seqs];
        if (int rc = S.seq_raw.ensure((size_t)bytes + 16)) return rc;
        if (int rc = S.seq_codes.ensure((size_t)bytes + 16)) return rc;
        if (int rc = S.seq_off.ensure((size_t)(n_seqs + 1) * 8)) return rc;
        if (int rc = S.out.ensure((size_t)n_pairs * PB_REC * 4)) return rc;
        if (int rc = S.pair_seq.ensure((size_t)n_pairs * 4)) return rc;
        if (int rc = S.pair_ad.ensure((size_t)n_pairs * 4)) return rc;
        if (int rc = S.order.ensure((size_t)n_pairs * 4)) return rc;
        if (int rc = reset_misc(S, stream)) return rc;
        if (bytes) CK(cudaMemcpyAsync(S.seq_raw.p, seqs, (size_t)bytes, cudaMemcpyHostToDevice, stream));
        CK(cudaMemcpyAsync(S.seq_off.p, seq_off, (size_t)(n_seqs + 1) * 8, cudaMemcpyHostToDevice, stream));
        CK(cudaMemcpyAsync(S.pair_seq.p, pair_seq, (size_t)n_pairs * 4, cudaMemcpyHostToDevice, stream));
        CK(cudaMemcpyAsync(S.pair_ad.p, pair_adapter, (size_t)n_pairs * 4, cudaMemcpyHostToDevice, stream));
        if (int rc = launch_encode(stream, S.seq_raw.as<uint8_t>(), S.seq_codes.as<uint8_t>(), bytes, E.sm_count)) return rc;
        // class of every adapter, then per-class ordering (adapter, length) so that slot halves have similar shapes
        std::vector<int> ad_class(n_adapters);
        for (int a = 0; a < n_adapters; ++a) ad_class[a] = class_of(P.si, ad_off[a + 1] - ad_off[a]);
        std::vector<std::vector<int32_t>> per_class(N_CLASSES);
        for (int64_t p = 0; p < n_pairs; ++p) per_class[ad_class[pair_adapter[p]]].push_back((int32_t)p);
        int *status = S.misc.as<int>();
        unsigned long long *counter = reinterpret_cast<unsigned long long *>(S.misc.as<char>() + 16);
        for (int c = 0; c < N_CLASSES; ++c) {
            auto &ord = per_class[c];
            if (ord.empty()) continue;
            int m_max = 0;
            int64_t max_n = 0;
            for (int32_t p : ord) {
                m_max = std::max(m_max, ad_off[pair_adapter[p] + 1] - ad_off[pair_adapter[p]]);
                max_n = std::max(max_n, seq_off[pair_seq[p] + 1] - seq_off[pair_seq[p]]);
            }
            if (max_n > 0x7fff0000ll) return fail(PB200_ERR_ARG, "sequence longer than 2^31");
            if (c == GENERIC_CLASS) {
                GenericBatch G{E, stream, S.seq_codes.as<uint8_t>(), P.d_ad_codes, P.sc, S.out.as<int32_t>()};
                for (int32_t p : ord) {
                    const int64_t s = pair_seq[p];
                    const int a = pair_adapter[p];
                    if (int rc = G.add(seq_off[s], (int32_t)(seq_off[s + 1] - seq_off[s]), ad_off[a + 1] - ad_off[a], ad_off[a], p))
                        return rc;
                }
                if (int rc = G.flush()) return rc;
                continue;
            }
            std::sort(ord.begin(), ord.end(), [&](int32_t x, int32_t y) {
                int ax = pair_adapter[x], ay = pair_adapter[y];
                if (ax != ay) return ax < ay;
                int64_t nx = seq_off[pair_seq[x] + 1] - seq_off[pair_seq[x]], ny = seq_off[pair_seq[y] + 1] - seq_off[pair_seq[y]];
                if (nx != ny) return nx < ny;
                return x < y;
            });
            const int64_t n_tasks = (int64_t)ord.size();
            if (int rc = S.tasks.ensure((size_t)n_tasks * sizeof(Task))) return rc;
            CK(cudaMemcpyAsync(S.order.p, ord.data(), (size_t)n_tasks * 4, cudaMemcpyHostToDevice, stream));
            CK(cudaStreamSynchronize(stream));  // ord is pageable and reused per class
            build_tasks_pairs_kernel<<<(unsigned)((n_tasks + 255) / 256), 256, 0, stream>>>(
                S.tasks.as<Task>(), n_tasks, S.order.as<int32_t>(), S.pair_seq.as<int32_t>(), S.pair_ad.as<int32_t>(),
                S.seq_off.as<int64_t>(), P.d_ad_off);
            g_launches++;
            CK(cudaGetLastError());
            TaskSrc ts;
            ts.tasks = S.tasks.as<Task>(); ts.n_tasks = n_tasks;
            ts.cls_ad = nullptr; ts.n_cls_ad = 0; ts.n_adapters = n_adapters; ts.n_seqs = n_seqs;
            ts.seq_off = S.seq_off.as<int64_t>(); ts.ad_off = P.d_ad_off; ts.seq_order = nullptr;
            if (int rc = run_class_tasks(E, S, stream, c, m_max, ts, max_n, S.seq_codes.as<uint8_t>(), P.d_ad_codes,
                                         P.sc, P.si, S.out.as<int32_t>(), status, counter)) return rc;
        }
        CK(cudaMemcpyAsync(out, S.out.p, (size_t)n_pairs * PB_REC * 4, cudaMemcpyDeviceToHost, stream));
        return check_status(S, stream);
    });
}

int batch_host_multi(const pb200_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    if (n_batches < 0 || (n_batches > 0 && !batches)) return fail(PB200_ERR_ARG, "bad batch list");
    load_env_options();
    std::vector<CrossJob> jobs;
    for (int b = 0; b < n_batches; ++b) {
        const pb200_batch_t &B = batches[b];
        if (B.n_seqs < 0 || B.n_adapters < 0) return fail(PB200_ERR_ARG, "negative count");
        if (B.n_seqs == 0 || B.n_adapters == 0) continue;
        if (!B.seq_off || !B.ad_off || !B.out) return fail(PB200_ERR_ARG, "NULL pointer");
        jobs.push_back(CrossJob{B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, B.out});
        if (int rc = validate_args(B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, nullptr, nullptr,
                                   B.n_seqs * (int64_t)B.n_adapters, true)) return rc;
    }
    if (jobs.empty()) return 0;
    return with_engine(CallOn::stages, nullptr, [&](Engine &E, cudaStream_t) { return run_cross_jobs(E, jobs, ma, mi, go, ge); });
}

// float("%f" % (100.0*c/l)) exactly as the reference chain produces it: std::to_string(double) = sprintf("%f")
// (porechop/src/alignment.cpp:113-121), then Python's float() = strtod (nanopore_read.py:488-489)
double printed_exact(double d) {
    char buf[512];                    // "%f" of any double up to 100.0 needs a few bytes; DBL_MAX would need 317
    snprintf(buf, sizeof buf, "%f", d);
    return strtod(buf, nullptr);
}
double percent_exact(int32_t c, int32_t l) {
    volatile double cd = (double)c, ld = (double)l;
    return printed_exact(100.0 * cd / ld);
}
// inclusive = false: the end-trim test (value > thr); true: the middle-hit test (value >= thr)
void threshold_table(double thr, int32_t len, bool inclusive, int32_t *cmin) {
    if (len > 0) cmin[0] = INT32_MAX;
    for (int32_t l = 1; l < len; ++l) {
        // percent_exact(., l) is non-decreasing: binary search for the first c that passes
        int32_t lo = 0, hi = l + 1;
        while (lo < hi) {
            const int32_t mid = lo + (hi - lo) / 2;
            const double v = percent_exact(mid, l);
            if (inclusive ? v >= thr : v > thr) hi = mid; else lo = mid + 1;
        }
        cmin[l] = lo;
    }
}

// threshold tables are pure functions of (threshold, length, test): built once, reused by every later call
std::shared_ptr<const std::vector<int32_t>> cached_threshold_table(double thr, int32_t len, bool inclusive = false) {
    static std::mutex mu;
    static std::map<std::tuple<double, int32_t, bool>, std::shared_ptr<const std::vector<int32_t>>> cache;
    std::lock_guard<std::mutex> lk(mu);
    const auto key = std::make_tuple(thr, len, inclusive);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    auto t = std::make_shared<std::vector<int32_t>>((size_t)len);
    threshold_table(thr, len, inclusive, t->data());
    if (cache.size() >= 64) cache.clear();                     // growth guard (thresholds are few in practice)
    cache[key] = t;
    return t;
}

// a side without adapters: nothing aligns, nothing is trimmed, and the ranking has no pairs
void fill_no_adapters(int32_t *trim, int32_t *top2, int64_t n_seqs) {
    memset(trim, 0, (size_t)n_seqs * 4);
    if (top2) for (int64_t s = 0; s < n_seqs; ++s) { int32_t *o = top2 + s * 6; o[0] = o[3] = -1; o[1] = o[4] = 0; o[2] = o[5] = 1; }
}

// The decision tables of decision job (or trim side) j: the end-trim threshold table and the score columns, on `stream`
int upload_decision_tables(Engine &E, int j, cudaStream_t stream, double thr, int32_t cmin_len, const int32_t *score_cols,
                           int32_t n_score_cols) {
    const auto table = cached_threshold_table(thr, cmin_len);
    if (int rc = E.dec_cmin[j].ensure((size_t)cmin_len * 4)) return rc;
    if (int rc = E.dec_cols[j].ensure((size_t)std::max<int32_t>(n_score_cols, 1) * 4)) return rc;
    CK(cudaMemcpyAsync(E.dec_cmin[j].p, table->data(), (size_t)cmin_len * 4, cudaMemcpyHostToDevice, stream));
    if (n_score_cols > 0) CK(cudaMemcpyAsync(E.dec_cols[j].p, score_cols, (size_t)n_score_cols * 4, cudaMemcpyHostToDevice, stream));
    return 0;
}

int batch_end_decisions(const pb200_end_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    if (n_batches < 0 || (n_batches > 0 && !batches)) return fail(PB200_ERR_ARG, "bad batch list");
    load_env_options();
    std::vector<CrossJob> jobs;
    for (int b = 0; b < n_batches; ++b) {
        const pb200_end_batch_t &D = batches[b];
        const pb200_batch_t &B = D.batch;
        if (B.n_seqs < 0 || B.n_adapters < 0 || D.n_score_cols < 0) return fail(PB200_ERR_ARG, "negative count");
        if (B.n_seqs == 0) continue;
        if (!D.trim || (D.n_score_cols > 0 && ((!D.score_pairs && !D.top2) || !D.score_cols))) return fail(PB200_ERR_ARG, "NULL pointer");
        if (!(D.end_threshold >= 0.0)) return fail(PB200_ERR_ARG, "end_threshold must be >= 0 for the device decisions");
        for (int32_t k = 0; k < D.n_score_cols; ++k)
            if (D.score_cols[k] < 0 || D.score_cols[k] >= B.n_adapters) return fail(PB200_ERR_ARG, "score column out of range");
        if (B.n_adapters == 0) {
            fill_no_adapters(D.trim, D.top2, B.n_seqs);
            continue;
        }
        if (!B.seq_off || !B.ad_off) return fail(PB200_ERR_ARG, "NULL pointer");
        CrossJob J{B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, B.out};
        if (int rc = validate_args(B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, nullptr, nullptr,
                                   B.n_seqs * (int64_t)B.n_adapters, true)) return rc;
        // a window is seq[:end_size] / seq[-end_size:] (nanopore_read.py:172,194) and the aligned region is at most
        // window + adapter columns long: that sizes the threshold table (windows are checked chunk by chunk)
        if (D.end_size < 0) return fail(PB200_ERR_ARG, "negative end_size");
        int64_t m_max = 0;
        for (int32_t a = 0; a < B.n_adapters; ++a) m_max = std::max<int64_t>(m_max, B.ad_off[a + 1] - B.ad_off[a]);
        if ((int64_t)D.end_size + m_max + 2 > 65535) return fail(PB200_ERR_ARG, "windows too long for the device decisions (use the record API)");
        if (D.top2 && ((int64_t)D.end_size + m_max + 2 > 4095 || D.n_score_cols >= 0xFFFF))
            return fail(PB200_ERR_ARG, "windows too long / too many score columns for the device barcode ranking (use score_pairs)");
        J.dec = &D;
        J.max_seq_len = D.end_size;
        J.cmin_len = (int32_t)(D.end_size + m_max + 2);
        jobs.push_back(std::move(J));
    }
    if (jobs.empty()) return 0;
    if ((int)jobs.size() > Engine::MAX_DEC_JOBS) return fail(PB200_ERR_ARG, "too many decision batches in one call");
    return with_engine(CallOn::stages, nullptr, [&](Engine &E, cudaStream_t s0) -> int {
        for (size_t j = 0; j < jobs.size(); ++j) {
            const pb200_end_batch_t &D = *jobs[j].dec;
            if (int rc = upload_decision_tables(E, (int)j, s0, D.end_threshold, jobs[j].cmin_len, D.score_cols, D.n_score_cols))
                return rc;
            jobs[j].d_cmin = E.dec_cmin[j].as<int32_t>();
            jobs[j].d_cols = E.dec_cols[j].as<int32_t>();
        }
        CK(cudaStreamSynchronize(s0));           // tables are in place before any stage's stream uses them
        return run_cross_jobs(E, jobs, ma, mi, go, ge);
    });
}

// Phase A on the device: every batch's records are max-reduced per adapter column (search_best_kernel) on the stage that made
// them, into that stage's own accumulator slice; after the final drain the host takes the maximum over the slices and turns
// the key back into float("%f" % d).
int batch_search(const pb200_search_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    if (n_batches < 0 || (n_batches > 0 && !batches)) return fail(PB200_ERR_ARG, "bad batch list");
    load_env_options();
    std::vector<CrossJob> jobs;
    std::vector<double *> bests;
    int64_t cols = 0;
    for (int b = 0; b < n_batches; ++b) {
        const pb200_batch_t &B = batches[b].batch;
        if (B.n_seqs < 0 || B.n_adapters < 0) return fail(PB200_ERR_ARG, "negative count");
        if (B.n_adapters == 0) continue;
        double *best = batches[b].best;
        if (!best) return fail(PB200_ERR_ARG, "NULL pointer");
        if (B.n_seqs == 0) continue;
        if (!B.seq_off || !B.ad_off) return fail(PB200_ERR_ARG, "NULL pointer");
        if (int rc = validate_args(B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, nullptr, nullptr,
                                   B.n_seqs * (int64_t)B.n_adapters, true)) return rc;
        CrossJob J{B.seqs, B.seq_off, B.n_seqs, B.adapters, B.ad_off, B.n_adapters, B.out};
        J.search_col = cols;
        cols += B.n_adapters;
        jobs.push_back(std::move(J));
        bests.push_back(best);
    }
    // every batch that has adapters starts from the reference's 0.0 (a batch without sequences keeps it)
    for (int b = 0; b < n_batches; ++b)
        if (batches[b].batch.n_adapters > 0) std::fill(batches[b].best, batches[b].best + batches[b].batch.n_adapters, 0.0);
    if (jobs.empty()) return 0;
    return with_engine(CallOn::stages, nullptr, [&](Engine &E, cudaStream_t s0) -> int {
        if (int rc = E.search_acc.ensure((size_t)NSTAGE * cols * 8)) return rc;
        E.search_cols = cols;
        for (int i = 0; i < NSTAGE; ++i)         // each slice is zeroed on the stream of the only stage that reduces into it
            CK(cudaMemsetAsync(E.search_acc.as<unsigned long long>() + (size_t)i * cols, 0, (size_t)cols * 8, E.st[i].stream));
        if (int rc = run_cross_jobs(E, jobs, ma, mi, go, ge)) return rc;
        // run_cross_jobs drained every stage: the slices are final
        std::vector<unsigned long long> keys((size_t)NSTAGE * cols);
        CK(cudaMemcpyAsync(keys.data(), E.search_acc.p, keys.size() * 8, cudaMemcpyDeviceToHost, s0));
        CK(cudaStreamSynchronize(s0));
        for (size_t j = 0; j < jobs.size(); ++j) {
            for (int32_t a = 0; a < jobs[j].n_adapters; ++a) {
                unsigned long long k = 0;
                for (int i = 0; i < NSTAGE; ++i) k = std::max(k, keys[(size_t)i * cols + jobs[j].search_col + a]);
                double d;
                memcpy(&d, &k, sizeof d);
                bests[j][a] = printed_exact(d);
            }
        }
        return 0;
    });
}

// longest sequence of a device-resident batch, measured when *max_len < 0 (unknown); S.misc must hold 64 bytes
int device_max_len(Stage &S, cudaStream_t stream, const int64_t *d_seq_off, int64_t n_seqs, int64_t *max_len) {
    if (*max_len < 0) {
        unsigned long long *d_max = reinterpret_cast<unsigned long long *>(S.misc.as<char>() + 32);
        CK(cudaMemsetAsync(d_max, 0, 8, stream));
        int64_t blocks = std::min<int64_t>((n_seqs + 255) / 256, 1024);
        max_len_kernel<<<(unsigned)blocks, 256, 0, stream>>>(d_seq_off, n_seqs, d_max);
        g_launches++;
        CK(cudaGetLastError());
        unsigned long long h = 0;
        CK(cudaMemcpyAsync(&h, d_max, 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        *max_len = (int64_t)h;
    }
    return *max_len > 0x7fff0000ll ? fail(PB200_ERR_ARG, "sequence longer than 2^31") : 0;
}

int batch_device_queue(Engine &E, cudaStream_t stream, const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs,
                       int64_t total_seq_bytes, int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off,
                       int32_t n_adapters, int ma, int mi, int go, int ge, int32_t *d_out) {
    Stage &S = E.st[0];
    NvtxRange submit_range("pb200:submit_device");
    AdapterPlan P;
    if (int rc = plan_adapters(E, stream, adapters, ad_off, n_adapters, ma, mi, go, ge, P)) return rc;
    if (int rc = reset_misc(S, stream)) return rc;
    if (int rc = device_max_len(S, stream, d_seq_off, n_seqs, &max_seq_len)) return rc;
    const bool ascii = single_pass_ascii(P, max_seq_len);
    const uint8_t *seqs = d_seqs;
    if (!ascii) {
        if (int rc = S.seq_codes.ensure((size_t)total_seq_bytes + 16)) return rc;
        if (int rc = launch_encode(stream, d_seqs, S.seq_codes.as<uint8_t>(), total_seq_bytes, E.sm_count)) return rc;
        seqs = S.seq_codes.as<uint8_t>();
    }
    std::vector<int64_t> h_off;   // only fetched when a generic class exists
    for (auto &c : P.classes) if (c.cls == GENERIC_CLASS) {
        h_off.resize((size_t)n_seqs + 1);
        CK(cudaMemcpyAsync(h_off.data(), d_seq_off, (size_t)(n_seqs + 1) * 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        break;
    }
    int64_t max_cnt = std::max<int64_t>(1, g_opt.device_chunk_tasks / std::max<int32_t>(n_adapters, 1));
    for (int64_t s0 = 0; s0 < n_seqs; s0 += max_cnt) {
        const int64_t cnt = std::min(max_cnt, n_seqs - s0);
        if (int rc = run_cross_chunk(E, S, stream, P, seqs, d_seq_off + s0, cnt, 0, max_seq_len,
                                     n_adapters, d_out + (size_t)s0 * n_adapters * PB_REC,
                                     h_off.empty() ? nullptr : h_off.data(), s0, ad_off, nullptr, ascii)) return rc;
    }
#ifdef PB_TEST_DEFERRED_STATUS
    // tests of the host-simulated engine only (through PB200_SIM_FLAGS): the call's last operation sets the status word's
    // "window bound violated" bit, as a trace kernel does when a traceback leaves its window, so that the deferred-error
    // path of the device-resident API can be tested
    CK(cudaMemsetAsync(S.misc.p, 1, 1, stream));
#endif
    return 0;
}

int batch_device(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                 int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters, int ma, int mi,
                 int go, int ge, int32_t *d_out, void *user_stream) {
    if (n_seqs < 0 || n_adapters < 0 || total_seq_bytes < 0) return fail(PB200_ERR_ARG, "negative count");
    if (n_seqs == 0 || n_adapters == 0) return 0;
    if (!d_seq_off || !ad_off || !d_out) return fail(PB200_ERR_ARG, "NULL pointer");
    return with_engine(CallOn::library, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        // the work is queued on `stream` and the call returns without waiting for it: whatever happens below, the next call
        // must wait for what was queued
        const int rc = batch_device_queue(E, stream, d_seqs, d_seq_off, n_seqs, total_seq_bytes, max_seq_len, adapters, ad_off,
                                          n_adapters, ma, mi, go, ge, d_out);
        const std::string first_err = g_err;
        const int rc_last = record_last(E, stream);
        if (rc) { g_err = first_err; return rc; }
        return rc_last;
    });
}

// ---- middle-adapter scan (adapterMiddleScan, Phase C) ------------------------------------------------------------
// Host-side checks that make the device loop exact and finite (include/porechop_b200.h): threshold > 0, adapters of A/C/G/T/U
// only, every adapter in an int16 class with a finite window bound.  cmin_len = W(m_max) + 2 covers every len_ad a traced
// path (score >= 0) can have.
int middle_preconditions(const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters, int ma, int mi, int go, int ge,
                         double thr, int32_t *cmin_len) {
    if (!(thr > 0.0)) return fail(PB200_ERR_ARG, "middle_threshold must be > 0 for the device middle scan");
    const SchemeInfo si = scheme_info(ma, mi, go, ge);
    if (!si.bounded) return fail(PB200_ERR_ARG, "the device middle scan needs negative gap scores (a finite window bound)");
    int64_t m_max = 0;
    for (int32_t a = 0; a < n_adapters; ++a) {
        const int32_t m = ad_off[a + 1] - ad_off[a];
        if (class_of(si, m) == GENERIC_CLASS) return fail(PB200_ERR_ARG, "adapter or scheme outside the int16 kernels");
        for (int32_t k = ad_off[a]; k < ad_off[a + 1]; ++k)
            if (!strchr("ACGTUacgtu", adapters[k]) || adapters[k] == 0)
                return fail(PB200_ERR_ARG, "the device middle scan takes adapters of A/C/G/T/U only");
        m_max = std::max<int64_t>(m_max, m);
    }
    *cmin_len = (int32_t)(m_max + (m_max * si.wnum) / si.wden + 2);
    return 0;
}

// the hits of one round of one segment, as they came back: read (segment-relative) and {adapter, record} per append position
struct MiddleRound { int64_t s0; std::vector<int32_t> reads, hits; };

size_t device_free_bytes() {
#if defined(__CUDACC__)
    size_t f = 0, t = 0;
    if (cudaMemGetInfo(&f, &t) != cudaSuccess) { cudaGetLastError(); return 1ull << 30; }
    return f;
#else
    return 4ull << 30;     // host builds of these sources have no device-memory query
#endif
}

// The reads [a, b) of the next segment: its resident buffers take at most half of the free device memory (plus what the
// engine already holds for them) and n * n_adapters stays below 2^31 (records are indexed with int32 out_idx).
// h_seq_off: host offsets when the segment's codes are part of its resident buffers (host API), else nullptr.
// extra_per_read / byte_weight / extra_held: what a caller keeps resident next to the scan's buffers (adapterTrimReads: the
// end windows per read, the ASCII reads next to their codes, and the buffers it already holds for them).
int64_t middle_segment_end(const Engine &E, int64_t a, int64_t n_seqs, int32_t n_adapters, const int64_t *h_seq_off,
                           double extra_per_read = 0, double byte_weight = 1, size_t extra_held = 0) {
    const size_t held = E.mid_codes.cap + E.mid_off.cap + E.mid_rec.cap + E.mid_next_ad.cap + E.mid_hits.cap +
                        E.mid_active[0].cap + E.mid_active[1].cap + extra_held;
    const double budget = (double)(device_free_bytes() + held) / 2;
    // per read: offset, records, next adapter, hit slot, two active-list entries, the two-pass task and end-cell records
    const double per_read = 8 + (double)n_adapters * (PB_REC * 4 + sizeof(Task) + 16) + 4 + PB_HIT_INTS * 4 + 8 + extra_per_read;
    const int64_t max_reads = std::max<int64_t>(1, std::min<int64_t>(0x7fffffffll / std::max<int32_t>(n_adapters, 1),
                                                                     (int64_t)(budget / per_read)));
    int64_t b = std::min(n_seqs, a + max_reads);
    if (h_seq_off)
        while (b > a + 1 && byte_weight * (double)(h_seq_off[b] - h_seq_off[a]) + (double)(b - a) * per_read > budget)
            b = a + (b - a) / 2;
    return b;
}

int middle_segment_buffers(Engine &E, int64_t n, int32_t n_adapters, size_t code_bytes, MiddleSeg &M) {
    if (code_bytes) {
        if (int rc = E.mid_codes.ensure(code_bytes + 16)) return rc;
        M.codes = E.mid_codes.as<uint8_t>();
    }
    if (int rc = E.mid_off.ensure((size_t)(n + 1) * 8)) return rc;
    if (int rc = E.mid_rec.ensure((size_t)n * n_adapters * PB_REC * 4)) return rc;
    if (int rc = E.mid_next_ad.ensure((size_t)n * 4)) return rc;
    if (int rc = E.mid_hits.ensure((size_t)n * PB_HIT_INTS * 4)) return rc;
    if (int rc = E.mid_active[0].ensure((size_t)n * 4)) return rc;
    if (int rc = E.mid_active[1].ensure((size_t)n * 4)) return rc;
    if (int rc = E.mid_ctr.ensure(64)) return rc;
    M.n = n;
    M.rec = E.mid_rec.as<int32_t>(); M.next_ad = E.mid_next_ad.as<int32_t>(); M.hits = E.mid_hits.as<int32_t>();
    M.active[0] = E.mid_active[0].as<int32_t>(); M.active[1] = E.mid_active[1].as<int32_t>();
    M.count = E.mid_ctr.as<unsigned>();
    M.max_len_d = reinterpret_cast<unsigned long long *>(E.mid_ctr.as<char>() + 8);
    M.cmin = E.mid_cmin.as<int32_t>();
    return 0;
}

// Rounds >= 1 of a segment whose round 0 (DP over every read + middle_decide_kernel) has been enqueued on `stream` (or has
// completed on other streams): each round reads back its hit count and longest active read, copies the round's hits home,
// and runs the DP over the active reads only (slot i = read active[i]: records land in each read's own slots, nothing is
// copied or re-encoded) followed by the next middle_decide_kernel.
int middle_rounds(Engine &E, Stage &S, cudaStream_t stream, const AdapterPlan &P, MiddleSeg &M, int32_t n_adapters,
                  const int32_t *h_ad_off, int64_t s0, std::vector<MiddleRound> &out) {
    int cur = 0;                      // round 0 appended to active[0]
    for (int64_t round = 1;; ++round) {
        unsigned c = 0;
        unsigned long long mx = 0;
        CK(cudaMemcpyAsync(&c, M.count, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&mx, M.max_len_d, 8, cudaMemcpyDeviceToHost, stream));
        if (int rc = check_status(S, stream)) return rc;
        if (c == 0) return 0;
        out.push_back(MiddleRound{s0, std::vector<int32_t>(c), std::vector<int32_t>((size_t)c * PB_HIT_INTS)});
        CK(cudaMemcpyAsync(out.back().reads.data(), M.active[cur], (size_t)c * 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(out.back().hits.data(), M.hits, (size_t)c * PB_HIT_INTS * 4, cudaMemcpyDeviceToHost, stream));
        // every hit masks at least one base that was not masked before (include/porechop_b200.h): a read has at most
        // max_len hits, so more rounds than that mean a broken invariant, not a long input
        if (round > M.max_len) return fail(PB200_ERR_INTERNAL, "middle scan: more rounds than the longest sequence has bases");
        CK(cudaMemsetAsync(E.mid_ctr.p, 0, 16, stream));
        if (int rc = run_cross_chunk(E, S, stream, P, M.codes, M.off, (int64_t)c, 0, (int64_t)mx, n_adapters, M.rec, nullptr, 0,
                                     h_ad_off, M.active[cur])) return rc;
        if (int rc = launch_middle_decide(E, stream, M, n_adapters, M.active[cur], 0, (int64_t)c, M.active[cur ^ 1],
                                          S.misc.as<int>())) return rc;
        cur ^= 1;
    }
}

// hits of every round of every segment -> n_hits / hits, sequence-major, each sequence's hits in round order
int middle_emit(const std::vector<MiddleRound> &rounds, int64_t n_seqs, int32_t *n_hits, int32_t *hits, int64_t hits_cap,
                int64_t *n_total) {
    if (n_seqs > 0) memset(n_hits, 0, (size_t)n_seqs * 4);
    int64_t total = 0;
    for (const MiddleRound &R : rounds) {
        for (int32_t s : R.reads) n_hits[R.s0 + s]++;
        total += (int64_t)R.reads.size();
    }
    *n_total = total;
    if (total > hits_cap) return fail(PB200_ERR_SPACE, "hits_cap is smaller than the number of hits (*n_total)");
    std::vector<int64_t> at((size_t)n_seqs + 1, 0);
    for (int64_t s = 0; s < n_seqs; ++s) at[s + 1] = at[s] + n_hits[s];
    for (const MiddleRound &R : rounds)
        for (size_t p = 0; p < R.reads.size(); ++p)
            memcpy(hits + (size_t)(at[R.s0 + R.reads[p]]++) * PB_HIT_INTS, R.hits.data() + p * PB_HIT_INTS, PB_HIT_INTS * 4);
    return 0;
}

int middle_table(Engine &E, cudaStream_t stream, double thr, int32_t cmin_len) {
    const auto table = cached_threshold_table(thr, cmin_len, true);
    if (int rc = E.mid_cmin.ensure((size_t)cmin_len * 4)) return rc;
    CK(cudaMemcpyAsync(E.mid_cmin.p, table->data(), (size_t)cmin_len * 4, cudaMemcpyHostToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    return 0;
}

// Host reads: the buffer and the offsets checked, *max_len the longest read.
int host_max_len(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, int64_t *max_len) {
    if (int rc = validate_args(seqs, seq_off, n_seqs, nullptr, nullptr, 0, nullptr, nullptr, 0, true)) return rc;
    *max_len = 0;
    for (int64_t s = 0; s < n_seqs; ++s) {
        const int64_t len = seq_off[s + 1] - seq_off[s];
        if (len < 0) return fail(PB200_ERR_ARG, "sequence offsets not monotone");
        *max_len = std::max(*max_len, len);
    }
    return *max_len > 0x7fff0000ll ? fail(PB200_ERR_ARG, "sequence longer than 2^31") : 0;
}

// Phase C of a segment whose reads are resident as codes (M.codes, M.off, longest M.max_len): round 0 over every read, chunk by
// chunk, each chunk's DP followed by middle_decide_kernel from adapter 0; then the masking rounds.
int middle_scan_resident(Engine &E, Stage &S, cudaStream_t stream, const AdapterPlan &P, MiddleSeg &M, int32_t n_adapters,
                         const int32_t *h_ad_off, int64_t s0, std::vector<MiddleRound> &rounds) {
    CK(cudaMemsetAsync(E.mid_ctr.p, 0, 16, stream));
    const int64_t max_cnt = std::max<int64_t>(1, g_opt.device_chunk_tasks / n_adapters);
    for (int64_t c0 = 0; c0 < M.n; c0 += max_cnt) {
        const int64_t cnt = std::min(max_cnt, M.n - c0);
        if (int rc = run_cross_chunk(E, S, stream, P, M.codes, M.off + c0, cnt, 0, M.max_len, n_adapters,
                                     M.rec + (size_t)c0 * n_adapters * PB_REC, nullptr, 0, h_ad_off)) return rc;
        if (int rc = launch_middle_decide(E, stream, M, n_adapters, nullptr, c0, cnt, M.active[0], S.misc.as<int>())) return rc;
    }
    return middle_rounds(E, S, stream, P, M, n_adapters, h_ad_off, s0, rounds);
}

// Entry checks of a middle scan (adapterMiddleScan*, and the middle adapters of adapterTrimReads*): the counts, the output
// pointers, the adapters and the scan's preconditions; *cmin_len: the length of its threshold table.  The reads are the
// caller's to check.
int middle_entry_checks(int64_t n_seqs, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters, int ma, int mi,
                        int go, int ge, double thr, const int32_t *n_hits, const int32_t *hits, int64_t hits_cap,
                        const int64_t *n_total, int32_t *cmin_len) {
    if (n_seqs < 0 || n_adapters < 0 || hits_cap < 0) return fail(PB200_ERR_ARG, "negative count");
    if (!n_total || (n_seqs > 0 && !n_hits) || (hits_cap > 0 && !hits) || (n_adapters > 0 && !ad_off))
        return fail(PB200_ERR_ARG, "NULL pointer");
    *cmin_len = 0;
    if (n_adapters == 0) return thr > 0.0 ? 0 : fail(PB200_ERR_ARG, "middle_threshold must be > 0 for the device middle scan");
    if (int rc = validate_args(nullptr, nullptr, 0, adapters, ad_off, n_adapters, nullptr, nullptr, 0, true)) return rc;
    return middle_preconditions(adapters, ad_off, n_adapters, ma, mi, go, ge, thr, cmin_len);
}

int middle_host(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters, const int32_t *ad_off,
                int32_t n_adapters, int ma, int mi, int go, int ge, double thr, int32_t *n_hits, int32_t *hits,
                int64_t hits_cap, int64_t *n_total) {
    load_env_options();
    int32_t cmin_len = 0;
    if (int rc = middle_entry_checks(n_seqs, adapters, ad_off, n_adapters, ma, mi, go, ge, thr, n_hits, hits, hits_cap, n_total,
                                     &cmin_len)) return rc;
    if (n_seqs > 0 && !seq_off) return fail(PB200_ERR_ARG, "NULL pointer");
    if (n_seqs == 0 || n_adapters == 0) return middle_emit({}, n_seqs, n_hits, hits, hits_cap, n_total);
    int64_t max_len = 0;
    if (int rc = host_max_len(seqs, seq_off, n_seqs, &max_len)) return rc;
    std::vector<MiddleRound> rounds;
    const int rc = sync_call(CallOn::stages, nullptr, [&](Engine &E, cudaStream_t stream) -> int {
        NvtxRange submit_range("pb200:submit_middle");
        Stage &S = E.st[0];
        if (int rc = middle_table(E, stream, thr, cmin_len)) return rc;
        for (int64_t a = 0; a < n_seqs;) {
            const int64_t b = middle_segment_end(E, a, n_seqs, n_adapters, seq_off);
            MiddleSeg M;
            if (int rc = middle_segment_buffers(E, b - a, n_adapters, (size_t)(seq_off[b] - seq_off[a]), M)) return rc;
            M.off = E.mid_off.as<int64_t>();
            M.cmin_len = cmin_len;
            M.max_len = max_len;
            CK(cudaMemsetAsync(E.mid_ctr.p, 0, 16, stream));
            CK(cudaStreamSynchronize(stream));
            // round 0: the chunk pipeline of every other host-buffer call, into the segment's resident buffers
            std::vector<CrossJob> jobs(1);
            jobs[0] = CrossJob{seqs, seq_off + a, b - a, adapters, ad_off, n_adapters, nullptr};
            jobs[0].mid = &M;
            if (int rc = run_cross_jobs(E, jobs, ma, mi, go, ge)) return rc;
            AdapterPlan P;
            if (int rc = plan_adapters(E, stream, adapters, ad_off, n_adapters, ma, mi, go, ge, P)) return rc;
            if (int rc = middle_rounds(E, S, stream, P, M, n_adapters, ad_off, a, rounds)) return rc;
            a = b;
        }
        return 0;
    });
    if (rc) return rc;
    return middle_emit(rounds, n_seqs, n_hits, hits, hits_cap, n_total);
}

int middle_device(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                  int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters, int ma, int mi,
                  int go, int ge, double thr, int32_t *n_hits, int32_t *hits, int64_t hits_cap, int64_t *n_total,
                  void *user_stream) {
    if (total_seq_bytes < 0) return fail(PB200_ERR_ARG, "negative count");
    load_env_options();
    int32_t cmin_len = 0;
    if (int rc = middle_entry_checks(n_seqs, adapters, ad_off, n_adapters, ma, mi, go, ge, thr, n_hits, hits, hits_cap, n_total,
                                     &cmin_len)) return rc;
    if (n_seqs > 0 && !d_seq_off) return fail(PB200_ERR_ARG, "NULL pointer");
    if (n_seqs == 0 || n_adapters == 0) return middle_emit({}, n_seqs, n_hits, hits, hits_cap, n_total);
    std::vector<MiddleRound> rounds;
    const int rc = sync_call(CallOn::library, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        NvtxRange submit_range("pb200:submit_middle");
        Stage &S = E.st[0];
        if (!S.misc.p) {
            if (int rc = S.misc.ensure(64)) return rc;
            CK(cudaMemsetAsync(S.misc.p, 0, 64, stream));
        }
        if (int rc = check_status(S, stream)) return rc;     // a deferred error of an earlier device-resident call
        AdapterPlan P;
        if (int rc = plan_adapters(E, stream, adapters, ad_off, n_adapters, ma, mi, go, ge, P)) return rc;
        if (int rc = device_max_len(S, stream, d_seq_off, n_seqs, &max_seq_len)) return rc;
        if (int rc = middle_table(E, stream, thr, cmin_len)) return rc;
        // the library's encoded copy of the caller's sequences is what the rounds mask
        if (int rc = E.mid_codes.ensure((size_t)total_seq_bytes + 16)) return rc;
        if (int rc = launch_encode(stream, d_seqs, E.mid_codes.as<uint8_t>(), total_seq_bytes, E.sm_count)) return rc;
        for (int64_t a = 0; a < n_seqs;) {
            const int64_t b = middle_segment_end(E, a, n_seqs, n_adapters, nullptr);
            MiddleSeg M;
            if (int rc = middle_segment_buffers(E, b - a, n_adapters, 0, M)) return rc;
            M.codes = E.mid_codes.as<uint8_t>();
            M.off = const_cast<int64_t *>(d_seq_off + a);          // read only: offsets are written by the host-buffer path only
            M.cmin_len = cmin_len;
            M.max_len = max_seq_len;
            if (int rc = middle_scan_resident(E, S, stream, P, M, n_adapters, ad_off, a, rounds)) return rc;
            a = b;
        }
        return 0;
    });
    if (rc) return rc;
    return middle_emit(rounds, n_seqs, n_hits, hits, hits_cap, n_total);
}

// ---- whole-read trimming (adapterTrimReads, Phase B + Phase C) ---------------------------------------------------------
// Lengths in x[1 .. n] (x[0] = 0) -> their exclusive offsets in x[0 .. n], in place on `stream`.
int scan_offsets(Engine &E, cudaStream_t stream, int64_t *x, int64_t n) {
    if (n <= 0) return 0;
    const int64_t tiles = (n + PB_SCAN_TILE - 1) / PB_SCAN_TILE;
    if (int rc = E.trim_scan.ensure((size_t)tiles * 8)) return rc;
    int64_t *sums = E.trim_scan.as<int64_t>();
    scan_tiles_kernel<<<(unsigned)tiles, PB_SCAN_THREADS, 0, stream>>>(static_cast<const int64_t *>(x + 1), n, sums);
    scan_tile_sums_kernel<<<1, PB_SCAN_THREADS, 0, stream>>>(sums, tiles);
    scan_apply_kernel<<<(unsigned)tiles, PB_SCAN_THREADS, 0, stream>>>(x + 1, n, static_cast<const int64_t *>(sums));
    g_launches += 3;
    CK(cudaGetLastError());
    return 0;
}

// One side of Phase B: preconditions (those of adapterEndDecisions plus int16 classes with a finite window bound) and the
// threshold table's length.  rank: the demux stage ranks the score columns on the device (top2 may then be NULL).
int trim_side_check(const pb200_trim_side_t &T, int64_t n_seqs, int32_t end_size, const SchemeInfo &si, int32_t *cmin_len,
                    bool rank = false) {
    if (T.n_adapters < 0 || T.n_score_cols < 0) return fail(PB200_ERR_ARG, "negative count");
    if (n_seqs > 0 && !T.trim) return fail(PB200_ERR_ARG, "NULL pointer");
    if (T.n_score_cols > 0 && ((!T.score_pairs && !T.top2 && !rank) || !T.score_cols)) return fail(PB200_ERR_ARG, "NULL pointer");
    for (int32_t k = 0; k < T.n_score_cols; ++k)
        if (T.score_cols[k] < 0 || T.score_cols[k] >= T.n_adapters) return fail(PB200_ERR_ARG, "score column out of range");
    *cmin_len = 0;
    if (T.n_adapters == 0) return 0;
    if (!T.ad_off) return fail(PB200_ERR_ARG, "NULL pointer");
    if (int rc = validate_args(nullptr, nullptr, 0, T.adapters, T.ad_off, T.n_adapters, nullptr, nullptr, 0, true)) return rc;
    if (!si.bounded) return fail(PB200_ERR_ARG, "whole-read trimming needs negative gap scores (a finite window bound)");
    int64_t m_max = 0;
    for (int32_t a = 0; a < T.n_adapters; ++a) {
        const int32_t m = T.ad_off[a + 1] - T.ad_off[a];
        if (class_of(si, m) == GENERIC_CLASS) return fail(PB200_ERR_ARG, "adapter or scheme outside the int16 kernels");
        m_max = std::max<int64_t>(m_max, m);
    }
    if ((int64_t)end_size + m_max + 2 > 65535) return fail(PB200_ERR_ARG, "windows too long for the device decisions");
    if ((T.top2 || (rank && T.n_score_cols > 0)) && ((int64_t)end_size + m_max + 2 > 4095 || T.n_score_cols >= 0xFFFF))
        return fail(PB200_ERR_ARG, "windows too long / too many score columns for the device barcode ranking");
    *cmin_len = (int32_t)(end_size + m_max + 2);
    return 0;
}

// The reads [a, b) of the next segment: the middle scan's budget (middle_segment_end) with, per read, the two end windows (and
// their codes when they are encoded), window offsets, two trims, the trimmed range's first base and -- host API -- the
// segment's ASCII reads and offsets next to their codes.
// split: the output stage's buffers too (hit row, records and bases per read, the source offset of up to two records per read);
// demux: the two sides' top-2 rankings.
int64_t trim_segment_end(const Engine &E, int64_t a, int64_t n_seqs, int32_t n_mid, int64_t wl_max, const int64_t *h_seq_off,
                         bool split = false, bool demux = false) {
    size_t held = E.trim_reads.cap + E.trim_off.cap + E.trim_win_off.cap + E.trim_win[0].cap + E.trim_win[1].cap +
                  E.trim_d[0].cap + E.trim_d[1].cap + E.trim_first.cap;
    if (split) held += E.split_hit_of.cap + E.split_cnt.cap + E.split_bytes.cap + E.split_src.cap;
    if (demux) held += E.demux_top2[0].cap + E.demux_top2[1].cap;
    int64_t b = middle_segment_end(E, a, n_seqs, n_mid, h_seq_off,
                                   3.0 * (double)wl_max + 40 + (split ? 44.0 : 0.0) + (demux ? 48.0 : 0.0),
                                   h_seq_off ? 2.0 : 1.0, held);
#ifdef PB_TEST_SEGMENT_READS
    // tests of the host-simulated engine only (through sim_engine.load): small segments, so that a few reads span several
    b = std::min<int64_t>(b, a + PB_TEST_SEGMENT_READS);
#endif
    return b;
}

// Output stage of adapterTrimSplitReadsDevice: the running totals over the segments, and whether the records still fit parts_cap
// (once they do not, the stage only counts).
struct SplitTotals { int64_t parts = 0, bases = 0; bool write = true; };

// Demux stage of adapterDemuxReadsDevice: the shape of the score table (tab_c match counts x tab_l lengths; 0 x 0 without
// barcode columns).
struct DemuxStage {
    int32_t tab_c = 0, tab_l = 0;
};

// tab[c * l_n + l] = percent_exact(c, max(l, 1)) for c < c_n, l < l_n: the barcode scores of the top-2 pairs (match_ad, len_ad),
// the doubles Top2Scores.ranked() gives them.  A pure function of the shape: built once, reused by every later call.
std::shared_ptr<const std::vector<double>> cached_score_table(int32_t c_n, int32_t l_n) {
    static std::mutex mu;
    static std::map<std::pair<int32_t, int32_t>, std::shared_ptr<const std::vector<double>>> cache;
    std::lock_guard<std::mutex> lk(mu);
    const auto key = std::make_pair(c_n, l_n);
    auto it = cache.find(key);
    if (it != cache.end()) return it->second;
    auto t = std::make_shared<std::vector<double>>((size_t)c_n * (size_t)l_n);
    for (int32_t c = 0; c < c_n; ++c)
        for (int32_t l = 0; l < l_n; ++l) (*t)[(size_t)c * l_n + l] = percent_exact(c, std::max<int32_t>(l, 1));
    if (cache.size() >= 16) cache.clear();                     // growth guard (window shapes are few in practice)
    cache[key] = t;
    return t;
}

// b grown to at least `bytes` with its first `keep` bytes kept (copied on `stream`): the call-wide record arrays of the demux
// stage, which grow segment by segment
int grow_keep(DevBuf &b, size_t bytes, size_t keep, cudaStream_t stream) {
    if (bytes <= b.cap) return 0;
    DevBuf g;
    if (int rc = g.ensure(bytes)) return rc;
    if (keep) CK(cudaMemcpyAsync(g.p, b.p, keep, cudaMemcpyDeviceToDevice, stream));
    CK(cudaStreamSynchronize(stream));
    if (b.p) cudaFree(b.p);
    b.p = g.p;
    b.cap = g.cap;
    return 0;
}

// One segment's records [a, a + n): reads at reads[off[s] ..], trimmed ranges first[s] / toff (scanned lengths) on the device;
// the segment's hits are the rounds from rounds[r0] on (segment-relative reads, {adapter, record} each).
// Dm: the records go to the demux stage's call-wide arrays in read order (their bins group them once all are known), not to
// the caller's buffers.
int split_segment(Engine &E, cudaStream_t stream, const pb200_split_args_t &X, const uint8_t *reads, const int64_t *off, int64_t a,
                  int64_t n, const int64_t *first, const int64_t *toff, const std::vector<MiddleRound> &rounds, size_t r0,
                  SplitTotals &T, const DemuxStage *Dm = nullptr) {
    // ---- the hit reads and their extended ranges (rs - left, re + right) sorted by start: a CSR, a few ints per hit ----
    struct Rng { int32_t read, x, y; };
    std::vector<Rng> all;
    for (size_t k = r0; k < rounds.size(); ++k) {
        const MiddleRound &R = rounds[k];
        for (size_t p = 0; p < R.reads.size(); ++p) {
            const int32_t *h = R.hits.data() + p * PB_HIT_INTS;
            const auto clamp = [](int64_t v) { return (int32_t)std::min<int64_t>(std::max<int64_t>(v, INT32_MIN), INT32_MAX); };
            // record ends are inclusive: the reference masks and trims up to readEnd + 1
            all.push_back(Rng{R.reads[p], clamp((int64_t)h[1] - X.mid_extra_left[h[0]]),
                              clamp((int64_t)h[2] + 1 + X.mid_extra_right[h[0]])});
        }
    }
    std::sort(all.begin(), all.end(), [](const Rng &u, const Rng &v) { return u.read != v.read ? u.read < v.read : u.x < v.x; });
    std::vector<int32_t> hit_reads, rng_off(1, 0), rng;
    rng.reserve(all.size() * 2);
    for (size_t k = 0; k < all.size(); ++k) {
        if (k == 0 || all[k].read != all[k - 1].read) {
            if (k) rng_off.push_back((int32_t)k);
            hit_reads.push_back(all[k].read);
        }
        rng.push_back(all[k].x);
        rng.push_back(all[k].y);
    }
    if (!all.empty()) rng_off.push_back((int32_t)all.size());
    const int64_t n_h = (int64_t)hit_reads.size();
    if (int rc = E.split_hit_of.ensure((size_t)n * 4 + 16)) return rc;
    if (int rc = E.split_hits.ensure((size_t)n_h * 4 + 16)) return rc;
    if (int rc = E.split_rng_off.ensure((size_t)(n_h + 1) * 4 + 16)) return rc;
    if (int rc = E.split_rng.ensure(rng.size() * 4 + 16)) return rc;
    if (int rc = E.split_cnt.ensure((size_t)(n + 1) * 8)) return rc;
    if (int rc = E.split_bytes.ensure((size_t)(n + 1) * 8)) return rc;
    CK(cudaMemsetAsync(E.split_hit_of.p, 0xFF, (size_t)n * 4, stream));
    if (n_h) {
        CK(cudaMemcpyAsync(E.split_hits.p, hit_reads.data(), (size_t)n_h * 4, cudaMemcpyHostToDevice, stream));
        CK(cudaMemcpyAsync(E.split_rng_off.p, rng_off.data(), (size_t)(n_h + 1) * 4, cudaMemcpyHostToDevice, stream));
        CK(cudaMemcpyAsync(E.split_rng.p, rng.data(), rng.size() * 4, cudaMemcpyHostToDevice, stream));
        split_mark_kernel<<<(unsigned)((n_h + 255) / 256), 256, 0, stream>>>(static_cast<const int32_t *>(E.split_hits.as<int32_t>()),
                                                                             n_h, E.split_hit_of.as<int32_t>());
        g_launches++;
    }
    // the segment as the output stage's kernels read it (PB_SPLIT_READS_PARAMS)
    const int32_t *hit_of = E.split_hit_of.as<int32_t>(), *rng_off_d = E.split_rng_off.as<int32_t>(),
                  *rng_d = E.split_rng.as<int32_t>();
    const int64_t min_split = X.min_split_read_size;
    // ---- records and bases per read, scanned; the segment's totals come home ----
    int64_t *cnt = E.split_cnt.as<int64_t>(), *bytes = E.split_bytes.as<int64_t>();
    split_count_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(off, first, toff, hit_of, rng_off_d, rng_d, n, min_split,
                                                                        X.discard_middle, X.untrimmed, cnt, bytes);
    g_launches++;
    CK(cudaGetLastError());
    if (int rc = scan_offsets(E, stream, cnt, n)) return rc;
    if (int rc = scan_offsets(E, stream, bytes, n)) return rc;
    int64_t seg[2] = {0, 0};
    CK(cudaMemcpyAsync(&seg[0], cnt + n, 8, cudaMemcpyDeviceToHost, stream));
    CK(cudaMemcpyAsync(&seg[1], bytes + n, 8, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    if (!Dm && T.write && T.parts + seg[0] > X.parts_cap) T.write = false;     // PB200_ERR_SPACE: from here on only count
    if (Dm || T.write) {
        // ---- each record's output offset, read, part and source; then the gather, one warp per record.  Demux: the records
        // are appended to the call's records in read order instead, and gathered once their bins are known ----
        int64_t *src, *rec_off = X.d_out_off;
        int32_t *rec_read = X.d_out_read, *rec_part = X.d_out_part;
        if (Dm) {
            const size_t n_rec = (size_t)(T.parts + seg[0]), have = (size_t)T.parts;
            if (int rc = grow_keep(E.demux_rsrc, n_rec * 8 + 16, have * 8, stream)) return rc;
            if (int rc = grow_keep(E.demux_roff, (n_rec + 1) * 8 + 16, have * 8, stream)) return rc;
            if (int rc = grow_keep(E.demux_rread, n_rec * 4 + 16, have * 4, stream)) return rc;
            if (int rc = grow_keep(E.demux_rpart, n_rec * 4 + 16, have * 4, stream)) return rc;
            src = E.demux_rsrc.as<int64_t>() + T.parts;
            rec_off = E.demux_roff.as<int64_t>();
            rec_read = E.demux_rread.as<int32_t>();
            rec_part = E.demux_rpart.as<int32_t>();
        } else {
            if (int rc = E.split_src.ensure((size_t)seg[0] * 8 + 16)) return rc;
            src = E.split_src.as<int64_t>();
        }
        split_write_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(off, first, toff, hit_of, rng_off_d, rng_d, n, min_split,
                                                                            X.discard_middle, X.untrimmed,
                                                                            static_cast<const int64_t *>(cnt),
                                                                            static_cast<const int64_t *>(bytes), T.parts, T.bases, a,
                                                                            src, rec_off, rec_read, rec_part);
        g_launches++;
        if (!Dm && seg[0] > 0) {
            const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((seg[0] + 7) / 8, (int64_t)E.sm_count * 8));
            split_gather_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reads, X.d_quals, static_cast<const int64_t *>(src),
                                                                      static_cast<const int64_t *>(X.d_out_off + T.parts), seg[0],
                                                                      X.d_out_seq, X.d_out_qual);
            g_launches++;
        }
        CK(cudaGetLastError());
    }
    T.parts += seg[0];
    T.bases += seg[1];
    return 0;
}

// Demux stage, once per call after the last segment: the read bins come home, the call's records (T.parts of them, in read
// order) are partitioned stably by bin into the caller's buffers, and the bin offsets come home.  T becomes the totals of the
// records that are kept; when they do not fit parts_cap nothing is written (the caller reports PB200_ERR_SPACE).
int demux_finalize(Engine &E, Stage &S, cudaStream_t stream, const pb200_split_args_t &X, const pb200_demux_args_t &Dm,
                   const uint8_t *seqs, int64_t n_seqs, SplitTotals &T) {
    const int64_t n_rec = T.parts;
    const int32_t n_bins = Dm.n_bins, n_keys = n_bins + 2;              // the bins, 'none', dropped
    const int64_t tiles = (n_rec + PB_DEMUX_TILE - 1) / PB_DEMUX_TILE;
    const int32_t *read_bin = E.demux_bin.as<int32_t>();
    CK(cudaMemcpyAsync(Dm.read_bin, read_bin, (size_t)n_seqs * 4, cudaMemcpyDeviceToHost, stream));
    std::vector<int64_t> parts((size_t)n_keys + 1, 0);
    unsigned long long kept_bytes = 0;
    int64_t *cnt = nullptr;
    if (n_rec > 0) {
        // ---- (key x tile) counts, scanned key-major: every (key, tile) its first output record; the key offsets come home ----
        const int64_t m = (int64_t)n_keys * tiles;
        if (int rc = E.demux_cnt.ensure((size_t)(m + 1) * 8)) return rc;
        if (int rc = E.demux_parts.ensure((size_t)(n_keys + 1) * 8)) return rc;
        if (int rc = E.demux_kept.ensure(16)) return rc;
        cnt = E.demux_cnt.as<int64_t>();
        CK(cudaMemsetAsync(E.demux_kept.p, 0, 8, stream));
        demux_count_kernel<<<(unsigned)tiles, PB_DEMUX_TILE, 0, stream>>>(static_cast<const int32_t *>(E.demux_rread.as<int32_t>()),
                                                                          static_cast<const int64_t *>(E.demux_roff.as<int64_t>()), n_rec,
                                                                          read_bin, n_bins, Dm.discard_unassigned, tiles,
                                                                          cnt, E.demux_kept.as<unsigned long long>());
        g_launches++;
        CK(cudaGetLastError());
        if (int rc = scan_offsets(E, stream, cnt, m)) return rc;
        demux_bin_parts_kernel<<<(unsigned)((n_keys + 1 + 255) / 256), 256, 0, stream>>>(static_cast<const int64_t *>(cnt), tiles,
                                                                                          n_keys, E.demux_parts.as<int64_t>());
        g_launches++;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(parts.data(), E.demux_parts.p, (size_t)(n_keys + 1) * 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&kept_bytes, E.demux_kept.p, 8, cudaMemcpyDeviceToHost, stream));
    }
    if (int rc = check_status(S, stream)) return rc;    // (synchronises the stream) a score outside the table
    memcpy(Dm.bin_parts, parts.data(), (size_t)(n_bins + 2) * 8);
    const int64_t kept = parts[(size_t)n_bins + 1];
    T.parts = kept;
    T.bases = (int64_t)kept_bytes;
    if (kept > X.parts_cap) return 0;
    // ---- the kept records in bin order: lengths (scanned into offsets), reads, parts, permuted sources; then the gather ----
    CK(cudaMemsetAsync(X.d_out_off, 0, 8, stream));
    if (kept > 0) {
        if (int rc = E.demux_perm.ensure((size_t)kept * 8 + 16)) return rc;
        int64_t *perm = E.demux_perm.as<int64_t>();
        demux_scatter_kernel<<<(unsigned)tiles, PB_DEMUX_TILE, 0, stream>>>(
            static_cast<const int32_t *>(E.demux_rread.as<int32_t>()), static_cast<const int32_t *>(E.demux_rpart.as<int32_t>()),
            static_cast<const int64_t *>(E.demux_roff.as<int64_t>()), static_cast<const int64_t *>(E.demux_rsrc.as<int64_t>()), n_rec,
            read_bin, n_bins, Dm.discard_unassigned, tiles, static_cast<const int64_t *>(cnt), X.d_out_off + 1, X.d_out_read,
            X.d_out_part, perm);
        g_launches++;
        CK(cudaGetLastError());
        if (int rc = scan_offsets(E, stream, X.d_out_off, kept)) return rc;
        const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((kept + 7) / 8, (int64_t)E.sm_count * 8));
        split_gather_kernel<<<(unsigned)blocks, 256, 0, stream>>>(seqs, X.d_quals, static_cast<const int64_t *>(perm),
                                                                  static_cast<const int64_t *>(X.d_out_off), kept, X.d_out_seq,
                                                                  X.d_out_qual);
        g_launches++;
        CK(cudaGetLastError());
    }
    return 0;
}

// What the preconditions of a whole-read call establish before anything touches the device: the threshold-table lengths of
// both sides and of the middle scan, the longest read (-1: measured on the device) and the demux stage's score table.
struct TrimPlan {
    int32_t cmin_len[2] = {0, 0}, mid_cmin_len = 0;
    int64_t max_len = -1;
    DemuxStage dstage;
};

int trim_plan(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, bool device, int64_t total_seq_bytes,
              int64_t max_seq_len, const pb200_trim_args_t *A, int ma, int mi, int go, int ge, const pb200_split_args_t *X,
              const pb200_demux_args_t *Dm, TrimPlan &TP) {
    if (!A) return fail(PB200_ERR_ARG, "NULL pointer");
    if (n_seqs < 0 || total_seq_bytes < 0) return fail(PB200_ERR_ARG, "negative count");
    if (A->end_size < 1) return fail(PB200_ERR_ARG, "end_size must be >= 1");
    if (!(A->end_threshold >= 0.0)) return fail(PB200_ERR_ARG, "end_threshold must be >= 0 for the device decisions");
    load_env_options();
    const SchemeInfo si = scheme_info(ma, mi, go, ge);
    const pb200_trim_side_t *side[2] = {&A->start, &A->end};
    for (int k = 0; k < 2; ++k)
        if (int rc = trim_side_check(*side[k], n_seqs, A->end_size, si, &TP.cmin_len[k], Dm != nullptr)) return rc;
    const int32_t n_mid = A->n_mid_adapters;
    if (n_mid < 0) return fail(PB200_ERR_ARG, "negative count");
    if (n_mid > 0) {
        if (int rc = middle_entry_checks(n_seqs, A->mid_adapters, A->mid_ad_off, n_mid, ma, mi, go, ge, A->middle_threshold,
                                         A->n_hits, A->hits, A->hits_cap, A->n_total, &TP.mid_cmin_len)) return rc;
    }
    if (n_seqs > 0 && !seq_off) return fail(PB200_ERR_ARG, "NULL pointer");
    TP.max_len = max_seq_len;
    if (!device && n_seqs > 0) { if (int rc = host_max_len(seqs, seq_off, n_seqs, &TP.max_len)) return rc; }
    if (TP.max_len > 0x7fff0000ll) return fail(PB200_ERR_ARG, "sequence longer than 2^31");
    if (X) {
        if (!device) return fail(PB200_ERR_ARG, "the output stage takes device reads only");
        if (X->parts_cap < 0) return fail(PB200_ERR_ARG, "negative count");
        if (!X->n_parts || !X->n_out_bases) return fail(PB200_ERR_ARG, "NULL pointer");
        if (n_mid > 0 && (!X->mid_extra_left || !X->mid_extra_right)) return fail(PB200_ERR_ARG, "NULL pointer");
        if (!X->d_quals != !X->d_out_qual) return fail(PB200_ERR_ARG, "d_out_qual must be NULL exactly when d_quals is NULL");
        if (n_seqs > 0 && (!X->d_out_off || (X->parts_cap > 0 && (!X->d_out_read || !X->d_out_part ||
                                                                  (total_seq_bytes > 0 && !X->d_out_seq)))))
            return fail(PB200_ERR_ARG, "NULL pointer");
    }
    if (Dm) {
        if (!X) return fail(PB200_ERR_ARG, "the demux stage needs the output stage");
        if (!Dm->read_bin || !Dm->bin_parts) return fail(PB200_ERR_ARG, "NULL pointer");
        if (Dm->n_bins < 0 || Dm->n_bins >= 4096) return fail(PB200_ERR_ARG, "n_bins must be in [0, 4096)");
        if (std::isnan(Dm->barcode_threshold) || std::isnan(Dm->barcode_diff))
            return fail(PB200_ERR_ARG, "barcode_threshold / barcode_diff is NaN");
        std::vector<char> seen((size_t)Dm->n_bins);
        for (int k = 0; k < 2; ++k) {
            const int32_t *map = k ? Dm->end_bin : Dm->start_bin;
            const int32_t n_cols = side[k]->n_score_cols;
            if (n_cols == 0) continue;
            if (!map) return fail(PB200_ERR_ARG, "NULL pointer");
            std::fill(seen.begin(), seen.end(), 0);
            for (int32_t j = 0; j < n_cols; ++j) {
                if (map[j] < 0 || map[j] >= Dm->n_bins) return fail(PB200_ERR_ARG, "bin id out of range");
                if (seen[(size_t)map[j]]) return fail(PB200_ERR_ARG, "a bin appears twice on one side");
                seen[(size_t)map[j]] = 1;
            }
            // the score table covers every (match_ad, len_ad) of the side: match_ad <= its longest adapter, len_ad < cmin_len
            TP.dstage.tab_c = std::max(TP.dstage.tab_c, TP.cmin_len[k] - A->end_size - 1);
            TP.dstage.tab_l = std::max(TP.dstage.tab_l, TP.cmin_len[k]);
        }
    }
    return 0;
}

// The device work of a whole-read call on its stream, stage by stage.  device: seqs / seq_off are device pointers
// (adapterTrimReadsDevice), else host buffers uploaded segment by segment.  X: the output stage of adapterTrimSplitReadsDevice
// (device reads only), or nullptr.  Dm: the demux stage of adapterDemuxReadsDevice (with X), or nullptr.
struct TrimCall {
    Engine &E; Stage &S; cudaStream_t stream;
    const uint8_t *seqs; const int64_t *seq_off; int64_t n_seqs; bool device; int64_t total_seq_bytes;
    const pb200_trim_args_t &A; const pb200_split_args_t *X; const pb200_demux_args_t *Dm;
    TrimPlan &TP;
    std::vector<MiddleRound> &rounds;
    SplitTotals &totals;
    AdapterPlan P[2], PM;                 // the adapter plans of both sides and of the middle scan
    int64_t wl_max = 0;                   // the longest end window

    const pb200_trim_side_t &side(int k) const { return k ? A.end : A.start; }

    int run(int ma, int mi, int go, int ge) {
        if (int rc = reset_misc(S, stream)) return rc;
        if (int rc = check_status(S, stream)) return rc;     // a deferred error of an earlier device-resident call
        if (int rc = upload_tables(ma, mi, go, ge)) return rc;
        if (int rc = device_max_len(S, stream, seq_off, n_seqs, &TP.max_len)) return rc;
        wl_max = std::min<int64_t>(A.end_size, TP.max_len);
        if (device && A.n_mid_adapters > 0) { if (int rc = E.mid_codes.ensure((size_t)total_seq_bytes + 16)) return rc; }
        for (int64_t a = 0; a < n_seqs;) {
            const int64_t b = trim_segment_end(E, a, n_seqs, A.n_mid_adapters, wl_max, device ? nullptr : seq_off, X != nullptr,
                                               Dm != nullptr);
            if (int rc = segment(a, b - a)) return rc;
            a = b;
        }
        if (Dm) { if (int rc = demux_finalize(E, S, stream, *X, *Dm, seqs, n_seqs, totals)) return rc; }
        if (X) CK(cudaStreamSynchronize(stream));      // the device outputs are written when the call returns
        return 0;
    }

    // Reads [a, a + n): end windows, Phase B of both sides, the barcode call; then, with middle adapters or an output stage,
    // the trimmed ranges, Phase C and the output records.
    int segment(int64_t a, int64_t n) {
        const uint8_t *reads = nullptr;
        const int64_t *off = nullptr;
        if (int rc = segment_reads(a, n, reads, off)) return rc;
        int64_t win_total = -1;
        for (int k = 0; k < 2; ++k)
            if (int rc = end_side(k, a, n, win_total)) return rc;
        if (Dm) { if (int rc = barcode_call(a, n)) return rc; }
        const int32_t n_mid = A.n_mid_adapters;
        if (n_mid == 0) {
            if (int rc = check_status(S, stream)) return rc;
            if (!X) return 0;
        }
        MiddleSeg M;
        if (n_mid > 0) {
            if (int rc = middle_segment_buffers(E, n, n_mid, device ? 0 : (size_t)(seq_off[a + n] - seq_off[a]), M)) return rc;
        }
        if (int rc = trimmed_ranges(off, n)) return rc;
        const size_t r0 = rounds.size();
        if (n_mid > 0) { if (int rc = middle_scan(reads, off, a, M)) return rc; }
        if (!X) return 0;
        return split_segment(E, stream, *X, reads, off, a, n, E.trim_first.as<int64_t>(), E.mid_off.as<int64_t>(), rounds, r0,
                             totals, Dm ? &TP.dstage : nullptr);
    }

    // Per call: both sides' adapter plans and decision tables; the demux stage's bin of each score column, score table and
    // per-read bins; the middle scan's plan and threshold table.
    int upload_tables(int ma, int mi, int go, int ge) {
        for (int k = 0; k < 2; ++k) {
            const pb200_trim_side_t &T = side(k);
            if (T.n_adapters == 0) continue;
            if (int rc = plan_adapters(E, stream, T.adapters, T.ad_off, T.n_adapters, ma, mi, go, ge, P[k])) return rc;
            if (int rc = upload_decision_tables(E, k, stream, A.end_threshold, TP.cmin_len[k], T.score_cols, T.n_score_cols))
                return rc;
        }
        if (Dm) {                             // the call rule's inputs: bin of each score column, score table; a bin per read
            for (int k = 0; k < 2; ++k) {
                const int32_t n_cols = side(k).n_score_cols;
                if (n_cols == 0) continue;
                if (int rc = E.demux_map[k].ensure((size_t)n_cols * 4)) return rc;
                CK(cudaMemcpyAsync(E.demux_map[k].p, k ? Dm->end_bin : Dm->start_bin, (size_t)n_cols * 4, cudaMemcpyHostToDevice,
                                   stream));
            }
            if (TP.dstage.tab_c > 0) {
                const auto tab = cached_score_table(TP.dstage.tab_c, TP.dstage.tab_l);
                if (int rc = E.demux_tab.ensure(tab->size() * 8)) return rc;
                CK(cudaMemcpyAsync(E.demux_tab.p, tab->data(), tab->size() * 8, cudaMemcpyHostToDevice, stream));
            }
            if (int rc = E.demux_bin.ensure((size_t)n_seqs * 4 + 16)) return rc;
        }
        if (A.n_mid_adapters > 0) {
            if (int rc = plan_adapters(E, stream, A.mid_adapters, A.mid_ad_off, A.n_mid_adapters, ma, mi, go, ge, PM)) return rc;
            if (int rc = middle_table(E, stream, A.middle_threshold, TP.mid_cmin_len)) return rc;   // (synchronises the stream)
        }
        return 0;
    }

    // The segment's reads [a, a + n), ASCII at reads[off[s] .. off[s + 1]) -- host reads are uploaded here (their only upload),
    // offsets rebased to the segment -- and their end windows: lengths, offsets (shared by both sides), the cut into trim_win.
    int segment_reads(int64_t a, int64_t n, const uint8_t *&reads, const int64_t *&off) {
        reads = seqs;
        off = seq_off + a;
        if (!device) {
            const int64_t bytes = seq_off[a + n] - seq_off[a];
            if (int rc = E.trim_reads.ensure((size_t)bytes + 16)) return rc;
            if (int rc = E.trim_off.ensure((size_t)(n + 1) * 8)) return rc;
            if (bytes) CK(cudaMemcpyAsync(E.trim_reads.p, seqs + seq_off[a], (size_t)bytes, cudaMemcpyHostToDevice, stream));
            CK(cudaMemcpyAsync(E.trim_off.p, seq_off + a, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, stream));
            rebase_kernel<<<(unsigned)((n + 1 + 255) / 256), 256, 0, stream>>>(E.trim_off.as<int64_t>(), n + 1, seq_off[a]);
            g_launches++;
            reads = E.trim_reads.as<uint8_t>();
            off = E.trim_off.as<int64_t>();
        }
        const size_t win_bytes = (size_t)n * (size_t)wl_max;
        if (int rc = E.trim_win_off.ensure((size_t)(n + 1) * 8)) return rc;
        if (int rc = E.trim_win[0].ensure(win_bytes + 16)) return rc;
        if (int rc = E.trim_win[1].ensure(win_bytes + 16)) return rc;
        int64_t *win_off = E.trim_win_off.as<int64_t>();
        window_len_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(off, n, (int64_t)A.end_size, win_off);
        g_launches++;
        if (int rc = scan_offsets(E, stream, win_off, n)) return rc;
        const int64_t warp_blocks = std::max<int64_t>(1, std::min<int64_t>((n + 3) / 4, (int64_t)E.sm_count * 16));
        cut_windows_kernel<<<(unsigned)warp_blocks, 128, 0, stream>>>(reads, off, static_cast<const int64_t *>(win_off), n,
                                                                     E.trim_win[0].as<uint8_t>(), E.trim_win[1].as<uint8_t>());
        g_launches++;
        CK(cudaGetLastError());
        return 0;
    }

    // Phase B of side k over the segment's reads [a, a + n): DP chunks, each followed by decide_kernel into the segment-wide
    // trims trim_d[k].  win_total: the windows' total length, fetched (once per segment) when a side encodes them first.
    int end_side(int k, int64_t a, int64_t n, int64_t &win_total) {
        const pb200_trim_side_t &T = side(k);
        if (int rc = E.trim_d[k].ensure((size_t)n * 4 + 16)) return rc;
        if (T.n_adapters == 0) {
            CK(cudaMemsetAsync(E.trim_d[k].p, 0, (size_t)n * 4, stream));
            return 0;
        }
        const int64_t *win_off = E.trim_win_off.as<int64_t>();
        const bool ascii = single_pass_ascii(P[k], wl_max);
        const uint8_t *w = E.trim_win[k].as<uint8_t>();
        if (!ascii) {                // two-pass windows: encode first, as batch_device_queue does
            if (win_total < 0) {
                CK(cudaMemcpyAsync(&win_total, win_off + n, 8, cudaMemcpyDeviceToHost, stream));
                CK(cudaStreamSynchronize(stream));
            }
            if (int rc = S.seq_codes.ensure((size_t)win_total + 16)) return rc;
            if (int rc = launch_encode(stream, w, S.seq_codes.as<uint8_t>(), win_total, E.sm_count)) return rc;
            w = S.seq_codes.as<uint8_t>();
        }
        pb200_end_batch_t D;
        memset(&D, 0, sizeof D);
        D.is_start = k == 0 ? 1 : 0; D.end_size = A.end_size; D.extra_trim_size = A.extra_trim_size;
        D.min_trim_size = A.min_trim_size; D.end_threshold = A.end_threshold;
        D.score_cols = T.score_cols; D.n_score_cols = T.n_score_cols;
        D.trim = T.trim; D.score_pairs = T.score_pairs; D.top2 = T.top2;
        const int64_t max_cnt = std::max<int64_t>(1, g_opt.device_chunk_tasks / T.n_adapters);
        int32_t *top2 = nullptr;     // demux: the segment's ranking stays on the device for barcode_call_kernel
        if (Dm && T.n_score_cols > 0) {
            if (int rc = E.demux_top2[k].ensure((size_t)n * 6 * 4 + 16)) return rc;
            top2 = E.demux_top2[k].as<int32_t>();
        }
        for (int64_t c0 = 0; c0 < n; c0 += max_cnt) {
            const int64_t cnt = std::min(max_cnt, n - c0);
            if (int rc = S.out.ensure((size_t)cnt * T.n_adapters * PB_REC * 4)) return rc;
            if (int rc = run_cross_chunk(E, S, stream, P[k], w, win_off + c0, cnt, 0, wl_max, T.n_adapters, S.out.as<int32_t>(),
                                         nullptr, 0, T.ad_off, nullptr, ascii)) return rc;
            if (int rc = launch_decide(E, S, stream, D, S.out.as<int32_t>(), cnt, T.n_adapters, E.dec_cmin[k].as<int32_t>(),
                                       TP.cmin_len[k], E.dec_cols[k].as<int32_t>(), E.trim_d[k].as<int32_t>() + c0, a + c0,
                                       top2 ? top2 + c0 * 6 : nullptr))
                return rc;
        }
        return 0;
    }

    // The barcode call of every read of the segment [a, a + n), into the call-wide bins.
    int barcode_call(int64_t a, int64_t n) {
        const int32_t *t[2] = {nullptr, nullptr};
        for (int k = 0; k < 2; ++k) if (side(k).n_score_cols > 0) t[k] = E.demux_top2[k].as<int32_t>();
        barcode_call_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
            t[0], t[1], static_cast<const int32_t *>(E.demux_map[0].as<int32_t>()),
            static_cast<const int32_t *>(E.demux_map[1].as<int32_t>()), static_cast<const double *>(E.demux_tab.as<double>()),
            TP.dstage.tab_c, TP.dstage.tab_l, n, Dm->n_bins, Dm->barcode_threshold, Dm->barcode_diff, Dm->require_two_barcodes,
            Dm->d_albacore ? Dm->d_albacore + a : nullptr, E.demux_bin.as<int32_t>() + a, S.misc.as<int>());
        g_launches++;
        CK(cudaGetLastError());
        return 0;
    }

    // The trims -> every read's trimmed range: its first base in trim_first, the lengths scanned into offsets in mid_off.
    int trimmed_ranges(const int64_t *off, int64_t n) {
        if (int rc = E.trim_first.ensure((size_t)n * 8 + 16)) return rc;
        if (int rc = E.mid_off.ensure((size_t)(n + 1) * 8)) return rc;
        int64_t *toff = E.mid_off.as<int64_t>();
        trimmed_range_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(
            off, static_cast<const int32_t *>(E.trim_d[0].as<int32_t>()), static_cast<const int32_t *>(E.trim_d[1].as<int32_t>()),
            n, E.trim_first.as<int64_t>(), toff);
        g_launches++;
        return scan_offsets(E, stream, toff, n);
    }

    // Phase C of the segment that starts at read a: the trimmed reads encoded into the middle scan's resident codes, then
    // round 0 and the masking rounds, as in middle_device.
    int middle_scan(const uint8_t *reads, const int64_t *off, int64_t a, MiddleSeg &M) {
        M.codes = E.mid_codes.as<uint8_t>();
        M.off = E.mid_off.as<int64_t>();
        M.cmin_len = TP.mid_cmin_len;
        const int64_t warp_blocks = std::max<int64_t>(1, std::min<int64_t>((M.n + 3) / 4, (int64_t)E.sm_count * 16));
        gather_encode_kernel<<<(unsigned)warp_blocks, 128, 0, stream>>>(reads, off, static_cast<const int64_t *>(E.trim_first.as<int64_t>()),
                                                                       static_cast<const int64_t *>(M.off), M.n, M.codes);
        g_launches++;
        CK(cudaGetLastError());
        M.max_len = -1;
        if (int rc = device_max_len(S, stream, M.off, M.n, &M.max_len)) return rc;
        return middle_scan_resident(E, S, stream, PM, M, A.n_mid_adapters, A.mid_ad_off, a, rounds);
    }
};

int trim_reads(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, bool device, int64_t total_seq_bytes,
               int64_t max_seq_len, const pb200_trim_args_t *A, int ma, int mi, int go, int ge, void *user_stream,
               const pb200_split_args_t *X = nullptr, const pb200_demux_args_t *Dm = nullptr) {
    TrimPlan TP;
    if (int rc = trim_plan(seqs, seq_off, n_seqs, device, total_seq_bytes, max_seq_len, A, ma, mi, go, ge, X, Dm, TP)) return rc;
    // the host outputs the device does not write
    if (Dm) memset(Dm->bin_parts, 0, (size_t)(Dm->n_bins + 2) * 8);
    if (A->n_hits && n_seqs > 0) memset(A->n_hits, 0, (size_t)n_seqs * 4);
    if (A->n_total) *A->n_total = 0;
    for (const pb200_trim_side_t *T : {&A->start, &A->end})
        if (T->n_adapters == 0 && n_seqs > 0) fill_no_adapters(T->trim, T->top2, n_seqs);
    // without adapters nothing is trimmed or split; the output stage still writes every non-empty read ("No adapters found")
    if (n_seqs == 0 || (!X && A->start.n_adapters == 0 && A->end.n_adapters == 0 && A->n_mid_adapters == 0)) return 0;

    std::vector<MiddleRound> rounds;
    SplitTotals totals;
    const int rc = sync_call(device ? CallOn::library : CallOn::stage0, user_stream, [&](Engine &E, cudaStream_t stream) {
        NvtxRange submit_range(Dm ? "pb200:submit_demux" : X ? "pb200:submit_trim_split" : "pb200:submit_trim");
        TrimCall C{E, E.st[0], stream, seqs, seq_off, n_seqs, device, total_seq_bytes, *A, X, Dm, TP, rounds, totals};
        return C.run(ma, mi, go, ge);
    });
    if (rc) return rc;
    if (X) { *X->n_parts = totals.parts; *X->n_out_bases = totals.bases; }
    if (A->n_mid_adapters > 0) { if (int rc2 = middle_emit(rounds, n_seqs, A->n_hits, A->hits, A->hits_cap, A->n_total)) return rc2; }
    if (X && totals.parts > X->parts_cap) return fail(PB200_ERR_SPACE, "parts_cap is smaller than the number of records (*n_parts)");
    return 0;
}

// ---- output files (pb200EmitReadsDevice) -------------------------------------------------------------------------------
// Record lengths (checked on the device) scanned into d_out_off; the total, the check flag and the sticky status word come home
// in one synchronise; then, when everything holds, one warp per record writes the bytes.
int emit_reads(const pb200_emit_args_t *A, int64_t n_rec, void *user_stream) {
    if (!A) return fail(PB200_ERR_ARG, "NULL pointer");
    if (A->n_out_bytes) *A->n_out_bytes = 0;
    if (A->fmt != 0 && A->fmt != 1) return fail(PB200_ERR_ARG, "fmt must be 0 (FASTQ) or 1 (FASTA)");
    if (A->fmt == 0 && !A->d_qual) return fail(PB200_ERR_ARG, "FASTQ needs d_qual");
    if (n_rec < 0 || A->seq_bytes < 0 || A->n_reads < 0 || A->name_bytes < 0 || A->out_cap < 0)
        return fail(PB200_ERR_ARG, "negative count");
    if (!A->n_out_bytes || !A->d_out_off || (A->seq_bytes > 0 && !A->d_seq) || (A->name_bytes > 0 && !A->d_names) ||
        (A->n_reads > 0 && !A->d_name_off) || (A->out_cap > 0 && !A->d_out) ||
        (n_rec > 0 && (!A->d_off || !A->d_read || !A->d_part)))
        return fail(PB200_ERR_ARG, "NULL pointer");
    return sync_call(CallOn::library, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        NvtxRange range("pb200:emit");
        Stage &S = E.st[0];
        int64_t total = 0;
        if (int rc = reset_misc(S, stream)) return rc;
        int *bad = reinterpret_cast<int *>(S.misc.as<char>() + 48);
        if (n_rec > 0) {
            emit_count_kernel<<<(unsigned)((n_rec + 255) / 256), 256, 0, stream>>>(A->d_off, A->d_read, A->d_part, A->d_name_off, n_rec,
                                                                                   A->seq_bytes, A->n_reads, A->name_bytes, A->fmt,
                                                                                   A->d_out_off, bad);
            g_launches++;
            CK(cudaGetLastError());
            if (int rc = scan_offsets(E, stream, A->d_out_off, n_rec)) return rc;
        } else {
            CK(cudaMemsetAsync(A->d_out_off, 0, 8, stream));
        }
        int st[2] = {0, 0};
        CK(cudaMemcpyAsync(&total, A->d_out_off + n_rec, 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&st[0], S.misc.p, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&st[1], bad, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        *A->n_out_bytes = total;
        if (int rc = status_error(st[0])) return rc;       // a deferred error of an earlier device-resident call
        if (st[1]) return fail(PB200_ERR_ARG, "a record's offsets, read, part or name range is out of range");
        if (total > A->out_cap) return fail(PB200_ERR_SPACE, "out_cap is smaller than the output (*n_out_bytes)");
        if (n_rec > 0) {
            const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((n_rec + 7) / 8, (int64_t)E.sm_count * 8));
            emit_write_kernel<<<(unsigned)blocks, 256, 0, stream>>>(A->d_seq, A->d_qual, A->d_off, A->d_read, A->d_part, A->d_names,
                                                                    A->d_name_off, A->d_rna, A->fmt,
                                                                    static_cast<const int64_t *>(A->d_out_off), n_rec, A->d_out);
            g_launches++;
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(stream));              // the device outputs are written when the call returns
        }
        return 0;
    });
}

// ---- parsing (pb200ParseReadsDevice) -----------------------------------------------------------------------------------
// The lines are counted per tile and the count comes home (it sizes the line index); the line ends, the record or line index
// and its scans follow, and the counts, totals and check flags come home in one synchronise.  When the input is well formed
// and everything fits, the offsets are copied out and one warp per record (FASTQ) or line (FASTA) writes the bytes; one warp
// per read then normalises the bases.
int parse_reads(const pb200_parse_args_t *A, void *user_stream) {
    if (!A) return fail(PB200_ERR_ARG, "NULL pointer");
    for (int64_t *p : {A->n_reads, A->n_name_bytes, A->n_seq_bytes}) if (p) *p = 0;
    if (A->error) *A->error = PB200_PARSE_OK;
    if (A->error_index) *A->error_index = -1;
    if (!A->n_reads || !A->n_name_bytes || !A->n_seq_bytes || !A->error || !A->error_index) return fail(PB200_ERR_ARG, "NULL pointer");
    if (A->fmt != 0 && A->fmt != 1) return fail(PB200_ERR_ARG, "fmt must be 0 (FASTQ) or 1 (FASTA)");
    if (A->n_in < 0 || A->names_cap < 0 || A->seq_cap < 0 || A->reads_cap < 0) return fail(PB200_ERR_ARG, "negative count");
    if ((A->n_in > 0 && !A->d_in) || !A->d_name_off || !A->d_seq_off || (A->names_cap > 0 && !A->d_names) ||
        (A->seq_cap > 0 && !A->d_seq) || (A->reads_cap > 0 && !A->d_rna))
        return fail(PB200_ERR_ARG, "NULL pointer");
    const int64_t n = A->n_in;
    const bool fastq = A->fmt == 0;
    return sync_call(CallOn::library, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        NvtxRange range("pb200:parse");
        if (n == 0) {                                      // no reads: the offsets' first entries only
            CK(cudaMemsetAsync(A->d_name_off, 0, 8, stream));
            CK(cudaMemsetAsync(A->d_seq_off, 0, 8, stream));
            CK(cudaStreamSynchronize(stream));
            return 0;
        }
        Stage &S = E.st[0];
        if (int rc = reset_misc(S, stream)) return rc;
        int *flags = reinterpret_cast<int *>(S.misc.as<char>() + 56);
        // ---- the line index ----
        const int64_t tiles = (n + PB_PARSE_TILE - 1) / PB_PARSE_TILE;
        if (int rc = E.parse_tiles.ensure((size_t)(tiles + 1) * 8)) return rc;
        int64_t *first_line = E.parse_tiles.as<int64_t>();
        parse_count_lines_kernel<<<(unsigned)tiles, PB_PARSE_THREADS, 0, stream>>>(A->d_in, n, first_line);
        g_launches++;
        CK(cudaGetLastError());
        if (int rc = scan_offsets(E, stream, first_line, tiles)) return rc;
        int64_t n_nl = 0;
        uint8_t last = 0;
        CK(cudaMemcpyAsync(&n_nl, first_line + tiles, 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&last, A->d_in + n - 1, 1, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        const int64_t n_lines = n_nl + (last != '\n');
        if (fastq && n_lines % 4 != 0) {
            *A->error = PB200_PARSE_LINES;
            *A->error_index = n_lines / 4;
            return fail(PB200_ERR_ARG, "FASTQ chunk is not a whole number of 4-line records");
        }
        if (int rc = E.parse_lines.ensure((size_t)n_lines * 8)) return rc;
        int64_t *line_end = E.parse_lines.as<int64_t>();
        parse_line_ends_kernel<<<(unsigned)tiles, PB_PARSE_THREADS, 0, stream>>>(A->d_in, n, static_cast<const int64_t *>(first_line),
                                                                                 line_end);
        g_launches++;
        CK(cudaGetLastError());
        // ---- records (FASTQ) or lines (FASTA): spans, checks, lengths scanned into offsets ----
        const int64_t m = fastq ? n_lines / 4 : n_lines;   // index entries: records or lines
        if (int rc = E.parse_index.ensure((size_t)(m + 1) * 8 * 7)) return rc;
        if (int rc = E.parse_status.ensure((size_t)m)) return rc;
        int64_t *ix = E.parse_index.as<int64_t>();
        int64_t *col[7];
        for (int c = 0; c < 7; ++c) col[c] = ix + (size_t)c * (m + 1);
        uint8_t *status = E.parse_status.as<uint8_t>();
        const unsigned grid = (unsigned)std::max<int64_t>(1, (m + 255) / 256);
        // FASTQ: name_a, name_off, seq_a, seq_off, qual_a, qual_len.  FASTA: span_a, span_len, hdr, nm, body, name_off, seq_off.
        int64_t *name_off = fastq ? col[1] : col[5], *seq_off = fastq ? col[3] : col[6];
        int64_t tot[3] = {0, 0, 0};                        // reads, name bytes, bases
        if (fastq) {
            parse_fastq_index_kernel<<<grid, 256, 0, stream>>>(A->d_in, static_cast<const int64_t *>(line_end), m, A->d_qual != nullptr,
                                                               col[0], col[1], col[2], col[3], col[4], col[5], status, flags);
            g_launches++;
            CK(cudaGetLastError());
            if (int rc = scan_offsets(E, stream, name_off, m)) return rc;
            if (int rc = scan_offsets(E, stream, seq_off, m)) return rc;
            tot[0] = m;
        } else {
            parse_fasta_lines_kernel<<<grid, 256, 0, stream>>>(A->d_in, static_cast<const int64_t *>(line_end), m, col[0], col[1],
                                                               col[2], col[3], col[4]);
            g_launches++;
            CK(cudaGetLastError());
            for (int c = 2; c < 5; ++c)
                if (int rc = scan_offsets(E, stream, col[c], m)) return rc;
            parse_fasta_records_kernel<<<grid, 256, 0, stream>>>(col[1], col[2], col[3], col[4], A->d_in, col[0], m, name_off, seq_off,
                                                                 status, flags);
            g_launches++;
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(&tot[0], col[2] + m, 8, cudaMemcpyDeviceToHost, stream));
        }
        int st[2] = {0, 0};
        CK(cudaMemcpyAsync(&tot[1], (fastq ? name_off : col[3]) + m, 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&tot[2], (fastq ? seq_off : col[4]) + m, 8, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&st[0], S.misc.p, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaMemcpyAsync(&st[1], flags, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        *A->n_reads = tot[0];
        *A->n_name_bytes = tot[1];
        *A->n_seq_bytes = tot[2];
        if (int rc = status_error(st[0])) return rc;       // a deferred error of an earlier device-resident call
        if (st[1]) {                                       // malformed input: the first record / line of the first failing check
            const int bad = (st[1] & 2) ? 1 : 2;
            std::vector<uint8_t> h((size_t)m);
            CK(cudaMemcpyAsync(h.data(), status, (size_t)m, cudaMemcpyDeviceToHost, stream));
            CK(cudaStreamSynchronize(stream));
            *A->error_index = std::find(h.begin(), h.end(), (uint8_t)bad) - h.begin();
            if (fastq) {
                *A->error = bad == 1 ? PB200_PARSE_HEADER : PB200_PARSE_LONG_QUAL;
                return fail(PB200_ERR_ARG, bad == 1 ? "FASTQ record does not start with @"
                                                    : "a quality line is longer than its bases (parse this chunk on the host)");
            }
            *A->error = bad == 1 ? PB200_PARSE_FASTA_START : PB200_PARSE_FASTA_NAME;
            return fail(PB200_ERR_ARG, bad == 1 ? "FASTA does not start with a > line" : "FASTA record with an empty name");
        }
        if (tot[0] > A->reads_cap || tot[1] > A->names_cap || tot[2] > A->seq_cap)
            return fail(PB200_ERR_SPACE, "reads_cap, names_cap or seq_cap is smaller than the parse (*n_reads, *n_name_bytes, *n_seq_bytes)");
        // ---- the outputs ----
        const int64_t r = tot[0];
        CK(cudaMemcpyAsync(A->d_name_off, name_off, (size_t)(r + 1) * 8, cudaMemcpyDeviceToDevice, stream));
        CK(cudaMemcpyAsync(A->d_seq_off, seq_off, (size_t)(r + 1) * 8, cudaMemcpyDeviceToDevice, stream));
        const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((m + 7) / 8, (int64_t)E.sm_count * 8));
        if (fastq) {
            parse_fastq_write_kernel<<<(unsigned)blocks, 256, 0, stream>>>(A->d_in, col[0], name_off, col[2], seq_off, col[4], col[5], m,
                                                                           A->d_names, A->d_seq, A->d_qual);
        } else {
            parse_fasta_write_kernel<<<(unsigned)blocks, 256, 0, stream>>>(A->d_in, col[0], col[1], col[3], col[4], m, A->d_names,
                                                                           A->d_seq);
            if (A->d_qual && tot[2] > 0) CK(cudaMemsetAsync(A->d_qual, '+', (size_t)tot[2], stream));
        }
        g_launches++;
        CK(cudaGetLastError());
        if (r > 0) {
            const int64_t nb = std::max<int64_t>(1, std::min<int64_t>((r + 7) / 8, (int64_t)E.sm_count * 8));
            parse_normalise_kernel<<<(unsigned)nb, 256, 0, stream>>>(static_cast<const int64_t *>(A->d_seq_off), r, A->d_seq, A->d_rna);
            g_launches++;
            CK(cudaGetLastError());
        }
        CK(cudaStreamSynchronize(stream));                 // the device outputs are written when the call returns
        return 0;
    });
}

// ---- gzip members (pb200GzipDevice) ------------------------------------------------------------------------------------
int64_t gzip_block_of(int32_t block) { return block == 0 ? PB_GZ_DEFAULT_BLOCK : block; }
// most bytes for n bytes in n_segs segments: every member stored; a segment adds at most one short block
int64_t gzip_bound(int64_t n, int64_t n_segs, int64_t block) {
    const int64_t members = n == 0 ? 0 : (n + block - 1) / block + n_segs - 1;
    return n + members * (gz_member_bound(block) - block);
}
// The block table goes up, one CTA per block writes its member into its slot, the sizes are scanned into offsets and come home
// with the status word in one synchronise; then, when the total fits, split_gather_kernel packs the members into d_out.
int gzip_device(const pb200_gzip_args_t *A, void *user_stream) {
    if (!A) return fail(PB200_ERR_ARG, "NULL pointer");
    if (A->n_out_bytes) *A->n_out_bytes = 0;
    if (!A->n_out_bytes || !A->seg_off || !A->out_seg_off) return fail(PB200_ERR_ARG, "NULL pointer");
    if (A->n < 0 || A->n_segs < 1 || A->out_cap < 0) return fail(PB200_ERR_ARG, "negative count (or no segment)");
    if ((A->n > 0 && !A->d_src) || (A->out_cap > 0 && !A->d_out)) return fail(PB200_ERR_ARG, "NULL pointer");
    if (A->block != 0 && (A->block < PB_GZ_MIN_BLOCK || A->block > PB_GZ_MAX_BLOCK))
        return fail(PB200_ERR_ARG, "block must be 0 (default) or 4096 .. 131072");
    const int64_t ns = A->n_segs, n = A->n;
    if (A->seg_off[0] != 0 || A->seg_off[ns] != n) return fail(PB200_ERR_ARG, "seg_off must run from 0 to n");
    for (int64_t s = 0; s < ns; ++s)
        if (A->seg_off[s + 1] < A->seg_off[s]) return fail(PB200_ERR_ARG, "seg_off is not ascending");
    const int32_t block = (int32_t)gzip_block_of(A->block);
    const int64_t stride = (gz_member_bound(block) + 15) & ~(int64_t)15;
    std::vector<int64_t> start, len, first(ns + 1);        // blocks; the first block of every segment
    for (int64_t s = 0; s < ns; ++s) {
        first[s] = (int64_t)start.size();
        for (int64_t p = A->seg_off[s]; p < A->seg_off[s + 1]; p += block) {
            start.push_back(p);
            len.push_back(std::min<int64_t>(block, A->seg_off[s + 1] - p));
        }
    }
    const int64_t nb = (int64_t)start.size();
    first[ns] = nb;
    std::vector<int64_t> table(3 * nb);
    for (int64_t b = 0; b < nb; ++b) { table[b] = start[b]; table[nb + b] = len[b]; table[2 * nb + b] = b * stride; }
    return sync_call(CallOn::library, user_stream, [&](Engine &E, cudaStream_t stream) -> int {
        NvtxRange range("pb200:gzip");
        Stage &S = E.st[0];
        if (int rc = reset_misc(S, stream)) return rc;
        std::vector<int64_t> off(nb + 1, 0);
        int st = 0;
        if (nb > 0) {
            if (int rc = E.gz_table.ensure((size_t)nb * 24)) return rc;
            if (int rc = E.gz_slots.ensure((size_t)(nb * stride))) return rc;
            if (int rc = E.gz_tokens.ensure((size_t)nb * block * 4)) return rc;
            if (int rc = E.gz_sizes.ensure((size_t)(nb + 1) * 8)) return rc;
            int64_t *tab = E.gz_table.as<int64_t>(), *sizes = E.gz_sizes.as<int64_t>();
            CK(cudaMemcpyAsync(tab, table.data(), (size_t)nb * 24, cudaMemcpyHostToDevice, stream));
            const size_t smem = (size_t)gz_smem_bytes(block);
            int bps = 0;
            if (int rc = E.blocks_per_sm(reinterpret_cast<const void *>(&gzip_block_kernel), PB_GZ_THREADS, smem, &bps)) return rc;
            gzip_block_kernel<<<(unsigned)nb, PB_GZ_THREADS, smem, stream>>>(A->d_src, static_cast<const int64_t *>(tab),
                                                                            static_cast<const int64_t *>(tab + nb), block,
                                                                            E.gz_slots.as<uint8_t>(), stride,
                                                                            E.gz_tokens.as<uint32_t>(), sizes);
            g_launches++;
            CK(cudaGetLastError());
            if (int rc = scan_offsets(E, stream, sizes, nb)) return rc;
            CK(cudaMemcpyAsync(off.data(), sizes, (size_t)(nb + 1) * 8, cudaMemcpyDeviceToHost, stream));
        }
        CK(cudaMemcpyAsync(&st, S.misc.p, 4, cudaMemcpyDeviceToHost, stream));
        CK(cudaStreamSynchronize(stream));
        for (int64_t s = 0; s <= ns; ++s) A->out_seg_off[s] = off[first[s]];
        *A->n_out_bytes = off[nb];
        if (int rc = status_error(st)) return rc;          // a deferred error of an earlier device-resident call
        if (off[nb] > A->out_cap) return fail(PB200_ERR_SPACE, "out_cap is smaller than the output (*n_out_bytes)");
        if (nb > 0) {
            const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>((nb + 7) / 8, (int64_t)E.sm_count * 8));
            split_gather_kernel<<<(unsigned)blocks, 256, 0, stream>>>(E.gz_slots.as<uint8_t>(), nullptr,
                                                                      static_cast<const int64_t *>(E.gz_table.as<int64_t>() + 2 * nb),
                                                                      static_cast<const int64_t *>(E.gz_sizes.as<int64_t>()), nb,
                                                                      A->d_out, nullptr);
            g_launches++;
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(stream));              // the device output is written when the call returns
        }
        return 0;
    });
}

}  // namespace

// =====================================================================================================
extern "C" {

int adapterAlignmentBatch(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
                          const int32_t *ad_off, int32_t n_adapters, const int32_t *pair_seq,
                          const int32_t *pair_adapter, int64_t n_pairs, int ma, int mi, int go, int ge, int32_t *out) {
    g_err.clear();
    return batch_host(seqs, seq_off, n_seqs, adapters, ad_off, n_adapters, pair_seq, pair_adapter, n_pairs, ma, mi, go, ge, out);
}

int adapterAlignmentBatchMulti(const pb200_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    g_err.clear();
    return batch_host_multi(batches, n_batches, ma, mi, go, ge);
}

int adapterEndDecisions(const pb200_end_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    g_err.clear();
    return batch_end_decisions(batches, n_batches, ma, mi, go, ge);
}

int adapterSetSearch(const pb200_search_batch_t *batches, int n_batches, int ma, int mi, int go, int ge) {
    g_err.clear();
    return batch_search(batches, n_batches, ma, mi, go, ge);
}

int pb200TrimThresholdTable(double end_threshold, int32_t len, int32_t *cmin) {
    if (len < 0 || (len > 0 && !cmin) || !(end_threshold >= 0.0)) return PB200_ERR_ARG;
    threshold_table(end_threshold, len, false, cmin);
    return 0;
}

int adapterMiddleScan(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const uint8_t *adapters,
                      const int32_t *ad_off, int32_t n_adapters, int ma, int mi, int go, int ge, double middle_threshold,
                      int32_t *n_hits, int32_t *hits, int64_t hits_cap, int64_t *n_total) {
    g_err.clear();
    return middle_host(seqs, seq_off, n_seqs, adapters, ad_off, n_adapters, ma, mi, go, ge, middle_threshold, n_hits, hits,
                       hits_cap, n_total);
}

int adapterMiddleScanDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                            int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters, int ma,
                            int mi, int go, int ge, double middle_threshold, int32_t *n_hits, int32_t *hits, int64_t hits_cap,
                            int64_t *n_total, void *stream) {
    g_err.clear();
    return middle_device(d_seqs, d_seq_off, n_seqs, total_seq_bytes, max_seq_len, adapters, ad_off, n_adapters, ma, mi, go, ge,
                         middle_threshold, n_hits, hits, hits_cap, n_total, stream);
}

int adapterTrimReads(const uint8_t *seqs, const int64_t *seq_off, int64_t n_seqs, const pb200_trim_args_t *args, int ma, int mi,
                     int go, int ge) {
    g_err.clear();
    return trim_reads(seqs, seq_off, n_seqs, false, 0, -1, args, ma, mi, go, ge, nullptr);
}

int adapterTrimReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                           int64_t max_seq_len, const pb200_trim_args_t *args, int ma, int mi, int go, int ge, void *stream) {
    g_err.clear();
    return trim_reads(d_seqs, d_seq_off, n_seqs, true, total_seq_bytes, max_seq_len, args, ma, mi, go, ge, stream);
}

int adapterTrimSplitReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                                int64_t max_seq_len, const pb200_trim_args_t *args, const pb200_split_args_t *split, int ma, int mi,
                                int go, int ge, void *stream) {
    g_err.clear();
    if (!split) return fail(PB200_ERR_ARG, "NULL pointer");
    if (split->n_parts) *split->n_parts = 0;
    if (split->n_out_bases) *split->n_out_bases = 0;
    return trim_reads(d_seqs, d_seq_off, n_seqs, true, total_seq_bytes, max_seq_len, args, ma, mi, go, ge, stream, split);
}

int adapterDemuxReadsDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                            int64_t max_seq_len, const pb200_trim_args_t *args, const pb200_split_args_t *split,
                            const pb200_demux_args_t *demux, int ma, int mi, int go, int ge, void *stream) {
    g_err.clear();
    if (!split) return fail(PB200_ERR_ARG, "NULL pointer");
    if (split->n_parts) *split->n_parts = 0;
    if (split->n_out_bases) *split->n_out_bases = 0;
    if (!demux) return fail(PB200_ERR_ARG, "NULL pointer");
    return trim_reads(d_seqs, d_seq_off, n_seqs, true, total_seq_bytes, max_seq_len, args, ma, mi, go, ge, stream, split, demux);
}

int pb200EmitReadsDevice(const pb200_emit_args_t *args, int64_t n_rec, void *stream) {
    g_err.clear();
    return emit_reads(args, n_rec, stream);
}

int pb200ParseReadsDevice(const pb200_parse_args_t *args, void *stream) {
    g_err.clear();
    return parse_reads(args, stream);
}

int pb200GzipDevice(const pb200_gzip_args_t *args, void *stream) {
    g_err.clear();
    return gzip_device(args, stream);
}

int64_t pb200GzipBound(int64_t n, int64_t n_segs, int32_t block) {
    if (n < 0 || n_segs < 1 || (block != 0 && (block < PB_GZ_MIN_BLOCK || block > PB_GZ_MAX_BLOCK))) return -1;
    return gzip_bound(n, n_segs, gzip_block_of(block));
}

int pb200MiddleThresholdTable(double middle_threshold, int32_t len, int32_t *cmin) {
    if (len < 0 || (len > 0 && !cmin) || !(middle_threshold > 0.0)) return PB200_ERR_ARG;
    threshold_table(middle_threshold, len, true, cmin);
    return 0;
}

int adapterAlignmentBatchDevice(const uint8_t *d_seqs, const int64_t *d_seq_off, int64_t n_seqs, int64_t total_seq_bytes,
                                int64_t max_seq_len, const uint8_t *adapters, const int32_t *ad_off, int32_t n_adapters,
                                int ma, int mi, int go, int ge, int32_t *d_out, void *stream) {
    g_err.clear();
    return batch_device(d_seqs, d_seq_off, n_seqs, total_seq_bytes, max_seq_len, adapters, ad_off, n_adapters, ma, mi, go,
                        ge, d_out, stream);
}

int pb200FormatRecord(const int32_t *r, char *buf, int buflen) {
    int n;
    if (r[0] == -1 && r[4] == PB_SCORE_EMPTY) {
        n = snprintf(buf, (size_t)buflen, "-1,0,-1,0,-2147483648,0.000000,0.000000");
    } else {
        // the two divisions of porechop/src/alignment.cpp:82,90 in double; 0/0 prints "-nan" like the reference
        volatile double c1 = (double)r[5], l1 = (double)r[6], c2 = (double)r[7], l2 = (double)r[8];
        double p1 = 100.0 * c1 / l1, p2 = 100.0 * c2 / l2;
        n = snprintf(buf, (size_t)buflen, "%d,%d,%d,%d,%d,%f,%f", r[0], r[1], r[2], r[3], r[4], p1, p2);
    }
    return (n < 0 || n >= buflen) ? -1 : n;
}

int pb200PackNibbles(const uint8_t *ascii, int64_t n, uint8_t *packed, int threads) {
    if (n < 0 || (n > 0 && (!ascii || !packed))) return PB200_ERR_ARG;
    pb_pack_nibbles(ascii, n, packed, threads);
    return 0;
}

char *adapterAlignment(char *readSeq, char *adapterSeq, int ma, int mi, int go, int ge) {
    g_err.clear();
    const int64_t n = readSeq ? (int64_t)strlen(readSeq) : 0;
    const int64_t m = adapterSeq ? (int64_t)strlen(adapterSeq) : 0;
    int32_t rec[PB_REC];
    if (n == 0 || m == 0) {
        rec[0] = -1; rec[1] = 0; rec[2] = -1; rec[3] = 0; rec[4] = PB_SCORE_EMPTY; rec[5] = rec[6] = rec[7] = rec[8] = 0;
    } else {
        int64_t soff[2] = {0, n};
        int32_t aoff[2] = {0, (int32_t)m};
        int rc = batch_host((const uint8_t *)readSeq, soff, 1, (const uint8_t *)adapterSeq, aoff, 1, nullptr, nullptr, 1, ma, mi,
                            go, ge, rec);
        if (rc != 0) {
            fprintf(stderr, "porechop_b200: adapterAlignment failed (%d): %s\n", rc, g_err.c_str());
            return nullptr;
        }
    }
    char *buf = (char *)malloc(96);
    if (!buf) return nullptr;
    if (pb200FormatRecord(rec, buf, 96) < 0) { free(buf); return nullptr; }
    return buf;
}

void freeCString(char *p) { free(p); }

int pb200DeviceCount(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int pb200SetDevice(int device) {
    g_err.clear();
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(PB200_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e));
    return 0;
}
const char *pb200LastError(void) { return g_err.c_str(); }
long long pb200KernelLaunches(void) { return g_launches.load(); }
void pb200TimingEnable(int on) { g_timing.store(on ? 1 : 0); }

int pb200TimingReadKinds(double *ms, long long *launches, double *window_cells, int reset) {
    Engine *Ep = nullptr;
    if (int rc = get_engine(&Ep)) return rc;
    Engine &E = *Ep;
    std::lock_guard<std::mutex> lk(E.mu);
    for (auto &tl : E.timed) {
        float f = 0.f;
        if (cudaEventSynchronize(tl.b) == cudaSuccess && cudaEventElapsedTime(&f, tl.a, tl.b) == cudaSuccess) {
            E.timed_ms_acc[tl.kind] += f; E.timed_n_acc[tl.kind]++;
        }
        cudaEventDestroy(tl.a); cudaEventDestroy(tl.b);
    }
    E.timed.clear();
    for (int k = 0; k < TK_N; ++k) {
        if (ms) ms[k] = E.timed_ms_acc[k];
        if (launches) launches[k] = E.timed_n_acc[k];
    }
    unsigned long long wc = 0;
    if (E.wcells.p) {
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpyAsync(&wc, E.wcells.p, 8, cudaMemcpyDeviceToHost, E.st[0].stream));
        if (reset) CK(cudaMemsetAsync(E.wcells.p, 0, 8, E.st[0].stream));
        CK(cudaStreamSynchronize(E.st[0].stream));
    }
    if (window_cells) *window_cells = (double)wc;
    if (reset) for (int k = 0; k < TK_N; ++k) { E.timed_ms_acc[k] = 0; E.timed_n_acc[k] = 0; }
    return 0;
}

int pb200TimingRead(double *ms, long long *launches, double *cells, int reset) {
    double m[TK_N]; long long n[TK_N]; double wc = 0;
    if (int rc = pb200TimingReadKinds(m, n, &wc, reset)) return rc;
    if (ms) { *ms = 0; for (int k = 0; k < TK_N; ++k) *ms += m[k]; }
    if (launches) { *launches = 0; for (int k = 0; k < TK_N; ++k) *launches += n[k]; }
    if (cells) *cells = wc;
    return 0;
}

int pb200Synchronize(void) {
    g_err.clear();
    Engine *Ep = nullptr;
    if (int rc = get_engine(&Ep)) return rc;
    Engine &E = *Ep;
    std::lock_guard<std::mutex> lk(E.mu);
    if (!E.init_done) return 0;
    CK(cudaDeviceSynchronize());
    E.last_pending = false;
    int rc_final = 0;
    for (int i = 0; i < NSTAGE; ++i) {
        if (!E.st[i].misc.p) continue;
        if (int rc = check_status(E.st[i], E.st[i].stream)) rc_final = rc;
        CK(cudaMemsetAsync(E.st[i].misc.p, 0, 4, E.st[i].stream));
        CK(cudaStreamSynchronize(E.st[i].stream));
    }
    return rc_final;
}

// Pinned staging memory for host callers (fastq.py gathers the trimmed reads of a chunk before the middle scan): `slot` 0..3,
// grown on demand, owned by the library, valid until the next call for the same slot.  NULL without a device (callers then
// use ordinary memory).  A pinned source makes the engine's uploads asynchronous DMA at PCIe speed and is reused chunk after
// chunk instead of page-faulting in a fresh gigabyte every time.
void *pb200HostBuffer(int slot, size_t bytes) {
    static HostBuf bufs[4];
    static std::mutex mu;
    if (slot < 0 || slot >= 4) return nullptr;
    Engine *Ep = nullptr;
    if (get_engine(&Ep)) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    if (bufs[slot].ensure(bytes ? bytes : 1)) return nullptr;
    return bufs[slot].p;
}

int pb200GetOption(const char *name) {
    load_env_options();
    if (!name) return -1;
    if (!strcmp(name, "h2d_pack")) return g_opt.h2d_pack;
    if (!strcmp(name, "h2d_pack_large_submit")) return pack_wanted(1ll << 40) ? 1 : 0;   // what "auto" resolves to for a large submit
    if (!strcmp(name, "pack_threads")) return g_opt.pack_threads;
    if (!strcmp(name, "tight_window")) return g_opt.tight_window;
    if (!strcmp(name, "profile")) return g_opt.profile;
    if (!strcmp(name, "scratch_mb")) return g_opt.scratch_mb;
    if (!strcmp(name, "hbuf")) return g_opt.hbuf_mode;
    if (!strcmp(name, "direct_max")) return (int)std::min<int64_t>(g_opt.direct_max, INT_MAX);
    if (!strcmp(name, "chunk_tasks")) return (int)std::min<int64_t>(g_opt.chunk_tasks, INT_MAX);
    return -1;
}

int pb200SetOption(const char *name, const char *value) {
    load_env_options();
    if (!name || !value) return PB200_ERR_ARG;
    if (!strcmp(name, "direct_max")) g_opt.direct_max = atoll(value);
    else if (!strcmp(name, "chunk_tasks")) g_opt.chunk_tasks = std::max(1ll, atoll(value));
    else if (!strcmp(name, "scratch_mb")) g_opt.scratch_mb = std::max(1, atoi(value));
    else if (!strcmp(name, "tight_window")) g_opt.tight_window = atoi(value);
    else if (!strcmp(name, "h2d_pack")) g_opt.h2d_pack = atoi(value);
    else if (!strcmp(name, "profile")) g_opt.profile = atoi(value);
    else if (!strcmp(name, "pack_threads")) { if (atoi(value) > 0) g_opt.pack_threads = atoi(value); }
    else if (!strcmp(name, "hbuf")) g_opt.hbuf_mode = !strcmp(value, "smem") ? 1 : !strcmp(value, "global") ? 2 : 0;
    else return PB200_ERR_ARG;
    return 0;
}

}  // extern "C"
