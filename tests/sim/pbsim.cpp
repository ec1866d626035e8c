// tests/sim/pbsim.cpp -- block scheduler of the host CUDA stand-in (see pbsim_cuda.h).  TESTS ONLY.
#include "pbsim_cuda.h"

#include <memory>
#include <mutex>
#include <set>

#if defined(__x86_64__) && !defined(PBSIM_NO_FAST_SWITCH)
// swapcontext() saves and restores the signal mask with a system call on every switch; a fiber switch here only needs the
// callee-saved registers and the stack pointer.
extern "C" void pbsim_swap(void **save_sp, void *load_sp);
asm(R"(
    .text
    .globl pbsim_swap
    .type pbsim_swap, @function
pbsim_swap:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
    .size pbsim_swap, .-pbsim_swap
)");
#define PBSIM_FAST_SWITCH 1
#endif

namespace pbsim {

Block *g_block = nullptr;

void poison_shared(void *p, size_t bytes) {
    static std::vector<std::pair<void *, unsigned long long>> seen;      // (array, epoch of its last poisoning)
    for (auto &e : seen)
        if (e.first == p) {
            if (e.second == g_block->epoch) return;
            e.second = g_block->epoch;
            memset(p, 0xA5, bytes);
            return;
        }
    seen.emplace_back(p, g_block->epoch);
    memset(p, 0xA5, bytes);
}

static inline void to_scheduler(Fiber *f) {
#ifdef PBSIM_FAST_SWITCH
    pbsim_swap(&f->sp, g_block->sched_sp);
#else
    swapcontext(&f->ctx, &g_block->sched);
#endif
}

unsigned long long collective(Op op, unsigned mask, unsigned long long val, int arg, int width) {
    Fiber *f = g_block->cur;
    f->op = op; f->mask = mask; f->val = val; f->arg = arg; f->width = width; f->waiting = true; f->n_collectives++;
    to_scheduler(f);
    return f->result;
}

static void fiber_entry() {
    g_block->body();
    g_block->cur->done = true;
#ifdef PBSIM_FAST_SWITCH
    to_scheduler(g_block->cur);           // never resumed
    abort();
#endif
}

// complete every collective all of whose (live) participants have arrived; returns whether anything was released
static bool resolve(Block &B) {
    bool released = false;
    const int n = (int)B.fibers.size();
    // block-wide barrier
    {
        bool any = false, all = true;
        for (auto &f : B.fibers) {
            if (f.done) continue;
            if (f.waiting && f.op == OP_SYNCTHREADS) any = true; else all = false;
        }
        if (any && all) {
            for (auto &f : B.fibers) if (!f.done) { f.waiting = false; f.op = OP_NONE; }
            return true;
        }
    }
    for (int w0 = 0; w0 < n; w0 += 32) {
        const int wn = std::min(32, n - w0);
        for (int l = 0; l < wn; ++l) {
            Fiber &f = B.fibers[w0 + l];
            if (f.done || !f.waiting || f.op == OP_SYNCTHREADS) continue;
            const unsigned m = f.mask;
            const Op op = f.op;                  // (f itself is reset in the release loop below)
            bool ready = true;
            for (int k = 0; k < wn && ready; ++k) {
                if (!((m >> k) & 1u)) continue;
                Fiber &o = B.fibers[w0 + k];
                if (o.done) continue;
                if (!o.waiting || o.op != op || o.mask != m) ready = false;
            }
            if (!ready) continue;
            // gather inputs first (results must not depend on the release order)
            unsigned long long in[32]; bool part[32];
            for (int k = 0; k < wn; ++k) {
                part[k] = ((m >> k) & 1u) && !B.fibers[w0 + k].done;
                in[k] = part[k] ? B.fibers[w0 + k].val : 0ull;
            }
            long long red = 0; bool first = true; int allv = 1;
            for (int k = 0; k < wn; ++k) if (part[k]) {
                const long long v = (long long)in[k];
                if (op == OP_REDUCE_MAX) red = first ? v : std::max(red, v);
                if (op == OP_REDUCE_MIN) red = first ? v : std::min(red, v);
                if (!in[k]) allv = 0;
                first = false;
            }
            for (int k = 0; k < wn; ++k) if (part[k]) {
                Fiber &o = B.fibers[w0 + k];
                const int wd = o.width > 0 ? o.width : 32;
                const int seg = (k / wd) * wd;
                unsigned long long r = in[k];
                switch (op) {
                    case OP_SHFL_UP: { const int s = k - o.arg; if (s >= seg && part[s]) r = in[s]; break; }
                    case OP_SHFL_IDX: { const int s = seg + (((o.arg % wd) + wd) % wd); if (s < wn && part[s]) r = in[s]; break; }
                    case OP_SHFL_XOR: { const int s = k ^ o.arg; if (s >= seg && s < seg + wd && s < wn && part[s]) r = in[s]; break; }
                    case OP_REDUCE_MAX: case OP_REDUCE_MIN: r = (unsigned long long)red; break;
                    case OP_ALL: r = (unsigned long long)allv; break;
                    default: r = 0; break;
                }
                o.result = r; o.waiting = false; o.op = OP_NONE;
            }
            released = true;
        }
    }
    return released;
}

void run_grid(dim3 grid, dim3 block, size_t smem, const std::function<void()> &body) {
    const size_t STACK = 256 * 1024;
    static std::vector<char *> pool;                      // fiber stacks, allocated once and reused by every launch
    Block B;
    B.bdim = block; B.gdim = grid; B.body = body;
    B.dyn_smem.assign(smem / 4 + 64, 0xDEADBEEFu);          // dynamic shared memory is NOT zero-initialised on the device
    const int nthreads = (int)(block.x * block.y * block.z);
    Block *outer = g_block;
    g_block = &B;
    for (unsigned b = 0; b < grid.x; ++b) {
        B.bid = dim3(b, 0, 0);
        static unsigned long long epoch_counter = 0;
        B.epoch = ++epoch_counter;
        std::fill(B.dyn_smem.begin(), B.dyn_smem.end(), 0xDEADBEEFu);
        B.fibers.clear();
        B.fibers.resize((size_t)nthreads);
        for (int t = 0; t < nthreads; ++t) {
            Fiber &f = B.fibers[(size_t)t];
            f.tid = dim3((unsigned)t, 0, 0);
            while (pool.size() <= (size_t)t) pool.push_back((char *)malloc(STACK));
#ifdef PBSIM_FAST_SWITCH
            {
                void **sp = reinterpret_cast<void **>(reinterpret_cast<uintptr_t>(pool[(size_t)t] + STACK) & ~(uintptr_t)15);
                *--sp = nullptr;                                   // keeps the ABI's stack alignment at fiber_entry
                *--sp = reinterpret_cast<void *>(&fiber_entry);    // `ret` target of the first switch
                for (int r = 0; r < 6; ++r) *--sp = nullptr;       // rbp rbx r12 r13 r14 r15
                f.sp = sp;
            }
#else
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = pool[(size_t)t];
            f.ctx.uc_stack.ss_size = STACK;
            f.ctx.uc_link = &B.sched;
            makecontext(&f.ctx, fiber_entry, 0);
#endif
        }
        // Lane interleaving between two collectives is not defined on the device (independent thread scheduling): the order
        // in which runnable fibers are resumed can be reversed or shuffled (PBSIM_ORDER=reverse | random[:seed]) -- code that
        // relies on one particular interleaving, e.g. a missing __syncwarp around shared memory, then changes its results.
        static const char *order_env = getenv("PBSIM_ORDER");
        static unsigned long long rng = (order_env && strchr(order_env, ':')) ? strtoull(strchr(order_env, ':') + 1, nullptr, 10) * 2654435761ull + 1 : 88172645463325252ull;
        std::vector<int> order((size_t)nthreads);
        for (int t = 0; t < nthreads; ++t) order[(size_t)t] = t;
        if (order_env && !strncmp(order_env, "reverse", 7)) std::reverse(order.begin(), order.end());
        for (;;) {
            bool progress = false, alive = false;
            if (order_env && !strncmp(order_env, "random", 6))
                for (int t = nthreads - 1; t > 0; --t) {
                    rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
                    std::swap(order[(size_t)t], order[(size_t)(rng % (unsigned long long)(t + 1))]);
                }
            for (int oi = 0; oi < nthreads; ++oi) {
                Fiber &f = B.fibers[(size_t)order[(size_t)oi]];
                if (f.done) continue;
                alive = true;
                if (f.waiting) continue;
                B.cur = &f;
#ifdef PBSIM_FAST_SWITCH
                pbsim_swap(&B.sched_sp, f.sp);
#else
                swapcontext(&B.sched, &f.ctx);
#endif
                progress = true;
            }
            if (!alive) break;
            if (resolve(B)) progress = true;
            if (!progress) {
                fprintf(stderr, "pbsim: deadlock in block %u -- a collective is waiting for lanes that never arrive\n", b);
                for (size_t t = 0; t < B.fibers.size(); ++t) {
                    const Fiber &f = B.fibers[t];
                    fprintf(stderr, "  thread %3zu: %s op=%d mask=%08x arg=%d width=%d ncoll=%ld\n", t, f.done ? "done" : f.waiting ? "waiting" : "runnable", (int)f.op, f.mask, f.arg, f.width, f.n_collectives);
                }
                abort();
            }
        }
    }
    g_block = outer;
}

}  // namespace pbsim

// ---- stream ordering: vector clocks, accesses, races (see pbsim_cuda.h) ---------------------------------------------
namespace pbsim {
namespace {

typedef std::vector<unsigned> VC;
void join(VC &a, const VC &b) {
    if (a.size() < b.size()) a.resize(b.size(), 0);
    for (size_t i = 0; i < b.size(); ++i) a[i] = std::max(a[i], b[i]);
}
unsigned at(const VC &v, int i) { return (size_t)i < v.size() ? v[(size_t)i] : 0; }

struct StreamObj { int id; bool blocking; };
struct EventObj { VC clock; };
struct Access {
    size_t lo, hi;                  // byte range inside the allocation
    Acc kind;
    int stream; unsigned epoch;     // the operation: its stream and that stream's clock component
    std::shared_ptr<const std::string> op;
    std::string what;
};
struct Alloc { size_t size; std::vector<Access> acc; };

std::mutex mu;
std::vector<VC> streams(1);         // [0] = the legacy default stream
std::vector<bool> blocking(1, true);
VC host;
std::map<uintptr_t, Alloc> allocs;
std::set<std::string> races;
long long n_races = 0;
thread_local int cur_stream = -1;
thread_local VC cur_clock;
thread_local std::shared_ptr<const std::string> cur_op;

const char *kind_name(Acc k) { return k == ACC_READ ? "read" : k == ACC_WRITE ? "write" : "atomic"; }

int stream_id(void *s) {            // NULL, cudaStreamLegacy and cudaStreamPerThread are the legacy stream here
    if (s == nullptr || s == (void *)0x1 || s == (void *)0x2) return 0;
    return static_cast<StreamObj *>(s)->id;
}

}  // namespace

void *hb_stream_create(bool is_blocking) {
    std::lock_guard<std::mutex> lk(mu);
    StreamObj *o = new StreamObj{(int)streams.size(), is_blocking};
    streams.emplace_back();
    blocking.push_back(is_blocking);
    return o;
}
void hb_stream_destroy(void *s) { (void)s; }   // ids stay valid: accesses of the stream may still be checked against

void hb_op_begin(void *s, const std::string &what) {
    std::lock_guard<std::mutex> lk(mu);
    const int id = stream_id(s);
    VC &c = streams[(size_t)id];
    join(c, host);
    if (id == 0) { for (size_t k = 1; k < streams.size(); ++k) if (blocking[k]) join(c, streams[k]); }
    else if (blocking[(size_t)id]) join(c, streams[0]);
    if (c.size() <= (size_t)id) c.resize((size_t)id + 1, 0);
    c[(size_t)id]++;
    cur_stream = id;
    cur_clock = c;
    cur_op = std::make_shared<const std::string>(what + " [stream " + std::to_string(id) + "]");
}
void hb_op_end() { cur_stream = -1; cur_op.reset(); }

void hb_access(const void *p, size_t bytes, Acc kind, const std::string &what) {
    if (cur_stream < 0 || p == nullptr) return;
    std::lock_guard<std::mutex> lk(mu);
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    auto it = allocs.upper_bound(a);
    if (it == allocs.begin()) return;
    --it;
    Alloc &A = it->second;
    if (a >= it->first + A.size) return;            // not device memory of this library (host memory, caller's buffers)
    const size_t lo = a - it->first;
    const size_t hi = bytes == 0 ? lo + 1 : bytes == (size_t)-1 || bytes > A.size - lo ? A.size : lo + bytes;
    // accesses the host has synchronised with happen before every later operation: drop them
    A.acc.erase(std::remove_if(A.acc.begin(), A.acc.end(), [](const Access &x) { return at(host, x.stream) >= x.epoch; }),
                A.acc.end());
    for (const Access &x : A.acc) {
        if (x.stream == cur_stream || at(cur_clock, x.stream) >= x.epoch) continue;      // ordered
        if (x.hi <= lo || hi <= x.lo) continue;
        if (x.kind == ACC_READ && kind == ACC_READ) continue;
        if (x.kind == ACC_ATOMIC && kind == ACC_ATOMIC) continue;
        ++n_races;
        races.insert("race on a " + std::to_string(A.size) + "-byte allocation, bytes [" + std::to_string(std::max(lo, x.lo)) +
                     ", " + std::to_string(std::min(hi, x.hi)) + "):\n  " + kind_name(x.kind) + " of " + x.what + " by " + *x.op +
                     "\n  " + kind_name(kind) + " of " + what + " by " + *cur_op);
    }
    A.acc.push_back(Access{lo, hi, kind, cur_stream, at(cur_clock, cur_stream), cur_op, what});
}

void hb_malloc(void *p, size_t n) {
    std::lock_guard<std::mutex> lk(mu);
    allocs[reinterpret_cast<uintptr_t>(p)] = Alloc{n, {}};
}
void hb_sync_device() {
    std::lock_guard<std::mutex> lk(mu);
    for (const VC &c : streams) join(host, c);
}
void hb_free(void *p) {
    hb_sync_device();                                // cudaFree synchronises the device
    std::lock_guard<std::mutex> lk(mu);
    allocs.erase(reinterpret_cast<uintptr_t>(p));
}
void hb_sync_stream(void *s) {
    std::lock_guard<std::mutex> lk(mu);
    const int id = stream_id(s);
    join(host, streams[(size_t)id]);
    if (id == 0) for (size_t k = 1; k < streams.size(); ++k) if (blocking[k]) join(host, streams[k]);
}
void *hb_event_create() { return new EventObj(); }
void hb_event_destroy(void *e) { delete static_cast<EventObj *>(e); }
void hb_event_record(void *e, void *s) {
    if (!e) return;
    hb_op_begin(s, "cudaEventRecord");
    hb_op_end();
    std::lock_guard<std::mutex> lk(mu);
    static_cast<EventObj *>(e)->clock = streams[(size_t)stream_id(s)];
}
void hb_event_sync(void *e) {
    if (!e) return;
    std::lock_guard<std::mutex> lk(mu);
    join(host, static_cast<EventObj *>(e)->clock);
}
void hb_stream_wait(void *s, void *e) {
    if (!e) return;
    std::lock_guard<std::mutex> lk(mu);
    join(streams[(size_t)stream_id(s)], static_cast<EventObj *>(e)->clock);
}

std::string site_arg(const Site &s, int idx) {
    const char *p = s.args;
    for (int k = 0; k < idx && p; ++k) { p = strchr(p, '\037'); if (p) ++p; }
    if (!p) return std::string(s.kernel) + " arg " + std::to_string(idx);
    const char *e = strchr(p, '\037');
    return std::string(s.kernel) + " arg `" + std::string(p, e ? (size_t)(e - p) : strlen(p)) + "`";
}

}  // namespace pbsim

extern "C" {
// a blocking stream (cudaStreamCreate) for tests that call the engine on streams of their own
void *pbsim_stream_create(void) { return pbsim::hb_stream_create(true); }
// "device" memory the check tracks, and an upload into it on a stream: a test's reads and records then take part in it
void *pbsim_device_alloc(long long n) { void *p = nullptr; return cudaMalloc(&p, (size_t)n) == cudaSuccess ? p : nullptr; }
void pbsim_device_free(void *p) { cudaFree(p); }
void pbsim_upload(void *dst, const void *src, long long n, void *stream) {
    cudaMemcpyAsync(dst, src, (size_t)n, cudaMemcpyHostToDevice, (cudaStream_t)stream);
}
long long pbsim_race_count(void) { std::lock_guard<std::mutex> lk(pbsim::mu); return pbsim::n_races; }
void pbsim_race_clear(void) { std::lock_guard<std::mutex> lk(pbsim::mu); pbsim::n_races = 0; pbsim::races.clear(); }
// the distinct races found since the last clear, one paragraph each; returns the length of the whole text (buf may be NULL)
long long pbsim_race_report(char *buf, long long cap) {
    std::lock_guard<std::mutex> lk(pbsim::mu);
    std::string t;
    for (const std::string &r : pbsim::races) t += r + "\n";
    if (buf && cap > 0) { const size_t n = std::min((size_t)cap - 1, t.size()); memcpy(buf, t.data(), n); buf[n] = 0; }
    return (long long)t.size();
}
}
