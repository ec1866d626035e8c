// tests/sim/pbsim_cuda.h -- a host stand-in for <cuda_runtime.h> + the CUDA execution model, for TESTS ONLY.
//
// tests/sim/build_sim.py rewrites the product's engine.cu / kernels.cuh (kernel launches `k<<<g, b, s, st>>>(args)` become
// pbsim::launch(k, g, b, s, st, args), <cuda_runtime.h> becomes this header) and compiles the result with g++ into
// tests/sim/_build/libengine_sim.so.  The kernels then run on the CPU exactly as written: every CUDA thread of a block is a
// fiber (ucontext), warp collectives (__shfl_*_sync, __reduce_*_sync, __all_sync, __syncwarp, __syncthreads) are rendezvous
// points of the fibers they name, blocks run one after the other, streams are synchronous.  This is how the no-GPU tier
// checks the kernels' ORCHESTRATION (chunking, staging rings, slot refill, trace addressing, launch sequences of the host
// engine) and not only the arithmetic of dp_core.cuh.  It is slow (about 10^4 alignments/s) and is not a fallback: nothing
// in porechop_b200/ builds, loads or references it.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <functional>
#include <map>
#include <string>
#include <type_traits>
#include <vector>

// ---- vector types / qualifiers ---------------------------------------------------------------------------
struct uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(16) int4 { int x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 v; v.x = x; v.y = y; v.z = z; v.w = w; return v; }
inline uint2 make_uint2(unsigned x, unsigned y) { uint2 v; v.x = x; v.y = y; return v; }
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

// ---- runtime API (synchronous, one "device") --------------------------------------------------------------
typedef int cudaError_t;
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind { cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
enum { cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0, cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { int major, minor, multiProcessorCount; size_t sharedMemPerBlockOptin; };
inline const char *cudaGetErrorString(cudaError_t) { return "simulated CUDA error"; }
// launch-configuration errors are reported the CUDA way: the launch does nothing and cudaGetLastError() returns the error once
inline cudaError_t &pbsim_last_error() { static thread_local cudaError_t e = cudaSuccess; return e; }
inline cudaError_t cudaGetLastError() { cudaError_t e = pbsim_last_error(); pbsim_last_error() = cudaSuccess; return e; }
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) {
    p->major = 9; p->minor = 0;
    p->multiProcessorCount = getenv("PBSIM_SMS") ? atoi(getenv("PBSIM_SMS")) : 2;   // small grids: the grid-stride loops really loop
    p->sharedMemPerBlockOptin = 227 * 1024;
    return cudaSuccess;
}
// ---- stream ordering: happens-before checking (pbsim.cpp) -----------------------------------------------------
// Streams still execute synchronously, but every stream operation also gets the vector clock that CUDA guarantees for it:
// join(its stream's clock, the host's clock) -- plus, on the legacy stream and on blocking streams, the implicit
// synchronisation between the two -- and then a tick of its stream's own component.  cudaEventRecord captures a stream's
// clock and cudaStreamWaitEvent joins it into another stream; the synchronise calls (and cudaFree, which synchronises the
// device) join stream clocks into the host's.  Each operation's accesses to cudaMalloc'd memory are recorded, and two
// accesses of different streams to overlapping bytes race when neither operation happens before the other and at least one
// writes.  Atomics (64-bit counters, append slots) race only with plain accesses.  pbsim_race_count / _report / _clear
// (extern "C") expose the races found.
namespace pbsim {
enum Acc { ACC_READ = 0, ACC_WRITE = 1, ACC_ATOMIC = 2 };
void hb_op_begin(void *stream, const std::string &what);   // one operation of `stream`: its accesses follow, then hb_op_end
void hb_access(const void *p, size_t bytes, Acc kind, const std::string &what);   // bytes = 0: the address p itself
void hb_op_end();
void hb_malloc(void *p, size_t n);
void hb_free(void *p);
void hb_sync_stream(void *stream);
void hb_sync_device();
void *hb_stream_create(bool blocking);
void hb_stream_destroy(void *stream);
void *hb_event_create();
void hb_event_destroy(void *event);
void hb_event_record(void *event, void *stream);
void hb_event_sync(void *event);
void hb_stream_wait(void *stream, void *event);
}  // namespace pbsim
#define cudaStreamLegacy ((cudaStream_t)0x1)
#define cudaStreamPerThread ((cudaStream_t)0x2)
inline cudaError_t cudaMalloc(void **p, size_t n) {
    *p = malloc(n ? n : 1);
    if (*p) pbsim::hb_malloc(*p, n ? n : 1);
    return *p ? cudaSuccess : 2;
}
template <class T> inline cudaError_t cudaMalloc(T **p, size_t n) { return cudaMalloc(reinterpret_cast<void **>(p), n); }
inline cudaError_t cudaFree(void *p) { pbsim::hb_free(p); free(p); return cudaSuccess; }     // synchronises the device
inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : 2; }
inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
// the copy / memset calls are macros so that a race report can quote the call's arguments and line
inline cudaError_t pbsim_memcpy_async(const char *args, const char *fn, int line, void *d, const void *s, size_t n, cudaMemcpyKind,
                                      cudaStream_t st = nullptr) {
    const std::string what = std::string("cudaMemcpyAsync(") + args + ") in " + fn + "(), line " + std::to_string(line);
    pbsim::hb_op_begin(st, what);
    pbsim::hb_access(s, n, pbsim::ACC_READ, "source");
    pbsim::hb_access(d, n, pbsim::ACC_WRITE, "destination");
    pbsim::hb_op_end();
    memcpy(d, s, n);
    return cudaSuccess;
}
inline cudaError_t pbsim_memset_async(const char *args, const char *fn, int line, void *d, int v, size_t n, cudaStream_t st = nullptr) {
    pbsim::hb_op_begin(st, std::string("cudaMemsetAsync(") + args + ") in " + fn + "(), line " + std::to_string(line));
    pbsim::hb_access(d, n, pbsim::ACC_WRITE, "destination");
    pbsim::hb_op_end();
    memset(d, v, n);
    return cudaSuccess;
}
#define cudaMemcpyAsync(...) pbsim_memcpy_async(#__VA_ARGS__, __func__, __LINE__, __VA_ARGS__)
#define cudaMemsetAsync(...) pbsim_memset_async(#__VA_ARGS__, __func__, __LINE__, __VA_ARGS__)
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned flags) { *s = pbsim::hb_stream_create(!(flags & 1u)); return cudaSuccess; }
inline cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = pbsim::hb_stream_create(true); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t s) { pbsim::hb_stream_destroy(s); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t s) { pbsim::hb_sync_stream(s); return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { pbsim::hb_sync_device(); return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = pbsim::hb_event_create(); return cudaSuccess; }
#define cudaEventDisableTiming 2u
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = pbsim::hb_event_create(); return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s = nullptr) { pbsim::hb_event_record(e, s); return cudaSuccess; }
inline cudaError_t cudaEventSynchronize(cudaEvent_t e) { pbsim::hb_event_sync(e); return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned = 0) { pbsim::hb_stream_wait(s, e); return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t e) { pbsim::hb_event_destroy(e); return cudaSuccess; }
// cudaFuncAttributeMaxDynamicSharedMemorySize is a property of the KERNEL (last value set wins); a launch asking for more
// dynamic shared memory than the attribute (48 KB if never set) fails with "invalid argument" on the device -- reproduced here
// (round 2: a per-size cache of the attribute call let a later, smaller value stand while a larger launch followed).
inline std::map<const void *, size_t> &pbsim_smem_attr() { static std::map<const void *, size_t> m; return m; }
template <class F> inline cudaError_t cudaFuncSetAttribute(F f, int, int v) {
    pbsim_smem_attr()[reinterpret_cast<const void *>(f)] = (size_t)v;
    return cudaSuccess;
}
template <class F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) {
    *n = getenv("PBSIM_BLOCKS_PER_SM") ? atoi(getenv("PBSIM_BLOCKS_PER_SM")) : 2;
    return cudaSuccess;
}

// ---- the block scheduler: one fiber per CUDA thread ---------------------------------------------------------
namespace pbsim {

enum Op { OP_NONE, OP_SHFL_UP, OP_SHFL_IDX, OP_SHFL_XOR, OP_REDUCE_MAX, OP_REDUCE_MIN, OP_ALL, OP_SYNCWARP, OP_SYNCTHREADS };

struct Fiber {
    ucontext_t ctx;                 // portable context switch (other architectures)
    void *sp = nullptr;             // x86-64: saved stack pointer of the hand-written switch (no sigprocmask syscalls)
    dim3 tid;
    bool done = false;
    // pending collective
    Op op = OP_NONE;
    unsigned mask = 0;
    unsigned long long val = 0, result = 0;
    int arg = 0, width = 32;
    bool waiting = false;
    long n_collectives = 0;
};

struct Block {
    std::vector<Fiber> fibers;
    ucontext_t sched;
    void *sched_sp = nullptr;
    Fiber *cur = nullptr;
    dim3 bid, bdim, gdim;
    std::function<void()> body;
    std::vector<uint32_t> dyn_smem;
    unsigned long long epoch = 0;           // one per block: static shared arrays are poisoned once per epoch
};
extern Block *g_block;

inline uint32_t *dynamic_smem() { return g_block->dyn_smem.data(); }
// static __shared__ arrays are function-local statics here; the first thread of every block that reaches the declaration
// fills the array with a poison pattern -- shared memory has no defined initial contents on the device
void poison_shared(void *p, size_t bytes);

// a fiber calls this at every collective: park, let the scheduler run the others, return the collective's result
unsigned long long collective(Op op, unsigned mask, unsigned long long val, int arg, int width);
void run_grid(dim3 grid, dim3 block, size_t smem, const std::function<void()> &body);

// A launch site, filled in by build_sim.py: kernel name, its argument expressions (separated by \037), function and line.
struct Site { const char *kernel, *args, *func; int line; };
std::string site_arg(const Site &s, int idx);        // "kernel arg `expr`"

// Kernel arguments as accesses: a `const T *` argument is a read and a `T *` argument a write of the data at the address it
// points to (a kernel's extent is not known here: two launches handed the same buffer conflict, launches handed disjoint
// pieces of one buffer do not); `unsigned long long *` arguments are the 64-bit atomic counters.  Pointers inside by-value
// struct arguments are classified by pbsim_fields() -- overloads for the kernels' argument structs are in pbsim_fields.h.
template <class T> inline void pbsim_fields(const T &, const std::string &) {}
template <class T> inline void classify_arg(const T &v, const Site &s, int idx) {
    if constexpr (std::is_pointer<T>::value) {
        using P = typename std::remove_pointer<T>::type;
        if (!v) return;
        const Acc k = std::is_const<P>::value ? ACC_READ
                    : std::is_same<typename std::remove_cv<P>::type, unsigned long long>::value ? ACC_ATOMIC : ACC_WRITE;
        hb_access(reinterpret_cast<const void *>(v), 0, k, site_arg(s, idx));
    } else {
        pbsim_fields(v, site_arg(s, idx));
    }
}

template <class F, class... Args>
inline void launch(const Site &site, F f, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    {   // the kernel's dynamic shared-memory limit: 48 KB unless the attribute was set -- then exactly that value
        auto it = pbsim_smem_attr().find(reinterpret_cast<const void *>(f));
        const size_t limit = it == pbsim_smem_attr().end() ? (size_t)48 * 1024 : it->second;
        if (smem > limit) { pbsim_last_error() = cudaErrorInvalidValue; return; }
    }
    hb_op_begin(stream, std::string(site.kernel) + "<<<>>> in " + site.func + "(), line " + std::to_string(site.line));
    int idx = 0;
    (classify_arg(args, site, idx++), ...);
    hb_op_end();
    run_grid(grid, block, smem, [=]() { f(args...); });
}

}  // namespace pbsim

#define threadIdx (pbsim::g_block->cur->tid)
#define blockIdx (pbsim::g_block->bid)
#define blockDim (pbsim::g_block->bdim)
#define gridDim (pbsim::g_block->gdim)

// ---- device intrinsics --------------------------------------------------------------------------------------
template <class T> inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    static_assert(sizeof(T) <= 8, "shuffle of up to 64 bits");
    unsigned long long raw = 0; memcpy(&raw, &v, sizeof(T));
    raw = pbsim::collective(pbsim::OP_SHFL_UP, mask, raw, (int)delta, width);
    T r; memcpy(&r, &raw, sizeof(T)); return r;
}
template <class T> inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    unsigned long long raw = 0; memcpy(&raw, &v, sizeof(T));
    raw = pbsim::collective(pbsim::OP_SHFL_IDX, mask, raw, src, width);
    T r; memcpy(&r, &raw, sizeof(T)); return r;
}
template <class T> inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    unsigned long long raw = 0; memcpy(&raw, &v, sizeof(T));
    raw = pbsim::collective(pbsim::OP_SHFL_XOR, mask, raw, lanemask, width);
    T r; memcpy(&r, &raw, sizeof(T)); return r;
}
inline int __reduce_max_sync(unsigned mask, int v) { return (int)(long long)pbsim::collective(pbsim::OP_REDUCE_MAX, mask, (unsigned long long)(long long)v, 0, 32); }
inline int __reduce_min_sync(unsigned mask, int v) { return (int)(long long)pbsim::collective(pbsim::OP_REDUCE_MIN, mask, (unsigned long long)(long long)v, 0, 32); }
inline int __all_sync(unsigned mask, int pred) { return (int)pbsim::collective(pbsim::OP_ALL, mask, pred ? 1 : 0, 0, 32); }
inline void __syncwarp(unsigned mask = 0xffffffffu) { pbsim::collective(pbsim::OP_SYNCWARP, mask, 0, 0, 32); }
inline void __syncthreads() { pbsim::collective(pbsim::OP_SYNCTHREADS, 0xffffffffu, 0, 0, 32); }

template <class T> inline T __ldg(const T *p) { return *p; }
template <class T> inline T __ldcs(const T *p) { return *p; }
template <class T> inline void __stcs(T *p, T v) { *p = v; }
inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
    const unsigned long long xy = ((unsigned long long)y << 32) | x;
    unsigned r = 0;
    for (int i = 0; i < 4; ++i) r |= (unsigned)((xy >> (8 * ((s >> (4 * i)) & 7))) & 0xFF) << (8 * i);
    return r;
}
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) {
    const unsigned long long v = ((unsigned long long)hi << 32) | lo;
    return (unsigned)(v >> (sh & 31));
}
inline unsigned long long atomicAdd(unsigned long long *p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
inline unsigned atomicAdd(unsigned *p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
inline unsigned long long atomicMax(unsigned long long *p, unsigned long long v) { unsigned long long o = *p; if (v > o) *p = v; return o; }
inline int atomicOr(int *p, int v) { int o = *p; *p = o | v; return o; }
using std::max;
using std::min;
