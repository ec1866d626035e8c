// porechop_b200/csrc/hostpack.cpp -- host half of the packed upload path of cpp_functions.so (option "h2d_pack").
//
// The sequences cross the reference's ABI as ASCII, one byte per base (porechop/src/adapter_align.cpp:15-16 turns them
// into Dna5 codes first thing: seqan/basic/alphabet_residue_tabs.h:113-140).  The end-to-end path of the engine is bound
// by those bytes crossing PCIe, not by the kernels (DESIGN.md section 6), so this file does the Dna5 conversion on the
// host cores instead and packs two 4-bit codes per byte: half the bytes over the link, and the device unpacks
// (kernels.cuh unpack_kernel) into exactly the code bytes encode_kernel would have produced.
//
// Plain C++ (g++), linked into cpp_functions.so by build.py; AVX-512BW / AVX2 body selected at run time, scalar table otherwise;
// its own sleeping thread team (no OpenMP: see PackTeam).
// No alignment arithmetic here -- only the alphabet conversion.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <stdio.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <vector>

#if defined(__x86_64__)
#include <immintrin.h>
#endif

namespace {

// same mapping as pb::encode_byte (dp_core.cuh): A/a=0 C/c=1 G/g=2 T/t/U/u=3, every other byte = 4
struct CodeTable {
    uint8_t t[256];
    CodeTable() {
        memset(t, 4, sizeof t);
        t[(int)'A'] = t[(int)'a'] = 0; t[(int)'C'] = t[(int)'c'] = 1; t[(int)'G'] = t[(int)'g'] = 2;
        t[(int)'T'] = t[(int)'t'] = t[(int)'U'] = t[(int)'u'] = 3;
    }
};
const CodeTable g_tab;

// bytes [i0, i1) of `in` -> nibbles; i0 is even, so every output byte belongs to exactly one caller
void pack_scalar(const uint8_t *in, int64_t i0, int64_t i1, int64_t n, uint8_t *out) {
    int64_t i = i0;
    for (; i + 1 < i1; i += 2) out[i >> 1] = (uint8_t)(g_tab.t[in[i]] | (g_tab.t[in[i + 1]] << 4));
    if (i < i1) out[i >> 1] = (uint8_t)(g_tab.t[in[i]] | ((i + 1 < n ? g_tab.t[in[i + 1]] : 0) << 4));
}

#if defined(__x86_64__)
__attribute__((target("avx2"))) void pack_avx2(const uint8_t *in, int64_t i0, int64_t i1, int64_t n, uint8_t *out) {
    // per 128-bit lane tables indexed by the low nibble of the case-folded byte: the letter that nibble must be,
    // and its code ('A' 0x41, 'C' 0x43, 'T' 0x54, 'U' 0x55, 'G' 0x47)
    const __m256i tchar = _mm256_setr_epi8((char)0xFF, 0x41, (char)0xFF, 0x43, 0x54, 0x55, (char)0xFF, 0x47, (char)0xFF, (char)0xFF,
                                           (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF,
                                           (char)0xFF, 0x41, (char)0xFF, 0x43, 0x54, 0x55, (char)0xFF, 0x47, (char)0xFF, (char)0xFF,
                                           (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF);
    const __m256i tcode = _mm256_setr_epi8(4, 0, 4, 1, 3, 3, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4, 4, 0, 4, 1, 3, 3, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4);
    const __m256i fold = _mm256_set1_epi8((char)0xDF), lo4 = _mm256_set1_epi8(0x0F), four = _mm256_set1_epi8(4);
    const __m256i w = _mm256_set1_epi16(0x1001);      // bytes (1, 16): even code + 16 * odd code
    const __m256i zero = _mm256_setzero_si256();
    int64_t i = i0;
    for (; i + 32 <= i1; i += 32) {
        const __m256i x = _mm256_loadu_si256(reinterpret_cast<const __m256i *>(in + i));
        const __m256i f = _mm256_and_si256(x, fold);
        const __m256i nib = _mm256_and_si256(f, lo4);
        const __m256i ok = _mm256_cmpeq_epi8(_mm256_shuffle_epi8(tchar, nib), f);
        const __m256i code = _mm256_blendv_epi8(four, _mm256_shuffle_epi8(tcode, nib), ok);
        const __m256i pr = _mm256_maddubs_epi16(code, w);                 // 16 x (c0 + 16*c1)
        const __m256i pk = _mm256_permute4x64_epi64(_mm256_packus_epi16(pr, zero), 0x08);
        _mm_storeu_si128(reinterpret_cast<__m128i *>(out + (i >> 1)), _mm256_castsi256_si128(pk));
    }
    if (i < i1) pack_scalar(in, i, i1, n, out);
}
bool have_avx2() {
    static const bool v = __builtin_cpu_supports("avx2");
    return v;
}
// the same conversion 64 bases at a time (AVX-512BW: byte shuffles per 128-bit lane, compare into a mask, vpmovwb)
__attribute__((target("avx512f,avx512bw"))) void pack_avx512(const uint8_t *in, int64_t i0, int64_t i1, int64_t n, uint8_t *out) {
    const __m512i tchar = _mm512_broadcast_i32x4(_mm_setr_epi8((char)0xFF, 0x41, (char)0xFF, 0x43, 0x54, 0x55, (char)0xFF, 0x47, (char)0xFF,
                                                               (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF, (char)0xFF));
    const __m512i tcode = _mm512_broadcast_i32x4(_mm_setr_epi8(4, 0, 4, 1, 3, 3, 4, 2, 4, 4, 4, 4, 4, 4, 4, 4));
    const __m512i fold = _mm512_set1_epi8((char)0xDF), lo4 = _mm512_set1_epi8(0x0F), four = _mm512_set1_epi8(4);
    const __m512i w = _mm512_set1_epi16(0x1001);
    int64_t i = i0;
    // the packed bytes are only read back by the DMA engine: non-temporal stores skip the read-for-ownership of the output
    // lines (a third of the loop's memory traffic) when the destination is 32-byte aligned (the engine's pinned buffers are)
    static const bool want_stream = getenv("PB200_PACK_NT") && atoi(getenv("PB200_PACK_NT")) != 0;   // A/B switch, default off
    const bool stream = want_stream && ((reinterpret_cast<uintptr_t>(out) + (uintptr_t)(i0 >> 1)) & 31) == 0;
    for (; i + 64 <= i1; i += 64) {
        const __m512i x = _mm512_loadu_si512(reinterpret_cast<const void *>(in + i));
        const __m512i f = _mm512_and_si512(x, fold);
        const __m512i nib = _mm512_and_si512(f, lo4);
        const __mmask64 ok = _mm512_cmpeq_epi8_mask(_mm512_shuffle_epi8(tchar, nib), f);
        const __m512i code = _mm512_mask_blend_epi8(ok, four, _mm512_shuffle_epi8(tcode, nib));
        const __m512i pr = _mm512_maddubs_epi16(code, w);                  // 32 x (c0 + 16*c1)
        if (stream) _mm256_stream_si256(reinterpret_cast<__m256i *>(out + (i >> 1)), _mm512_cvtepi16_epi8(pr));
        else _mm256_storeu_si256(reinterpret_cast<__m256i *>(out + (i >> 1)), _mm512_cvtepi16_epi8(pr));
    }
    if (stream) _mm_sfence();
    if (i < i1) pack_avx2(in, i, i1, n, out);
}
bool have_avx512() {
    static const bool v = __builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw") && !getenv("PB200_PACK_NO_AVX512");
    return v;
}
#endif

void pack_range(const uint8_t *in, int64_t i0, int64_t i1, int64_t n, uint8_t *out) {
#if defined(__x86_64__)
    if (have_avx512()) { pack_avx512(in, i0, i1, n, out); return; }
    if (have_avx2()) { pack_avx2(in, i0, i1, n, out); return; }
#endif
    pack_scalar(in, i0, i1, n, out);
}

// A small persistent team for the packer.  Under OpenMP the team's idle threads spin after every parallel region; inside a
// cgroup CPU quota smaller than the host's hardware threads a spinning team eats the quota and the whole process gets
// throttled.  These workers sleep on a condition
// variable between calls and take 64-KB blocks from a shared counter while a call runs.
class PackTeam {
    std::vector<std::thread> workers;
    std::mutex mu;
    std::condition_variable cv_work, cv_done;
    std::mutex call_mu;                      // one pack call at a time (concurrent callers take turns)
    const uint8_t *in = nullptr; uint8_t *out = nullptr;
    int64_t n = 0, nblk = 0;
    std::atomic<int64_t> next{0};
    int use = 0, pending = 0;
    std::atomic<uint64_t> gen{0};
    static constexpr int64_t BLK = 1 << 16;  // bytes per work item (even)

    void blocks() {
        for (;;) {
            const int64_t b = next.fetch_add(1, std::memory_order_relaxed);
            if (b >= nblk) return;
            pack_range(in, b * BLK, (b + 1) * BLK < n ? (b + 1) * BLK : n, n, out);
        }
    }
    void loop(int idx, uint64_t seen) {          // seen = the job generation at creation: only LATER jobs are this worker's
        for (;;) {
            bool got = false;
            const auto t0 = std::chrono::steady_clock::now();
            for (unsigned i = 1;; ++i) {                     // bounded polling, then sleep
                if (gen.load(std::memory_order_acquire) != seen) { got = true; break; }
                if ((i & 127u) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::microseconds(200)) break;
#if defined(__x86_64__)
                _mm_pause();
#endif
            }
            std::unique_lock<std::mutex> lk(mu);
            if (!got) cv_work.wait(lk, [&] { return gen.load(std::memory_order_acquire) != seen; });
            seen = gen.load(std::memory_order_acquire);
            const bool mine = idx < use;
            lk.unlock();
            if (mine) blocks();
            lk.lock();
            if (--pending == 0) cv_done.notify_one();
        }
    }

public:
    void pack(const uint8_t *src, int64_t count, uint8_t *dst, int threads) {
        std::lock_guard<std::mutex> call(call_mu);
        const int64_t blocks_total = (count + BLK - 1) / BLK;
        int nt = threads;
        if ((int64_t)nt > blocks_total) nt = (int)blocks_total;
        if (nt <= 1) { pack_range(src, 0, count, count, dst); return; }
        while ((int)workers.size() < nt - 1) {
            const int idx = (int)workers.size();
            uint64_t g0;
            { std::lock_guard<std::mutex> lk(mu); g0 = gen.load(); }
            workers.emplace_back([this, idx, g0] { loop(idx, g0); });
            workers.back().detach();             // process-lifetime team (the library is never unloaded while a call runs)
        }
        {
            std::lock_guard<std::mutex> lk(mu);
            in = src; out = dst; n = count; nblk = blocks_total;
            next.store(0, std::memory_order_relaxed);
            use = nt - 1; pending = (int)workers.size();
            gen.fetch_add(1, std::memory_order_release);
        }
        cv_work.notify_all();
        blocks();                                // the caller is the team's last member
        std::unique_lock<std::mutex> lk(mu);
        cv_done.wait(lk, [&] { return pending == 0; });
    }
};
PackTeam *g_team = new PackTeam;                 // intentionally leaked: detached workers may outlive static destructors

}  // namespace

// n ASCII bytes -> (n+1)/2 bytes, base 2k in the low nibble and base 2k+1 in the high nibble of byte k (a missing last
// base packs as 0).  threads <= 0: the hardware threads, capped by the cgroup CPU quota (see PackTeam).  Safe to call
// concurrently on different buffers (calls take turns).
extern "C" void pb_pack_nibbles(const uint8_t *in, int64_t n, uint8_t *out, int threads) {
    if (n <= 0) return;
    if (threads <= 0) {
        static const int dflt = [] {
            long hw = (long)std::thread::hardware_concurrency();
            if (hw < 1) hw = 1;
            if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
                char q[64]; long long period = 0;
                if (fscanf(f, "%63s %lld", q, &period) == 2 && strcmp(q, "max") != 0 && period > 0 && atoll(q) > 0)
                    hw = std::min<long>(hw, (long)std::max<long long>(1, (atoll(q) + period - 1) / period));
                fclose(f);
            }
            return (int)hw;
        }();
        threads = dflt;
    }
    g_team->pack(in, n, out, threads);
}
