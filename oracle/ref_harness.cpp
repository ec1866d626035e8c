// oracle/ref_harness.cpp -- TEST / BASELINE INFRASTRUCTURE ONLY.
//
// Native timing harness for the reference CPU path (BASELINE.md section 3, SURVEY.md 8(d)):
// dlopen()s a library exporting the reference C-ABI (porechop/include/adapter_align.h:12-16:
// adapterAlignment / freeCString) -- normally oracle/_ref/cpp_functions.so, the UNMODIFIED reference
// C++ -- and calls it over a pair list from T std::threads (the Python --threads path anti-scales,
// SURVEY section 6, so the fair multi-core baseline is a native caller).
//
// usage: ref_harness <lib.so> <workload.bin> <threads> [answers.txt]
//   env REF_HARNESS_PROCS=P (P > 1): P forked worker PROCESSES x <threads> threads each pull chunks from one shared
//   counter -- every process has its own heap, which separates the machine's capacity from glibc-arena contention
//   (the reference mallocs an (n+1)(m+1) trace matrix per call, so many threads of one process can contend on the
//   allocator).  Answers are only written in the single-process mode.
//   workload.bin (little endian), written by porechop_b200.workloads.write_harness_file():
//     int64 n_seqs, n_adapters, n_pairs ; int32 ma, mi, go, ge ; int32 cross, pad
//     int64 seq_off[n_seqs+1] ; bytes seqs ; int32 ad_off[n_adapters+1] ; bytes adapters
//     if !cross: int32 pair_seq[n_pairs] ; int32 pair_adapter[n_pairs]
//   prints one JSON line: {"seconds":..,"pairs":..,"cells":..,"threads":..}
//   with answers.txt: also writes one result string per pair (in pair order).
#include <dlfcn.h>
#include <sys/mman.h>
#include <sys/wait.h>
#include <unistd.h>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

typedef char *(*align_fn)(char *, char *, int, int, int, int);
typedef void (*free_fn)(char *);

static bool read_all(FILE *f, void *dst, size_t n) { return n == 0 || fread(dst, 1, n, f) == n; }

int main(int argc, char **argv)
{
    if (argc < 4) { fprintf(stderr, "usage: %s lib.so workload.bin threads [answers.txt]\n", argv[0]); return 2; }
    void *lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
    if (!lib) { fprintf(stderr, "dlopen failed: %s\n", dlerror()); return 2; }
    align_fn align = (align_fn)dlsym(lib, "adapterAlignment");
    free_fn release = (free_fn)dlsym(lib, "freeCString");
    if (!align || !release) { fprintf(stderr, "missing symbols\n"); return 2; }
    int threads = atoi(argv[3]);
    if (threads < 1) threads = 1;

    FILE *f = fopen(argv[2], "rb");
    if (!f) { perror("workload"); return 2; }
    int64_t hdr[3]; int32_t sc[6];
    if (!read_all(f, hdr, sizeof hdr) || !read_all(f, sc, sizeof sc)) return 2;
    int64_t n_seqs = hdr[0], n_ad = hdr[1], n_pairs = hdr[2];
    bool cross = sc[4] != 0;
    std::vector<int64_t> seq_off(n_seqs + 1);
    if (!read_all(f, seq_off.data(), sizeof(int64_t) * (n_seqs + 1))) return 2;
    std::vector<char> seqs(seq_off[n_seqs]);
    if (!read_all(f, seqs.data(), seqs.size())) return 2;
    std::vector<int32_t> ad_off(n_ad + 1);
    if (!read_all(f, ad_off.data(), sizeof(int32_t) * (n_ad + 1))) return 2;
    std::vector<char> ads(ad_off[n_ad]);
    if (!read_all(f, ads.data(), ads.size())) return 2;
    std::vector<int32_t> ps, pa;
    if (!cross) {
        ps.resize(n_pairs); pa.resize(n_pairs);
        if (!read_all(f, ps.data(), 4 * n_pairs) || !read_all(f, pa.data(), 4 * n_pairs)) return 2;
    }
    fclose(f);

    // NUL-terminated copies (the ABI takes C strings; strlen is part of the reference's cost)
    std::vector<std::string> S(n_seqs), A(n_ad);
    for (int64_t i = 0; i < n_seqs; ++i) S[i].assign(seqs.data() + seq_off[i], seq_off[i + 1] - seq_off[i]);
    for (int64_t i = 0; i < n_ad; ++i) A[i].assign(ads.data() + ad_off[i], ad_off[i + 1] - ad_off[i]);

    bool want = argc > 4;
    int procs = getenv("REF_HARNESS_PROCS") ? atoi(getenv("REF_HARNESS_PROCS")) : 1;
    if (procs < 1 || want) procs = 1;
    std::vector<std::string> answers(want ? n_pairs : 0);
    // the work counter and the cell total live in a shared anonymous mapping so that forked workers can use them too
    struct Shared { std::atomic<int64_t> next; std::atomic<long long> cells; };
    Shared *sh = (Shared *)mmap(nullptr, sizeof(Shared), PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
    if (sh == MAP_FAILED) { perror("mmap"); return 2; }
    new (&sh->next) std::atomic<int64_t>(0);
    new (&sh->cells) std::atomic<long long>(0);
    auto worker = [&]() {
        long long my = 0;
        const int64_t CH = 64;
        for (;;) {
            int64_t b = sh->next.fetch_add(CH);
            if (b >= n_pairs) break;
            int64_t e = b + CH < n_pairs ? b + CH : n_pairs;
            for (int64_t p = b; p < e; ++p) {
                int64_t s = cross ? p / n_ad : ps[p];
                int64_t a = cross ? p % n_ad : pa[p];
                char *r = align(const_cast<char *>(S[s].c_str()), const_cast<char *>(A[a].c_str()),
                                sc[0], sc[1], sc[2], sc[3]);
                if (want) answers[p] = r;
                release(r);
                my += (long long)S[s].size() * (long long)A[a].size();
            }
        }
        sh->cells += my;
    };
    auto run_threads = [&]() {
        std::vector<std::thread> pool;
        for (int t = 1; t < threads; ++t) pool.emplace_back(worker);
        worker();
        for (auto &t : pool) t.join();
    };
    auto t0 = std::chrono::steady_clock::now();
    if (procs > 1) {
        std::vector<pid_t> kids;
        for (int k = 0; k < procs; ++k) {
            pid_t pid = fork();
            if (pid < 0) { perror("fork"); break; }
            if (pid == 0) { run_threads(); _exit(0); }
            kids.push_back(pid);
        }
        for (pid_t pid : kids) { int st = 0; waitpid(pid, &st, 0); }
    } else {
        run_threads();
    }
    double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (want) {
        FILE *o = fopen(argv[4], "w");
        if (!o) { perror("answers"); return 2; }
        for (auto &s : answers) fprintf(o, "%s\n", s.c_str());
        fclose(o);
    }
    printf("{\"seconds\": %.6f, \"pairs\": %lld, \"cells\": %lld, \"threads\": %d, \"procs\": %d}\n",
           sec, (long long)n_pairs, (long long)sh->cells.load(), threads, procs);
    return 0;
}
