// tools/ubench_pipes.cu -- which PIPE the instructions of the DP kernels issue on, and at what rate (sm_90a).
// Each kernel runs 8 independent chains per thread of one op (or two ops alternating), 8 warps per scheduler.  Printed:
// warp-instructions per clock and scheduler from clock64; run under
//   ncu --metrics smsp__inst_executed.sum,smsp__issue_active.avg.pct_of_peak_sustained_active,\
//       sm__pipe_alu_cycles_active.avg.pct_of_peak_sustained_active,sm__pipe_fmaheavy_cycles_active.avg.pct_of_peak_sustained_active,\
//       sm__pipe_fmalite_cycles_active.avg.pct_of_peak_sustained_active,sm__pipe_fma_cycles_active.avg.pct_of_peak_sustained_active
// the pipe counters of every kernel say where its instructions went.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ubench_pipes tools/ubench_pipes.cu ; run on an H100.
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#define ITER 2048
enum { VMAX, VADDMAX, VADD2, ADD32, PADD, POR, LOP, IMADOP, VMAX3, MIX_VMAX_VADD2, MIX_VMAX_ADD32, MIX_VADD2_ADD32, MIX_VMAX_LOP,
       MIX_VADDMAX_IMAD, CELL_TRACE, N_OPS };

__device__ __forceinline__ uint32_t op_vmax(uint32_t a, uint32_t b) { return __vmaxs2(a, b); }
__device__ __forceinline__ uint32_t op_vaddmax(uint32_t a, uint32_t b, uint32_t c) { return __viaddmax_s16x2(a, b, c); }
__device__ __forceinline__ uint32_t op_vadd2(uint32_t a, uint32_t b) { return __vadd2(a, b); }
__device__ __forceinline__ uint32_t op_lop(uint32_t a, uint32_t b) { uint32_t d; asm("lop3.b32 %0, %1, %2, 0, 0xC3;" : "=r"(d) : "r"(a), "r"(b)); return d; }

template <int OP>
__global__ void __launch_bounds__(512) k(uint32_t *out, uint32_t seed, long long *cycles) {
    uint32_t a[8], acc = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = seed + threadIdx.x * 17 + i * 1237;
    uint32_t c1 = seed | 0x00030003u, c2 = seed ^ 0x7fff7fffu;
    const long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < ITER; ++it) {
        c2 += 0x00010001u;      // operands change every iteration: nothing is loop-invariant or idempotent
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (OP == VMAX) a[i] = op_vmax(a[i], c2) ^ 0;
            if (OP == VADDMAX) a[i] = op_vaddmax(a[i], c1, c2);
            if (OP == VADD2) a[i] = op_vadd2(a[i], c2);
            if (OP == ADD32) a[i] = a[i] - c2;
            if (OP == PADD) { asm("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %1, %2;\n\t@p add.u32 %0, %0, %3;\n\t}" : "+r"(a[i]) : "r"(c2), "r"(seed), "r"(1u << i)); }
            if (OP == POR) { asm("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %1, %2;\n\t@p or.b32 %0, %0, %3;\n\t}" : "+r"(a[i]) : "r"(c2), "r"(seed), "r"(c2)); }
            if (OP == LOP) a[i] = op_lop(a[i], c2);
            if (OP == IMADOP) a[i] = a[i] * 3 + c2;
            if (OP == VMAX3) a[i] = __vimax3_s16x2(a[i], c1, c2);
            if (OP == MIX_VMAX_VADD2) a[i] = (i & 1) ? op_vmax(a[i], c2) : op_vadd2(a[i], c2);
            if (OP == MIX_VMAX_ADD32) a[i] = (i & 1) ? op_vmax(a[i], c2) : a[i] - c2;
            if (OP == MIX_VADD2_ADD32) a[i] = (i & 1) ? op_vadd2(a[i], c2) : a[i] - c2;
            if (OP == MIX_VMAX_LOP) a[i] = (i & 1) ? op_vmax(a[i], c2) : op_lop(a[i], c2);
            if (OP == MIX_VADDMAX_IMAD) a[i] = (i & 1) ? op_vaddmax(a[i], c1, c2) : a[i] * 3 + c2;
            if (OP == CELL_TRACE) {   // one row of the trace cell as the kernel issues it: 4 x (VIMNMX.P + 2 predicated adds) + 3 packed adds + LOP3 + VIADDMNMX + sub
                uint32_t x = a[i], v;
                const uint32_t sub = op_vaddmax(op_lop(x, c2), c1, c2);
                const uint32_t d = op_vadd2(x, sub);
                uint32_t hs = op_vadd2(x, c1), vs = op_vadd2(d, c1);
#define MAXACC(dst, p, q, bit)                                                                                          \
    asm("{\n\t.reg .pred plo, phi;\n\t.reg .s16 a0, a1, b0, b1;\n\tmax.s16x2 %0, %2, %3;\n\tmov.b32 {a0, a1}, %0;\n\t" \
        "mov.b32 {b0, b1}, %2;\n\tsetp.eq.s16 plo, a0, b0;\n\tsetp.eq.s16 phi, a1, b1;\n\t"                           \
        "@plo add.u32 %1, %1, %4;\n\t@phi add.u32 %1, %1, %5;\n\t}"                                                   \
        : "=r"(dst), "+r"(acc) : "r"(p), "r"(q), "r"(1u << (bit)), "r"(0x10000u << (bit)))
                MAXACC(v, hs, x, 0); hs = v;
                MAXACC(v, vs, d, 1); vs = v;
                MAXACC(v, vs, hs, 2);
                uint32_t s; MAXACC(s, d, v, 3);
                a[i] = s - c1;
            }
        }
    }
    const long long t1 = clock64();
    uint32_t s = acc;
#pragma unroll
    for (int i = 0; i < 8; ++i) s ^= a[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cycles = t1 - t0;
}

template <int OP> void run(const char *name, int per_chain_instr) {
    uint32_t *out; long long *cyc, h;
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&out, (size_t)sms * 2 * 512 * 4); cudaMalloc(&cyc, 8);
    for (int rep = 0; rep < 2; ++rep) { k<OP><<<sms * 2, 512>>>(out, 12345u, cyc); cudaDeviceSynchronize(); }   // 32 warps / SM
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    const double warp_instr = 8.0 * ITER * 8 * per_chain_instr;   // per scheduler: 8 warps x ITER x 8 chains
    printf("%-44s %.3f warp-instr/clk/scheduler\n", name, warp_instr / h);
    cudaFree(out); cudaFree(cyc);
}
int main() {
    run<VMAX>("VIMNMX.S16x2", 1);
    run<VADDMAX>("VIADDMNMX.S16x2", 1);
    run<VADD2>("VIADD.16x2", 1);
    run<ADD32>("32-bit sub (VIADD / IADD3 / IMAD.IADD)", 1);
    run<PADD>("predicated add", 1);
    run<POR>("predicated or", 1);
    run<LOP>("LOP3", 1);
    run<IMADOP>("IMAD", 1);
    run<VMAX3>("VIMNMX3.S16x2", 1);
    run<MIX_VMAX_VADD2>("VIMNMX / VIADD.16x2 alternating", 1);
    run<MIX_VMAX_ADD32>("VIMNMX / 32-bit sub alternating", 1);
    run<MIX_VADD2_ADD32>("VIADD.16x2 / 32-bit sub alternating", 1);
    run<MIX_VMAX_LOP>("VIMNMX / LOP3 alternating", 1);
    run<MIX_VADDMAX_IMAD>("VIADDMNMX / IMAD alternating", 1);
    run<CELL_TRACE>("trace cell row (18 instructions)", 18);
    return 0;
}
