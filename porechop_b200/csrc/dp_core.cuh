// porechop_b200/csrc/dp_core.cuh
//
// Core of the H100 adapter-alignment engine: the packed-int16 (s16x2, DPX) cell recurrence, the
// per-lane wavefront step, best-end-cell tracking, traceback and alignment statistics.
//
// Semantics follow the reference hot path (paths relative to a Porechop v0.2.4 checkout, seqan/ =
// porechop/include/seqan/) -- nothing here is ported code, only the arithmetic contract:
//   cell        seqan/align/dp_formula_affine.h:459-495 ; linear case dp_formula_linear.h:156-188
//   borders     seqan/align/dp_formula.h:204-220, dp_cell_affine.h:62-64
//   scout       seqan/align/dp_scout.h:168-181, dp_meta_info.h:200-213
//   traceback   seqan/align/dp_algorithm_impl.h:1354-1369, dp_traceback_impl.h:379-555
//   statistics  porechop/src/alignment.cpp:6-110
//
// Everything in this header is `PB_HD` (host+device) so that tests/emu (a CPU emulation of one
// sub-warp group, compiled with g++) runs exactly the code the kernels run; only warp shuffles,
// shared-memory addressing and the launch glue live in kernels.cu.
//
// Mapping (see DESIGN.md): a *slot* is two independent alignments carried in the two int16 halves of
// every 32-bit register (half A = low 16 bits, half B = high 16 bits).  A slot is processed by a group
// of G consecutive lanes; lane g owns adapter rows g*R+1 .. g*R+R and at step t computes read column
// j = t-g+1 for those rows (anti-diagonal wavefront); the bottom row's (S, Vs) move to lane g+1 by
// one warp shuffle per step.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PB_HD __host__ __device__ __forceinline__
#else
#define PB_HD inline
#endif

namespace pb {

#if !defined(__CUDA_ARCH__) && defined(PB_CHECK_RANGES)
void pb_range_violation();   // defined by the CPU emulation: counts int16-domain violations
#endif

// ---- int16 domain ---------------------------------------------------------------------------------------
// All DP values are kept BIASED by PB_BIAS so that every 16-bit half is a non-negative number: adding a
// (negative) gap score to both halves is then ONE plain 32-bit subtraction of the packed magnitudes with no
// borrow between the halves -- an instruction ptxas may place on either the ALU or the FMA pipe, which is what
// balances the two pipes (the packed DPX max / add-max instructions only exist on the ALU pipe).
//   genuine values   |x| <= PB_I16_LIMIT (+ one more score)      (host check: A*(m+3) <= PB_I16_LIMIT)
//   "-infinity"      PB_NEG16 (borders, left edge of a windowed pass); pseudo-infinite values of a windowed
//                    pass stay within PB_NEG16 +- PB_I16_LIMIT, below every genuine value
//   smallest value ever formed: PB_NEG16 - PB_I16_LIMIT - PB_LINEAR_EXT  > -PB_BIAS   (no wrap, no borrow)
constexpr int PB_BIAS = 24576;
constexpr int PB_NEG16 = -14000;
constexpr int PB_I16_LIMIT = 4000;
constexpr int PB_LINEAR_EXT = 4096;    // magnitude of the "never extend" pseudo score that runs go==ge through the affine cell
constexpr int PB_CODE_SHIFT = 12;      // base codes live in bits 12..14 of each half: x^y is 0 or >= 4096
constexpr int PB_MAX_SUBW = 4096;      // ma - mi must not exceed this for the xnor/addmax substitution trick
constexpr uint8_t PB_PAD_H = 0x50;     // encoded-byte value (code<<4) for read padding (matches nothing)
constexpr uint8_t PB_PAD_V = 0x60;     // encoded-byte value for adapter padding rows

// record layout of one alignment (9 x int32): rs, re, as, ae, score, match_aln, len_aln, match_ad, len_ad
constexpr int PB_REC = 9;
constexpr int32_t PB_SCORE_EMPTY = (int32_t)0x80000000;

PB_HD uint32_t pack2(int lo, int hi) { return ((uint32_t)lo & 0xFFFFu) | (((uint32_t)hi & 0xFFFFu) << 16); }
PB_HD int half16(uint32_t x, int h) { return (int)(int16_t)(h ? (x >> 16) : (x & 0xFFFFu)); }

// ASCII -> encoded byte (Dna5 code << 4): A/a=0 C/c=1 G/g=2 T/t/U/u=3, every other byte = 4
// (seqan/basic/alphabet_residue_tabs.h:113-140)
PB_HD uint32_t encode_byte(uint32_t c) {
    uint32_t u = c & 0xDFu;  // fold case
    uint32_t code = 4u;
    code = (u == 'A') ? 0u : code;
    code = (u == 'C') ? 1u : code;
    code = (u == 'G') ? 2u : code;
    code = (u == 'T' || u == 'U') ? 3u : code;
    return code << 4;
}

// Packed upload path (option h2d_pack): the host converts ASCII to Dna5 codes itself and ships two 4-bit codes per byte
// (hostpack.cpp: base 2k in the low nibble of byte k, base 2k+1 in the high nibble).  One packed 32-bit word = 8 bases ->
// the same 8 encoded bytes (code << 4) encode_byte would have produced, as two words in memory order.
PB_HD void unpack_nibbles8(uint32_t w, uint32_t &first4, uint32_t &next4) {
    const uint32_t e = (w & 0x0F0F0F0Fu) << 4;      // even bases of the 4 packed bytes, already code << 4
    const uint32_t o = w & 0xF0F0F0F0u;             // odd bases
#if defined(__CUDA_ARCH__)
    first4 = __byte_perm(e, o, 0x5140);
    next4 = __byte_perm(e, o, 0x7362);
#else
    first4 = (e & 0xFFu) | ((o & 0xFFu) << 8) | ((e & 0xFF00u) << 8) | ((o & 0xFF00u) << 16);
    next4 = ((e >> 16) & 0xFFu) | (((o >> 16) & 0xFFu) << 8) | (((e >> 24) & 0xFFu) << 16) | ((o >> 24) << 24);
#endif
}
PB_HD uint32_t unpack_nibble1(uint32_t packed_byte, int odd) { return odd ? (packed_byte & 0xF0u) : ((packed_byte & 0x0Fu) << 4); }

// ---- packed s16x2 primitives (DPX instructions of sm_90: __viaddmax_s16x2, __vibmax_s16x2, __vimax3_s16x2) ----
PB_HD uint32_t add2(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __vadd2(a, b);
#else
    return (((a & 0xFFFFu) + (b & 0xFFFFu)) & 0xFFFFu) | ((((a >> 16) + (b >> 16)) & 0xFFFFu) << 16);
#endif
}
// max with "first operand wins ties" predicates: p = (a >= b) per half
PB_HD uint32_t max2p(uint32_t a, uint32_t b, bool &plo, bool &phi) {
#if defined(__CUDA_ARCH__)
    return __vibmax_s16x2(a, b, &phi, &plo);
#else
    int al = half16(a, 0), bl = half16(b, 0), ah = half16(a, 1), bh = half16(b, 1);
    plo = al >= bl; phi = ah >= bh;
    return pack2(plo ? al : bl, phi ? ah : bh);
#endif
}
PB_HD uint32_t max2(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    return __vmaxs2(a, b);
#else
    bool p, q; return max2p(a, b, p, q);
#endif
}
// max(a+b, c) per half
PB_HD uint32_t addmax2(uint32_t a, uint32_t b, uint32_t c) {
#if defined(__CUDA_ARCH__)
    return __viaddmax_s16x2(a, b, c);
#else
    return max2(add2(a, b), c);
#endif
}
PB_HD uint32_t max3(uint32_t a, uint32_t b, uint32_t c) {
#if defined(__CUDA_ARCH__)
    return __vimax3_s16x2(a, b, c);
#else
    return max2(max2(a, b), c);
#endif
}

// ---- scoring scheme as the kernels see it --------------------------------------------------------------
// The state of a cell is X = S + go (+bias): it is what both the cell to the right (horizontal open) and the cell
// below (vertical open) need, so the "+ go" is added once per cell; the diagonal use compensates by folding "- go"
// into the substitution constants.
struct Scoring {
    uint32_t goMag2;  // packed |go|  (linear mode: |ge|)            X = S_biased - goMag
    uint32_t geMag2;  // packed |ge|  (linear mode: PB_LINEAR_EXT)   h_ext = Hs_biased - geMag   (trace pass)
    uint32_t ge2;     // packed signed ge (linear: -PB_LINEAR_EXT)   for the fused add-max of the score pass
    uint32_t subA2;   // packed (match + 1 - go)
    uint32_t subF2;   // packed (mismatch - go)
    uint32_t padF2;   // packed (-go): substitution operand of the border-emulating pad rows
    uint32_t borderX2;// packed biased X of the zero border: 0 + go + bias
    uint32_t negb2;   // packed biased -infinity
    int32_t goEff;    // go (linear: ge)
    int32_t linear;   // go == ge : NW recurrence of dp_formula_linear.h, no end-cell correction
    int32_t ma, mi, go, ge;
};

PB_HD Scoring make_scoring(int ma, int mi, int go, int ge) {
    Scoring s;
    s.linear = (go == ge) ? 1 : 0;
    s.ma = ma; s.mi = mi; s.go = go; s.ge = ge;
    const int goE = s.linear ? ge : go;
    const int geE = s.linear ? -PB_LINEAR_EXT : ge;
    s.goEff = goE;
    s.goMag2 = pack2(-goE, -goE);
    s.geMag2 = pack2(-geE, -geE);
    s.ge2 = pack2(geE, geE);
    s.subA2 = pack2(ma + 1 - goE, ma + 1 - goE);
    s.subF2 = pack2(mi - goE, mi - goE);
    s.padF2 = pack2(-goE, -goE);
    s.borderX2 = pack2(PB_BIAS + goE, PB_BIAS + goE);
    s.negb2 = pack2(PB_BIAS + PB_NEG16, PB_BIAS + PB_NEG16);
    return s;
}

// One alignment as the kernels see it (64 bytes).  `n` columns of the encoded read starting at seq_off
// are aligned against `m` adapter rows.  A windowed task (second pass over a long read) starts at global
// column col0 with a -infinity left boundary (unless col0 == 0) and has its end cell given.
struct Task {
    int64_t seq_off;     // offset of the first column's base in the encoded sequence buffer
    int32_t n;           // number of columns (window length)
    int32_t m;           // adapter length (rows)
    int32_t ad_off;      // offset of the adapter in the encoded adapter buffer
    int32_t out_idx;     // index of the 9-int result record
    int32_t flags;       // TASK_* bits
    int32_t end_j;       // given end cell: column local to the window (TASK_END_GIVEN)
    int32_t end_i;       //                 row
    int32_t end_corr;    // bit0: Vs* == S*, bit1: Hs* == S*   (dp_algorithm_impl.h:1354-1369)
    int32_t end_score;
    int32_t col0;        // global column of the window start (read coordinates = local + col0)
    int32_t n_total;     // full read length
    int32_t pad0, pad1, pad2;
};
static_assert(sizeof(Task) == 64, "Task must be 64 bytes");
enum { TASK_LEFT_INF = 1, TASK_END_GIVEN = 2 };

// End cell of one alignment found by the score pass.
struct EndCell {
    int32_t j, i, score, corr;
};

// Window of the second pass of a long read: how many columns left of its end cell (j*, i*) the traced path can reach.
// The path has score S* >= 0 and consumes at most i* adapter rows, hence d <= i* diagonals, each worth at most
// wnum = max(ma, mi, 0); every read-only gap column costs at least wden = min(|go|, |ge|) > 0 and every vertical step
// costs something, so  S* <= wnum*d - wden*hg  and the path spans  d + hg <= i* + (wnum*i* - S*)/wden  columns -- with
// strict inequality as soon as it contains a vertical step, which is what lets the -infinity left edge of the window
// stand in for the real column (DESIGN.md "two-pass scheme").
//   classic bound (tight == false): i* <= m, S* >= 0  ->  W(m) = m + m*wnum/wden, the same for every alignment of an adapter
//   tight bound: uses the end cell the score pass found; never larger than the classic one.
PB_HD int64_t window_cols(int m, int end_i, int end_score, int wnum, int wden, bool tight) {
    const int64_t wc = (int64_t)m + ((int64_t)m * wnum) / wden;
    if (!tight) return wc;
    int64_t num = (int64_t)wnum * end_i - (int64_t)end_score;
    if (num < 0) num = 0;
    const int64_t wt = (int64_t)end_i + num / wden;
    return wt < wc ? wt : wc;
}

// ---- one lane of a group ------------------------------------------------------------------------------
// Row layout: the G*R rows of a group are BOTTOM-aligned per half: real adapter row i (1..m) lives at group row
// q = i + pad, pad = G*R - m, so the last row m is always the bottom row of lane G-1 (static register, no
// per-step row selection for the scout).  The `pad` rows above row 1 reproduce the zero border row without
// extra instructions: they carry a code that matches nothing and the substitution operand -go, so they compute
// S = 0 in every column (d = 0 beats both gaps), and their gap values are never better than what the true
// border would present to row 1.
template <int R>
struct Lane {
    uint32_t X[R];    // X[j-1][row] = S + go (biased, packed halves); becomes X[j][row] after the step
    uint32_t Hs[R];   // Hs[j-1][row] (biased)
    uint32_t v2[R];   // adapter code << PB_CODE_SHIFT of the owned rows, packed halves
    uint32_t sf2[R];  // per-row mismatch operand (real rows: mi - go, pad rows: -go)
    uint32_t prevRecvX;  // X[j-1][top-1]  (diagonal input of the top row)
    uint32_t botX, botV; // X[j][bottom], Vs[j][bottom] -> shuffled to the next lane
    // scout state: last-row running best (X domain), packed, with the Vs / Hs of that cell (the end-cell correction flags
    // are derived from them once, in make_cand) -- lane G-1 only: the other lanes start at +infinity and never update ...
    uint32_t lrBest2, lrV2, lrH2;
    int lrJ[2];
    // ... and the best of this lane's rows in the final column, per half (X domain, biased)
    int fcBest[2], fcI[2], fcCorr[2];
};

// geometry of one half of a slot
struct HalfGeom {
    int n, m;
    int pad;      // G*R - m : number of border-emulating rows above row 1
};
PB_HD HalfGeom make_geom(int n, int m, int G, int R) {
    HalfGeom h; h.n = n; h.m = m; h.pad = G * R - m;
    return h;
}

// x - P per half where P holds magnitudes and every half of x is >= the half of P: one plain 32-bit subtraction
PB_HD uint32_t subm2(uint32_t x, uint32_t P) {
#if !defined(__CUDA_ARCH__) && defined(PB_CHECK_RANGES)
    if ((x & 0xFFFFu) < (P & 0xFFFFu) || (x >> 16) < (P >> 16) || (x & 0x80008000u)) pb_range_violation();
#endif
    return x - P;
}

template <int R>
PB_HD void lane_init(Lane<R> &L, int g, int G, const Scoring &sc, const uint8_t *adA, int mA, bool leftInfA,
                     const uint8_t *adB, int mB, bool leftInfB) {
    const int padA = G * R - mA, padB = G * R - mB;
    // column 0: X = S0 + go + bias with S0 = 0 (border / pad rows) or -inf (real rows of a windowed task)
    const uint32_t x0 = sc.borderX2;
    const uint32_t xinf = add2(sc.negb2, pack2(sc.goEff, sc.goEff));
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int q = g * R + r + 1;
        const int iA = q - padA, iB = q - padB;      // real rows (>= 1) or pad rows (<= 0)
        const bool realA = iA >= 1, realB = iB >= 1;
        const uint32_t a = realA ? (uint32_t)adA[iA - 1] : (uint32_t)PB_PAD_V;
        const uint32_t b = realB ? (uint32_t)adB[iB - 1] : (uint32_t)PB_PAD_V;
        L.v2[r] = (a << 8) | (b << 24);               // code<<4 in a byte -> code<<12 in the half
        L.sf2[r] = ((realA ? sc.subF2 : sc.padF2) & 0xFFFFu) | ((realB ? sc.subF2 : sc.padF2) & 0xFFFF0000u);
        L.X[r] = (((realA && leftInfA) ? xinf : x0) & 0xFFFFu) | (((realB && leftInfB) ? xinf : x0) & 0xFFFF0000u);
        L.Hs[r] = sc.negb2;
    }
    {   // X[0][row above this lane's top row]
        const int q = g * R;
        const bool realA = (q - padA) >= 1, realB = (q - padB) >= 1;
        L.prevRecvX = (((realA && leftInfA) ? xinf : x0) & 0xFFFFu) | (((realB && leftInfB) ? xinf : x0) & 0xFFFF0000u);
    }
    L.botX = L.X[R - 1]; L.botV = sc.negb2;
    // candidate (0, m): S = 0, no correction.  Only the bottom row of lane G-1 is the last row: every other lane starts from
    // +infinity, so its compare never fires and the scout branch of the step loops is taken for real candidates only
    // (with all 32 lanes tracking their own bottom rows the "rare" branch would run in most steps).
    L.lrBest2 = (g == G - 1) ? sc.borderX2 : 0x7FFF7FFFu;
    L.lrV2 = sc.negb2; L.lrH2 = sc.negb2;
    for (int h = 0; h < 2; ++h) {
        L.lrJ[h] = 0;
        L.fcBest[h] = -1; L.fcI[h] = 0; L.fcCorr[h] = 0;   // biased X values are >= 0
    }
}

// ~(a ^ b) as ONE LOP3 (the compiler otherwise splits it into xor + not)
PB_HD uint32_t xnor2(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
    uint32_t d;
    asm("lop3.b32 %0, %1, %2, 0, 0xC3;" : "=r"(d) : "r"(a), "r"(b));
    return d;
#else
    return ~(a ^ b);
#endif
}

// max(a, b) per half; sets the bits `clo` / `chi` in acc when a >= b in the low / high half ("first operand wins ties").
// Device: ptxas fuses this into one VIMNMX.S16x2 with two predicate outputs plus two predicated accumulations.
// on_alu picks the PIPE of the two accumulations: the flag bits of a step are disjoint, so add / or / xor give the same word,
// but a predicated add issues on the FMA-heavy pipe (VIADD / IMAD.IADD) and a predicated logic op on the ALU pipe (LOP3).
// Both pipes take one warp instruction per two cycles and scheduler and the FMA-lite pipe takes no integer work
// (tools/ubench_pipes.cu measures which pipe each instruction issues on).  With every accumulation an add the trace pass
// has 12 heavy and 6 ALU instructions per row and is bound by the heavy pipe; lane_step mixes the two forms (PB_FLAG_ALU_*).
// (on_alu is a constant after unrolling: the dead form is eliminated)
PB_HD uint32_t max2acc(bool on_alu, uint32_t a, uint32_t b, uint32_t &accLo, uint32_t clo, uint32_t &accHi, uint32_t chi) {
#if defined(__CUDA_ARCH__)
    uint32_t val;
    if (on_alu) {
        asm("{\n\t.reg .pred plo, phi;\n\t.reg .s16 a0, a1, b0, b1;\n\t"
            "max.s16x2 %0, %3, %4;\n\t"
            "mov.b32 {a0, a1}, %0;\n\tmov.b32 {b0, b1}, %3;\n\t"
            "setp.eq.s16 plo, a0, b0;\n\tsetp.eq.s16 phi, a1, b1;\n\t"
            "@plo xor.b32 %1, %1, %5;\n\t@phi xor.b32 %2, %2, %6;\n\t}"      // xor, not or: ptxas turns an `or` of provably disjoint bits back into an add
            : "=r"(val), "+r"(accLo), "+r"(accHi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
    } else {
        asm("{\n\t.reg .pred plo, phi;\n\t.reg .s16 a0, a1, b0, b1;\n\t"
            "max.s16x2 %0, %3, %4;\n\t"
            "mov.b32 {a0, a1}, %0;\n\tmov.b32 {b0, b1}, %3;\n\t"
            "setp.eq.s16 plo, a0, b0;\n\tsetp.eq.s16 phi, a1, b1;\n\t"
            "@plo add.u32 %1, %1, %5;\n\t@phi add.u32 %2, %2, %6;\n\t}"
            : "=r"(val), "+r"(accLo), "+r"(accHi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
    }
    return val;
#else
    bool plo, phi;
    uint32_t v = max2p(a, b, plo, phi);
    if (plo) accLo = on_alu ? (accLo ^ clo) : (accLo + clo);
    if (phi) accHi = on_alu ? (accHi ^ chi) : (accHi + chi);
    return v;
#endif
}
// which of a cell's four flag accumulations use the ALU-pipe form: bit 0 tH, 1 tV, 2 tM, 3 tD; _A for even rows of a lane,
// _B for odd rows.  The default (tD) puts 2 of the 8 accumulations per row on the ALU pipe, which makes the hot loop's ALU
// and FMA-heavy instruction counts about equal (279 / 286 per 4 steps x 7 rows of the end-trim class).
#ifndef PB_FLAG_ALU_A
#define PB_FLAG_ALU_A 0x8
#endif
#ifndef PB_FLAG_ALU_B
#define PB_FLAG_ALU_B 0x8
#endif

// Query profile of the score pass (option "profile", default on).  The substitution operand of group row q depends only
// on the read base -- six possible codes (0..4 and the read padding code 5).  When both halves of a slot read the same
// sequence (cross mode: one read, two adapters), score_kernel<.., PROF> keeps those words per lane group in shared memory
// and fetches a column's R operands with two 128-bit loads instead of computing them with LOP3 + VIADDMNMX per row.
// The word is produced by the very expression
// lane_step uses, so both paths are identical by construction.
// the two base-independent operands of a group row (adapter codes and mismatch operands, as lane_init sets them up) ...
PB_HD void profile_row(int q, const Scoring &sc, const uint8_t *adA, int mA, int padA, const uint8_t *adB, int mB, int padB,
                       uint32_t &v2, uint32_t &sf2) {
    const int iA = q - padA, iB = q - padB;
    const bool realA = iA >= 1 && iA <= mA, realB = iB >= 1 && iB <= mB;
    const uint32_t a = realA ? (uint32_t)adA[iA - 1] : (uint32_t)PB_PAD_V;
    const uint32_t b = realB ? (uint32_t)adB[iB - 1] : (uint32_t)PB_PAD_V;
    v2 = (a << 8) | (b << 24);
    sf2 = ((realA ? sc.subF2 : sc.padF2) & 0xFFFFu) | ((realB ? sc.subF2 : sc.padF2) & 0xFFFF0000u);
}
// ... and the operand for a read base code (both halves): exactly lane_step's expression
PB_HD uint32_t profile_from(uint32_t v2, uint32_t sf2, uint32_t bcode, const Scoring &sc) {
    const uint32_t e = (bcode & 7u) << 4;                         // encoded byte (code << 4)
    const uint32_t h2 = (e << 8) | (e << 24);
    return addmax2(xnor2(h2, v2), sc.subA2, sf2);
}
// The profile word in a form that a PLAIN 32-bit add applies to both halves at once.  A packed s16x2 addend whose low half is
// negative carries 1 into the high half when added as one 32-bit number (the low half of a biased X is always larger than
// the addend's magnitude), so that 1 is taken off the high half up front; a non-negative low half never carries (biased
// values stay below 2^15 + |addend|).  The diagonal term S_diag + sub then is an ordinary integer add (FMA-heavy pipe) --
// which ptxas cannot fuse into a VIADDMNMX on the ALU pipe, the busier pipe of the score pass -- and the cell's maximum
// becomes one three-input VIMNMX3: 3 ALU + 2 heavy instructions per row instead of 4 + 1, and fewer registers.
PB_HD uint32_t profile_plain(uint32_t sub2) { return (sub2 & 0x8000u) ? sub2 - 0x10000u : sub2; }
#define PB_PROF_ENCODE(x) profile_plain(x)
PB_HD uint32_t profile_word(int q, uint32_t bcode, const Scoring &sc, const uint8_t *adA, int mA, int padA, const uint8_t *adB,
                            int mB, int padB) {
    uint32_t v2, sf2;
    profile_row(q, sc, adA, mA, padA, adB, mB, padB, v2, sf2);
    return profile_from(v2, sf2, bcode, sc);
}

// R <= 4: one word per step (half A in bits 0..15, half B in bits 16..31); R = 5..8: word 0 = half A, word 1 = half B.
template <int R> struct TraceWords { static constexpr int value = (R <= 4) ? 1 : 2; };
template <int R> PB_HD int trace_word(int h, int r) { (void)r; return (R <= 4) ? 0 : h; }
template <int R> PB_HD int trace_shift(int h, int r) { return (R <= 4) ? (4 * r + 16 * h) : 4 * r; }

// end-cell correction flags of a cell (dp_algorithm_impl.h:1354-1369): bit0 Vs == S, bit1 Hs == S.
// x = biased X (= S + go + bias), vs/hs biased.
PB_HD int corr_flags(int x, int vs, int hs, int goEff) {
    const int sb = x - goEff;      // biased S
    return (vs == sb ? 1 : 0) | (hs == sb ? 2 : 0);
}
// Final-column scout of one row (lane_step<.., FCOL>): fc.mask bit h = the step's column is the final column of half h
struct FinalCol { int mask; int i0[2]; };   // i0[h]: real row of this lane's first row in half h (<= 0: pad row)
template <int R>
PB_HD void final_col_row(Lane<R> &L, const FinalCol &fc, int r, uint32_t x, uint32_t vs, uint32_t hs, const Scoring &sc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int i = fc.i0[h] + r;
        if (((fc.mask >> h) & 1) && i >= 1) {
            const int c = half16(x, h);
            if (c > L.fcBest[h]) {
                L.fcBest[h] = c; L.fcI[h] = i;
                L.fcCorr[h] = corr_flags(c, half16(vs, h), half16(hs, h), sc.goEff);
            }
        }
    }
}

// One wavefront step of one lane: column j with inputs from the lane above.
//   recvX/recvV : X[j][top-1], Vs[j][top-1]  (for g == 0 the caller passes the row-0 border: sc.borderX2 / sc.negb2)
//   h2          : read bases of column j, encoded << PB_CODE_SHIFT, packed halves
//   tw          : trace words of this step (TRACE only), TraceWords<R>::value entries.  4 flags per cell:
//       bit0 tD : diagonal chosen          (g <= d,  ties -> diagonal)
//       bit1 tM : vertical gap is the max  (vs >= hs, ties -> vertical)
//       bit2 tV : vertical gap extended    (v_ext >= v_open, ties -> extend)
//       bit3 tH : horizontal gap extended  (h_ext >= h_open, ties -> extend)
//   vr          : KEEPV only -- Vs[j][row] of every owned row (the final-column scout needs it for the end-cell
//                 correction flags); the hot path does not keep these registers alive
// Pipe balance of the trace pass (per row, see max2acc): VIMNMX x4, VIADDMNMX, LOP3 and the
// two xor flag ops run on the ALU pipe (8); the three packed adds (VIADD.16x2), the six predicated flag adds and the X
// update run on the FMA-heavy pipe (10); the per-step overhead (selects, scout, index arithmetic) is mostly ALU work, which
// evens the two out over a chunk.  (The gap extension as a plain subtraction instead of the packed add -- both are
// FMA-heavy work -- measured the same.)
#define PB_EXT(x) add2((x), sc.ge2)
//   PROF / subs : the R substitution operands of this column are given (query profile, see profile_word) instead of being
//                 computed from h2 -- two ALU-pipe instructions per row less; only when both halves read the same base
//   FCOL / fc   : the final-column scout of lane_track_general, done row by row as the rows are computed (top to bottom, the
//                 same visiting order) -- no Vs registers kept for it; fc.mask bit h: column j is the final column of half h
template <int R, bool TRACE, bool KEEPV = false, bool PROF = false, bool FCOL = false>
PB_HD void lane_step(Lane<R> &L, uint32_t recvX, uint32_t recvV, uint32_t h2, const Scoring &sc, uint32_t *tw,
                     uint32_t *vr = nullptr, const uint32_t *subs = nullptr, const FinalCol *fc = nullptr) {
    uint32_t diagX = L.prevRecvX, upX = recvX, upV = recvV;
    uint32_t accLo = 0u, accHi = 0u;
#pragma unroll
    for (int r = 0; r < R; ++r) {
        // substitution (minus go) per half: codes equal -> ~(h^v) == -1 -> max(-1 + ma + 1 - go, mi - go) = ma - go
        const uint32_t sub = PROF ? subs[r] : addmax2(xnor2(h2, L.v2[r]), sc.subA2, L.sf2[r]);
        const uint32_t d = PROF ? diagX + sub : add2(diagX, sub);   // S_diag + sub (biased); PROF: carry-compensated word, plain add
#if !defined(__CUDA_ARCH__) && defined(PB_CHECK_RANGES)
        if (PROF && d != add2(diagX, (sub & 0x8000u) ? sub + 0x10000u : sub)) pb_range_violation();   // the plain add IS the packed add
#endif
        uint32_t hs, vs, s;
        if (TRACE) {
            const uint32_t bl = 1u << trace_shift<R>(0, r);
            const uint32_t bh = 1u << trace_shift<R>(1, r);
            const int alu_sites = (r & 1) ? (PB_FLAG_ALU_B) : (PB_FLAG_ALU_A);
            hs = max2acc((alu_sites & 1) != 0, PB_EXT(L.Hs[r]), L.X[r], accLo, bl << 3, accHi, bh << 3);   // ext vs open (= X left)
            vs = max2acc((alu_sites & 2) != 0, PB_EXT(upV), upX, accLo, bl << 2, accHi, bh << 2);          // ext vs open (= X up)
            const uint32_t gmx = max2acc((alu_sites & 4) != 0, vs, hs, accLo, bl << 1, accHi, bh << 1);
            s = max2acc((alu_sites & 8) != 0, d, gmx, accLo, bl, accHi, bh);
        } else {
            hs = addmax2(L.Hs[r], sc.ge2, L.X[r]);
            vs = addmax2(upV, sc.ge2, upX);
            s = max3(d, vs, hs);
        }
        diagX = L.X[r];
        const uint32_t xn = subm2(s, sc.goMag2);                    // X = S + go
        L.X[r] = xn; L.Hs[r] = hs;
        if (KEEPV) vr[r] = vs;
        if (FCOL) final_col_row<R>(L, *fc, r, xn, vs, hs, sc);
        upX = xn; upV = vs;
    }
    if (TRACE) {
        if (TraceWords<R>::value == 1) tw[0] = accLo + accHi; else { tw[0] = accLo; tw[1] = accHi; }
    }
    L.prevRecvX = recvX;
    L.botX = upX; L.botV = upV;
}

// Scout, fast path: inner columns (j < n for both halves).  Only the bottom row of lane G-1 is the last row, but every
// lane may run this on its own bottom row -- scout_combine reads lane G-1 only.  One VIMNMX + a rarely taken branch.
template <int R>
PB_HD void lane_track_lastrow(Lane<R> &L, int j, const Scoring &sc) {
    bool plo, phi;
    const uint32_t nb = max2p(L.lrBest2, L.botX, plo, phi);     // p = (old best >= candidate): strict '>' replaces
    (void)sc;
    if (!(plo && phi)) {
        L.lrBest2 = nb;          // the improved half of nb IS botX's half: only column, Vs and Hs remain to be noted
        if (!plo) { L.lrJ[0] = j; L.lrV2 = (L.lrV2 & 0xFFFF0000u) | (L.botV & 0xFFFFu); L.lrH2 = (L.lrH2 & 0xFFFF0000u) | (L.Hs[R - 1] & 0xFFFFu); }
        if (!phi) { L.lrJ[1] = j; L.lrV2 = (L.lrV2 & 0xFFFFu) | (L.botV & 0xFFFF0000u); L.lrH2 = (L.lrH2 & 0xFFFFu) | (L.Hs[R - 1] & 0xFFFF0000u); }
    }
}

// Scout, general path: handles halves of different lengths and the final column (every real row of the final
// column is a candidate, visited top to bottom; dp_scout.h:168-181).
// FCOL = false: inner columns only (the final column was scanned inside lane_step<.., FCOL>; vr is not used)
template <int R, bool FCOL = true>
PB_HD void lane_track_general(Lane<R> &L, int g, int j, const HalfGeom &A, const HalfGeom &B, const uint32_t *vr,
                              const Scoring &sc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const HalfGeom &H = h ? B : A;
        if (j < H.n) {
            const int c = half16(L.botX, h);
            if (c > half16(L.lrBest2, h)) {
                const uint32_t keep = h ? 0xFFFFu : 0xFFFF0000u;
                L.lrBest2 = (L.lrBest2 & keep) | (L.botX & ~keep);
                L.lrV2 = (L.lrV2 & keep) | (L.botV & ~keep);
                L.lrH2 = (L.lrH2 & keep) | (L.Hs[R - 1] & ~keep);
                L.lrJ[h] = j;
            }
        } else if (FCOL && j == H.n) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int i = g * R + r + 1 - H.pad;
                if (i >= 1) {
                    const int c = half16(L.X[r], h);
                    if (c > L.fcBest[h]) {
                        L.fcBest[h] = c; L.fcI[h] = i;
                        L.fcCorr[h] = corr_flags(c, half16(vr[r], h), half16(L.Hs[r], h), sc.goEff);
                    }
                }
            }
        }
    }
}

// Combine the per-lane scout state of a group into the end cell of half h.  Scores are converted from the biased
// X domain (S + go + bias) back to raw scores here.
struct ScoutCand { int fcBest, fcI, fcCorr, lrBest, lrJ, lrCorr; };
template <int R>
PB_HD ScoutCand make_cand(const Lane<R> &L, int h, const Scoring &sc) {
    ScoutCand c;
    c.fcBest = L.fcBest[h] < 0 ? -0x40000000 : L.fcBest[h] - PB_BIAS - sc.goEff;
    c.fcI = L.fcI[h]; c.fcCorr = L.fcCorr[h];
    c.lrBest = half16(L.lrBest2, h) - PB_BIAS - sc.goEff; c.lrJ = L.lrJ[h];
    c.lrCorr = L.lrJ[h] > 0 ? corr_flags(half16(L.lrBest2, h), half16(L.lrV2, h), half16(L.lrH2, h), sc.goEff) : 0;
    return c;
}
PB_HD EndCell scout_combine(const ScoutCand *c, int G, const HalfGeom &H) {
    EndCell e;
    if (H.n <= 0 || H.m <= 0) { e.j = 0; e.i = 0; e.score = PB_SCORE_EMPTY; e.corr = 0; return e; }
    const ScoutCand &lr = c[G - 1];
    int best = lr.lrBest, bj = lr.lrJ, bi = H.m, corr = lr.lrCorr;
    for (int g = 0; g < G; ++g) {
        if (c[g].fcBest > best) { best = c[g].fcBest; bj = H.n; bi = c[g].fcI; corr = c[g].fcCorr; }
    }
    e.j = bj; e.i = bi; e.score = best; e.corr = corr;
    return e;
}

// ---- traceback + statistics ---------------------------------------------------------------------------
// Cursor: walks the trace.  cur.flags() = 4 trace flags of the current cell, cur.move(consR, consA) steps to the cell one
// column left (consR) and / or one row up (consA), cur.eq() = read base of the current column equals the adapter base of the
// current row (code equality, N == N).  The kernels keep incremental addresses in the cursor (trace_kernel) or index a plain
// array (generic_kernel, tests); RandomCursor adapts a pair of (column, row) functions.
template <class NibFn, class EqFn>
struct RandomCursor {
    NibFn nib; EqFn eqf; int j, i;
    PB_HD RandomCursor(NibFn n, EqFn e, int j0, int i0) : nib(n), eqf(e), j(j0), i(i0) {}
    PB_HD uint32_t flags() { return nib(j, i); }
    PB_HD bool eq() { return eqf(j, i); }
    PB_HD void move(bool consR, bool consA) { j -= consR ? 1 : 0; i -= consA ? 1 : 0; }
};

// Writes the 9-int record.  Returns 0, or 1 if the path ran into the left edge of a window with
// col0 > 0 (window too small -- must never happen when the window bound of DESIGN.md holds).
// `cur` must be positioned on the end cell (end.j, end.i) when both are > 0.
// FROM_SCORE (needs sc->ma != sc->mi): the matches are not compared base by base (cur.eq() is never called) but follow from
// the score.  The path follows the argmax decisions of the DP that found end.score, and the end-cell correction only picks a
// state of the same value, so the path scores exactly S* = ma*M + mi*(D - M) + (gap costs), D = diagonal steps, M = matches;
// a gap run of k steps costs go + (k-1)*ge (linear: k*ge), and a run starts (walking backwards: ends) at the step whose
// cell does not say "extended".  tests/test_trace_cursor.py checks the identity against the oracle.
template <bool FROM_SCORE = false, class Cursor>
PB_HD int traceback_stats_cur(Cursor &cur, const EndCell &end, bool linear, int col0, int n_total, int m, int32_t *rec,
                              const Scoring *sc = nullptr) {
    if (end.score == PB_SCORE_EMPTY) {
        rec[0] = -1; rec[1] = 0; rec[2] = -1; rec[3] = 0; rec[4] = PB_SCORE_EMPTY;
        rec[5] = 0; rec[6] = 0; rec[7] = 0; rec[8] = 0;
        return 0;
    }
    int j = end.j, i = end.i;      // local column, row
    int L = 0, matches = 0, opens = 0;
    // The statistics need the first / last (in forward order) path operation that consumes a read base and the first / last
    // that consumes an adapter base.  Walking backwards these are the last / first step that consumes one, and what is needed
    // of each is its step index k and the row (column) the path is on after it.  The "first" events are noted in every step
    // that starts on the end cell's column (row) -- the last such note is the step that leaves it -- and the "last" events in
    // every step that consumes a base.  No per-step event records, no run-length bookkeeping.
    int kR1 = 0, iR1 = 0, kA1 = 0, jA1 = 0;      // first step (backwards) that consumes a read / an adapter base
    int kR2 = 0, iR2 = 0, kA2 = 0, jA2 = 0;      // last step that does
    // direction of the current cell as the bases its step consumes: diagonal both, vertical the adapter's, horizontal the read's
    // (ints, not bools: loop-carried bools cost byte moves on the device)
    int consR = 1, consA = 1;
    uint32_t b = 0;
    bool ext = false;
    if (j > 0 && i > 0) {
        b = cur.flags();
        consR = (b & 3u) != 2u; consA = (b & 3u) != 0u;  // tD -> diagonal, else tM -> vertical, else horizontal
        if (!linear) {                                  // dp_algorithm_impl.h:1354-1369
            if (end.corr & 1) { consR = 0; consA = 1; } else if (end.corr & 2) { consR = 1; consA = 0; }
        }
    }
    // ONE path step per loop iteration with the step kind as data (no per-direction code paths, no inner gap-run loops):
    // the lanes of a warp that trace at the same time run the same instruction stream instead of serialising diagonal /
    // vertical / horizontal branches and waiting for each other's gap runs.
    while (j > 0 && i > 0) {
        const bool isD = (consR & consA) != 0;
        if (!FROM_SCORE && isD && cur.eq()) ++matches;
        // a gap run continues while the current cell says "extended" (dp_traceback_impl.h:225-341).  A vertical step from row
        // 1 or a horizontal one from column 1 ends the path, so what its flag says only matters to the count of runs, which
        // the test after the loop corrects.
        ext = (b & (linear ? 0u : (!consR ? 4u : (!consA ? 8u : 0u)))) != 0u;
        if (FROM_SCORE && !isD && !ext) ++opens;
        const bool onR = j == end.j, onA = i == end.i;
        if (consR) --j;
        if (consA) --i;
        if (onR) { kR1 = L; iR1 = i; }
        if (onA) { kA1 = L; jA1 = j; }
        if (consR) { kR2 = L; iR2 = i; }
        if (consA) { kA2 = L; jA2 = j; }
        ++L;
        cur.move(consR != 0, consA != 0);
        if (j > 0 && i > 0) {
            b = cur.flags();
            if (!ext) { consR = (b & 3u) != 2u; consA = (b & 3u) != 0u; }
        }
    }
    if (FROM_SCORE) {
        if (ext) ++opens;          // the last step (into row 0 or column 0) opened its run
        const int diag = (end.i - i) + (end.j - j) - L, gaps = L - diag;
        const int gapcost = linear ? sc->ge * gaps : sc->go * opens + sc->ge * (gaps - opens);
        matches = (end.score - sc->mi * diag - gapcost) / (sc->ma - sc->mi);
    }
    const bool haveR = j < end.j, haveA = i < end.i;
    int status = (j == 0 && i > 0 && col0 > 0) ? 1 : 0;

    // whole alignment = [H x a][V x bb] . path . [H x c][V x e]   (dp_traceback_impl.h:532-554)
    const int a = col0 + j, bb = i;
    const int jend = col0 + end.j;
    const int c = n_total - jend, e = m - end.i;
    const int Ltot = a + bb + L + c + e;
#define PB_COL(k) (a + bb + (L - 1 - (k)))
    // first column with a read base (r0) / adapter base (a0) and the bases of the OTHER sequence before it
    int r0, AB_r0, a0, RB_a0;
    if (a > 0) { r0 = 0; AB_r0 = 0; }
    else if (haveR) { r0 = PB_COL(kR2); AB_r0 = iR2; }
    else { r0 = bb + L; AB_r0 = end.i; }
    if (bb > 0) { a0 = 0; RB_a0 = 0; }
    else if (haveA) { a0 = PB_COL(kA2); RB_a0 = col0 + jA2; }
    else { a0 = a + L + c; RB_a0 = n_total; }
    int rs, as;
    int start;
    if (r0 >= a0) { start = r0; rs = 0; as = AB_r0; } else { start = a0; as = 0; rs = RB_a0; }
    // last column with a read base (r1) / adapter base (a1)
    int r1, AB_r1, a1, RB_a1;
    if (c > 0) { r1 = Ltot - 1; AB_r1 = m; }
    else if (haveR) { r1 = PB_COL(kR1); AB_r1 = iR1; }
    else { r1 = a - 1; AB_r1 = 0; }
    if (e > 0) { a1 = Ltot - 1; RB_a1 = n_total; }
    else if (haveA) { a1 = PB_COL(kA1); RB_a1 = col0 + jA1; }
    else { a1 = a + bb - 1; RB_a1 = 0; }
#undef PB_COL
    int re, ae, endc;
    if (r1 <= a1) { endc = r1; re = n_total - 1; ae = AB_r1; } else { endc = a1; ae = m - 1; re = RB_a1; }
    rec[0] = rs; rec[1] = re; rec[2] = as; rec[3] = ae; rec[4] = end.score;
    rec[5] = matches; rec[6] = endc - start + 1; rec[7] = matches; rec[8] = a1 - a0 + 1;
    return status;
}

// NibFn(jl, i) -> 4 trace flags of cell (local column jl >= 1, row i >= 1); EqFn(jl, i) -> bases equal
template <class NibFn, class EqFn>
PB_HD int traceback_stats(NibFn nib, EqFn eq, const EndCell &end, bool linear, int col0, int n_total, int m,
                          int32_t *rec) {
    RandomCursor<NibFn, EqFn> cur(nib, eq, end.j, end.i);
    return traceback_stats_cur(cur, end, linear, col0, n_total, m, rec);
}

// ---- end-trim decisions on the device (SURVEY 8(f) row 3) ------------------------------------------------------
// find_start_trim / find_end_trim (porechop/nanopore_read.py:166-208) for one record: the trim amount this adapter asks
// for, or 0.  The reference compares  float("%f" % (100.0*match_aln/len_aln)) > end_threshold ; printf's rounding and
// strtod are monotone, so for every len_aln there is a smallest match count that passes: cmin[len_aln], built on the
// host with the very same snprintf/strtod chain (engine.cu pb200TrimThresholdTable).  A failed alignment (empty read or
// adapter) parses as 0.0 / read_start -1 / read_end 0 in the reference (nanopore_read.py:479-485).
PB_HD int32_t end_trim_candidate(const int32_t *r, int is_start, int32_t end_size, int32_t extra_trim, int32_t min_trim,
                                 const int32_t *cmin, int32_t cmin_len, int *overflow) {
    const bool failed = r[0] == -1 && r[4] == PB_SCORE_EMPTY;
    if (failed) return 0;                                   // 0.0 > threshold only for negative thresholds: see host check
    const int32_t l = r[6], c = r[5];
    if (l < 0 || l >= cmin_len) { *overflow = 1; return 0; }
    if (c < cmin[l]) return 0;                              // partial identity does not pass (also 0/0 = NaN: cmin[0] is huge)
    const int32_t rs = r[0], re = r[1] + 1;
    if (re - rs < min_trim) return 0;
    if (is_start) return (re == end_size) ? 0 : re + extra_trim;
    return (rs == 0) ? 0 : (end_size - rs) + extra_trim;
}
// ---- middle-adapter hits on the device ----------------------------------------------------------------------------
// find_middle_adapters (porechop/nanopore_read.py:216-243) for one record: float("%f" % (100.0*match_ad/len_ad)) >=
// middle_threshold, with cmin[len_ad] the smallest passing match count (engine.cu pb200MiddleThresholdTable).  A failed
// alignment has len_ad = 0 and never hits (cmin[0] is huge, and the threshold is > 0).  The table covers the window bound
// W(m_max) + 2; a length outside it sets *overflow.
PB_HD bool middle_hit(const int32_t *r, const int32_t *cmin, int32_t cmin_len, int *overflow) {
    const int32_t l = r[8], c = r[7];
    if (l < 0 || l >= cmin_len) { *overflow = 1; return false; }
    return l > 0 && c >= cmin[l];
}
// barcode score column of a record: (match_ad, len_ad) as two uint16 -- the host turns the pair into the exact double
// the reference parses (full-adapter identity); a failed alignment scores 0.0 = the pair (0, 1).
PB_HD uint32_t score_pair(const int32_t *r, int *overflow) {
    if (r[0] == -1 && r[4] == PB_SCORE_EMPTY) return 1u << 16;
    if ((uint32_t)r[7] > 0xFFFFu || (uint32_t)r[8] > 0xFFFFu) { *overflow = 1; return 0u; }
    return (uint32_t)r[7] | ((uint32_t)r[8] << 16);
}

}  // namespace pb
