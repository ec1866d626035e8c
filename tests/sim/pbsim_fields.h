// tests/sim/pbsim_fields.h -- the pointers inside the kernels' by-value argument structs, as accesses of the stream-ordering
// check (pbsim_cuda.h).  TESTS ONLY: build_sim.py includes it after kernels.cuh.  Found by argument-dependent lookup from
// pbsim::classify_arg; a struct without an overload here carries no pointers the check needs.
#pragma once

namespace pb {

// every pointer of a task source is read: explicit tasks, the class's adapter ids, offsets, the sequence order
inline void pbsim_fields(const TaskSrc &t, const std::string &w) {
    if (t.tasks) pbsim::hb_access(t.tasks, 0, pbsim::ACC_READ, w + ".tasks");
    if (t.cls_ad) pbsim::hb_access(t.cls_ad, 0, pbsim::ACC_READ, w + ".cls_ad");
    if (t.seq_off) pbsim::hb_access(t.seq_off, 0, pbsim::ACC_READ, w + ".seq_off");
    if (t.ad_off) pbsim::hb_access(t.ad_off, 0, pbsim::ACC_READ, w + ".ad_off");
    if (t.seq_order) pbsim::hb_access(t.seq_order, 0, pbsim::ACC_READ, w + ".seq_order");
}

// decide_kernel reads the records, the threshold table and the score columns, and writes trim / pairs / top2
inline void pbsim_fields(const DecideArgs &a, const std::string &w) {
    if (a.records) pbsim::hb_access(a.records, 0, pbsim::ACC_READ, w + ".records");
    if (a.cmin) pbsim::hb_access(a.cmin, 0, pbsim::ACC_READ, w + ".cmin");
    if (a.cols) pbsim::hb_access(a.cols, 0, pbsim::ACC_READ, w + ".cols");
    if (a.trim) pbsim::hb_access(a.trim, 0, pbsim::ACC_WRITE, w + ".trim");
    if (a.pairs) pbsim::hb_access(a.pairs, 0, pbsim::ACC_WRITE, w + ".pairs");
    if (a.top2) pbsim::hb_access(a.top2, 0, pbsim::ACC_WRITE, w + ".top2");
}

// middle_decide_kernel gets the whole segment's buffers.  Round 0 (active == nullptr) touches only the rows of reads
// [first, first + n): records and offsets read, next adapter and codes (the masking) written -- chunks of one host call run
// it on different streams at once, on disjoint rows.  A later round's reads come from the active list: the whole buffer
// from the pointer on.  The hit slots and the active list are claimed with atomicAdd on `count`: atomic accesses.
// (The offsets' end entry [first + n] is also the next chunk's first entry, which both chunks write with the same value.)
inline void pbsim_fields(const MiddleArgs &a, const std::string &w) {
    const bool round0 = a.active == nullptr;
    const size_t rec_row = (size_t)a.n_adapters * PB_REC * 4, all = (size_t)-1;
    if (a.records) {
        if (round0) pbsim::hb_access(a.records + (size_t)a.first * a.n_adapters * PB_REC, (size_t)a.n * rec_row, pbsim::ACC_READ, w + ".records");
        else pbsim::hb_access(a.records, all, pbsim::ACC_READ, w + ".records");
    }
    if (a.active) pbsim::hb_access(a.active, 0, pbsim::ACC_READ, w + ".active");
    if (a.next_ad) {
        if (round0) pbsim::hb_access(a.next_ad + a.first, (size_t)a.n * 4, pbsim::ACC_WRITE, w + ".next_ad");
        else pbsim::hb_access(a.next_ad, all, pbsim::ACC_WRITE, w + ".next_ad");
    }
    if (a.seq_off) {
        if (round0) pbsim::hb_access(a.seq_off + a.first, (size_t)a.n * 8, pbsim::ACC_READ, w + ".seq_off");
        else pbsim::hb_access(a.seq_off, all, pbsim::ACC_READ, w + ".seq_off");
    }
    if (a.codes) {
        if (round0 && a.seq_off && a.n > 0) {
            const int64_t b = a.seq_off[a.first], e = a.seq_off[a.first + a.n];
            if (e > b) pbsim::hb_access(a.codes + b, (size_t)(e - b), pbsim::ACC_WRITE, w + ".codes");
        } else if (!round0) {
            pbsim::hb_access(a.codes, all, pbsim::ACC_WRITE, w + ".codes");
        }
    }
    if (a.cmin) pbsim::hb_access(a.cmin, 0, pbsim::ACC_READ, w + ".cmin");
    if (a.hits) pbsim::hb_access(a.hits, 0, pbsim::ACC_ATOMIC, w + ".hits");
    if (a.next_active) pbsim::hb_access(a.next_active, 0, pbsim::ACC_ATOMIC, w + ".next_active");
    if (a.count) pbsim::hb_access(a.count, 0, pbsim::ACC_ATOMIC, w + ".count");
    if (a.max_len) pbsim::hb_access(a.max_len, 0, pbsim::ACC_ATOMIC, w + ".max_len");
}

}  // namespace pb
